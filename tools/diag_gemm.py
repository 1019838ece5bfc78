"""GPU diagnostic (not a test): accuracy and speed of the GEMM engines."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from anyloc_b200 import _lib as L
L.load()

def split(x):
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    L.check(L.load().anyloc_split_tf32(L.ptr(x), L.ptr(hi), L.ptr(lo), x.numel(), L.stream_ptr()), "split")
    return hi, lo

def gemm(a_hi, a_lo, b_hi, b_lo, engine, out=None):
    M, K = a_hi.shape; N = b_hi.shape[0]
    if out is None: out = torch.empty(M, N, device="cuda")
    rc = L.load().anyloc_gemm_nt(L.ptr(a_hi), L.ptr(a_lo), K, L.ptr(b_hi), L.ptr(b_lo), K, M, N, K, L.PAIR["tf32"],
                                 1.0, L.EPI["bias"], None, None, None, L.ptr(out), None, N, L.PAIR["tf32"],
                                 L.ENGINE[engine], L.stream_ptr())
    L.check(rc, "gemm")
    return out

print("== accuracy: err = max|out-ref|/max|ref| ; bias = mean((out-ref)*sign(ref))/mean|ref|")
for K in (64, 384, 1536, 4096, 16384):
    g = torch.Generator(device="cuda").manual_seed(K)
    a = torch.randn(512, K, device="cuda", generator=g); b = torch.randn(512, K, device="cuda", generator=g) * 0.05
    ref = a.double() @ b.double().T
    ah, al = split(a); bh, bl = split(b)
    rows = []
    for name, out in (("simt", gemm(ah, al, bh, bl, "simt")), ("tc3", gemm(ah, al, bh, bl, "tc3")),
                      ("tc1(hi only)", gemm(ah, None, bh, None, "tc3")),
                      ("torch fp32", (a @ b.T))):
        d = out.double() - ref
        rows.append(f"{name}: err {float(d.abs().max()/ref.abs().max()):.2e} bias {float((d*ref.sign()).mean()/ref.abs().mean()):+.2e}")
    print(f"K={K}: " + " | ".join(rows))

print("== speed (CUDA events, 5 reps after 2 warmups)")
for (M, N, K) in [(16960, 4608, 1536), (16960, 1536, 1536), (16960, 8192, 1536), (16960, 1536, 4096), (1000, 10000, 49152)]:
    a = torch.randn(M, K, device="cuda"); b = torch.randn(N, K, device="cuda") * 0.05
    ah, al = split(a); bh, bl = split(b)
    out = torch.empty(M, N, device="cuda")
    for eng in ("tc3", "simt"):
        if eng == "simt" and M * N * K > 2e11: continue
        for _ in range(2): gemm(ah, al, bh, bl, eng, out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(5): gemm(ah, al, bh, bl, eng, out)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        print(f"{eng} M={M} N={N} K={K}: {ms:.3f} ms  {2*M*N*K/ms/1e9:.1f} TFLOP/s fp32-equivalent ({3*2*M*N*K/ms/1e9:.0f} TF/s tf32 issued)" if eng == "tc3" else
              f"{eng} M={M} N={N} K={K}: {ms:.3f} ms  {2*M*N*K/ms/1e9:.1f} TFLOP/s")
    torch.backends.cuda.matmul.allow_tf32 = False
    for _ in range(2): torch.matmul(a, b.T, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(5): torch.matmul(a, b.T, out=out)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    print(f"cublas-fp32 M={M} N={N} K={K}: {ms:.3f} ms  {2*M*N*K/ms/1e9:.1f} TFLOP/s")
