"""GPU diagnostic (not a test): accuracy and speed of the GEMM engines.

    python tools/diag_gemm.py [--speed-only] [--reps N]

The speed section times the tensor-core engine at the shapes the flagship workloads run: the four GEMMs of a ViT-G/14
block at bench c2 (M = 32 x 530 tokens, fp16 pairs, each with the epilogue, bias, LayerScale gamma, aliased residual
and leading dimension `vit_block` (csrc/api.cu) gives it), the VLAD coarse pass at c2 (hi-only tf32) and the c3
retrieval coarse pass (hi-only fp16).  Each shape is also timed with its epilogue discarded
(ANYLOC_GEMM_DEBUG_SKIP_EPI, in a subprocess: the library reads it once per process) to expose the epilogue's share.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from anyloc_b200 import _lib as L
from tests.util import gemm_nt, split_f16
L.load()

# name: (M, N, K, pair, lom, epilogue, ldo, n_out)  -- lom: lo operands present (3 = both, 0 = hi-only)
M_C2, D, HF = 32 * 530, 1536, 4096
SPEED_SHAPES = {
    "c2 qkv": (M_C2, 3 * D, D, "f16", 3, "bias_split", 3 * D, 3 * D),
    "c2 proj": (M_C2, D, D, "f16", 3, "ls_resid", D, D),
    "c2 w12": (M_C2, 2 * HF, D, "f16", 3, "swiglu_split", HF, HF),
    "c2 w3": (M_C2, D, HF, "f16", 3, "ls_resid", D, D),
    "c2 vlad coarse": (M_C2, 32, D, "tf32", 0, "bias", 32, 32),
    "c3 coarse": (1000, 10000, 49152, "f16", 0, "bias", 10000, 10000),
}


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


def accuracy():
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


def shape_call(name):
    """buffers of one speed shape -> a function that issues the GEMM once"""
    M, N, K, pair, lom, epi, ldo, n_out = SPEED_SHAPES[name]
    g = torch.Generator(device="cuda").manual_seed(7)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g) * 0.02
    if pair == "f16":
        s_b = 2.0 ** int(torch.floor(torch.log2(16384.0 / b.abs().max())).item())
        (a_hi, a_lo), (b_hi, b_lo) = split_f16(L, a, L.ACT_SCALE), split_f16(L, b, s_b)
        alpha = 1.0 / (L.ACT_SCALE * s_b)
    else:
        (a_hi, a_lo), (b_hi, b_lo), alpha = (a, None), (b, None), 1.0
    if not lom & 1: a_lo = None
    if not lom & 2: b_lo = None
    del a, b
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.randn(N, device="cuda", generator=g) * 1e-2 if epi == "ls_resid" else None
    odt = torch.float16 if ("split" in epi and pair == "f16") else torch.float32
    out = torch.randn(M, ldo, device="cuda", generator=g).to(odt)
    out_lo = torch.empty(M, ldo, device="cuda", dtype=odt) if "split" in epi else None
    resid = out if epi == "ls_resid" else None             # in place, as the ViT's residual stream

    def call():
        L.check(gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, pair=pair, alpha=alpha, epi=epi, bias=bias, gamma=gamma,
                        resid=resid, out=out, out_lo=out_lo, ldo=ldo, engine="tc3"), name)
    return call


def sm_clock():
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return r.stdout.strip() or "?"


def time_shapes(reps):
    """{name: (ms per launch, SM clock MHz sampled while the timed launches run)}"""
    res = {}
    for name in SPEED_SHAPES:
        call = shape_call(name)
        for _ in range(3): call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): call()
        e1.record()
        clk = sm_clock()                                   # sampled while the queued launches run
        torch.cuda.synchronize()
        res[name] = (e0.elapsed_time(e1) / reps, clk)
        del call
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--speed-only", action="store_true")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", action="store_true", help="print the speed table as one JSON line (used for the "
                    "epilogue-discarding subprocess)")
    args = ap.parse_args()
    if args.json:
        print(json.dumps(time_shapes(args.reps)))
        return
    if not args.speed_only:
        accuracy()
    name = torch.cuda.get_device_name()
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"== speed: {name}, power limit / max SM clock {q.stdout.strip()}; CUDA events, {args.reps} launches after "
          "3 warm-ups; TFLOP/s algorithmic (2MNK) and issued (x MMAs per product)")
    full = time_shapes(args.reps)
    env = dict(os.environ, ANYLOC_GEMM_DEBUG_SKIP_EPI=str(0b11111))    # every epilogue mode discards its result
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--json", "--reps", str(args.reps)], env=env,
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stderr)
        raise SystemExit("epilogue-discarding run failed")
    bare = json.loads(r.stdout.strip().splitlines()[-1])
    sms = C.c_int(0)
    L.load().anyloc_device_info(C.byref(sms), None)
    print(f"{'shape':16s} {'M x N x K':>20s} {'ms':>8s} {'TF/s alg':>9s} {'TF/s iss':>9s} {'no-epi ms':>9s} "
          f"{'epi %':>6s} {'SM MHz':>7s}  grid")
    for nm, (M, N, K, pair, lom, epi, ldo, n_out) in SPEED_SHAPES.items():
        ms, clk = full[nm]
        ms0 = bare[nm][0]
        mmas = 1 + (lom & 1) + ((lom >> 1) & 1)
        tf = 2.0 * M * N * K / ms / 1e9
        grid = f"{min(-(-M // 128) * -(-N // 128), sms.value)} CTAs on {sms.value} SMs"     # persistent grid
        print(f"{nm:16s} {f'{M}x{N}x{K}':>20s} {ms:8.3f} {tf:9.1f} {tf * mmas:9.1f} {ms0:9.3f} "
              f"{100 * (ms - ms0) / ms:6.1f} {clk:>7s}  {grid}")


if __name__ == "__main__":
    main()
