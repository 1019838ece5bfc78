"""Device time of the tensor-core attention kernel alone at the flagship shapes, in both 2-byte formats.

Shapes (images B, tokens T, heads; head_dim 64), the attention of bench.py's ViT workloads:
  c2   ViT-G/14 at 322x322: B = 32, T = 530, 24 heads
  c5   ViT-L/14 at 518x518: B = 64, T = 1370, 16 heads
  c1   ViT-S/14 at 224x224: B = 16, T = 257, 6 heads
Formats: f16x3 (fp16 pairs of 8x, three MMAs per product) and bf16 (one bf16 array, one MMA per product).  The call is
anyloc_attention on seeded random inputs; the fp16-pair route converts its fp32 input first, so the time reported is
the attention kernel's own, read from torch.profiler's per-kernel device-time totals (the kernel whose name contains
"attention"), averaged over --iters launches after --warmup.  Prints the card, its power limit and clocks, then one JSON line per (shape,
format): ms per call, algorithmic TFLOP/s (4 B T^2 D) and issued TFLOP/s (x3 for the fp16 pairs).  Writes nothing
unless --out is given.

    python tools/bench_attention.py [--iters 50] [--shapes c2,c5,c1] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"c2": (32, 530, 24), "c5": (64, 1370, 16), "c1": (16, 257, 6)}
FORMATS = {"f16x3": 3, "bf16": 1}          # MMAs issued per product


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


def make_call(L, fmt, B, T, heads):
    import torch
    D = heads * 64
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T)
    x = torch.randn(B * T, 3 * D, device="cuda", generator=g)
    lib = L.load()
    if fmt == "bf16":
        q = x.to(torch.bfloat16)
        o = torch.empty(B * T, D, device="cuda", dtype=torch.bfloat16)
        return lambda: L.check(lib.anyloc_attention(L.ptr(q), None, B, T, D, heads, L.ptr(o), None, L.PAIR["bf16"],
                                                    L.ENGINE["tc3"], L.stream_ptr()), "attention")
    lo = torch.zeros_like(x)
    hi, olo = torch.empty(B * T, D, device="cuda", dtype=torch.float16), torch.empty(B * T, D, device="cuda",
                                                                                      dtype=torch.float16)
    return lambda: L.check(lib.anyloc_attention(L.ptr(x), L.ptr(lo), B, T, D, heads, L.ptr(hi), L.ptr(olo),
                                                L.PAIR["f16"], L.ENGINE["tc3"], L.stream_ptr()), "attention")


def kernel_ms(call, iters, warmup):
    """mean device time of the attention kernel per call, from the profiler's per-kernel totals"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    hits = [e for e in prof.key_averages() if "attention" in e.key and "qkv_to_f16" not in e.key and
            "anyloc" in e.key and e.self_device_time_total > 0]
    if len(hits) != 1 or hits[0].count != iters:
        raise RuntimeError("expected %d launches of one attention kernel, found %s" %
                           (iters, [(e.key, e.count) for e in hits]))
    return hits[0].self_device_time_total / iters / 1e3, hits[0].key


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="c2,c5,c1")
    ap.add_argument("--formats", default="f16x3,bf16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention: no CUDA device")
    from anyloc_b200 import _lib as L
    print("card:", card_info(), flush=True)
    rows = []
    for name in a.shapes.split(","):
        B, T, heads = SHAPES[name]
        flop = 4.0 * B * T * T * heads * 64
        for fmt in a.formats.split(","):
            ms, kernel = kernel_ms(make_call(L, fmt, B, T, heads), a.iters, a.warmup)
            row = {"shape": name, "B": B, "T": T, "heads": heads, "format": fmt, "ms": round(ms, 4),
                   "tflops_alg": round(flop / ms / 1e9, 1), "tflops_issued": round(FORMATS[fmt] * flop / ms / 1e9, 1),
                   "kernel": kernel[:60]}
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card_info(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
