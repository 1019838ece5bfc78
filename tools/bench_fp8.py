"""Throughput and error of the single-e4m3 precision against single bf16, alternating in one process.

bf16 runs one bf16 MMA per product; fp8 runs the block GEMMs as one e4m3 MMA per product (twice the data-sheet rate)
on e4m3 weights and per-row-scaled e4m3 activations, with extra quantiser passes over the attention output and the FFN
hidden layer, and keeps the bf16 patch embedding and attention.  Configurations
(random-init weights, vit.random_state_dict; auto engine), the ViT part of bench.py's pipeline workloads:
  c2   ViT-G/14 layer 31 value, 322x322, B = 32
  c5   ViT-L/14 layer 20 value, 518x518, B = 64
  c1   ViT-S/14 layer 9 value, 224x224, B = 16
Every shape is warmed up, then the arms alternate inside each of --rounds rounds (host clock around a device
synchronise); the median gives img/s.  One profiled call per arm splits the device time into GEMM / attention /
LayerNorm / other, and the ViT's algorithmic FLOPs (bench.vit_flops_per_image) over the median time give TFLOP/s and
its share of the 989 TFLOP/s dense BF16 data-sheet peak of the H100 SXM (the FP8 peak is 1,979).  The feature error of each arm,
max|f - f32| / max|f32|, is measured at full size on 2 images against the restated model in fp32 on the GPU (TF32
off).  Prints the card, its power limit and clocks, then one JSON line per configuration; writes nothing unless --out
is given.

    python tools/bench_fp8.py [--rounds 7] [--configs c2,c5,c1] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {
    "c2": ("dinov2_vitg14", 31, 322, 32),
    "c5": ("dinov2_vitl14", 20, 518, 64),
    "c1": ("dinov2_vits14", 9, 224, 16),
}
ARMS = {"bf16": "bf16", "fp8": "fp8"}
PEAK_TFLOPS = 989.0


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else
            f"unavailable ({r.stderr.strip()})"}


def feature_error(name, layer, sd, models, side, dev):
    """max|f - f32| / max|f32| of each arm on 2 images against the restated model in fp32 on the GPU"""
    import torch
    from oracle import anyloc_oracle as ao
    from oracle import dinov2_restated as dr
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    model = dr.build(name, depth_override=layer + 1)
    model.load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=False)
    model = model.to(dev)
    img = torch.randn(2, 3, side, side, generator=torch.Generator().manual_seed(99)).to(dev)
    ref = ao.extract_features(model, img, layer, "value").double()
    err = {arm: float((m.extract(img, layer, "value").double() - ref).abs().max() / ref.abs().max())
           for arm, m in models.items()}
    del model
    return err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 times the GPU path and needs a CUDA device")
    from anyloc_b200 import _lib
    from anyloc_b200.vit import VitWeights, random_state_dict
    from bench import vit_flops_per_image
    dev = torch.device("cuda", 0)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []
    for key in args.configs.split(","):
        name, layer, side, B = CONFIGS[key]
        sd = random_state_dict(name, seed=0, device=dev, depth=layer + 1)
        models = {arm: VitWeights(name, sd, dev, pair=pair) for arm, pair in ARMS.items()}
        err = feature_error(name, layer, sd, models, side, dev)
        del sd
        torch.cuda.empty_cache()
        img = torch.randn(B, 3, side, side, generator=torch.Generator().manual_seed(1234)).to(dev)
        fns = {arm: (lambda m=m: m.extract(img, layer, "value")) for arm, m in models.items()}
        prof = {}
        for arm, fn in fns.items():
            fn()                                  # warm-up
            torch.cuda.synchronize()
            _lib.profile_enable(True)
            fn()
            p = _lib.profile_read()
            _lib.profile_enable(False)
            prof[arm] = {c: round(p[c][0], 2) for c in ("gemm_tc", "gemm_simt", "attention", "layernorm", "vit_misc")}
        torch.cuda.synchronize()
        times = {a: [] for a in fns}
        for r in range(args.rounds):
            order = list(fns) if r % 2 == 0 else list(fns)[::-1]
            for arm in order:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = fns[arm]()
                torch.cuda.synchronize()
                times[arm].append(time.perf_counter() - t0)
                del res
        med = {a: sorted(t)[len(t) // 2] for a, t in times.items()}
        flops = vit_flops_per_image(name, layer, side, side) * B
        line = {"config": key, "model": name, "layer": layer, "size": side, "batch": B,
                "ms": {a: round(1e3 * t, 2) for a, t in med.items()},
                "img_per_s": {a: round(B / t, 1) for a, t in med.items()},
                "speedup_fp8": round(med["bf16"] / med["fp8"], 3),
                "spread_ms": {a: [round(1e3 * min(t), 2), round(1e3 * max(t), 2)] for a, t in times.items()},
                "vit_tflops": {a: round(flops / t / 1e12, 1) for a, t in med.items()},
                "share_of_989": {a: round(flops / t / 1e12 / PEAK_TFLOPS, 3) for a, t in med.items()},
                "profiled_ms": prof, "feature_rel_err_vs_fp32": err, **info}
        results.append(line)
        print(json.dumps(line), flush=True)
        del models, fns, img
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
