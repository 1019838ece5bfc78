"""Throughput and error of the bf16-pair precision (bf16pair) against the fp16 pairs (f16x3) and the tf32 pairs (tf32x3),
alternating in one process.

bf16pair and f16x3 both run three 2-byte MMAs per product on operands of the same bytes; tf32x3 runs three tf32 MMAs on
4-byte words.  Configurations (random-init weights, vit.random_state_dict; auto engine), the ViT part of bench.py's
pipeline workloads:
  c2   ViT-G/14 layer 31 value, 322x322, B = 32
  c5   ViT-L/14 layer 20 value, 518x518, B = 64
  c1   ViT-S/14 layer 9 value, 224x224, B = 16
Every shape is warmed up, then the three arms alternate inside each of --rounds rounds, in an order that rotates from
round to round (host clock around a device synchronise); the median gives img/s.  One profiled call per arm splits the
device time into GEMM / attention / LayerNorm / other.  For c2 the feature error of each arm, max|f - f64| / max|f64|
and |f - f64|_F / |f64|_F, is measured on 2 images against the restated model in fp64 on the GPU.  All of it uses
random-init weights, not a trained checkpoint.  Prints the card, its power limit and clocks, then one JSON line per
configuration; writes nothing unless --out is given.

    python tools/bench_bf16x3.py [--rounds 7] [--configs c2,c5,c1] [--out results.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_bf16 import CONFIGS, card_info      # noqa: E402

ARMS = {"f16x3": "f16", "bf16pair": "bf16pair", "tf32x3": "tf32"}


def errors(name, layer, sd, models, side, dev):
    """(max-element, RMS) error of each arm against the restated model in fp64 on 2 images"""
    import torch
    from oracle import anyloc_oracle as ao
    from oracle import dinov2_restated as dr
    model = dr.build(name, depth_override=layer + 1)
    model.load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=False)
    model = model.double().to(dev)
    img = torch.randn(2, 3, side, side, generator=torch.Generator().manual_seed(99)).to(dev)
    with torch.no_grad():
        ref = ao.extract_features(model, img.double(), layer, "value")
    del model
    torch.cuda.empty_cache()
    err = {}
    for arm, m in models.items():
        f = m.extract(img, layer, "value").double()
        err[arm] = [float((f - ref).abs().max() / ref.abs().max()), float((f - ref).norm() / ref.norm())]
    return err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_bf16x3 times the GPU path and needs a CUDA device")
    from anyloc_b200 import _lib
    from anyloc_b200.vit import VitWeights, random_state_dict
    dev = torch.device("cuda", 0)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []
    for key in args.configs.split(","):
        name, layer, side, B = CONFIGS[key]
        sd = random_state_dict(name, seed=0, device=dev, depth=layer + 1)
        models = {arm: VitWeights(name, sd, dev, pair=pair) for arm, pair in ARMS.items()}
        err = errors(name, layer, sd, models, side, dev) if key == "c2" else None
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
        arms = list(fns)
        for r in range(args.rounds):
            order = arms[r % len(arms):] + arms[:r % len(arms)]
            for arm in order:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = fns[arm]()
                torch.cuda.synchronize()
                times[arm].append(time.perf_counter() - t0)
                del res
        med = {a: sorted(t)[len(t) // 2] for a, t in times.items()}
        line = {"config": key, "model": name, "layer": layer, "size": side, "batch": B, "weights": "random-init",
                "ms": {a: round(1e3 * t, 2) for a, t in med.items()},
                "img_per_s": {a: round(B / t, 1) for a, t in med.items()},
                "bf16pair_over_f16x3_time": round(med["bf16pair"] / med["f16x3"], 3),
                "bf16pair_over_tf32x3_time": round(med["bf16pair"] / med["tf32x3"], 3),
                "spread_ms": {a: [round(1e3 * min(t), 2), round(1e3 * max(t), 2)] for a, t in times.items()},
                "profiled_ms": prof, **info}
        if err is not None:
            line["feature_err_vs_fp64_max_rms"] = err
        results.append(line)
        print(json.dumps(line), flush=True)
        del models, fns, img
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
