"""Throughput and error of the single-fp16 precision (f16x1) against single bf16, alternating in one process.

Both run one 2-byte MMA per product on the same bytes; f16x1 rounds every operand to fp16's 11 significant bits (the
hi half of the f16x3 pair), bf16 to 8.  Configurations (random-init weights, vit.random_state_dict; auto engine), the
ViT part of bench.py's pipeline workloads:
  c2   ViT-G/14 layer 31 value, 322x322, B = 32
  c5   ViT-L/14 layer 20 value, 518x518, B = 64
  c1   ViT-S/14 layer 9 value, 224x224, B = 16
Every shape is warmed up, then the f16x1 and bf16 arms alternate inside each of --rounds rounds (host clock around a
device synchronise); the median gives img/s.  One profiled call per arm splits the device time into GEMM / attention /
LayerNorm / other.  The feature error of f16x3, f16x1, bf16 and fp8, max|f - f32| / max|f32| and |f - f32|_F / |f32|_F,
is measured at full size on 2 images against the restated model in fp32 on the GPU (TF32 off).  A pipeline proxy: a
K = 32 cosine k-means vocabulary is fitted on the f16x3 features of those images, and the share of patches whose hard
VLAD label under each other precision differs from the f16x3 label is reported.  All of it uses random-init weights,
not a trained checkpoint.  Prints the card, its power limit and clocks, then one JSON line per configuration; writes
nothing unless --out is given.

    python tools/bench_f16x1.py [--rounds 7] [--configs c2,c5,c1] [--out results.json]
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

TIMED = {"f16x1": "f16x1", "bf16": "bf16"}
ERR_ONLY = {"f16x3": "f16", "fp8": "fp8"}


def cosine_kmeans(x, k, iters=25, seed=0):
    """centres [k, D] of a cosine k-means on the rows of x (unit rows; fixed seed, fixed iteration count)"""
    import torch
    x = torch.nn.functional.normalize(x.double(), dim=1)
    g = torch.Generator().manual_seed(seed)
    c = x[torch.randperm(x.shape[0], generator=g)[:k].to(x.device)]
    for _ in range(iters):
        lab = (x @ c.T).argmax(dim=1)
        for j in range(k):
            m = lab == j
            if m.any():
                c[j] = torch.nn.functional.normalize(x[m].sum(0), dim=0)
    return c


def errors(name, layer, sd, models, side, dev):
    """(max-element, RMS) error of each arm against the restated fp32 model on 2 images, and the share of hard labels
    (K = 32, vocabulary of the f16x3 features) that differ from f16x3's"""
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
    del model
    feats = {arm: m.extract(img, layer, "value").double() for arm, m in models.items()}
    err = {arm: [float((f - ref).abs().max() / ref.abs().max()), float((f - ref).norm() / ref.norm())]
           for arm, f in feats.items()}
    base = feats["f16x3"].reshape(-1, feats["f16x3"].shape[-1])
    centres = cosine_kmeans(base, 32)
    lab0 = (torch.nn.functional.normalize(base, dim=1) @ centres.T).argmax(dim=1)
    changed = {}
    for arm in ("f16x1", "bf16", "fp8"):
        f = torch.nn.functional.normalize(feats[arm].reshape(base.shape), dim=1)
        changed[arm] = round(float(((f @ centres.T).argmax(dim=1) != lab0).double().mean()), 5)
    return err, changed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_f16x1 times the GPU path and needs a CUDA device")
    from anyloc_b200 import _lib
    from anyloc_b200.vit import VitWeights, random_state_dict
    dev = torch.device("cuda", 0)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []
    for key in args.configs.split(","):
        name, layer, side, B = CONFIGS[key]
        sd = random_state_dict(name, seed=0, device=dev, depth=layer + 1)
        models = {arm: VitWeights(name, sd, dev, pair=pair) for arm, pair in {**TIMED, **ERR_ONLY}.items()}
        err, changed = errors(name, layer, sd, models, side, dev)
        for arm in ERR_ONLY:
            del models[arm]
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
        line = {"config": key, "model": name, "layer": layer, "size": side, "batch": B, "weights": "random-init",
                "ms": {a: round(1e3 * t, 2) for a, t in med.items()},
                "img_per_s": {a: round(B / t, 1) for a, t in med.items()},
                "f16x1_over_bf16_time": round(med["f16x1"] / med["bf16"], 3),
                "spread_ms": {a: [round(1e3 * min(t), 2), round(1e3 * max(t), 2)] for a, t in times.items()},
                "profiled_ms": prof, "feature_err_vs_fp32_max_rms": err,
                "vlad_k32_labels_changed_vs_f16x3": changed, **info}
        results.append(line)
        print(json.dumps(line), flush=True)
        del models, fns, img
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
