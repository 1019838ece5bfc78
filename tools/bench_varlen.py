"""Throughput of differently sized images through the extractor, three ways on the same seeded images:
  loop    one call per image (ext(img[None])[0]) -- what a caller without list input runs
  grouped images of equal size stacked into one uniform call each -- the best a caller without list input can do
  list    one call on the whole list (one packed forward pass, anyloc_vit_extract_varlen)
Models: ViT-S/14 layer 9 and ViT-G/14 layer 31, value facet, random-init weights (vit.random_state_dict), f16x3, the
fp16-range check off (it adds one reduction per call and, synchronous, one host sync).  Size mixes:
  dataset  32 images cycling 224x224, 322x322, 476x630, 518x518
  demo     16 images at the sizes the reference demo's rule (longest side shrunk to 1024 when larger, centre crop to a
           multiple of 14) gives 4:3, 3:4, 16:9 and 1:1 photos: 756x1022, 1022x756, 574x1022, 1022x1022
Each arm is warmed up on every shape, then timed over --rounds rounds with the arms alternating inside each round
(host clock around a device synchronise); the median is reported.  The list arm's features are checked bit-identical
to the loop arm's before any timing.  Prints the card, its power limit and clocks, then one JSON line per
(model, mix, arm); writes nothing unless --out is given.

    python tools/bench_varlen.py [--rounds 5] [--models vits14,vitg14] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODELS = {"vits14": ("dinov2_vits14", 9), "vitg14": ("dinov2_vitg14", 31)}
MIXES = {
    "dataset": ([(224, 224), (322, 322), (476, 630), (518, 518)], 32),
    "demo": ([(756, 1022), (1022, 756), (574, 1022), (1022, 1022)], 16),
}


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else
            f"unavailable ({r.stderr.strip()})"}


def mix_images(sizes, n, seed, device):
    import torch
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, *sizes[i % len(sizes)], generator=g).to(device) for i in range(n)]


def arms(ext, imgs):
    import torch
    groups = {}
    for i, x in enumerate(imgs):
        groups.setdefault(tuple(x.shape), []).append(i)

    def loop():
        return [ext(x[None])[0] for x in imgs]

    def grouped():
        out = [None] * len(imgs)
        for idx in groups.values():
            feats = ext(torch.stack([imgs[i] for i in idx]))
            for k, i in enumerate(idx):
                out[i] = feats[k]
        return out

    def packed():
        return ext(imgs)

    return {"loop": loop, "grouped": grouped, "list": packed}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--models", default="vits14,vitg14")
    ap.add_argument("--mixes", default="dataset,demo")
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_varlen times the GPU path and needs a CUDA device")
    from anyloc_b200 import utilities as u
    from anyloc_b200.vit import random_state_dict
    dev = torch.device("cuda", 0)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []
    for mk in args.models.split(","):
        name, layer = MODELS[mk]
        sd = random_state_dict(name, seed=0, device=dev, depth=layer + 1)
        ext = u.DinoV2ExtractFeatures(name, layer, "value", device=dev, weights=sd, precision="f16x3")
        ext.check_finite = "off"
        del sd
        for mix in args.mixes.split(","):
            sizes, n = MIXES[mix]
            imgs = mix_images(sizes, n, seed=1234, device=dev)
            tokens = sum((x.shape[1] // 14) * (x.shape[2] // 14) + 1 for x in imgs)
            fns = arms(ext, imgs)
            ref = fns["loop"]()
            for arm, fn in fns.items():             # warm-up of every shape each arm launches
                out = fn()
                if arm == "list":
                    same = all(torch.equal(a, b) for a, b in zip(out, ref))
                    if not same:
                        raise SystemExit(f"{mk}/{mix}: list features are not bit-identical to the per-image calls")
            del ref, out
            torch.cuda.synchronize()
            times = {a: [] for a in fns}
            for r in range(args.rounds):
                order = list(fns) if r % 2 == 0 else list(fns)[::-1]
                for arm in order:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fns[arm]()
                    torch.cuda.synchronize()
                    times[arm].append(time.perf_counter() - t0)
            med = {a: sorted(t)[len(t) // 2] for a, t in times.items()}
            for arm in fns:
                line = {"model": mk, "layer": layer, "mix": mix, "arm": arm, "images": n, "tokens": tokens,
                        "median_s": round(med[arm], 5), "min_s": round(min(times[arm]), 5),
                        "max_s": round(max(times[arm]), 5), "img_per_s": round(n / med[arm], 2),
                        "tokens_per_s": round(tokens / med[arm]), "list_bit_identical_to_loop": True,
                        "speedup_vs_loop": round(med["loop"] / med[arm], 3),
                        "speedup_vs_grouped": round(med["grouped"] / med[arm], 3), **info}
                results.append(line)
                print(json.dumps(line), flush=True)
            del imgs
        del ext
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
