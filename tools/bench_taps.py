"""Cost of reading several (layer, facet) taps of the same images, two ways on one uploaded weight set:
  loop    VitWeights.extract(img, layer, facet) once per tap -- what one DinoV2ExtractFeatures per tap costs, minus
          their separate weight uploads
  taps    one VitWeights.extract_taps call (one forward pass to the deepest tapped layer)
and, as the cost of tapping itself, one extract(img, L_max, "token") call: the same blocks without keeping anything.
Configurations (random-init weights, vit.random_state_dict; f16x3; auto engine), the tap lists AnyLoc's ablations read:
  vits_all    ViT-S/14 224x224, B = 16, all 12 layers x 4 facets
  vitg_value  ViT-G/14 322x322, B = 8, all 40 layers, value facet
  vitg_l31    ViT-G/14 322x322, B = 8, layer 31, all 4 facets
Each arm is warmed up on every shape, then timed over --rounds rounds with the arms alternating inside each round (host
clock around a device synchronise); the median is reported.  The taps arm's outputs are checked torch.equal to the loop
arm's before any timing.  Prints the card, its power limit and clocks, then one JSON line per configuration; writes
nothing unless --out is given.

    python tools/bench_taps.py [--rounds 5] [--configs vits_all,vitg_value,vitg_l31] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FACETS = ("query", "key", "value", "token")
CONFIGS = {
    "vits_all": ("dinov2_vits14", 224, 16, [(l, f) for l in range(12) for f in FACETS]),
    "vitg_value": ("dinov2_vitg14", 322, 8, [(l, "value") for l in range(40)]),
    "vitg_l31": ("dinov2_vitg14", 322, 8, [(31, f) for f in FACETS]),
}


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else
            f"unavailable ({r.stderr.strip()})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_taps times the GPU path and needs a CUDA device")
    from anyloc_b200.vit import VitWeights, random_state_dict
    dev = torch.device("cuda", 0)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []
    for key in args.configs.split(","):
        name, side, B, taps = CONFIGS[key]
        l_max = max(l for l, _ in taps)
        sd = random_state_dict(name, seed=0, device=dev, depth=l_max + 1)
        m = VitWeights(name, sd, dev, pair="f16")
        del sd
        img = torch.randn(B, 3, side, side, generator=torch.Generator().manual_seed(1234)).to(dev)

        def loop():
            return [m.extract(img, l, f) for l, f in taps]

        def tapped():
            return m.extract_taps(img, taps)

        def token():
            return m.extract(img, l_max, "token")

        fns = {"loop": loop, "taps": tapped, "token_only": token}
        ref = loop()
        out = tapped()           # warm-up of every shape each arm launches, and the equality check
        token()
        if not all(torch.equal(out[k], r) for k, r in enumerate(ref)):
            raise SystemExit(f"{key}: the taps call is not bit-identical to the per-tap calls")
        del ref, out
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
        line = {"config": key, "model": name, "size": side, "batch": B, "taps": len(taps), "l_max": l_max,
                "precision": "f16x3", "taps_equal_loop": True,
                **{f"{a}_ms_per_img": round(1e3 * med[a] / B, 3) for a in fns},
                **{f"{a}_spread_ms": [round(1e3 * min(times[a]), 2), round(1e3 * max(times[a]), 2)] for a in fns},
                "loop_over_taps": round(med["loop"] / med["taps"], 3),
                "taps_over_token_only": round(med["taps"] / med["token_only"], 3), **info}
        results.append(line)
        print(json.dumps(line), flush=True)
        del m, img
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
