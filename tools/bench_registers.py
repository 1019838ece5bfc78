"""Cost of the 4 register tokens of the dinov2_vit*14_reg backbones: the same extraction on a plain model and on its
register twin, alternating in one process.  A register model runs 4 more token rows per image through every block
(T = 1 + 4 + N instead of 1 + N), so its cost should follow the token ratio in the GEMMs and LayerNorms and the square
of it in the attention.
Configurations (random-init weights, vit.random_state_dict -- the register model's other tensors equal the plain
model's; f16x3; auto engine), the two deep ones of bench.py:
  vitg_l31   ViT-G/14 layer 31 value, 322x322, B = 32   (T = 530 -> 534)
  vitl_l20   ViT-L/14 layer 20 value, 518x518, B = 64   (T = 1370 -> 1374)
Each arm is warmed up, then timed over --rounds rounds with the arms alternating inside each round (host clock around a
device synchronise); the median is reported, with one profiled call per arm split into GEMM / attention / LayerNorm
device time.  Prints the card, its power limit and clocks, then one JSON line per configuration; writes nothing unless
--out is given.

    python tools/bench_registers.py [--rounds 7] [--configs vitg_l31,vitl_l20] [--out results.json]
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
    "vitg_l31": ("dinov2_vitg14", 31, 322, 32),
    "vitl_l20": ("dinov2_vitl14", 20, 518, 64),
}


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else
            f"unavailable ({r.stderr.strip()})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_registers times the GPU path and needs a CUDA device")
    from anyloc_b200 import _lib
    from anyloc_b200.vit import VitWeights, random_state_dict
    dev = torch.device("cuda", 0)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []
    for key in args.configs.split(","):
        name, layer, side, B = CONFIGS[key]
        models = {}
        for arm in (name, name + "_reg"):
            sd = random_state_dict(arm, seed=0, device=dev, depth=layer + 1)
            models[arm] = VitWeights(arm, sd, dev, pair="f16")
            del sd
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
            prof[arm] = {c: round(p[c][0], 2) for c in ("gemm_tc", "attention", "layernorm", "vit_misc")}
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
        n = (side // 14) ** 2
        plain, reg = name, name + "_reg"
        line = {"config": key, "model": name, "layer": layer, "size": side, "batch": B, "precision": "f16x3",
                "tokens": [1 + n, 5 + n], "token_ratio": round((5 + n) / (1 + n), 4),
                "plain_ms": round(1e3 * med[plain], 2), "reg_ms": round(1e3 * med[reg], 2),
                "reg_over_plain": round(med[reg] / med[plain], 4),
                "spread_ms": {a: [round(1e3 * min(t), 2), round(1e3 * max(t), 2)] for a, t in times.items()},
                "profiled_ms": prof,
                "attention_ratio": round(prof[reg]["attention"] / max(prof[plain]["attention"], 1e-9), 4), **info}
        results.append(line)
        print(json.dumps(line), flush=True)
        del models, fns, img
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
