"""Measure a vocabulary-size sweep's descriptors from generate_vocabularies against one VLAD.generate_multi per
vocabulary, on the GPU.

    python tools/bench_generate_sweep.py [--images 2000] [--patches 529] [--dim 1536] [--ks 32 64 128 256]
                                         [--reps 3] [--inputs host device list] [--json out.json]

For each input form the two arms alternate, --reps times each: the sequential arm calls v.generate_multi(x) for every
vocabulary in turn, the shared arm calls generate_vocabularies(vlads, x) once.  "host" passes a CPU tensor
[images, patches, dim] (what the reference driver hands generate_multi), "device" the same tensor on the GPU, "list" a
list of device views of one buffer with 0.5x to 1.5x the patches per image (what ext(list) returns).  The sweep runs
with all --ks and again with the first K alone (V = 1), which separates the host staging from the sharing.  Every
run's descriptors must be bit-identical between the arms.  The features are clustered (64 seeded centres plus noise);
the vocabularies are seeded random centres.  Reported: the median wall time of each arm and their ratio, with the
card, its power limit and the SM clock sampled during the timed runs.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyloc_b200 import _lib, utilities as u  # noqa: E402
from tools.bench_fit_sweep import ClockSampler, device_rows, smi  # noqa: E402


def vocabularies(ks, D):
    out = []
    for i, K in enumerate(ks):
        v = u.VLAD(K)
        v.kmeans = u._KMeans(K, mode=v.mode)
        g = torch.Generator().manual_seed(100 + i)
        v.kmeans.centroids = v.c_centers = torch.randn(K, D, generator=g)
        v.desc_dim = D
        out.append(v)
    return out


def run_arm(arm, vlads, x):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    outs = [v.generate_multi(x) for v in vlads] if arm == "seq" else u.generate_vocabularies(vlads, x)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=2000)
    ap.add_argument("--patches", type=int, default=529)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--ks", type=int, nargs="+", default=[32, 64, 128, 256])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--inputs", nargs="+", default=["host", "device", "list"])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_generate_sweep needs a CUDA device")
    _lib.load()
    print(f"gpu {smi('name')}, power limit {smi('power.limit')}, max SM clock {smi('clocks.max.sm')}", flush=True)
    n, N, D = a.images, a.patches, a.dim
    Xd = device_rows(n * N, D).view(n, N, D)
    rng = np.random.default_rng(0)
    lens = [int(m) for m in rng.integers(N // 2, N + N // 2 + 1, n)]
    buf = device_rows(sum(lens), D, seed=1)
    out = {"gpu": smi("name"), "power_limit": smi("power.limit"), "images": n, "patches": N, "dim": D, "ks": a.ks,
           "runs": {}}
    for form in a.inputs:
        x = {"host": lambda: Xd.cpu(), "device": lambda: Xd, "list": lambda: list(torch.split(buf, lens))}[form]()
        for ks in (a.ks, a.ks[:1]):
            vlads = vocabularies(ks, D)
            run_arm("multi", vlads, x[:2])                         # warm-up: workspaces, prepared blobs
            res = {"seq": [], "multi": []}
            same = True
            with ClockSampler() as clk:
                for rep in range(a.reps):
                    runs = {}
                    for arm in ("seq", "multi") if rep % 2 == 0 else ("multi", "seq"):
                        runs[arm] = run_arm(arm, vlads, x)
                    ok = all(torch.equal(p, q) for p, q in zip(runs["seq"][1], runs["multi"][1]))
                    same = same and ok
                    for arm in runs:
                        res[arm].append(runs[arm][0])
                    del runs
                    print(f"{form} V={len(ks)} rep {rep}: seq {res['seq'][-1]:.3f} s, shared {res['multi'][-1]:.3f} s, "
                          f"bit-identical {ok}", flush=True)
            m = {"seq_s": float(np.median(res["seq"])), "shared_s": float(np.median(res["multi"])),
                 "bit_identical": same, "sm_clock_mhz_median": float(np.median(clk.samples)) if clk.samples else None}
            m["ratio_shared_over_seq"] = m["shared_s"] / m["seq_s"]
            out["runs"][f"{form}_V{len(ks)}"] = m
            print(f"{form} V={len(ks)}: seq {m['seq_s']:.3f} s, shared {m['shared_s']:.3f} s "
                  f"(x{m['ratio_shared_over_seq']:.3f}); bit-identical {same}; SM clock {m['sm_clock_mhz_median']} MHz",
                  flush=True)
        del x
        torch.cuda.empty_cache()
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
