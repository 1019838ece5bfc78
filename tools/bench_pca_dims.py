"""Measure a PCA-dimension sweep from reduce_pca_dims against one reduce_pca call per dimension, on the GPU.

    python tools/bench_pca_dims.py [--dims 1024 512 256 128 64 32 16] [--cases exact uploaded streamed] [--reps 1]
                                   [--json out.json]

The two arms alternate, --reps times each, in one process: the sequential arm calls reduce_pca(db, qu, k,
whitening=True) for every k in turn, the shared arm calls reduce_pca_dims(db, qu, dims, whitening=True) once, both
from the same numpy seed.  Cases, all on host fp32 rows of dimension 49 152 (a VLAD of 32 x 1536) with 1000 query
rows:
  exact     10 000 rows, svd_solver="full" (the in-memory Gram route);
  uploaded  100 000 rows, svd_solver="randomized", the rows uploaded once per call (per sweep);
  streamed  the same rows with the device budget set a byte below the rows' size, so every member's pass streams
            them from host memory in 1 GiB pieces.
Every run's outputs must be bit-identical between the arms.  The rows are seeded: a decaying 2048-dimensional
spectrum plus noise.  Reported: each arm's wall times and their ratio, with the card, its power limit, its max SM
clock and the SM clock sampled during the timed runs.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyloc_b200 import utilities as u  # noqa: E402
from tools.bench_fit_sweep import ClockSampler, smi  # noqa: E402

D = 49_152


def host_rows(n, seed, rank=2048, block=4096):
    """n x D host fp32 rows: a decaying rank-`rank` spectrum, a mean and noise, made on the device in blocks"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    basis = torch.randn(rank, D, device="cuda", generator=g) / np.sqrt(D)
    scale = 10.0 * 0.998 ** torch.arange(rank, device="cuda", dtype=torch.float32)
    mean = torch.randn(D, device="cuda", generator=g)
    out = np.empty((n, D), np.float32)
    for i in range(0, n, block):
        b = min(block, n - i)
        x = (torch.randn(b, rank, device="cuda", generator=g) * scale) @ basis + mean
        out[i:i + b] = (x + 0.05 * torch.randn(b, D, device="cuda", generator=g)).cpu().numpy()
    return out


def run_arm(arm, db, qu, dims, solver):
    np.random.seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if arm == "seq":
        outs = [u.reduce_pca(db, qu, k, svd_solver=solver, whitening=True) for k in dims]
    else:
        outs = u.reduce_pca_dims(db, qu, dims, svd_solver=solver, whitening=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs="+", default=[1024, 512, 256, 128, 64, 32, 16])
    ap.add_argument("--cases", nargs="+", default=["exact", "uploaded", "streamed"])
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pca_dims: no CUDA device")
    card = {"card": smi("name"), "power_limit": smi("power.limit"), "max_sm_clock": smi("clocks.max.sm")}
    print(json.dumps(card), flush=True)
    results = []
    rows = {}
    for case in a.cases:
        n = 10_000 if case == "exact" else 100_000
        if n not in rows:
            rows.clear()
            rows[n] = host_rows(n, seed=1), host_rows(1000, seed=2)
        db, qu = rows[n]
        solver = "full" if case == "exact" else "randomized"
        real_budget = u._device_budget
        if case == "streamed":
            u._device_budget = lambda dev, release_cache=True: 4 * n * D - 1
        try:
            times = {"seq": [], "shared": []}
            with ClockSampler() as clk:
                for rep in range(a.reps):
                    ref = None
                    for arm in ("seq", "shared") if rep % 2 == 0 else ("shared", "seq"):
                        t, outs = run_arm(arm, db, qu, a.dims, solver)
                        times[arm].append(t)
                        if ref is None:
                            ref = outs
                        else:
                            same = all(np.array_equal(x, y) for o, r in zip(outs, ref) for x, y in zip(o, r))
                            if not same:
                                sys.exit(f"bench_pca_dims: {case}: the arms' outputs differ")
                        del outs
                    del ref
        finally:
            u._device_budget = real_budget
        res = {"case": case, "n": n, "d": D, "queries": 1000, "dims": a.dims, "solver": solver,
               "seq_s": times["seq"], "shared_s": times["shared"],
               "ratio": float(np.median(times["shared"]) / np.median(times["seq"])), "identical": True,
               "sm_clock_mhz": sorted(clk.samples)[len(clk.samples) // 2] if clk.samples else None}
        results.append(res)
        print(json.dumps(res), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({**card, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
