"""Measure the streamed k-means fit (VLAD.fit on host descriptors larger than the device) on the GPU.

    python tools/fit_stream.py [--rows 4000000] [--dim 1536] [--clusters 32] [--iters 4] [--reps 2] [--large 15300000]

1. Same size, three paths: at --rows x --dim (fits on the device) the in-memory fit, a fully streamed fit and a
   half-resident fit run alternately, --reps times each, with --iters Lloyd iterations (no convergence stop).  Their
   centres must be bit-identical; per-iteration times are the spacing of the iterations after the first.
2. Overlap: for the rounds one fully streamed iteration moves, the plain pinned host-to-device copy, the gather into
   the pinned staging buffer and the per-round device work (normalise + assign + accumulate), each timed alone.  A
   streamed iteration should take at most 1.2x the largest of the three, which is the one that bounds it.
3. Larger than the device: one fit of --large rows (Pitts30k: 10 000 images x 1 530 patches), or the most rows the
   host's available memory holds, through the plan VLAD.fit picks.  It must complete.
Host rows are tiles of one seeded random block (generating 94 GB of random numbers would dominate the run).
Prints the card, its power limit, a sampled SM clock, the host's available memory and usable cores beside the results.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyloc_b200 import _lib, utilities as u  # noqa: E402


def smi(query):
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={query}",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def mem_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def host_rows(R, D, seed=0, block=1 << 18):
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(min(R, block), D, generator=g)
    X = torch.empty(R, D)
    for i in range(0, R, base.shape[0]):
        n = min(base.shape[0], R - i)
        X[i:i + n] = base[:n]
    return X


class IterClock:
    """timestamps of the iterations of a fit: the in-memory loop calls _update once per iteration (plus one
    speculative call), the streamed loop calls anyloc_kmeans_finalize and waits for its shift"""

    def __init__(self):
        self.t = []
        self.lib = _lib.load()
        self.upd, self.fin = u._KMeans._update, self.lib.anyloc_kmeans_finalize

    def __enter__(self):
        clock, upd, fin = self, self.upd, self.fin

        def update(km, *a):
            clock.t.append(time.perf_counter())
            return upd(km, *a)

        def finalize(*a):
            clock.t.append(time.perf_counter())
            return fin(*a)
        u._KMeans._update = update
        self.lib.anyloc_kmeans_finalize = finalize
        return self

    def __exit__(self, *exc):
        u._KMeans._update = self.upd
        self.lib.anyloc_kmeans_finalize = self.fin

    def per_iter(self, iters):
        t = self.t[:iters]                      # drops the in-memory loop's speculative call
        return (t[-1] - t[1]) / (len(t) - 2) if len(t) > 2 else float("nan")


def fit(X, K, iters, dev, plan):
    """one VLAD.fit-style fit (rows normalised, cosine) with a fixed iteration count -> (centres, s per iteration, total s)"""
    km = u._KMeans(K, max_iter=iters, tol=-1.0, mode="cosine")
    np.random.seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with IterClock() as clock:
        if plan is None:
            km.fit(u._normalize_rows_dev(u._as_device_f32(X, dev)))
        else:
            km._fit_streamed(X, None, True, plan, dev)
        torch.cuda.synchronize()
    total = time.perf_counter() - t0
    return km.centroids.cpu(), clock.per_iter(iters), total


def overlap_parts(X, K, plan, dev):
    """the three parts of one fully streamed iteration, each alone: H2D, staging gather, device work (seconds)"""
    lib = _lib.load()
    R, D = X.shape
    chunks, rows_per = u._kmeans_partition(R, D)
    rounds = u._stream_rounds(R, chunks, rows_per, plan[0])
    sizes = [(chunks - 1) * p[0][1] + p[-1][1] for p in rounds]
    host = torch.empty(sizes[0], D, pin_memory=True)
    dbuf = torch.empty(sizes[0], D, device=dev)
    t0 = time.perf_counter()
    for j, pieces in enumerate(rounds):
        for ci, (lo, m) in enumerate(pieces):
            host[ci * pieces[0][1]:ci * pieces[0][1] + m].copy_(X[lo:lo + m])
    t_stage = time.perf_counter() - t0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for n in sizes:
        dbuf[:n].copy_(host[:n], non_blocking=True)
    torch.cuda.synchronize()
    t_h2d = time.perf_counter() - t0
    km = u._KMeans(K, mode="cosine")
    c = u._normalize_rows_dev(dbuf[:K].clone())
    ws = _lib.workspaces.get(dev, lib.anyloc_kmeans_round_workspace_bytes(R, D, K), "kmeans_upd")
    for rep in range(2):                        # the first pass warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j, n in enumerate(sizes):
            x = u._normalize_rows_dev(dbuf[:n])
            lab = km._assign(x, c)
            _lib.check(lib.anyloc_kmeans_accumulate_round(_lib.ptr(x), _lib.ptr(lab), R, n, rounds[j][0][1], D, K,
                                                          int(j > 0), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                       "accumulate_round")
        torch.cuda.synchronize()
        t_dev = time.perf_counter() - t0
    nbytes = sum(sizes) * D * 4
    return {"h2d": t_h2d, "staging": t_stage, "device": t_dev}, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--clusters", type=int, default=32)
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--large", type=int, default=15_300_000)
    args = ap.parse_args()
    dev = _lib.require_cuda()
    torch.cuda.set_device(dev)
    D, K = args.dim, args.clusters
    cores = len(os.sched_getaffinity(0))
    print(f"== {torch.cuda.get_device_name(dev)}; power limit / max SM clock {smi('power.limit,clocks.max.sm')}; "
          f"host memory available {mem_available() / 2**30:.0f} GiB; usable cores {cores}; torch threads "
          f"{torch.get_num_threads()}; staging buffers 2 x {u._STAGE_BYTES / 2**30:.1f} GiB pinned")

    X = host_rows(args.rows, D)
    R = X.shape[0]
    chunks, rows_per = u._kmeans_partition(R, D)
    P, _ = u._kmeans_plan(R, D, chunks, rows_per, 0, 2, lambda n: 0, u._STAGE_BYTES)
    n_rounds = -(-rows_per // P)
    plans = {"in-memory": None, "streamed": (P, 0), "half-resident": (P, n_rounds // 2)}
    print(f"== same size: {R} x {D} fp32 ({R * D * 4 / 1e9:.1f} GB), K={K}, {args.iters} iterations; {chunks} chunks "
          f"of {rows_per} rows, P={P}, {n_rounds} rounds of <= {chunks * P * D * 4 / 2**20:.0f} MiB")
    centres, times = {}, {k: [] for k in plans}
    for rep in range(args.reps):
        for name, plan in plans.items():
            c, per_it, total = fit(X, K, args.iters, dev, plan)
            times[name].append(per_it)
            if name in centres:
                assert torch.equal(centres[name], c), f"{name}: not reproducible"
            centres[name] = c
            print(f"   rep {rep} {name:14s} {per_it * 1e3:9.1f} ms/iteration   total {total:6.2f} s")
    same = all(torch.equal(centres["in-memory"], c) for c in centres.values())
    print(f"   centres bit-identical across the three paths: {same}; SM clock sampled after the last fit "
          f"{smi('clocks.sm')}")

    parts, nbytes = overlap_parts(X, K, plans["streamed"], dev)
    it = min(times["streamed"])
    bound = max(parts, key=parts.get)
    print(f"== overlap, per fully streamed iteration ({nbytes / 1e9:.1f} GB): " +
          ", ".join(f"{k} alone {v * 1e3:.1f} ms ({nbytes / v / 1e9:.1f} GB/s)" for k, v in parts.items()))
    print(f"   streamed iteration {it * 1e3:.1f} ms = {it / parts[bound]:.2f} x the largest part ({bound}); "
          f"{'within' if it <= 1.2 * parts[bound] else 'OVER'} the 1.2x target")
    del X, centres

    free_dev = torch.cuda.mem_get_info(dev)[1]
    R_big = min(args.large, (mem_available() - (12 << 30) - 2 * u._STAGE_BYTES) // (4 * D))
    label = "Pitts30k size" if R_big == args.large else "the most rows the host memory holds"
    label += ", larger than the device" if R_big * 4 * D > free_dev else ", NOT larger than the device"
    X = host_rows(R_big, D, seed=1)
    plan = u._host_fit_plan(X, dev, K, copies=2)
    print(f"== larger than the device: {R_big} x {D} fp32 = {R_big * D * 4 / 1e9:.1f} GB ({label}; device "
          f"{free_dev / 1e9:.1f} GB), plan {plan}")
    c, per_it, total = fit(X, K, 3, dev, plan)
    print(f"   completed: 3 iterations in {total:.1f} s ({per_it * 1e3:.0f} ms per iteration after the first); "
          f"centres finite {bool(torch.isfinite(c).all())}")


if __name__ == "__main__":
    main()
