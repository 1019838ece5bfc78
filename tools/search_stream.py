"""Measure the streamed search (FlatIndex over host rows larger than the device) on the GPU.

    python tools/search_stream.py [--sizes 10000,100000] [--dim 49152] [--queries 1000] [--k 5] [--reps 3]
                                  [--budget-gb 8] [--large 150000]

1. Same size, three paths: at each --sizes database (c3's 10k and c4's 100k x 49152 by default, both fit the device)
   the resident, the fully streamed and the half-resident search run alternately in one process, --reps times each.
   Their (dist, idx) must be identical; the median time of each is reported.  The streamed paths are forced with an
   in-process budget override, as the tests force them.
2. Overlap: for one fully streamed search of the largest size, the gather into the pinned staging buffer, the pinned
   host-to-device copy and the per-piece device work (prepare + search + merge), each timed alone.  The streamed search
   should take at most 1.2x the largest of the three, which is the one that bounds it.
3. Larger than the budget: one search of --large rows (or the most the host's available memory holds) with the
   device budget set to --budget-gb.  It must complete.
Host rows are tiles of one seeded random block.  Prints the card, its power limit, a sampled SM clock, the host's
available memory and usable cores beside the results.
"""
import argparse
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyloc_b200 import _lib, utilities as u  # noqa: E402
from tools.fit_stream import host_rows, mem_available, smi  # noqa: E402


def byte_fns(D):
    lib = _lib.load()
    return (lambda n: lib.anyloc_index_bytes(n, D, 1),
            lambda n, q=u._SEARCH_Q_CHUNK: lib.anyloc_index_search_workspace_bytes(n, q, D, 1))


def budget_for(n_db, D, resident_pieces, stage):
    """the device budget under which an n_db-row index streams in pieces that fill `stage` bytes, with
    `resident_pieces` of them kept"""
    ib, wb = byte_fns(D)
    P = max(1, min(n_db, stage // (4 * D)))
    return u._stream_fixed_bytes(P, 4 * D, ib, wb) + resident_pieces * ib(P), P


def build(X, budget, stage):
    """a cosine FlatIndex over host rows X, under `budget` (None: the real free memory) and `stage` staging bytes"""
    real = u._device_budget, u._STAGE_BYTES
    if budget is not None:
        u._device_budget = lambda dev, release_cache=True: budget
    u._STAGE_BYTES = stage
    try:
        ix = u.FlatIndex(X.shape[1], "cosine", True, device="cuda")
        ix.add(X)
    finally:
        u._device_budget, u._STAGE_BYTES = real
    return ix


def timed_search(ix, qu, k):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    d, i = ix.search(qu, k)
    torch.cuda.synchronize()
    return d, i, time.perf_counter() - t0


def overlap_parts(ix, qu, k):
    """the three parts of one search of a fully streamed index, each alone (seconds)"""
    lib = _lib.load()
    P, D = ix._stream["P"], ix.dp
    pieces = u._search_pieces(ix.ntotal, min(ix.ntotal, ix.capacity), P)
    host = torch.empty(P, D, pin_memory=True)
    raw = torch.empty(P, D, device="cuda")
    t0 = time.perf_counter()
    for r0, m, _ in pieces:
        ix._gather(host, r0, m)
    t_stage = time.perf_counter() - t0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r0, m, _ in pieces:
        raw[:m].copy_(host[:m], non_blocking=True)
    torch.cuda.synchronize()
    t_h2d = time.perf_counter() - t0
    blob = torch.empty(lib.anyloc_index_bytes(P, D, 1), dtype=torch.uint8, device="cuda")
    n_q = qu.shape[0]
    dist = torch.full((n_q, k), -float("inf"), device="cuda")
    idx = torch.full((n_q, k), -1, dtype=torch.int64, device="cuda")
    ws = _lib.workspaces.get(qu.device, lib.anyloc_index_search_workspace_bytes(P, n_q, D, 1), "topk")
    for rep in range(2):                        # the first pass warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for r0, m, _ in pieces:
            _lib.check(lib.anyloc_index_init(_lib.ptr(blob), blob.numel(), P, D, 1, _lib.stream_ptr()), "init")
            _lib.check(lib.anyloc_index_add(_lib.ptr(blob), blob.numel(), P, 0, _lib.ptr(raw), m, D, 1,
                                            _lib.stream_ptr()), "add")
            _lib.check(lib.anyloc_index_search_continue(_lib.ptr(blob), blob.numel(), P, 0, m, r0, ix.ntotal,
                                                        _lib.ptr(qu), n_q, D, k, 0, 1, _lib.ptr(dist), _lib.ptr(idx),
                                                        _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "continue")
        torch.cuda.synchronize()
        t_dev = time.perf_counter() - t0
    return {"staging": t_stage, "h2d": t_h2d, "device": t_dev}, ix.ntotal * D * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,100000")
    ap.add_argument("--dim", type=int, default=49152)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--budget-gb", type=float, default=8.0)
    ap.add_argument("--large", type=int, default=150_000)
    args = ap.parse_args()
    dev = _lib.require_cuda()
    torch.cuda.set_device(dev)
    D, k = args.dim, args.k
    print(f"== {torch.cuda.get_device_name(dev)}; power limit / max SM clock {smi('power.limit,clocks.max.sm')}; "
          f"host memory available {mem_available() / 2**30:.0f} GiB; usable cores {len(os.sched_getaffinity(0))}; "
          f"torch threads {torch.get_num_threads()}; staging buffers 2 x {u._STAGE_BYTES / 2**30:.1f} GiB pinned")
    qu = host_rows(args.queries, D, seed=7).cuda()
    last = None
    for n_db in [int(s) for s in args.sizes.split(",")]:
        need = 2.5 * n_db * D * 4 + (8 << 30)       # the rows, the streamed and half-resident host copies, slack
        if need > mem_available():
            print(f"== {n_db} x {D}: skipped, needs {need / 2**30:.0f} GiB of host memory")
            continue
        X = host_rows(n_db, D, seed=n_db)
        # at least 8 pieces: at c3's size one 1 GiB piece's buffers would take more than the resident index
        stage = min(u._STAGE_BYTES, n_db * D * 4 // 8)
        b0, P = budget_for(n_db, D, 0, stage)
        n_pieces = -(-n_db // P)
        b_half, _ = budget_for(n_db, D, n_pieces // 2, stage)
        print(f"== same size: {n_db} x {D} fp32 ({n_db * D * 4 / 1e9:.1f} GB), {args.queries} queries, k={k}; "
              f"pieces of {P} rows ({P * D * 4 / 2**20:.0f} MiB), {n_pieces} pieces")
        paths = {"resident": build(X, None, stage), "streamed": build(X, b0, stage),
                 "half-resident": build(X, b_half, stage)}
        assert paths["resident"]._stream is None and paths["streamed"]._stream is not None
        assert paths["half-resident"].capacity == min(n_db, P * (n_pieces // 2))
        times, outs = {n: [] for n in paths}, {}
        for rep in range(args.reps + 1):        # rep 0 warms up
            for name, ix in paths.items():
                d, i, t = timed_search(ix, qu, k)
                if rep:
                    times[name].append(t)
                if name in outs:
                    assert torch.equal(outs[name][0], d) and torch.equal(outs[name][1], i), f"{name}: not reproducible"
                outs[name] = (d, i)
        same = all(torch.equal(outs["resident"][0], d) and torch.equal(outs["resident"][1], i) for d, i in outs.values())
        for name in paths:
            med = statistics.median(times[name])
            print(f"   {name:14s} median {med * 1e3:9.1f} ms over {args.reps}  ({n_db * D * 4 / med / 1e9:6.1f} GB/s of "
                  f"database)   all {[round(t * 1e3, 1) for t in times[name]]}")
        print(f"   (dist, idx) identical across the three paths: {same}; SM clock sampled {smi('clocks.sm')}")
        assert same
        last = (paths["streamed"], statistics.median(times["streamed"]))
        del paths, X, outs
        torch.cuda.empty_cache()

    ix, t_stream = last
    parts, nbytes = overlap_parts(ix, qu, k)
    bound = max(parts, key=parts.get)
    print(f"== overlap, one fully streamed search ({nbytes / 1e9:.1f} GB): " +
          ", ".join(f"{n} alone {v * 1e3:.1f} ms ({nbytes / v / 1e9:.1f} GB/s)" for n, v in parts.items()))
    print(f"   streamed search {t_stream * 1e3:.1f} ms = {t_stream / parts[bound]:.2f} x the largest part ({bound}); "
          f"{'within' if t_stream <= 1.2 * parts[bound] else 'OVER'} the 1.2x target")
    del ix, last
    torch.cuda.empty_cache()

    budget = int(args.budget_gb * 2**30)
    n_big = min(args.large, (mem_available() - (12 << 30) - 2 * u._STAGE_BYTES) // (2 * 4 * D))
    X = host_rows(n_big, D, seed=1)
    ix = build(X, budget, u._STAGE_BYTES)
    print(f"== larger than the budget: {n_big} x {D} fp32 = {n_big * D * 4 / 1e9:.1f} GB, budget "
          f"{budget / 1e9:.1f} GB; streams {ix._stream is not None}, {ix.capacity} rows resident, pieces of "
          f"{ix._stream['P'] if ix._stream else '-'} rows")
    d, i, t = timed_search(ix, qu, k)
    print(f"   completed in {t:.2f} s ({n_big * D * 4 / t / 1e9:.1f} GB/s of database); indices in range "
          f"{bool(((i >= 0) & (i < n_big)).all())}, distances finite {bool(torch.isfinite(d).all())}")


if __name__ == "__main__":
    main()
