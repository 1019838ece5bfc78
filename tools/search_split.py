"""Measure the split index (FlatIndex(placement="split"): lo halves in page-locked host memory) on the GPU.

    python tools/search_split.py [--sizes 10000,100000] [--dim 49152] [--queries 1000] [--k 5] [--reps 3]
                                 [--large-dim 196608] [--large 100000]

1. Same size, the placements: at each --sizes database (c3's 10k and c4's 100k x 49152 by default) the resident,
   the split and the fully streamed index are searched alternately in one process, --reps times each.  Their
   (dist, idx) must be identical; the median time of each is reported.  The streamed index is forced with an
   in-process budget override, as tools/search_stream.py forces it.
   The split index runs twice: gathering the unique candidate rows into a device stage first ("split"), and with the
   re-scoring reading lo from host memory directly ("split-direct", what runs when no stage fits).
2. The coarse route's lo traffic: per search, the candidate rows summed over the queries (what split-direct reads
   from host memory) and the unique rows among them (what split gathers).  The link rate of each is those lo bytes
   over its search time less the resident one's: they run the same launches, except where lo is read from.
3. The largest database host memory allows at --large-dim (K = 128 ViT-G VLADs by default): seeded random rows made
   on the device and added in chunks to a split index reserved at its full capacity, so that the host holds lo only.
   Its coarse search of --queries queries, and the exact route of 8 queries, which moves every lo row.
Other host rows are tiles of one seeded random block.  Prints the card, its power limit, a sampled SM clock and the host's
available memory beside the results.
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
from tools.search_stream import budget_for, build, timed_search  # noqa: E402


def counts(ix):
    """(unique, all) candidate rows of the last search, summed over its coarse query chunks"""
    return tuple(sum(c[j] for c in ix._split_counts) for j in range(2))


def direct(ix):
    """the same split index, re-scoring from host lo directly (the path taken when no stage fits)"""
    ix._split_stage = lambda nbytes, dev: None
    return ix


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,100000")
    ap.add_argument("--dim", type=int, default=49152)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--k", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--large-dim", type=int, default=128 * 1536)
    ap.add_argument("--large", type=int, default=100_000)
    args = ap.parse_args()
    dev = _lib.require_cuda()
    torch.cuda.set_device(dev)
    D, k = args.dim, args.k
    print(f"== {torch.cuda.get_device_name(dev)}; power limit / max SM clock {smi('power.limit,clocks.max.sm')}; "
          f"host memory available {mem_available() / 2**30:.0f} GiB; usable cores {len(os.sched_getaffinity(0))}")
    qu = host_rows(args.queries, D, seed=7).cuda()
    for n_db in [int(s) for s in args.sizes.split(",")]:
        need = 2.5 * n_db * D * 4 + (8 << 30)       # the rows, the streamed host copy, the split lo, slack
        if need > mem_available():
            print(f"== {n_db} x {D}: skipped, needs {need / 2**30:.0f} GiB of host memory")
            continue
        X = host_rows(n_db, D, seed=n_db)
        stage = min(u._STAGE_BYTES, n_db * D * 4 // 8)
        b0, P = budget_for(n_db, D, 0, stage)
        sp = u.FlatIndex(D, device="cuda", placement="split")
        sp.add(X)
        sd = direct(u.FlatIndex(D, device="cuda", placement="split"))
        sd.add(X)
        paths = {"resident": build(X, None, stage), "split": sp, "split-direct": sd, "streamed": build(X, b0, stage)}
        assert paths["resident"]._stream is None and paths["streamed"]._stream is not None
        print(f"== same size: {n_db} x {D} ({n_db * D * 4 / 1e9:.1f} GB fp32), {args.queries} queries, k={k}; "
              f"device blob resident {paths['resident']._blob.numel() / 1e9:.2f} GB, split "
              f"{sp._blob.numel() / 1e9:.2f} GB + {sp._lo.nbytes / 1e9:.2f} GB pinned lo; "
              f"streamed in pieces of {P} rows")
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
            print(f"   {name:12s} median {statistics.median(times[name]) * 1e3:9.1f} ms over {args.reps}   "
                  f"all {[round(t * 1e3, 1) for t in times[name]]}")
        print(f"   (dist, idx) identical across all: {same}; SM clock sampled {smi('clocks.sm')}")
        assert same
        uniq, total = counts(sp)
        med = {n: statistics.median(t) for n, t in times.items()}
        print(f"   candidates: {total} rows over {args.queries} queries ({total / args.queries:.1f} a query), "
              f"{uniq} unique; lo bytes {total * D * 2 / 1e9:.2f} GB direct, {uniq * D * 2 / 1e9:.2f} GB gathered")
        for name, b in (("split", uniq * D * 2), ("split-direct", total * D * 2)):
            extra = med[name] - med["resident"]
            print(f"   {name:12s} - resident {extra * 1e3:.1f} ms: {b / extra / 1e9:.1f} GB/s of lo over the link")
        del paths, sp, sd, X, outs
        torch.cuda.empty_cache()

    Dl = args.large_dim
    lo_row = Dl * 2
    n_big = int(min(args.large, (mem_available() - (16 << 30)) // lo_row))
    chunk = 1000
    g = torch.Generator(device="cuda").manual_seed(3)
    t0 = time.perf_counter()
    ix = u.FlatIndex(Dl, device="cuda", placement="split", capacity=n_big)
    for r0 in range(0, n_big, chunk):           # device rows: the host holds lo only
        ix.add(torch.randn(min(chunk, n_big - r0), Dl, device="cuda", generator=g))
    torch.cuda.synchronize()
    t_add = time.perf_counter() - t0
    q = host_rows(args.queries, Dl, seed=8).cuda()
    print(f"== largest: {n_big} x {Dl} (fp32 {n_big * Dl * 4 / 1e9:.1f} GB; resident index "
          f"{_lib.load().anyloc_index_bytes(n_big, Dl, 1) / 1e9:.1f} GB); split device blob "
          f"{ix._blob.numel() / 1e9:.1f} GB + {ix._lo.nbytes / 1e9:.1f} GB pinned lo; added in chunks of {chunk} "
          f"device rows in {t_add:.1f} s")
    ts = {"split": [], "split-direct": []}
    for rep in range(args.reps + 1):
        for name in ts:
            if name == "split-direct":
                direct(ix)
            d, i, t = timed_search(ix, q, k)
            if name == "split-direct":
                del ix._split_stage                 # back to the class's staging
            if rep:
                ts[name].append(t)
    uniq, total = counts(ix)
    for name, v in ts.items():
        print(f"   {args.queries} queries, k={k}, {name}: median {statistics.median(v) * 1e3:.1f} ms, all "
              f"{[round(t * 1e3, 1) for t in v]}")
    print(f"   candidates {total} ({uniq} unique; lo {total * lo_row / 1e9:.2f} GB direct, {uniq * lo_row / 1e9:.2f} GB "
          f"gathered); indices in range {bool(((i >= 0) & (i < n_big)).all())}; SM clock sampled {smi('clocks.sm')}")
    d, i, t = timed_search(ix, q[:8], k)
    print(f"   8 queries (the exact route, every lo row over the link): {t * 1e3:.0f} ms "
          f"({n_big * lo_row / t / 1e9:.1f} GB/s of lo)")


if __name__ == "__main__":
    main()
