"""Measure reduce_pca's streamed route (the rows fed through the fp64 Gram / covariance accumulation) on the GPU.

    python tools/pca_stream.py [--both 10000x49152,60000x4096] [--large 26000x196608] [--k 512] [--reps 3]

1. Where both routes fit (--both, n x d host fp32 rows with a decaying spectrum, 1000 test rows): the in-memory route
   and the streamed route, forced with an in-process budget override, run alternately --reps times each in one process;
   the median wall time of each (host clock around the call, which ends in a device-to-host copy) and the largest
   difference of their outputs.
2. Where only the stream fits (--large): the streamed route alone, lower_dim = --k with whitening, once.
3. For each streamed run, per stage: the mean pass, the accumulation, eigh, vt and the projections.  Kernel times are
   CUDA events around each launch, summed; stage wall times are host clocks between device synchronisations.  The
   accumulation's fp64 rate counts K m (m + 1) flops (the lower triangle, K the contracted length), against the 67
   TFLOP/s FP64 data sheet figure; the host gather rate counts the bytes gathered into the pinned stages over the gather
   time; the H2D rate is one pinned staging buffer copied to the device, timed with events.
Prints the card, its power limit and max SM clock, read in the same run.
"""
import argparse
import os
import statistics
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyloc_b200 import _lib, utilities as u  # noqa: E402

FP64_PEAK = 67e12


def smi(query):
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={query}",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def spectrum_rows(n, n_te, d, seed, rank=640, decay=0.99, chunk=4096):
    """host fp32 [n, d] and [n_te, d]: rank-`rank` rows with geometrically decaying scales plus a non-zero mean, made on
    the device in chunks.  The rank is above lower_dim, so that every retained component is determined by the data."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    basis = torch.linalg.qr(torch.randn(d, rank, device="cuda", generator=g))[0]
    scales = decay ** torch.arange(rank, device="cuda", dtype=torch.float32)
    offset = 0.3 * torch.randn(d, device="cuda", generator=g)
    out = []
    for m in (n, n_te):
        x = torch.empty(m, d)
        for r in range(0, m, chunk):
            h = min(chunk, m - r)
            x[r:r + h] = ((torch.randn(h, rank, device="cuda", generator=g) * scales) @ basis.T + offset).cpu()
        out.append(x.numpy())
    return out


class Stages:
    """per-stage kernel times (events around each launch) and gather times, collected through wrappers of
    utilities' streamed-route helpers"""

    def __init__(self):
        self.ev = defaultdict(list)
        self.gather_s, self.gather_bytes = 0.0, 0
        self.flops = 0.0

    def install(self):
        real_colsum, real_acc, real_gather = u._pca_colsum, u._pca_accumulate, u._PcaRows.gather
        real_eigh = torch.linalg.eigh

        def timed(name, fn, *a, **kw):
            b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            b.record()
            r = fn(*a, **kw)
            e.record()
            self.ev[name].append((b, e))
            return r

        def acc(mode, x, mu, out, uu=None):
            if mode != "vt":
                m = out.shape[0]
                self.flops += (x.shape[0] if mode == "cov" else x.shape[1]) * m * (m + 1)
            return timed("accumulate" if mode != "vt" else "vt", real_acc, mode, x, mu, out, uu)

        def gather(rows, dst, box):
            t = time.perf_counter()
            real_gather(rows, dst, box)
            self.gather_s += time.perf_counter() - t
            self.gather_bytes += dst.numel() * 4

        u._pca_colsum = lambda x, out: timed("mean", real_colsum, x, out)
        u._pca_accumulate = acc
        u._PcaRows.gather = gather
        torch.linalg.eigh = lambda a: timed("eigh", real_eigh, a)

        def restore():
            u._pca_colsum, u._pca_accumulate, u._PcaRows.gather = real_colsum, real_acc, real_gather
            torch.linalg.eigh = real_eigh
        return restore

    def ms(self, name):
        return sum(b.elapsed_time(e) for b, e in self.ev[name])


def forced(n, d, n_te):
    """a budget just under the in-memory footprint: the streamed route"""
    return lambda dev, release_cache=True: u._pca_in_memory_bytes(n, d, n_te) - 1


def run(tr, te, k, budget=None, stages=None):
    """-> (wall seconds, outputs, {stage: wall seconds})"""
    walls = {}
    real_budget, real_fit, real_proj = u._device_budget, u._PcaDev.fit_streamed, u._pca_project_streamed
    if budget is not None:
        u._device_budget = budget

    def fit(pca, *a):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = real_fit(pca, *a)
        torch.cuda.synchronize()
        walls["fit"] = walls.get("fit", 0) + time.perf_counter() - t
        return r

    def proj(*a):
        t = time.perf_counter()
        r = real_proj(*a)
        walls["projections"] = walls.get("projections", 0) + time.perf_counter() - t
        return r
    u._PcaDev.fit_streamed, u._pca_project_streamed = fit, proj
    restore = stages.install() if stages else None
    try:
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = u.reduce_pca(tr, te, k, whitening=True)
        torch.cuda.synchronize()
        return time.perf_counter() - t, out, walls
    finally:
        u._device_budget, u._PcaDev.fit_streamed, u._pca_project_streamed = real_budget, real_fit, real_proj
        if restore:
            restore()


def h2d_rate(dev):
    host = torch.empty(u._STAGE_BYTES // 4, pin_memory=True)
    dst = torch.empty(host.numel(), device=dev)
    for _ in range(2):
        dst.copy_(host, non_blocking=True)
    b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    b.record()
    for _ in range(5):
        dst.copy_(host, non_blocking=True)
    e.record()
    e.synchronize()
    return 5 * host.numel() * 4 / (b.elapsed_time(e) / 1e3)


def report(label, n, d, wall, walls, st):
    m = min(n, d)
    acc_ms = st.ms("accumulate")
    print(f"   {label}: {wall:.2f} s end to end; fit {walls.get('fit', 0):.2f} s, projections "
          f"{walls.get('projections', 0):.2f} s (host clocks)")
    print(f"     kernels (events): mean {st.ms('mean'):.1f} ms, accumulation {acc_ms:.1f} ms, eigh {st.ms('eigh'):.1f} "
          f"ms, vt {st.ms('vt'):.1f} ms")
    rate = st.flops / (acc_ms / 1e3) if acc_ms else 0.0
    print(f"     accumulation: {st.flops:.3e} flops (K m (m+1), m = {m}) at {rate / 1e12:.1f} TFLOP/s fp64 = "
          f"{100 * rate / FP64_PEAK:.0f} % of the 67 TFLOP/s data sheet")
    if st.gather_s:
        print(f"     host gather: {st.gather_bytes / 1e9:.1f} GB in {st.gather_s:.2f} s = "
              f"{st.gather_bytes / st.gather_s / 1e9:.1f} GB/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--both", default="10000x49152,60000x4096")
    ap.add_argument("--large", default="26000x196608")
    ap.add_argument("--k", type=int, default=512)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--test-rows", type=int, default=1000)
    args = ap.parse_args()
    dev = _lib.require_cuda()
    torch.cuda.set_device(dev)
    print(f"== {torch.cuda.get_device_name(dev)}; name, power limit, max SM clock: "
          f"{smi('name,power.limit,clocks.max.sm')}")
    print(f"== H2D of one pinned {u._STAGE_BYTES >> 20} MiB stage: {h2d_rate(dev) / 1e9:.1f} GB/s")
    n_te, k = args.test_rows, args.k
    for shape in filter(None, args.both.split(",")):
        n, d = map(int, shape.split("x"))
        tr, te = spectrum_rows(n, n_te, d, seed=n + d)
        print(f"== both routes fit: {n} x {d} ({tr.nbytes / 1e9:.2f} GB host fp32), lower_dim={k}, whitening=True, "
              f"{'Gram' if n <= d else 'covariance'} route, in-memory footprint "
              f"{u._pca_in_memory_bytes(n, d, n_te) / 1e9:.1f} GB")
        run(tr, te, k)                                             # warm-up of both routes
        run(tr, te, k, forced(n, d, n_te))
        times, diffs = {"in-memory": [], "streamed": []}, []
        for _ in range(args.reps):
            w0, (a_tr, a_te), _ = run(tr, te, k)
            w1, (b_tr, b_te), _ = run(tr, te, k, forced(n, d, n_te))
            times["in-memory"].append(w0)
            times["streamed"].append(w1)
            diffs.append(max(float(np.abs(a_tr - b_tr).max()), float(np.abs(a_te - b_te).max())))
            scale = max(float(np.abs(a_tr).max()), float(np.abs(a_te).max()))
        print(f"   median of {args.reps}: in-memory {statistics.median(times['in-memory']):.2f} s, streamed "
              f"{statistics.median(times['streamed']):.2f} s (each: {times})")
        print(f"   max |streamed - in-memory| = {max(diffs):.3e} (outputs up to {scale:.3e}, relative "
              f"{max(diffs) / scale:.2e})")
        st = Stages()
        wall, _, walls = run(tr, te, k, forced(n, d, n_te), st)
        report("streamed, staged", n, d, wall, walls, st)
        del tr, te
    if args.large:
        n, d = map(int, args.large.split("x"))
        tr, te = spectrum_rows(n, n_te, d, seed=1)
        budget = u._device_budget(dev)
        print(f"== only the stream fits: {n} x {d} ({tr.nbytes / 1e9:.2f} GB host fp32), lower_dim={k}, "
              f"whitening=True; in-memory footprint {u._pca_in_memory_bytes(n, d, n_te) / 1e9:.1f} GB, device budget "
              f"{budget / 1e9:.1f} GB, plan {u._pca_plan(n, d, n_te, budget, u._STAGE_BYTES)}")
        st = Stages()
        wall, (o_tr, o_te), walls = run(tr, te, k, None, st)
        report("streamed", n, d, wall, walls, st)
        print(f"   outputs {tuple(o_tr.shape)} {tuple(o_te.shape)}, finite: {bool(np.isfinite(o_tr).all())}")


if __name__ == "__main__":
    main()
