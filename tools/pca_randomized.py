"""Measure reduce_pca(svd_solver="randomized") on the GPU.

    python tools/pca_randomized.py [--both 10000x49152] [--large 40000x49152,100000x49152] [--k 512] [--reps 2]

1. Where the exact fit also runs (--both, host fp32 rows with a decaying spectrum, 1000 test rows): svd_solver="full"
   and "randomized" alternately --reps times each in one process; the median wall time of each (host clock around the
   call, which ends in a device-to-host copy) and how far their top-32 projections differ.
2. Beyond the exact solver's limit (--large): the randomized fit on host rows, uploaded once, then forced to stream
   (an in-process budget override just under the upload's footprint), once each.
3. For each randomized run, per phase: the mean pass; the sketch and vt passes (CUDA events around each launch, summed;
   fp64 rate from 2 n d l flops per pass); LU, QR and SVD (events around each torch.linalg call); the projections (host
   clock).  Host rows are gathered into the pinned stages; the gather rate is over the gather time.
Prints the card, its power limit and max SM clock, read in the same run.
"""
import argparse
import os
import statistics
import sys
import time
from collections import defaultdict

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from anyloc_b200 import _lib, utilities as u  # noqa: E402
from pca_stream import smi, spectrum_rows  # noqa: E402

FP64_PEAK = 67e12


class Phases:
    """per-phase times, collected through wrappers of utilities' helpers and of torch.linalg"""

    def __init__(self):
        self.ev = defaultdict(list)
        self.flops = 0.0
        self.gather_s, self.gather_bytes, self.proj_s = 0.0, 0, 0.0

    def install(self):
        saved = [(u, "_pca_colsum"), (u, "_pca_accumulate"), (u._PcaRows, "gather"), (u, "_pca_project_streamed"),
                 (torch.linalg, "lu_factor"), (torch.linalg, "qr"), (torch.linalg, "svd")]
        real = {(o, a): getattr(o, a) for o, a in saved}

        def timed(name, fn):
            def run(*a, **kw):
                b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                b.record()
                r = fn(*a, **kw)
                e.record()
                self.ev[name].append((b, e))
                return r
            return run

        def acc(mode, x, mu, out, q=None):
            self.flops += 2 * x.shape[0] * x.shape[1] * q.shape[1]
            return timed("sketch / vt passes", real[(u, "_pca_accumulate")])(mode, x, mu, out, q)

        def gather(rows, dst, box):
            t = time.perf_counter()
            real[(u._PcaRows, "gather")](rows, dst, box)
            self.gather_s += time.perf_counter() - t
            self.gather_bytes += dst.numel() * 4

        def proj(*a):
            t = time.perf_counter()
            r = real[(u, "_pca_project_streamed")](*a)
            self.proj_s += time.perf_counter() - t
            return r
        u._pca_colsum = timed("mean", real[(u, "_pca_colsum")])
        u._pca_accumulate, u._PcaRows.gather, u._pca_project_streamed = acc, gather, proj
        for name in ("lu_factor", "qr", "svd"):
            setattr(torch.linalg, name, timed(name, real[(torch.linalg, name)]))

        def restore():
            for (o, a), f in real.items():
                setattr(o, a, f)
        return restore

    def ms(self, name):
        return sum(b.elapsed_time(e) for b, e in self.ev[name])


def run(tr, te, k, solver, budget=None, phases=None):
    """-> (wall seconds, outputs)"""
    real_budget = u._device_budget
    if budget is not None:
        u._device_budget = budget
    restore = phases.install() if phases else None
    try:
        np.random.seed(0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = u.reduce_pca(tr, te, k, svd_solver=solver)
        torch.cuda.synchronize()
        return time.perf_counter() - t, out
    finally:
        u._device_budget = real_budget
        if restore:
            restore()


def report(label, n, d, k, wall, ph):
    l, n_iter, _ = u._pca_randomized_params(n, d, k)
    pass_ms = ph.ms("sketch / vt passes")
    rate = ph.flops / (pass_ms / 1e3)
    print(f"   {label}: {wall:.2f} s end to end (l = {l}, n_iter = {n_iter}, {2 * n_iter + 2} passes)")
    print(f"     mean {ph.ms('mean'):.0f} ms; sketch / vt passes {pass_ms:.0f} ms for {ph.flops:.3e} flops = "
          f"{rate / 1e12:.2f} TFLOP/s fp64 ({100 * rate / FP64_PEAK:.0f} % of the 67 TFLOP/s data sheet); "
          f"LU {ph.ms('lu_factor'):.0f} ms, QR {ph.ms('qr'):.0f} ms, SVD {ph.ms('svd'):.0f} ms; "
          f"test-row projections {ph.proj_s * 1e3:.0f} ms (host clock)")
    if ph.gather_s:
        print(f"     host gather: {ph.gather_bytes / 1e9:.1f} GB in {ph.gather_s:.2f} s = "
              f"{ph.gather_bytes / ph.gather_s / 1e9:.1f} GB/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--both", default="10000x49152")
    ap.add_argument("--large", default="40000x49152,100000x49152")
    ap.add_argument("--k", type=int, default=512)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--test-rows", type=int, default=1000)
    args = ap.parse_args()
    dev = _lib.require_cuda()
    torch.cuda.set_device(dev)
    print(f"== {torch.cuda.get_device_name(dev)}; name, power limit, max SM clock: "
          f"{smi('name,power.limit,clocks.max.sm')}")
    n_te, k = args.test_rows, args.k
    for shape in filter(None, args.both.split(",")):
        n, d = map(int, shape.split("x"))
        tr, te = spectrum_rows(n, n_te, d, seed=n + d)
        print(f"== full and randomized: {n} x {d} ({tr.nbytes / 1e9:.2f} GB host fp32), lower_dim={k}")
        run(tr, te, k, "full")                                  # warm-up of both
        run(tr, te, k, "randomized")
        times = {"full": [], "randomized": []}
        for _ in range(args.reps):
            for solver in times:
                w, out = run(tr, te, k, solver)
                times[solver].append(w)
                if solver == "full":
                    f_tr, f_te = out
                else:
                    r_tr, r_te = out
        print(f"   median of {args.reps}: full {statistics.median(times['full']):.2f} s, randomized "
              f"{statistics.median(times['randomized']):.2f} s (each: {times})")
        for name, f, r in (("train", f_tr, r_tr), ("test", f_te, r_te)):
            f32, r32 = f[:, :32].astype(np.float64), r[:, :32].astype(np.float64)
            sign = np.sign((f32 * r32).sum(0))                  # the two fits may pick opposite component signs
            diff = np.abs(f32 - r32 * sign).max() / np.abs(f32).max()
            print(f"   top-32 projections, {name} rows: max |full - randomized| / max |full| = {diff:.2e}")
        ph = Phases()
        wall, _ = run(tr, te, k, "randomized", phases=ph)
        report("randomized, rows uploaded once", n, d, k, wall, ph)
        del tr, te
    for shape in filter(None, args.large.split(",")):
        n, d = map(int, shape.split("x"))
        tr, te = spectrum_rows(n, n_te, d, seed=1)
        l = u._pca_randomized_params(n, d, k)[0]
        budget = u._device_budget(dev)
        print(f"== randomized only: {n} x {d} ({tr.nbytes / 1e9:.2f} GB host fp32), lower_dim={k}; fit matrices "
              f"{u._pca_randomized_bytes(n, d, l) / 1e9:.2f} GB, device budget {budget / 1e9:.1f} GB, plan "
              f"{u._pca_randomized_plan(n, d, l, budget, u._STAGE_BYTES)}")
        ph = Phases()
        wall, (o_tr, o_te) = run(tr, te, k, "randomized", phases=ph)
        report("uploaded once", n, d, k, wall, ph)
        forced = u._pca_randomized_bytes(n, d, l) + 4 * n * d - 1
        ph = Phases()
        wall, (s_tr, s_te) = run(tr, te, k, "randomized", lambda dev, release_cache=True: forced, ph)
        report(f"streamed (budget {forced / 1e9:.1f} GB)", n, d, k, wall, ph)
        diff = max(float(np.abs(o_tr - s_tr).max()) / float(np.abs(o_tr).max()),
                   float(np.abs(o_te - s_te).max()) / float(np.abs(o_te).max()))
        print(f"   outputs {tuple(o_tr.shape)} {tuple(o_te.shape)}, finite {bool(np.isfinite(o_tr).all())}; "
              f"max |streamed - uploaded| relative {diff:.2e}")
        del tr, te


if __name__ == "__main__":
    main()
