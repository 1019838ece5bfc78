"""Measure a vocabulary-size sweep fitted with fit_vocabularies against one VLAD.fit per vocabulary, on the GPU.

    python tools/bench_fit_sweep.py [--rows 4000000] [--dim 1536] [--ks 32 64 128 256] [--max-iter 8] [--reps 3]
                                    [--modes memory streamed] [--json out.json]

For each mode the two arms alternate, --reps times each, from the same numpy seed: the sequential arm calls
VLAD(K).fit(rows) for every K in turn, the shared arm calls fit_vocabularies once.  "memory" passes device rows;
"streamed" passes host rows with the device budget set to zero, so every round crosses the host link in every
iteration (fully streamed).  Every member's Lloyd loop is capped at --max-iter iterations (tol stays 1e-4), because
a full sweep from host rows takes minutes per run; the cap applies to both arms alike.  The centres of the two arms
must be bit-identical in every run.

Reported per mode: the median wall time per sweep of each arm and their ratio; the shared arm's time per iteration
while all members are active and the sequential arm's per-iteration time summed over the vocabularies (the spacing of
the iterations after the first); the iterations each member ran.  The rows are clustered (64 seeded centres plus
noise), generated on the device.  The card, its power limit and the SM clock sampled during the timed runs are
printed beside the results.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from anyloc_b200 import _lib, utilities as u  # noqa: E402


def smi(query):
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={query}",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


class ClockSampler:
    """samples the SM clock every half second while active"""

    def __init__(self):
        self.samples, self.on = [], False

    def __enter__(self):
        self.on = True
        self.th = threading.Thread(target=self.run, daemon=True)
        self.th.start()
        return self

    def run(self):
        while self.on:
            v = smi("clocks.sm").split()
            if v and v[0].isdigit():
                self.samples.append(int(v[0]))
            time.sleep(0.5)

    def __exit__(self, *exc):
        self.on = False
        self.th.join()


def device_rows(R, D, seed=0, n_centres=64, block=1 << 18):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn(n_centres, D, device="cuda", generator=g)
    X = torch.empty(R, D, device="cuda")
    for i in range(0, R, block):
        n = min(block, R - i)
        idx = torch.randint(0, n_centres, (n,), device="cuda", generator=g)
        X[i:i + n] = centres[idx] + 0.8 * torch.randn(n, D, device="cuda", generator=g)
    return X


class Passes:
    """timestamps and member sizes of every Lloyd iteration: _finalize_multi (shared arm), or _KMeans._update and
    _finalize (sequential arm, in memory and streamed)"""

    def __init__(self, arm):
        self.t, self.arm = [], arm

    def __enter__(self):
        self.saved = (u._finalize_multi, u._KMeans._update, u._finalize)
        fm, upd, fin = self.saved

        def finalize_multi(c, R, ws):
            self.t.append((time.perf_counter(), tuple(ci.shape[0] for ci in c)))
            return fm(c, R, ws)

        def update(km, x, labels, c):
            self.t.append((time.perf_counter(), (c.shape[0],)))
            return upd(km, x, labels, c)

        def finalize(c, R, c_next, err, ws):
            self.t.append((time.perf_counter(), (c.shape[0],)))
            return fin(c, R, c_next, err, ws)
        if self.arm == "multi":
            u._finalize_multi = finalize_multi
        else:
            u._KMeans._update, u._finalize = update, finalize
        return self

    def __exit__(self, *exc):
        u._finalize_multi, u._KMeans._update, u._finalize = self.saved


def run_arm(arm, X, ks):
    np.random.seed(0)
    vl = [u.VLAD(K) for K in ks]
    torch.cuda.synchronize()
    with Passes(arm) as p:
        t0 = time.perf_counter()
        if arm == "seq":
            for v in vl:
                v.fit(X)
        else:
            u.fit_vocabularies(vl, X)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    return wall, [v.c_centers for v in vl], p.t


def per_iteration(arm, t, ks):
    """-> (seconds per iteration with every member active, iterations per member)"""
    if arm == "multi":
        full = [ti for ti, kk in t if len(kk) == len(ks)]
        step = float(np.median(np.diff(full))) if len(full) > 1 else float("nan")
        return step, {K: sum(K in kk for _, kk in t) for K in ks}
    step, its = 0.0, {}
    for K in ks:
        tk = [ti for ti, kk in t if kk == (K,)]
        its[K] = len(tk)
        step += float(np.median(np.diff(tk))) if len(tk) > 1 else float("nan")
    return step, its


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--ks", type=int, nargs="+", default=[32, 64, 128, 256])
    ap.add_argument("--max-iter", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--modes", nargs="+", default=["memory", "streamed"])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fit_sweep needs a CUDA device")
    _lib.load()
    defaults = list(u._KMeans.__init__.__defaults__)
    defaults[0] = a.max_iter                                   # max_iter of every member's k-means
    u._KMeans.__init__.__defaults__ = tuple(defaults)
    print(f"gpu {smi('name')}, power limit {smi('power.limit')}, max SM clock {smi('clocks.max.sm')}")
    Xd = device_rows(a.rows, a.dim)
    out = {"gpu": smi("name"), "power_limit": smi("power.limit"), "rows": a.rows, "dim": a.dim, "ks": a.ks,
           "max_iter": a.max_iter, "modes": {}}
    for mode in sorted(a.modes):                           # "memory" first: "streamed" frees the device rows
        if mode == "streamed":
            X = Xd.cpu()
            del Xd
            torch.cuda.empty_cache()
            u._device_budget = lambda dev, release_cache=True: 0
        else:
            X = Xd
        res = {"seq": [], "multi": []}
        run_arm("multi", X, a.ks[:1])                          # warm-up: module loads and workspace allocations
        with ClockSampler() as clk:
            for rep in range(a.reps):
                runs = {}
                for arm in ("seq", "multi") if rep % 2 == 0 else ("multi", "seq"):
                    runs[arm] = run_arm(arm, X, a.ks)
                same = all(torch.equal(p, q) for p, q in zip(runs["seq"][1], runs["multi"][1]))
                for arm in runs:
                    step, its = per_iteration(arm, runs[arm][2], a.ks)
                    res[arm].append((runs[arm][0], step, its, same))
                print(f"{mode} rep {rep}: seq {runs['seq'][0]:.2f} s, shared {runs['multi'][0]:.2f} s, "
                      f"centres bit-identical {same}", flush=True)
        m = {}
        for arm in res:
            m[arm] = {"wall_s": float(np.median([r[0] for r in res[arm]])),
                      "iter_s_all_active": float(np.median([r[1] for r in res[arm]])),
                      "iterations": res[arm][-1][2]}
        m["ratio_shared_over_seq"] = m["multi"]["wall_s"] / m["seq"]["wall_s"]
        m["bit_identical"] = all(r[3] for r in res["multi"])
        m["sm_clock_mhz_median"] = float(np.median(clk.samples)) if clk.samples else None
        out["modes"][mode] = m
        print(f"{mode}: sweep seq {m['seq']['wall_s']:.2f} s, shared {m['multi']['wall_s']:.2f} s "
              f"(x{m['ratio_shared_over_seq']:.3f}); per iteration, all members active: seq (sum over K) "
              f"{1e3 * m['seq']['iter_s_all_active']:.1f} ms, shared {1e3 * m['multi']['iter_s_all_active']:.1f} ms; "
              f"iterations seq {m['seq']['iterations']} shared {m['multi']['iterations']}; "
              f"bit-identical {m['bit_identical']}; SM clock {m['sm_clock_mhz_median']} MHz", flush=True)
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
