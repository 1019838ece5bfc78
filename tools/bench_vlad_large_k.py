"""Time hard VLAD's sorted route (any vocabulary size) and a large-K VLAD.fit on the GPU.

    python tools/bench_vlad_large_k.py [--reps 20] [--fit-rows 200000] [--out results/vlad_large_k.json]

1. Inside accumulate3's envelope, c2 (B = 32, N = 529, D = 1536, K = 32) and c5 (B = 32, N = 1369, D = 1024, K = 128):
   anyloc_vlad_generate_prepared (accumulate3, what VLAD uses there) and anyloc_vlad_generate_sorted, alternated on
   the same inputs; their outputs must be bitwise equal.
2. K = 256 at N = 3942, D = 1536 (a demo 1024-px photo on ViT-G, B = 8) and K = 1024 at N = 2000, D = 1024 (B = 8):
   outside the envelope, the sorted route alone.  K = 1024 at N = 1369, D = 1024 (B = 8) still fits accumulate3's
   100 KB, so both routes are timed there.
3. VLAD(1024).fit on --fit-rows host rows of D = 1536 streamed in rounds (the fit is forced onto the streamed route
   by a budget of zero resident rounds), a fixed number of Lloyd iterations.
Times are CUDA-event medians per call after a warm-up.  Prints the card, its power limit and max SM clock beside the
results.
"""
import argparse
import json
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


def inputs(B, N, D, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, N, D, device="cuda", generator=g) * (0.5 + torch.rand(B, N, 1, device="cuda", generator=g))
    c = 0.5 * torch.nn.functional.normalize(torch.randn(K, D, device="cuda", generator=g), dim=1)
    return x.contiguous(), c.contiguous()


def call(lib, fn, x, c, blob, B, N, D, K, out, ws):
    _lib.check(fn(_lib.ptr(x), None, _lib.ptr(c), _lib.ptr(blob), blob.numel(), B, N, D, K, 0, 1, 1, _lib.ptr(out),
                  None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "generate")


def timed(f, reps):
    for _ in range(3):
        f()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def generate_case(lib, B, N, D, K, reps, with_acc3):
    x, c = inputs(B, N, D, K, seed=N + K)
    blob = torch.empty(lib.anyloc_vlad_prepared_bytes(D, K), dtype=torch.uint8, device="cuda")
    _lib.check(lib.anyloc_vlad_prepare(_lib.ptr(c), D, K, 0, _lib.ptr(blob), blob.numel(), _lib.stream_ptr()), "prep")
    res = {"B": B, "N": N, "D": D, "K": K, "route": lib.anyloc_vlad_generate_route(B, N, D, K)}
    out_s = torch.empty(B, K * D, device="cuda")
    ws_s = torch.empty(lib.anyloc_vlad_sorted_workspace_bytes(B, N, D, K), dtype=torch.uint8, device="cuda")
    sorted_f = lambda: call(lib, lib.anyloc_vlad_generate_sorted, x, c, blob, B, N, D, K, out_s, ws_s)
    if with_acc3:
        out_3 = torch.empty(B, K * D, device="cuda")
        ws_3 = torch.empty(lib.anyloc_vlad_workspace_bytes(B, N, D, K), dtype=torch.uint8, device="cuda")
        acc3_f = lambda: call(lib, lib.anyloc_vlad_generate_prepared, x, c, blob, B, N, D, K, out_3, ws_3)
        t3, ts = [], []
        for _ in range(3):                       # alternate the two routes
            t3.append(timed(acc3_f, reps))
            ts.append(timed(sorted_f, reps))
        torch.cuda.synchronize()
        res["bitwise_equal"] = bool(torch.equal(out_3, out_s))
        res["accumulate3_ms"] = [t[0] for t in t3]
        res["sorted_ms"] = [t[0] for t in ts]
    else:
        res["sorted_ms"] = [timed(sorted_f, reps)[0]]
    res["sorted_ms_per_image"] = min(res["sorted_ms"]) / B
    return res


def fit_case(rows, D, K, iters):
    g = torch.Generator().manual_seed(1)
    base = torch.randn(20_000, D, generator=g)
    X = base.repeat(-(-rows // base.shape[0]), 1)[:rows] + 0.01 * torch.randn(rows, 1, generator=g)
    saved = u._device_budget
    u._device_budget = lambda dev, release_cache=True: 0              # streamed, no resident round
    try:
        np.random.seed(0)
        v = u.VLAD(K)
        km_init = u._KMeans.__init__

        def init(self, *a, **k):
            km_init(self, *a, **k)
            self.max_iter, self.tol = iters, -1.0                    # a fixed number of iterations
        u._KMeans.__init__ = init
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v.fit(X)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        u._device_budget = saved
        u._KMeans.__init__ = km_init
    return {"rows": rows, "D": D, "K": K, "iterations": iters, "seconds": dt, "seconds_per_iteration": dt / iters}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--fit-rows", type=int, default=200_000)
    ap.add_argument("--fit-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    lib = _lib.load()
    res = {"gpu": torch.cuda.get_device_name(), "power_limit": smi("power.limit"), "max_sm_clock": smi("clocks.max.sm")}
    res["c2"] = generate_case(lib, 32, 529, 1536, 32, a.reps, True)
    res["c5"] = generate_case(lib, 32, 1369, 1024, 128, a.reps, True)
    res["K256_N3942"] = generate_case(lib, 8, 3942, 1536, 256, a.reps, False)
    res["K1024_N1369"] = generate_case(lib, 8, 1369, 1024, 1024, a.reps, True)       # still inside accumulate3
    res["K1024_N2000"] = generate_case(lib, 8, 2000, 1024, 1024, a.reps, False)
    res["fit_K1024"] = fit_case(a.fit_rows, 1536, 1024, a.fit_iters)
    res["sm_clock_after"] = smi("clocks.sm")
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
