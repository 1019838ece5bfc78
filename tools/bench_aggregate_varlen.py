"""Aggregation of differently sized images' features, the packed list route against the paths it replaces:
  padded  VLAD: the list zero-padded into one [B, max n, D] tensor with a Python copy per item, then the padded
          kernels with n_valid (VLAD.generate_multi(list) before the packed route)
          GeM: one pool_descriptors call per image (a list had no other way in)
  packed  VLAD.generate_multi(list) / pool_descriptors(list): the items' own buffer and a row table, one launch
          sequence per call
Features: ViT-G/14-sized rows (D = 1536) with the token counts preprocess_images(..., max_side=1024) gives photos of
mixed aspect ratios (portrait, landscape and panorama), as consecutive views of one buffer like ext(list) returns.
Lists of 16 and 64 images; hard VLAD at K = 32 and K = 256, soft VLAD at K = 32, GeM (p = 3).

The packed descriptors are checked bit-identical to the padded path's (GeM: to anyloc_pool on the padded batch with
n_valid) before any timing.  Each arm is warmed up, then timed over --rounds rounds with the arms alternating inside
each round (host clock around a device synchronise, the median reported); peak device memory
(torch.cuda.max_memory_allocated over the memory held before the call, the workspace pool emptied first) comes from
one more call of each arm.

Prints the card, its power limit and clocks, then one JSON line per result; writes nothing unless --out is given.

    python tools/bench_aggregate_varlen.py [--rounds 7] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (height, width) of the photos, cycled through a list: phone portrait / landscape, 16:9, and panoramas
PHOTO_SIZES = [(4032, 3024), (3024, 4032), (1080, 1920), (1920, 1080), (2000, 8000), (3264, 2448), (1500, 6000),
               (720, 1280)]
D = 1536


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unavailable ({r.stderr})"


def token_counts(u, n, patch=14, max_side=1024):
    out = []
    for i in range(n):
        h, w = PHOTO_SIZES[i % len(PHOTO_SIZES)]
        if max(h, w) > max_side:
            h, w = u.max_side_size(h, w, max_side)
        out.append((h // patch) * (w // patch))
    return out


def padded_generate(u, v, items, dev):
    """VLAD.generate_multi(list) before the packed route"""
    import torch
    n_max = max(q.shape[0] for q in items)
    feats = torch.zeros(len(items), n_max, items[0].shape[1], device=dev, dtype=torch.float32)
    for i, q in enumerate(items):
        feats[i, :q.shape[0]] = q
    n_valid = torch.tensor([q.shape[0] for q in items], dtype=torch.int32, device=dev)
    return v._run(feats, n_valid, dev)[0]


def timed(fn, torch):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def peak(fn, torch, L):
    L.workspaces.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--lists", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from anyloc_b200 import _lib as L
    from anyloc_b200 import utilities as u
    if not torch.cuda.is_available():
        raise SystemExit("bench_aggregate_varlen needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(f"[card] {card_info()}")
    results = []
    for n in a.lists:
        lens = token_counts(u, n)
        g = torch.Generator(device=dev).manual_seed(n)
        buf = torch.randn(sum(lens), D, device=dev, generator=g)
        items = list(buf.split(lens))
        cases = []
        for mode, K in (("hard", 32), ("hard", 256), ("soft", 32)):
            v = u.VLAD(K, vlad_mode=mode)
            v.kmeans = u._KMeans(K, mode="cosine")
            v.kmeans.centroids = v.c_centers = torch.nn.functional.normalize(
                torch.randn(K, D, generator=torch.Generator().manual_seed(K)), dim=1)
            v.desc_dim = D
            ref, got = padded_generate(u, v, items, dev), v.generate_multi(items)
            assert torch.equal(ref, got), f"{mode} K={K}: packed != padded"
            cases.append((f"vlad_{mode}_k{K}", lambda v=v: padded_generate(u, v, items, dev),
                          lambda v=v: v.generate_multi(items)))
        x = torch.zeros(n, max(lens), D, device=dev)
        for i, q in enumerate(items):
            x[i, :q.shape[0]] = q
        nv = torch.tensor(lens, dtype=torch.int32, device=dev)
        ref = torch.empty(n, D, device=dev)
        L.check(L.load().anyloc_pool(L.ptr(x), L.ptr(nv), n, max(lens), D, 2, 3.0, 0, L.ptr(ref), L.stream_ptr()),
                "anyloc_pool")
        assert torch.equal(ref, u.pool_descriptors(items, "gem")), "gem: packed != padded"
        del x
        cases.append(("gem", lambda: torch.cat([u.pool_descriptors(q[None], "gem") for q in items]),
                      lambda: u.pool_descriptors(items, "gem")))
        for name, padded_fn, packed_fn in cases:
            for _ in range(2):
                padded_fn(), packed_fn()
            tp, tk = [], []
            for _ in range(a.rounds):
                tp.append(timed(padded_fn, torch))
                tk.append(timed(packed_fn, torch))
            tp.sort(), tk.sort()
            r = {"case": name, "images": n, "rows": sum(lens), "max_rows": max(lens), "D": D,
                 "padded_ms": round(1e3 * tp[len(tp) // 2], 3), "packed_ms": round(1e3 * tk[len(tk) // 2], 3),
                 "padded_peak_mib": round(peak(padded_fn, torch, L) / 2 ** 20, 1),
                 "packed_peak_mib": round(peak(packed_fn, torch, L) / 2 ** 20, 1),
                 "bit_identical": True}
            r["speedup"] = round(r["padded_ms"] / r["packed_ms"], 2)
            print(json.dumps(r), flush=True)
            results.append(r)
    print(f"[card] {card_info()}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card_info(), "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
