"""Pre-processing of differently sized uint8 photos, two ways on the same seeded images:
  loop    one preprocess_images call per photo -- what a caller without list input runs
  list    one preprocess_images call on the whole list (anyloc_preprocess_u8_varlen)
Mixes of seeded random uint8 photos:
  demo     16 photos from 4032x3024 down to 1280x720, portrait and landscape; max_side=1024, bicubic (the reference
           demo's rule, demo/anyloc_vlad_generate.py:160-185)
  dataset  32 photos of mixed sizes; resize=(480, 640), bilinear (the dataset loader, dvgl_benchmark/datasets_ws.py)
Each arm runs on host inputs (uint8 tensors in ordinary host memory, as decoded photos arrive) and on device inputs.
The list arm's outputs are checked bit-identical to the loop arm's before any timing; each arm is warmed up, then
timed over --rounds rounds with the arms alternating inside each round (host clock around a device synchronise); the
median is reported with the source bytes it read per second.

Also, on the demo mix with device inputs: the single-image resize kernel (anyloc_preprocess_resize_u8, one launch per
photo) against the tiled list kernel on the same photos and outputs, timed with CUDA events over --reps launches of
each; and the share of pre-processing in "list pre-processing + ViT-G/14 layer 31 value list extraction" (random-init
weights, f16x3, the fp16-range check off).

Prints the card, its power limit and clocks, then one JSON line per result; writes nothing unless --out is given.

    python tools/bench_preprocess_list.py [--rounds 5] [--reps 10] [--no-vit] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEMO_SIZES = [(3024, 4032), (4032, 3024), (2268, 4032), (4032, 2268), (2448, 3264), (3264, 2448), (1080, 1920),
              (720, 1280)]
DATASET_SIZES = [(480, 640), (720, 1280), (1080, 1920), (600, 800), (375, 500), (1536, 2048), (640, 480), (333, 517)]
MIXES = {
    "demo": (DEMO_SIZES, 16, dict(max_side=1024, interpolation="bicubic")),
    "dataset": (DATASET_SIZES, 32, dict(resize=(480, 640), interpolation="bilinear")),
}


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else
            f"unavailable ({r.stderr.strip()})"}


def mix_photos(sizes, n, seed):
    import numpy as np
    import torch
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (*sizes[i % len(sizes)], 3), dtype=np.uint8)) for i in range(n)]


def timed(fns, rounds):
    """median / min / max seconds of each fn, the fns alternating inside each round"""
    import torch
    times = {a: [] for a in fns}
    for r in range(rounds):
        for arm in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fns[arm]()
            torch.cuda.synchronize()
            times[arm].append(time.perf_counter() - t0)
    return {a: (sorted(t)[len(t) // 2], min(t), max(t)) for a, t in times.items()}


def kernel_comparison(u, lib, photos, kw, reps):
    """the single-image kernel (one launch per photo) against the tiled list kernel, same device photos and outputs,
    CUDA events over `reps` passes of each, alternating"""
    import torch
    from anyloc_b200 import _lib
    dev = torch.device("cuda", 0)
    xs = [x.to(dev) for x in photos]
    geo = u._list_geometry([tuple(x.shape[:2]) for x in xs], 14, None, kw["max_side"])
    interp = u._INTERP[kw["interpolation"]]
    outs = [torch.empty(3, g[5], g[6], device=dev) for g in geo]
    m3 = (C.c_float * 3)(*u.IMAGENET_MEAN)
    s3 = (C.c_float * 3)(*u.IMAGENET_STD)
    sizes = [3 * g[5] * g[6] for g in geo]
    flat = torch.empty(sum(sizes), device=dev)
    n = len(xs)
    res = [k for k, g in enumerate(geo) if g[2]]
    crop = [k for k, g in enumerate(geo) if not g[2]]
    offs = [sum(sizes[:k]) for k in range(n)]

    def varlen(idx, it):
        m = len(idx)

        def ints(f):
            return (C.c_int * m)(*[int(f(k)) for k in idx])
        return lib.anyloc_preprocess_u8_varlen(
            m, (C.c_void_p * m)(*[xs[k].data_ptr() for k in idx]), ints(lambda k: xs[k].shape[0]),
            ints(lambda k: xs[k].shape[1]), ints(lambda k: geo[k][0]), ints(lambda k: geo[k][1]), it,
            ints(lambda k: geo[k][3]), ints(lambda k: geo[k][4]), ints(lambda k: geo[k][5]), ints(lambda k: geo[k][6]),
            m3, s3, _lib.ptr(flat), (C.c_int64 * m)(*[offs[k] for k in idx]), _lib.stream_ptr())

    def single():
        for k in range(n):
            x, g = xs[k], geo[k]
            if g[2]:
                rc = lib.anyloc_preprocess_resize_u8(_lib.ptr(x), 1, x.shape[0], x.shape[1], g[0], g[1], interp, g[3],
                                                     g[4], g[5], g[6], m3, s3, _lib.ptr(outs[k]), _lib.stream_ptr())
            else:
                rc = lib.anyloc_preprocess_u8(_lib.ptr(x), 1, x.shape[0], x.shape[1], g[3], g[4], g[5], g[6], m3, s3,
                                              _lib.ptr(outs[k]), _lib.stream_ptr())
            _lib.check(rc, "single-image kernel")

    def tiled():
        if res:
            _lib.check(varlen(res, interp), "anyloc_preprocess_u8_varlen")
        if crop:
            _lib.check(varlen(crop, -1), "anyloc_preprocess_u8_varlen")

    single()
    tiled()
    torch.cuda.synchronize()
    if not all(torch.equal(flat[offs[k]:offs[k] + sizes[k]].view(outs[k].shape), outs[k]) for k in range(n)):
        raise SystemExit("tiled kernel output differs from the single-image kernel")
    ms = {"single_image_kernel": [], "tiled_kernel": []}
    for r in range(reps):
        for arm, fn in (("single_image_kernel", single), ("tiled_kernel", tiled))[::1 if r % 2 == 0 else -1]:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms[arm].append(a.elapsed_time(b))
    return {arm: sorted(t)[len(t) // 2] for arm, t in ms.items()}, len(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--mixes", default="demo,dataset")
    ap.add_argument("--no-vit", action="store_true", help="skip the ViT-G/14 share")
    ap.add_argument("--out", default=None, help="also write every result line to this JSON file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_preprocess_list times the GPU path and needs a CUDA device")
    from anyloc_b200 import _lib
    from anyloc_b200 import utilities as u
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card_info()
    print(json.dumps(info), flush=True)
    results = []

    def emit(line):
        line.update(info)
        results.append(line)
        print(json.dumps(line), flush=True)

    for mix in args.mixes.split(","):
        sizes, n, kw = MIXES[mix]
        photos = mix_photos(sizes, n, seed=1234)
        src_bytes = sum(x.numel() for x in photos)
        for where in ("host", "device"):
            imgs = photos if where == "host" else [x.to(dev) for x in photos]
            fns = {"loop": lambda: [u.preprocess_images(x[None], **kw)[0] for x in imgs],
                   "list": lambda: u.preprocess_images(imgs, **kw)}
            ref, out = fns["loop"](), fns["list"]()
            if not all(torch.equal(a, b) for a, b in zip(out, ref)):
                raise SystemExit(f"{mix}/{where}: list outputs are not bit-identical to the per-photo calls")
            del ref, out
            med = timed(fns, args.rounds)
            for arm in fns:
                emit({"mix": mix, "inputs": where, "arm": arm, "photos": n, "source_MB": round(src_bytes / 1e6, 1),
                      "median_ms": round(med[arm][0] * 1e3, 3), "min_ms": round(med[arm][1] * 1e3, 3),
                      "max_ms": round(med[arm][2] * 1e3, 3), "source_GB_per_s": round(src_bytes / med[arm][0] / 1e9, 2),
                      "list_bit_identical_to_loop": True, "loop_over_list": round(med["loop"][0] / med[arm][0], 3)})
            del imgs
        if mix == "demo":
            ms, nres = kernel_comparison(u, lib, photos, kw, args.reps)
            emit({"mix": mix, "inputs": "device", "what": "kernels", "photos": n, "resized": nres,
                  **{k: round(v, 3) for k, v in ms.items()},
                  "single_over_tiled": round(ms["single_image_kernel"] / ms["tiled_kernel"], 2),
                  "tiled_source_GB_per_s": round(src_bytes / ms["tiled_kernel"] / 1e6, 1)})
            if not args.no_vit:
                from anyloc_b200.vit import random_state_dict
                sd = random_state_dict("dinov2_vitg14", seed=0, device=dev, depth=32)
                ext = u.DinoV2ExtractFeatures("dinov2_vitg14", 31, "value", device=dev, weights=sd, precision="f16x3")
                ext.check_finite = "off"
                del sd
                for where in ("host", "device"):
                    imgs = photos if where == "host" else [x.to(dev) for x in photos]
                    pre = u.preprocess_images(imgs, **kw)
                    ext(pre)
                    fns = {"preprocess": lambda: u.preprocess_images(imgs, **kw), "extract": lambda: ext(pre),
                           "both": lambda: ext(u.preprocess_images(imgs, **kw))}
                    med = timed(fns, args.rounds)
                    emit({"mix": mix, "inputs": where, "what": "share in list preprocess + ViT-G/14 L31 value list",
                          "photos": n, **{f"{a}_ms": round(v[0] * 1e3, 2) for a, v in med.items()},
                          "preprocess_share": round(med["preprocess"][0] / med["both"][0], 4)})
                    del imgs, pre
                del ext
                torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
