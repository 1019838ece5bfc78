"""Every (layer, facet) output of the single-format ViT forwards (precision "bf16" and "f16x1") against the same model
in fp64, calibrated against an fp64 emulation of each precision's rounding points; and the fp16-range guard of f16x1 at
each of its rounding points.

tests/test_vit_bf16_gpu.py and tests/test_vit_f16x1_gpu.py hold one layer per model to torch.autocast by statistics over
the whole output.  That lets through an error confined to a few rows (an M tail, the cls or register rows), an error at
another layer or facet, and a rounding point that is wrong by a small factor (autocast rounds elsewhere, and the ratio
to it swings from 0.7x to 1.4x from one output to the next).  Here, as in tests/test_vit_accuracy_gpu.py, each output f
of a forward and its fp64 reference f64 give
  worst row  max_r |f_r - f64_r| / |f64_r|      and      RMS  |f - f64|_F / |f64|_F,
and the control is emulated(): the restated model in fp64, rounded exactly where the precision rounds (DESIGN 4.8,
4.10).  Weights: every weight matrix, the patch embedding included, as bf16_rn(w), or for f16x1 as fp16(s_w w) / s_w
with s_w = 2^floor(log2(16384 / max|w|)) per matrix.  Rounded values: the im2col pixels, both LayerNorm outputs, q / k /
v where they feed the attention, the attention output and the GELU / SwiGLU output, to bf16_rn(v), or for f16x1 to
fp16(8 v) / 8 (fp16 subnormals and overflow kept).  P is rounded as the kernel rounds it (bf16_rn(p), fp16(1024 p) /
1024) and the softmax denominator sums the unrounded p.  Left unrounded: the tapped q / k / v facets, the residual
stream, the LayerScale / residual adds and the features.  The emulation takes p relative to the row's final maximum,
where the kernel's online softmax rounds p relative to the running maximum of the key blocks read so far, and it sums
in fp64 where the kernel accumulates in fp32; both are left out, so ratios somewhat above 1 are normal.  Each statistic
must stay within KAPPA_* x the control's.  tests/test_vit_single_emulation_cpu.py checks the emulation itself.

Covered: the four MODELS of test_vit_accuracy_gpu.py (ViT-S at full depth, ViT-B with registers, ViT-L, ViT-G with
SwiGLU), random and trained-like weights (LayerScale 1e-5 .. 1, outlier channels x100), B = 2 images of 224^2 (T = 257),
98x154 (T = 78), 112^2 (T = 65, one row past a 64-row tile) and 14x28 (T = 3, far below one tile), both
(use_cls, norm_descs) settings and both precisions.  Every tap comes from one DinoV2MultiExtractFeatures call; one
DinoV2ExtractFeatures adds the deepest layer's value facet through its own N = D third of the qkv GEMM.

Measured on an H100 80GB HBM3 (700 W power limit), worst (row, RMS) ratio over the four images and both options
("taps": the DinoV2MultiExtractFeatures call, "single": the deepest value facet alone):
               random                                           trained-like
               bf16 taps   bf16 single f16x1 taps  f16x1 single  bf16 taps   bf16 single f16x1 taps  f16x1 single
  ViT-S        1.16, 1.02  1.06, 1.00  1.16, 1.03  1.01, 1.00    1.73, 1.27  1.03, 1.03  3.26, 1.98  1.49, 1.20
  ViT-B reg    1.07, 1.00  1.07, 1.00  1.07, 1.01  1.04, 1.00    1.09, 1.08  1.06, 1.08  1.68, 1.23  1.09, 1.10
  ViT-L        1.07, 1.01  1.02, 1.01  1.05, 1.01  1.01, 1.00    1.07, 1.04  1.00, 1.03  1.43, 1.15  1.42, 1.15
  ViT-G        1.05, 1.01  1.05, 1.00  1.08, 1.01  1.04, 1.00    1.19, 1.03  1.19, 1.03  1.25, 1.24  1.12, 1.05
KAPPA_* are at least 1.5x the worst (3.26 and 1.98, both at a trained-like ViT-S layer-10 query, T = 3).  The subnormal
case (test_f16x1_at_the_fp16_subnormal_floor) measured 1.13 / 1.08.  The file runs in about a minute on an H100.
Deliberately broken kernels, one per build, run on ViT-S with random weights (ViT-G for SwiGLU):
  - the last row of the last query tile dividing by the other half-row's l: 162 / 81 in f16x1, 20.6 / 10.3 in bf16;
  - the SwiGLU epilogue pairing x1_j with x2_(j+1) in the last column tile: 563 / 267 in f16x1, 70 / 33 in bf16;
  - P rounded to 8 significant bits in the f16x1 attention: 1.94 / 1.40, inside KAPPA_* (the worst rows are the
    layer-0 token of the 14x28 image; a random-init P is nearly uniform, so the lost bits average out);
  - a tanh GELU in the single-format epilogue: 1.17 / 1.04, inside KAPPA_*: the tanh form differs from erf's by at
    most ~1e-3 of |x|, below bf16's and fp16's rounding of the hidden layer.
So this file catches row-local and pairing faults by a wide margin; a wrong P rounding or GELU form that stays below the
format's own rounding is left to the kernel tests (tests/test_f16x1_kernels_gpu.py and tests/test_bf16_kernels_gpu.py
bound the attention and the GELU epilogue against fp64 of their operands).

The fp16-range guard: small crafted ViT-S models make one f16x1 rounding point overflow (|8 x| > 65504) while every
other point of the fp64 model stays below half the limit: the im2col pixels, the LayerNorm output, q / k / v and
the FFN hidden layer.  A later layer is tapped, so the Inf has to travel.  check_finite="sync" raises naming bf16,
"deferred" raises at the next call, "off" returns non-finite rows, bf16 stays finite.  The last case overflows a key
channel alone, in one sign and in 7 of 514 rows, against a query channel of -1e-3: its logits are -Inf.  Before the
wgmma softmax turned a live key's infinite logit into NaN, the key got p = 0, every row stayed finite and f16x1 raised
in no mode (measured on an H100; the fp64 emulation, which rounds the same way, is 16 % off fp64 at layer 2).  With
the fix every case raises, and "auto" (f16x3) switches to tf32x3 and returns its result bit for bit."""
import copy
import math
import time

import pytest
import torch

from oracle import dinov2_restated as dr
from tests.test_vit_accuracy_gpu import (FACETS, IMAGES, MODELS, OPTS, finish, forward_taps, image, measure,
                                         model_of, report)

pytestmark = pytest.mark.gpu

KAPPA_ROW = 5.0
KAPPA_RMS = 3.0
HWS = list(IMAGES.values()) + [(14, 28)]
PRECISIONS = ("bf16", "f16x1")
POINTS = ("pixels", "ln", "qkv", "attn", "hidden")       # the rounded activations, in forward order
F16_MAX = 65504.0
ACT = 8.0                                                 # f16x1 stores 8 x for an activation x
P_SCALE = 1024.0                                          # ... and 1024 p for the attention's P


def bf16_rn(x):
    return x.to(torch.bfloat16).to(x.dtype)


def f16_scaled(x, s):
    """fp16(s x) / s: the value whose fp16 word of s x f16x1 stores; fp16 subnormals and overflow are kept"""
    return (x * s).to(torch.float16).to(x.dtype) / s


def f16_weight_scale(w):
    """vit.VitWeights' per-matrix scale of the fp16 formats: max |s_w w| in (8192, 16384]"""
    amax = float(w.abs().max())
    return 2.0 ** math.floor(math.log2(16384.0 / amax)) if amax > 0 else 1.0


def rounding(precision):
    """{point: the rounding f(x) there} of a precision: POINTS, "weight" (every weight matrix) and "p" (the attention's P)"""
    if precision == "bf16":
        return dict.fromkeys(POINTS + ("weight", "p"), bf16_rn)
    rnd = dict.fromkeys(POINTS, lambda x: f16_scaled(x, ACT))
    rnd["weight"] = lambda w: f16_scaled(w, f16_weight_scale(w))
    rnd["p"] = lambda p: f16_scaled(p, P_SCALE)
    return rnd


def identity():
    return dict.fromkeys(POINTS + ("weight", "p"), lambda x: x)


def emulated(model, rnd):
    """an fp64 copy of the restated model that applies rnd[point] at each rounding point of a single-format forward"""
    m = copy.deepcopy(model).double()
    lins = [m.patch_embed.proj]
    m.patch_embed.proj.register_forward_pre_hook(lambda mod, a: (rnd["pixels"](a[0]),))
    for blk in m.blocks:
        ffn = blk.mlp
        lin_in, lin_out = (ffn.fc1, ffn.fc2) if hasattr(ffn, "fc1") else (ffn.w12, ffn.w3)
        attn = blk.attn
        lins += [attn.qkv, attn.proj, lin_in, lin_out]
        for lin in (attn.qkv, lin_in):                         # LayerNorm outputs
            lin.register_forward_pre_hook(lambda mod, a: (rnd["ln"](a[0]),))
        attn.proj.register_forward_pre_hook(lambda mod, a: (rnd["attn"](a[0]),))
        lin_out.register_forward_pre_hook(lambda mod, a: (rnd["hidden"](a[0]),))

        def fwd(x, attn=attn):
            B, N, C = x.shape
            qkv = rnd["qkv"](attn.qkv(x)).reshape(B, N, 3, attn.num_heads, C // attn.num_heads).permute(2, 0, 3, 1, 4)
            q, k, v = qkv[0] * attn.scale, qkv[1], qkv[2]
            s = q @ k.transpose(-2, -1)
            a = s.softmax(dim=-1)
            # P as the kernel rounds it, over the sum of the unrounded p: a + (rnd(p) - p) / l ~ rnd(p) / l, and exactly
            # the restated model's softmax when rnd is the identity
            p = torch.exp(s - s.amax(dim=-1, keepdim=True))
            a = a + (rnd["p"](p) - p) / p.sum(dim=-1, keepdim=True)
            return attn.proj((a @ v).transpose(1, 2).reshape(B, N, C))
        attn.forward = fwd
    with torch.no_grad():
        for lin in lins:
            lin.weight.copy_(rnd["weight"](lin.weight))
    return m


def recording(rnd, seen, inputs=False):
    """rnd with every point's values (its inputs, or its outputs) appended to seen[point]"""
    def wrap(point, f):
        def g(x):
            y = f(x)
            seen.setdefault(point, []).append((x if inputs else y).detach())
            return y
        return g
    return {point: wrap(point, f) for point, f in rnd.items()}


def peaks(model, img):
    """{point: max |x| over the fp64 forward} of every activation rounding point"""
    seen = {}
    with torch.no_grad():
        emulated(model, recording(identity(), seen, inputs=True))(img.double())
    return {p: max(float(x.abs().max()) for x in seen[p]) for p in POINTS}


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def check_taps(u, name, model, hws, label, weights, precisions=PRECISIONS):
    """ACC lines, and the cases over KAPPA_*, of every precision and image of one model"""
    depth = len(model.blocks)
    taps = [(l, f) for l in range(depth) for f in FACETS]
    sd = model.state_dict()
    exts = {}
    for precision in precisions:
        multi = u.DinoV2MultiExtractFeatures(name, taps, device="cuda", weights=sd, precision=precision)
        single = u.DinoV2ExtractFeatures(name, depth - 1, "value", device="cuda", weights=sd, precision=precision)
        assert multi.precision == single.precision == precision
        exts[precision] = (multi, single)
    bad = []
    for hw in hws:
        img = image(hw)
        r64 = forward_taps(copy.deepcopy(model).double(), img.double())        # shared by both precisions
        img_d = img.cuda()
        for precision, (multi, single) in exts.items():
            emu = [forward_taps(emulated(model, rounding(precision)), img.double())]

            def every_tap(use_cls, norm, multi=multi):
                multi.use_cls, multi.norm_descs = use_cls, norm
                return multi(img_d)

            def deepest_value(use_cls, norm, single=single):
                single.use_cls, single.norm_descs = use_cls, norm
                return {(depth - 1, "value"): single(img_d)}

            for what, outs_of in (("taps", every_tap), ("single", deepest_value)):
                worst = measure(outs_of, r64, emu, OPTS)
                case = f"{label}|{weights}|{precision}|{what}|{hw[0]}x{hw[1]}"
                report(case, worst)
                if worst["row"][0] > KAPPA_ROW or worst["rms"][0] > KAPPA_RMS:
                    bad.append((case, worst))
    return bad


@pytest.mark.parametrize("weights", ["random", "trained"])
@pytest.mark.parametrize("key", list(MODELS))
def test_every_tap_against_fp64(u, key, weights):
    t0 = time.perf_counter()
    bad = check_taps(u, MODELS[key][0], model_of(key, weights), HWS, key, weights)
    print(f"TIME|{key}|{weights}|{time.perf_counter() - t0:.1f} s")
    assert not bad, bad


SUB_BLOCK, SUB_SCALE = 5, 4e-6
F16_SUBNORMAL = 2.0 ** -14            # the smallest normal fp16: 8 y below it is an fp16 subnormal


def subnormal_model():
    """ViT-S with block SUB_BLOCK's LayerNorm gains and biases, and the qkv / fc1 biases, scaled by SUB_SCALE: most of
    that block's f16x1 operands (8 y) are fp16 subnormals"""
    m = dr.perturb(dr.build("dinov2_vits14", seed=0), seed=1)
    blk = m.blocks[SUB_BLOCK]
    with torch.no_grad():
        for p in (blk.norm1.weight, blk.norm1.bias, blk.norm2.weight, blk.norm2.bias, blk.attn.qkv.bias,
                  blk.mlp.fc1.bias):
            p.mul_(SUB_SCALE)
    return m.float().eval()


def flush_f16(x):
    """fp16(8 x) / 8 with fp16 subnormals flushed to zero, as a kernel that flushed them would round"""
    y = f16_scaled(x, ACT)
    return torch.where((ACT * y).abs() < F16_SUBNORMAL, torch.zeros_like(y), y)


def test_f16x1_at_the_fp16_subnormal_floor(u):
    """ViT-S with one block's normalised activations at ~SUB_SCALE (subnormal_model).  f16x1 rounds 8 y to fp16, so
    below |y| = 2^-17 its error is the absolute fp16 subnormal step, 2^-24 / 8 = 2^-27 in y, not a relative one.  That
    block's LayerNorm outputs are checked to be mostly fp16 subnormals, and every tap is held to the KAPPA_* of the other
    cases: the emulation models the subnormals because .half() keeps them.  The same emulation with fp16 subnormals
    flushed to zero (flush_f16 at every activation point) is measured against that bound too and must exceed it twice
    over, which is what a kernel that flushed them would show."""
    m = subnormal_model()
    hw = (112, 112)
    img = image(hw).double()
    seen = {}
    with torch.no_grad():
        emulated(m, recording(identity(), seen, inputs=True))(img)
    share = [float(((ACT * x).abs() < F16_SUBNORMAL).double().mean()) for x in seen["ln"]]   # norm1, norm2 per block
    print(f"SUBNORMAL|share of the LayerNorm outputs y with 8 y an fp16 subnormal, per block: "
          f"{[round(max(share[2 * b:2 * b + 2]), 3) for b in range(len(m.blocks))]}")
    assert min(share[2 * SUB_BLOCK:2 * SUB_BLOCK + 2]) > 0.5, share
    assert max(s for i, s in enumerate(share) if i // 2 != SUB_BLOCK) < 0.01, share
    bad = check_taps(u, "dinov2_vits14", m, [hw], "vits-subnormal", "random", ("f16x1",))
    flushed = rounding("f16x1")
    flushed.update(dict.fromkeys(POINTS, flush_f16))
    r64 = forward_taps(copy.deepcopy(m).double(), img)
    emu = [forward_taps(emulated(m, rounding("f16x1")), img)]
    ftz = forward_taps(emulated(m, flushed), img)
    worst = measure(lambda use_cls, norm: {t: finish(f, use_cls, norm) for t, f in ftz.items()}, r64, emu, OPTS)
    report(f"vits-subnormal|random|f16x1 flushing subnormals (emulated)|taps|{hw[0]}x{hw[1]}", worst)
    assert worst["row"][0] > 2 * KAPPA_ROW, worst
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- the fp16-range guard
GUARD_DEPTH, GUARD_LAYER, GUARD_HW = 3, 2, (224, 224)
LIMIT = F16_MAX / ACT                 # |x| beyond this overflows f16x1's fp16 word of 8 x
C_IN, C_OUT = 17, 70                  # a LayerNorm channel and the head-1 channel of q / k / v it feeds


def guard_case(point):
    """(model, image, the rounding point that overflows) of one crafted ViT-S: block 0 or 1 made to push exactly one
    f16x1 rounding point past the fp16 range"""
    m = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=GUARD_DEPTH), seed=1)
    img = image(GUARD_HW)
    D = 384
    blk = m.blocks[0]
    with torch.no_grad():
        if point == "pixels":                   # one pixel at 9000: 8 x = 72 000
            img[0, 1, 100, 100] = 9000.0
        elif point == "ln":                     # norm2 gain 4000 on one channel: |y| > LIMIT where |n| > 2
            m.blocks[1].norm2.weight[C_IN] = 4000.0
        elif point == "qkv":                    # one q bias at 9000: the logits saturate, the attention output does not
            blk.attn.qkv.bias[C_OUT] = 9000.0
        elif point == "hidden":                 # one fc1 bias at 9000: GELU keeps it
            blk.mlp.fc1.bias[C_OUT] = 9000.0
        else:                                   # "key": k channel C_OUT = 5 y, y = 400 n + 800 in [-400, 2000]: +Inf in
            blk.norm1.weight[C_IN], blk.norm1.bias[C_IN] = 400.0, 800.0      # the rows with n > 2; q channel -1e-3
            blk.attn.qkv.weight[D + C_OUT].zero_()
            blk.attn.qkv.weight[D + C_OUT, C_IN] = 5.0
            blk.attn.qkv.bias[D + C_OUT] = 0.0
            blk.attn.qkv.weight[C_OUT].zero_()
            blk.attn.qkv.bias[C_OUT] = -1e-3
    return m.float().eval(), img, "qkv" if point == "key" else point


GUARD_CASES = ("pixels", "ln", "qkv", "hidden", "key")


@pytest.mark.parametrize("case", GUARD_CASES)
def test_the_fp16_range_guard_at_each_rounding_point(u, case):
    from anyloc_b200 import _lib
    m, img, point = guard_case(case)
    pk = peaks(m, img)
    print(f"GUARD|{case}|peak |x| per point of the fp64 forward (limit {LIMIT:.0f}): " +
          ", ".join(f"{p} {v:.4g}" for p, v in pk.items()))
    assert pk[point] > LIMIT, pk
    assert all(v < LIMIT / 2 for p, v in pk.items() if p != point), pk
    if case == "key":
        # the key channel overflows in one sign, in some rows only; the query channel is small and negative
        m64 = copy.deepcopy(m).double()
        with torch.no_grad():
            qkv = m64.blocks[0].attn.qkv(m64.blocks[0].norm1(m64.prepare_tokens(img.double())))
        k, q = qkv[..., 384 + C_OUT], qkv[..., C_OUT]
        over = k > LIMIT
        assert 0 < int(over.sum()) < over.numel() // 10 and float(k.min()) > -LIMIT, (int(over.sum()), float(k.min()))
        assert float(q.max()) < 0 and float(q.min()) > -2e-3
    sd = m.state_dict()
    img_d = img.cuda()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", GUARD_LAYER, "token", device="cuda", weights=sd, precision="f16x1")
    with pytest.raises(_lib.AnylocError, match="precision='bf16'"):
        ext(img_d)
    ext.check_finite = "deferred"
    ext(img_d)
    with pytest.raises(_lib.AnylocError, match="precision='bf16'"):
        ext(img_d)
    ext.check_finite = "off"
    assert not bool(torch.isfinite(ext(img_d)).all())
    b16 = u.DinoV2ExtractFeatures("dinov2_vits14", GUARD_LAYER, "token", device="cuda", weights=sd, precision="bf16")
    assert bool(torch.isfinite(b16(img_d)).all())
    # "auto" (f16x3) ends with the tf32x3 result or raises, never a silent f16x3 result
    tf32 = u.DinoV2ExtractFeatures("dinov2_vits14", GUARD_LAYER, "token", device="cuda", weights=sd, precision="tf32x3")
    want = tf32(img_d)
    auto = u.DinoV2ExtractFeatures("dinov2_vits14", GUARD_LAYER, "token", device="cuda", weights=sd, precision="auto")
    try:
        got = auto(img_d)
    except _lib.AnylocError:
        return
    print(f"GUARD|{case}|auto ran {auto.precision}")
    assert auto.precision == "tf32x3" and torch.equal(got, want)
