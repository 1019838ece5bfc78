"""The fp64 emulation of the single-format forwards (tests/test_vit_single_accuracy_gpu.emulated), without a GPU: with
every rounding replaced by the identity it is the fp64 model bit for bit, so its hooks change nothing but the rounding;
every value it rounds lies on the format's grid, fp16 subnormals included, and the f16x1 weights follow the per-matrix
scale rule; and its error against fp64 sits where each format's precision puts it."""
import copy

import pytest
import torch

from tests.test_vit_accuracy_gpu import MODELS, forward_taps, image, model_of
from tests.test_vit_single_accuracy_gpu import (ACT, F16_SUBNORMAL, P_SCALE, POINTS, emulated, f16_scaled,
                                                f16_weight_scale, identity, recording, rounding, subnormal_model)

HW = (28, 42)                   # T = 7: the fp64 forwards of every model stay quick


def on_bf16_grid(x):
    """x is an fp32 value with the low 16 bits of its word zero (or +-Inf)"""
    f = x.float()
    return bool((f.double() == x).all()) and bool(((f.view(torch.int32) & 0xFFFF) == 0).all())


def on_f16_grid(v):
    """v is an fp16 value: 11 significant bits at or above 2^-14, a multiple of 2^-24 below, or +-Inf"""
    fin = torch.isfinite(v)
    f = v[fin].float()
    if not bool((f.double() == v[fin]).all()) or bool((f.abs() > 65504).any()):
        return False
    normal = f.abs() >= F16_SUBNORMAL
    return bool(((f[normal].view(torch.int32) & 0x1FFF) == 0).all()) and \
        bool((f[~normal].double() * 2.0 ** 24 == torch.round(f[~normal].double() * 2.0 ** 24)).all())


@pytest.mark.parametrize("key", list(MODELS))
def test_identity_rounding_is_the_fp64_model_bit_for_bit(key):
    m = model_of(key, "random")
    img = image(HW).double()
    want = forward_taps(copy.deepcopy(m).double(), img)
    got = forward_taps(emulated(m, identity()), img)
    assert want.keys() == got.keys()
    for tap in want:
        assert torch.equal(got[tap], want[tap]), tap


def test_f16_rounding_keeps_subnormals_and_overflow():
    k = torch.arange(-3000, 3000, dtype=torch.float64)
    x = k * 2.0 ** -27 / 3                      # 8 x spans the fp16 subnormals, 2^-24 apart, and a third of a step
    want = torch.round(x * 2.0 ** 27) * 2.0 ** -27          # round half to even on the subnormal grid
    assert torch.equal(f16_scaled(x, ACT), want)
    assert bool((f16_scaled(x, ACT) != 0).sum() > 5000)
    big = torch.tensor([8187.0, 8191.0, -8200.0, 1e6], dtype=torch.float64)
    assert f16_scaled(big, ACT).tolist() == [8188.0, float("inf"), float("-inf"), float("inf")]


@pytest.mark.parametrize("precision", ["bf16", "f16x1"])
@pytest.mark.parametrize("key", ["vits", "vitg"])
def test_rounded_values_lie_on_the_grid(key, precision):
    m = model_of(key, "trained")
    seen = {}
    with torch.no_grad():
        emu = emulated(m, recording(rounding(precision), seen))
        emu(image(HW).double())
    assert set(seen) == set(POINTS + ("weight", "p"))
    for point, vals in seen.items():
        for v in vals:
            if precision == "bf16":
                assert on_bf16_grid(v), point
            elif point == "weight":
                continue
            else:
                assert on_f16_grid(v * (P_SCALE if point == "p" else ACT)), point
    # the weights: every matrix of the original model rounded by its own rule
    orig = dict(m.named_parameters())
    for name, w in emu.named_parameters():
        if not name.endswith("weight") or w.dim() < 2:
            continue
        w0 = orig[name].detach().double()
        if precision == "bf16":
            assert torch.equal(w, w0.to(torch.bfloat16).double()), name
            continue
        s = f16_weight_scale(w0)
        assert 8192 < float(w0.abs().max()) * s <= 16384, name
        assert on_f16_grid(w.detach() * s) and torch.equal(w, (w0 * s).half().double() / s), name
        assert float(((w - w0).abs() / w0.abs().clamp_min(1e-30))[w0.abs() * s >= F16_SUBNORMAL].max()) <= 2.0 ** -11


def test_f16x1_subnormal_model_rounds_onto_the_subnormal_grid():
    """the floor test's model: most of block 5's f16x1 LayerNorm operands are fp16 subnormals, on their grid"""
    m = subnormal_model()
    seen = {}
    with torch.no_grad():
        emulated(m, recording(rounding("f16x1"), seen))(image((56, 56)).double())
    ln = seen["ln"][10:12]                    # block 5's norm1 and norm2 outputs
    for v in ln:
        assert on_f16_grid(ACT * v)
        sub = (ACT * v).abs() < F16_SUBNORMAL
        assert float(sub.double().mean()) > 0.5
        assert int(((ACT * v)[sub] != 0).sum()) > 0.4 * sub.numel()      # mostly subnormal, not flushed to zero


def rel_rms(a, b):
    return float((a - b).norm() / b.norm())


def test_emulation_error_sits_in_each_formats_band():
    """per rounded operand, the relative RMS rounding error is about 0.42 u, u = 2^-8 for bf16 (8 significant bits) and
    2^-11 for fp16 (11; measured 0.42 u for both on ViT-S); at the taps, the f16x1 emulation's RMS error against fp64
    is about 8x below bf16's (measured 7.9x; the existing GPU files measured 7.95x and more for the kernels)"""
    m = model_of("vits", "random")
    img = image((56, 70)).double()
    band = {}
    for precision in ("bf16", "f16x1"):
        xs, ys = {}, {}
        with torch.no_grad():
            emulated(m, recording(rounding(precision), xs, inputs=True))(img)
            emulated(m, recording(rounding(precision), ys))(img)
        for point in POINTS:
            x, y = torch.cat([v.flatten() for v in xs[point]]), torch.cat([v.flatten() for v in ys[point]])
            e = rel_rms(y, x)
            unit = 2.0 ** -8 if precision == "bf16" else 2.0 ** -11
            assert 0.3 * unit < e < 0.55 * unit, (precision, point, e)
            band[(precision, point)] = e
        r64 = forward_taps(copy.deepcopy(m).double(), img)
        emu = forward_taps(emulated(m, rounding(precision)), img)
        band[precision] = max(rel_rms(emu[t], r64[t]) for t in r64)
        assert band[precision] < (2.0 ** -5 if precision == "bf16" else 2.0 ** -8), band
    print(band)
    assert band["bf16"] > 6 * band["f16x1"], band
