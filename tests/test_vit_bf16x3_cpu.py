"""The bf16-pair precision (precision="bf16pair", ANYLOC_PAIR_BF16X3) without a GPU: the precision choice (argument and
$ANYLOC_B200_PRECISION, "auto" and the default never picking it), the C ABI's refusals (which return before anything
touches the device), the documented workspace sizes, and the fp64 emulation of the format that
tests/test_vit_bf16x3_gpu.py holds the kernels to.

The emulation (rounding_bf16x3 with tests/test_vit_single_accuracy_gpu.emulated): every value the forward rounds --
the weights, the im2col pixels, both LayerNorm outputs, q / k / v where they feed the attention, P, the attention output
and the GELU / SwiGLU output -- becomes the value of its bf16 pair, hi + lo with hi = bf16_rn(x), lo = bf16_rn(x - hi).
It leaves out the kernels' one other approximation, the dropped lo.lo term of each product, which is of the same
order (2^-16 relative) as the rounding it does model."""
import copy
import ctypes as C

import pytest
import torch

from anyloc_b200 import _lib, vit
from anyloc_b200 import utilities as u
from tests.test_vit_accuracy_gpu import forward_taps, image, model_of
from tests.test_vit_single_accuracy_gpu import POINTS, emulated, identity, recording, rounding

ARG, UNSUPPORTED = _lib.ERR["arg"], _lib.ERR["unsupported"]
FAKE = 4096                      # placeholder device pointer (16-byte aligned); every checked error returns first
X3 = _lib.PAIR["bf16pair"]


def bf16_pair(x):
    """hi + lo of the bf16 pair of x (round to nearest even, as .to(torch.bfloat16) and the kernels' cvt.rn round)"""
    hi = x.to(torch.bfloat16).to(x.dtype)
    return hi + (x - hi).to(torch.bfloat16).to(x.dtype)


def rounding_bf16x3():
    """{point: rounding} of the bf16-pair forward, in the form of tests/test_vit_single_accuracy_gpu.rounding()"""
    return dict.fromkeys(POINTS + ("weight", "p"), bf16_pair)


def test_format_constant():
    assert _lib.PAIR["bf16pair"] == 5 and "bf16pair" in u.PRECISIONS and "bf16pair" not in u._FP16_RANGE


def test_precision_choice(monkeypatch):
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    assert u.resolve_precision("bf16pair") == "bf16pair" and u.resolve_precision("bf16pair", "tc3") == "bf16pair"
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "bf16pair")
    assert u.resolve_precision(None) == "bf16pair"
    assert u.resolve_precision("f16x3") == "f16x3"          # the argument wins
    with pytest.raises(ValueError, match="tensor cores"):
        u.resolve_precision(None, "simt")
    with pytest.raises(ValueError, match="tensor cores"):
        u.resolve_precision("bf16pair", "simt")
    # "bf16x3" stays refused: tests/test_vit_bf16_cpu.py lists it among the names that are not precisions
    for bad in ("bf16x3", "BF16PAIR", "bf16pairs", "bf16_pair", "bf16x2"):
        with pytest.raises(ValueError, match="precision must be"):
            u.resolve_precision(bad)


@pytest.mark.parametrize("precision", [None, "auto"])
def test_auto_and_the_default_never_pick_bf16x3(monkeypatch, precision):
    """the extractor's default and "auto" upload f16x3 pairs; only an explicit bf16pair uploads bf16 pairs, with no
    fp16-range guard"""
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    seen = []

    class Fake:
        def __init__(self, name, sd, dev, depth=None, pair="tf32"):
            seen.append(pair)

    monkeypatch.setattr(u._vit, "VitWeights", Fake)
    ext = u.DinoV2ExtractFeatures.__new__(u.DinoV2ExtractFeatures)
    ext.layer = 1
    ext._load("dinov2_vits14", None, {}, "auto", precision)
    assert seen == ["f16"] and ext.precision == "f16x3" and ext._auto
    ext._load("dinov2_vits14", None, {}, "tc3", "bf16pair")
    assert seen[-1] == "bf16pair" and ext.precision == "bf16pair" and not ext._auto and ext._state_dict is None
    with pytest.raises(ValueError):
        ext._load("dinov2_vits14", None, {}, "simt", "bf16pair")


def _cfg(dim=384, heads=6, depth=4, ffn="mlp", pair="bf16pair", reg=0):
    return _lib.VitCfg(dim, depth, heads, _lib.FFN[ffn], vit.ffn_hidden(dim, ffn), vit.PATCH, _lib.PAIR[pair], reg)


def A(x):
    return (x + 255) // 256 * 256


def documented_bytes(cfg, n_patch, M, qkv32=False):
    """the workspace formula of include/anyloc_b200.h for pair_dtype = ANYLOC_PAIR_BF16X3"""
    D, Kp, Hf = cfg.embed_dim, 608, cfg.ffn_hidden
    return (2 * A(2 * n_patch * Kp) + A(4 * n_patch * D) + A(4 * M * D) + 2 * A(2 * M * D) + 2 * A(6 * M * D) +
            2 * A(2 * M * Hf) + (A(12 * M * D) if qkv32 else 0) + 4096)


def _taps(pairs):
    return (_lib.VitTap * len(pairs))(*[_lib.VitTap(l, _lib.FACET[f], FAKE) for l, f in pairs])


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


@pytest.mark.parametrize("dim,heads,ffn,reg", [(384, 6, "mlp", 0), (1536, 24, "swiglufused", 0), (768, 12, "mlp", 4)])
def test_workspace_is_the_documented_formula(lib, dim, heads, ffn, reg):
    """the bf16 pairs take the 2-byte GEMM inputs of the fp16 pairs' bytes: less than the f16x3 workspace (whose pair
    buffers hold fp32 words), more than single bf16's"""
    cfg = _cfg(dim, heads, ffn=ffn, reg=reg)
    f16, bf16 = _cfg(dim, heads, ffn=ffn, reg=reg, pair="f16"), _cfg(dim, heads, ffn=ffn, reg=reg, pair="bf16")
    for B, H, W in [(1, 224, 224), (3, 98, 126), (32, 322, 322)]:
        N = (H // 14) * (W // 14)
        M = B * (N + 1 + reg)
        got = lib.anyloc_vit_workspace_bytes(C.byref(cfg), B, H, W)
        assert got == documented_bytes(cfg, B * N, M), (dim, B, H, W)
        assert lib.anyloc_vit_workspace_bytes(C.byref(bf16), B, H, W) < got < \
            lib.anyloc_vit_workspace_bytes(C.byref(f16), B, H, W)
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps([(1, "query"), (3, "value")]), 2) == \
            documented_bytes(cfg, B * N, M, qkv32=True)
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps([(3, "value")]), 1) == got
    sizes = [(98, 126), (224, 224), (14, 14)]
    n_patch = sum((h // 14) * (w // 14) for h, w in sizes)
    M = n_patch + len(sizes) * (1 + reg)
    assert lib.anyloc_vit_varlen_workspace_bytes(C.byref(cfg), 3, _hw(sizes)) == documented_bytes(cfg, n_patch, M)
    assert lib.anyloc_vit_taps_varlen_workspace_bytes(C.byref(cfg), 3, _hw(sizes), _taps([(0, "key"), (2, "token")]),
                                                      2) == documented_bytes(cfg, n_patch, M, qkv32=True)


def _weights(null_field=None):
    blocks = (_lib.VitBlock * 4)()
    for b in blocks:
        for n in ("qkv_w", "proj_w", "in_w", "out_w"):
            setattr(b, n + "_hi", FAKE)
            setattr(b, n + "_lo", FAKE)
        b.qkv_alpha = b.proj_alpha = b.in_alpha = b.out_alpha = 1.0
    w = _lib.VitWeightsStruct(FAKE, FAKE, FAKE, FAKE, blocks, 1.0, None)
    if null_field == "patch_w_lo":
        w.patch_w_lo = None
    elif null_field:
        setattr(blocks[2], null_field, None)
    return w, blocks


@pytest.mark.parametrize("call", ["single", "taps", "varlen", "taps_varlen"])
@pytest.mark.parametrize("lo", ["patch_w_lo", "qkv_w_lo", "proj_w_lo", "in_w_lo", "out_w_lo"])
def test_vit_refuses_missing_lo_weights_and_the_simt_engine(lib, call, lo):
    cfg = _cfg()

    def run(w, engine="tc3"):
        taps, ptrs, hw = _taps([(3, "value")]), (C.c_void_p * 2)(FAKE, FAKE), _hw([(224, 224), (98, 126)])
        f, eng = C.c_void_p(FAKE), _lib.ENGINE[engine]
        if call == "single":
            return lib.anyloc_vit_extract(C.byref(cfg), C.byref(w), f, 2, 224, 224, f, 3, 2, 0, 1, f, f, 1 << 40, eng,
                                          None)
        if call == "taps":
            return lib.anyloc_vit_extract_taps(C.byref(cfg), C.byref(w), f, 2, 224, 224, f, taps, 1, 0, 1, f, 1 << 40,
                                               eng, None)
        if call == "varlen":
            return lib.anyloc_vit_extract_varlen(C.byref(cfg), C.byref(w), 2, ptrs, hw, ptrs, 3, 2, 0, 1, f, f,
                                                 1 << 40, eng, None)
        return lib.anyloc_vit_extract_taps_varlen(C.byref(cfg), C.byref(w), 2, ptrs, hw, ptrs, taps, 1, 0, 1, f,
                                                  1 << 40, eng, None)

    w, keep = _weights(lo)
    assert run(w) == ARG
    assert "ANYLOC_PAIR_BF16X3" in _lib.last_error() and "*_w_lo must be non-NULL" in _lib.last_error()
    w, keep = _weights()
    assert run(w, "simt") == UNSUPPORTED
    assert "bf16-pair" in _lib.last_error() or "tensor-core" in _lib.last_error()


def test_gemm_argument_checks(lib):
    f = C.c_void_p(FAKE)

    def gemm(a_lo=f, b_lo=f, out_lo=f, in_dt=X3, out_dt=X3, engine="tc3", epi="bias_split", K=64):
        return lib.anyloc_gemm_nt(f, a_lo, K, f, b_lo, K, 128, 128, K, in_dt, C.c_float(1.0), _lib.EPI[epi], None,
                                  None, None, f, out_lo, 128, out_dt, _lib.ENGINE[engine], None)

    # each lo operand is mandatory: without it the operand is single bf16
    assert gemm(a_lo=None) == ARG and "both lo operands" in _lib.last_error()
    assert gemm(b_lo=None) == ARG and "both lo operands" in _lib.last_error()
    assert gemm(out_lo=None) == ARG and "out_lo" in _lib.last_error()
    assert gemm(a_lo=None, b_lo=None, out_lo=None) == ARG
    for epi in ("gelu_split", "swiglu_split"):
        assert gemm(out_lo=None, epi=epi) == ARG
    # mixed formats, in either direction
    for dt in ("tf32", "f16", "bf16", "f16x1"):
        assert gemm(out_dt=_lib.PAIR[dt]) == ARG
        assert gemm(in_dt=_lib.PAIR[dt], out_dt=X3) == ARG
    assert gemm(in_dt=_lib.PAIR["fp8"], out_dt=X3) == ARG
    # the next value is not a format
    for bad in (6, 7, -1):
        assert gemm(in_dt=bad, out_dt=bad) == ARG and "bad in_dtype" in _lib.last_error()
        assert gemm(out_dt=bad) == ARG and "bad out_dtype" in _lib.last_error()
    # tensor cores only, at every shape
    assert gemm(engine="simt") == UNSUPPORTED and "bf16-pair" in _lib.last_error()
    assert gemm(engine="simt", epi="bias", out_lo=None) == UNSUPPORTED
    assert gemm(engine="auto", K=60) == UNSUPPORTED      # K not a multiple of 8 bf16 elements


def test_layernorm_and_attention_argument_checks(lib):
    f = C.c_void_p(FAKE)
    ln = lib.anyloc_layernorm_split
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), f, None, X3, None) == ARG
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), C.c_void_p(FAKE + 4), f, X3, None) == ARG     # 4 bf16 = 8 bytes
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), f, C.c_void_p(FAKE + 4), X3, None) == ARG
    assert ln(f, f, f, 0, 384, C.c_float(1e-6), C.c_void_p(FAKE + 8), C.c_void_p(FAKE + 8), X3, None) == 0
    att = lib.anyloc_attention
    tc3, simt = _lib.ENGINE["tc3"], _lib.ENGINE["simt"]
    assert att(f, None, 1, 64, 128, 2, f, f, X3, tc3, None) == ARG
    assert att(f, f, 1, 64, 128, 2, f, None, X3, tc3, None) == ARG
    assert "bf16-pair" in _lib.last_error() and "qkv_lo and o_lo" in _lib.last_error()
    assert att(f, f, 1, 64, 128, 2, f, C.c_void_p(FAKE + 4), X3, tc3, None) == ARG       # o_lo 8-byte
    assert att(f, f, 1, 64, 96, 2, f, f, X3, tc3, None) == ARG                              # head_dim 48
    assert att(f, f, 1, 64, 128, 2, f, f, X3, simt, None) == UNSUPPORTED
    assert att(f, C.c_void_p(FAKE + 8), 1, 64, 128, 2, f, f, X3, _lib.ENGINE["auto"], None) == UNSUPPORTED
    assert att(f, f, 0, 64, 128, 2, f, f, X3, tc3, None) == 0                               # nothing to do
    row0, len_ = (C.c_int32 * 1)(0), (C.c_int32 * 1)(64)
    av = lib.anyloc_attention_varlen
    assert av(f, None, 1, row0, len_, 128, 2, f, f, X3, None) == ARG
    assert av(f, f, 1, row0, len_, 128, 2, f, None, X3, None) == ARG
    assert "pair formats need qkv_lo and o_lo" in _lib.last_error()
    assert av(f, C.c_void_p(FAKE + 8), 1, row0, len_, 128, 2, f, f, X3, None) == UNSUPPORTED
    for bad in (6, 7):
        assert av(f, f, 1, row0, len_, 128, 2, f, f, bad, None) == ARG and "bad fmt" in _lib.last_error()


# --------------------------------------------------------------------------------------------------------- emulation
HW = (28, 42)


def test_bf16_pair_rounding():
    """hi + lo keeps 16 significant bits of x (17 with a sign change between hi and lo), round to nearest; hi and lo
    are both bf16 values; x beyond bf16's largest finite value rounds to Inf"""
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(100000, generator=g) * 10.0 ** torch.randint(-30, 30, (100000,), generator=g)).double()
    x = x.float().double()                                   # fp32 inputs, as the kernels see them
    y = bf16_pair(x)
    hi = x.to(torch.bfloat16)
    lo = (x - hi.double()).to(torch.bfloat16)
    assert torch.equal(y, hi.double() + lo.double())
    assert torch.equal((x.float() - hi.float()).double(), x - hi.double())    # x - hi is exact in fp32
    rel = ((y - x).abs() / x.abs()).max()
    assert 2.0 ** -18 < rel <= 2.0 ** -16, float(rel)
    big = torch.tensor([3.38e38, 3.4e38, -3.4e38], dtype=torch.float32).double()
    assert torch.isfinite(bf16_pair(big[:1])).all() and not torch.isfinite(bf16_pair(big[1:])).any()


def test_identity_and_the_pair_rounding_hooks():
    """the emulation with every rounding the identity is the fp64 model bit for bit, and with the pair rounding every
    rounded value is a sum of two bf16 values"""
    m = model_of("vits", "random")
    img = image(HW).double()
    want = forward_taps(copy.deepcopy(m).double(), img)
    got = forward_taps(emulated(m, identity()), img)
    for tap in want:
        assert torch.equal(got[tap], want[tap]), tap
    seen = {}
    with torch.no_grad():
        emulated(m, recording(rounding_bf16x3(), seen))(img)
    assert set(seen) == set(POINTS) | {"weight", "p"}
    for point, vals in seen.items():
        y = torch.cat([v.flatten() for v in vals])
        hi = y.to(torch.bfloat16).double()
        assert torch.equal((y - hi).to(torch.bfloat16).double(), y - hi), point


def rel_rms(a, b):
    return float((a - b).norm() / b.norm())


def test_emulation_error_sits_between_f16x1_and_fp32():
    """per rounded operand the pair's relative RMS rounding error is far below single fp16's 2^-11 (measured on ViT-S:
    2.45e-6 = 0.32 x 2^-17 at every point, against 0.42 x 2^-11 for f16x1; lo rounds x - hi, whose size is spread below
    2^-8 |x|); at the taps, the bf16pair emulation's RMS error against fp64 is over 32x below f16x1's (measured 83x)"""
    m = model_of("vits", "random")
    img = image((56, 70)).double()
    band = {}
    for precision, rnd in (("f16x1", rounding("f16x1")), ("bf16pair", rounding_bf16x3())):
        xs, ys = {}, {}
        with torch.no_grad():
            emulated(m, recording(rnd, xs, inputs=True))(img)
            emulated(m, recording(rnd, ys))(img)
        for point in POINTS:
            x, y = torch.cat([v.flatten() for v in xs[point]]), torch.cat([v.flatten() for v in ys[point]])
            band[(precision, point)] = rel_rms(y, x)
        r64 = forward_taps(copy.deepcopy(m).double(), img)
        emu = forward_taps(emulated(m, rnd), img)
        band[precision] = max(rel_rms(emu[t], r64[t]) for t in r64)
    print(band)
    for point in POINTS:
        assert 2.0 ** -21 < band[("bf16pair", point)] < 2.0 ** -16, (point, band)
    assert 0 < band["bf16pair"] < band["f16x1"] / 32, band
