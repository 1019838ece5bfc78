"""The single-fp16 precision without a GPU: the precision choice (argument and $ANYLOC_B200_PRECISION, "auto" and the
default never picking it), the format's constant, the C ABI's refusals for ANYLOC_PAIR_F16X1 (which return before
anything touches the device) and the documented workspace sizes."""
import ctypes as C

import pytest

from anyloc_b200 import _lib, vit
from anyloc_b200 import utilities as u

ARG, UNSUPPORTED = _lib.ERR["arg"], _lib.ERR["unsupported"]
FAKE = 4096                      # placeholder device pointer (16-byte aligned); every checked error returns first
H1 = _lib.PAIR["f16x1"]


def test_format_constant():
    assert _lib.PAIR["f16x1"] == 4


def test_precision_choice(monkeypatch):
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    assert u.resolve_precision("f16x1") == "f16x1" and u.resolve_precision("f16x1", "tc3") == "f16x1"
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "f16x1")
    assert u.resolve_precision(None) == "f16x1"
    assert u.resolve_precision("bf16") == "bf16"          # the argument wins
    with pytest.raises(ValueError, match="tensor cores"):
        u.resolve_precision(None, "simt")
    with pytest.raises(ValueError, match="tensor cores"):
        u.resolve_precision("f16x1", "simt")
    for bad in ("F16X1", "f16x2", "fp16x1", "f16"):
        with pytest.raises(ValueError, match="precision must be"):
            u.resolve_precision(bad)


@pytest.mark.parametrize("precision", [None, "auto"])
def test_auto_and_the_default_never_pick_f16x1(monkeypatch, precision):
    """the extractor's default and "auto" upload f16x3 pairs; only an explicit f16x1 uploads single fp16 weights"""
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    seen = []

    class Fake:
        def __init__(self, name, sd, dev, depth=None, pair="tf32"):
            seen.append(pair)

    monkeypatch.setattr(u._vit, "VitWeights", Fake)
    ext = u.DinoV2ExtractFeatures.__new__(u.DinoV2ExtractFeatures)
    ext.layer = 1
    ext._load("dinov2_vits14", None, {}, "auto", precision)
    assert seen == ["f16"] and ext.precision == "f16x3" and ext._overflow_msg() == ext._OVERFLOW_MSG
    ext._load("dinov2_vits14", None, {}, "auto", "f16x1")
    assert seen[-1] == "f16x1" and ext.precision == "f16x1" and not ext._auto
    assert "precision='bf16'" in ext._overflow_msg()
    with pytest.raises(ValueError):
        ext._load("dinov2_vits14", None, {}, "simt", "f16x1")


def _cfg(dim=384, heads=6, depth=4, ffn="mlp", pair="f16x1", reg=0):
    return _lib.VitCfg(dim, depth, heads, _lib.FFN[ffn], vit.ffn_hidden(dim, ffn), vit.PATCH, _lib.PAIR[pair], reg)


def A(x):
    return (x + 255) // 256 * 256


def documented_bytes(cfg, n_patch, M, qkv32=False):
    """the workspace formula of include/anyloc_b200.h for pair_dtype = ANYLOC_PAIR_F16X1"""
    D, Kp, Hf = cfg.embed_dim, 608, cfg.ffn_hidden
    return (A(2 * n_patch * Kp) + A(4 * n_patch * D) + A(4 * M * D) + A(2 * M * D) + A(6 * M * D) + A(2 * M * Hf) +
            (A(12 * M * D) if qkv32 else 0) + 4096)


def _taps(pairs):
    return (_lib.VitTap * len(pairs))(*[_lib.VitTap(l, _lib.FACET[f], FAKE) for l, f in pairs])


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


@pytest.mark.parametrize("dim,heads,ffn,reg", [(384, 6, "mlp", 0), (1536, 24, "swiglufused", 0), (768, 12, "mlp", 4)])
def test_workspace_is_the_documented_formula_and_smaller_than_f16x3(lib, dim, heads, ffn, reg):
    cfg = _cfg(dim, heads, ffn=ffn, reg=reg)
    f16 = _cfg(dim, heads, ffn=ffn, reg=reg, pair="f16")
    for B, H, W in [(1, 224, 224), (3, 98, 126), (32, 322, 322)]:
        N = (H // 14) * (W // 14)
        M = B * (N + 1 + reg)
        got = lib.anyloc_vit_workspace_bytes(C.byref(cfg), B, H, W)
        assert got == documented_bytes(cfg, B * N, M), (dim, B, H, W)
        assert got < lib.anyloc_vit_workspace_bytes(C.byref(f16), B, H, W)
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps([(1, "query"), (3, "value")]), 2) == \
            documented_bytes(cfg, B * N, M, qkv32=True)
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps([(3, "value")]), 1) == got
    sizes = [(98, 126), (224, 224), (14, 14)]
    n_patch = sum((h // 14) * (w // 14) for h, w in sizes)
    M = n_patch + len(sizes) * (1 + reg)
    assert lib.anyloc_vit_varlen_workspace_bytes(C.byref(cfg), 3, _hw(sizes)) == documented_bytes(cfg, n_patch, M)
    assert lib.anyloc_vit_taps_varlen_workspace_bytes(C.byref(cfg), 3, _hw(sizes), _taps([(0, "key"), (2, "token")]),
                                                      2) == documented_bytes(cfg, n_patch, M, qkv32=True)


def _weights(lo_field=None):
    blocks = (_lib.VitBlock * 4)()
    for b in blocks:
        for n in ("qkv_w_hi", "proj_w_hi", "in_w_hi", "out_w_hi"):
            setattr(b, n, FAKE)
        b.qkv_alpha = b.proj_alpha = b.in_alpha = b.out_alpha = 2.0 ** -17
    w = _lib.VitWeightsStruct(FAKE, None, FAKE, FAKE, blocks, 2.0 ** -17, None)
    if lo_field == "patch_w_lo":
        w.patch_w_lo = FAKE
    elif lo_field:
        setattr(blocks[1], lo_field, FAKE)
    return w, blocks


@pytest.mark.parametrize("call", ["single", "taps", "varlen", "taps_varlen"])
@pytest.mark.parametrize("lo", ["patch_w_lo", "qkv_w_lo", "proj_w_lo", "in_w_lo", "out_w_lo"])
def test_vit_refuses_lo_weights_and_the_simt_engine(lib, call, lo):
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
    assert "ANYLOC_PAIR_F16X1" in _lib.last_error() and "*_w_lo must be NULL" in _lib.last_error()
    w, keep = _weights()
    assert run(w, "simt") == UNSUPPORTED
    assert "single-fp16" in _lib.last_error() or "tensor-core" in _lib.last_error()


def test_building_block_argument_checks(lib):
    f = C.c_void_p(FAKE)

    def gemm(a_lo=None, b_lo=None, out_lo=None, in_dt=H1, out_dt=H1, engine="tc3", epi="bias_split", K=64):
        return lib.anyloc_gemm_nt(f, a_lo, K, f, b_lo, K, 128, 128, K, in_dt, C.c_float(1.0), _lib.EPI[epi], None,
                                  None, None, f, out_lo, 128, out_dt, _lib.ENGINE[engine], None)

    assert gemm(a_lo=f) == ARG and gemm(b_lo=f) == ARG and gemm(out_lo=f) == ARG
    assert "single-fp16" in _lib.last_error() and "no lo arrays" in _lib.last_error()
    for dt in ("tf32", "f16", "bf16", "fp8"):
        assert gemm(out_dt=_lib.PAIR[dt], out_lo=f) == ARG
        assert gemm(in_dt=_lib.PAIR[dt], out_lo=f) == ARG
    assert gemm(in_dt=5, out_dt=5) == ARG
    assert gemm(engine="simt") == UNSUPPORTED and gemm(engine="simt", epi="bias") == UNSUPPORTED
    assert gemm(K=60) == UNSUPPORTED          # K not a multiple of 8 fp16 elements: outside the tensor-core contract
    ln = lib.anyloc_layernorm_split
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), f, f, H1, None) == ARG
    assert "single-fp16" in _lib.last_error()
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), C.c_void_p(FAKE + 2), None, H1, None) == ARG      # y_hi misaligned
    att = lib.anyloc_attention
    assert att(f, f, 1, 64, 128, 2, f, None, H1, _lib.ENGINE["tc3"], None) == ARG
    assert att(f, None, 1, 64, 128, 2, f, f, H1, _lib.ENGINE["tc3"], None) == ARG
    assert att(f, None, 1, 64, 128, 2, f, None, H1, _lib.ENGINE["simt"], None) == UNSUPPORTED
    assert att(f, None, 1, 64, 96, 2, f, None, H1, _lib.ENGINE["tc3"], None) == ARG          # head_dim 48
    row0, ln_ = (C.c_int32 * 1)(0), (C.c_int32 * 1)(64)
    av = lib.anyloc_attention_varlen
    assert av(f, f, 1, row0, ln_, 128, 2, f, None, H1, None) == ARG
    assert av(f, None, 1, row0, ln_, 128, 2, f, f, H1, None) == ARG
    assert "single-fp16" in _lib.last_error()
    assert av(f, None, 1, row0, ln_, 128, 2, f, None, 5, None) == ARG
