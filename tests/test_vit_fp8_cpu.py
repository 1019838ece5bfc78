"""The single-e4m3 precision without a GPU: the precision choice (argument and $ANYLOC_B200_PRECISION, "auto" never
picking it), the C ABI's refusals for ANYLOC_PAIR_FP8 (which return before anything touches the device), the documented
workspace sizes, and the power-of-two scale rule of the quantisers against a numpy restatement."""
import ctypes as C

import numpy as np
import pytest

from anyloc_b200 import _lib, vit
from anyloc_b200 import utilities as u

ARG, UNSUPPORTED = _lib.ERR["arg"], _lib.ERR["unsupported"]
FAKE = 4096                      # placeholder device pointer (16-byte aligned); every checked error returns first
FP8 = _lib.PAIR["fp8"]


def test_precision_choice(monkeypatch):
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    assert _lib.PAIR["fp8"] == 3
    assert u.resolve_precision("fp8") == "fp8" and u.resolve_precision("fp8", "tc3") == "fp8"
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "fp8")
    assert u.resolve_precision(None) == "fp8"
    assert u.resolve_precision("bf16") == "bf16"          # the argument wins
    with pytest.raises(ValueError, match="tensor cores"):
        u.resolve_precision(None, "simt")
    for bad in ("FP8", "fp8x3", "e4m3", "fp8_e5m2"):
        with pytest.raises(ValueError, match="precision must be"):
            u.resolve_precision(bad)


@pytest.mark.parametrize("precision", [None, "auto"])
def test_auto_never_picks_fp8(monkeypatch, precision):
    """the extractor's default and "auto" upload f16x3 pairs; only an explicit fp8 uploads e4m3 weights"""
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    seen = []

    class Fake:
        def __init__(self, name, sd, dev, depth=None, pair="tf32"):
            seen.append(pair)

    monkeypatch.setattr(u._vit, "VitWeights", Fake)
    ext = u.DinoV2ExtractFeatures.__new__(u.DinoV2ExtractFeatures)
    ext.layer = 1
    ext._load("dinov2_vits14", None, {}, "auto", precision)
    assert seen == ["f16"] and ext.precision == "f16x3"
    ext._load("dinov2_vits14", None, {}, "auto", "fp8")
    assert seen[-1] == "fp8" and ext.precision == "fp8"
    with pytest.raises(ValueError):
        ext._load("dinov2_vits14", None, {}, "simt", "fp8")


def restated_scale(amax):
    """s = 2^ceil(log2(amax / 448)), at least 2^-126; 1 for amax = 0"""
    amax = np.float64(amax)
    if amax == 0:
        return 1.0
    return float(2.0 ** max(np.ceil(np.log2(amax / 448.0)), -126))


def test_scale_rule_matches_numpy(lib):
    vals = [0.0, 448.0, 1.0, 0.5, 3.0e38, 1.0e-30, 1.0e-40, 2.0 ** -149, 2.0 ** -126 * 448]
    for k in range(-157, 120, 3):            # every boundary 448 2^k that fp32 holds, and its neighbours
        b = 448.0 * 2.0 ** k
        if 2.0 ** -149 <= b <= 3.0e38:
            b = np.float32(b)
            vals += [float(b), float(np.nextafter(b, np.float32(np.inf))), float(np.nextafter(b, np.float32(0)))]
    rng = np.random.default_rng(0)
    vals += [float(v) for v in np.exp(rng.uniform(-80, 80, 2000)).astype(np.float32)]
    for v in vals:
        v32 = float(np.float32(v))
        got = lib.anyloc_fp8_scale(v32)
        assert got == restated_scale(v32), (v32, got, restated_scale(v32))
        if v32 > 0:
            assert v32 / got <= 448.0 and (got == 2.0 ** -126 or v32 / got > 224.0), v32


def _cfg(dim=384, heads=6, depth=4, ffn="mlp", pair="fp8", reg=0):
    return _lib.VitCfg(dim, depth, heads, _lib.FFN[ffn], vit.ffn_hidden(dim, ffn), vit.PATCH, _lib.PAIR[pair], reg)


def A(x):
    return (x + 255) // 256 * 256


def documented_bytes(cfg, n_patch, M, qkv32=False):
    """the workspace formula of include/anyloc_b200.h for pair_dtype = ANYLOC_PAIR_FP8"""
    D, Kp, Hf = cfg.embed_dim, 608, cfg.ffn_hidden
    return (A(2 * n_patch * Kp) + A(4 * n_patch * D) + A(4 * M * D) + A(M * D) + A(4 * M) + A(6 * M * D) +
            A(2 * M * Hf) + A(M * Hf) + A(4 * M) + (A(12 * M * D) if qkv32 else 0) + 4096)


def _taps(pairs):
    return (_lib.VitTap * len(pairs))(*[_lib.VitTap(l, _lib.FACET[f], FAKE) for l, f in pairs])


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


@pytest.mark.parametrize("dim,heads,ffn,reg", [(384, 6, "mlp", 0), (1536, 24, "swiglufused", 0), (768, 12, "mlp", 4)])
def test_workspace_is_the_documented_formula(lib, dim, heads, ffn, reg):
    cfg = _cfg(dim, heads, ffn=ffn, reg=reg)
    bf = _cfg(dim, heads, ffn=ffn, reg=reg, pair="bf16")
    for B, H, W in [(1, 224, 224), (3, 98, 126), (32, 322, 322)]:
        N = (H // 14) * (W // 14)
        M = B * (N + 1 + reg)
        got = lib.anyloc_vit_workspace_bytes(C.byref(cfg), B, H, W)
        assert got == documented_bytes(cfg, B * N, M), (dim, B, H, W)
        assert got < lib.anyloc_vit_workspace_bytes(C.byref(bf), B, H, W) * 1.6
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps([(1, "query"), (3, "value")]), 2) == \
            documented_bytes(cfg, B * N, M, qkv32=True)
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
        b.qkv_alpha = b.proj_alpha = b.in_alpha = b.out_alpha = 2.0 ** -10
    w = _lib.VitWeightsStruct(FAKE, None, FAKE, FAKE, blocks, 1.0, None)
    if lo_field == "patch_w_lo":
        w.patch_w_lo = FAKE
    elif lo_field:
        setattr(blocks[3], lo_field, FAKE)
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
    assert "ANYLOC_PAIR_FP8" in _lib.last_error() and "*_w_lo must be NULL" in _lib.last_error()
    w, keep = _weights()
    assert run(w, "simt") == UNSUPPORTED
    assert "single-e4m3" in _lib.last_error() or "tensor-core" in _lib.last_error()


def test_building_block_argument_checks(lib):
    f, bf = C.c_void_p(FAKE), _lib.PAIR["bf16"]

    def gemm(a_lo=f, b_lo=None, out_lo=None, out_dt=bf, engine="tc3", epi="bias_split", K=384, lda=384, ldb=384):
        return lib.anyloc_gemm_nt(f, a_lo, lda, f, b_lo, ldb, 128, 128, K, FP8, C.c_float(1.0), _lib.EPI[epi], None,
                                  None, None, f, out_lo, 128, out_dt, _lib.ENGINE[engine], None)

    assert gemm(a_lo=None) == ARG and "row scales" in _lib.last_error()
    assert gemm(b_lo=f) == ARG and gemm(out_lo=f) == ARG
    for dt in ("tf32", "f16", "fp8"):
        assert gemm(out_dt=_lib.PAIR[dt]) == ARG
    assert gemm(engine="simt") == UNSUPPORTED and gemm(engine="simt", epi="bias") == UNSUPPORTED
    assert gemm(K=392, lda=392, ldb=392) == UNSUPPORTED          # K not a multiple of 16 e4m3 elements
    assert gemm(lda=392) == UNSUPPORTED and gemm(ldb=392) == UNSUPPORTED
    assert gemm(a_lo=C.c_void_p(FAKE + 2)) == UNSUPPORTED       # misaligned row scales
    ln = lib.anyloc_layernorm_split
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), f, None, FP8, None) == ARG     # the row scales are required
    q = lib.anyloc_quantize_fp8_rows
    assert q(None, 8, 384, f, f, None) == ARG and q(f, 8, 384, None, f, None) == ARG and q(f, 8, 384, f, None, None) == ARG
    assert q(f, 8, 388, f, f, None) == ARG and q(f, -1, 384, f, f, None) == ARG and q(f, 8, 0, f, f, None) == ARG
    assert q(C.c_void_p(FAKE + 8), 8, 384, f, f, None) == ARG and q(f, 8, 384, C.c_void_p(FAKE + 4), f, None) == ARG
    assert q(f, 0, 384, f, f, None) == 0                        # nothing to do, nothing launched
    s = C.c_float()
    t = lib.anyloc_quantize_fp8_tensor
    assert t(None, f, 16, C.byref(s), None) == ARG and t(f, None, 16, C.byref(s), None) == ARG
    assert t(f, f, 16, None, None) == ARG and t(f, f, 0, C.byref(s), None) == ARG
