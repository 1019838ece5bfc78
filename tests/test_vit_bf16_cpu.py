"""The single-bf16 precision without a GPU: the precision choice (argument and $ANYLOC_B200_PRECISION), the C ABI's
argument checks for ANYLOC_PAIR_BF16 (which return before anything touches the device), the documented workspace
sizes, and the extractors failing loudly without a device."""
import ctypes as C

import pytest
import torch

from anyloc_b200 import _lib, vit
from anyloc_b200 import utilities as u

ARG, UNSUPPORTED = _lib.ERR["arg"], _lib.ERR["unsupported"]
FAKE = 4096                      # placeholder device pointer (16-byte aligned); every checked error returns first


def test_precision_choice(monkeypatch):
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    assert u.resolve_precision(None) == "auto"
    for p in ("auto", "tf32x3", "f16x3", "bf16"):
        assert u.resolve_precision(p) == p
        assert u.resolve_precision(p, "tc3") == p
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "bf16")
    assert u.resolve_precision(None) == "bf16"
    assert u.resolve_precision("f16x3") == "f16x3"          # the argument wins
    with pytest.raises(ValueError, match="tensor cores"):
        u.resolve_precision(None, "simt")
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "fp16")
    with pytest.raises(ValueError, match="precision must be"):
        u.resolve_precision(None)
    for bad in ("BF16", "bf16x3", "fp32"):
        with pytest.raises(ValueError):
            u.resolve_precision(bad)
    with pytest.raises(ValueError):
        u.resolve_precision("bf16", "simt")
    assert u.resolve_precision("tf32x3", "simt") == "tf32x3"
    assert _lib.PAIR["bf16"] == 2


def _cfg(dim=384, heads=6, depth=4, ffn="mlp", pair="bf16", reg=0):
    return _lib.VitCfg(dim, depth, heads, _lib.FFN[ffn], vit.ffn_hidden(dim, ffn), vit.PATCH, _lib.PAIR[pair], reg)


def A(x):
    return (x + 255) // 256 * 256


def documented_bytes(cfg, n_patch, M, qkv32=False):
    """the workspace formula of include/anyloc_b200.h for pair_dtype = ANYLOC_PAIR_BF16"""
    D, Kp, Hf = cfg.embed_dim, 608, cfg.ffn_hidden
    return (A(2 * n_patch * Kp) + A(4 * n_patch * D) + A(4 * M * D) + A(2 * M * D) + A(6 * M * D) + A(2 * M * Hf) +
            (A(12 * M * D) if qkv32 else 0) + 4096)


def _taps(pairs):
    return (_lib.VitTap * len(pairs))(*[_lib.VitTap(l, _lib.FACET[f], FAKE) for l, f in pairs])


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


@pytest.mark.parametrize("dim,heads,ffn,reg", [(384, 6, "mlp", 0), (1536, 24, "swiglufused", 0), (768, 12, "mlp", 4)])
def test_workspace_is_the_documented_formula_and_smaller(lib, dim, heads, ffn, reg):
    cfg = _cfg(dim, heads, ffn=ffn, reg=reg)
    f16 = _cfg(dim, heads, ffn=ffn, reg=reg, pair="f16")
    for B, H, W in [(1, 224, 224), (3, 98, 126), (32, 322, 322)]:
        N = (H // 14) * (W // 14)
        M = B * (N + 1 + reg)
        got = lib.anyloc_vit_workspace_bytes(C.byref(cfg), B, H, W)
        assert got == documented_bytes(cfg, B * N, M), (dim, B, H, W)
        assert got < lib.anyloc_vit_workspace_bytes(C.byref(f16), B, H, W)
        taps = [(1, "query"), (3, "value")]
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps(taps), 2) == \
            documented_bytes(cfg, B * N, M, qkv32=True)
        assert lib.anyloc_vit_taps_workspace_bytes(C.byref(cfg), B, H, W, _taps([(3, "value")]), 1) == got
    sizes = [(98, 126), (224, 224), (14, 14)]
    n_patch = sum((h // 14) * (w // 14) for h, w in sizes)
    M = n_patch + len(sizes) * (1 + reg)
    assert lib.anyloc_vit_varlen_workspace_bytes(C.byref(cfg), 3, _hw(sizes)) == documented_bytes(cfg, n_patch, M)
    assert lib.anyloc_vit_taps_varlen_workspace_bytes(C.byref(cfg), 3, _hw(sizes), _taps([(0, "key"), (2, "token")]),
                                                      2) == documented_bytes(cfg, n_patch, M, qkv32=True)


def test_existing_formats_keep_their_workspace(lib):
    """tf32 / f16 pairs: 4-byte-element (hi, lo) buffers as before"""
    for pair in ("tf32", "f16"):
        cfg = _cfg(pair=pair)
        N, M = 256, 257
        want = (2 * A(4 * N * 608) + A(4 * N * 384) + A(4 * M * 384) + 2 * A(4 * M * 384) + 2 * A(12 * M * 384) +
                2 * A(4 * M * 1536) + 4096)
        assert lib.anyloc_vit_workspace_bytes(C.byref(cfg), 1, 224, 224) == want


def _weights(lo_field=None):
    blocks = (_lib.VitBlock * 4)()
    for b in blocks:
        for n in ("qkv_w_hi", "proj_w_hi", "in_w_hi", "out_w_hi"):
            setattr(b, n, FAKE)
        b.qkv_alpha = b.proj_alpha = b.in_alpha = b.out_alpha = 1.0
    w = _lib.VitWeightsStruct(FAKE, None, FAKE, FAKE, blocks, 1.0, None)
    if lo_field == "patch_w_lo":
        w.patch_w_lo = FAKE
    elif lo_field:
        setattr(blocks[2], lo_field, FAKE)
    return w, blocks


@pytest.mark.parametrize("varlen", [False, True])
@pytest.mark.parametrize("lo", ["patch_w_lo", "qkv_w_lo", "proj_w_lo", "in_w_lo", "out_w_lo"])
def test_vit_refuses_lo_weights_and_the_simt_engine(lib, varlen, lo):
    cfg = _cfg()

    def call(w, engine="tc3"):
        taps = _taps([(3, "value")])
        if varlen:
            ptrs = (C.c_void_p * 2)(FAKE, FAKE)
            return lib.anyloc_vit_extract_taps_varlen(C.byref(cfg), C.byref(w), 2, ptrs, _hw([(224, 224), (98, 126)]),
                                                      ptrs, taps, 1, 0, 1, C.c_void_p(FAKE), 1 << 40,
                                                      _lib.ENGINE[engine], None)
        return lib.anyloc_vit_extract_taps(C.byref(cfg), C.byref(w), C.c_void_p(FAKE), 2, 224, 224, C.c_void_p(FAKE),
                                           taps, 1, 0, 1, C.c_void_p(FAKE), 1 << 40, _lib.ENGINE[engine], None)

    w, keep = _weights(lo)
    assert call(w) == ARG
    assert "*_w_lo must be NULL" in _lib.last_error()
    w, keep = _weights()
    assert call(w, "simt") == UNSUPPORTED
    assert "tensor-core" in _lib.last_error()


def test_single_image_extract_refusals(lib):
    cfg = _cfg()
    w, keep = _weights("in_w_lo")
    args = (C.c_void_p(FAKE), 2, 224, 224, C.c_void_p(FAKE), 3, 2, 0, 1, C.c_void_p(FAKE), C.c_void_p(FAKE), 1 << 40)
    assert lib.anyloc_vit_extract(C.byref(cfg), C.byref(w), *args, _lib.ENGINE["auto"], None) == ARG
    w, keep = _weights()
    assert lib.anyloc_vit_extract(C.byref(cfg), C.byref(w), *args, _lib.ENGINE["simt"], None) == UNSUPPORTED


def test_building_block_argument_checks(lib):
    f, bf = C.c_void_p(FAKE), _lib.PAIR["bf16"]

    def gemm(a_lo=None, b_lo=None, out_lo=None, in_dt=bf, out_dt=bf, engine="tc3", epi="bias_split"):
        return lib.anyloc_gemm_nt(f, a_lo, 64, f, b_lo, 64, 128, 128, 64, in_dt, C.c_float(1.0), _lib.EPI[epi], None,
                                  None, None, f, out_lo, 128, out_dt, _lib.ENGINE[engine], None)

    assert gemm(a_lo=f) == ARG and gemm(b_lo=f) == ARG and gemm(out_lo=f) == ARG
    assert "no lo arrays" in _lib.last_error()
    assert gemm(out_dt=_lib.PAIR["f16"]) == ARG and gemm(in_dt=_lib.PAIR["tf32"], out_lo=f) == ARG
    assert gemm(in_dt=3, out_dt=3) == ARG
    assert gemm(engine="simt") == UNSUPPORTED
    assert gemm(engine="simt", epi="bias") == UNSUPPORTED
    # K not a multiple of 8 bf16 elements (16 bytes): outside the tensor-core contract, and there is no other engine
    assert lib.anyloc_gemm_nt(f, None, 60, f, None, 60, 128, 128, 60, bf, C.c_float(1.0), _lib.EPI["bias"], None, None,
                              None, f, None, 128, bf, _lib.ENGINE["auto"], None) == UNSUPPORTED
    ln = lib.anyloc_layernorm_split
    assert ln(f, f, f, 8, 384, C.c_float(1e-6), f, f, bf, None) == ARG
    att = lib.anyloc_attention
    assert att(f, f, 1, 64, 128, 2, f, None, bf, _lib.ENGINE["tc3"], None) == ARG
    assert att(f, None, 1, 64, 128, 2, f, f, bf, _lib.ENGINE["tc3"], None) == ARG
    assert att(f, None, 1, 64, 128, 2, f, None, bf, _lib.ENGINE["simt"], None) == UNSUPPORTED
    assert att(f, None, 1, 64, 96, 2, f, None, bf, _lib.ENGINE["tc3"], None) == ARG          # head_dim 48


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_extractors_fail_loudly_without_gpu(lib):
    with pytest.raises(_lib.AnylocError):
        u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", precision="bf16")
    with pytest.raises(_lib.AnylocError):
        u.DinoV2MultiExtractFeatures("dinov2_vits14", [(3, "value")], device="cuda", precision="bf16")
    with pytest.raises(_lib.AnylocError):
        vit.VitWeights("dinov2_vits14", {}, "cuda", pair="bf16")
