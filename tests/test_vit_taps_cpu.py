"""Several (layer, facet) taps from one forward pass, without a GPU: what a tap means on the oracle model (one forward
with hooks on several layers gives each tap's own oracle run), the tap-list validation, the workspace the C ABI asks
for and its argument checks (which return before anything touches the device)."""
import ctypes as C

import pytest
import torch
from torch.nn import functional as F

from anyloc_b200 import _lib, vit
from oracle import anyloc_oracle as ao
from oracle import dinov2_restated as dr

QKV = {"query": 0, "key": 1, "value": 2}


def test_hooks_on_several_layers_in_one_forward_equal_the_per_tap_oracle_runs():
    """q/k/v of layer l read block l's INPUT (the qkv projection of norm1(x_l)); token reads block l's OUTPUT"""
    model = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=5), seed=1)
    img = torch.randn(2, 3, 56, 70, generator=torch.Generator().manual_seed(3))
    layers = [0, 2, 3]
    captured, handles = {}, []
    for l in layers:
        blk = model.blocks[l]
        handles.append(blk.attn.qkv.register_forward_hook(lambda m, i, o, l=l: captured.__setitem__((l, "qkv"), o)))
        handles.append(blk.register_forward_hook(lambda m, i, o, l=l: captured.__setitem__((l, "token"), o)))
    try:
        with torch.no_grad():
            model(img)
    finally:
        for h in handles:
            h.remove()
    for l in layers:
        for facet in ("query", "key", "value", "token"):
            for use_cls, norm in ((False, True), (True, False)):
                res = captured[(l, "token" if facet == "token" else "qkv")]
                if not use_cls:
                    res = res[:, 1:]
                if facet != "token":
                    d = res.shape[2] // 3
                    res = res[:, :, QKV[facet] * d:(QKV[facet] + 1) * d]
                if norm:
                    res = F.normalize(res, dim=-1)
                ref = ao.extract_features(model, img, l, facet, use_cls, norm)
                assert torch.equal(res, ref), (l, facet, use_cls, norm)


def test_tap_list_validation():
    assert vit.check_taps([(3, "value"), (0, "token"), [1, "key"]], 4) == [(3, "value"), (0, "token"), (1, "key")]
    assert vit.check_taps(((l, "value") for l in range(4)), 4) == [(l, "value") for l in range(4)]
    for bad in ([], (), "value", [(1, "values")], [(1,)], [(1, "key", 2)], [("1", "key")], [(1.0, "key")],
                [(True, "key")], [(1, "key"), (1, "key")], [3]):
        with pytest.raises(ValueError):
            vit.check_taps(bad, 4)
    for bad in ([(4, "value")], [(-1, "token")], [(0, "key"), (7, "key")]):
        with pytest.raises(IndexError):
            vit.check_taps(bad, 4)


def _cfg(dim=384, heads=6, depth=4):
    return _lib.VitCfg(dim, depth, heads, _lib.FFN["mlp"], 4 * dim, vit.PATCH, _lib.PAIR["f16"])


def _taps(pairs, out=4096):
    return (_lib.VitTap * max(len(pairs), 1))(*[_lib.VitTap(l, _lib.FACET[f] if isinstance(f, str) else f, out)
                                                for l, f in pairs])


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


# (tap list, whether some layer's fp32 qkv rows are kept)
CASES = [([(3, "value")], False), ([(3, "token")], False), ([(0, "token"), (1, "token"), (3, "query")], False),
         ([(3, "query"), (3, "key")], True), ([(3, "query"), (3, "key"), (3, "value")], True),
         ([(3, "value"), (3, "token")], True), ([(1, "value"), (3, "token")], True),
         ([(0, "key"), (3, "value")], True), ([(2, "token"), (3, "key"), (0, "token")], False)]


def test_taps_workspace_adds_the_fp32_qkv_rows_exactly_when_needed(lib):
    for dim, heads in ((384, 6), (1536, 24)):
        cfg = C.byref(_cfg(dim, heads))
        for B, H, W in [(1, 224, 224), (3, 98, 126), (16, 224, 224)]:
            M = B * ((H // 14) * (W // 14) + 1)
            base = lib.anyloc_vit_workspace_bytes(cfg, B, H, W)
            for pairs, extra in CASES:
                got = lib.anyloc_vit_taps_workspace_bytes(cfg, B, H, W, _taps(pairs), len(pairs))
                assert got == base + (M * 3 * dim * 4 if extra else 0), (dim, B, H, W, pairs)
            sizes = [(98, 126), (224, 224), (14, 14)][:B]
            M = sum((h // 14) * (w // 14) + 1 for h, w in sizes)
            base = lib.anyloc_vit_varlen_workspace_bytes(cfg, len(sizes), _hw(sizes))
            for pairs, extra in CASES:
                got = lib.anyloc_vit_taps_varlen_workspace_bytes(cfg, len(sizes), _hw(sizes), _taps(pairs), len(pairs))
                assert got == base + (M * 3 * dim * 4 if extra else 0), (dim, sizes, pairs)
    cfg = C.byref(_cfg())
    for pairs in ([(4, "value")], [(1, "key"), (1, "key")], [(1, 4)], [(1, -1)]):
        assert lib.anyloc_vit_taps_workspace_bytes(cfg, 1, 224, 224, _taps(pairs), len(pairs)) == 0, pairs
        assert lib.anyloc_vit_taps_varlen_workspace_bytes(cfg, 1, _hw([(224, 224)]), _taps(pairs), len(pairs)) == 0
    assert lib.anyloc_vit_taps_workspace_bytes(cfg, 1, 224, 224, _taps([]), 0) == 0
    assert lib.anyloc_vit_taps_workspace_bytes(cfg, 1, 224, 224, None, 1) == 0


def _call(lib, pairs, n=None, varlen=False, ws_bytes=1 << 40, out=4096):
    """the tap entry points with placeholder device pointers: every checked error returns before any is used"""
    n = len(pairs) if n is None else n
    w, fake = _lib.VitWeightsStruct(), C.c_void_p(4096)
    taps = _taps(pairs, out)
    if varlen:
        ptrs = (C.c_void_p * 2)(4096, 4096)
        return lib.anyloc_vit_extract_taps_varlen(C.byref(_cfg()), C.byref(w), 2, ptrs, _hw([(224, 224), (98, 126)]),
                                                  ptrs, taps, n, 0, 1, fake, ws_bytes, _lib.ENGINE["tc3"], None)
    return lib.anyloc_vit_extract_taps(C.byref(_cfg()), C.byref(w), fake, 2, 224, 224, fake, taps, n, 0, 1, fake,
                                       ws_bytes, _lib.ENGINE["tc3"], None)


@pytest.mark.parametrize("varlen", [False, True])
def test_taps_abi_argument_errors(lib, varlen):
    arg = _lib.ERR["arg"]
    assert _call(lib, [(3, "value")], n=0, varlen=varlen) == arg and "no taps" in _lib.last_error()
    assert _call(lib, [(4, "value")], varlen=varlen) == arg and "out of range" in _lib.last_error()
    assert _call(lib, [(1, "token"), (-1, "value")], varlen=varlen) == arg and "out of range" in _lib.last_error()
    assert _call(lib, [(1, 4)], varlen=varlen) == arg and "bad facet" in _lib.last_error()
    assert _call(lib, [(1, "key"), (3, "value"), (1, "key")], varlen=varlen) == arg
    assert "twice" in _lib.last_error()
    assert _call(lib, [(1, "key")], out=None, varlen=varlen) == arg and "null output" in _lib.last_error()
    assert _call(lib, [(1, "key"), (3, "value")], ws_bytes=1 << 20, varlen=varlen) == _lib.ERR["workspace"]
    assert "workspace too small" in _lib.last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_multi_extractor_fails_loudly_without_gpu(lib):
    from anyloc_b200 import utilities as u
    with pytest.raises(_lib.AnylocError):
        u.DinoV2MultiExtractFeatures("dinov2_vits14", [(3, "value"), (5, "token")], device="cuda")
    with pytest.raises(_lib.AnylocError):
        u.DinoV2MultiExtractFeatures("dinov2_vits14", [(3, "value")])         # default device "cpu"
