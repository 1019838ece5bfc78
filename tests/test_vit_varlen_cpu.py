"""Host side of list input to the extractor, without a GPU: where each image's rows land in the packed output, how a
long list splits into library calls, input validation, and the C ABI's size and argument checks (which return before
anything touches the device)."""
import ctypes as C

import pytest
import torch

from anyloc_b200 import _lib, vit


def test_layout_rows_tokens_and_offsets():
    sizes = [(224, 224), (98, 126), (14, 14), (756, 1022), (112, 224)]
    lay = vit.VarlenLayout(sizes, use_cls=False, max_b=128)
    assert lay.grids == [(16, 16), (7, 9), (1, 1), (54, 73), (8, 16)]
    assert lay.tokens == [257, 64, 2, 3943, 129]
    assert lay.n_out == [256, 63, 1, 3942, 128]
    assert lay.row0 == [0, 256, 319, 320, 4262, 4390] and lay.rows == 4390
    assert lay.chunks == [(0, 5)]
    cls = vit.VarlenLayout(sizes, use_cls=True, max_b=128)
    assert cls.n_out == cls.tokens and cls.rows == sum(cls.tokens)
    packed = torch.arange(lay.rows)
    parts = packed.split(lay.n_out)
    assert [p[0].item() for p in parts] == lay.row0[:-1]


def test_layout_splits_long_lists_at_the_library_limit():
    assert _lib.VIT_VARLEN_MAX_B >= 128
    lay = vit.VarlenLayout([(28, 42)] * 300, use_cls=False, max_b=128)
    assert lay.chunks == [(0, 128), (128, 256), (256, 300)]
    assert lay.row0[128] == 128 * 6 and lay.rows == 300 * 6
    assert vit.VarlenLayout([(14, 14)] * 128, False, 128).chunks == [(0, 128)]


def test_list_input_validation():
    cpu = torch.device("cpu")
    ok = [torch.zeros(3, 28, 42), torch.zeros(1, 3, 14, 14, dtype=torch.float64)]
    out = vit.check_varlen_images(ok, cpu)
    assert [tuple(x.shape) for x in out] == [(3, 28, 42), (3, 14, 14)] and all(x.dtype == torch.float32 for x in out)
    assert out[0].data_ptr() == ok[0].data_ptr()          # used in place, not copied
    bad = [[], (), [torch.zeros(3, 28, 30)], [torch.zeros(3, 30, 28)], [torch.zeros(28, 28)], [torch.zeros(4, 28, 28)],
           [torch.zeros(2, 3, 28, 28)], [torch.zeros(3, 0, 28)], [torch.zeros(3, 28, 28), "img"]]
    for imgs in bad:
        with pytest.raises(ValueError):
            vit.check_varlen_images(imgs, cpu)
    with pytest.raises(ValueError, match="on cpu"):
        vit.check_varlen_images([torch.zeros(3, 28, 28)], torch.device("cuda", 0))


def _cfg(dim=384, heads=6):
    return _lib.VitCfg(dim, 4, heads, _lib.FFN["mlp"], 4 * dim, vit.PATCH, _lib.PAIR["f16"])


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


def test_varlen_workspace_is_sized_from_the_totals(lib):
    cfg = C.byref(_cfg())
    for H, W, B in [(224, 224, 1), (98, 126, 3), (518, 518, 2)]:
        assert lib.anyloc_vit_varlen_workspace_bytes(cfg, B, _hw([(H, W)] * B)) == \
            lib.anyloc_vit_workspace_bytes(cfg, B, H, W)
    mixed = [(756, 1022)] + [(14, 14)] * 15
    ws = lib.anyloc_vit_varlen_workspace_bytes(cfg, 16, _hw(mixed))
    # from sum N_i and sum T_i, not from 16 copies of the largest image
    assert lib.anyloc_vit_workspace_bytes(cfg, 1, 756, 1022) < ws < lib.anyloc_vit_workspace_bytes(cfg, 2, 756, 1022)
    assert lib.anyloc_vit_varlen_workspace_bytes(cfg, 0, _hw([(14, 14)])) == 0
    assert lib.anyloc_vit_varlen_workspace_bytes(cfg, 129, _hw([(14, 14)] * 129)) == 0
    assert lib.anyloc_vit_varlen_workspace_bytes(cfg, 128, _hw([(14, 14)] * 128)) > 0
    assert lib.anyloc_vit_varlen_workspace_bytes(cfg, 2, _hw([(14, 14), (14, 15)])) == 0
    assert lib.anyloc_vit_varlen_workspace_bytes(cfg, 1, None) == 0


def _call(lib, sizes, engine="tc3", ws_bytes=1 << 40, B=None, layer=3):
    """anyloc_vit_extract_varlen with placeholder device pointers: every checked error returns before any is used"""
    B = len(sizes) if B is None else B
    fake = (C.c_void_p * max(B, 1))(*([4096] * max(B, 1)))
    w = _lib.VitWeightsStruct()
    return lib.anyloc_vit_extract_varlen(C.byref(_cfg()), C.byref(w), B, fake, _hw(sizes), fake, layer,
                                         _lib.FACET["value"], 0, 1, C.c_void_p(4096), C.c_void_p(4096), ws_bytes,
                                         _lib.ENGINE[engine], None)


def test_varlen_abi_argument_errors(lib):
    assert _call(lib, [(14, 14)] * 129) == _lib.ERR["arg"] and "out of range" in _lib.last_error()
    assert _call(lib, [], B=0) == _lib.ERR["arg"]
    assert _call(lib, [(224, 224), (224, 230)]) == _lib.ERR["arg"] and "multiples of the patch" in _lib.last_error()
    assert _call(lib, [(224, 224)], layer=4) == _lib.ERR["arg"]
    assert _call(lib, [(224, 224)], engine="simt") == _lib.ERR["unsupported"] and "simt" in _lib.last_error()
    assert _call(lib, [(224, 224), (98, 126)], ws_bytes=1 << 20) == _lib.ERR["workspace"]
    assert "workspace too small" in _lib.last_error()
