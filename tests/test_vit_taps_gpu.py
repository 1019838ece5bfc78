"""Several (layer, facet) taps from one forward pass (anyloc_vit_extract_taps / _varlen, DinoV2MultiExtractFeatures).
Every tap must be BIT-IDENTICAL to the single-tap call on the same weights, images, precision and GEMM engine, so the
feature adds no tolerance; the launch counts show that the blocks run once each."""
import ctypes as C

import pytest
import torch

from oracle import dinov2_restated as dr

pytestmark = pytest.mark.gpu
FACETS = ("query", "key", "value", "token")


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


@pytest.fixture(scope="module")
def vits_sd():
    return dr.perturb(dr.build("dinov2_vits14", seed=0), seed=1).state_dict()


def _img(B, H, W, seed=1234):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed)).cuda()


def _check(ext, img, opts):
    """every tap of ext equals the single-tap call of its weights, for each (use_cls, norm_descs) in opts"""
    m = ext.dino_model
    for use_cls, norm in opts:
        ext.use_cls, ext.norm_descs = use_cls, norm
        out = ext(img)
        assert list(out) == ext.taps
        for (layer, facet), got in out.items():
            ref = m.extract(img, layer, facet, use_cls, norm, ext.gemm_engine)
            assert got.shape == ref.shape and torch.equal(got, ref), (
                ext.precision, ext.gemm_engine, layer, facet, use_cls, norm, (got - ref).abs().max().item())


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("engine", ["tc3", "simt", "auto"])
def test_all_vits_taps_in_one_call(u, vits_sd, precision, engine):
    taps = [(l, f) for l in range(12) for f in FACETS]
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps[::-1], device="cuda", weights=vits_sd,
                                       gemm_engine=engine, precision=precision)
    assert ext.dino_model.depth == 12
    _check(ext, _img(3, 56, 70), [(False, True), (True, False)])
    if engine == "auto":        # T = 5: the GEMMs take the SIMT engine under "auto"
        _check(ext, _img(1, 28, 28), [(False, True), (True, True)])


def test_single_tap_class_agrees(u, vits_sd):
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", [(4, "key"), (2, "token"), (7, "value")], device="cuda",
                                       weights=vits_sd)
    img = _img(2, 42, 98)
    out = ext(img)
    for layer, facet in ext.taps:
        one = u.DinoV2ExtractFeatures("dinov2_vits14", layer, facet, device="cuda", weights=vits_sd)
        assert one.precision == ext.precision and torch.equal(out[(layer, facet)], one(img)), (layer, facet)


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_vitg_swiglu_taps(u, precision):
    from anyloc_b200 import vit
    sd = vit.random_state_dict("dinov2_vitg14", seed=3, device="cuda", depth=4)
    taps = [(l, f) for l in range(4) for f in FACETS]
    ext = u.DinoV2MultiExtractFeatures("dinov2_vitg14", taps, device="cuda", weights=sd, gemm_engine="tc3",
                                       precision=precision)
    _check(ext, _img(2, 42, 56), [(False, True), (True, False)])


# the deepest layer: one q/k/v facet (its own N = D GEMM), two or three (the N = 3D GEMM and the tap kernel without
# pairs), and a token tap (the whole block runs, with or without q/k/v taps of its own)
DEEPEST = [[(1, "token"), (5, "value")], [(0, "query"), (5, "key"), (5, "value")],
           [(5, "query"), (5, "key"), (5, "value")], [(5, "value"), (5, "token")], [(2, "key"), (5, "token")],
           [(5, "query"), (5, "value"), (5, "token"), (3, "value")]]


@pytest.mark.parametrize("taps", DEEPEST)
def test_deepest_layer_cases(u, vits_sd, taps):
    for precision in ("f16x3", "tf32x3"):
        ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=vits_sd, gemm_engine="tc3",
                                           precision=precision)
        assert ext.dino_model.depth == 6
        for B in (1, 3):
            _check(ext, _img(B, 70, 42, seed=B), [(False, True), (True, False), (False, False)])


def test_list_input(u, vits_sd):
    sizes = [(56, 70), (14, 14), (98, 42), (224, 224)]
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(sizes)]
    for precision in ("f16x3", "tf32x3"):
        for taps in ([(l, f) for l in (0, 3, 5) for f in FACETS], [(2, "token"), (5, "value")],
                     [(5, "key"), (5, "query")]):
            ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=vits_sd,
                                               gemm_engine="tc3", precision=precision)
            for use_cls, norm in ((False, True), (True, False)):
                ext.use_cls, ext.norm_descs = use_cls, norm
                out = ext(imgs)
                for (layer, facet), items in out.items():
                    assert len(items) == len(imgs)
                    for x, got in zip(imgs, items):
                        ref = ext.dino_model.extract(x[None], layer, facet, use_cls, norm, "tc3")[0]
                        assert torch.equal(got, ref), (precision, layer, facet, use_cls, norm, tuple(x.shape))


def _count(fn):
    from anyloc_b200 import _lib
    fn()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    return _lib.launch_count() - n0


def test_launch_counts(u, vits_sd):
    """One-tap calls launch what the single-tap schedule gives (blocks 0..layer-1, then the whole block or norm1 + the
    facet's GEMM, then the facet slice); a multi-tap call launches one forward pass to the deepest layer plus one tap
    kernel per layer with q/k/v taps and one facet slice per token tap."""
    from anyloc_b200 import _lib
    lib = _lib.load()
    B, H, W, D = 2, 56, 70, 384
    M = B * ((H // 14) * (W // 14) + 1)
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", [(l, "token") for l in range(12)], device="cuda",
                                       weights=vits_sd, gemm_engine="tc3", precision="tf32x3")
    m, img = ext.dino_model, _img(B, H, W)
    # launches of one GEMM and of the attention, from the building blocks themselves
    a = torch.randn(M, D, device="cuda")
    b = torch.randn(3 * D, D, device="cuda")
    o = torch.empty(M, 3 * D, device="cuda")
    o_lo = torch.empty(M, 3 * D, device="cuda")
    g = _count(lambda: lib.anyloc_gemm_nt(_lib.ptr(a), _lib.ptr(a), D, _lib.ptr(b), _lib.ptr(b), D, M, 3 * D, D,
                                          _lib.PAIR["tf32"], C.c_float(1.0), _lib.EPI["bias"], None, None, None,
                                          _lib.ptr(o), None, 3 * D, _lib.PAIR["tf32"], _lib.ENGINE["tc3"],
                                          _lib.stream_ptr()))
    y = torch.empty(M, D, device="cuda")
    at = _count(lambda: lib.anyloc_attention(_lib.ptr(o), _lib.ptr(o_lo), B, M // B, D, 6, _lib.ptr(y), _lib.ptr(y),
                                             _lib.PAIR["tf32"], _lib.ENGINE["tc3"], _lib.stream_ptr()))
    assert g >= 1 and at >= 1
    prefix, block = 1 + g + 1, 2 + at + 4 * g           # im2col, patch GEMM, assembly | 2 LayerNorms, 4 GEMMs
    for layer in (0, 4, 11):
        assert _count(lambda: m.extract(img, layer, "token", engine="tc3")) == prefix + (layer + 1) * block + 1
        assert _count(lambda: m.extract(img, layer, "key", engine="tc3")) == prefix + layer * block + 1 + g + 1
    cases = [([(l, f) for l in range(12) for f in FACETS], 12 * block + 12 + 12),
             ([(2, "value"), (5, "token"), (7, "query"), (7, "key")], 7 * block + 1 + g + 1 + 1 + 1),
             ([(2, "token"), (5, "token"), (7, "value")], 7 * block + 1 + g + 1 + 2)]
    for taps, n in cases:
        _lib.profile_enable(True)
        got = _count(lambda: m.extract_taps(img, taps, engine="tc3"))
        prof = _lib.profile_read()
        _lib.profile_enable(False)
        assert got == prefix + n, (taps, got, prefix + n)
        n_tap_kernels = len({l for l, f in taps if f != "token"} - ({7} if taps[-1] == (7, "value") else set()))
        assert prof["vit_misc"][1] == 2 * n_tap_kernels, (taps, prof["vit_misc"])     # both counted calls


def test_refusals_leave_outputs_untouched(u, vits_sd):
    from anyloc_b200 import _lib
    lib = _lib.load()
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", [(5, "value")], device="cuda", weights=vits_sd,
                                       gemm_engine="tc3", precision="tf32x3")
    m = ext.dino_model
    B, H, W, canary = 2, 56, 42, 7
    img = _img(B, H, W)
    rows = B * (H // 14) * (W // 14)
    pairs = [(1, "key"), (5, "token"), (3, "value"), (3, "query")]
    outs = [torch.full((rows + canary, m.dim), float("nan"), device="cuda") for _ in pairs]
    pos = m.pos_for(H // 14, W // 14)

    def call(taps, ws_bytes=None):
        arr = (_lib.VitTap * len(taps))(*[_lib.VitTap(l, f, p) for l, f, p in taps])
        nbytes = lib.anyloc_vit_taps_workspace_bytes(C.byref(m.cfg), B, H, W, arr, len(taps))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")
        return lib.anyloc_vit_extract_taps(C.byref(m.cfg), C.byref(m.struct), _lib.ptr(img), B, H, W, _lib.ptr(pos),
                                           arr, len(taps), 0, 1, _lib.ptr(ws), nbytes if ws_bytes is None else ws_bytes,
                                           _lib.ENGINE["tc3"], _lib.stream_ptr())

    good = [(l, _lib.FACET[f], o.data_ptr()) for (l, f), o in zip(pairs, outs)]
    refusals = [(good + [(1, _lib.FACET["key"], outs[0].data_ptr())], _lib.ERR["arg"]),
                (good[:2] + [(6, 0, outs[2].data_ptr())], _lib.ERR["arg"]),
                (good[:2] + [(2, 4, outs[2].data_ptr())], _lib.ERR["arg"]),
                (good[:3] + [(3, 0, None)], _lib.ERR["arg"])]
    for taps, rc in refusals:
        assert call(taps) == rc, _lib.last_error()
    assert call(good, ws_bytes=4096) == _lib.ERR["workspace"]
    torch.cuda.synchronize()
    assert all(bool(torch.isnan(o).all()) for o in outs)
    assert call(good) == 0, _lib.last_error()
    torch.cuda.synchronize()
    for (layer, facet), o in zip(pairs, outs):
        assert bool(torch.isnan(o[rows:]).all()), (layer, facet)
        assert torch.equal(o[:rows].view(B, rows // B, -1), m.extract(img, layer, facet, engine="tc3"))


def test_precision_auto_switches_to_tf32(u):
    from tests.test_vit_gpu import _outlier_weights
    wild = _outlier_weights("dinov2_vits14", 4, 3000.0).state_dict()
    taps = [(1, "token"), (3, "value"), (3, "query"), (2, "key")]
    img = _img(2, 224, 224)
    ref = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=wild, precision="tf32x3")(img)
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=wild)
    assert ext.precision == "f16x3"
    out = ext(img)
    assert ext.precision == "tf32x3" and ext.dino_model.pair == "tf32" and ext.dino_model.depth == 4
    assert all(torch.equal(out[t], ref[t]) for t in taps)
    assert all(torch.equal(a, b) for t in taps for a, b in zip(ext([img[0], img[1]])[t], [ref[t][0], ref[t][1]]))
