"""List input to the extractor: differently sized images in one packed forward pass (anyloc_vit_extract_varlen).
Every image's features must be BIT-IDENTICAL to a call on that image alone with the same GEMM engine, so the feature
adds no tolerance; the oracle check ties the packed path to the reference model as well."""
import ctypes as C
import random

import pytest
import torch

from oracle import anyloc_oracle as ao
from oracle import dinov2_restated as dr
from tests.util import rel_inf

pytestmark = pytest.mark.gpu
TOL = 1e-4
# T = 257, 64, 65, 2, 1370 (the pretrained grid: identity positional table), 1531, 257 again (a repeated grid, not
# adjacent), 129, 3943 (a 4032x3024 photo under the demo's resize rule)
SIZES = [(224, 224), (98, 126), (112, 112), (14, 14), (518, 518), (476, 630), (224, 224), (112, 224), (756, 1022)]


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def _imgs(sizes, seed=1234):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(3, H, W, generator=g).cuda() for H, W in sizes]


def _check_bit_identical(u, name, sd, layer, sizes, precision, facets, engines=("tc3", "auto")):
    imgs = _imgs(sizes)
    for engine in engines:
        ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd, gemm_engine=engine,
                                      precision=precision)
        for facet in facets:
            for use_cls in (False, True):
                for norm in (True, False):
                    ext.facet, ext.use_cls, ext.norm_descs = facet, use_cls, norm
                    out = ext(imgs)
                    assert isinstance(out, list) and len(out) == len(imgs)
                    for i, x in enumerate(imgs):
                        T = (x.shape[1] // 14) * (x.shape[2] // 14) + 1
                        if engine == "auto" and T < 32:
                            continue        # alone, this image's GEMMs take the SIMT engine under "auto"
                        ref = ext(x[None])[0]
                        assert out[i].shape == ref.shape, (i, out[i].shape, ref.shape)
                        assert torch.equal(out[i], ref), (engine, facet, use_cls, norm, sizes[i],
                                                          (out[i] - ref).abs().max().item())


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_list_bit_identical_to_per_image_calls_vits(u, precision):
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=4), seed=1).state_dict()
    _check_bit_identical(u, "dinov2_vits14", sd, 3, SIZES, precision, ("query", "key", "value", "token"))


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_list_bit_identical_to_per_image_calls_vitg(u, precision):
    """SwiGLU blocks, D = 1536 (24 heads)"""
    sd = dr.perturb(dr.build("dinov2_vitg14", seed=0, depth_override=2), seed=1).state_dict()
    _check_bit_identical(u, "dinov2_vitg14", sd, 1, [(322, 322), (224, 308), (518, 518)], precision,
                         ("value", "token"), engines=("tc3",))


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_equal_sizes_match_the_stacked_batch(u, precision):
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=4), seed=1).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=sd, precision=precision)
    imgs = _imgs([(98, 154)] * 5)
    assert torch.equal(torch.stack(ext(imgs)), ext(torch.stack(imgs)))
    assert torch.equal(torch.stack(ext(tuple(x[None] for x in imgs))), ext(torch.stack(imgs)))


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_list_vs_oracle(u, precision):
    model = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=4), seed=2)
    imgs = _imgs([(98, 154), (224, 224), (14, 28), (140, 112)], seed=7)
    for facet in ("value", "token"):
        ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, facet, device="cuda", weights=model.state_dict(),
                                      precision=precision)
        out = ext(imgs)
        for x, o in zip(imgs, out):
            ref = ao.extract_features(model, x[None].cpu(), 3, facet)[0]
            err = rel_inf(o.cpu(), ref)
            assert err < TOL, (facet, tuple(x.shape), err)


def _small_sizes(n, seed):
    """n images with sides of 14..126 px (1..9 patches), among them equal patch counts in different shapes"""
    rng = random.Random(seed)
    sides = [14 * k for k in range(1, 10)]
    sizes = [(28, 56), (56, 28), (14, 112), (112, 14), (42, 84), (84, 42), (14, 126), (126, 14), (14, 14), (126, 126)]
    sizes += [(rng.choice(sides), rng.choice(sides)) for _ in range(n - len(sizes))]
    rng.shuffle(sizes)
    return sizes


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3", "bf16"])
def test_full_tables_bit_identical_to_per_image_calls(u, precision):
    """ViT-S with 2 blocks: 128 small images fill one call's table (ANYLOC_VIT_VARLEN_MAX_B entries), 300 run as three
    calls (128, 128, 44) into one output; every image's rows equal its lone call's"""
    from anyloc_b200 import _lib
    assert _lib.VIT_VARLEN_MAX_B == 128
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=2), seed=1).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd, gemm_engine="tc3",
                                  precision=precision)
    for n in (128, 300):
        imgs = _imgs(_small_sizes(n, seed=n), seed=n)
        for facet in ("value", "token"):
            ext.facet = facet
            out = ext(imgs)
            assert len(out) == n
            for i, x in enumerate(imgs):
                assert torch.equal(out[i], ext(x[None])[0]), (precision, n, facet, i, tuple(x.shape))


def test_list_is_one_forward_pass(u):
    from anyloc_b200 import _lib
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=4), seed=1).state_dict()
    for facet in ("value", "token"):
        ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, facet, device="cuda", weights=sd, gemm_engine="tc3",
                                      precision="tf32x3")
        imgs = _imgs(SIZES)
        ext(imgs[:1]); ext(imgs[0][None])                 # first use: nothing lazily launched inside the count
        n0 = _lib.launch_count(); ext(imgs[0][None]); one = _lib.launch_count() - n0
        n0 = _lib.launch_count(); ext(imgs); many = _lib.launch_count() - n0
        assert one == many, (facet, one, many)


def test_list_feeds_vlad(u):
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=4), seed=1).state_dict()
    # tc3: the list holds a 14x14 image, whose lone call would take the SIMT GEMMs under "auto"
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=sd, gemm_engine="tc3")
    imgs = _imgs(SIZES[:8])
    feats = ext(imgs)
    v = u.VLAD(8)
    v.fit(torch.cat(feats).cpu())
    per_image = [ext(x[None])[0] for x in imgs]
    vl = v.generate_multi(feats)
    assert torch.equal(vl, v.generate_multi(per_image))
    assert torch.equal(vl, torch.stack([v.generate(f) for f in per_image]))


def test_varlen_abi_edges(u):
    from anyloc_b200 import _lib, vit
    lib = _lib.load()
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=4), seed=1).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=sd, gemm_engine="tc3",
                                  precision="tf32x3")
    m = ext.dino_model
    sizes = [(98, 126), (224, 224), (14, 14)]
    imgs = _imgs(sizes)
    B, D, canary = len(sizes), m.dim, 5
    lay = vit.VarlenLayout(sizes, use_cls=False, max_b=_lib.VIT_VARLEN_MAX_B)
    hw = (C.c_int32 * (2 * B))(*[v for s in sizes for v in s])
    img_p = (C.c_void_p * B)(*[x.data_ptr() for x in imgs])
    pos_p = (C.c_void_p * B)(*[m.pos_for(*g).data_ptr() for g in lay.grids])
    nbytes = lib.anyloc_vit_varlen_workspace_bytes(C.byref(m.cfg), B, hw)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")

    def call(out, ws_bytes=nbytes, engine="tc3", n=B, hw_=hw):
        return lib.anyloc_vit_extract_varlen(C.byref(m.cfg), C.byref(m.struct), n, img_p, hw_, pos_p, 3,
                                             _lib.FACET["value"], 0, 1, _lib.ptr(out), _lib.ptr(ws), ws_bytes,
                                             _lib.ENGINE[engine], _lib.stream_ptr())

    out = torch.full((lay.rows + canary, D), float("nan"), device="cuda")
    assert call(out) == 0, _lib.last_error()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out[:lay.rows]).all())
    assert bool(torch.isnan(out[lay.rows:]).all())
    for i, x in enumerate(imgs):
        assert torch.equal(out[lay.row0[i]:lay.row0[i + 1]], ext(x[None])[0])
    assert call(out, ws_bytes=nbytes - 8192) == _lib.ERR["workspace"]
    assert call(out, engine="simt") == _lib.ERR["unsupported"]
    assert call(out, n=_lib.VIT_VARLEN_MAX_B + 1) == _lib.ERR["arg"]
    bad = (C.c_int32 * (2 * B))(98, 126, 224, 220, 14, 14)
    assert call(out, hw_=bad) == _lib.ERR["arg"] and "multiples of the patch size" in _lib.last_error()


def test_list_precision_guards(u):
    from anyloc_b200 import _lib
    from tests.test_vit_gpu import _outlier_weights
    wild = _outlier_weights("dinov2_vits14", 4, 3000.0).state_dict()
    imgs = _imgs([(224, 224), (98, 126), (140, 112)])
    ref = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=wild, precision="tf32x3")(imgs)
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=wild)       # auto
    assert ext.precision == "f16x3"
    out = ext(imgs)
    assert ext.precision == "tf32x3"
    assert all(torch.equal(a, b) for a, b in zip(out, ref))
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=wild, precision="f16x3")
    with pytest.raises(_lib.AnylocError, match="overflowed the fp16 operand range"):
        ext(imgs)
    ext.check_finite = "deferred"
    ext(imgs)
    with pytest.raises(_lib.AnylocError):
        ext.raise_if_overflowed()


def test_list_input_errors(u):
    sd = dr.build("dinov2_vits14", seed=0, depth_override=4).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 3, "value", device="cuda", weights=sd)
    good = torch.randn(3, 28, 28, device="cuda")
    for bad in ([], [good, torch.randn(28, 28, device="cuda")], [good, torch.randn(2, 3, 28, 28, device="cuda")],
                [good, torch.randn(3, 28, 30, device="cuda")], [good, torch.randn(3, 28, 28)]):
        with pytest.raises(ValueError):
            ext(bad)
