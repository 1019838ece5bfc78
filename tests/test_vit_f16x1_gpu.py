"""The single-fp16 precision of the DINOv2 extractor (precision="f16x1") on the GPU.

Every error below is measured against the restated model in fp64, on ViT-S at full depth, a 4-block SwiGLU ViT-G and a
register model, all four facets, two image sizes and both (use_cls, norm_descs) settings.  Two errors per output:
the relative RMS error |f - f64|_F / |f64|_F and the max-element error max|f - f64| / max|f64|.
  - Autocast yardstick: the same model run the common PyTorch way, under torch.autocast("cuda", torch.float16).  Each
    output's RMS error must not exceed autocast's, and its max-element error must stay within 1.5x autocast's (one
    element's luck; see tests/test_vit_bf16_gpu.py for why the max-element error alone is not a sound yardstick).
  - Against bf16: this tier exists to be several times more accurate than precision="bf16" at the same speed, so its
    RMS error must be below bf16's divided by BF16_MARGIN on every output.  fp16 keeps 11 significant bits against
    bf16's 8, an 8x finer rounding per operand.  BF16_MARGIN = 4, half the smallest ratio measured on an H100 (7.95 on
    ViT-S, 8.01 on ViT-G, 7.96 on the register model); the worst f16x1 / autocast ratios there were 0.77 (RMS) and
    1.13 (max-element).
Beside that: the bitwise invariances of bf16 (list input equals single calls at every size, with up to 128 images in
one table; every tap equals the single-tap call, which makes the qkv tap kernel's single-fp16 operands those of the
GEMM epilogue), and the fp16-range guard on outlier activations."""
import copy

import pytest
import torch

from oracle import anyloc_oracle as ao
from oracle import dinov2_restated as dr
from tests import dinov2_reg_restated as rr
from tests.test_vit_gpu import _outlier_weights

pytestmark = pytest.mark.gpu
FACETS = ("query", "key", "value", "token")
CLS_NORM = ((False, True), (True, False))
BF16_MARGIN = 4.0


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def _img(B, H, W, seed=1234):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed))


def rel_err(f, ref):
    """(max-element, RMS) relative error"""
    f, ref = f.double().cpu(), ref.double().cpu()
    return float((f - ref).abs().max() / ref.abs().max()), float((f - ref).norm() / ref.norm())


ACCURACY = [("dinov2_vits14", None, 11), ("dinov2_vitg14", 4, 3), ("dinov2_vitb14_reg", 3, 2)]


@pytest.mark.parametrize("name,depth,layer", ACCURACY, ids=[a[0] for a in ACCURACY])
def test_error_against_fp16_autocast_and_bf16(u, name, depth, layer):
    from anyloc_b200 import vit
    model = rr.model(name, depth) if name.endswith("_reg") else dr.perturb(dr.build(name, depth_override=depth), 1)
    sd = model.state_dict()
    h1, b16 = (vit.VitWeights(name, sd, "cuda", pair=p) for p in ("f16x1", "bf16"))
    model64 = copy.deepcopy(model).double()
    model_gpu = copy.deepcopy(model).cuda()
    rows = []
    for hw in ((224, 224), (98, 154)):
        img = _img(2, *hw)
        for facet in FACETS:
            for use_cls, norm in CLS_NORM:
                ref = ao.extract_features(model64, img.double(), layer, facet, use_cls, norm)
                with torch.autocast("cuda", dtype=torch.float16):
                    amp = ao.extract_features(model_gpu, img.cuda(), layer, facet, use_cls, norm)
                out = h1.extract(img.cuda(), layer, facet, use_cls, norm)
                assert out.dtype == torch.float32 and out.shape == ref.shape
                e_bf = rel_err(b16.extract(img.cuda(), layer, facet, use_cls, norm), ref)
                rows.append((hw, facet, use_cls, norm, rel_err(out, ref), rel_err(amp, ref), e_bf))
    for hw, facet, use_cls, norm, e, e_amp, e_bf in rows:
        print(f"{name} L{layer} {hw} {facet:5s} cls={int(use_cls)} norm={int(norm)}: max-element f16x1 {e[0]:.3e} "
              f"autocast {e_amp[0]:.3e} bf16 {e_bf[0]:.3e}; RMS f16x1 {e[1]:.3e} autocast {e_amp[1]:.3e} "
              f"bf16 {e_bf[1]:.3e} (bf16 / f16x1 {e_bf[1] / e[1]:.2f})")
    print(f"{name}: smallest bf16 / f16x1 RMS ratio {min(r[6][1] / r[4][1] for r in rows):.2f}")
    bad = [r for r in rows if r[4][1] > r[5][1] or r[4][0] > 1.5 * r[5][0]]
    assert not bad, bad
    bad = [r for r in rows if r[4][1] * BF16_MARGIN > r[6][1]]
    assert not bad, bad


SIZES = [(56, 70), (14, 14), (98, 42), (224, 224), (42, 28)]      # 21, 2, 22, 257 and 7 tokens


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vits14_reg"])
def test_list_input_equals_single_calls_at_every_size(u, name):
    """no SIMT route for f16x1: a lone image of fewer than 32 tokens is bit-identical under the default engine too"""
    sd = (rr.model(name, 4) if name.endswith("_reg") else dr.perturb(dr.build(name, depth_override=4), 1)).state_dict()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for facet in FACETS:
        for use_cls, norm in CLS_NORM:
            ext = u.DinoV2ExtractFeatures(name, 3, facet, use_cls, norm, device="cuda", weights=sd, precision="f16x1")
            assert ext.precision == "f16x1" and ext.gemm_engine == "auto" and ext.dino_model.pair == "f16x1"
            out = ext(imgs)
            for x, got in zip(imgs, out):
                assert torch.equal(got, ext(x[None])[0]), (name, facet, use_cls, norm, tuple(x.shape))


def test_a_full_table_of_128_images(u):
    sd = dr.perturb(dr.build("dinov2_vits14", depth_override=2), 1).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 1, "key", device="cuda", weights=sd, precision="f16x1")
    g = torch.Generator().manual_seed(3)
    imgs = [torch.randn(3, 14 * (1 + i % 5), 14 * (1 + (i * 7) % 4), generator=g).cuda() for i in range(130)]
    out = ext(imgs)
    for i in (0, 1, 63, 127, 128, 129):
        assert torch.equal(out[i], ext(imgs[i][None])[0]), i


def test_multi_taps_equal_single_taps(u):
    sd = dr.perturb(dr.build("dinov2_vits14"), 1).state_dict()
    taps = [(l, f) for l in range(12) for f in FACETS][::-1]
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=sd, precision="f16x1")
    m = ext.dino_model
    assert m.pair == "f16x1"
    img = _img(3, 70, 42).cuda()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for use_cls, norm in CLS_NORM:
        ext.use_cls, ext.norm_descs = use_cls, norm
        out, out_list = ext(img), ext(imgs)
        for layer, facet in taps:
            assert torch.equal(out[(layer, facet)], m.extract(img, layer, facet, use_cls, norm)), (layer, facet)
            ref, _ = m.extract_varlen(imgs, layer, facet, use_cls, norm)
            assert torch.equal(torch.cat(out_list[(layer, facet)]), ref), (layer, facet)


def test_register_model_taps_and_rows_do_not_depend_on_the_batch(u):
    name = "dinov2_vitb14_reg"
    sd = rr.model(name, 3).state_dict()
    taps = [(0, "value"), (2, "token"), (2, "query"), (1, "key")]
    ext = u.DinoV2MultiExtractFeatures(name, taps, device="cuda", weights=sd, precision="f16x1")
    img = _img(4, 56, 84).cuda()
    out = ext(img)
    for layer, facet in taps:
        one = ext.dino_model.extract(img[1:2], layer, facet)
        assert torch.equal(out[(layer, facet)][1:2], one), (layer, facet)


def test_outliers_stay_finite_or_raise_with_the_bf16_remedy(u):
    """x100 outlier channels stay inside fp16's range; x3000 ones (|8 x| > 65504) raise in the default sync mode, at
    the next call in the deferred mode, and come back non-finite with the guard off"""
    from anyloc_b200 import _lib
    name, layer = "dinov2_vits14", 3
    img = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(1234)).cuda()
    mild = _outlier_weights(name, 4, 100.0)
    ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=mild.state_dict(), precision="f16x1")
    assert torch.isfinite(ext(img)).all()
    wild = _outlier_weights(name, 4, 3000.0).float().state_dict()
    ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=wild, precision="f16x1")
    with pytest.raises(_lib.AnylocError, match="precision='bf16'"):
        ext(img)
    assert ext.precision == "f16x1"
    ext.check_finite = "deferred"
    ext(img)
    with pytest.raises(_lib.AnylocError, match="precision='bf16'"):
        ext(img)
    ext.check_finite = "off"
    assert not bool(torch.isfinite(ext(img)).all())
    ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=wild, precision="bf16")
    assert torch.isfinite(ext(img)).all()


def test_precision_from_the_environment_and_simt_refusal(u, monkeypatch):
    sd = dr.build("dinov2_vits14", depth_override=2).state_dict()
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "f16x1")
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd)
    assert ext.precision == "f16x1" and ext.dino_model.pair == "f16x1"
    img = _img(2, 56, 56).cuda()
    assert torch.isfinite(ext(img)).all()
    with pytest.raises(ValueError):
        u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd, gemm_engine="simt")
    from anyloc_b200 import _lib
    with pytest.raises(_lib.AnylocError, match="tensor-core"):
        ext.dino_model.extract(img, 1, "value", engine="simt")
    monkeypatch.delenv("ANYLOC_B200_PRECISION")
    assert u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd).precision == "f16x3"
