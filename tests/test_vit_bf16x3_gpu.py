"""The bf16-pair precision of the DINOv2 extractor (precision="bf16pair") on the GPU.

Accuracy: every (layer, facet) output f of a forward against the restated model in fp64, as the worst row error
max_r |f_r - f64_r| / |f64_r| and the RMS error |f - f64|_F / |f64|_F, each divided by the same statistic of the fp64
emulation of the format (tests/test_vit_bf16x3_cpu.rounding_bf16x3: every rounding point of the forward rounded to its
bf16 pair).  The kernels also drop each product's lo.lo term (2^-16 relative, the order of the pair rounding itself),
round P relative to the running maximum and accumulate in fp32, none of which the emulation models, so ratios
somewhat above 1 are normal; each must stay within KAPPA_ROW / KAPPA_RMS.  Covered: ViT-S at full depth, a 3-block
ViT-B with registers and a 3-block SwiGLU ViT-G, random weights, two image sizes and both (use_cls, norm_descs).

Outliers: the x3000 outlier-channel weights of tests/test_vit_gpu.test_outlier_activations_precision_contract overflow
fp16 (f16x3 raises); bf16pair has fp32's exponent range, so it returns finite features, held to the same KAPPA_* against
its emulation.

Beside that, the invariances of the single-MMA formats: list input equals single calls at every size (no SIMT route),
up to 128 images in one table; every tap equals the single-tap call; a register model's rows do not depend on the
batch; and precision="auto" is unchanged (f16x3, then tf32x3 on an overflow, never bf16pair)."""
import copy

import pytest
import torch

from oracle import dinov2_restated as dr
from tests import dinov2_reg_restated as rr
from tests.test_vit_accuracy_gpu import FACETS, OPTS, forward_taps, image, measure, report
from tests.test_vit_bf16x3_cpu import rounding_bf16x3
from tests.test_vit_gpu import _outlier_weights
from tests.test_vit_single_accuracy_gpu import emulated

pytestmark = pytest.mark.gpu
KAPPA_ROW = 5.0
KAPPA_RMS = 3.0
CLS_NORM = ((False, True), (True, False))


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def _img(B, H, W, seed=1234):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed))


def check_every_tap(u, name, model, hws, label):
    """ACC lines, and the cases over KAPPA_*, of every tap of one model (one DinoV2MultiExtractFeatures call) and of
    the deepest value facet alone (its own N = D third of the qkv GEMM)"""
    depth = len(model.blocks)
    taps = [(l, f) for l in range(depth) for f in FACETS]
    sd = model.state_dict()
    multi = u.DinoV2MultiExtractFeatures(name, taps, device="cuda", weights=sd, precision="bf16pair")
    single = u.DinoV2ExtractFeatures(name, depth - 1, "value", device="cuda", weights=sd, precision="bf16pair")
    assert multi.precision == single.precision == "bf16pair" and multi.dino_model.pair == "bf16pair"
    bad = []
    for hw in hws:
        img = image(hw)
        r64 = forward_taps(copy.deepcopy(model).double(), img.double())
        emu = [forward_taps(emulated(model, rounding_bf16x3()), img.double())]
        img_d = img.cuda()

        def every_tap(use_cls, norm):
            multi.use_cls, multi.norm_descs = use_cls, norm
            return multi(img_d)

        def deepest_value(use_cls, norm):
            single.use_cls, single.norm_descs = use_cls, norm
            return {(depth - 1, "value"): single(img_d)}

        for what, outs_of in (("taps", every_tap), ("single", deepest_value)):
            worst = measure(outs_of, r64, emu, OPTS)
            case = f"{label}|bf16pair|{what}|{hw[0]}x{hw[1]}"
            report(case, worst)
            if worst["row"][0] > KAPPA_ROW or worst["rms"][0] > KAPPA_RMS:
                bad.append((case, worst))
    return bad


ACCURACY = [("dinov2_vits14", None), ("dinov2_vitb14_reg", 3), ("dinov2_vitg14", 3)]


@pytest.mark.parametrize("name,depth", ACCURACY, ids=[a[0] for a in ACCURACY])
def test_every_tap_against_fp64(u, name, depth):
    model = rr.model(name, depth) if name.endswith("_reg") else dr.perturb(dr.build(name, depth_override=depth), 1)
    bad = check_every_tap(u, name, model.float().eval(), [(224, 224), (98, 154)], name)
    assert not bad, bad


def test_outliers_stay_finite_where_f16x3_raises(u):
    from anyloc_b200 import _lib
    name, layer = "dinov2_vits14", 3
    wild = _outlier_weights(name, 4, 3000.0).float().eval()
    sd = wild.state_dict()
    img = _img(2, 224, 224)
    ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd, precision="f16x3")
    with pytest.raises(_lib.AnylocError, match="overflowed"):
        ext(img.cuda())
    bad = check_every_tap(u, name, wild, [(224, 224)], "vits-outliers-x3000")
    assert not bad, bad
    ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd, precision="bf16pair")
    ext.check_finite = "sync"
    assert torch.isfinite(ext(img.cuda())).all()


SIZES = [(56, 70), (14, 14), (98, 42), (224, 224), (42, 28)]      # 21, 2, 22, 257 and 7 tokens


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vits14_reg"])
def test_list_input_equals_single_calls_at_every_size(u, name):
    """no SIMT route for bf16pair: a lone image of fewer than 32 tokens is bit-identical under the default engine too"""
    sd = (rr.model(name, 4) if name.endswith("_reg") else dr.perturb(dr.build(name, depth_override=4), 1)).state_dict()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for facet in FACETS:
        for use_cls, norm in CLS_NORM:
            ext = u.DinoV2ExtractFeatures(name, 3, facet, use_cls, norm, device="cuda", weights=sd, precision="bf16pair")
            assert ext.precision == "bf16pair" and ext.gemm_engine == "auto" and ext.dino_model.pair == "bf16pair"
            out = ext(imgs)
            for x, got in zip(imgs, out):
                assert torch.equal(got, ext(x[None])[0]), (name, facet, use_cls, norm, tuple(x.shape))


def test_a_full_table_of_128_images(u):
    sd = dr.perturb(dr.build("dinov2_vits14", depth_override=2), 1).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 1, "key", device="cuda", weights=sd, precision="bf16pair")
    g = torch.Generator().manual_seed(3)
    imgs = [torch.randn(3, 14 * (1 + i % 5), 14 * (1 + (i * 7) % 4), generator=g).cuda() for i in range(130)]
    out = ext(imgs)
    for i in (0, 1, 63, 127, 128, 129):
        assert torch.equal(out[i], ext(imgs[i][None])[0]), i


def test_multi_taps_equal_single_taps(u):
    """every tap of a 12-layer call equals the single-tap call, padded and packed: the qkv tap kernel's bf16 pairs are
    the GEMM epilogue's"""
    sd = dr.perturb(dr.build("dinov2_vits14"), 1).state_dict()
    taps = [(l, f) for l in range(12) for f in FACETS][::-1]
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=sd, precision="bf16pair")
    m = ext.dino_model
    assert m.pair == "bf16pair"
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
    ext = u.DinoV2MultiExtractFeatures(name, taps, device="cuda", weights=sd, precision="bf16pair")
    img = _img(4, 56, 84).cuda()
    out = ext(img)
    for layer, facet in taps:
        one = ext.dino_model.extract(img[1:2], layer, facet)
        assert torch.equal(out[(layer, facet)][1:2], one), (layer, facet)
        lst, _ = ext.dino_model.extract_varlen([img[1], img[3]], layer, facet)
        assert torch.equal(lst, torch.cat([one[0], ext.dino_model.extract(img[3:4], layer, facet)[0]])), (layer, facet)


def test_auto_is_unchanged(u, monkeypatch):
    """"auto" starts in f16x3 and, on the x3000 outliers, redoes the call in tf32x3 -- never bf16pair; the environment
    variable selects bf16pair, and gemm_engine="simt" refuses it"""
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)
    name, layer = "dinov2_vits14", 3
    sd = _outlier_weights(name, 4, 3000.0).float().state_dict()
    img = _img(2, 224, 224).cuda()
    ext = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd)
    assert ext.precision == "f16x3" and ext._auto
    out = ext(img)
    assert ext.precision == "tf32x3" and ext.dino_model.pair == "tf32"
    ref = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd, precision="tf32x3")
    assert torch.equal(out, ref(img))
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "bf16pair")
    env = u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd)
    assert env.precision == "bf16pair" and env.dino_model.pair == "bf16pair" and torch.isfinite(env(img)).all()
    with pytest.raises(ValueError):
        u.DinoV2ExtractFeatures(name, layer, "value", device="cuda", weights=sd, gemm_engine="simt")
    from anyloc_b200 import _lib
    with pytest.raises(_lib.AnylocError, match="tensor-core"):
        env.dino_model.extract(img, layer, "value", engine="simt")
