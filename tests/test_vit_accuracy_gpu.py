"""Every (layer, facet) output of the fp32-equivalent ViT forward (precision "tf32x3" and "f16x3") against the same
model in fp64, calibrated against that model in IEEE fp32.

The parity tests (test_vit_gpu.py and its siblings) bound max|f - f32| / max|f32| by 1e-4 against the fp32 oracle;
an operand that loses its lo word at one conversion point (2^-11 instead of ~2^-21), a LayerNorm eps of 1e-5 or a
tanh GELU moves the features by 1e-6 .. 1e-4 of their maximum and can pass that.  Here each output f of a forward
and its fp64 reference f64 (the restated model, oracle/dinov2_restated.py and tests/dinov2_reg_restated.py, on the
CPU in fp64) give, with rows taken along D,
  worst row  max_r |f_r - f64_r| / |f64_r|      and      RMS  |f - f64|_F / |f64|_F,
and the same two statistics of the CPU fp32 forward (the control, checked to run IEEE fp32; the worst of three
evaluations in different summation orders, see refs) set the scale: each statistic must stay within
KAPPA_* x max(control's statistic, 4u), u = 2^-24.  A 3-term GEMM reads its lo words as tf32, so operand errors of
about 2^-21 against fp32's 2^-24 are expected and ratios of a few are normal.

Covered: ViT-S at full depth (MLP, LayerNorm template 4), dinov2_vitb14_reg 3 blocks (registers, template 8),
ViT-L 3 blocks (D = 1024), ViT-G 4 blocks (SwiGLU, template 16, 24 heads); perturbed random weights and "trained-like"
ones (LayerScale log-uniform 1e-5 .. 1, outlier channels x100 inside the fp16 range); tf32x3 and f16x3 on the
tensor-core and the SIMT engine, and "auto" on a 14x28 image (T = 3: SIMT GEMMs); B = 2 images of 224^2 (T = 257),
98x154 (T = 78) and 112^2 (T = 65, one row past a 64-row tile); (use_cls, norm_descs) = (False, True), (True, False).
All taps come from one DinoV2MultiExtractFeatures call (test_vit_taps_gpu.py proves each bit-identical to its
single-tap call, so this covers every route of the forward); one DinoV2ExtractFeatures with the drop-in defaults
per case adds the deepest layer's value facet through its own third of the qkv GEMM.

Measured on an H100 80GB HBM3 (700 W power limit), worst (row, RMS) ratio over both weight sets and all images
("single": DinoV2ExtractFeatures on the deepest value facet, the drop-in default and tf32x3 on the tensor cores):
             tf32x3 tc3  tf32x3 simt  f16x3 tc3  f16x3 simt  auto 14x28  single default  single tf32x3
  ViT-S      1.9, 1.6    5.9, 2.5     5.6, 4.7   5.3, 2.3    5.8, 3.5    4.3, 3.4        1.9, 1.2
  ViT-B reg  2.1, 1.6    2.1, 1.7     6.1, 5.0   2.6, 1.7    4.4, 3.1    3.7, 3.7        1.5, 1.2
  ViT-L      2.0, 1.6    2.2, 2.0     6.5, 5.6   2.3, 2.0    3.4, 2.7    4.1, 4.0        1.4, 1.2
  ViT-G      2.2, 1.7    3.4, 2.0     8.3, 5.8   3.2, 2.0    3.0, 2.8    4.5, 4.2        1.5, 1.3
KAPPA_* are at least 1.5x the worst (8.3 and 5.8), rounded up to a power of two.  Zeroing the lo word of the im2col
rows, of the qkv tap's operand pairs, of the GELU / SwiGLU outputs or of the fp16-pair attention's output, a LayerNorm
eps of 1e-5 in the forward or a tanh GELU each exceed KAPPA_ROW by 25x .. 760x.

The fp16 pair has an absolute floor: its lo half rounds to the fp16 subnormal step, 2^-25 / 8 = 2^-28 in x at the
activation scale 8, coarser than fp32 rounding below |x| ~ 2^-4.  test_small_activations_f16_floor scales one ViT-S
block's LayerNorm gains and biases and the qkv / fc1 biases by 1e-3, so that block's GEMM inputs have an RMS of 1e-3
(checked) and its q, k, v carry operand errors of ~36 u.  Measured: those taps are the worst of the forward on the
SIMT engine (row 3.6, RMS 3.6) and reach the RMS maximum on the tensor cores (5.4 / 4.7); both stay within KAPPA_*,
so the variant needs no bound of its own.  The single-tap cases assert which precision ran: "auto" stays f16x3 on
every weight set here."""
import copy
import math

import pytest
import torch
from torch.nn import functional as F

from oracle import anyloc_oracle as ao
from oracle import dinov2_restated as dr
from tests import dinov2_reg_restated as dreg

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FLOOR = 4 * U
KAPPA_ROW = 16.0
KAPPA_RMS = 16.0
FACETS = ("query", "key", "value", "token")
MODELS = {"vits": ("dinov2_vits14", 12), "vitb_reg": ("dinov2_vitb14_reg", 3), "vitl": ("dinov2_vitl14", 3),
          "vitg": ("dinov2_vitg14", 4)}
IMAGES = {"224x224": (224, 224), "98x154": (98, 154), "112x112": (112, 112)}
CONFIGS = [(p, e) for p in ("tf32x3", "f16x3") for e in ("tc3", "simt")]
OPTS = [(False, True), (True, False)]


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def check_ieee_fp32():
    """The control must be IEEE fp32: no reduced-precision fp32 matmul or convolution on the CPU backends."""
    assert torch.get_float32_matmul_precision() == "highest"
    for be in (torch.backends.mkldnn, torch.backends.mkldnn.matmul, torch.backends.mkldnn.conv):
        assert getattr(be, "fp32_precision", "none") in ("none", "ieee"), be
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(256, 512, generator=g), torch.randn(512, 256, generator=g)
    err = ((a @ b).double() - a.double() @ b.double()).abs().max() / (a.double().abs() @ b.double().abs()).max()
    assert float(err) < 64 * U, float(err)      # tf32 or bf16 would miss by 2^-11 .. 2^-8


def forward_taps(model, img):
    """{(layer, facet): [B, T, D]} of every layer and facet of one forward pass, with the cls row and not normalised:
    facet "token" is the output of blocks[layer], q/k/v the thirds of blocks[layer].attn.qkv(norm1(x)) (the hooks of
    ao.extract_features)"""
    out = {}
    with torch.no_grad():
        x = model.prepare_tokens(img)
        for layer, blk in enumerate(model.blocks):
            qkv = blk.attn.qkv(blk.norm1(x))
            for i, facet in enumerate(FACETS[:3]):
                out[(layer, facet)] = qkv[..., i * x.shape[-1]:(i + 1) * x.shape[-1]]
            x = blk(x)
            out[(layer, "token")] = x
    return out


def finish(raw, use_cls, norm_descs):
    """ao.extract_features' row selection and normalisation of a forward_taps output"""
    res = raw if use_cls else raw[:, 1:]
    return F.normalize(res, dim=-1) if norm_descs else res


def all_taps(model, img, use_cls, norm_descs):
    """every (layer, facet) output of one forward, as ao.extract_features returns each"""
    return {t: finish(r, use_cls, norm_descs) for t, r in forward_taps(model, img).items()}


_MODELS, _REFS = {}, {}


def _trained_like(key):
    from tests.test_vit_gpu import _outlier_weights
    name, depth = MODELS[key]
    if not name.endswith("_reg"):
        return _outlier_weights(name, depth, 100.0)
    model = dreg.model(name, depth_override=depth)
    sd = _outlier_weights(name[:-len("_reg")], depth, 100.0).state_dict()
    sd["register_tokens"] = model.register_tokens.detach().clone()
    model.load_state_dict(sd)
    return model


def model_of(key, weights):
    """the fp32 CPU model of a case (cached)"""
    if (key, weights) not in _MODELS:
        name, depth = MODELS[key]
        if weights == "trained":
            m = _trained_like(key)
        elif name.endswith("_reg"):
            m = dreg.model(name, depth_override=depth)
        else:
            m = dr.perturb(dr.build(name, seed=0, depth_override=depth), seed=1)
        _MODELS[(key, weights)] = m.float().eval()
    return _MODELS[(key, weights)]


def image(hw, seed=1234):
    return torch.randn(2, 3, *hw, generator=torch.Generator().manual_seed(seed + hw[0] * 1000 + hw[1]))


CONTROL_THREADS = (1, 2, 4)


def refs(key, weights, hw, model=None):
    """(fp64 raw taps, [fp32 raw taps, ...]) of a case, shared across precisions and engines.  The fp32 control runs
    once per count in CONTROL_THREADS: the CPU GEMMs block their sums by thread count, and on an ill-conditioned tap one
    summation order can be 10x luckier than another (ViT-S, trained-like weights, T = 3, layer 5: 7 u .. 94 u), so
    the control's statistic is the worst of these fp32 evaluations, each fixed whatever the machine's core count."""
    ck = (key, weights, hw) if model is None else None
    if ck in _REFS:
        return _REFS[ck]
    check_ieee_fp32()
    m32 = model_of(key, weights) if model is None else model
    img = image(hw)
    threads = torch.get_num_threads()
    try:
        r32 = []
        for n in CONTROL_THREADS:
            torch.set_num_threads(n)
            r32.append(forward_taps(m32, img))
        r64 = forward_taps(copy.deepcopy(m32).double(), img.double())
    finally:
        torch.set_num_threads(threads)
    if ck is not None:
        _REFS[ck] = (r64, r32)
    return r64, r32


def stats(f, ref):
    """(worst row, RMS) relative error of f against ref, rows along the last dimension"""
    f, ref = f.double(), ref.double()
    d = f - ref
    row = float((d.norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-300)).max())
    return row, float(d.norm() / ref.norm().clamp_min(1e-300))


def ratios(out, r64, r32, tap, use_cls, norm_descs):
    """(worst-row ratio, RMS ratio, kernel stats, control stats) of one output; r32: the fp32 controls (refs)"""
    ref = finish(r64[tap], use_cls, norm_descs)
    s = stats(out.cpu(), ref)
    cs = [stats(finish(r[tap], use_cls, norm_descs), ref) for r in r32]
    c = (max(x[0] for x in cs), max(x[1] for x in cs))
    return s[0] / max(c[0], FLOOR), s[1] / max(c[1], FLOOR), s, c


def report(case, worst):
    """print one table line: the case's worst ratios and the tap they came from"""
    (rr, tr), (rm, tm) = worst["row"], worst["rms"]
    print(f"ACC|{case}|row {rr:7.3f} @ {tr}|rms {rm:7.3f} @ {tm}")


def measure(outs_of, r64, r32, opts):
    """the worst ratios over every tap and option of one configuration; outs_of(use_cls, norm) -> {tap: tensor}"""
    worst = {"row": (0.0, None), "rms": (0.0, None)}
    for use_cls, norm in opts:
        for tap, out in outs_of(use_cls, norm).items():
            rr, rm, _, _ = ratios(out, r64, r32, tap, use_cls, norm)
            assert math.isfinite(rr) and math.isfinite(rm), (tap, use_cls, norm)
            if rr > worst["row"][0]:
                worst["row"] = (rr, (*tap, use_cls, norm))
            if rm > worst["rms"][0]:
                worst["rms"] = (rm, (*tap, use_cls, norm))
    return worst


def test_all_taps_helper_matches_extract_features():
    """forward_taps / all_taps give what ao.extract_features gives for a tap, bit for bit"""
    for key in ("vits", "vitb_reg"):
        m = model_of(key, "random")
        img = image((56, 70))
        for use_cls, norm in OPTS + [(False, False)]:
            got = all_taps(m, img, use_cls, norm)
            assert len(got) == 4 * MODELS[key][1]
            for tap in ((0, "query"), (1, "key"), (2, "token"), (2, "value")):
                assert torch.equal(got[tap], ao.extract_features(m, img, *tap, use_cls, norm)), (key, tap)


@pytest.mark.parametrize("weights", ["random", "trained"])
@pytest.mark.parametrize("key", list(MODELS))
def test_every_tap_against_fp64(u, monkeypatch, key, weights):
    monkeypatch.delenv("ANYLOC_B200_PRECISION", raising=False)        # the drop-in default is "auto"
    name, depth = MODELS[key]
    taps = [(l, f) for l in range(depth) for f in FACETS]
    sd = model_of(key, weights).state_dict()
    _REFS.clear()           # one case's references at a time: shared by its precisions and engines
    bad = []

    def check(case, worst):
        report(case, worst)
        if worst["row"][0] > KAPPA_ROW or worst["rms"][0] > KAPPA_RMS:
            bad.append((case, worst))

    for precision, engine in CONFIGS + [("tf32x3", "auto"), ("f16x3", "auto")]:
        ext = u.DinoV2MultiExtractFeatures(name, taps, device="cuda", weights=sd, gemm_engine=engine,
                                           precision=precision)
        assert ext.precision == precision
        sizes = [(14, 28)] if engine == "auto" else list(IMAGES.values())
        for hw in sizes:
            r64, r32 = refs(key, weights, hw)
            img = image(hw).cuda()

            def outs_of(use_cls, norm):
                ext.use_cls, ext.norm_descs = use_cls, norm
                return ext(img)

            check(f"{key}|{weights}|{precision}|{engine}|{hw[0]}x{hw[1]}", measure(outs_of, r64, r32, OPTS))
        del ext
    # the deepest layer's value facet alone (its own third of the qkv GEMM): the drop-in default (precision "auto",
    # which must stay f16x3 on these weights, engine "auto") and tf32x3 on the tensor cores
    for precision, engine in ((None, "auto"), ("tf32x3", "tc3")):
        ext = u.DinoV2ExtractFeatures(name, depth - 1, "value", device="cuda", weights=sd, gemm_engine=engine,
                                      precision=precision)
        for hw in IMAGES.values():
            r64, r32 = refs(key, weights, hw)
            img = image(hw).cuda()

            def one(use_cls, norm):
                ext.use_cls, ext.norm_descs = use_cls, norm
                return {(depth - 1, "value"): ext(img)}

            check(f"{key}|{weights}|{precision or 'default'}|single|{hw[0]}x{hw[1]}", measure(one, r64, r32, OPTS))
        assert ext.precision == (precision or "f16x3"), (precision, ext.precision)
        del ext
    assert not bad, bad


SMALL_BLOCK, SMALL = 5, 1e-3
F16_FLOOR = 2.0 ** -28       # the fp16 pair's absolute error in x at the activation scale 8: 2^-25 / 8


def small_activations_model():
    """ViT-S with block SMALL_BLOCK's LayerNorm gains and biases, and the biases of the GEMMs reading them (qkv, fc1),
    scaled by SMALL: that block's normalised activations and its q, k, v are ~SMALL instead of ~1"""
    m = dr.perturb(dr.build("dinov2_vits14", seed=0), seed=1)
    blk = m.blocks[SMALL_BLOCK]
    with torch.no_grad():
        for p in (blk.norm1.weight, blk.norm1.bias, blk.norm2.weight, blk.norm2.bias, blk.attn.qkv.bias,
                  blk.mlp.fc1.bias):
            p.mul_(SMALL)
    return m


def layernorm_rms(model, img):
    """{layer: (RMS, max |.|) of norm1's output} of one fp32 forward"""
    seen = {}

    def keep(layer):
        def hook(mod, inp, out):       # returns None: the output is left as it is
            seen[layer] = (float(out.pow(2).mean().sqrt()), float(out.abs().max()))
        return hook

    hooks = [blk.norm1.register_forward_hook(keep(l)) for l, blk in enumerate(model.blocks)]
    try:
        with torch.no_grad():
            model(img)
    finally:
        for h in hooks:
            h.remove()
    return seen


def test_small_activations_f16_floor(u):
    """ViT-S with one block's normalised activations at ~1e-3 (small_activations_model), in f16x3.  The fp16 pair of
    8 y rounds its lo half to the fp16 subnormal step 2^-24 once |8 y| < 2^-3, an absolute error of up to
    F16_FLOOR = 2^-28 in y: at an RMS of 1e-3 that is 2^-28 / sqrt(3) / 1e-3 ~ 36 u relative per operand, far above
    fp32's u.  It enters that block's q, k and v directly; the block's attention and FFN outputs reach the residual
    stream through LayerScale next to O(1) values, where it vanishes.  The LayerNorm outputs are checked to be that
    small, and every tap is held to the KAPPA_* of the other cases (see the module docstring for what it measures)."""
    m = small_activations_model()
    taps = [(l, f) for l in range(12) for f in FACETS]
    bad = []
    for hw in ((224, 224), (112, 112)):
        ln = layernorm_rms(m, image(hw))
        rms, amax = ln[SMALL_BLOCK]
        assert 0.3 * SMALL < rms < 3 * SMALL and amax < 30 * SMALL, (rms, amax)        # the operands really are small
        assert F16_FLOOR / rms > 16 * U                     # ... so small that the floor is above fp32 rounding
        assert all(0.3 < ln[l][0] for l in ln if l != SMALL_BLOCK), ln
        r64, r32 = refs(None, None, hw, model=m)
        img = image(hw).cuda()
        for engine in ("tc3", "simt"):
            ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=m.state_dict(),
                                               gemm_engine=engine, precision="f16x3")

            def outs_of(use_cls, norm):
                ext.use_cls, ext.norm_descs = use_cls, norm
                return ext(img)

            worst = measure(outs_of, r64, r32, OPTS)
            case = f"vits-small-activations|random|f16x3|{engine}|{hw[0]}x{hw[1]}"
            report(case, worst)
            if worst["row"][0] > KAPPA_ROW or worst["rms"][0] > KAPPA_RMS:
                bad.append((case, worst))
    assert not bad, bad
