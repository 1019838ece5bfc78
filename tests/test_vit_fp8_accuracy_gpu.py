"""Every (layer, facet) output of the single-e4m3 ViT forward (precision "fp8") against the same model in fp64,
calibrated against an fp64 emulation of the same quantisation points.

tests/test_vit_fp8_gpu.py holds one tap per model, by RMS over all rows, to within 1.1x of the emulation's RMS.  That
lets through an error confined to a few rows (an M tail, the cls or register rows: the RMS over 500 rows dilutes it),
an error at another layer or facet, and one that only trained checkpoints provoke (one x100 channel sets a whole row's
e4m3 scale).  Here, as in tests/test_vit_accuracy_gpu.py, each output f of a forward and its fp64 reference f64 give
  worst row  max_r |f_r - f64_r| / |f64_r|      and      RMS  |f - f64|_F / |f64|_F,
and the control is test_vit_fp8_gpu.emulated(): the restated model in fp64 with this precision's quantisation points
(bf16 pixels and patch weights, e4m3 weights with one power-of-two scale each, e4m3 rows in front of every block GEMM,
bf16 q / k / v and GEMM outputs), whose own statistics against f64 set the scale.  Each statistic must stay within
KAPPA_* x the control's.  The emulation leaves out the attention's bf16 rounding of P and the GEMMs' fp32
accumulation, so ratios somewhat above 1 are normal.

Covered: the four MODELS of test_vit_accuracy_gpu.py (ViT-S at full depth, ViT-B with registers, ViT-L, ViT-G with
SwiGLU), random and trained-like weights (LayerScale 1e-5 .. 1, outlier channels x100), B = 2 images of 224^2 (T = 257),
98x154 (T = 78), 112^2 (T = 65, one row past a 64-row tile) and 14x28 (T = 3, far below one tile), and both
(use_cls, norm_descs) settings.  Every tap comes from one DinoV2MultiExtractFeatures call; one DinoV2ExtractFeatures
adds the deepest layer's value facet through its own third of the qkv GEMM.

Measured on an H100 80GB HBM3 (700 W power limit), worst (row, RMS) ratio over the four images and both options
("taps": the DinoV2MultiExtractFeatures call, "single": the deepest value facet alone):
                 random taps   random single   trained taps   trained single
  ViT-S          1.15, 1.06    1.15, 1.06      2.75, 1.49     1.24, 1.06
  ViT-B reg      1.11, 1.01    1.06, 1.01      1.49, 1.08     1.21, 1.06
  ViT-L          1.06, 1.02    1.06, 1.00      1.19, 1.06     1.19, 1.06
  ViT-G          1.07, 1.01    1.02, 1.00      1.36, 1.34     1.31, 1.16
KAPPA_* are at least 1.5x the worst (2.75 at a trained-like ViT-S layer-8 query row, T = 65; 1.49 at T = 3).
Deliberately broken kernels, one per build: the dequantisation applying row r's scale to row r + 8 when
r + 8 = M - 1 reaches ratios of 13.1 (row) and 6.0 (RMS), 2.9x and 2.4x over KAPPA_* (test_vit_fp8_gpu.py's RMS check
sees 1.8x against its 1.1); reading the upper half's scale from row r reaches 275 / 16.5 (61x over).  A row quantiser
taking amax over the first 256 elements only reaches 4.0 / 1.7, inside KAPPA_*: the bit-exact quantiser tests and
test_vit_fp8_gpu.py's RMS check (1.5x against 1.1) catch it instead.  Dropping a partial k-block cannot show here:
every K of these models is a multiple of 128.  The file runs in about 50 s on an H100, most of it the CPU's fp64 forwards."""
import copy
import time

import pytest

from tests.test_vit_accuracy_gpu import FACETS, IMAGES, MODELS, OPTS, forward_taps, image, measure, model_of, report
from tests.test_vit_fp8_gpu import emulated

pytestmark = pytest.mark.gpu

KAPPA_ROW = 4.5
KAPPA_RMS = 2.5
HWS = list(IMAGES.values()) + [(14, 28)]


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


_REFS = {}


def refs(key, weights, hw):
    """(fp64 raw taps, [emulated raw taps]) of a case, cached: the fp64 model and its emulation run once per image"""
    ck = (key, weights, hw)
    if ck not in _REFS:
        m = model_of(key, weights)
        img = image(hw).double()
        _REFS[ck] = (forward_taps(copy.deepcopy(m).double(), img), [forward_taps(emulated(m), img)])
    return _REFS[ck]


@pytest.mark.parametrize("weights", ["random", "trained"])
@pytest.mark.parametrize("key", list(MODELS))
def test_every_tap_against_fp64(u, key, weights):
    t0 = time.perf_counter()
    name, depth = MODELS[key]
    taps = [(l, f) for l in range(depth) for f in FACETS]
    sd = model_of(key, weights).state_dict()
    _REFS.clear()
    multi = u.DinoV2MultiExtractFeatures(name, taps, device="cuda", weights=sd, precision="fp8")
    single = u.DinoV2ExtractFeatures(name, depth - 1, "value", device="cuda", weights=sd, precision="fp8")
    assert multi.precision == single.precision == "fp8"
    bad = []
    for hw in HWS:
        r64, emu = refs(key, weights, hw)
        img = image(hw).cuda()

        def every_tap(use_cls, norm):
            multi.use_cls, multi.norm_descs = use_cls, norm
            return multi(img)

        def deepest_value(use_cls, norm):
            single.use_cls, single.norm_descs = use_cls, norm
            return {(depth - 1, "value"): single(img)}

        for what, outs_of in (("taps", every_tap), ("single", deepest_value)):
            worst = measure(outs_of, r64, emu, OPTS)
            case = f"{key}|{weights}|fp8|{what}|{hw[0]}x{hw[1]}"
            report(case, worst)
            if worst["row"][0] > KAPPA_ROW or worst["rms"][0] > KAPPA_RMS:
                bad.append((case, worst))
    print(f"TIME|{key}|{weights}|{time.perf_counter() - t0:.1f} s")
    assert not bad, bad
