"""The single-e4m3 precision of the DINOv2 extractor (precision="fp8") on the GPU.

The yardstick is a restated model with the same quantisation points, run in fp64: the patch embedding on bf16-rounded
pixels and weights; every block weight matrix as e4m3_rn(w / s_w); the input rows of the qkv and fc1 / w12 GEMMs (the
LayerNorm outputs) as e4m3 rows with their power-of-two scales; the qkv output rounded to bf16 where it feeds the
attention; the attention output and the FFN hidden layer rounded to bf16, then to e4m3 rows, before the proj and fc2 /
w3 GEMMs.  (The attention's own bf16 rounding of P is not emulated.)  Each output's relative RMS error against the
unquantised fp64 model must be within 1.1x of the emulation's; the errors against fp64 of this precision, the
emulation and bf16 are printed side by side.  Beside that: list input and taps bit-identical to single calls,
including a full 128-image table, and a register model."""
import copy

import pytest
import torch

from oracle import anyloc_oracle as ao
from oracle import dinov2_restated as dr
from tests import dinov2_reg_restated as rr

pytestmark = pytest.mark.gpu
FACETS = ("query", "key", "value", "token")
CLS_NORM = ((False, True), (True, False))


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def _img(B, H, W, seed=1234):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed))


def _vit(name, sd, pair="fp8", depth=None):
    from anyloc_b200 import vit
    return vit.VitWeights(name, sd, "cuda", depth=depth, pair=pair)


def e4m3_rows(x):
    """x [..., K] (fp64) -> its e4m3 rows dequantised: q s with s = 2^ceil(log2(max|x| / 448)) per row"""
    amax = x.abs().amax(dim=-1, keepdim=True)
    s = torch.where(amax > 0, 2.0 ** torch.ceil(torch.log2(amax / 448.0)).clamp_min(-126), torch.ones_like(amax))
    return (x / s).float().to(torch.float8_e4m3fn).double() * s


def bf16(x):
    return x.float().to(torch.bfloat16).double()


def e4m3_weight(w):
    s = 2.0 ** float(torch.ceil(torch.log2(w.abs().max().double() / 448.0)))
    return (w / s).float().to(torch.float8_e4m3fn).double() * s


def emulated(model):
    """an fp64 copy of the restated model with this precision's quantisation points"""
    m = copy.deepcopy(model).double()
    with torch.no_grad():
        m.patch_embed.proj.weight.copy_(bf16(m.patch_embed.proj.weight))
    m.patch_embed.proj.register_forward_pre_hook(lambda mod, a: (bf16(a[0]),))
    for blk in m.blocks:
        ffn = blk.mlp
        lin_in, lin_out = (ffn.fc1, ffn.fc2) if hasattr(ffn, "fc1") else (ffn.w12, ffn.w3)
        for lin in (blk.attn.qkv, blk.attn.proj, lin_in, lin_out):
            with torch.no_grad():
                lin.weight.copy_(e4m3_weight(lin.weight))
        for lin in (blk.attn.qkv, lin_in):                     # LayerNorm -> e4m3
            lin.register_forward_pre_hook(lambda mod, a: (e4m3_rows(a[0]),))
        for lin in (blk.attn.proj, lin_out):                   # bf16 output of the attention / first FFN GEMM
            lin.register_forward_pre_hook(lambda mod, a: (e4m3_rows(bf16(a[0])),))
        attn = blk.attn

        def fwd(x, attn=attn):
            B, N, C = x.shape
            qkv = bf16(attn.qkv(x)).reshape(B, N, 3, attn.num_heads, C // attn.num_heads).permute(2, 0, 3, 1, 4)
            q, k, v = qkv[0] * attn.scale, qkv[1], qkv[2]
            p = (q @ k.transpose(-2, -1)).softmax(dim=-1)
            return attn.proj((p @ v).transpose(1, 2).reshape(B, N, C))
        attn.forward = fwd
    return m


def rms(f, ref):
    f, ref = f.double().cpu(), ref.double().cpu()
    return float((f - ref).norm() / ref.norm())


ACCURACY = [("dinov2_vits14", None, 11), ("dinov2_vitg14", 4, 3), ("dinov2_vitb14_reg", 3, 2)]


@pytest.mark.parametrize("name,depth,layer", ACCURACY, ids=[a[0] for a in ACCURACY])
def test_error_within_the_emulated_model(u, name, depth, layer):
    model = rr.model(name, depth) if name.endswith("_reg") else dr.perturb(dr.build(name, depth_override=depth), 1)
    sd = model.state_dict()
    m8, m16 = _vit(name, sd), _vit(name, sd, "bf16")
    model64, emu = copy.deepcopy(model).double(), emulated(model)
    rows = []
    for hw in ((224, 224), (98, 154)):
        img = _img(2, *hw)
        for facet in FACETS:
            for use_cls, norm in CLS_NORM:
                ref = ao.extract_features(model64, img.double(), layer, facet, use_cls, norm)
                e_emu = rms(ao.extract_features(emu, img.double(), layer, facet, use_cls, norm), ref)
                out = m8.extract(img.cuda(), layer, facet, use_cls, norm)
                assert out.dtype == torch.float32 and out.shape == ref.shape
                e8, e16 = rms(out, ref), rms(m16.extract(img.cuda(), layer, facet, use_cls, norm), ref)
                rows.append((hw, facet, use_cls, norm, e8, e_emu, e16))
    for hw, facet, use_cls, norm, e8, e_emu, e16 in rows:
        print(f"{name} L{layer} {hw} {facet:5s} cls={int(use_cls)} norm={int(norm)}: RMS fp8 {e8:.3e} "
              f"emulated {e_emu:.3e} bf16 {e16:.3e}")
    bad = [r for r in rows if r[4] > 1.1 * r[5]]
    assert not bad, bad


SIZES = [(56, 70), (14, 14), (98, 42), (224, 224), (42, 28)]      # 21, 2, 22, 257 and 7 tokens


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vits14_reg"])
def test_list_input_equals_single_calls(u, name):
    sd = (rr.model(name, 4) if name.endswith("_reg") else dr.perturb(dr.build(name, depth_override=4), 1)).state_dict()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for facet in FACETS:
        for use_cls, norm in CLS_NORM:
            ext = u.DinoV2ExtractFeatures(name, 3, facet, use_cls, norm, device="cuda", weights=sd, precision="fp8")
            assert ext.precision == "fp8" and ext.dino_model.pair == "fp8"
            out = ext(imgs)
            for x, got in zip(imgs, out):
                assert torch.equal(got, ext(x[None])[0]), (name, facet, use_cls, norm, tuple(x.shape))


def test_full_table_of_128_images(u):
    sd = dr.perturb(dr.build("dinov2_vits14", depth_override=2), 1).state_dict()
    m = _vit("dinov2_vits14", sd)
    g = torch.Generator().manual_seed(11)
    sizes = [(14 * int(torch.randint(1, 6, (1,), generator=g)), 14 * int(torch.randint(1, 6, (1,), generator=g)))
             for _ in range(128)]
    imgs = [torch.randn(3, H, W, generator=g).cuda() for H, W in sizes]
    packed, n = m.extract_varlen(imgs, 1, "value")
    for x, got in zip(imgs, packed.split(n)):
        assert torch.equal(got, m.extract(x[None], 1, "value")[0]), tuple(x.shape)


def test_multi_taps_equal_single_taps(u):
    sd = dr.perturb(dr.build("dinov2_vits14"), 1).state_dict()
    taps = [(l, f) for l in range(12) for f in FACETS][::-1]
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14", taps, device="cuda", weights=sd, precision="fp8")
    m = ext.dino_model
    img = _img(3, 70, 42).cuda()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for use_cls, norm in CLS_NORM:
        ext.use_cls, ext.norm_descs = use_cls, norm
        out, out_list = ext(img), ext(imgs)
        for layer, facet in taps:
            assert torch.equal(out[(layer, facet)], m.extract(img, layer, facet, use_cls, norm)), (layer, facet)
            ref, _ = m.extract_varlen(imgs, layer, facet, use_cls, norm)
            assert torch.equal(torch.cat(out_list[(layer, facet)]), ref), (layer, facet)


def test_rows_do_not_depend_on_the_batch(u):
    sd = dr.perturb(dr.build("dinov2_vitg14", depth_override=2), 1).state_dict()
    m = _vit("dinov2_vitg14", sd)
    img = _img(5, 126, 98).cuda()
    for facet in FACETS:
        full = m.extract(img, 1, facet)
        for i in (0, 3):
            assert torch.equal(full[i], m.extract(img[i:i + 1], 1, facet)[0]), (facet, i)


def test_weights_take_a_quarter_of_the_f16_pairs(u):
    sd = dr.build("dinov2_vitg14", depth_override=2).state_dict()
    m8, f16 = _vit("dinov2_vitg14", sd), _vit("dinov2_vitg14", sd, "f16")

    def block_bytes(m, dtypes):
        return sum(t.numel() * t.element_size() for t in m._keep if t.dtype in dtypes)

    assert block_bytes(m8, (torch.float8_e4m3fn,)) * 4 == block_bytes(f16, (torch.float16,)) - 2 * 2 * 1536 * 608
    blk = m8.blocks[0]
    assert not any(getattr(blk, n) for n in ("qkv_w_lo", "proj_w_lo", "in_w_lo", "out_w_lo"))
    assert m8.struct.patch_w_lo is None and m8.patch_w[0].dtype == torch.bfloat16
    w = sd["blocks.0.attn.qkv.weight"]
    assert blk.qkv_alpha == 2.0 ** float(torch.ceil(torch.log2(w.abs().max().double() / 448.0)))


def test_precision_from_the_environment_and_simt_refusal(u, monkeypatch):
    sd = dr.build("dinov2_vits14", depth_override=2).state_dict()
    monkeypatch.setenv("ANYLOC_B200_PRECISION", "fp8")
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd)
    assert ext.precision == "fp8" and ext.dino_model.pair == "fp8"
    img = _img(2, 56, 56).cuda()
    assert torch.isfinite(ext(img)).all()
    with pytest.raises(ValueError):
        u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd, gemm_engine="simt")
    from anyloc_b200 import _lib
    with pytest.raises(_lib.AnylocError, match="tensor-core"):
        ext.dino_model.extract(img, 1, "value", engine="simt")
    monkeypatch.delenv("ANYLOC_B200_PRECISION")
    assert u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=sd).precision == "f16x3"
