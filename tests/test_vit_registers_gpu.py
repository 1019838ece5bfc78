"""The DINOv2 backbones with register tokens (dinov2_vit{s,b,l,g}14_reg) on the GPU: parity with the oracle and with
the reference's own outputs (tests/golden/extract_reg.npz) at the 1e-4 of tests/test_vit_gpu.py, bit-identity of list
input and of several taps with the single calls, the output row layout, the launch count, the fp16-range contract and
the refusals."""
import ctypes as C

import pytest
import torch

from oracle import anyloc_oracle as ao
from tests import dinov2_reg_restated as rr
from tests.test_vit_registers_cpu import EXTRACT_REG, golden_image, golden_view
from tests.util import load_cases, rel_inf

pytestmark = pytest.mark.gpu
TOL = 1e-4
FACETS = ("query", "key", "value", "token")
ENGINES = [("tc3", "tf32x3"), ("tc3", "f16x3"), ("simt", "tf32x3"), ("simt", "f16x3")]


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def _model(name, depth, seed=2):
    return rr.model(name, depth, seed=seed)


def _img(B, H, W, seed=1234):
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(seed))


def _weights(name, sd, precision, depth=None):
    from anyloc_b200 import vit
    return vit.VitWeights(name, sd, "cuda", depth=depth, pair="f16" if precision == "f16x3" else "tf32")


# model, depth_override, layer, (H, W): full-depth ViT-S, a 4-block SwiGLU ViT-G, shallow B and L; non-square grids and
# the 518x518 identity grid of the positional table
PARITY = [("dinov2_vits14_reg", None, 11, (56, 70)), ("dinov2_vitg14_reg", 4, 3, (42, 70)),
          ("dinov2_vitb14_reg", 2, 1, (98, 154)), ("dinov2_vitl14_reg", 2, 1, (518, 518))]


@pytest.mark.parametrize("name,depth,layer,hw", PARITY, ids=[p[0] for p in PARITY])
def test_parity_with_oracle(u, name, depth, layer, hw):
    model = _model(name, depth)
    sd = model.state_dict()
    worst = 0.0
    for B in (1, 3):
        img = _img(B, *hw)
        refs = {(f, c, n): ao.extract_features(model, img, layer, f, c, n)
                for f in FACETS for c, n in ((False, True), (True, False))}
        for engine, precision in ENGINES:
            m = _weights(name, sd, precision)
            for (facet, use_cls, norm), ref in refs.items():
                out = m.extract(img.cuda(), layer, facet, use_cls, norm, engine)
                assert out.shape == ref.shape == (B, (1 if use_cls else 0) + 4 + (hw[0] // 14) * (hw[1] // 14),
                                                  m.dim)
                err = rel_inf(out.cpu(), ref)
                worst = max(worst, err)
                assert err < TOL, (name, B, engine, precision, facet, use_cls, norm, err)
    print(f"{name} L{layer} {hw}: worst rel err {worst:.2e}")


@pytest.mark.parametrize("engine", ENGINES)
def test_golden_replay(u, engine):
    """the reference's own DinoV2ExtractFeatures outputs on the register models"""
    engine, precision = engine
    for tag, name, depth, layer in EXTRACT_REG:
        g = load_cases("extract_reg.npz")[tag]
        sd = _model(name, depth, seed=1).state_dict()
        img = golden_image(g).cuda()
        for facet in FACETS:
            out = u.DinoV2ExtractFeatures(name, layer, facet, device="cuda", weights=sd, gemm_engine=engine,
                                          precision=precision)(img)
            err = rel_inf(golden_view(out.cpu(), g, facet), g[facet])
            assert err < TOL, (tag, facet, err)
        out = u.DinoV2ExtractFeatures(name, layer, "value", use_cls=True, norm_descs=False, device="cuda", weights=sd,
                                      gemm_engine=engine, precision=precision)(img)
        err = rel_inf(golden_view(out.cpu(), g, "value_cls_nonorm"), g["value_cls_nonorm"])
        assert err < TOL, (tag, "value_cls_nonorm", err)


SIZES = [(56, 70), (14, 14), (532, 546), (98, 42), (224, 224)]


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_list_input_equals_single_calls(u, precision):
    sd = _model("dinov2_vits14_reg", 4).state_dict()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for facet in FACETS:
        for use_cls, norm in ((False, True), (True, False)):
            ext = u.DinoV2ExtractFeatures("dinov2_vits14_reg", 3, facet, use_cls, norm, device="cuda", weights=sd,
                                          gemm_engine="tc3", precision=precision)
            out = ext(imgs)
            assert len(out) == len(imgs)
            for x, got in zip(imgs, out):
                ref = ext(x[None])[0]
                assert got.shape == ref.shape == ((1 if use_cls else 0) + 4 + (x.shape[1] // 14) * (x.shape[2] // 14),
                                                  384)
                assert torch.equal(got, ref), (precision, facet, use_cls, norm, tuple(x.shape))


@pytest.mark.parametrize("precision", ["f16x3", "tf32x3"])
def test_multi_taps_equal_single_taps(u, precision):
    sd = _model("dinov2_vits14_reg", None).state_dict()
    taps = [(l, f) for l in range(12) for f in FACETS][::-1]
    ext = u.DinoV2MultiExtractFeatures("dinov2_vits14_reg", taps, device="cuda", weights=sd, gemm_engine="tc3",
                                       precision=precision)
    m = ext.dino_model
    img = _img(3, 70, 42).cuda()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(i)).cuda() for i, (H, W) in enumerate(SIZES)]
    for use_cls, norm in ((False, True), (True, False)):
        ext.use_cls, ext.norm_descs = use_cls, norm
        out, out_list = ext(img), ext(imgs)
        for layer, facet in taps:
            ref = m.extract(img, layer, facet, use_cls, norm, "tc3")
            assert torch.equal(out[(layer, facet)], ref), (precision, layer, facet, use_cls, norm)
            for x, got in zip(imgs, out_list[(layer, facet)]):
                assert torch.equal(got, m.extract(x[None], layer, facet, use_cls, norm, "tc3")[0]), (layer, facet)


def test_row_layout(u):
    """With use_cls, row 0 is cls and rows 1-4 are the registers.  Checked at layer 0 without the oracle's token order:
    the value of a register row is v(norm1(reg)) -- the registers carry no positional embedding -- and the cls row's is
    v(norm1(cls + pos[0])); without use_cls the same rows shift up by one."""
    model = _model("dinov2_vits14_reg", 1)
    sd = model.state_dict()
    img = _img(2, 56, 70).cuda()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14_reg", 0, "value", use_cls=True, norm_descs=False, device="cuda",
                                  weights=sd, gemm_engine="tc3", precision="tf32x3")
    out = ext(img).cpu()
    blk, D = model.blocks[0], 384
    with torch.no_grad():
        heads = torch.cat([sd["cls_token"][0] + sd["pos_embed"][0, :1], sd["register_tokens"][0]])
        want = blk.attn.qkv(blk.norm1(heads))[:, 2 * D:]
    for b in range(2):
        assert rel_inf(out[b, :5], want) < TOL, (b, rel_inf(out[b, :5], want))
    ext.use_cls = False
    assert torch.equal(ext(img).cpu(), out[:, 1:])


def _count(fn):
    from anyloc_b200 import _lib
    fn()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    return _lib.launch_count() - n0


def test_same_launches_as_plain(u):
    from anyloc_b200 import vit
    plain = vit.random_state_dict("dinov2_vits14", seed=1, device="cuda", depth=6)
    reg = vit.random_state_dict("dinov2_vits14_reg", seed=1, device="cuda", depth=6)
    img = _img(2, 56, 70).cuda()
    imgs = [img[0], img[1, :, :42, :28]]
    taps = [(1, "key"), (3, "token"), (5, "value"), (5, "query")]
    for precision in ("f16x3", "tf32x3"):
        mp, mr = _weights("dinov2_vits14", plain, precision), _weights("dinov2_vits14_reg", reg, precision)
        for layer, facet in ((5, "value"), (5, "token"), (2, "key")):
            assert _count(lambda: mr.extract(img, layer, facet)) == _count(lambda: mp.extract(img, layer, facet))
            assert _count(lambda: mr.extract_varlen(imgs, layer, facet)) == \
                _count(lambda: mp.extract_varlen(imgs, layer, facet))
        assert _count(lambda: mr.extract_taps(img, taps)) == _count(lambda: mp.extract_taps(img, taps))
        assert _count(lambda: mr.extract_taps_varlen(imgs, taps)) == _count(lambda: mp.extract_taps_varlen(imgs, taps))


def _loud_registers(depth, scale, ln_gain=None, seed=5):
    """registers x scale; with ln_gain also the traits of trained checkpoints that test_vit_gpu._outlier_weights gives
    the plain models: LayerScale spread log-uniformly over 1e-5 .. 1 and a few massive LayerNorm channels"""
    model = _model("dinov2_vits14_reg", depth, seed=seed)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        model.register_tokens.mul_(scale)
        for blk in model.blocks if ln_gain is not None else []:
            D = blk.ls1.gamma.shape[0]
            blk.ls1.gamma.copy_(10 ** (-5 * torch.rand(D, generator=g)))
            blk.ls2.gamma.copy_(10 ** (-5 * torch.rand(D, generator=g)))
            hot = torch.randperm(D, generator=g)[:3]
            blk.norm1.weight[hot] *= ln_gain
            blk.norm2.weight[hot] *= ln_gain
            blk.norm2.bias[hot] += 0.5 * ln_gain
    return model


def test_register_outliers_precision_contract(u):
    """Trained register models keep their high-norm tokens in the registers.  Registers x3000 alone stay out of the fp16
    operands (every GEMM input passes a LayerNorm first), so f16x3 stays inside the tolerance; with the massive
    LayerNorm channels of test_outlier_activations_precision_contract as well, f16x3 raises and precision='auto' redoes
    the call in tf32x3 and stays there, inside 3x the oracle's own fp32 error against fp64."""
    from anyloc_b200 import _lib
    layer = 3
    img = _img(2, 224, 224)
    loud = _loud_registers(4, 3000.0)
    ref = ao.extract_features(loud, img, layer, "value")
    for precision in ("f16x3", "tf32x3"):
        ext = u.DinoV2ExtractFeatures("dinov2_vits14_reg", layer, "value", device="cuda", weights=loud.state_dict(),
                                      precision=precision)
        err = rel_inf(ext(img.cuda()).cpu(), ref)
        assert ext.precision == precision and err < TOL, (precision, err)
    wild = _loud_registers(4, 3000.0, ln_gain=3000.0)
    ref = ao.extract_features(wild, img, layer, "value")
    ref64 = ao.extract_features(wild.double(), img.double(), layer, "value")
    wild = wild.float()
    tol = max(TOL, 3.0 * rel_inf(ref, ref64))
    ext = u.DinoV2ExtractFeatures("dinov2_vits14_reg", layer, "value", device="cuda", weights=wild.state_dict(),
                                  precision="f16x3")
    with pytest.raises(_lib.AnylocError, match="overflowed the fp16 operand range"):
        ext(img.cuda())
    ext = u.DinoV2ExtractFeatures("dinov2_vits14_reg", layer, "value", device="cuda", weights=wild.state_dict())
    assert ext.precision == "f16x3"
    out = ext(img.cuda())
    assert ext.precision == "tf32x3" and rel_inf(out.cpu(), ref64) < tol
    assert rel_inf(ext(img.cuda()).cpu(), ref64) < tol
    print(f"register outliers: oracle fp32 vs fp64 {rel_inf(ref, ref64):.2e}, auto vs fp64 {rel_inf(out.cpu(), ref64):.2e}")


def test_state_dict_refusals(u):
    sd = _model("dinov2_vits14_reg", 2).state_dict()
    with pytest.raises(ValueError, match="register_tokens"):
        u.DinoV2ExtractFeatures("dinov2_vits14_reg", 1, "value", device="cuda",
                                weights={k: v for k, v in sd.items() if k != "register_tokens"})
    with pytest.raises(ValueError, match="register_tokens"):
        u.DinoV2MultiExtractFeatures("dinov2_vits14_reg", [(1, "value")], device="cuda",
                                     weights={**sd, "register_tokens": sd["register_tokens"][:, :3]})


def test_abi_refusals_write_nothing(u):
    from anyloc_b200 import _lib
    lib = _lib.load()
    m = _weights("dinov2_vits14_reg", _model("dinov2_vits14_reg", 2).state_dict(), "tf32x3")
    B, H, W, canary = 2, 56, 42, 7
    img = _img(B, H, W).cuda()
    rows = B * (4 + (H // 14) * (W // 14))
    out = torch.full((rows + canary, m.dim), float("nan"), device="cuda")
    pos = m.pos_for(H // 14, W // 14)
    nbytes = lib.anyloc_vit_workspace_bytes(C.byref(m.cfg), B, H, W)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    img_p = (C.c_void_p * B)(img[0].data_ptr(), img[1].data_ptr())
    pos_p = (C.c_void_p * B)(pos.data_ptr(), pos.data_ptr())
    hw = (C.c_int32 * (2 * B))(H, W, H, W)
    tap = (_lib.VitTap * 1)(_lib.VitTap(1, _lib.FACET["value"], out.data_ptr()))

    def calls(cfg, w):
        tc3, st = _lib.ENGINE["tc3"], _lib.stream_ptr()
        return [lib.anyloc_vit_extract(C.byref(cfg), C.byref(w), _lib.ptr(img), B, H, W, _lib.ptr(pos), 1, 2, 0, 1,
                                       _lib.ptr(out), _lib.ptr(ws), nbytes, tc3, st),
                lib.anyloc_vit_extract_varlen(C.byref(cfg), C.byref(w), B, img_p, hw, pos_p, 1, 2, 0, 1, _lib.ptr(out),
                                              _lib.ptr(ws), nbytes, tc3, st),
                lib.anyloc_vit_extract_taps(C.byref(cfg), C.byref(w), _lib.ptr(img), B, H, W, _lib.ptr(pos), tap, 1, 0,
                                            1, _lib.ptr(ws), nbytes, tc3, st),
                lib.anyloc_vit_extract_taps_varlen(C.byref(cfg), C.byref(w), B, img_p, hw, pos_p, tap, 1, 0, 1,
                                                   _lib.ptr(ws), nbytes, tc3, st)]

    neg = _lib.VitCfg.from_buffer_copy(m.cfg)
    neg.num_registers = -1
    null = _lib.VitWeightsStruct.from_buffer_copy(m.struct)
    null.register_tokens = None
    assert calls(neg, m.struct) == [_lib.ERR["arg"]] * 4
    assert calls(m.cfg, null) == [_lib.ERR["arg"]] * 4
    torch.cuda.synchronize()
    assert bool(torch.isnan(out).all())
    assert calls(m.cfg, m.struct)[0] == 0, _lib.last_error()
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[rows:]).all())
    assert torch.equal(out[:rows].view(B, rows // B, -1), m.extract(img, 1, "value", engine="tc3"))


def test_vlad_accepts_register_output(u):
    """VLAD aggregates every row it is given, registers included, as the reference does with [B, 4 + N, D]"""
    sd = _model("dinov2_vits14_reg", 3).state_dict()
    ext = u.DinoV2ExtractFeatures("dinov2_vits14_reg", 2, "value", device="cuda", weights=sd)
    feats = ext(_img(3, 56, 70).cuda())
    assert feats.shape == (3, 4 + 20, 384)
    c = torch.nn.functional.normalize(torch.randn(8, 384, generator=torch.Generator().manual_seed(0)), dim=1).cuda()
    v = u.VLAD(8)
    v.kmeans = u._KMeans(8, mode="cosine")
    v.kmeans.centroids, v.c_centers, v.desc_dim = c, c, 384
    batch = v.generate_multi(feats)
    assert batch.shape == (3, 8 * 384)
    for f, got in zip(feats, batch):
        ref = ao.vlad_generate(f.cpu(), c.cpu(), labels=v.kmeans.predict(f).cpu())
        assert rel_inf(got.cpu(), ref) < 1e-5
    items = ext([x for x in _img(2, 42, 98).cuda()] + [_img(1, 56, 56).cuda()[0]])
    lst = v.generate_multi(items)
    assert len(lst) == 3
    for f, got in zip(items, lst):
        assert torch.allclose(got, v.generate(f), atol=1e-6, rtol=0)
