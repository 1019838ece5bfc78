"""The DINOv2 backbones with register tokens (dinov2_vit{s,b,l,g}14_reg) without a GPU: the restated models against the
independent HuggingFace port (transformers.models.dinov2_with_registers) and against the reference's own outputs
(tests/golden/extract_reg.npz), three wrong restatements that the goldens must reject, and the host side of the
extractor: the positional tables, the packed-list layout, the workspace sizes and the C ABI's argument checks."""
import ctypes as C
import math

import pytest
import torch

from anyloc_b200 import _lib, vit
from oracle import anyloc_oracle as ao
from oracle import dinov2_restated as dr
from tests import dinov2_reg_restated as rr
from tests.util import load_cases, rel_inf

GOLDEN_TOL = 1e-5     # as tests/test_oracle_cpu.py
FACETS = ("value", "key", "query", "token")
REG = ["dinov2_vits14_reg", "dinov2_vitb14_reg", "dinov2_vitl14_reg", "dinov2_vitg14_reg"]
# the cases of tests/golden/extract_reg.npz (tests/golden/make_golden_reg.py): (tag, model, depth_override, layer); the
# image shape B, H, W is stored with each case
EXTRACT_REG = [
    ("vits14_reg_l9_56x70", "dinov2_vits14_reg", None, 9),
    ("vits14_reg_d2_l1_532x546", "dinov2_vits14_reg", 2, 1),
    ("vitg14_reg_d2_l1_42x42", "dinov2_vitg14_reg", 2, 1),
]


def golden_image(case):
    """the input of an extract_reg.npz case, regenerated from its seed as make_golden_reg.py does"""
    B, H, W = (int(v) for v in case["shape"])
    return torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(1234))


def golden_view(out, case, key):
    """the rows and channels of an output [B, n, D] that extract_reg.npz stores for `key`"""
    return out[:, torch.from_numpy(case[key + "_rows"])][:, :, torch.from_numpy(case["cols"])]


def _model(name, depth, seed=1):
    return rr.model(name, depth, seed=seed) if name in rr.ARCHS else \
        dr.perturb(dr.build(name, seed=0, depth_override=depth), seed=seed)


# ------------------------------------------------------------------ the restated models
def _hf_reg_model_from(model, name, depth):
    """HuggingFace's Dinov2WithRegistersModel holding the restated model's weights, with the RAW 37x37 positional table:
    the port resizes it itself, like upstream (size=(gh, gw), bicubic, antialias)"""
    from transformers import Dinov2WithRegistersConfig, Dinov2WithRegistersModel
    dim, _, heads, ffn = rr.ARCHS[name]
    cfg = Dinov2WithRegistersConfig(hidden_size=dim, num_hidden_layers=depth, num_attention_heads=heads, mlp_ratio=4,
                                    image_size=518, patch_size=14, num_register_tokens=4,
                                    use_swiglu_ffn=(ffn != "mlp"), layer_norm_eps=1e-6, hidden_act="gelu",
                                    qkv_bias=True, layerscale_value=1.0, attn_implementation="eager")
    hf = Dinov2WithRegistersModel(cfg).eval()
    sd = model.state_dict()
    with torch.no_grad():
        e = hf.embeddings
        e.cls_token.copy_(sd["cls_token"])
        e.register_tokens.copy_(sd["register_tokens"])
        e.position_embeddings.copy_(sd["pos_embed"])
        e.patch_embeddings.projection.weight.copy_(sd["patch_embed.proj.weight"])
        e.patch_embeddings.projection.bias.copy_(sd["patch_embed.proj.bias"])
        for i, layer in enumerate(hf.encoder.layer):
            p = f"blocks.{i}."
            layer.norm1.weight.copy_(sd[p + "norm1.weight"]); layer.norm1.bias.copy_(sd[p + "norm1.bias"])
            layer.norm2.weight.copy_(sd[p + "norm2.weight"]); layer.norm2.bias.copy_(sd[p + "norm2.bias"])
            w, b = sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]
            att = layer.attention.attention
            for j, lin in enumerate((att.query, att.key, att.value)):
                lin.weight.copy_(w[j * dim:(j + 1) * dim]); lin.bias.copy_(b[j * dim:(j + 1) * dim])
            layer.attention.output.dense.weight.copy_(sd[p + "attn.proj.weight"])
            layer.attention.output.dense.bias.copy_(sd[p + "attn.proj.bias"])
            layer.layer_scale1.lambda1.copy_(sd[p + "ls1.gamma"])
            layer.layer_scale2.lambda1.copy_(sd[p + "ls2.gamma"])
            if ffn == "mlp":
                layer.mlp.fc1.weight.copy_(sd[p + "mlp.fc1.weight"]); layer.mlp.fc1.bias.copy_(sd[p + "mlp.fc1.bias"])
                layer.mlp.fc2.weight.copy_(sd[p + "mlp.fc2.weight"]); layer.mlp.fc2.bias.copy_(sd[p + "mlp.fc2.bias"])
            else:
                layer.mlp.weights_in.weight.copy_(sd[p + "mlp.w12.weight"]); layer.mlp.weights_in.bias.copy_(sd[p + "mlp.w12.bias"])
                layer.mlp.weights_out.weight.copy_(sd[p + "mlp.w3.weight"]); layer.mlp.weights_out.bias.copy_(sd[p + "mlp.w3.bias"])
    return hf


@pytest.mark.parametrize("name,depth", [("dinov2_vits14_reg", 3), ("dinov2_vitg14_reg", 2)])
def test_restated_register_vit_matches_hf_port(name, depth):
    """Token order [cls, r0..r3, patches], no positional embedding on the registers, and the offset-0 antialiased resize,
    pinned by the independent port: the embeddings and every block's output at the identity grid (518x518), a smaller
    and a larger one."""
    model = _model(name, depth)
    hf = _hf_reg_model_from(model, name, depth)
    for H, W in ((518, 518), (56, 70), (546, 532)):
        img = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(3))
        with torch.no_grad():
            hs = hf(pixel_values=img, output_hidden_states=True).hidden_states     # [emb, blk0, blk1, ...]
            x = model.prepare_tokens(img)
            assert x.shape[1] == 1 + 4 + (H // 14) * (W // 14)
            assert torch.allclose(x, hs[0], atol=2e-5, rtol=1e-5), (H, W, (x - hs[0]).abs().max().item())
            for i, blk in enumerate(model.blocks):
                x = blk(x)
                assert torch.allclose(x, hs[i + 1], atol=2e-5, rtol=1e-5), (H, W, i, (x - hs[i + 1]).abs().max().item())


@pytest.mark.parametrize("case", EXTRACT_REG, ids=[c[0] for c in EXTRACT_REG])
def test_extract_reg_oracle_matches_golden(case):
    """The reference's own DinoV2ExtractFeatures on the register models returns the 4 register rows after cls (it drops
    row 0 only); the oracle matches it, and its early exit equals the full forward + hook bit for bit."""
    tag, name, depth, layer = case
    g = load_cases("extract_reg.npz")[tag]
    model = _model(name, depth)
    img = golden_image(g)
    n = 4 + (img.shape[2] // 14) * (img.shape[3] // 14)
    for facet, kw, key in [(f, {}, f) for f in FACETS] + [("value", dict(use_cls=True, norm_descs=False),
                                                           "value_cls_nonorm")]:
        out = ao.extract_features(model, img, layer, facet, **kw)
        assert out.shape[1] == n + (1 if kw else 0)
        assert torch.equal(out, ao.extract_features_full_forward(model, img, layer, facet, **kw)), key
        out = golden_view(out, g, key)
        assert rel_inf(out, g[key]) < GOLDEN_TOL, (key, rel_inf(out, g[key]))


def test_extract_reg_oracle_matches_live_reference():
    from oracle import reference_import as ri
    if not ri.available():
        pytest.skip("reference tree not present")
    ref = ri.load_reference_utilities()
    tag, name, depth, layer = EXTRACT_REG[0]
    model = _model(name, depth)
    img = golden_image(load_cases("extract_reg.npz")[tag])
    for facet in FACETS:
        with ri.hub_patched(lambda n: model):
            ext = ref.DinoV2ExtractFeatures(name, layer, facet, device="cpu")
        assert torch.equal(ext(img), ao.extract_features(model, img, layer, facet)), facet


# ------------------------------------------------------------------ negative controls
def _registers_after_patches(model):
    def prepare_tokens(x):
        B, _, w, h = x.shape
        x = model.patch_embed(x)
        x = torch.cat((model.cls_token.expand(B, -1, -1), x), dim=1)
        x = x + model.interpolate_pos_encoding(x, w, h)
        return torch.cat((x, model.register_tokens.expand(B, -1, -1)), dim=1)
    model.prepare_tokens = prepare_tokens


def _registers_with_pos_embed(model):
    """the registers take the cls token's positional embedding, as if they were inserted before the table is added"""
    def prepare_tokens(x):
        B, _, w, h = x.shape
        x = model.patch_embed(x)
        x = torch.cat((model.cls_token.expand(B, -1, -1), x), dim=1)
        pos = model.interpolate_pos_encoding(x, w, h)
        x = x + pos
        return torch.cat((x[:, :1], model.register_tokens.expand(B, -1, -1) + pos[:, :1], x[:, 1:]), dim=1)
    model.prepare_tokens = prepare_tokens


def _plain_interpolation(model):
    model.interpolate_offset, model.interpolate_antialias = 0.1, False


@pytest.mark.parametrize("wrong", [_registers_after_patches, _registers_with_pos_embed, _plain_interpolation])
def test_wrong_register_oracles_miss_the_goldens(wrong):
    """Each plausible mistake misses the reference's outputs by far more than the 1e-4 parity tolerance; the printed
    factor is the smallest miss over the cases and facets, in units of 1e-4 (measured: 12470x registers after the
    patches, 128x positional embedding on the registers, 45x the plain models' resize)."""
    worst = math.inf
    for tag, name, depth, layer in EXTRACT_REG:
        g = load_cases("extract_reg.npz")[tag]
        model = _model(name, depth)
        wrong(model)
        img = golden_image(g)
        for facet in FACETS:
            out = ao.extract_features(model, img, layer, facet)
            worst = min(worst, rel_inf(golden_view(out, g, facet), g[facet]))
    print(f"{wrong.__name__}: misses the goldens by >= {worst / 1e-4:.0f}x the 1e-4 tolerance")
    assert worst > 20 * 1e-4, worst


# ------------------------------------------------------------------ host side
@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vits14_reg"])
def test_pos_table_equals_the_oracle(name):
    model = _model(name, 1)
    off, aa = vit.TOKENS[name][1:]
    assert (off, aa) == (model.interpolate_offset, getattr(model, "interpolate_antialias", False))
    for gh, gw in ((37, 37), (4, 5), (38, 39), (3, 3), (46, 38), (37, 40)):
        x = torch.zeros(1, 1 + gh * gw, model.embed_dim)
        want = model.interpolate_pos_encoding(x, gh * 14, gw * 14)[0]
        got = vit.interpolate_pos_embed(model.pos_embed, gh, gw, off, aa)
        assert torch.equal(got, want), (name, gh, gw)
    # the two recipes differ wherever the table is resized
    a = vit.interpolate_pos_embed(model.pos_embed, 38, 39)
    b = vit.interpolate_pos_embed(model.pos_embed, 38, 39, 0.0, True)
    assert not torch.equal(a, b)


def test_varlen_layout_counts_the_registers():
    sizes = [(56, 70), (14, 14), (532, 546)]
    for use_cls in (False, True):
        lay = vit.VarlenLayout(sizes, use_cls, 2, registers=4)
        assert lay.tokens == [25, 6, 1487]
        assert lay.n_out == [t - (0 if use_cls else 1) for t in lay.tokens]
        assert lay.row0 == [0, lay.n_out[0], lay.n_out[0] + lay.n_out[1], sum(lay.n_out)] and lay.rows == sum(lay.n_out)
        assert lay.chunks == [(0, 2), (2, 3)]
        assert vit.VarlenLayout(sizes, use_cls, 2).tokens == [21, 2, 1483]


def _cfg(dim=384, heads=6, depth=4, registers=0, kind="mlp"):
    return _lib.VitCfg(dim, depth, heads, _lib.FFN[kind], vit.ffn_hidden(dim, kind), vit.PATCH, _lib.PAIR["f16"],
                       registers)


def _carve_bytes(n_patch, M, D, hidden, kp, qkv32=False):
    """the workspace the ViT carves: the patch pairs and GEMM output, then M token rows of every activation"""
    counts = [n_patch * kp] * 2 + [n_patch * D] + [M * D] * 3 + [M * 3 * D] * 2 + [M * hidden] * 2
    counts += [M * 3 * D] if qkv32 else []
    return sum((4 * c + 255) // 256 * 256 for c in counts) + 4096


def _hw(sizes):
    return (C.c_int32 * (2 * len(sizes)))(*[v for s in sizes for v in s])


def test_workspace_counts_the_registers(lib):
    kp = lib.anyloc_vit_patch_k(14)
    for dim, heads, kind in ((384, 6, "mlp"), (1536, 24, "swiglufused")):
        hid = vit.ffn_hidden(dim, kind)
        for R in (0, 4):
            cfg = C.byref(_cfg(dim, heads, registers=R, kind=kind))
            for B, H, W in ((1, 224, 224), (3, 98, 126), (32, 322, 322)):
                N = (H // 14) * (W // 14)
                assert lib.anyloc_vit_workspace_bytes(cfg, B, H, W) == _carve_bytes(B * N, B * (1 + R + N), dim, hid, kp)
                taps = (_lib.VitTap * 2)(_lib.VitTap(1, 0, 4096), _lib.VitTap(3, 2, 4096))
                assert lib.anyloc_vit_taps_workspace_bytes(cfg, B, H, W, taps, 2) == \
                    _carve_bytes(B * N, B * (1 + R + N), dim, hid, kp, qkv32=True)
            sizes = [(98, 126), (224, 224), (14, 14)]
            n = [(h // 14) * (w // 14) for h, w in sizes]
            assert lib.anyloc_vit_varlen_workspace_bytes(cfg, 3, _hw(sizes)) == \
                _carve_bytes(sum(n), sum(1 + R + k for k in n), dim, hid, kp)
    bad = C.byref(_cfg(registers=-1))
    assert lib.anyloc_vit_workspace_bytes(bad, 1, 224, 224) == 0
    assert lib.anyloc_vit_varlen_workspace_bytes(bad, 1, _hw([(224, 224)])) == 0
    taps = (_lib.VitTap * 1)(_lib.VitTap(1, 0, 4096))
    assert lib.anyloc_vit_taps_workspace_bytes(bad, 1, 224, 224, taps, 1) == 0
    assert lib.anyloc_vit_taps_varlen_workspace_bytes(bad, 1, _hw([(224, 224)]), taps, 1) == 0


def _calls(lib, registers, reg_ptr):
    """the four extraction entry points with placeholder device pointers: a refused call returns before any is used"""
    cfg, fake = _cfg(registers=registers), C.c_void_p(4096)
    w = _lib.VitWeightsStruct()
    w.register_tokens = reg_ptr
    cfg_p, w_p = C.byref(cfg), C.byref(w)
    taps = (_lib.VitTap * 1)(_lib.VitTap(3, 2, 4096))
    ptrs = (C.c_void_p * 2)(4096, 4096)
    hw = _hw([(224, 224), (98, 126)])
    tc3, ws = _lib.ENGINE["tc3"], 1 << 40
    return {
        "extract": lambda: lib.anyloc_vit_extract(cfg_p, w_p, fake, 2, 224, 224, fake, 3, 2, 0, 1, fake, fake, ws, tc3,
                                                  None),
        "extract_varlen": lambda: lib.anyloc_vit_extract_varlen(cfg_p, w_p, 2, ptrs, hw, ptrs, 3, 2, 0, 1, fake, fake, ws,
                                                                tc3, None),
        "extract_taps": lambda: lib.anyloc_vit_extract_taps(cfg_p, w_p, fake, 2, 224, 224, fake, taps, 1, 0, 1, fake, ws,
                                                            tc3, None),
        "extract_taps_varlen": lambda: lib.anyloc_vit_extract_taps_varlen(cfg_p, w_p, 2, ptrs, hw, ptrs, taps, 1, 0, 1,
                                                                          fake, ws, tc3, None),
    }


def test_abi_refuses_bad_registers(lib):
    for fn, call in _calls(lib, -1, 4096).items():
        assert call() == _lib.ERR["arg"] and "num_registers=-1" in _lib.last_error(), fn
    for fn, call in _calls(lib, 4, None).items():
        assert call() == _lib.ERR["arg"] and "register_tokens is null" in _lib.last_error(), fn


def test_abi_version_and_layout(lib):
    assert lib.anyloc_version() == 101
    # appended fields: a 7-field configuration and a zero-initialised weight table keep today's models
    assert _lib.VitCfg(384, 4, 6, 0, 1536, 14, 0).num_registers == 0
    assert _lib.VitWeightsStruct().register_tokens is None
    assert [f for f, _ in _lib.VitCfg._fields_][-1] == "num_registers"
    assert [f for f, _ in _lib.VitWeightsStruct._fields_][-1] == "register_tokens"


@pytest.mark.parametrize("name", REG)
def test_random_state_dict_has_register_tokens(name):
    plain = vit.random_state_dict(name[:-4], seed=3, depth=1)
    sd = vit.random_state_dict(name, seed=3, depth=1)
    dim = vit.ARCHS[name][0]
    assert set(sd) == set(plain) | {"register_tokens"}
    assert sd["register_tokens"].shape == (1, 4, dim) and float(sd["register_tokens"].abs().max()) < 1e-4
    assert all(torch.equal(sd[k], plain[k]) for k in plain)     # drawn last: the rest is the plain model's
    assert vit.TOKENS[name] == (4, 0.0, True) and vit.TOKENS[name[:-4]] == (0, 0.1, False)
    assert vit.ARCHS[name] == vit.ARCHS[name[:-4]] == rr.ARCHS[name] == dr.ARCHS[name[:-4]]


def test_state_dict_without_registers_is_refused():
    """the check runs before the weights go anywhere, so it needs no device"""
    sd = vit.random_state_dict("dinov2_vits14_reg", depth=1)
    with pytest.raises(ValueError, match="'register_tokens' missing"):
        vit.VitWeights("dinov2_vits14_reg", {k: v for k, v in sd.items() if k != "register_tokens"}, "cuda")
    with pytest.raises(ValueError, match=r"'register_tokens' has shape \(1, 5, 384\)"):
        vit.VitWeights("dinov2_vits14_reg", {**sd, "register_tokens": torch.zeros(1, 5, 384)}, "cuda")
