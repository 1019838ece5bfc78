"""TEST INFRASTRUCTURE -- CPU restatement of the facebookresearch/dinov2 backbones with register tokens,
dinov2_vit{s,b,l,g}14_reg (hub/backbones.py), on top of the plain restatement in oracle/dinov2_restated.py.

The register models are the plain architectures with three differences:
  num_register_tokens=4    prepare_tokens adds the positional table to [cls, patches], then inserts
                           register_tokens.expand(B, -1, -1) between cls and the patches -> [cls, r0..r3, patches];
                           the registers get no positional embedding
  interpolate_offset=0     the 37x37 table is resized to size=(gh, gw) instead of scale_factor=((g + 0.1) / 37)
  interpolate_antialias    ... with antialias=True
and the state dict holds `register_tokens` [1, 4, D] (init N(0, 1e-6)).  Cross-checked in
tests/test_vit_registers_cpu.py against the independent HuggingFace port (transformers.models.dinov2_with_registers),
and the reference's own DinoV2ExtractFeatures over this model makes tests/golden/extract_reg.npz
(tests/golden/make_golden_reg.py).
"""
import math

import torch
from torch import nn
from torch.nn import functional as F

from oracle import dinov2_restated as dr

NUM_REGISTERS = 4
ARCHS = {n + "_reg": a for n, a in dr.ARCHS.items()}


class DinoVisionTransformerReg(dr.DinoVisionTransformer):
    def __init__(self, name="dinov2_vits14_reg", depth_override=None):
        if name not in ARCHS:
            raise KeyError(f"{name!r} is not a register model; expected one of {sorted(ARCHS)}")
        super().__init__(name[:-len("_reg")], depth_override=depth_override)
        self.num_register_tokens = NUM_REGISTERS
        self.interpolate_offset, self.interpolate_antialias = 0.0, True
        self.register_tokens = nn.Parameter(torch.zeros(1, NUM_REGISTERS, self.embed_dim))
        nn.init.normal_(self.register_tokens, std=1e-6)

    def interpolate_pos_encoding(self, x, w, h):
        npatch = x.shape[1] - 1
        N = self.pos_embed.shape[1] - 1
        if npatch == N and w == h:
            return self.pos_embed
        pos_embed = self.pos_embed.float()
        class_pos_embed = pos_embed[:, 0]
        patch_pos_embed = pos_embed[:, 1:]
        dim = x.shape[-1]
        w0 = w // self.patch_size
        h0 = h // self.patch_size
        M = int(math.sqrt(N))
        if self.interpolate_offset:      # upstream keeps both recipes; the register models take the second
            kwargs = {"scale_factor": (float(w0 + self.interpolate_offset) / M, float(h0 + self.interpolate_offset) / M)}
        else:
            kwargs = {"size": (w0, h0)}
        patch_pos_embed = F.interpolate(
            patch_pos_embed.reshape(1, M, M, dim).permute(0, 3, 1, 2),
            mode="bicubic", antialias=self.interpolate_antialias, **kwargs)
        assert (w0, h0) == tuple(patch_pos_embed.shape[-2:])
        patch_pos_embed = patch_pos_embed.permute(0, 2, 3, 1).view(1, -1, dim)
        return torch.cat((class_pos_embed.unsqueeze(0), patch_pos_embed), dim=1).to(x.dtype)

    def prepare_tokens(self, x):
        B, nc, w, h = x.shape
        x = self.patch_embed(x)
        x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
        x = x + self.interpolate_pos_encoding(x, w, h)
        return torch.cat((x[:, :1], self.register_tokens.expand(B, -1, -1), x[:, 1:]), dim=1)


def build(name, seed=0, dtype=torch.float32, depth_override=None):
    """Random-init register model, deterministic in `seed` (CPU generator), eval mode (as oracle.dinov2_restated.build)"""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    m = DinoVisionTransformerReg(name, depth_override=depth_override).eval().to(dtype)
    torch.random.set_rng_state(g)
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def perturb(model, seed=1, scale=0.05):
    """oracle.dinov2_restated.perturb, then O(1) register tokens: at their init of 1e-6 a misplaced register would not
    show in any output"""
    dr.perturb(model, seed=seed, scale=scale)
    gen = torch.Generator().manual_seed(seed + 7919)
    with torch.no_grad():
        model.register_tokens.copy_(torch.randn(model.register_tokens.shape, generator=gen))
    return model


def model(name, depth_override=None, seed=1):
    """the perturbed model the golden vectors and the tests use"""
    return perturb(build(name, seed=0, depth_override=depth_override), seed=seed)
