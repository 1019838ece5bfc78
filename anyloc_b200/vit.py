"""Host side of the DINOv2 extractor: weight preparation (tf32 hi/lo split, SwiGLU row
interleave, patch-embed flattening), positional-embedding interpolation (upstream
`interpolate_pos_encoding`, done once per resolution) and the call into
`anyloc_vit_extract` (include/anyloc_b200.h).

Reference: /root/reference/utilities.py:219-288 (DinoV2ExtractFeatures) and the hub model it
loads (facebookresearch/dinov2; spec in SURVEY.md Appendix A).
"""
import ctypes as C
import math
import operator
import os

import torch
from torch.nn import functional as F

from . import _lib

ARCHS = {
    # name: (embed_dim, depth, heads, ffn kind)
    "dinov2_vits14": (384, 12, 6, "mlp"),
    "dinov2_vitb14": (768, 12, 12, "mlp"),
    "dinov2_vitl14": (1024, 24, 16, "mlp"),
    "dinov2_vitg14": (1536, 40, 24, "swiglufused"),
}
# the register variants (upstream hub/backbones.py *_reg): same architectures with 4 register tokens between cls and
# the patches, and their own positional-embedding resize
ARCHS.update({n + "_reg": a for n, a in list(ARCHS.items())})
PATCH = 14
POS_GRID = 37           # pretrained at 518x518
INTERP_OFFSET = 0.1     # upstream interpolate_offset of the plain models
# name: (num_register_tokens, interpolate_offset, interpolate_antialias)
TOKENS = {n: (4, 0.0, True) if n.endswith("_reg") else (0, INTERP_OFFSET, False) for n in ARCHS}


def ffn_hidden(dim, kind):
    return 4 * dim if kind == "mlp" else (int(4 * dim * 2 / 3) + 7) // 8 * 8


def random_state_dict(name, seed=0, device="cpu", depth=None):
    """Random weights with the upstream init recipe (trunc_normal std .02 for Linear / pos_embed,
    cls ~ N(0,1e-6), zero bias, LayerNorm (1,0), LayerScale 1.0), generated directly on `device`.
    Register models get `register_tokens` ~ N(0,1e-6), drawn last, so every other tensor equals the plain model's of the
    same seed.  Synthetic-benchmark use only: no pretrained checkpoint can be fetched offline."""
    dim, full_depth, heads, kind = ARCHS[name]
    depth = full_depth if depth is None else depth
    hid = ffn_hidden(dim, kind)
    g = torch.Generator(device=device).manual_seed(seed)

    def tn(*shape):
        t = torch.empty(*shape, device=device, dtype=torch.float32)
        # trunc_normal_(std=.02, a=-2, b=2): the +-2 bounds are 100 sigma away -> plain normal
        return t.normal_(0.0, 0.02, generator=g)

    def zeros(*s):
        return torch.zeros(*s, device=device)

    def ones(*s):
        return torch.ones(*s, device=device)

    sd = {
        "cls_token": torch.empty(1, 1, dim, device=device).normal_(0.0, 1e-6, generator=g),
        "pos_embed": tn(1, 1 + POS_GRID * POS_GRID, dim),
        "patch_embed.proj.weight": tn(dim, 3, PATCH, PATCH),
        "patch_embed.proj.bias": zeros(dim),
    }
    for i in range(depth):
        p = f"blocks.{i}."
        sd[p + "norm1.weight"], sd[p + "norm1.bias"] = ones(dim), zeros(dim)
        sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"] = tn(3 * dim, dim), zeros(3 * dim)
        sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"] = tn(dim, dim), zeros(dim)
        sd[p + "ls1.gamma"] = ones(dim)
        sd[p + "norm2.weight"], sd[p + "norm2.bias"] = ones(dim), zeros(dim)
        if kind == "mlp":
            sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = tn(hid, dim), zeros(hid)
            sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = tn(dim, hid), zeros(dim)
        else:
            sd[p + "mlp.w12.weight"], sd[p + "mlp.w12.bias"] = tn(2 * hid, dim), zeros(2 * hid)
            sd[p + "mlp.w3.weight"], sd[p + "mlp.w3.bias"] = tn(dim, hid), zeros(dim)
        sd[p + "ls2.gamma"] = ones(dim)
    n_reg = TOKENS[name][0]
    if n_reg:
        sd["register_tokens"] = torch.empty(1, n_reg, dim, device=device).normal_(0.0, 1e-6, generator=g)
    return sd


def interpolate_pos_embed(pos_embed, gh, gw, offset=INTERP_OFFSET, antialias=False):
    """Upstream DinoVisionTransformer.interpolate_pos_encoding for a gh x gw patch grid
    (gh = H//14 rows, gw = W//14 columns).  pos_embed [1, 1+37*37, D] -> [1+gh*gw, D].
    offset / antialias: the model's interpolate_offset / interpolate_antialias (TOKENS); offset 0 resizes to
    size=(gh, gw) instead of scale_factor=((g + offset) / 37)."""
    pos_embed = pos_embed.detach().float().cpu()
    n = pos_embed.shape[1] - 1
    m = int(math.sqrt(n))
    if gh * gw == n and gh == gw:
        return pos_embed[0].contiguous()
    dim = pos_embed.shape[-1]
    cls_pos, patch_pos = pos_embed[:, 0], pos_embed[:, 1:]
    kw = {"scale_factor": (float(gh + offset) / m, float(gw + offset) / m)} if offset else {"size": (gh, gw)}
    patch_pos = F.interpolate(patch_pos.reshape(1, m, m, dim).permute(0, 3, 1, 2), mode="bicubic",
                              antialias=antialias, **kw)
    if tuple(patch_pos.shape[-2:]) != (gh, gw):
        raise _lib.AnylocError(f"pos-embed interpolation produced {tuple(patch_pos.shape[-2:])}, wanted {(gh, gw)}")
    patch_pos = patch_pos.permute(0, 2, 3, 1).reshape(-1, dim)
    return torch.cat([cls_pos, patch_pos], dim=0).contiguous()


class VitWeights:
    """Device-resident, kernel-ready weights of one DINOv2 backbone (blocks 0..depth-1).  A register model's outputs
    hold its num_registers register rows between the cls row and the patch rows, as the reference returns them."""

    def __init__(self, name, state_dict, device, depth=None, pair="tf32"):
        if name not in ARCHS:
            raise ValueError(f"unknown DINOv2 model {name!r}; expected one of {sorted(ARCHS)}")
        if pair not in _lib.PAIR:
            raise ValueError(f"pair must be one of {sorted(_lib.PAIR)}, got {pair!r}")
        self.name = name
        self.pair = pair
        self.dim, full_depth, self.heads, self.ffn_kind = ARCHS[name]
        self.num_registers, self.interp_offset, self.interp_antialias = TOKENS[name]
        if self.num_registers:
            reg = state_dict.get("register_tokens")
            want = (1, self.num_registers, self.dim)
            if reg is None or tuple(reg.shape) != want:
                got = "missing" if reg is None else f"has shape {tuple(reg.shape)}"
                raise ValueError(f"{name} state_dict: 'register_tokens' {got}, expected shape {want}")
        self.device = _lib.require_cuda(device)
        n_blocks = 1 + max([int(k.split(".")[1]) for k in state_dict if k.startswith("blocks.")], default=-1)
        self.depth = min(n_blocks, full_depth if depth is None else depth)
        self.hidden = ffn_hidden(self.dim, self.ffn_kind)
        self._keep = []          # owning references of every device tensor handed to the C side
        self._pos_cache = {}
        lib = _lib.load()
        self.patch_k = lib.anyloc_vit_patch_k(PATCH)
        dev = self.device

        def f32(t):
            return t.detach().to(device=dev, dtype=torch.float32).contiguous()

        def split(t):
            """-> (hi, lo, alpha): the kernel-ready pair of a weight matrix and the accumulator scale
            1/(s_act*s_w) its GEMM epilogue applies (1.0 for tf32 pairs)."""
            t = f32(t)
            with torch.cuda.device(dev):
                if pair == "tf32":
                    hi, lo = torch.empty_like(t), torch.empty_like(t)
                    _lib.check(lib.anyloc_split_tf32(_lib.ptr(t), _lib.ptr(hi), _lib.ptr(lo), t.numel(),
                                                     _lib.stream_ptr()), "split_tf32")
                    alpha = 1.0
                else:
                    # per-tensor power-of-two scale: largest |w| lands in [8192, 16384) -- far from fp16's 65504
                    # ceiling, and typical weights sit well inside the normal range (hi+lo keeps ~22 bits)
                    amax = float(t.abs().max().item())
                    s_w = 2.0 ** math.floor(math.log2(16384.0 / amax)) if amax > 0 else 1.0
                    hi = torch.empty(t.shape, dtype=torch.float16, device=dev)
                    lo = torch.empty(t.shape, dtype=torch.float16, device=dev)
                    _lib.check(lib.anyloc_split_f16(_lib.ptr(t), _lib.ptr(hi), _lib.ptr(lo), t.numel(),
                                                    C.c_float(s_w), _lib.stream_ptr()), "split_f16")
                    alpha = 1.0 / (_lib.ACT_SCALE * s_w)
            self._keep += [hi, lo]
            return hi, lo, alpha

        def keep(t):
            t = f32(t)
            self._keep.append(t)
            return t

        sd = state_dict
        pw = f32(sd["patch_embed.proj.weight"]).reshape(self.dim, -1)
        pw = F.pad(pw, (0, self.patch_k - pw.shape[1]))
        self.patch_w = split(pw)
        patch_alpha = self.patch_w[2]
        self.patch_b = keep(sd["patch_embed.proj.bias"])
        self.cls_token = keep(sd["cls_token"].reshape(-1))
        self.register_tokens = keep(sd["register_tokens"].reshape(self.num_registers, self.dim)) if self.num_registers \
            else None
        self.pos_embed = sd["pos_embed"].detach().float().cpu()
        self.blocks = (_lib.VitBlock * self.depth)()
        for i in range(self.depth):
            p = f"blocks.{i}."
            blk = self.blocks[i]

            def put(field, t):
                setattr(blk, field, t.data_ptr())

            put("ln1_w", keep(sd[p + "norm1.weight"])); put("ln1_b", keep(sd[p + "norm1.bias"]))
            hi, lo, blk.qkv_alpha = split(sd[p + "attn.qkv.weight"]); put("qkv_w_hi", hi); put("qkv_w_lo", lo)
            put("qkv_b", keep(sd[p + "attn.qkv.bias"]))
            hi, lo, blk.proj_alpha = split(sd[p + "attn.proj.weight"]); put("proj_w_hi", hi); put("proj_w_lo", lo)
            put("proj_b", keep(sd[p + "attn.proj.bias"]))
            put("ls1", keep(sd[p + "ls1.gamma"]))
            put("ln2_w", keep(sd[p + "norm2.weight"])); put("ln2_b", keep(sd[p + "norm2.bias"]))
            if self.ffn_kind == "mlp":
                w_in, b_in = sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]
                w_out, b_out = sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"]
            else:
                # interleave so GEMM columns (2j, 2j+1) = (x1_j, x2_j): the SwiGLU epilogue needs
                # both halves of `w12(x).chunk(2)` for the same j in one thread
                h = self.hidden
                perm = torch.stack([torch.arange(h), torch.arange(h) + h], dim=1).reshape(-1)
                w_in = sd[p + "mlp.w12.weight"].detach().cpu()[perm]
                b_in = sd[p + "mlp.w12.bias"].detach().cpu()[perm]
                w_out, b_out = sd[p + "mlp.w3.weight"], sd[p + "mlp.w3.bias"]
            hi, lo, blk.in_alpha = split(w_in); put("in_w_hi", hi); put("in_w_lo", lo); put("in_b", keep(b_in))
            hi, lo, blk.out_alpha = split(w_out); put("out_w_hi", hi); put("out_w_lo", lo); put("out_b", keep(b_out))
            put("ls2", keep(sd[p + "ls2.gamma"]))
        self.cfg = _lib.VitCfg(self.dim, self.depth, self.heads, _lib.FFN[self.ffn_kind], self.hidden, PATCH,
                               _lib.PAIR[pair], self.num_registers)
        self.struct = _lib.VitWeightsStruct(self.patch_w[0].data_ptr(), self.patch_w[1].data_ptr(),
                                            self.patch_b.data_ptr(), self.cls_token.data_ptr(), self.blocks,
                                            patch_alpha,
                                            self.register_tokens.data_ptr() if self.num_registers else None)
        torch.cuda.synchronize(dev)

    def pos_for(self, gh, gw):
        key = (gh, gw)
        if key not in self._pos_cache:
            self._pos_cache[key] = interpolate_pos_embed(self.pos_embed, gh, gw, self.interp_offset,
                                                         self.interp_antialias).to(self.device)
        return self._pos_cache[key]

    def extract(self, img, layer, facet="value", use_cls=False, norm_descs=True, engine="auto"):
        """img [B,3,H,W] fp32 on self.device -> [B, (1 +) R + N, D] fp32 (utilities.py:263-285): the cls row with
        use_cls, then the R = num_registers register rows, then the N patch rows."""
        if img.dim() != 4 or img.shape[1] != 3:
            raise ValueError(f"expected an image batch [B,3,H,W], got {tuple(img.shape)}")
        B, _, H, W = img.shape
        if H % PATCH or W % PATCH:
            raise ValueError(f"image size {(H, W)} is not a multiple of the patch size {PATCH}")
        if not 0 <= layer < self.depth:
            raise IndexError(f"layer {layer} out of range for {self.name} with {self.depth} blocks loaded")
        img = img.to(device=self.device, dtype=torch.float32).contiguous()
        gh, gw = H // PATCH, W // PATCH
        n_out = gh * gw + self.num_registers + (1 if use_cls else 0)
        out = torch.empty(B, n_out, self.dim, device=self.device, dtype=torch.float32)
        lib = _lib.load()
        pos = self.pos_for(gh, gw)
        with torch.cuda.device(self.device):
            nbytes = lib.anyloc_vit_workspace_bytes(C.byref(self.cfg), B, H, W)
            ws = _lib.workspaces.get(self.device, nbytes, "vit")
            rc = lib.anyloc_vit_extract(C.byref(self.cfg), C.byref(self.struct), _lib.ptr(img), B, H, W,
                                        _lib.ptr(pos), layer, _lib.FACET[facet], int(bool(use_cls)),
                                        int(bool(norm_descs)), _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                        _lib.ENGINE[engine], _lib.stream_ptr())
        _lib.check(rc, "anyloc_vit_extract")
        return out

    def extract_varlen(self, imgs, layer, facet="value", use_cls=False, norm_descs=True, engine="auto"):
        """A list of differently sized images [3,H_i,W_i] (or [1,3,H_i,W_i]) fp32 on self.device in one packed forward
        pass (anyloc_vit_extract_varlen) -> (packed [sum n_i, D] fp32, [n_i]), n_i = R + gh_i*gw_i (+1 with use_cls).
        Image i's rows equal extract(imgs[i][None])[0] bit for bit.  Lists longer than the library's per-call limit
        run as consecutive calls into the same packed output."""
        if not 0 <= layer < self.depth:
            raise IndexError(f"layer {layer} out of range for {self.name} with {self.depth} blocks loaded")
        imgs = check_varlen_images(imgs, self.device)
        lay = VarlenLayout([tuple(x.shape[1:]) for x in imgs], use_cls, _lib.VIT_VARLEN_MAX_B, self.num_registers)
        out = torch.empty(lay.rows, self.dim, device=self.device, dtype=torch.float32)
        lib = _lib.load()
        with torch.cuda.device(self.device):
            for s, e in lay.chunks:
                B = e - s
                hw = (C.c_int32 * (2 * B))(*[v for x in imgs[s:e] for v in x.shape[1:]])
                img_p = (C.c_void_p * B)(*[x.data_ptr() for x in imgs[s:e]])
                pos_p = (C.c_void_p * B)(*[self.pos_for(*g).data_ptr() for g in lay.grids[s:e]])
                nbytes = lib.anyloc_vit_varlen_workspace_bytes(C.byref(self.cfg), B, hw)
                ws = _lib.workspaces.get(self.device, nbytes, "vit")
                rc = lib.anyloc_vit_extract_varlen(C.byref(self.cfg), C.byref(self.struct), B, img_p, hw, pos_p, layer,
                                                   _lib.FACET[facet], int(bool(use_cls)), int(bool(norm_descs)),
                                                   C.c_void_p(out[lay.row0[s]:].data_ptr()), _lib.ptr(ws), ws.numel(),
                                                   _lib.ENGINE[engine], _lib.stream_ptr())
                _lib.check(rc, "anyloc_vit_extract_varlen")
        return out, lay.n_out

    def _tap_array(self, taps, out):
        """taps [(layer, facet)] and their outputs out[k] -> the library's tap array"""
        return (_lib.VitTap * len(taps))(*[_lib.VitTap(l, _lib.FACET[f], o.data_ptr()) for (l, f), o in zip(taps, out)])

    def extract_taps(self, img, taps, use_cls=False, norm_descs=True, engine="auto"):
        """Several (layer, facet) features of img [B,3,H,W] from one forward pass (anyloc_vit_extract_taps) ->
        [len(taps), B, (1 +) R + N, D] fp32; item k is taps[k]'s output, equal bit for bit to extract(img, *taps[k])."""
        if img.dim() != 4 or img.shape[1] != 3:
            raise ValueError(f"expected an image batch [B,3,H,W], got {tuple(img.shape)}")
        B, _, H, W = img.shape
        if H % PATCH or W % PATCH:
            raise ValueError(f"image size {(H, W)} is not a multiple of the patch size {PATCH}")
        taps = check_taps(taps, self.depth)
        img = img.to(device=self.device, dtype=torch.float32).contiguous()
        gh, gw = H // PATCH, W // PATCH
        n_out = gh * gw + self.num_registers + (1 if use_cls else 0)
        out = torch.empty(len(taps), B, n_out, self.dim, device=self.device, dtype=torch.float32)
        arr = self._tap_array(taps, out)
        lib = _lib.load()
        pos = self.pos_for(gh, gw)
        with torch.cuda.device(self.device):
            nbytes = lib.anyloc_vit_taps_workspace_bytes(C.byref(self.cfg), B, H, W, arr, len(taps))
            ws = _lib.workspaces.get(self.device, nbytes, "vit")
            rc = lib.anyloc_vit_extract_taps(C.byref(self.cfg), C.byref(self.struct), _lib.ptr(img), B, H, W,
                                             _lib.ptr(pos), arr, len(taps), int(bool(use_cls)), int(bool(norm_descs)),
                                             _lib.ptr(ws), ws.numel(), _lib.ENGINE[engine], _lib.stream_ptr())
        _lib.check(rc, "anyloc_vit_extract_taps")
        return out

    def extract_taps_varlen(self, imgs, taps, use_cls=False, norm_descs=True, engine="auto"):
        """extract_taps for a list of differently sized images (anyloc_vit_extract_taps_varlen) -> (packed
        [len(taps), sum n_i, D] fp32, [n_i]), laid out per tap as extract_varlen's output.  Lists longer than the
        library's per-call limit run as consecutive calls into the same packed output."""
        taps = check_taps(taps, self.depth)
        imgs = check_varlen_images(imgs, self.device)
        lay = VarlenLayout([tuple(x.shape[1:]) for x in imgs], use_cls, _lib.VIT_VARLEN_MAX_B, self.num_registers)
        out = torch.empty(len(taps), lay.rows, self.dim, device=self.device, dtype=torch.float32)
        lib = _lib.load()
        with torch.cuda.device(self.device):
            for s, e in lay.chunks:
                B = e - s
                hw = (C.c_int32 * (2 * B))(*[v for x in imgs[s:e] for v in x.shape[1:]])
                img_p = (C.c_void_p * B)(*[x.data_ptr() for x in imgs[s:e]])
                pos_p = (C.c_void_p * B)(*[self.pos_for(*g).data_ptr() for g in lay.grids[s:e]])
                arr = self._tap_array(taps, out[:, lay.row0[s]:])
                nbytes = lib.anyloc_vit_taps_varlen_workspace_bytes(C.byref(self.cfg), B, hw, arr, len(taps))
                ws = _lib.workspaces.get(self.device, nbytes, "vit")
                rc = lib.anyloc_vit_extract_taps_varlen(C.byref(self.cfg), C.byref(self.struct), B, img_p, hw, pos_p,
                                                        arr, len(taps), int(bool(use_cls)), int(bool(norm_descs)),
                                                        _lib.ptr(ws), ws.numel(), _lib.ENGINE[engine],
                                                        _lib.stream_ptr())
                _lib.check(rc, "anyloc_vit_extract_taps_varlen")
        return out, lay.n_out


def check_taps(taps, depth):
    """A tap list as [(layer, facet)] in the given order; ValueError on an empty list, an item that is not a
    (layer, facet) pair, an unknown facet or a repeated tap, IndexError on a layer outside [0, depth)."""
    if isinstance(taps, (str, bytes)) or not hasattr(taps, "__iter__"):
        raise ValueError(f"expected a list of (layer, facet) taps, got {taps!r}")
    res = []
    for t in taps:
        if not isinstance(t, (tuple, list)) or len(t) != 2 or isinstance(t[0], bool):
            raise ValueError(f"a tap is a (layer, facet) pair, got {t!r}")
        try:
            layer = operator.index(t[0])
        except TypeError:
            raise ValueError(f"tap {t!r}: the layer must be an integer") from None
        facet = t[1]
        if facet not in _lib.FACET:
            raise ValueError(f"tap {t!r}: facet must be one of {sorted(_lib.FACET)}")
        if not 0 <= layer < depth:
            raise IndexError(f"tap {t!r}: layer out of range for {depth} blocks")
        if (layer, facet) in res:
            raise ValueError(f"tap {(layer, facet)!r} is requested twice")
        res.append((layer, facet))
    if not res:
        raise ValueError("expected a non-empty list of (layer, facet) taps")
    return res


def check_varlen_images(imgs, device):
    """The items of a list input as [3,H,W] fp32 contiguous tensors on `device`; ValueError on an empty list, a wrong
    rank or channel count, a size that is not a positive multiple of the patch size, or an image on another device.
    Images are used in place (their data pointers go to the library), converted only if not fp32 contiguous."""
    if not isinstance(imgs, (list, tuple)) or len(imgs) == 0:
        raise ValueError("expected a non-empty list of images [3,H,W] or [1,3,H,W]")
    res = []
    for i, x in enumerate(imgs):
        if not isinstance(x, torch.Tensor):
            raise ValueError(f"image {i} is a {type(x).__name__}, not a tensor")
        if x.dim() == 4 and x.shape[0] == 1:
            x = x[0]
        if x.dim() != 3 or x.shape[0] != 3:
            raise ValueError(f"image {i}: expected [3,H,W] or [1,3,H,W], got {tuple(x.shape)}")
        H, W = x.shape[1:]
        if H == 0 or W == 0 or H % PATCH or W % PATCH:
            raise ValueError(f"image {i}: size {(H, W)} is not a multiple of the patch size {PATCH}")
        if x.device != device:
            raise ValueError(f"image {i} is on {x.device}, the extractor on {device}")
        res.append(x.to(dtype=torch.float32).contiguous())
    return res


class VarlenLayout:
    """Where each image of a list input lands: grids (gh_i, gw_i), tokens T_i = 1 + registers + gh_i*gw_i, output rows
    n_i (T_i - 1 without the cls token), their offsets row0 in the packed output (row0[-1] = rows) and the consecutive
    (start, stop) slices of at most max_b images, one library call each."""

    def __init__(self, sizes, use_cls, max_b, registers=0):
        self.grids = [(H // PATCH, W // PATCH) for H, W in sizes]
        self.tokens = [1 + registers + gh * gw for gh, gw in self.grids]
        self.n_out = [t - (0 if use_cls else 1) for t in self.tokens]
        self.row0 = [0]
        for n in self.n_out:
            self.row0.append(self.row0[-1] + n)
        self.rows = self.row0[-1]
        self.chunks = [(s, min(s + max_b, len(sizes))) for s in range(0, len(sizes), max_b)]


def resolve_state_dict(name, device):
    """Where the weights come from, in order: $ANYLOC_B200_WEIGHTS_DIR/<name>.pth (a plain upstream
    state_dict), the torch.hub checkpoint the reference itself loads (utilities.py:239-240; needs
    network or a warm hub cache), or -- only when ANYLOC_B200_RANDOM_INIT=1 -- a seeded random init
    for synthetic benchmarks."""
    wdir = os.environ.get("ANYLOC_B200_WEIGHTS_DIR")
    if wdir:
        path = os.path.join(wdir, f"{name}.pth")
        if os.path.isfile(path):
            return torch.load(path, map_location="cpu")
    if os.environ.get("ANYLOC_B200_RANDOM_INIT") == "1":
        return random_state_dict(name, seed=int(os.environ.get("ANYLOC_B200_SEED", "0")), device=device)
    try:
        model = torch.hub.load("facebookresearch/dinov2", name)
    except Exception as e:  # offline box
        raise _lib.AnylocError(
            f"cannot obtain weights for {name}: torch.hub.load failed ({type(e).__name__}: {e}). Put an upstream "
            f"state_dict at $ANYLOC_B200_WEIGHTS_DIR/{name}.pth, or set ANYLOC_B200_RANDOM_INIT=1 for "
            "synthetic benchmarking") from e
    if hasattr(model, "state_dict"):
        return model.state_dict()
    return model
