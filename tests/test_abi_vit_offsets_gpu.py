"""The four anyloc_vit_extract* entries at the pointer offsets their rows of the alignment table accept
(tests/test_abi_alignment_cpu.py ALIGN): every weight, image, positional table, output and the workspace at +16 / +48
bytes (16 required) or +4 / +12 (4 required) past a 256-byte boundary, inside NaN frames, in the six weight formats,
on a 2-block ViT-S/14 without and with 4 register tokens.  Each call must give, bit for bit, what the same call on
256-byte aligned buffers gives, with the same number of launches, the same number of tensor-core and SIMT GEMM groups
(the profiler's gemm_tc / gemm_simt counts: an accepted buffer never moves a GEMM off its route) and intact frames.
The single and tap calls run two 56x56 images (32 patch rows and 34 / 42 token rows: the tensor-core GEMMs under
ANYLOC_GEMM_AUTO); the list calls run a 28x42 and a 42x42 image (15 patch rows: the tf32 and fp16 pairs' patch GEMM takes
the SIMT kernel there, so both GEMM engines read offset weights; the single formats and the bf16 pairs have no SIMT
kernel).  The single calls return block 1's value facet, the tap
calls block 0's query (below the deepest layer: qkv_tap_kernel writes it) and block 1's token output
(facet_out_kernel).  One ViT-S forward at full depth is also held to
test_vit_accuracy_gpu.py's fp64 bounds at offsets, and VitWeights is shown to copy a state dict of misaligned views
before any pointer reaches the library.  No pointer below its alignment is passed here; the refusals are
test_abi_alignment_cpu.py's."""
import ctypes as C

import pytest
import torch

from tests.test_abi_alignment_cpu import ALIGN, VIT_BLOCK_FIELDS, VIT_DEPTH
from tests.test_abi_offsets_gpu import L, accepted, run  # noqa: F401  (L: the library fixture)

pytestmark = pytest.mark.gpu

PAIRS = ("tf32", "f16", "bf16", "fp8", "f16x1", "bf16pair")
KINDS = {"single": "anyloc_vit_extract", "taps": "anyloc_vit_extract_taps", "varlen": "anyloc_vit_extract_varlen",
         "taps_varlen": "anyloc_vit_extract_taps_varlen"}
TAPS = ((0, "query"), (1, "token"))
LIST_HW = ((28, 42), (42, 42))
_WEIGHTS = {}


def model(regs, depth=VIT_DEPTH):
    """the fp32 CPU model: perturbed random ViT-S/14 weights (non-zero biases, LayerNorm gains and LayerScales)"""
    from oracle import dinov2_restated as dr
    from tests import dinov2_reg_restated as dreg
    if regs:
        return dreg.model("dinov2_vits14_reg", depth_override=depth).float().eval()
    return dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=depth), seed=1).float().eval()


def weights(pair, regs):
    from anyloc_b200 import vit
    if (pair, regs) not in _WEIGHTS:
        name = "dinov2_vits14_reg" if regs else "dinov2_vits14"
        _WEIGHTS[(pair, regs)] = vit.VitWeights(name, model(regs).state_dict(), torch.device("cuda", 0), pair=pair)
    return _WEIGHTS[(pair, regs)]


def weight_tensors(w):
    """{table name: the device tensor that pointer of w's structs points at, or None}, for every block of w"""
    by_ptr = {t.data_ptr(): t for t in w._keep if t is not None}
    d = {"w.patch_w_hi": w.patch_w[0], "w.patch_w_lo": w.patch_w[1], "w.patch_b": w.patch_b,
         "w.cls_token": w.cls_token, "w.register_tokens": w.register_tokens}
    for l in range(w.depth):
        for f in VIT_BLOCK_FIELDS:
            p = getattr(w.blocks[l], f)
            d[f"blocks[{l}].{f}"] = None if p is None else by_ptr[p]
    return d


def align_of(entry, name):
    """the table's alignment of a name; block l of a deeper model has block 0's, tap i of a longer list tap 0's"""
    if name.startswith("blocks["):
        name = "blocks[0]." + name.split(".", 1)[1]
    elif name.startswith("taps["):
        name = "taps[0].out"
    return ALIGN[entry][name]


def struct_of(w, p):
    """w's AnylocVitWeights with the placed pointers p (ctypes pointers; 0 for a null one)"""
    from anyloc_b200 import _lib
    blocks = (_lib.VitBlock * w.depth)()
    for l in range(w.depth):
        C.pointer(blocks[l])[0] = w.blocks[l]                   # the alphas
        for f in VIT_BLOCK_FIELDS:
            setattr(blocks[l], f, p[f"blocks[{l}].{f}"].value)
    return _lib.VitWeightsStruct(p["w.patch_w_hi"].value, p["w.patch_w_lo"].value, p["w.patch_b"].value,
                                 p["w.cls_token"].value, blocks, w.struct.patch_alpha, p["w.register_tokens"].value)


def spec(L, w, kind, taps=TAPS, hw=(56, 56), seed=3):
    """(buffers, outputs, call) of one ViT call, as test_abi_offsets_gpu.spec; the call also records the profiler's
    GEMM groups in groups[0]"""
    from anyloc_b200 import _lib
    lib, st = L.load(), L.stream_ptr()
    D, R, B = w.dim, w.num_registers, 2
    bufs = weight_tensors(w)
    g = torch.Generator(device="cuda").manual_seed(seed)
    # the single calls: block 1's value facet (block 0 whole, then block 1's norm1 and the value third of its qkv GEMM)
    tap_list = [(l, _lib.FACET[f]) for l, f in (taps if kind.startswith("taps") else ((1, "value"),))]
    if kind in ("single", "taps"):
        H, W = hw
        bufs.update(img=torch.randn(B, 3, H, W, device="cuda", generator=g), pos_embed=w.pos_for(H // 14, W // 14))
        rows = B * (R + (H // 14) * (W // 14))
    else:
        for i, (H, W) in enumerate(LIST_HW):
            bufs[f"img[{i}]"] = torch.randn(3, H, W, device="cuda", generator=g)
            bufs[f"pos_embed[{i}]"] = w.pos_for(H // 14, W // 14)
        hw_arr = (C.c_int32 * 4)(*[v for s in LIST_HW for v in s])
        rows = sum(R + (H // 14) * (W // 14) for H, W in LIST_HW)
    outs = [f"taps[{i}].out" for i in range(len(tap_list))] if kind.startswith("taps") else ["out"]
    bufs.update({o: rows * D * 4 for o in outs})
    cfg = C.byref(w.cfg)
    arr = (_lib.VitTap * len(tap_list))(*[_lib.VitTap(l, f, None) for l, f in tap_list])
    bufs["ws"] = int({"single": lambda: lib.anyloc_vit_workspace_bytes(cfg, B, *hw),
                      "taps": lambda: lib.anyloc_vit_taps_workspace_bytes(cfg, B, *hw, arr, len(arr)),
                      "varlen": lambda: lib.anyloc_vit_varlen_workspace_bytes(cfg, 2, hw_arr),
                      "taps_varlen": lambda: lib.anyloc_vit_taps_varlen_workspace_bytes(cfg, 2, hw_arr, arr,
                                                                                         len(arr))}[kind]())
    groups = [None]

    def call(p, n):
        wst = struct_of(w, p)
        t = (_lib.VitTap * len(tap_list))(*[_lib.VitTap(l, f, p[o].value) for (l, f), o in zip(tap_list, outs)])
        if kind.startswith("taps"):
            t_args = (t, len(t))
        else:
            t_args = (tap_list[0][0], tap_list[0][1])
        L.profile_enable(True)
        if kind in ("single", "taps"):
            fn = lib.anyloc_vit_extract if kind == "single" else lib.anyloc_vit_extract_taps
            head = (C.byref(wst), p["img"], B, *hw, p["pos_embed"]) + t_args
        else:
            fn = lib.anyloc_vit_extract_varlen if kind == "varlen" else lib.anyloc_vit_extract_taps_varlen
            head = (C.byref(wst), 2, (C.c_void_p * 2)(p["img[0]"].value, p["img[1]"].value), hw_arr,
                    (C.c_void_p * 2)(p["pos_embed[0]"].value, p["pos_embed[1]"].value)) + t_args
        tail = (0, 1) + (() if kind.startswith("taps") else (p["out"],)) + (p["ws"], n["ws"], 0, st)
        rc = fn(cfg, *head, *tail)
        prof = L.profile_read()
        L.profile_enable(False)
        groups[0] = (prof["gemm_tc"][1], prof["gemm_simt"][1])
        return rc

    return bufs, outs, call, groups


def offsets(entry, bufs, pattern):
    """each present buffer at one of its accepted offsets, alternating from one buffer to the next"""
    names = [n for n, v in bufs.items() if v is not None]
    return {n: accepted(align_of(entry, n))[(k + pattern) % 2] for k, n in enumerate(names)}


CASES = [(pair, regs, kind) for pair in PAIRS for regs in (0, 4) for kind in KINDS]


@pytest.mark.parametrize("pair,regs,kind", CASES, ids=[f"{p}-r{r}-{k}" for p, r, k in CASES])
def test_vit_offsets_match_aligned_call(L, pair, regs, kind):
    w = weights(pair, regs)
    entry = KINDS[kind]
    bufs, outs, call, groups = spec(L, w, kind)
    assert {n for n, v in bufs.items() if v is not None} <= set(ALIGN[entry]), set(bufs) - set(ALIGN[entry])
    rc, launches, ref, intact, _ = run(L, bufs, outs, call, {})
    ref_groups = groups[0]
    assert rc == 0 and intact, (rc, L.last_error())
    assert all(torch.isfinite(ref[o].view(torch.float32)).all() for o in outs)
    if kind in ("single", "taps") or pair in ("bf16", "fp8", "f16x1", "bf16pair"):
        assert ref_groups[1] == 0, ref_groups          # M >= 32 or a single format: tensor cores only
    else:
        assert ref_groups[1] > 0, ref_groups           # the 15-row patch GEMM: SIMT
    for pattern in (0, 1):
        offs = offsets(entry, bufs, pattern)
        rc2, l2, got, intact2, _ = run(L, bufs, outs, call, offs)
        assert rc2 == 0, (pattern, L.last_error())
        assert l2 == launches and groups[0] == ref_groups, (pattern, l2, launches, groups[0], ref_groups)
        assert intact2, (pattern, "a frame was overwritten")
        for o in outs:
            assert torch.equal(got[o], ref[o]), (pattern, o)


def test_vit_offsets_hold_the_fp64_bound(L):
    # ViT-S at full depth, tf32 pairs on the tensor cores, two 112x112 images, every pointer at an accepted offset:
    # each tap within test_vit_accuracy_gpu.py's kappa of the fp64 forward
    from anyloc_b200 import vit
    from tests import test_vit_accuracy_gpu as A
    m = A.model_of("vits", "random")
    depth = len(m.blocks)
    w = vit.VitWeights("dinov2_vits14", m.state_dict(), torch.device("cuda", 0), pair="tf32")
    hw = (112, 112)
    taps = [(0, "query"), (depth // 2, "key"), (depth - 1, "value"), (depth - 1, "token")]
    bufs, outs, call, groups = spec(L, w, "taps", taps=taps, hw=hw)
    bufs["img"] = A.image(hw).cuda()
    rc, _, got, intact, _ = run(L, bufs, outs, call, offsets("anyloc_vit_extract_taps", bufs, 1))
    assert rc == 0 and intact, L.last_error()
    assert groups[0][1] == 0, groups[0]
    r64, r32 = A.refs("vits", "random", hw)
    for i, tap in enumerate(taps):
        out = got[f"taps[{i}].out"].view(torch.float32).view(2, -1, w.dim)
        rr, rm, s, c = A.ratios(out, r64, r32, tap, False, True)
        assert rr <= A.KAPPA_ROW and rm <= A.KAPPA_RMS, (tap, rr, rm, s, c)


def test_vit_weights_copy_misaligned_views(L):
    # every tensor of the state dict a view 4 bytes past a 16-byte boundary of one CUDA buffer: VitWeights must hand
    # the library 16-byte aligned copies (checked before anything runs), and extract what the aligned weights extract
    from anyloc_b200 import vit
    sd = model(4).state_dict()
    buf = torch.empty(sum(t.numel() + 8 for t in sd.values()) + 8, device="cuda")
    views, off = {}, 1
    for k, t in sd.items():
        views[k] = buf[off:off + t.numel()].view(t.shape)
        views[k].copy_(t)
        assert views[k].data_ptr() % 16 == 4
        off += (t.numel() + 3) // 4 * 4 + 4
    img = torch.randn(2, 3, 56, 42, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    for pair in PAIRS:
        w = vit.VitWeights("dinov2_vits14_reg", views, torch.device("cuda", 0), pair=pair)
        ptrs = {f: getattr(w.struct, f) for f in ("patch_w_hi", "patch_w_lo", "patch_b", "cls_token",
                                                   "register_tokens")}
        ptrs.update({f"blocks[{l}].{f}": getattr(w.blocks[l], f) for l in range(w.depth) for f in VIT_BLOCK_FIELDS})
        bad = {n: p % 16 for n, p in ptrs.items() if p is not None and p % 16}
        assert not bad, (pair, bad)
        got = w.extract(img, 1, "value")
        ref = weights(pair, 4).extract(img, 1, "value")
        assert torch.equal(got, ref), pair
        for k, t in sd.items():
            assert torch.equal(views[k].cpu(), t), k           # the caller's tensors are left as they were
