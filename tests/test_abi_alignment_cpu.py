"""Alignment checks of the C entry points, without a GPU.  anyloc_pool reads the features and writes the output with
float4 accesses, anyloc_preprocess_u8 stores pairs of columns as float2 when Wc is even, and every pre-processing kernel
stores fp32 elements, so a pointer those accesses would fault on is refused before any CUDA call: the placeholder device
pointers here are never touched.  Calls with nothing to do (B = 0, n = 0) and aligned pointers still return OK without
launching.  The table ALIGN below does the same for every other entry that takes device pointers, and the header's
prototypes and ViT structs are checked against it."""
import ctypes as C
import re

import pytest

from anyloc_b200 import _lib

P = 4096                    # placeholder device address, 16-byte aligned
ARG = _lib.ERR["arg"]
AVG, MAX, GEM = 0, 1, 2
M3 = (C.c_float * 3)(0.485, 0.456, 0.406)
S3 = (C.c_float * 3)(0.229, 0.224, 0.225)


def _pool(lib, B=2, N=9, D=36, mode=AVG, feats=P, out=P, n_valid=None, p=3.0):
    return lib.anyloc_pool(C.c_void_p(feats), C.c_void_p(n_valid), B, N, D, mode, C.c_float(p), 0, C.c_void_p(out),
                           None)


def _crop(lib, B=1, Wc=28, out=P):
    return lib.anyloc_preprocess_u8(C.c_void_p(P), B, 56, 57, 0, 0, 28, Wc, M3, S3, C.c_void_p(out), None)


def _resize(lib, B=1, Wc=28, out=P):
    return lib.anyloc_preprocess_resize_u8(C.c_void_p(P), B, 100, 90, 56, 57, 1, 0, 0, 28, Wc, M3, S3,
                                           C.c_void_p(out), None)


def _varlen(lib, n=1, interp=-1, out=P):
    def ints(v):
        return (C.c_int * 1)(v)
    return lib.anyloc_preprocess_u8_varlen(n, (C.c_void_p * 1)(P), ints(56), ints(57), ints(56), ints(57), interp,
                                           ints(0), ints(0), ints(28), ints(27), M3, S3, C.c_void_p(out),
                                           (C.c_int64 * 1)(0), None)


def test_pool_refuses_misaligned_pointers(lib):
    for mode in (AVG, MAX, GEM):
        for B in (0, 2):
            for kw in (dict(feats=P + 4), dict(feats=P + 8), dict(feats=P + 12), dict(feats=P + 1),
                       dict(out=P + 4), dict(out=P + 8), dict(out=P + 12), dict(out=P + 2)):
                assert _pool(lib, B=B, mode=mode, **kw) == ARG, (mode, B, kw)
                assert "16-byte aligned" in _lib.last_error()
        assert _pool(lib, B=0, mode=mode) == 0                  # nothing to do, nothing launched
        assert _pool(lib, B=0, mode=mode, feats=P + 16, out=P + 32, n_valid=P + 4) == 0


def test_pool_other_refusals_unchanged(lib):
    assert _pool(lib, feats=0) == ARG and "null pointer" in _lib.last_error()
    for B, N, D in ((-1, 9, 36), (2, 0, 36), (2, 9, 0), (2, 9, 38), (65536, 1, 4)):
        assert _pool(lib, B=B, N=N, D=D) == ARG, (B, N, D)
    assert _pool(lib, B=0, mode=3) == ARG and "unknown mode" in _lib.last_error()
    assert _pool(lib, B=0, mode=GEM, p=0.0) == ARG and "non-zero" in _lib.last_error()


def test_preprocess_u8_alignment(lib):
    # odd Wc: the kernel stores one float at a time, 4-byte alignment is enough
    for off in (1, 2, 3):
        assert _crop(lib, B=0, Wc=27, out=P + off) == ARG, off
        assert "4-byte aligned" in _lib.last_error()
    assert _crop(lib, B=0, Wc=27, out=P + 4) == 0
    # even Wc: pairs of columns are float2 stores
    for off in (1, 2, 3, 4, 5, 6, 7, 12):
        assert _crop(lib, B=0, Wc=28, out=P + off) == ARG, off
        assert "8-byte aligned when Wc is even" in _lib.last_error()
    assert _crop(lib, B=0, Wc=28, out=P + 8) == 0
    assert _crop(lib, B=3, Wc=28, out=P + 4) == ARG             # refused before the launch, whatever B


def test_preprocess_resize_and_list_alignment(lib):
    for Wc in (27, 28):
        for off in (1, 2, 3):
            assert _resize(lib, B=0, Wc=Wc, out=P + off) == ARG, (Wc, off)
            assert "4-byte aligned" in _lib.last_error()
            assert _resize(lib, B=1, Wc=Wc, out=P + off) == ARG, (Wc, off)
        assert _resize(lib, B=0, Wc=Wc, out=P + 4) == 0         # fp32 stores only
    for interp in (-1, 0, 1):
        for off in (1, 2, 3):
            assert _varlen(lib, n=1, interp=interp, out=P + off) == ARG, (interp, off)
            assert "4-byte aligned" in _lib.last_error()
            assert _varlen(lib, n=0, interp=interp, out=P + off) == ARG, (interp, off)
        assert _varlen(lib, n=0, interp=interp, out=P + 4) == 0


# ---------------------------------------------------------------------------------------------------------------------
# The alignment each entry requires of each pointer it takes: the widest access any of its routes makes through that
# pointer (float4 / uint4 / TMA: 16, int64 / fp64 / a 64-bit store: 8, fp32 / int32: 4).  A workspace or blob inherits
# the base's alignment in every buffer carved from it, so it needs what its strictest buffer needs.  Where the pointer
# reaches the tensor-core GEMM, TMA or the wgmma attention it is 16 even when the fallback kernel would accept less, so
# that an accepted buffer never changes the route.  Host arrays of device pointers are named by element (centers[1]),
# the fields of the ViT's structs as w.patch_b, blocks[1].ln2_w and taps[1].out.  test_abi_offsets_gpu.py and
# test_abi_vit_offsets_gpu.py hand every entry real buffers at the offsets this table accepts.  DESIGN.md section 2
# lists the kernels' 64- and 128-bit accesses that each entry traces back to.
VIT_BLOCK_FIELDS = ("ln1_w", "ln1_b", "qkv_w_hi", "qkv_w_lo", "qkv_b", "proj_w_hi", "proj_w_lo", "proj_b", "ls1",
                    "ln2_w", "ln2_b", "in_w_hi", "in_w_lo", "in_b", "out_w_hi", "out_w_lo", "out_b", "ls2")
VIT_DEPTH = 2                   # two blocks and two taps / images, so that a check of element 0 alone is caught


def _vit_row(images, outs):
    """a ViT entry's row: the workspace, the weights of blocks 0..VIT_DEPTH-1, the images and positional tables (named
    `images`), the outputs (named `outs`)"""
    row = {"ws": 16, "w.patch_w_hi": 16, "w.patch_w_lo": 16, "w.patch_b": 16, "w.cls_token": 4,
           "w.register_tokens": 4}
    row.update({f"blocks[{l}].{f}": 16 for l in range(VIT_DEPTH) for f in VIT_BLOCK_FIELDS})
    row.update({n: 4 for n in images})
    row.update({n: 16 for n in outs})
    return row


ALIGN = {
    "anyloc_vlad_assign": {"feats": 16, "centers": 4, "labels": 4, "ws": 16},
    "anyloc_vlad_assign_multi": {"feats": 16, "centers[0]": 4, "centers[1]": 4, "labels": 4, "ws": 16},
    "anyloc_vlad_prepare": {"centers": 4, "prepared": 16},
    "anyloc_vlad_generate": {"feats": 16, "n_valid": 4, "centers": 16, "vlad": 16, "labels": 4, "ws": 16},
    "anyloc_vlad_generate_prepared": {"feats": 16, "n_valid": 4, "centers": 16, "prepared": 16, "vlad": 16,
                                      "labels": 4, "ws": 16},
    "anyloc_vlad_generate_sorted": {"feats": 16, "n_valid": 4, "centers": 16, "prepared": 16, "vlad": 16,
                                    "labels": 4, "ws": 16},
    "anyloc_vlad_generate_soft": {"feats": 16, "n_valid": 4, "centers": 4, "vlad": 4, "assign": 4, "ws": 16},
    "anyloc_vlad_generate_varlen": {"feats": 16, "row0": 8, "len": 4, "centers": 16, "prepared": 16, "vlad": 16,
                                    "labels": 4, "ws": 16},
    "anyloc_vlad_generate_soft_varlen": {"feats": 16, "row0": 8, "len": 4, "centers": 4, "vlad": 16, "assign": 4,
                                         "ws": 16},
    "anyloc_vlad_residuals": {"feats": 16, "centers": 16, "out": 16},
    "anyloc_vlad_from_residuals": {"resid": 4, "labels": 4, "assign": 4, "vlad": 4, "ws": 4},
    "anyloc_kmeans_update": {"x": 4, "labels": 4, "old_centers": 4, "new_centers": 4, "err_out": 4, "ws": 4},
    "anyloc_kmeans_update_tiled": {"x": 4, "labels": 4, "old_centers": 4, "new_centers": 4, "err_out": 4, "ws": 4},
    "anyloc_kmeans_accumulate_round": {"x": 4, "labels": 4, "ws": 4},
    "anyloc_kmeans_accumulate_round_tiled": {"x": 4, "labels": 4, "ws": 4},
    "anyloc_kmeans_accumulate_round_multi": {"x": 4, "labels[0]": 4, "labels[1]": 4, "ws[0]": 4, "ws[1]": 4},
    "anyloc_kmeans_finalize": {"old_centers": 4, "new_centers": 4, "err_out": 4, "ws": 4},
    "anyloc_index_init": {"index": 16},
    "anyloc_index_add": {"index": 16, "rows": 16},
    "anyloc_index_copy": {"dst": 16, "src": 16},
    "anyloc_index_search": {"index": 16, "qu": 16, "dist": 4, "idx": 8, "ws": 16},
    "anyloc_index_search_continue": {"index": 16, "qu": 16, "dist": 4, "idx": 8, "ws": 16},
    "anyloc_index_split_init": {"index": 16},
    "anyloc_index_split_copy": {"dst": 16, "src": 16},
    "anyloc_index_split_add": {"index": 16, "lo": 16, "rows": 16},
    "anyloc_index_split_piece": {"dst": 16, "index": 16, "lo": 16},
    "anyloc_index_split_search": {"index": 16, "qu": 16, "ws": 16, "counts": 8},
    "anyloc_index_split_rescore": {"index": 16, "lo": 16, "ws": 16, "stage": 16, "dist": 4, "idx": 8},
    "anyloc_topk": {"db": 16, "qu": 16, "dist": 4, "idx": 8, "ws": 16},
    "anyloc_pca_colsum": {"x": 4, "sum": 8, "ws": 8},
    "anyloc_pca_accumulate": {"x": 4, "mu": 8, "u": 8, "out": 8},
    "anyloc_pca_mirror": {"a": 8},
    "anyloc_pool": {"feats": 16, "n_valid": 4, "out": 16},
    "anyloc_pool_varlen": {"feats": 16, "row0": 8, "len": 4, "out": 16},
    "anyloc_vlad_label_multi": {"feats": 16, "n_valid": 4, "centers[0]": 4, "centers[1]": 4, "prepared[0]": 16,
                                "prepared[1]": 16, "labels": 4, "inv_norm": 4, "ws": 16},
    "anyloc_vlad_soft_assign_multi": {"feats": 16, "n_valid": 4, "centers[0]": 4, "centers[1]": 4, "assign[0]": 4,
                                      "assign[1]": 4, "inv_norm": 4, "ws": 16},
    "anyloc_vlad_accumulate": {"feats": 16, "n_valid": 4, "labels": 4, "assign": 4, "inv_norm": 4, "centers": 16,
                               "vlad": 16, "ws": 16},
    "anyloc_vlad_accumulate_varlen": {"feats": 16, "row0": 8, "len": 4, "labels": 4, "assign": 4, "inv_norm": 4,
                                      "centers": 16, "vlad": 16, "ws": 16},
    # o: the 64-bit stores of attention_tc_kernel's epilogue (the SIMT and wgmma kernels store 32 bits)
    "anyloc_attention": {"qkv_hi": 16, "qkv_lo": 16, "o_hi": 8, "o_lo": 8},
    "anyloc_attention_varlen": {"qkv_hi": 16, "qkv_lo": 16, "o_hi": 8, "o_lo": 8},
    "anyloc_vit_extract": _vit_row(("img", "pos_embed"), ("out",)),
    "anyloc_vit_extract_taps": _vit_row(("img", "pos_embed"), ("taps[0].out", "taps[1].out")),
    "anyloc_vit_extract_varlen": _vit_row(("img[0]", "img[1]", "pos_embed[0]", "pos_embed[1]"), ("out",)),
    "anyloc_vit_extract_taps_varlen": _vit_row(("img[0]", "img[1]", "pos_embed[0]", "pos_embed[1]"),
                                               ("taps[0].out", "taps[1].out")),
}

# The attention entries' rows hold for every format they take; their refusals run in the tf32 pairs (format 0) and
# again in the bf16 pairs.
X3 = _lib.PAIR["bf16pair"]
ATTENTION_FMTS = (0, X3)

# Pointers whose alignment chooses a route instead of being refused, as documented: below 16 bytes a tf32-pair qkv runs
# anyloc_attention's SIMT kernel under ANYLOC_GEMM_AUTO (B = 0 here: OK, nothing to run); a bf16-pair qkv has no SIMT
# kernel, and anyloc_attention returns ANYLOC_ERR_UNSUPPORTED even at B = 0 (it checks the qkv before the empty batch);
# anyloc_attention_varlen returns ANYLOC_ERR_UNSUPPORTED in both formats.  (entry, pointer, format) -> the code
# expected below the alignment.
BELOW = {("anyloc_attention", "qkv_hi", 0): 0, ("anyloc_attention", "qkv_lo", 0): 0,
         ("anyloc_attention", "qkv_hi", X3): _lib.ERR["unsupported"],
         ("anyloc_attention", "qkv_lo", X3): _lib.ERR["unsupported"]}
BELOW.update({("anyloc_attention_varlen", n, f): _lib.ERR["unsupported"] for n in ("qkv_hi", "qkv_lo")
              for f in ATTENTION_FMTS})

# The entries with device pointers that the table leaves out: why, and the tests that cover their alignment.
EXEMPT = {
    "anyloc_gemm_nt": ("alignment chooses the tensor-core or SIMT route under AUTO", "test_gemm_engine_gpu.py"),
    "anyloc_layernorm_split": ("y_hi / y_lo need 4 elements of the output format", "test_vit_rows_cpu.py"),
    "anyloc_preprocess_u8": ("out needs 8 bytes when Wc is even, 4 when odd", "test_abi_alignment_cpu.py"),
    "anyloc_preprocess_resize_u8": ("fp32 stores only, refused above", "test_abi_alignment_cpu.py"),
    "anyloc_preprocess_u8_varlen": ("fp32 stores only, refused above", "test_abi_alignment_cpu.py"),
    "anyloc_l2_normalize_rows": ("one message names x and y together", "test_vit_rows_cpu.py"),
    "anyloc_quantize_fp8_rows": ("one message names x, q and scales together", "test_fp8_edges_gpu.py"),
    "anyloc_quantize_fp8_tensor": ("element-wise kernels, natural alignment", "test_fp8_kernels_gpu.py"),
    "anyloc_split_tf32": ("element-wise kernel, natural alignment", "test_ops_gpu.py"),
    "anyloc_split_f16": ("element-wise kernel, natural alignment", "test_f16x1_kernels_gpu.py"),
    "anyloc_split_bf16": ("element-wise kernel, natural alignment", "test_bf16_kernels_gpu.py"),
    "anyloc_allgather_desc": ("NCCL's all-gather reads and writes the buffers", "test_dist_gpu.py"),
    "anyloc_device_info": ("host pointers only", "test_abi_cpu.py"),
    "anyloc_profile_read": ("host pointers only", "test_retrieval_engine_gpu.py"),
    "anyloc_kmeans_partition": ("host pointers only", "test_kmeans_stream_cpu.py"),
}

OK, WS, UNS = 0, _lib.ERR["workspace"], _lib.ERR["unsupported"]
D_, K_ = 8, 4                   # every call below: 8 columns, 4 clusters
VIT_CFG = _lib.VitCfg(384, VIT_DEPTH, 6, 0, 1536, 14, 0, 4)   # ViT-S/14, tf32 pairs, 4 register tokens
VIT_TAPS = ((0, 0), (1, 3))     # block 0's query, block 1's token output
VIT_HW = (C.c_int32 * 4)(28, 42, 42, 42)


def _vp(*xs):
    return (C.c_void_p * len(xs))(*xs)


def _counts(addr):
    return C.cast(C.c_void_p(addr), C.POINTER(C.c_int64))


def _vit_weights(p):
    """the AnylocVitWeights of the addresses p["w.*"] and p["blocks[l].*"]"""
    blocks = (_lib.VitBlock * VIT_DEPTH)()
    for l in range(VIT_DEPTH):
        for f in VIT_BLOCK_FIELDS:
            setattr(blocks[l], f, p[f"blocks[{l}].{f}"])
    return _lib.VitWeightsStruct(p["w.patch_w_hi"], p["w.patch_w_lo"], p["w.patch_b"], p["w.cls_token"], blocks, 1.0,
                                 p["w.register_tokens"])     # the struct keeps `blocks` alive


def _vit_taps(p):
    return (_lib.VitTap * 2)(*[_lib.VitTap(l, f, p[f"taps[{i}].out"]) for i, (l, f) in enumerate(VIT_TAPS)])


def _attention_varlen(lib, p, fmt):
    # no shape of this entry runs nothing, so the other qkv pointer is kept below 16 bytes: each call stops at the
    # qkv check (ANYLOC_ERR_UNSUPPORTED), which follows the argument checks
    hi, lo = p["qkv_hi"], p["qkv_lo"]
    if lo != P:
        hi = P + 8
    else:
        lo = P + 8
    return lib.anyloc_attention_varlen(hi, lo, 2, (C.c_int32 * 2)(0, 70), (C.c_int32 * 2)(70, 50), 384, 6,
                                       p["o_hi"], p["o_lo"], fmt, None)


# Each entry's call at a shape that does no device work even without the alignment checks: nothing to do (B, R, N,
# n_q, n_rows, rows = 0: -> OK), or, where even an empty call would launch or copy something (the k-means, the index
# headers, the prepared blob, the residual descriptors), a workspace or blob of 0 bytes (-> ANYLOC_ERR_WORKSPACE, the
# refusal that follows the pointer checks).  p[name] is the address handed for that pointer; fmt the attention
# entries' format.
def _calls(lib, fmt=0):
    ib = lib.anyloc_index_bytes(4, D_, 1)
    sb = lib.anyloc_index_split_bytes(4, D_)
    return {
        "anyloc_vlad_assign": (OK, lambda p: lib.anyloc_vlad_assign(
            p["feats"], p["centers"], 0, D_, K_, 0, p["labels"], p["ws"], 1 << 20, None)),
        "anyloc_vlad_assign_multi": (OK, lambda p: lib.anyloc_vlad_assign_multi(
            p["feats"], 0, D_, 2, _vp(p["centers[0]"], p["centers[1]"]), (C.c_int * 2)(K_, 3), 0, p["labels"],
            p["ws"], 1 << 20, None)),
        "anyloc_vlad_prepare": (WS, lambda p: lib.anyloc_vlad_prepare(p["centers"], D_, K_, 0, p["prepared"], 0, None)),
        "anyloc_vlad_generate": (OK, lambda p: lib.anyloc_vlad_generate(
            p["feats"], p["n_valid"], p["centers"], 0, 9, D_, K_, 0, 1, 1, p["vlad"], p["labels"], p["ws"],
            1 << 20, None)),
        "anyloc_vlad_generate_prepared": (OK, lambda p: lib.anyloc_vlad_generate_prepared(
            p["feats"], p["n_valid"], p["centers"], p["prepared"], 1 << 20, 0, 9, D_, K_, 0, 1, 1, p["vlad"],
            p["labels"], p["ws"], 1 << 20, None)),
        "anyloc_vlad_generate_sorted": (OK, lambda p: lib.anyloc_vlad_generate_sorted(
            p["feats"], p["n_valid"], p["centers"], p["prepared"], 1 << 20, 0, 9, D_, K_, 0, 1, 1, p["vlad"],
            p["labels"], p["ws"], 1 << 20, None)),
        "anyloc_vlad_generate_soft": (OK, lambda p: lib.anyloc_vlad_generate_soft(
            p["feats"], p["n_valid"], p["centers"], 0, 9, D_, K_, C.c_float(0.1), 1, 1, p["vlad"], p["assign"],
            p["ws"], 1 << 20, None)),
        "anyloc_vlad_generate_varlen": (OK, lambda p: lib.anyloc_vlad_generate_varlen(
            p["feats"], 9, p["row0"], p["len"], 0, p["centers"], p["prepared"], 1 << 20, D_, K_, 0, 1, 1, p["vlad"],
            p["labels"], p["ws"], 1 << 20, None)),
        "anyloc_vlad_generate_soft_varlen": (OK, lambda p: lib.anyloc_vlad_generate_soft_varlen(
            p["feats"], 9, p["row0"], p["len"], 0, p["centers"], D_, K_, C.c_float(0.1), 1, 1, p["vlad"],
            p["assign"], p["ws"], 1 << 20, None)),
        "anyloc_vlad_residuals": (OK, lambda p: lib.anyloc_vlad_residuals(
            p["feats"], p["centers"], 0, D_, K_, 1, p["out"], None)),
        # hard (labels) unless the case is the soft weights' pointer
        "anyloc_vlad_from_residuals": (WS, lambda p: lib.anyloc_vlad_from_residuals(
            p["resid"], None if p["assign"] != P else p["labels"], p["assign"] if p["assign"] != P else None, 9, D_,
            K_, 1, p["vlad"], p["ws"], 0, None)),
        "anyloc_kmeans_update": (WS, lambda p: lib.anyloc_kmeans_update(
            p["x"], p["labels"], p["old_centers"], 9, D_, K_, p["new_centers"], p["err_out"], p["ws"], 0, None)),
        "anyloc_kmeans_update_tiled": (WS, lambda p: lib.anyloc_kmeans_update_tiled(
            p["x"], p["labels"], p["old_centers"], 9, D_, K_, 2, p["new_centers"], p["err_out"], p["ws"], 0, None)),
        "anyloc_kmeans_accumulate_round": (WS, lambda p: lib.anyloc_kmeans_accumulate_round(
            p["x"], p["labels"], 9, 9, 9, D_, K_, 0, p["ws"], 0, None)),
        "anyloc_kmeans_accumulate_round_tiled": (WS, lambda p: lib.anyloc_kmeans_accumulate_round_tiled(
            p["x"], p["labels"], 9, 9, 9, D_, K_, 2, 0, p["ws"], 0, None)),
        "anyloc_kmeans_accumulate_round_multi": (WS, lambda p: lib.anyloc_kmeans_accumulate_round_multi(
            p["x"], 2, _vp(p["labels[0]"], p["labels[1]"]), (C.c_int * 2)(K_, 3), 9, 9, 9, D_, 0,
            _vp(p["ws[0]"], p["ws[1]"]), (C.c_size_t * 2)(0, 0), None)),
        "anyloc_kmeans_finalize": (WS, lambda p: lib.anyloc_kmeans_finalize(
            p["old_centers"], 9, D_, K_, p["new_centers"], p["err_out"], p["ws"], 0, None)),
        "anyloc_index_init": (WS, lambda p: lib.anyloc_index_init(p["index"], 0, 4, D_, 1, None)),
        "anyloc_index_add": (OK, lambda p: lib.anyloc_index_add(p["index"], ib, 4, 0, p["rows"], 0, D_, 1, None)),
        "anyloc_index_copy": (WS, lambda p: lib.anyloc_index_copy(p["dst"], 0, 4, p["src"], ib, 4, 2, D_, 1, None)),
        "anyloc_index_search": (OK, lambda p: lib.anyloc_index_search(
            p["index"], ib, 4, 4, p["qu"], 0, D_, 2, 0, 1, p["dist"], p["idx"], p["ws"], 1 << 20, None)),
        "anyloc_index_search_continue": (OK, lambda p: lib.anyloc_index_search_continue(
            p["index"], ib, 4, 0, 4, 0, 4, p["qu"], 0, D_, 2, 0, 1, p["dist"], p["idx"], p["ws"], 1 << 20, None)),
        "anyloc_index_split_init": (WS, lambda p: lib.anyloc_index_split_init(p["index"], 0, 4, D_, None)),
        "anyloc_index_split_copy": (WS, lambda p: lib.anyloc_index_split_copy(
            p["dst"], 0, 4, p["src"], sb, 4, 2, D_, None)),
        "anyloc_index_split_add": (WS, lambda p: lib.anyloc_index_split_add(
            p["index"], 0, 4, p["lo"], 0, p["rows"], 0, D_, None)),
        "anyloc_index_split_piece": (WS, lambda p: lib.anyloc_index_split_piece(
            p["dst"], 0, 4, p["index"], sb, 4, p["lo"], 0, 2, D_, None)),
        "anyloc_index_split_search": (OK, lambda p: lib.anyloc_index_split_search(
            p["index"], sb, 4, 4, p["qu"], 0, D_, 2, p["ws"], 1 << 20, _counts(p["counts"]), None)),
        "anyloc_index_split_rescore": (WS, lambda p: lib.anyloc_index_split_rescore(
            p["index"], 0, 4, p["lo"], 4, 32, D_, 2, p["ws"], 1 << 20, 0, p["stage"], 1 << 20, p["dist"], p["idx"],
            None)),
        "anyloc_topk": (OK, lambda p: lib.anyloc_topk(
            p["db"], p["qu"], 4, 0, D_, 2, 0, 1, p["dist"], p["idx"], p["ws"], 1 << 20, None)),
        "anyloc_pca_colsum": (OK, lambda p: lib.anyloc_pca_colsum(p["x"], 7, 0, 0, p["sum"], p["ws"], 0, None)),
        "anyloc_pca_accumulate": (OK, lambda p: lib.anyloc_pca_accumulate(
            _lib.PCA["vt"], p["x"], 7, 0, 0, p["mu"], p["u"], 3, 0, p["out"], 5, None)),
        "anyloc_pca_mirror": (OK, lambda p: lib.anyloc_pca_mirror(p["a"], 0, 3, None)),
        "anyloc_pool": (OK, lambda p: lib.anyloc_pool(p["feats"], p["n_valid"], 0, 9, 36, AVG, C.c_float(3.0), 0,
                                                      p["out"], None)),
        "anyloc_pool_varlen": (OK, lambda p: lib.anyloc_pool_varlen(
            p["feats"], 9, p["row0"], p["len"], 0, 36, AVG, C.c_float(3.0), 0, p["out"], None)),
        "anyloc_vlad_label_multi": (OK, lambda p: lib.anyloc_vlad_label_multi(
            p["feats"], p["n_valid"], 9, 0, None, D_, 2, _vp(p["centers[0]"], p["centers[1]"]),
            _vp(p["prepared[0]"], p["prepared[1]"]), (C.c_size_t * 2)(1 << 20, 1 << 20), (C.c_int * 2)(K_, 3), 0,
            p["labels"], p["inv_norm"], p["ws"], 1 << 20, None)),
        "anyloc_vlad_soft_assign_multi": (OK, lambda p: lib.anyloc_vlad_soft_assign_multi(
            p["feats"], p["n_valid"], 9, 0, D_, 2, _vp(p["centers[0]"], p["centers[1]"]), (C.c_int * 2)(K_, 3),
            (C.c_float * 2)(0.1, 0.2), _vp(p["assign[0]"], p["assign[1]"]), p["inv_norm"], p["ws"], 1 << 20, None)),
        # hard (labels) unless the case is the soft weights' pointer
        "anyloc_vlad_accumulate": (OK, lambda p: lib.anyloc_vlad_accumulate(
            p["feats"], p["n_valid"], None if p["assign"] != P else p["labels"],
            p["assign"] if p["assign"] != P else None, p["inv_norm"], p["centers"], 0, 9, D_, K_, 1, 1, p["vlad"],
            p["ws"], 1 << 20, None)),
        "anyloc_vlad_accumulate_varlen": (OK, lambda p: lib.anyloc_vlad_accumulate_varlen(
            p["feats"], 9, p["row0"], p["len"], 0, None if p["assign"] != P else p["labels"],
            p["assign"] if p["assign"] != P else None, p["inv_norm"], p["centers"], D_, K_, 1, 1, p["vlad"], p["ws"],
            1 << 20, None)),
        "anyloc_attention": (OK, lambda p: lib.anyloc_attention(
            p["qkv_hi"], p["qkv_lo"], 0, 64, 384, 6, p["o_hi"], p["o_lo"], fmt, 0, None)),
        "anyloc_attention_varlen": (UNS, lambda p: _attention_varlen(lib, p, fmt)),
        # the ViT entries: a 0-byte workspace, refused after the pointers (the forward itself always launches)
        "anyloc_vit_extract": (WS, lambda p: lib.anyloc_vit_extract(
            C.byref(VIT_CFG), C.byref(_vit_weights(p)), p["img"], 1, 28, 42, p["pos_embed"], 1, 2, 0, 1, p["out"],
            p["ws"], 0, 0, None)),
        "anyloc_vit_extract_taps": (WS, lambda p: lib.anyloc_vit_extract_taps(
            C.byref(VIT_CFG), C.byref(_vit_weights(p)), p["img"], 1, 28, 42, p["pos_embed"], _vit_taps(p), 2, 0, 1,
            p["ws"], 0, 0, None)),
        "anyloc_vit_extract_varlen": (WS, lambda p: lib.anyloc_vit_extract_varlen(
            C.byref(VIT_CFG), C.byref(_vit_weights(p)), 2, _vp(p["img[0]"], p["img[1]"]), VIT_HW,
            _vp(p["pos_embed[0]"], p["pos_embed[1]"]), 1, 2, 0, 1, p["out"], p["ws"], 0, 0, None)),
        "anyloc_vit_extract_taps_varlen": (WS, lambda p: lib.anyloc_vit_extract_taps_varlen(
            C.byref(VIT_CFG), C.byref(_vit_weights(p)), 2, _vp(p["img[0]"], p["img[1]"]), VIT_HW,
            _vp(p["pos_embed[0]"], p["pos_embed[1]"]), _vit_taps(p), 2, 0, 1, p["ws"], 0, 0, None)),
    }


def below(a):
    """the offsets past an `a`-aligned address that are not `a`-aligned, of those a caller is likely to hand over"""
    return {4: (1, 2), 8: (1, 2, 4), 16: (1, 2, 4, 8, 12)}[a]


CASES = [(e, n) for e, ptrs in ALIGN.items() for n in ptrs]
_HOST = C.c_int64 * 8                           # split_search writes counts[0..1] on the host: a real array


def refuses_below_alignment(lib, entry, name, fmt=0):
    expect, call = _calls(lib, fmt)[entry]
    host = _HOST()
    base = C.addressof(host) if name == "counts" else P
    ptrs = {n: (C.addressof(host) if n == "counts" else P) for n in ALIGN[entry]}
    a = ALIGN[entry][name]
    for off in below(a):
        rc = call(dict(ptrs, **{name: base + off}))
        if (entry, name, fmt) in BELOW:
            assert rc == BELOW[entry, name, fmt], (entry, name, fmt, off, rc, _lib.last_error())
            continue
        assert rc == ARG, (entry, name, off, rc, _lib.last_error())
        assert f"{name} must be {a}-byte aligned" in _lib.last_error(), (entry, name, off, _lib.last_error())
    for off in (a, 2 * a, 3 * a):
        assert call(dict(ptrs, **{name: base + off})) == expect, (entry, name, off, _lib.last_error())


@pytest.mark.parametrize("entry,name", CASES, ids=[f"{e[7:]}-{n}" for e, n in CASES])
def test_entry_refuses_pointer_below_its_alignment(lib, entry, name):
    refuses_below_alignment(lib, entry, name)


ATTENTION_CASES = [(e, n) for e in ("anyloc_attention", "anyloc_attention_varlen") for n in ALIGN[e]]


@pytest.mark.parametrize("entry,name", ATTENTION_CASES, ids=[f"{e[7:]}-{n}" for e, n in ATTENTION_CASES])
def test_bf16pair_attention_refuses_pointer_below_its_alignment(lib, entry, name):
    refuses_below_alignment(lib, entry, name, X3)


def _header():
    import os
    return open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                             "anyloc_b200.h")).read()


# arguments the library reads on the CPU (host arrays, sizes, the stream), of every entry and of one entry
HOST_ARGS = {"K", "ws_bytes", "stream", "cfg", "hw", "route_rows", "prepared_bytes", "soft_temp"}
HOST_ARGS_OF = {"anyloc_attention_varlen": {"row0", "len"}}


def _argument_of(name):
    """the prototype argument a table name goes through: centers[1] -> centers, w.patch_b / blocks[1].ln2_w -> w_host,
    taps[1].out -> taps_host"""
    if name.startswith(("w.", "blocks[")):
        return "w_host"
    if name.startswith("taps["):
        return "taps_host"
    return re.sub(r"\[\d+\]", "", name)


def test_table_covers_every_pointer_argument_of_the_entries(lib):
    # every `int anyloc_*(` prototype of the header that takes a pointer is in the table, with each of its device
    # pointers, or exempt with a reason; a new entry with neither fails here
    protos = {m.group(1): m.group(2) for m in re.finditer(r"^int (anyloc_\w+)\(([^)]*)\)", _header(), re.M)}
    assert set(ALIGN) <= set(protos) and set(EXEMPT) <= set(protos), (set(ALIGN) | set(EXEMPT)) - set(protos)
    assert not set(ALIGN) & set(EXEMPT)
    for entry, args in protos.items():
        names = {re.sub(r"\W", "", a.split("*")[-1]) for a in args.split(",") if "*" in a}
        if not names:
            continue
        assert entry in ALIGN or entry in EXEMPT, f"{entry} takes pointers {sorted(names)} but has no row in ALIGN"
        if entry in ALIGN:
            covered = {_argument_of(n) for n in ALIGN[entry]}
            assert names - HOST_ARGS - HOST_ARGS_OF.get(entry, set()) == covered, (entry, names, covered)
    for entry, (reason, test) in EXEMPT.items():
        assert reason and test.startswith("test_"), entry


def _struct_pointers(src, struct):
    body = re.search(r"typedef struct \{([^}]*)\} " + struct + ";", src).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return {n for decl in body.split(";") for n in re.findall(r"\*\s*(\w+)", decl)}


def test_vit_rows_cover_every_pointer_field_of_the_vit_structs():
    # a pointer field added to AnylocVitBlock, AnylocVitWeights or AnylocVitTap needs its rows in every ViT entry, for
    # every block and tap
    src = _header()
    block, weights, tap = (_struct_pointers(src, s) for s in ("AnylocVitBlock", "AnylocVitWeights", "AnylocVitTap"))
    assert set(VIT_BLOCK_FIELDS) == block, block ^ set(VIT_BLOCK_FIELDS)
    assert "blocks" in weights and tap == {"out"}
    for entry in (e for e in ALIGN if e.startswith("anyloc_vit_extract")):
        row = ALIGN[entry]
        assert {f"w.{f}" for f in weights - {"blocks"}} <= set(row), entry
        assert {f"blocks[{l}].{f}" for l in range(VIT_DEPTH) for f in block} <= set(row), entry
        outs = {n for n in row if n.endswith("out")}
        assert outs == ({f"taps[{i}].{f}" for i in range(2) for f in tap} if "taps" in entry else {"out"}), entry
