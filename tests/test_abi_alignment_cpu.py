"""Alignment checks of the pooling and pre-processing entry points, without a GPU.  anyloc_pool reads the features and
writes the output with float4 accesses, anyloc_preprocess_u8 stores pairs of columns as float2 when Wc is even, and
every pre-processing kernel stores fp32 elements, so a pointer those accesses would fault on is refused before any
CUDA call: the placeholder device pointers here are never touched.  Calls with nothing to do (B = 0, n = 0) and
aligned pointers still return OK without launching."""
import ctypes as C

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
# The alignment each VLAD, k-means, retrieval and PCA entry requires of each pointer it takes: the widest access any of
# its routes makes through that pointer (float4 / uint4 / TMA: 16, int64 / fp64: 8, fp32 / int32: 4).  A workspace or
# blob inherits the base's alignment in every buffer carved from it, so it needs what its strictest buffer needs.  Where
# the pointer reaches the tensor-core GEMM it is 16 even when the fallback kernel would accept less, so that an accepted
# buffer never changes the route.  test_abi_offsets_gpu.py hands every entry real buffers at the offsets this table
# accepts.  DESIGN.md section 2 lists the kernels' 64- and 128-bit accesses that each entry traces back to.
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
}

OK, WS = 0, _lib.ERR["workspace"]
D_, K_ = 8, 4                   # every call below: 8 columns, 4 clusters


def _vp(*xs):
    return (C.c_void_p * len(xs))(*xs)


def _counts(addr):
    return C.cast(C.c_void_p(addr), C.POINTER(C.c_int64))


# Each entry's call at a shape that does no device work even without the alignment checks: nothing to do (B, R, N,
# n_q, n_rows, rows = 0: -> OK), or, where even an empty call would launch or copy something (the k-means, the index
# headers, the prepared blob, the residual descriptors), a workspace or blob of 0 bytes (-> ANYLOC_ERR_WORKSPACE, the
# refusal that follows the pointer checks).  p[name] is the address handed for that pointer.
def _calls(lib):
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
    }


def below(a):
    """the offsets past an `a`-aligned address that are not `a`-aligned, of those a caller is likely to hand over"""
    return {4: (1, 2), 8: (1, 2, 4), 16: (1, 2, 4, 8, 12)}[a]


CASES = [(e, n) for e, ptrs in ALIGN.items() for n in ptrs]
_HOST = C.c_int64 * 8                           # split_search writes counts[0..1] on the host: a real array


@pytest.mark.parametrize("entry,name", CASES, ids=[f"{e[7:]}-{n}" for e, n in CASES])
def test_entry_refuses_pointer_below_its_alignment(lib, entry, name):
    expect, call = _calls(lib)[entry]
    host = _HOST()
    base = C.addressof(host) if name == "counts" else P
    ptrs = {n: (C.addressof(host) if n == "counts" else P) for n in ALIGN[entry]}
    a = ALIGN[entry][name]
    for off in below(a):
        rc = call(dict(ptrs, **{name: base + off}))
        assert rc == ARG, (entry, name, off, rc, _lib.last_error())
        assert f"{name} must be {a}-byte aligned" in _lib.last_error(), (entry, name, off, _lib.last_error())
    for off in (a, 2 * a, 3 * a):
        assert call(dict(ptrs, **{name: base + off})) == expect, (entry, name, off, _lib.last_error())


def test_table_covers_every_pointer_argument_of_the_entries(lib):
    # the header's prototype of each entry names every pointer argument; each must be in the table (or be a host array
    # the library reads on the CPU, or the stream)
    import os
    import re
    host_only = {"K", "ws_bytes", "stream"}
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "anyloc_b200.h")).read()
    for entry, ptrs in ALIGN.items():
        m = re.search(r"^int " + entry + r"\(([^)]*)\)", src, re.M)
        assert m, entry
        names = set()
        for arg in m.group(1).split(","):
            arg = arg.strip()
            if "*" in arg:
                names.add(re.sub(r"\W", "", arg.split("*")[-1]))
        covered = {re.sub(r"\[\d+\]", "", n) for n in ptrs}
        assert names - host_only == covered, (entry, names - host_only, covered)
