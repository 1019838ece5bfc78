"""Shared helpers for the parity tests (the oracle is the checker, never the thing under test)."""
import ast
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_cases(fname):
    z = np.load(os.path.join(GOLDEN, fname), allow_pickle=False)
    cases = {}
    for key in z.files:
        if "/" in key:
            name, field = key.split("/", 1)
            cases.setdefault(name, {})[field] = z[key]
        else:
            cases.setdefault("", {})[key] = z[key]
    return cases


def case_kwargs(case):
    return ast.literal_eval(str(case["kw"])) if "kw" in case else {}


def rel_inf(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def split_tf32(L, x):
    """(hi, lo) tf32 pair of the fp32 tensor x through anyloc_split_tf32 (hi + lo == x exactly)."""
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    L.check(L.load().anyloc_split_tf32(L.ptr(x), L.ptr(hi), L.ptr(lo), x.numel(), L.stream_ptr()), "split")
    return hi, lo


def split_f16(L, x, scale):
    """(hi, lo) fp16 pair of scale*x through anyloc_split_f16."""
    import ctypes as C
    hi, lo = torch.empty_like(x, dtype=torch.float16), torch.empty_like(x, dtype=torch.float16)
    L.check(L.load().anyloc_split_f16(L.ptr(x), L.ptr(hi), L.ptr(lo), x.numel(), C.c_float(scale), L.stream_ptr()),
            "split_f16")
    return hi, lo


def dptr(t, offset_elems=0):
    """raw device pointer of tensor t's storage (plus an element offset); None -> NULL.  Unlike _lib.ptr it accepts
    buffers that are handed to the library with an explicit leading dimension."""
    import ctypes as C
    if t is None:
        return C.c_void_p(0)
    assert t.is_cuda and t.is_contiguous()
    return C.c_void_p(t.data_ptr() + offset_elems * t.element_size())


def gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, *, pair="tf32", alpha=1.0, epi="bias", bias=None, gamma=None,
            resid=None, out, out_lo=None, ldo, lda=None, ldb=None, engine="tc3", out_off=0, out_dtype=None):
    """anyloc_gemm_nt on raw buffers (lda/ldb default to K); returns the C ABI's return code.  out, out_lo and resid
    are buffers whose element `out_off` is the output's (0, 0), with leading dimension ldo.  out_dtype defaults to the
    input format (e4m3 inputs write bf16: out_dtype="bf16")."""
    import ctypes as C
    return L.load().anyloc_gemm_nt(
        dptr(a_hi), dptr(a_lo), K if lda is None else lda, dptr(b_hi), dptr(b_lo), K if ldb is None else ldb, M, N, K,
        L.PAIR[pair], C.c_float(alpha), L.EPI[epi], dptr(bias), dptr(gamma), dptr(resid, out_off),
        dptr(out, out_off), dptr(out_lo, out_off), ldo, L.PAIR[out_dtype or pair], L.ENGINE[engine], L.stream_ptr())


def gemm(L, a, b, epi="bias", bias=None, gamma=None, resid=None, engine="simt", pair="tf32"):
    """C = a @ b.T through the (hi,lo) pair format `pair` (3-term split); SPLIT epilogues return the reconstructed
    value.  LS_RESID runs in place (resid copied into out), as the ViT uses it."""
    M, K = a.shape
    N = b.shape[0]
    if pair == "tf32":
        (a_hi, a_lo), (b_hi, b_lo), alpha = split_tf32(L, a), split_tf32(L, b), 1.0
    else:
        s_b = 2.0 ** int(torch.floor(torch.log2(16384.0 / b.abs().max())).item())
        (a_hi, a_lo), (b_hi, b_lo) = split_f16(L, a, L.ACT_SCALE), split_f16(L, b, s_b)
        alpha = 1.0 / (L.ACT_SCALE * s_b)
    n_out = N // 2 if epi == "swiglu_split" else N
    is_split = "split" in epi
    odt = torch.float16 if (is_split and pair == "f16") else torch.float32
    out = torch.empty(M, n_out, device="cuda", dtype=odt)
    out_lo = torch.empty(M, n_out, device="cuda", dtype=odt) if is_split else None
    if epi == "ls_resid":
        out.copy_(resid)
        resid = out
    L.check(gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, pair=pair, alpha=alpha, epi=epi, bias=bias, gamma=gamma,
                    resid=resid, out=out, out_lo=out_lo, ldo=n_out, engine=engine), "gemm_nt")
    if not is_split:
        return out
    rec = out.double() + out_lo.double()
    return rec / L.ACT_SCALE if pair == "f16" else rec


def make_vlad(u, K, centers, **kw):
    """product VLAD object with a given vocabulary (what `fit` from a c_centers.pt cache yields)."""
    v = u.VLAD(K, **kw)
    v.kmeans = u._KMeans(K, mode=v.mode)
    v.kmeans.centroids = torch.as_tensor(centers)
    v.c_centers = torch.as_tensor(centers)
    v.desc_dim = centers.shape[1]
    return v
