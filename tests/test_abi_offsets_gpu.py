"""Every VLAD, k-means, retrieval, PCA, pooling and attention entry point at the pointer offsets its alignment table
accepts (tests/test_abi_alignment_cpu.py ALIGN) but that torch allocations never produce: +16 and +48 bytes where 16 is
required, +8 where 8 is, +4 and +12 where 4 is (PCA's x also with an odd leading dimension).  Each buffer sits inside a
NaN frame.  Each call must give, bit for bit, what the same call on 256-byte aligned buffers gives, with the same
number of launches (the same route: tensor-core or FFMA assignment, accumulate3 / accumulate2 / sorted, the tiled
k-means, the coarse or exact retrieval, the attention kernel), and leave every frame intact.  No pointer below its
alignment is ever passed here; the refusals are test_abi_alignment_cpu.py's.  One shape of the VLAD and of the
retrieval family is also held to the fp64 bounds of test_vlad_engine_gpu.py / test_retrieval_engine_gpu.py at an
offset.  The split index (host lo array) is left to test_retrieval_split_gpu.py's aligned buffers, the ViT entries to
test_abi_vit_offsets_gpu.py."""
import ctypes as C

import pytest
import torch

from tests.test_abi_alignment_cpu import ALIGN

pytestmark = pytest.mark.gpu

NAN32 = 0x7FC0DEAD
FRAME = 256


def accepted(a):
    return {16: (16, 48), 8: (8,), 4: (4, 12)}[a]


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


class Buf:
    """`t`'s bytes (a tensor) or `t` bytes of NaN (an int) at `off` bytes past a 256-byte boundary, inside a NaN
    frame of at least 256 bytes on each side"""

    def __init__(self, t, off):
        self.n = t if isinstance(t, int) else t.numel() * t.element_size()
        self.off = off
        self.buf = torch.full(((2 * FRAME + off + self.n + 3) // 4,), NAN32, dtype=torch.int32, device="cuda")
        assert self.buf.data_ptr() % 256 == 0
        if not isinstance(t, int):
            self.region().copy_(t.contiguous().reshape(-1).view(torch.uint8))
        self.ptr = C.c_void_p(self.buf.data_ptr() + FRAME + off)

    def region(self):
        return self.buf.view(torch.uint8)[FRAME + self.off:FRAME + self.off + self.n]

    def read(self, dtype=torch.uint8):
        return self.region().clone().view(dtype)

    def frame_intact(self):
        b, ref = self.buf.view(torch.uint8), torch.full_like(self.buf, NAN32).view(torch.uint8)
        lo, hi = FRAME + self.off, FRAME + self.off + self.n
        return torch.equal(b[:lo], ref[:lo]) and torch.equal(b[hi:], ref[hi:])


def g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rnd(*s, seed=0):
    return torch.randn(*s, device="cuda", generator=g(seed))


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def i64(v):
    return torch.tensor(v, dtype=torch.int64, device="cuda")


def nb(lib, name, *a):
    return int(getattr(lib, name)(*a))


# ------------------------------------------------------------------------------------------------------------------
# Per entry: shapes on both sides of the route switches, and for each shape the buffers (tensor: an input, int: the
# bytes of an output or workspace; None: a pointer this shape does not take), the call, and the outputs compared.
def vlad_inputs(R, D, K, seed=0):
    x = rnd(R, D, seed=seed)
    c = 0.5 * torch.nn.functional.normalize(rnd(K, D, seed=seed + 1), dim=1)
    return x, c


def prepared(L, c, D, K):
    lib = L.load()
    blob = torch.empty(nb(lib, "anyloc_vlad_prepared_bytes", D, K), dtype=torch.uint8, device="cuda")
    L.check(lib.anyloc_vlad_prepare(L.ptr(c), D, K, 0, L.ptr(blob), blob.numel(), L.stream_ptr()), "prepare")
    return blob


def spec(L, entry, shape):
    lib, st = L.load(), L.stream_ptr()
    if entry == "anyloc_vlad_assign":
        R, D, K = shape
        x, c = vlad_inputs(R, D, K)
        bufs = dict(feats=x, centers=c, labels=R * 4, ws=nb(lib, "anyloc_vlad_workspace_bytes", 1, R, D, K))
        return bufs, ["labels"], lambda p, n: lib.anyloc_vlad_assign(p["feats"], p["centers"], R, D, K, 0, p["labels"],
                                                                     p["ws"], n["ws"], st)
    if entry == "anyloc_vlad_assign_multi":
        R, D = shape
        Ks = (C.c_int * 2)(16, 8)
        x, c0 = vlad_inputs(R, D, 16)
        c1 = vlad_inputs(8, D, 8, seed=5)[1]
        bufs = {"feats": x, "centers[0]": c0, "centers[1]": c1, "labels": 2 * R * 4,
                "ws": nb(lib, "anyloc_vlad_assign_multi_workspace_bytes", R, D, 2, Ks)}
        return bufs, ["labels"], lambda p, n: lib.anyloc_vlad_assign_multi(
            p["feats"], R, D, 2, (C.c_void_p * 2)(p["centers[0]"].value, p["centers[1]"].value), Ks, 0, p["labels"],
            p["ws"], n["ws"], st)
    if entry == "anyloc_vlad_prepare":
        D, K = shape
        c = vlad_inputs(1, D, K)[1]
        bufs = dict(centers=c, prepared=nb(lib, "anyloc_vlad_prepared_bytes", D, K))
        return bufs, ["prepared"], lambda p, n: lib.anyloc_vlad_prepare(p["centers"], D, K, 0, p["prepared"],
                                                                        n["prepared"], st)
    if entry in ("anyloc_vlad_generate", "anyloc_vlad_generate_prepared", "anyloc_vlad_generate_sorted"):
        B, N, D, K = shape
        x, c = vlad_inputs(B * N, D, K)
        sorted_ = entry.endswith("sorted")
        ws = nb(lib, "anyloc_vlad_sorted_workspace_bytes" if sorted_ else "anyloc_vlad_workspace_bytes", B, N, D, K)
        bufs = dict(feats=x, n_valid=i32([N - 7 * b for b in range(B)]), centers=c, vlad=B * K * D * 4,
                    labels=B * N * 4, ws=ws, prepared=None if entry == "anyloc_vlad_generate" else prepared(L, c, D, K))
        if entry == "anyloc_vlad_generate":
            call = lambda p, n: lib.anyloc_vlad_generate(p["feats"], p["n_valid"], p["centers"], B, N, D, K, 0, 1, 1,
                                                         p["vlad"], p["labels"], p["ws"], n["ws"], st)
        else:
            fn = getattr(lib, entry)
            call = lambda p, n: fn(p["feats"], p["n_valid"], p["centers"], p["prepared"], n["prepared"], B, N, D, K,
                                   0, 1, 1, p["vlad"], p["labels"], p["ws"], n["ws"], st)
        return bufs, ["vlad", "labels"], call
    if entry == "anyloc_vlad_generate_soft":
        B, N, D, K = shape
        x, c = vlad_inputs(B * N, D, K)
        bufs = dict(feats=x, n_valid=i32([N - 5 * b for b in range(B)]), centers=c, vlad=B * K * D * 4,
                    assign=B * N * K * 4, ws=nb(lib, "anyloc_vlad_workspace_bytes", B, N, D, K))
        return bufs, ["vlad", "assign"], lambda p, n: lib.anyloc_vlad_generate_soft(
            p["feats"], p["n_valid"], p["centers"], B, N, D, K, C.c_float(30.0), 1, 1, p["vlad"], p["assign"],
            p["ws"], n["ws"], st)
    if entry in ("anyloc_vlad_generate_varlen", "anyloc_vlad_generate_soft_varlen"):
        D, K, lens = shape
        B, R = len(lens), sum(lens) + 20
        row0, r = [], 10
        for ln in lens:
            row0.append(r)
            r += ln
        x, c = vlad_inputs(R, D, K)
        if entry.endswith("soft_varlen"):
            bufs = dict(feats=x, row0=i64(row0), len=i32(lens), centers=c, vlad=B * K * D * 4, assign=R * K * 4,
                        ws=nb(lib, "anyloc_vlad_soft_varlen_workspace_bytes", R, B, D, K))
            return bufs, ["vlad", "assign"], lambda p, n: lib.anyloc_vlad_generate_soft_varlen(
                p["feats"], R, p["row0"], p["len"], B, p["centers"], D, K, C.c_float(30.0), 1, 1, p["vlad"],
                p["assign"], p["ws"], n["ws"], st)
        bufs = dict(feats=x, row0=i64(row0), len=i32(lens), centers=c, prepared=prepared(L, c, D, K),
                    vlad=B * K * D * 4, labels=R * 4,
                    ws=nb(lib, "anyloc_vlad_varlen_workspace_bytes", R, B, max(lens), D, K))
        return bufs, ["vlad", "labels"], lambda p, n: lib.anyloc_vlad_generate_varlen(
            p["feats"], R, p["row0"], p["len"], B, p["centers"], p["prepared"], n["prepared"], D, K, 0, 1, 1,
            p["vlad"], p["labels"], p["ws"], n["ws"], st)
    if entry == "anyloc_vlad_residuals":
        N, D, K = shape
        x, c = vlad_inputs(N, D, K)
        bufs = dict(feats=x, centers=c, out=N * K * D * 4)
        return bufs, ["out"], lambda p, n: lib.anyloc_vlad_residuals(p["feats"], p["centers"], N, D, K, 1, p["out"], st)
    if entry == "anyloc_vlad_from_residuals":
        N, D, K, soft = shape
        resid = rnd(N, K, D)
        bufs = dict(resid=resid, labels=None if soft else (torch.arange(N, device="cuda") % K).int(),
                    assign=torch.softmax(rnd(N, K, seed=3), 1) if soft else None, vlad=K * D * 4,
                    ws=nb(lib, "anyloc_vlad_from_residuals_workspace_bytes", D, K))
        return bufs, ["vlad"], lambda p, n: lib.anyloc_vlad_from_residuals(
            p["resid"], p["labels"], p["assign"], N, D, K, 1, p["vlad"], p["ws"], n["ws"], st)
    if entry.startswith("anyloc_kmeans"):
        R, D, K = shape
        x, c = vlad_inputs(R, D, K)
        lab = torch.randint(0, K, (R,), device="cuda", generator=g(9)).int()
        wsb = nb(lib, "anyloc_kmeans_round_workspace_bytes", R, D, K)
        part = C.c_int(0), C.c_int64(0)
        L.check(lib.anyloc_kmeans_partition(R, D, C.byref(part[0]), C.byref(part[1])), "partition")
        rows_per = part[1].value
        tiled = "tiled" in entry
        if entry in ("anyloc_kmeans_update", "anyloc_kmeans_update_tiled"):
            bufs = dict(x=x, labels=lab, old_centers=c, new_centers=K * D * 4, err_out=4, ws=wsb)
            if tiled:
                call = lambda p, n: lib.anyloc_kmeans_update_tiled(p["x"], p["labels"], p["old_centers"], R, D, K, 0,
                                                                   p["new_centers"], p["err_out"], p["ws"], n["ws"], st)
            else:
                call = lambda p, n: lib.anyloc_kmeans_update(p["x"], p["labels"], p["old_centers"], R, D, K,
                                                             p["new_centers"], p["err_out"], p["ws"], n["ws"], st)
            return bufs, ["new_centers", "err_out"], call
        if entry in ("anyloc_kmeans_accumulate_round", "anyloc_kmeans_accumulate_round_tiled"):
            bufs = dict(x=x, labels=lab, ws=wsb)
            if tiled:
                call = lambda p, n: lib.anyloc_kmeans_accumulate_round_tiled(p["x"], p["labels"], R, R, rows_per, D, K,
                                                                             0, 0, p["ws"], n["ws"], st)
            else:
                call = lambda p, n: lib.anyloc_kmeans_accumulate_round(p["x"], p["labels"], R, R, rows_per, D, K, 0,
                                                                       p["ws"], n["ws"], st)
            return bufs, ["ws"], call
        if entry == "anyloc_kmeans_finalize":
            ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
            L.check(lib.anyloc_kmeans_accumulate_round(L.ptr(x), L.ptr(lab), R, R, rows_per, D, K, 0, L.ptr(ws), wsb,
                                                       st), "round")
            bufs = dict(old_centers=c, new_centers=K * D * 4, err_out=4, ws=ws)
            return bufs, ["new_centers", "err_out"], lambda p, n: lib.anyloc_kmeans_finalize(
                p["old_centers"], R, D, K, p["new_centers"], p["err_out"], p["ws"], n["ws"], st)
        if entry == "anyloc_kmeans_accumulate_round_multi":
            Ks = (C.c_int * 2)(K, 5)
            w1 = nb(lib, "anyloc_kmeans_round_workspace_bytes", R, D, 5)
            bufs = {"x": x, "labels[0]": lab, "labels[1]": (lab % 5).int(), "ws[0]": wsb, "ws[1]": w1}
            return bufs, ["ws[0]", "ws[1]"], lambda p, n: lib.anyloc_kmeans_accumulate_round_multi(
                p["x"], 2, (C.c_void_p * 2)(p["labels[0]"].value, p["labels[1]"].value), Ks, R, R, rows_per, D, 0,
                (C.c_void_p * 2)(p["ws[0]"].value, p["ws[1]"].value), (C.c_size_t * 2)(n["ws[0]"], n["ws[1]"]), st)
    if entry.startswith("anyloc_index") or entry == "anyloc_topk":
        n_db, n_q, Dv, k, metric, norm = shape
        db, qu = rnd(n_db, Dv, seed=1), rnd(n_q, Dv, seed=2)
        ib = nb(lib, "anyloc_index_bytes", n_db, Dv, norm)
        wsb = nb(lib, "anyloc_index_search_workspace_bytes", n_db, n_q, Dv, norm)
        if entry == "anyloc_topk":
            bufs = dict(db=db, qu=qu, dist=n_q * k * 4, idx=n_q * k * 8,
                        ws=nb(lib, "anyloc_topk_workspace_bytes", n_db, n_q, Dv, k))
            return bufs, ["dist", "idx"], lambda p, n: lib.anyloc_topk(p["db"], p["qu"], n_db, n_q, Dv, k, metric,
                                                                       norm, p["dist"], p["idx"], p["ws"], n["ws"], st)
        blank = torch.zeros(ib, dtype=torch.uint8, device="cuda")
        L.check(lib.anyloc_index_init(L.ptr(blank), ib, n_db, Dv, norm, st), "init")
        full = blank.clone()
        L.check(lib.anyloc_index_add(L.ptr(full), ib, n_db, 0, L.ptr(db), n_db, Dv, norm, st), "add")
        if entry == "anyloc_index_init":
            return dict(index=ib), ["index"], lambda p, n: lib.anyloc_index_init(p["index"], ib, n_db, Dv, norm, st)
        if entry == "anyloc_index_add":
            return dict(index=blank, rows=db), ["index"], lambda p, n: lib.anyloc_index_add(
                p["index"], ib, n_db, 0, p["rows"], n_db, Dv, norm, st)
        if entry == "anyloc_index_copy":
            return dict(dst=blank, src=full), ["dst"], lambda p, n: lib.anyloc_index_copy(
                p["dst"], ib, n_db, p["src"], ib, n_db, n_db, Dv, norm, st)
        if entry == "anyloc_index_search":
            bufs = dict(index=full, qu=qu, dist=n_q * k * 4, idx=n_q * k * 8, ws=wsb)
            return bufs, ["dist", "idx"], lambda p, n: lib.anyloc_index_search(
                p["index"], ib, n_db, n_db, p["qu"], n_q, Dv, k, metric, norm, p["dist"], p["idx"], p["ws"], n["ws"],
                st)
        if entry == "anyloc_index_search_continue":
            half = n_db // 2
            w2 = nb(lib, "anyloc_index_search_workspace_bytes", n_db - half, n_q, Dv, norm)
            bufs = dict(index=full, qu=qu, dist=torch.full((n_q, k), -float("inf"), device="cuda"),
                        idx=torch.full((n_q, k), -1, dtype=torch.int64, device="cuda"), ws=w2)
            return bufs, ["dist", "idx"], lambda p, n: lib.anyloc_index_search_continue(
                p["index"], ib, n_db, half, n_db - half, half, n_db, p["qu"], n_q, Dv, k, metric, norm, p["dist"],
                p["idx"], p["ws"], n["ws"], st)
    if entry.startswith("anyloc_pca"):
        rows, cols, ld = shape
        x = rnd(rows, ld, seed=4)
        if entry == "anyloc_pca_colsum":
            bufs = dict(x=x, sum=torch.zeros(cols, dtype=torch.float64, device="cuda"),
                        ws=nb(lib, "anyloc_pca_colsum_workspace_bytes", rows, cols))
            return bufs, ["sum"], lambda p, n: lib.anyloc_pca_colsum(p["x"], ld, rows, cols, p["sum"], p["ws"],
                                                                     n["ws"], st)
        if entry == "anyloc_pca_accumulate":
            k = 5
            bufs = dict(x=x, mu=rnd(cols, seed=5).double(), u=rnd(rows, k, seed=6).double(),
                        out=torch.zeros(k, cols, dtype=torch.float64, device="cuda"))
            return bufs, ["out"], lambda p, n: lib.anyloc_pca_accumulate(
                2, p["x"], ld, rows, cols, p["mu"], p["u"], k, k, p["out"], cols, st)
        if entry == "anyloc_pca_mirror":
            return dict(a=rnd(cols, ld, seed=7).double()), ["a"], lambda p, n: lib.anyloc_pca_mirror(
                p["a"], cols, ld, st)
    if entry == "anyloc_pool":
        B, N, D = shape
        bufs = dict(feats=rnd(B, N, D), n_valid=i32([N - 3 * b for b in range(B)]), out=B * D * 4)
        return bufs, ["out"], lambda p, n: lib.anyloc_pool(p["feats"], p["n_valid"], B, N, D, 2, C.c_float(3.0), 0,
                                                           p["out"], st)
    if entry == "anyloc_pool_varlen":
        D, lens = shape
        row0, r = [], 3
        for ln in lens:
            row0.append(r)
            r += ln
        R, B = r + 2, len(lens)
        bufs = dict(feats=rnd(R, D), row0=i64(row0), len=i32(lens), out=B * D * 4)
        return bufs, ["out"], lambda p, n: lib.anyloc_pool_varlen(p["feats"], R, p["row0"], p["len"], B, D, 2,
                                                                  C.c_float(3.0), 0, p["out"], st)
    if entry in ("anyloc_vlad_label_multi", "anyloc_vlad_soft_assign_multi"):
        R, N, D = shape
        Ks = (C.c_int * 2)(16, 8)
        x, c0 = vlad_inputs(R, D, 16)
        c1 = vlad_inputs(8, D, 8, seed=5)[1]
        bufs = {"feats": x, "n_valid": i32([N - 5 * b for b in range(R // N)]), "centers[0]": c0, "centers[1]": c1,
                "inv_norm": R * 4}

        def vp(p, *names):
            return (C.c_void_p * len(names))(*[p[k].value for k in names])
        if entry == "anyloc_vlad_label_multi":
            bufs.update({"prepared[0]": prepared(L, c0, D, 16), "prepared[1]": prepared(L, c1, D, 8),
                         "labels": 2 * R * 4, "ws": nb(lib, "anyloc_vlad_label_multi_workspace_bytes", R, D, 2, Ks)})
            return bufs, ["labels", "inv_norm"], lambda p, n: lib.anyloc_vlad_label_multi(
                p["feats"], p["n_valid"], N, R, None, D, 2, vp(p, "centers[0]", "centers[1]"),
                vp(p, "prepared[0]", "prepared[1]"), (C.c_size_t * 2)(n["prepared[0]"], n["prepared[1]"]), Ks, 0,
                p["labels"], p["inv_norm"], p["ws"], n["ws"], st)
        bufs.update({"assign[0]": R * 16 * 4, "assign[1]": R * 8 * 4,
                     "ws": nb(lib, "anyloc_vlad_soft_assign_multi_workspace_bytes", D, 2, Ks)})
        return bufs, ["assign[0]", "assign[1]", "inv_norm"], lambda p, n: lib.anyloc_vlad_soft_assign_multi(
            p["feats"], p["n_valid"], N, R, D, 2, vp(p, "centers[0]", "centers[1]"), Ks, (C.c_float * 2)(30.0, 10.0),
            vp(p, "assign[0]", "assign[1]"), p["inv_norm"], p["ws"], n["ws"], st)
    if entry in ("anyloc_vlad_accumulate", "anyloc_vlad_accumulate_varlen"):
        # given per-row labels (some -1) or soft weights and 1/|x|: every accumulation route of the generate calls
        if entry == "anyloc_vlad_accumulate":
            B, N, D, K, soft = shape
            R = B * N
        else:
            D, K, lens, soft = shape
            B, R, N = len(lens), sum(lens) + 20, max(lens)
        x, c = vlad_inputs(R, D, K)
        lab = torch.randint(0, K, (R,), device="cuda", generator=g(9)).int()
        lab[::7] = -1
        bufs = dict(feats=x, labels=None if soft else lab, assign=torch.softmax(rnd(R, K, seed=3), 1) if soft else None,
                    inv_norm=1.0 / x.norm(dim=1), centers=c, vlad=B * K * D * 4,
                    ws=nb(lib, "anyloc_vlad_accumulate_workspace_bytes", B, N, D, K, int(soft)))
        if entry == "anyloc_vlad_accumulate":
            bufs["n_valid"] = i32([N - 7 * b for b in range(B)])
            return bufs, ["vlad"], lambda p, n: lib.anyloc_vlad_accumulate(
                p["feats"], p["n_valid"], p["labels"], p["assign"], p["inv_norm"], p["centers"], B, N, D, K, 1, 1,
                p["vlad"], p["ws"], n["ws"], st)
        row0, r = [], 10
        for ln in lens:
            row0.append(r)
            r += ln
        bufs.update(row0=i64(row0), len=i32(lens))
        return bufs, ["vlad"], lambda p, n: lib.anyloc_vlad_accumulate_varlen(
            p["feats"], R, p["row0"], p["len"], B, p["labels"], p["assign"], p["inv_norm"], p["centers"], D, K, 1, 1,
            p["vlad"], p["ws"], n["ws"], st)
    if entry in ("anyloc_attention", "anyloc_attention_varlen"):
        # fmt: ANYLOC_PAIR_TF32 (fp32 pairs), _F16 (anyloc_attention: tf32 pairs in, fp16 pairs out; _varlen: fp16
        # pairs of 8 x both ways), _BF16 / _F16X1 (one 2-byte array each way), _BF16X3 (bf16 pairs both ways)
        D, heads = 384, 6
        if entry == "anyloc_attention":
            B, T, fmt, engine = shape
            rows = B * T
        else:
            (fmt,) = shape
            row0, lens = (C.c_int32 * 2)(90, 0), (C.c_int32 * 2)(50, 70)     # out of order, rows 70..89 unused
            rows = 150
        x = 0.5 * rnd(rows, 3 * D, seed=6)
        if fmt in (2, 4):
            qkv = dict(qkv_hi=(x if fmt == 2 else 8 * x).to(torch.bfloat16 if fmt == 2 else torch.float16),
                       qkv_lo=None)
        elif fmt == 1 and entry == "anyloc_attention_varlen":
            hi = (8 * x).half()
            qkv = dict(qkv_hi=hi, qkv_lo=(8 * x - hi.float()).half())
        elif fmt == 5:
            hi = x.bfloat16()
            qkv = dict(qkv_hi=hi, qkv_lo=(x - hi.float()).bfloat16())
        else:
            qkv = dict(qkv_hi=x, qkv_lo=1e-4 * rnd(rows, 3 * D, seed=7))
        osz = rows * D * (4 if fmt == 0 else 2)
        bufs = dict(qkv, o_hi=osz, o_lo=osz if fmt in (0, 1, 5) else None)
        outs = [o for o in ("o_hi", "o_lo") if bufs[o] is not None]
        if entry == "anyloc_attention":
            return bufs, outs, lambda p, n: lib.anyloc_attention(p["qkv_hi"], p["qkv_lo"], B, T, D, heads, p["o_hi"],
                                                                 p["o_lo"], fmt, engine, st)
        return bufs, outs, lambda p, n: lib.anyloc_attention_varlen(p["qkv_hi"], p["qkv_lo"], 2, row0, lens, D, heads,
                                                                    p["o_hi"], p["o_lo"], fmt, st)
    raise KeyError(entry)


IDX_EXACT, IDX_COARSE, IDX_L2 = (500, 20, 256, 5, 0, 1), (2048, 40, 256, 5, 0, 1), (300, 12, 100, 4, 1, 0)
SHAPES = {
    # the tensor-core and FFMA assignments: R 255 / 256, D 2048 / 2052
    "anyloc_vlad_assign": [(255, 256, 16), (256, 256, 16), (300, 2048, 8), (300, 2052, 8)],
    "anyloc_vlad_assign_multi": [(255, 128), (256, 128)],
    "anyloc_vlad_prepare": [(256, 16)],
    # accumulate3, accumulate2 (acc3's shared memory over 100 KB), and the sorted route (K = 500)
    "anyloc_vlad_generate": [(2, 300, 256, 16), (1, 5000, 128, 64)],
    "anyloc_vlad_generate_prepared": [(2, 300, 256, 16), (1, 5000, 128, 64)],
    "anyloc_vlad_generate_sorted": [(1, 300, 64, 500)],
    "anyloc_vlad_generate_soft": [(2, 100, 128, 16)],
    "anyloc_vlad_generate_varlen": [(256, 16, (150, 0, 120)), (64, 500, (200, 90))],
    "anyloc_vlad_generate_soft_varlen": [(128, 16, (60, 40))],
    "anyloc_vlad_residuals": [(50, 128, 8)],
    "anyloc_vlad_from_residuals": [(40, 128, 8, False), (40, 128, 8, True)],
    "anyloc_kmeans_update": [(1000, 128, 16)],
    # the untiled limit: K 436 / 437
    "anyloc_kmeans_update_tiled": [(600, 128, 436), (600, 128, 437)],
    "anyloc_kmeans_accumulate_round": [(1000, 130, 16)],
    "anyloc_kmeans_accumulate_round_tiled": [(600, 128, 437)],
    "anyloc_kmeans_accumulate_round_multi": [(1000, 128, 16)],
    "anyloc_kmeans_finalize": [(1000, 128, 16)],
    "anyloc_index_init": [IDX_EXACT],
    "anyloc_index_add": [IDX_EXACT, IDX_L2],
    "anyloc_index_copy": [IDX_EXACT],
    # the exact and coarse retrieval routes
    "anyloc_index_search": [IDX_EXACT, IDX_COARSE, IDX_L2],
    "anyloc_index_search_continue": [IDX_EXACT, IDX_COARSE],
    "anyloc_topk": [IDX_EXACT, IDX_COARSE, IDX_L2],
    # odd leading dimensions
    "anyloc_pca_colsum": [(300, 70, 71)],
    "anyloc_pca_accumulate": [(300, 70, 73)],
    "anyloc_pca_mirror": [(0, 70, 73)],
    "anyloc_pool": [(2, 9, 36)],
    "anyloc_pool_varlen": [(36, (9, 0, 5))],
    # the coarse (R >= 256) and FFMA assignments
    "anyloc_vlad_label_multi": [(255, 85, 128), (256, 128, 128)],
    "anyloc_vlad_soft_assign_multi": [(200, 100, 128)],
    # accumulate3, accumulate2, sorted and soft
    "anyloc_vlad_accumulate": [(2, 300, 256, 16, False), (1, 5000, 128, 64, False), (1, 300, 64, 500, False),
                               (2, 100, 128, 16, True)],
    "anyloc_vlad_accumulate_varlen": [(256, 16, (150, 0, 120), False), (64, 500, (200, 90), False),
                                      (128, 16, (60, 40), True)],
    # the tensor-core, SIMT, fp16-pair, bf16, fp16 and bf16-pair kernels (ANYLOC_GEMM_AUTO = 0, _SIMT = 1)
    "anyloc_attention": [(2, 70, 0, 0), (2, 70, 0, 1), (2, 70, 1, 0), (2, 70, 2, 0), (2, 70, 4, 0), (2, 70, 5, 0)],
    "anyloc_attention_varlen": [(0,), (1,), (2,), (4,), (5,)],
}
CASES = [(e, i) for e in SHAPES for i in range(len(SHAPES[e]))]


def run(L, bufs, outs, call, offsets):
    """the call with each buffer at its offset -> (rc, launches, {output: bytes}, frames intact)"""
    placed = {k: (Buf(v, offsets.get(k, 0)) if v is not None else None) for k, v in bufs.items()}
    p = {k: (b.ptr if b is not None else C.c_void_p(0)) for k, b in placed.items()}
    n = {k: b.n for k, b in placed.items() if b is not None}
    torch.cuda.synchronize()
    n0 = L.launch_count()
    rc = call(p, n)
    launches = L.launch_count() - n0
    torch.cuda.synchronize()
    return (rc, launches, {o: placed[o].read() for o in outs},
            all(b.frame_intact() for b in placed.values() if b is not None), placed)


@pytest.mark.parametrize("entry,i", CASES, ids=[f"{e[7:]}-{i}" for e, i in CASES])
def test_offsets_match_aligned_call(L, entry, i):
    assert set(SHAPES) <= set(ALIGN)
    bufs, outs, call = spec(L, entry, SHAPES[entry][i])
    rc, launches, ref, intact, _ = run(L, bufs, outs, call, {})
    assert rc == 0 and intact, (rc, L.last_error())
    for name, a in ALIGN[entry].items():
        if bufs.get(name) is None:
            continue
        for off in accepted(a):
            rc2, l2, got, intact2, _ = run(L, bufs, outs, call, {name: off})
            assert rc2 == 0, (name, off, L.last_error())
            assert l2 == launches, (name, off, l2, launches)
            assert intact2, (name, off, "a frame was overwritten")
            for o in outs:
                assert torch.equal(got[o], ref[o]), (name, off, o)


def test_vlad_offsets_hold_the_fp64_bound(L):
    from tests import test_vlad_engine_gpu as V
    B, N, D, K = 2, 300, 256, 16
    x, c = V.make_inputs("clustered", B, N, D, K, seed=11)
    bufs, outs, call = spec(L, "anyloc_vlad_generate", (B, N, D, K))
    bufs.update(feats=x.reshape(B * N, D), centers=c, n_valid=None)
    rc, _, got, intact, _ = run(L, bufs, outs, call, dict(feats=48, centers=16, vlad=48, labels=12, ws=16))
    assert rc == 0 and intact, L.last_error()
    v, lab = got["vlad"].view(torch.float32).view(B, K, D), got["labels"].view(torch.int32).view(B, N)
    V.check_labels(x, c, lab, V.COS, "offsets")
    v64, bound, _ = V.hard_reference(x, c, lab)
    assert V.ratio(v, v64, bound) <= 1.0


def test_retrieval_offsets_hold_the_fp64_bound(L):
    from tests import test_retrieval_engine_gpu as T
    n_db, n_q, Dv, k, metric, norm = IDX_COARSE
    db, qu = T.make_rows("clustered", n_db, n_q, Dv, seed=3)
    bufs, outs, call = spec(L, "anyloc_topk", IDX_COARSE)
    bufs.update(db=db, qu=qu)
    rc, _, got, intact, _ = run(L, bufs, outs, call, dict(db=16, qu=48, dist=12, idx=8, ws=48))
    assert rc == 0 and intact, L.last_error()
    ref, B = T.reference(db, qu, norm, metric)
    r, _ = T.check(got["dist"].view(torch.float32).view(n_q, k), got["idx"].view(torch.int64).view(n_q, k), ref, B,
                   metric)
    assert r <= 1.0
