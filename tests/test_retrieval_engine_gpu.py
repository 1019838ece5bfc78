"""Every retrieval route of anyloc_index_search, the prepared index and the C ABI around them, checked element by element
against fp64 on raw buffers.

Let q^, y^_j be the query and database rows normalised in fp64 from the fp32 inputs (the raw rows when normalize = 0),
S64 = q^ . y^_j, L64 = |q^ - y^_j|^2 and P_qj = sum_i |q^_i y^_ji|.  Every returned distance must satisfy, element by
element, with u = 2^-24 and the sqrt-style constant of test_gemm_engine_gpu.py,

    IP:  |d - S64| <= 16 u (sqrt(Dv) + c_n) P_qj + sigma
    L2:  |d - L64| <= 16 u (sqrt(Dv) + c_n) (|q^|^2 + 2 P_qj + |y^_j|^2) + 2 sigma

    c_n = Dv / 4096 + 3 (normalize = 1; 0 for raw rows),   sigma = 2 sqrt(Dv) 2^-25 / 4096 (fp16 pairs; 0 for tf32).

Derivation from the kernels' arithmetic:
  * c_n, the two row normalisations.  |x|^2 is an fp32 sum of Dv squares: Dv/256 terms per thread in the grid-stride
    kernel (Dv/1024 .. Dv/4096 per thread in the register forms), a 5-level warp tree, then 8 or 32 warp totals in
    order: a relative error of at most (Dv/256 + 41) u.  The sqrt halves it and adds u, the division adds u, so each
    normalised row is off by a common factor of at most (Dv/512 + 22.5) u plus one rounding per element; both sides
    give (Dv/256 + 45) u |S| <= (Dv/256 + 45) u P.  Three more u P cover the pair formats below, so
    16 c_n = Dv/256 + 48.
  * The fp16 pairs hold 4096 y to 2^-22 relative (hi: 11 significant bits, lo: the next 11), 0.25 u P per side.  The
    tf32 pairs hold y exactly (hi + lo == y); the tensor cores truncate lo to tf32 (2^-21 of the element) and the
    3-term product drops lo.lo (2^-22): at most 20 u per product, which 16 u sqrt(Dv) covers for Dv >= 2 even when
    the truncation biases every term the same way (the all-positive family).
  * The rescore (coarse route) is an fma chain of exact products (hi + lo is exact in fp32 on both sides): Dv/128
    terms per accumulator, 2 + 5 tree levels, Dv/4096 slices added in order, then the exact 1/4096^2.  That is
    gamma_{Dv/128 + Dv/4096 + 7} P, inside 16 u sqrt(Dv) P in the sqrt form.  The GEMM engines (3-term fallback,
    exact tensor-core and SIMT routes) are covered by the same 16 u sqrt(Dv) (test_gemm_engine_gpu.py).
  * L2 forms (qq - 2 v) + dd: qq and dd are fp32 sums of Dv squares of the normalised rows (the c_n and sqrt(Dv)
    terms times |q^|^2 and |y^|^2), 2 v carries twice the IP error, and the two additions round once each (covered by
    the 16 u factor on the same magnitudes).
  * sigma, the fp16 subnormal slack: elements of |4096 y| < 2^-14 are rounded to the 2^-24 grid, hi and lo each by at
    most 2^-25; over a dot product with a unit row that is at most sqrt(Dv) 2^-24 / 4096 per side, i.e.
    2 sqrt(Dv) 2^-25 / 4096.  No family needed a larger constant.

Indices are checked conditioned on that bound rather than on a fixed gap: (a) the output is strictly ordered by
(dist desc, idx asc) for IP, (dist asc, idx asc) for L2, no index repeats, -1 / -inf (+inf for L2) exactly at ranks
>= the number of finite rows; (b) every dist is within the bound of the fp64 value of its row; (c) no row outside the
list beats a returned one by more than their two bounds; (d) where the fp64 gaps exceed the bounds the indices equal
the fp64 stable top-k; (e) bit-identical rows come out lowest index first.

Non-finite rows.  A database row with a NaN or an Inf is never returned, and the other rows' answers are those of the
database without it; a query with a NaN or an Inf gets -1 / -inf (+inf for L2) at every rank, on every route.  That
is this project's definition (faiss' behaviour there is a parity-unpinned boundary, DESIGN §2), the one the exact
route has always had.

The route that ran is identified for every call, never assumed: by the anyloc_launch_count() delta, by the
per-category launch groups of anyloc_profile_read (gemm_tc vs gemm_simt) and, for the 3-term fallback, by the
overflow flag in the caller's workspace.  Which path of topk_select2_kernel ran (shared-memory list or k ordered
sweeps) is derived from the scores it read, left in the workspace.  Three wrong references must violate the bound on
the same output.  The worst bound ratio per (route, family) is printed at the end."""
import ctypes as C

import pytest
import torch

from tests.util import dptr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ACC = 16
S_RET = 4096.0                              # kRetrievalScale
CAND_MAX, SEL_CAP, SEL_THREADS = 256, 4096, 1024
IP, L2 = 0, 1
OK, ERR_ARG, ERR_WS = 0, -1, -3
LEAD = 16                                   # canary elements before and after every output
NAN32 = 0x7FC0DEAD                          # a quiet-NaN pattern no kernel writes
CANARY64 = 0x0BADC0DE0BADC0DE
WORST = {}                                  # (route, family) -> worst ratio seen
SEEN = set()                                # routes and select2 paths identified


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    yield _lib
    if WORST:
        print("\n[worst |d - ref| / bound per route and family]")
        for (route, fam), r in sorted(WORST.items()):
            print(f"  {route:<22} {fam:<28} {r:.3f}")
    print(f"[routes and select paths identified] {sorted(SEEN)}")


@pytest.fixture(scope="module")
def sms(L):
    n = C.c_int(0)
    assert L.load().anyloc_device_info(C.byref(n), None) >= 90
    return n.value


def note(route, fam, r):
    WORST[(route, fam)] = max(WORST.get((route, fam), 0.0), r)


# ------------------------------------------------------------------------------------------------------ route mirror
# anyloc_index_search (topk.cu) and gemm_dispatch (api.cu):
#   route       taken when                                                               launches  GEMM group
#   coarse      IP, fp16-pair index (normalize, Dv % 8 == 0), k <= 64, n_db >= 1024,         6       gemm_tc
#               n_q >= 32; "fallback" when a candidate list overflowed (flag in the workspace)
#   exact_tc    anything else with n_q >= 32                                                    3       gemm_tc
#   exact_simt  anything else with n_q < 32                                                     3       gemm_simt
def uses_f16(Dv, normalize):
    return bool(normalize) and Dv % 8 == 0


def route_of(n_db, n_q, Dv, k, metric, normalize):
    """(route, launches, {profile category: launch groups})"""
    if n_q == 0:
        return "none", 0, {"gemm_tc": 0, "gemm_simt": 0, "topk": 0}
    if uses_f16(Dv, normalize) and metric == IP and k <= 64 and n_db >= 1024 and n_q >= 32:
        return "coarse", 6, {"gemm_tc": 1, "gemm_simt": 0, "topk": 3}    # the gated GEMM records nothing
    if n_q >= 32:
        return "exact_tc", 3, {"gemm_tc": 1, "gemm_simt": 0, "topk": 2}
    return "exact_simt", 3, {"gemm_tc": 0, "gemm_simt": 1, "topk": 2}


# ------------------------------------------------------------------------------------ carves of the caller's buffers
def a256(n):
    return (n + 255) // 256 * 256


def carve(parts):
    off, out = 0, {}
    for name, nbytes in parts:
        out[name] = off
        off += a256(nbytes)
    out["_total"] = off
    return out


def search_carve(n_db, n_q, Dv, normalize):
    """anyloc_index_search's workspace: qu_hi, qu_lo, qq, dnq, scores, cand, cand_n, flags (256 B aligned each)"""
    esz = 2 if uses_f16(Dv, normalize) else 4
    return carve([("qu_hi", n_q * Dv * esz), ("qu_lo", n_q * Dv * esz), ("qq", 4 * n_q), ("dnq", 4 * n_q),
                  ("scores", 4 * n_q * n_db), ("cand", 4 * n_q * CAND_MAX), ("cand_n", 4 * n_q), ("flags", 256)])


def index_carve(cap, Dv, normalize):
    """carve_index: hi, lo, sq, dn, header"""
    esz = 2 if uses_f16(Dv, normalize) else 4
    return carve([("hi", cap * Dv * esz), ("lo", cap * Dv * esz), ("sq", 4 * cap), ("dn", 4 * cap), ("hdr", 256)])


def view(buf, off, n, dtype):
    es = torch.empty((), dtype=dtype).element_size()
    return buf[off:off + n * es].view(dtype)


def index_sections(blob, cap, n, Dv, normalize):
    o = index_carve(cap, Dv, normalize)
    pd = torch.float16 if uses_f16(Dv, normalize) else torch.float32
    return dict(hi=view(blob, o["hi"], n * Dv, pd).view(n, Dv), lo=view(blob, o["lo"], n * Dv, pd).view(n, Dv),
                sq=view(blob, o["sq"], n, torch.float32), dn=view(blob, o["dn"], n, torch.float32),
                hdr=view(blob, o["hdr"], 1, torch.float32))


def query_sections(ws, n_db, n_q, Dv, normalize):
    o = search_carve(n_db, n_q, Dv, normalize)
    pd = torch.float16 if uses_f16(Dv, normalize) else torch.float32
    return dict(hi=view(ws, o["qu_hi"], n_q * Dv, pd).view(n_q, Dv), lo=view(ws, o["qu_lo"], n_q * Dv, pd).view(n_q, Dv),
                sq=view(ws, o["qq"], n_q, torch.float32), dn=view(ws, o["dnq"], n_q, torch.float32),
                scores=view(ws, o["scores"], n_q * n_db, torch.float32).view(n_q, n_db),
                cand=view(ws, o["cand"], n_q * CAND_MAX, torch.int32).view(n_q, CAND_MAX),
                cand_n=view(ws, o["cand_n"], n_q, torch.int32), flag=view(ws, o["flags"], 1, torch.int32))


# ------------------------------------------------------------------------------------------------------- buffers
def canary_f32(n):
    return torch.full((LEAD + n + LEAD,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def canary_i64(n):
    return torch.full((LEAD + n + LEAD,), CANARY64, dtype=torch.int64, device="cuda")


def assert_intact(buf, n, what, written=True):
    bits = buf.view(torch.int32) if buf.dtype == torch.float32 else buf
    pat = NAN32 if buf.dtype == torch.float32 else CANARY64
    outside = torch.cat([bits[:LEAD], bits[LEAD + n:]]) if written else bits
    bad = int((outside != pat).sum())
    assert bad == 0, f"{what}: {bad} canary words overwritten"


def workspace(nbytes):
    return torch.empty(int(nbytes), dtype=torch.uint8, device="cuda")


def build_index(L, db, normalize, cap=None, fill=None, offset=0):
    """an index blob of `cap` rows (default: len(db)) holding db at rows [offset, offset + len(db))"""
    n, Dv = db.shape
    cap = n + offset if cap is None else cap
    lib = L.load()
    blob = workspace(lib.anyloc_index_bytes(cap, Dv, normalize))
    if fill is not None:
        blob.fill_(fill)
    L.check(lib.anyloc_index_init(dptr(blob), blob.numel(), cap, Dv, normalize, L.stream_ptr()), "index_init")
    L.check(lib.anyloc_index_add(dptr(blob), blob.numel(), cap, offset, dptr(db), n, Dv, normalize, L.stream_ptr()),
            "index_add")
    return blob


class Result:
    pass


def search(L, blob, cap, n_db, qu, k, metric, normalize, *, ws=None, expect_rc=OK, Dv=None, tag=""):
    """one anyloc_index_search call with canaries around dist and idx; asserts the route it took"""
    lib = L.load()
    n_q = qu.shape[0]
    Dv = qu.shape[1] if Dv is None else Dv
    if ws is None:
        ws = workspace(lib.anyloc_index_search_workspace_bytes(n_db, n_q, Dv, normalize))
    dist, idx = canary_f32(n_q * k), canary_i64(n_q * k)
    torch.cuda.synchronize()
    L.profile_enable(True)
    n0 = L.launch_count()
    rc = lib.anyloc_index_search(dptr(blob), blob.numel(), cap, n_db, dptr(qu), n_q, Dv, k, metric, normalize,
                                 dptr(dist, LEAD), dptr(idx, LEAD), dptr(ws), ws.numel(), L.stream_ptr())
    launches = L.launch_count() - n0
    prof = L.profile_read()
    L.profile_enable(False)
    torch.cuda.synchronize()
    assert rc == expect_rc, (rc, L.last_error())
    ok = rc == OK and n_q > 0
    assert_intact(dist, n_q * k, "dist", written=ok)
    assert_intact(idx, n_q * k, "idx", written=ok)
    r = Result()
    r.rc, r.ws, r.launches = rc, ws, launches
    if rc != OK:
        assert launches == 0
        return r
    route, n_exp, groups = route_of(n_db, n_q, Dv, k, metric, normalize)
    got = {c: prof[c][1] for c in groups}
    assert launches == n_exp, (route, launches, n_exp)
    assert got == groups, (route, got, groups)
    r.flag = int(query_sections(ws, n_db, n_q, Dv, normalize)["flag"][0]) if route == "coarse" else 0
    r.route = "fallback" if r.flag else route
    r.dist, r.idx = dist[LEAD:LEAD + n_q * k].view(n_q, k), idx[LEAD:LEAD + n_q * k].view(n_q, k)
    SEEN.add(r.route)
    print(f"{tag} n_db={n_db} n_q={n_q} Dv={Dv} k={k} {'L2' if metric else 'IP'} norm={normalize}: route {r.route} "
          f"({launches} launches, {got})")
    return r


# ---------------------------------------------------------------------------------------------- fp64 reference
def reference(db, qu, normalize, metric, mutate=None):
    """(ref [n_q, n_db] fp64 scores (IP) or squared distances (L2), bound [n_q, n_db]); NaN where a row or query is
    not finite.  mutate: a wrong reference (see test_wrong_references)"""
    Dv = db.shape[1]
    y, q = db.double(), qu.double()
    fy, fq = torch.isfinite(y).all(1), torch.isfinite(q).all(1)
    y = torch.where(fy[:, None], y, torch.zeros((), dtype=torch.float64, device=y.device))
    q = torch.where(fq[:, None], q, torch.zeros((), dtype=torch.float64, device=q.device))
    q_raw = q
    if normalize:
        if mutate == "hi_norm":                      # the norm of the fp16 hi parts instead of the row's
            def hnorm(t):
                t = t / t.norm(dim=1, keepdim=True).clamp_min(1e-12)
                return t / ((t * S_RET).float().half().double() / S_RET).norm(dim=1, keepdim=True).clamp_min(1e-12)
            y, q = hnorm(y), hnorm(q)
        else:
            y = y / y.norm(dim=1, keepdim=True).clamp_min(1e-12)
            q = q / q.norm(dim=1, keepdim=True).clamp_min(1e-12)
    cn = Dv / 4096 + 3 if normalize else 0.0
    sig = 2 * Dv ** 0.5 * 2.0 ** -25 / S_RET if uses_f16(Dv, normalize) else 0.0
    c = C_ACC * U * (Dv ** 0.5 + cn)
    P = q.abs() @ y.abs().T
    if mutate == "drop_tail4":                       # the last 4 columns left out of the product
        S = q[:, :-4] @ y[:, :-4].T
    else:
        S = q @ y.T
    if metric == IP:
        ref, B = S, c * P + sig
    else:
        qn, yn = (q * q).sum(1), (y * y).sum(1)
        qn_used = (q_raw * q_raw).sum(1) if mutate == "raw_qq" else qn
        ref = qn_used[:, None] - 2 * S + yn[None, :]
        B = c * (qn[:, None] + 2 * P + yn[None, :]) + 2 * sig
    nan = torch.full((), float("nan"), dtype=torch.float64, device=ref.device)
    ref = torch.where(fy[None, :] & fq[:, None], ref, nan)
    return ref, B


def check(dist, idx, ref, B, metric, dup_groups=()):
    """(a)-(e) of the module docstring on one output; returns (worst ratio, fraction of ranks fixed by the bound)"""
    n_q, k = idx.shape
    n_db = ref.shape[1]
    dev = ref.device
    dist, idx = dist.to(dev), idx.to(dev)
    valid = torch.isfinite(ref)
    n_av = valid.sum(1)
    sign = 1.0 if metric == IP else -1.0
    pad = -float("inf") if metric == IP else float("inf")
    live = torch.arange(k, device=dev)[None, :] < n_av[:, None]
    # (a)
    assert bool((idx[~live] == -1).all()) and bool((dist[~live] == pad).all()), "padding is not -1 / inf"
    assert bool((idx[live] >= 0).all()) and bool((idx[live] < n_db).all()), "index out of range"
    g = idx.clamp_min(0)
    assert bool(valid.gather(1, g)[live].all()), "a non-finite row (or query) was returned"
    key = sign * dist.double()
    both = live[:, 1:]
    order = (key[:, :-1] > key[:, 1:]) | ((key[:, :-1] == key[:, 1:]) & (idx[:, :-1] < idx[:, 1:]))
    assert bool(order[both].all()), "output not strictly ordered by (dist, idx)"
    s = torch.where(live, idx, -1 - torch.arange(k, device=dev)[None, :]).sort(1).values
    assert not bool((s[:, 1:] == s[:, :-1]).any()), "an index repeats"
    # (b)
    r64, b = ref.gather(1, g), B.gather(1, g)
    err = (dist.double() - r64).abs()
    ratio = float((err / b)[live].max()) if bool(live.any()) else 0.0
    assert ratio <= 1.0, f"distance off its fp64 value by {ratio:.3g} bounds"
    # (c)
    sref = torch.where(valid, sign * ref, torch.full((), -float("inf"), dtype=torch.float64, device=dev))
    inlist = torch.zeros(n_q, n_db + 1, dtype=torch.bool, device=dev)
    inlist = inlist.scatter_(1, torch.where(live, idx, n_db), True)[:, :n_db]    # padded ranks land in a spare column
    best_out = torch.where(valid & ~inlist, sref - B, torch.full((), -float("inf"), dtype=torch.float64, device=dev))
    worst_in = torch.where(inlist, sref + B, torch.full((), float("inf"), dtype=torch.float64, device=dev))
    assert bool((best_out.max(1).values <= worst_in.min(1).values).all()), "a row outside the list beats a returned one"
    # (d)
    top = torch.sort(torch.where(valid, -sref, torch.full((), float("inf"), dtype=torch.float64, device=dev)), dim=1,
                     stable=True).indices[:, :k + 1]
    tv, tb = sref.gather(1, top), B.gather(1, top)
    kk = top.shape[1]
    ranks = torch.arange(kk, device=dev)[None, :]
    sep = torch.ones(n_q, kk, dtype=torch.bool, device=dev)
    sep[:, :-1] = (tv[:, :-1] - tv[:, 1:] > tb[:, :-1] + tb[:, 1:]) | (ranks[:, 1:] >= n_av[:, None])
    prev = torch.ones_like(sep)
    prev[:, 1:] = sep[:, :-1]
    kd = min(k, kk)
    det = (sep & prev)[:, :kd] & live[:, :kd]           # rank r is fixed when it is separated from r - 1 and r + 1
    assert bool((idx[:, :kd][det] == top[:, :kd][det]).all()), \
        "indices differ from the fp64 top-k where the gaps exceed the bounds"
    # (e)
    for grp in dup_groups:
        grp = grp.to(dev)
        for q in range(n_q):
            got = idx[q][torch.isin(idx[q], grp)]
            assert torch.equal(got, grp[:got.numel()]), f"query {q}: bit-identical rows not lowest index first"
            if got.numel() > 1:
                d = dist[q][torch.isin(idx[q], grp)]
                assert bool((d == d[0]).all()), f"query {q}: bit-identical rows with different distances"
    return ratio, float(det.sum()) / max(1, int(live.sum()))


def verify(res, db, qu, normalize, metric, fam, dup_groups=()):
    ref, B = reference(db, qu, normalize, metric)
    r, fixed = check(res.dist, res.idx, ref, B, metric, dup_groups)
    note(res.route, fam, r)
    print(f"  {fam}: worst ratio {r:.3f}, {fixed:.2f} of the ranks fixed by the bound")
    return ref, B, fixed


# ------------------------------------------------------------------------------------------------------ inputs
def make_rows(fam, n_db, n_q, Dv, seed, raw=False):
    """db [n_db, Dv], qu [n_q, Dv] on the device.  raw: row norms spread over 1e-2 .. 1e2 (normalize = 0 searches)"""
    from tests.test_coarse_bound_gpu import unit_rows
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    if fam in ("random", "positive", "spiky"):
        db, qu = unit_rows(fam, n_db, Dv, g), unit_rows(fam, n_q, Dv, g)
    elif fam == "near_dup":                            # scores near 1, L2 distances near 0
        base = unit_rows("random", 32, Dv, g)
        db, qu = unit_rows("near_dup", n_db, Dv, g, base=base), unit_rows("near_dup", n_q, Dv, g, base=base)
    elif fam == "clustered":
        centres = unit_rows("random", 8, Dv, g)
        pick = lambda n: centres[torch.randint(0, 8, (n,), device="cuda", generator=g)]
        db, qu = pick(n_db) + 0.3 * rn(n_db, Dv) / Dv ** 0.5, pick(n_q) + 0.3 * rn(n_q, Dv) / Dv ** 0.5
    else:
        raise ValueError(fam)
    if raw:
        db = db * 10.0 ** (4 * torch.rand(n_db, 1, device="cuda", generator=g) - 2)
        qu = qu * 10.0 ** (4 * torch.rand(n_q, 1, device="cuda", generator=g) - 2)
    return db.float().contiguous(), qu.float().contiguous()


def run(L, fam, n_db, n_q, Dv, k, metric, normalize, seed=0, tag=""):
    db, qu = make_rows(fam, n_db, n_q, Dv, seed, raw=not normalize)
    blob = build_index(L, db, normalize)
    res = search(L, blob, n_db, n_db, qu, k, metric, normalize, tag=tag)
    ref, B, fixed = verify(res, db, qu, normalize, metric, fam)
    return db, qu, blob, res, fixed


# ------------------------------------------------------------------------------------------- route table, thresholds
THRESHOLDS = {
    # name: (n_db, n_q, Dv, k, metric, normalize, expected route)
    "base": (1024, 32, 256, 10, IP, 1, "coarse"),
    "n_q31": (1024, 31, 256, 10, IP, 1, "exact_simt"),
    "n_db1023": (1023, 32, 256, 10, IP, 1, "exact_tc"),
    "k64": (1024, 32, 256, 64, IP, 1, "coarse"),
    "k65": (1024, 32, 256, 65, IP, 1, "exact_tc"),
    "Dv260_tf32": (1024, 32, 260, 10, IP, 1, "exact_tc"),
    "Dv260_n_q31": (1024, 31, 260, 10, IP, 1, "exact_simt"),
    "norm0": (1024, 32, 256, 10, IP, 0, "exact_tc"),
    "norm0_n_q31": (1024, 31, 256, 10, IP, 0, "exact_simt"),
    "L2": (1024, 32, 256, 10, L2, 1, "exact_tc"),
    "L2_n_q31": (1024, 31, 256, 10, L2, 1, "exact_simt"),
    "L2_norm0": (1024, 32, 260, 10, L2, 0, "exact_tc"),
    "wide_coarse": (3000, 96, 3072, 5, IP, 1, "coarse"),
    "wide_L2": (3000, 40, 3072, 5, L2, 1, "exact_tc"),
}


@pytest.mark.parametrize("name", sorted(THRESHOLDS))
def test_route_thresholds(L, name):
    n_db, n_q, Dv, k, metric, normalize, want = THRESHOLDS[name]
    assert route_of(n_db, n_q, Dv, k, metric, normalize)[0] == want
    _, _, _, res, fixed = run(L, "random", n_db, n_q, Dv, k, metric, normalize, seed=len(name), tag=name)
    assert res.route == want
    if normalize or metric == IP:        # raw L2 distances are dominated by |q|^2: most near ranks stay ambiguous
        assert fixed > 0.5, "the bound leaves most ranks of random rows ambiguous"


@pytest.mark.parametrize("fam", ["random", "positive", "spiky", "near_dup", "clustered"])
@pytest.mark.parametrize("route", ["coarse", "exact_tc", "exact_simt", "exact_tc_L2", "exact_tc_tf32"])
def test_families(L, route, fam):
    n_db, n_q, Dv, k, metric, normalize = {
        "coarse": (2048, 64, 1024, 10, IP, 1), "exact_tc": (2048, 64, 1024, 80, IP, 1),
        "exact_simt": (2048, 8, 1024, 10, IP, 1), "exact_tc_L2": (2048, 64, 1024, 10, L2, 1),
        "exact_tc_tf32": (2048, 64, 1028, 10, IP, 1)}[route]
    _, _, _, res, _ = run(L, fam, n_db, n_q, Dv, k, metric, normalize, seed=31 * len(route) + len(fam),
                          tag=f"{route}/{fam}")
    assert res.route == route.split("_L2")[0].split("_tf32")[0]


def test_flatindex_search_chunks(L):
    """FlatIndex.search with 4096 + 7 queries: the first chunk takes the coarse route, the tail of 7 the SIMT one"""
    from anyloc_b200 import utilities as u
    n_db, Dv, k = 2048, 256, 10
    db, qu = make_rows("random", n_db, 4096 + 7, Dv, seed=41)
    ix = u.FlatIndex(Dv, "cosine", True, device="cuda")
    ix.add(db)
    torch.cuda.synchronize()
    L.profile_enable(True)
    n0 = L.launch_count()
    dist, idx = ix.search(qu, k)
    launches = L.launch_count() - n0
    prof = L.profile_read()
    L.profile_enable(False)
    assert launches == route_of(n_db, 4096, Dv, k, IP, 1)[1] + route_of(n_db, 7, Dv, k, IP, 1)[1] == 9
    assert prof["gemm_tc"][1] == 1 and prof["gemm_simt"][1] == 1
    SEEN.update(("coarse", "exact_simt"))
    ref, B = reference(db, qu, 1, IP)
    r, fixed = check(dist, idx, ref, B, IP)
    note("coarse+simt (FlatIndex)", "random", r)
    assert fixed > 0.5


# ----------------------------------------------------------------------------------------- white box, coarse route
def thread_tau(key, k):
    """the k-th best of the 1024 per-thread maxima (thread t owns rows j = t mod 1024; NaN keys are never a maximum),
    -inf when fewer than k threads hold one: the tau of topk_select2_kernel and topk_candidates_kernel"""
    n_q, n = key.shape
    cols = (n + SEL_THREADS - 1) // SEL_THREADS * SEL_THREADS
    kp = torch.full((n_q, cols), float("nan"), dtype=key.dtype, device=key.device)
    kp[:, :n] = key
    kp = kp.view(n_q, -1, SEL_THREADS)
    present = ~torch.isnan(kp)
    m = torch.where(present, kp, torch.full((), -float("inf"), dtype=key.dtype, device=key.device)).max(1).values
    has = present.any(1)
    m = torch.where(has, m, torch.full((), -float("inf"), dtype=key.dtype, device=key.device))
    tau = m.sort(1, descending=True).values[:, min(k, SEL_THREADS) - 1]
    return torch.where(has.sum(1) >= k, tau, torch.full((), -float("inf"), dtype=key.dtype, device=key.device))


def coarse_whitebox(res, blob, cap, n_db, qu, k, ref):
    """the coarse scores, the candidate lists and the overflow flag the kernels left behind.  Every row whose fp64 score
    reaches the fp64 k-th best must be a candidate (|S~ - S64| <= eps_q makes S~_j >= tau - 2 eps_q for them)"""
    n_q, Dv = qu.shape
    w = query_sections(res.ws, n_db, n_q, Dv, 1)
    valid = torch.isfinite(ref)
    kth = torch.where(valid, ref, torch.full((), -float("inf"), dtype=torch.float64, device=ref.device))
    must = valid & (ref >= kth.topk(k, dim=1).values[:, -1:])
    assert bool((w["cand_n"] <= CAND_MAX).all())
    if res.flag:                      # the gated GEMM has overwritten the coarse scores: the flag must be justified
        forced = must.sum(1) > CAND_MAX
        assert bool(forced.any()), "the flag is set but no query has more than 256 guaranteed candidates"
        assert bool((w["cand_n"][forced] == 0).all())
        return
    DN = index_sections(blob, cap, n_db, Dv, 1)["hdr"][0]
    st, dq = w["scores"], w["dn"]
    eps = (dq.double() + DN.double() + dq.double() * DN.double()) * 1.001 + 3e-5
    r = float(((st.double() - ref).abs()[valid] / eps[:, None].expand_as(ref)[valid]).max())
    print(f"  coarse scores: worst |S~ - S64| / eps_q {r:.3f}")
    assert r <= 1.0
    tau = thread_tau(st, k)
    eps32 = (dq + DN + dq * DN) * 1.001 + 3.0e-5          # nvcc may contract these into FMAs: one ulp either way
    thr = tau - 2.0 * eps32
    inf = torch.full_like(thr, float("inf"))
    slack = 2 * (torch.nextafter(thr.abs(), inf) - thr.abs()) + 4 * (torch.nextafter(eps32, inf) - eps32)
    cand = st >= thr[:, None]
    either = (st - thr[:, None]).abs() <= slack[:, None]
    assert not bool(((cand | either).sum(1) > CAND_MAX).any()), "a list overflowed without setting the flag"
    for q in range(n_q):
        got = torch.zeros(n_db, dtype=torch.bool, device=st.device)
        lst = w["cand"][q, :int(w["cand_n"][q])].long()
        assert torch.unique(lst).numel() == lst.numel(), f"query {q}: a candidate repeats"
        got[lst] = True
        bad = (got != cand[q]) & ~either[q]
        assert not bool(bad.any()), f"query {q}: candidate set differs from {{S~ >= tau - 2 eps_q}} at {bad.nonzero()[:5]}"
        assert bool(got[must[q]].all()), f"query {q}: an fp64 top-k member is not a candidate"


@pytest.mark.parametrize("fam", ["random", "near_dup", "spiky", "clustered"])
def test_coarse_whitebox(L, fam):
    n_db, n_q, Dv, k = 3000, 64, 1024, 10
    db, qu = make_rows(fam, n_db, n_q, Dv, seed=7 + len(fam))
    blob = build_index(L, db, 1)
    res = search(L, blob, n_db, n_db, qu, k, IP, 1, tag=f"whitebox/{fam}")
    ref, _, _ = verify(res, db, qu, 1, IP, fam)
    coarse_whitebox(res, blob, n_db, n_db, qu, k, ref)


# ----------------------------------------------------------------------------------------- boundaries by construction
def dup_block(n_db, Dv, start, m, seed, n_q=40, noise=0.05):
    """random unit rows with rows [start, start + m) bit-identical; queries close to that row"""
    db, _ = make_rows("random", n_db, 1, Dv, seed)
    db[start:start + m] = db[start]
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    qu = (db[start][None] + noise * torch.randn(n_q, Dv, device="cuda", generator=g) / Dv ** 0.5).contiguous()
    return db.contiguous(), qu


@pytest.mark.parametrize("m", [256, 257])
def test_candidate_overflow_edge(L, m):
    """m bit-identical rows well above the others: 256 candidates fit (no flag), 257 set the flag and every query of
    the batch is answered by the 3-term fallback"""
    n_db, Dv, k, start = 2048, 256, 8, 100
    db, qu = dup_block(n_db, Dv, start, m, seed=m)
    blob = build_index(L, db, 1)
    res = search(L, blob, n_db, n_db, qu, k, IP, 1, tag=f"overflow m={m}")
    assert res.route == ("coarse" if m == 256 else "fallback")
    grp = torch.arange(start, start + m, device="cuda")
    ref, _, _ = verify(res, db, qu, 1, IP, f"dup_block{m}", dup_groups=[grp])
    assert torch.equal(res.idx, grp[:k].expand(qu.shape[0], k))
    coarse_whitebox(res, blob, n_db, n_db, qu, k, ref)
    if m == 256:
        assert bool((query_sections(res.ws, n_db, qu.shape[0], Dv, 1)["cand_n"] == 256).all())


def select_path(res, blob, n_db, qu, k, metric, normalize):
    """list / sweeps per query, from the scores topk_select2_kernel read (left in the workspace)"""
    n_q, Dv = qu.shape
    w = query_sections(res.ws, n_db, n_q, Dv, normalize)
    s = w["scores"]
    if metric == L2:
        key = -((w["sq"][:, None] - 2.0 * s) + index_sections(blob, n_db, n_db, Dv, normalize)["sq"][None, :])
    else:
        key = s
    tau = thread_tau(key, k)
    count = (key >= tau[:, None]).sum(1)
    return ["sweeps" if int(c) > SEL_CAP else "list" for c in count]


@pytest.mark.parametrize("metric", [IP, L2])
@pytest.mark.parametrize("m", [4096, 4097])
def test_select_list_and_sweeps(L, m, metric):
    """m bit-identical rows at the top: 4096 keys >= tau use the shared-memory list, 4097 the k ordered sweeps"""
    n_db, Dv, k, start = 6000, 128, 7, 1000
    db, qu = dup_block(n_db, Dv, start, m, seed=m + metric)
    blob = build_index(L, db, 1)
    res = search(L, blob, n_db, n_db, qu, k, metric, 1, tag=f"select m={m}")
    assert res.route == ("fallback" if metric == IP else "exact_tc")
    paths = select_path(res, blob, n_db, qu, k, metric, 1)
    want = "list" if m == 4096 else "sweeps"
    assert paths == [want] * qu.shape[0], paths
    SEEN.add(f"select2/{want}")
    grp = torch.arange(start, start + m, device="cuda")
    verify(res, db, qu, 1, metric, f"dup_block{m}", dup_groups=[grp])
    assert torch.equal(res.idx, grp[:k].expand(qu.shape[0], k))


@pytest.mark.parametrize("n_q", [8, 40])
def test_zero_query_sweeps(L, n_q):
    """an all-zero query over 5000 rows scores 0 everywhere: 0 .. k-1 with distance 0, through the sweeps (the coarse
    route overflows and falls back; below 32 queries the SIMT route runs)"""
    n_db, Dv, k = 5000, 256, 9
    db, qu = make_rows("random", n_db, n_q, Dv, seed=3)
    qu[0] = 0.0
    db[11] = 0.0                                          # an all-zero database row is an ordinary row of score 0
    blob = build_index(L, db, 1)
    res = search(L, blob, n_db, n_db, qu, k, IP, 1, tag="zero query")
    assert res.route == ("fallback" if n_q >= 32 else "exact_simt")
    assert select_path(res, blob, n_db, qu, k, IP, 1)[0] == "sweeps"
    SEEN.add("select2/sweeps")
    assert torch.equal(res.idx[0], torch.arange(k, device="cuda")) and bool((res.dist[0] == 0).all())
    verify(res, db, qu, 1, IP, "zero_query")


def test_k_beyond_thread_count(L):
    """k = 1100 > 1024 thread maxima: tau = -inf, so every row is a candidate and the sweeps run"""
    n_db, n_q, Dv, k = 5000, 32, 128, 1100
    db, qu = make_rows("clustered", n_db, n_q, Dv, seed=11)
    blob = build_index(L, db, 1)
    res = search(L, blob, n_db, n_db, qu, k, IP, 1, tag="k=1100")
    assert res.route == "exact_tc"
    assert set(select_path(res, blob, n_db, qu, k, IP, 1)) == {"sweeps"}
    SEEN.add("select2/sweeps")
    verify(res, db, qu, 1, IP, "clustered:k1100")


@pytest.mark.parametrize("n_q,metric", [(32, IP), (5, IP), (32, L2)])
def test_k_beyond_n_db(L, n_q, metric):
    n_db, Dv, k = 100, 64, 150
    db, qu = make_rows("random", n_db, n_q, Dv, seed=n_q)
    db[50:60] = db[50]
    blob = build_index(L, db, 1)
    res = search(L, blob, n_db, n_db, qu, k, metric, 1, tag="k>n_db")
    verify(res, db, qu, 1, metric, "k>n_db", dup_groups=[torch.arange(50, 60, device="cuda")])
    assert bool((res.idx[:, n_db:] == -1).all())


# -------------------------------------------------------------------------------------------------- non-finite rows
NONFINITE = {
    # name: (Dv, normalize, metric, n_q)
    "coarse": (256, 1, IP, 64), "simt": (256, 1, IP, 8), "L2": (256, 1, L2, 64), "tf32": (260, 1, IP, 64),
    "raw": (256, 0, IP, 64), "raw_L2": (256, 0, L2, 40),
}


@pytest.mark.parametrize("name", sorted(NONFINITE))
def test_nonfinite_rows(L, name):
    """database rows with a NaN, a +Inf and a -Inf are never returned and the other rows' answers are bitwise those of
    the database without them; queries with a NaN or an Inf get -1 / inf at every rank"""
    Dv, normalize, metric, n_q = NONFINITE[name]
    n_db, k = 2048, 10
    db, qu = make_rows("random", n_db, n_q, Dv, seed=19, raw=not normalize)
    bad = [5, 17, 1030]
    db[5, 3] = float("nan")
    db[17, 200] = float("inf")
    db[1030, 0] = -float("inf")
    qu[2, 7] = float("nan")
    qu[4, 9] = float("inf")
    blob = build_index(L, db, normalize)
    res = search(L, blob, n_db, n_db, qu, k, metric, normalize, tag=f"nonfinite/{name}")
    verify(res, db, qu, normalize, metric, f"nonfinite:{name}")
    pad = -float("inf") if metric == IP else float("inf")
    assert bool((res.idx[[2, 4]] == -1).all()) and bool((res.dist[[2, 4]] == pad).all())
    keep = torch.tensor([j for j in range(n_db) if j not in bad], device="cuda")
    clean = db[keep].contiguous()
    blob2 = build_index(L, clean, normalize)
    res2 = search(L, blob2, n_db - 3, n_db - 3, qu, k, metric, normalize, tag=f"nonfinite/{name} (rows removed)")
    assert res2.route == res.route
    mapped = torch.where(res2.idx >= 0, keep[res2.idx.clamp_min(0)], res2.idx)
    assert torch.equal(res.idx, mapped), "the non-finite rows changed the other rows' answers"
    assert torch.equal(res.dist, res2.dist), "the non-finite rows changed the other rows' distances"
    if normalize and Dv % 8 == 0:
        s = index_sections(blob, n_db, n_db, Dv, normalize)
        fin = torch.ones(n_db, dtype=torch.bool, device="cuda")
        fin[bad] = False
        assert s["hdr"].view(torch.int32)[0] == s["dn"][fin].max().view(torch.int32), "header != max finite dn"


# ------------------------------------------------------------------------------------------------ wrong references
def test_wrong_references(L):
    """the bound is tight enough to matter: on the same kernel outputs, a row norm taken from the fp16 hi parts only
    (near-duplicates, Dv = 64, coarse route), the last 4 columns left out (a planted value there, Dv = 260, tf32 pairs)
    and L2 with |q|^2 of the unnormalised query (Dv = 256) violate it"""
    cases = []
    db, qu = make_rows("near_dup", 2048, 64, 64, seed=5)
    res = search(L, build_index(L, db, 1), 2048, 2048, qu, 10, IP, 1, tag="wrong/hi_norm")
    cases.append(("hi_norm", res, db, qu, IP))
    db, qu = make_rows("random", 2048, 64, 260, seed=6)
    db[:, -4:] += 0.3
    qu[:, -4:] += 0.3
    res = search(L, build_index(L, db, 1), 2048, 2048, qu, 10, IP, 1, tag="wrong/drop_tail4")
    cases.append(("drop_tail4", res, db, qu, IP))
    db, qu = make_rows("random", 2048, 64, 256, seed=7)
    qu = (qu * 3.0).contiguous()
    res = search(L, build_index(L, db, 1), 2048, 2048, qu, 10, L2, 1, tag="wrong/raw_qq")
    cases.append(("raw_qq", res, db, qu, L2))
    for mutate, res, db, qu, metric in cases:
        ref, B = reference(db, qu, 1, metric)
        r_ok, _ = check(res.dist, res.idx, ref, B, metric)
        note(res.route, f"wrong-ref base:{mutate}", r_ok)
        wref, _ = reference(db, qu, 1, metric, mutate=mutate)
        g = res.idx.clamp_min(0)
        r = float(((res.dist.double() - wref.gather(1, g)).abs() / B.gather(1, g)).max())
        print(f"wrong reference {mutate}: worst ratio {r:.3g} (correct reference {r_ok:.3f})")
        assert r > 1.0, f"the bound does not catch the {mutate} reference ({r:.3g})"


# ------------------------------------------------------------------------------------------ normalise kernel forms
def norm_form(Dv):
    d4 = Dv // 4
    if 2048 < d4 <= 16384:
        return f"reg_nv{4 if d4 <= 4096 else 8 if d4 <= 8192 else 12 if d4 <= 12288 else 16}"
    return "grid_stride"


def rna_tf32(t):
    return ((t.view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def check_sections(s, x, normalize, what):
    """hi / lo / sq / dn / header of n rows (index or query pairs) against the fp64 normalisation of x"""
    n, Dv = x.shape
    x64 = x.double()
    fin = torch.isfinite(x64).all(1)
    y64 = x64 / x64.norm(dim=1, keepdim=True).clamp_min(1e-12) if normalize else x64
    y64 = y64[fin]
    cn = Dv / 4096 + 3 if normalize else 0.0
    hi, lo = s["hi"][fin], s["lo"][fin]
    if hi.dtype == torch.float16:
        a64 = S_RET * y64
        h, l = hi.double(), lo.double()
        assert bool(((h - a64).abs() <= (2.0 ** -11 + C_ACC * U * cn) * a64.abs() + 2.0 ** -24).all()), \
            f"{what}: hi is not 4096 y rounded to 11 significant bits"
        assert bool(((h + l - a64).abs() <= (2.0 ** -22 + C_ACC * U * cn) * a64.abs() + 2.0 ** -24).all()), \
            f"{what}: hi + lo is not 4096 y to 2^-22"
        if s.get("dn") is not None:
            ln = l.norm(dim=1) / S_RET                  # |s y - hi| / s as stored (lo = fp16(s y - hi), 2^-11)
            dn = s["dn"][fin].double()
            slack = Dv ** 0.5 * 2.0 ** -25 / S_RET
            assert bool((dn >= ln).all()), f"{what}: dn below |s y - hi| / s"
            assert bool((dn <= 1.0025 * ln + 1.001 * slack + 1e-12).all()), f"{what}: dn far above |s y - hi| / s"
        y = None
    else:
        assert bool(((hi.view(torch.int32) & 0x1FFF) == 0).all()), f"{what}: hi is not a tf32 word"
        y = hi + lo
        assert torch.equal(rna_tf32(y), hi) and torch.equal(y - hi, lo), f"{what}: (hi, lo) is not the split of hi + lo"
        if normalize:
            assert bool(((y.double() - y64).abs() <= C_ACC * U * cn * y64.abs() + 1e-30).all()), f"{what}: y != x / |x|"
        else:
            assert torch.equal(y, x[fin]), f"{what}: hi + lo != x bitwise"
    sq64 = (y64 * y64).sum(1)
    sq_err = (s["sq"][fin].double() - sq64).abs()
    assert bool((sq_err <= C_ACC * U * (Dv ** 0.5 + cn) * sq64).all()), f"{what}: |y|^2 off its bound"


FORMS = [8192, 8200, 16384, 16392, 32768, 32776, 49152, 49160, 65536, 65544, 131072,          # fp16 pairs
         8188, 8196, 16380, 16388, 32764, 32772, 49148, 49156, 65532, 65540, 131076]           # tf32 pairs


@pytest.mark.parametrize("Dv", FORMS)
def test_normalise_forms(L, sms, Dv):
    """every form of launch_normalize_rows for both pair formats, with more rows than the grid has CTAs: sections
    straight from the blob and from the search workspace, then a search within the bound"""
    form = norm_form(Dv)
    n = sms + 9 if form.startswith("reg") else 8 * sms + 17
    assert n > (sms if form.startswith("reg") else 8 * sms)
    db, qu = make_rows("random" if Dv % 3 else "positive", n, 32, Dv, seed=Dv)
    db[1] = 0.0                                           # an all-zero row
    blob = build_index(L, db, 1)
    pairs = "fp16" if uses_f16(Dv, 1) else "tf32"
    print(f"Dv={Dv}: {form}, {pairs} pairs, {n} rows")
    s = index_sections(blob, n, n, Dv, 1)
    check_sections(s, db, 1, f"index Dv={Dv}")
    if pairs == "fp16":
        assert s["hdr"].view(torch.int32)[0] == s["dn"].max().view(torch.int32), "header != max dn"
    res = search(L, blob, n, n, qu, 5, IP, 1, tag=f"form {form}/{pairs}")
    w = query_sections(res.ws, n, 32, Dv, 1)
    check_sections(dict(w, dn=w["dn"] if pairs == "fp16" else None), qu, 1, f"queries Dv={Dv}")
    verify(res, db, qu, 1, IP, f"form:{form}/{pairs}")
    SEEN.add(f"normalise/{form}/{pairs}")


def test_normalise_raw_rows(L, sms):
    """normalize = 0: tf32 pairs of the raw rows, hi + lo == x bitwise, in the grid-stride and a register form"""
    for Dv in (1024, 32768):
        n = 8 * sms + 17 if norm_form(Dv) == "grid_stride" else sms + 9
        db, qu = make_rows("random", n, 32, Dv, seed=Dv + 1, raw=True)
        blob = build_index(L, db, 0)
        check_sections(index_sections(blob, n, n, Dv, 0), db, 0, f"raw index Dv={Dv}")
        res = search(L, blob, n, n, qu, 5, IP, 0, tag=f"raw {norm_form(Dv)}")
        verify(res, db, qu, 0, IP, f"raw:{norm_form(Dv)}")


# --------------------------------------------------------------------------------------- adds and prefix searches
def test_add_at_offset_writes_only_its_rows(L):
    cap, Dv, r0, n = 3000, 256, 1000, 500
    db, _ = make_rows("random", n, 1, Dv, seed=2)
    blob = build_index(L, db, 1, cap=cap, fill=0xA5, offset=r0)
    o = index_carve(cap, Dv, 1)
    for sec, es in (("hi", 2 * Dv), ("lo", 2 * Dv), ("sq", 4), ("dn", 4)):
        part = blob[o[sec]:o[sec] + cap * es].view(cap, es)
        outside = torch.cat([part[:r0], part[r0 + n:]])
        assert bool((outside == 0xA5).all()), f"add at offset {r0} wrote outside its rows ({sec})"
        assert not bool((part[r0:r0 + n] == 0xA5).all(1).any()), f"add left a row of {sec} unwritten"
    s = index_sections(blob, cap, cap, Dv, 1)
    assert s["hdr"].view(torch.int32)[0] == s["dn"][r0:r0 + n].max().view(torch.int32)
    check_sections({key: (v[r0:r0 + n] if key != "hdr" else v) for key, v in s.items()}, db, 1, "offset add")


def flat_sections(ix, n):
    s = index_sections(ix._blob, ix.capacity, n, ix.dp, int(ix.norm_descs))
    return {key: v.clone() for key, v in s.items()}


@pytest.mark.parametrize("method,norm", [("cosine", True), ("l2", True), ("cosine", False)])
def test_index_builds_agree(L, method, norm):
    """chunked adds (growth through anyloc_index_copy), add_at out of order and reset() + re-add give the same blob
    sections and bitwise the same search results as one add"""
    from anyloc_b200 import utilities as u
    n, Dv, k = 3000, 256, 10
    db, qu = make_rows("random", n, 64, Dv, seed=13, raw=not norm)
    ix = u.FlatIndex(Dv, method, norm, capacity=n, device="cuda")
    ix.add(db)
    want, (d0, i0) = flat_sections(ix, n), ix.search(qu, k)
    builds = {}
    a = u.FlatIndex(Dv, method, norm, device="cuda")
    cuts = (0, 700, 1400, 2900, n)
    for c0, c1 in zip(cuts[:-1], cuts[1:]):
        a.add(db[c0:c1])
    builds["chunked+growth"] = a
    b = u.FlatIndex(Dv, method, norm, capacity=n, device="cuda")
    for c0 in (2000, 0, 1000):
        b.add_at(db[c0:c0 + 1000], c0)
    builds["add_at"] = b
    c = u.FlatIndex(Dv, method, norm, capacity=n, device="cuda")
    c.add(torch.flip(db, [0]) * 7.0)
    c.reset()
    c.add(db)
    builds["reset+re-add"] = c
    for name, x in builds.items():
        assert x.ntotal == n
        got = flat_sections(x, n)
        for sec in (("hi", "lo", "sq", "dn", "hdr") if norm else ("hi", "lo", "sq")):   # tf32 pairs keep no dn
            assert torch.equal(got[sec].view(torch.uint8), want[sec].view(torch.uint8)), \
                f"{name}: section {sec} differs from one add"
        d, i = x.search(qu, k)
        assert torch.equal(i, i0) and torch.equal(d, d0), f"{name}: search differs from one add"
    ref, B = reference(db, qu, int(norm), _lib_metric(method))
    r, _ = check(d0, i0, ref, B, _lib_metric(method))
    note("FlatIndex", f"builds:{method}:{int(norm)}", r)


def _lib_metric(method):
    return IP if method == "cosine" else L2


def test_prefix_search(L):
    """a search over the first n_db < capacity rows is within the bound and bitwise that of an index of those rows"""
    cap, n_db, Dv, k = 3000, 2000, 256, 10
    db, qu = make_rows("random", cap, 64, Dv, seed=17)
    big = build_index(L, db, 1)
    res = search(L, big, cap, n_db, qu, k, IP, 1, tag="prefix")
    verify(res, db[:n_db], qu, 1, IP, "prefix")
    small = build_index(L, db[:n_db].contiguous(), 1)
    res2 = search(L, small, n_db, n_db, qu, k, IP, 1, tag="prefix (own index)")
    assert torch.equal(res.idx, res2.idx) and torch.equal(res.dist, res2.dist)


# -------------------------------------------------------------------------------------------------- C ABI contract
@pytest.mark.parametrize("metric,normalize,n_q", [(IP, 1, 64), (L2, 1, 64), (IP, 0, 20), (IP, 1, 7)])
def test_anyloc_topk(L, metric, normalize, n_q):
    """the one-shot entry is bitwise FlatIndex add + search; one byte short of its workspace size is refused"""
    from anyloc_b200 import utilities as u
    lib = L.load()
    n_db, Dv, k = 2048, 256, 10
    db, qu = make_rows("random", n_db, n_q, Dv, seed=23, raw=not normalize)
    need = lib.anyloc_topk_workspace_bytes(n_db, n_q, Dv, k)
    for nbytes, rc_want in ((need - 1, ERR_WS), (need, OK)):
        ws = workspace(nbytes)
        dist, idx = canary_f32(n_q * k), canary_i64(n_q * k)
        rc = lib.anyloc_topk(dptr(db), dptr(qu), n_db, n_q, Dv, k, metric, normalize, dptr(dist, LEAD),
                             dptr(idx, LEAD), dptr(ws), ws.numel(), L.stream_ptr())
        torch.cuda.synchronize()
        assert rc == rc_want, (nbytes, rc, L.last_error())
        assert_intact(dist, n_q * k, "topk dist", written=rc == OK)
        assert_intact(idx, n_q * k, "topk idx", written=rc == OK)
    ix = u.FlatIndex(Dv, "cosine" if metric == IP else "l2", bool(normalize), capacity=n_db, device="cuda")
    ix.add(db)
    d, i = ix.search(qu, k)
    assert torch.equal(dist[LEAD:LEAD + n_q * k].view(n_q, k), d) and torch.equal(idx[LEAD:LEAD + n_q * k].view(n_q, k), i)
    ref, B = reference(db, qu, normalize, metric)
    r, _ = check(d, i, ref, B, metric)
    note("anyloc_topk", f"random:{'L2' if metric else 'IP'}:norm{normalize}:n_q{n_q}", r)


def test_refusals(L):
    """refused calls return their code and write nothing; n_q = 0 writes nothing"""
    lib = L.load()
    n_db, n_q, Dv, k = 2048, 40, 256, 10
    db, qu = make_rows("random", n_db, n_q, Dv, seed=29)
    blob = build_index(L, db, 1)
    carve_total = search_carve(n_db, n_q, Dv, 1)["_total"]
    search(L, blob, n_db, n_db, qu, k, IP, 1, ws=workspace(carve_total - 1), expect_rc=ERR_WS)
    search(L, blob, n_db, n_db, qu, k, IP, 1, ws=workspace(1024), expect_rc=ERR_WS)
    search(L, blob, n_db, n_db, qu, k, IP, 1, ws=workspace(carve_total), tag="exact carve size")
    bad = torch.zeros(n_q, 260, device="cuda")
    search(L, blob, n_db, n_db, bad, k, IP, 1, Dv=258, expect_rc=ERR_ARG)
    search(L, blob, n_db, n_db, qu, 0, IP, 1, expect_rc=ERR_ARG)
    dist, idx = canary_f32(4), canary_i64(4)
    ws = workspace(lib.anyloc_index_search_workspace_bytes(n_db, n_q, Dv, 1))
    for what, args in (("k=-1", (n_db, n_db, -1, IP)), ("n_db > capacity", (n_db, n_db + 1, k, IP)),
                       ("metric 2", (n_db, n_db, k, 2)), ("n_db = 0", (n_db, 0, k, IP))):
        cap, nd, kk, met = args
        rc = lib.anyloc_index_search(dptr(blob), blob.numel(), cap, nd, dptr(qu), n_q, Dv, kk, met, 1, dptr(dist, LEAD),
                                     dptr(idx, LEAD), dptr(ws), ws.numel(), L.stream_ptr())
        torch.cuda.synchronize()
        assert rc == ERR_ARG, (what, rc)
        assert_intact(dist, 4, what, written=False)
        assert_intact(idx, 4, what, written=False)
    n0 = L.launch_count()
    rc = lib.anyloc_index_search(dptr(blob), blob.numel(), n_db, n_db, dptr(qu), 0, Dv, k, IP, 1, dptr(dist, LEAD),
                                 dptr(idx, LEAD), dptr(ws), ws.numel(), L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == OK and L.launch_count() == n0, "n_q = 0 launched work"
    assert_intact(dist, 4, "n_q = 0", written=False)
    assert_intact(idx, 4, "n_q = 0", written=False)
    rc = lib.anyloc_index_add(dptr(blob), blob.numel(), n_db, 0, dptr(db), n_db, 258, 1, L.stream_ptr())
    assert rc == ERR_ARG


def test_bitwise_invariants(L):
    """the same search twice is bitwise identical (the atomicAdd order of the candidate lists does not leak), permuting
    the queries permutes the outputs bitwise, and the SIMT route on 31 of the queries agrees with the coarse route on
    all of them within the bound"""
    n_db, n_q, Dv, k = 3000, 64, 512, 10
    db, qu = make_rows("random", n_db, n_q, Dv, seed=31)
    db[200:230] = db[200]                                  # ties inside the candidate lists of the first 8 queries
    qu[:8] = db[200] + 0.05 * torch.randn(8, Dv, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    blob = build_index(L, db, 1)
    a = search(L, blob, n_db, n_db, qu, k, IP, 1, tag="twice (1)")
    b = search(L, blob, n_db, n_db, qu, k, IP, 1, tag="twice (2)")
    assert a.route == "coarse" and torch.equal(a.idx, b.idx) and torch.equal(a.dist, b.dist)
    perm = torch.randperm(n_q, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    p = search(L, blob, n_db, n_db, qu[perm].contiguous(), k, IP, 1, tag="permuted")
    assert p.route == "coarse" and torch.equal(p.idx, a.idx[perm]) and torch.equal(p.dist, a.dist[perm])
    s = search(L, blob, n_db, n_db, qu[:31].contiguous(), k, IP, 1, tag="first 31")
    assert s.route == "exact_simt"
    ref, B = reference(db, qu[:31], 1, IP)
    for res in (s, a):
        check(res.dist[:31], res.idx[:31], ref, B, IP, dup_groups=[torch.arange(200, 230, device="cuda")])
    same = s.idx == a.idx[:31]
    g = s.idx.clamp_min(0)
    assert bool(((s.dist.double() - a.dist[:31].double()).abs() <= 2 * B.gather(1, g))[same].all())
