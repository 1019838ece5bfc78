"""anyloc_pool (average, max, GeM) checked element by element against fp64 through the C ABI, with n_valid, every
output inside a NaN frame; and the Python entry points handed CUDA views at odd storage offsets.

The kernel: a CTA owns 128 columns of one image; 8 row groups each add rows grp, grp + 8, ... in order, then group 0
adds the other 7 groups' sums in order and divides by n = min(N, n_valid[b]).  So, with u = 2^-24 and
gamma_k = k u / (1 - k u):

  * average: |o - o64| <= gamma_{ceil(n/8)+8} sum|x| / n + u |o64|.
  * max: bit-exact against the max of the fp32 values (torch's, NaN propagating).  A NaN among the first n rows
    gives NaN; NaN or +-Inf past n_valid is never read.
  * GeM: each term x^p (|x|^p with use_abs) carries gamma_{p-1} |x|^p for integer p in [1, 16] (repeated products) and
    otherwise powf's documented maximum error of 4 ulp <= 8 u |x^p|.  The mean m then carries
    eps_m = (gamma_{ceil(n/8)+8} + k_pow u) sum|x|^p / n + u |m64| + 8 * 2^-149, the last term for powers that
    fall among fp32's subnormals (0.005^17 = 8e-40 keeps 17 significant bits, so without it an n = 1 image with
    p = 17 exceeds the relative bound 5e5-fold).  The root o = sign(m) powf(|m|, fl(1/p)):
      - when |m64| > 2 eps_m: |o - o64| <= max_{|m'| in [|m| - eps_m, |m| + eps_m]} (1/|p|) |m'|^(1/p - 1) eps_m
        + (8 + |ln|m64|| / |p|) u |o64|, the last term powf's 4 ulp and 1/p rounded to fp32 (a relative u in the
        exponent is u |ln m| / |p| in the result);
      - when |m64| <= 2 eps_m the computed mean may have either sign: |o - o64| <= 2 (|m64| + eps_m)^(1/p).
    The bound is applied with a factor 2 for second-order terms.  p in {1, 2, 3, 16, 17, 2.5, 0.5, -1} covers both
    sides of the kernel's integer-exponent switch; with use_abs off, fractional p on a negative value must give NaN
    exactly where the fp64 reference does.
  * An image with n_valid <= 0 is empty and written NaN in every mode.

Shapes: D in {4, 36, 388, 1540} (D % 128 != 0: a partial column slice), N in {1, 7, 8, 9, 1369, 5000}, B = 65 535
with tiny N D, and B = 65 536 refused without a write.  n_valid > N (clamped), 1 and 0, rows past n_valid holding NaN
and +-Inf.  Reruns are bit-identical and an image's output does not depend on the batch around it.  The worst share of
the bound per mode is printed at the end."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests.util import dptr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LEAD = 16
NAN32 = 0x7FC0DEAD
AVG, MAX, GEM = 0, 1, 2
ARG = -1
TINY = 8 * 2.0 ** -149                      # powf's 4 ulp and the mean's rounding where x^p falls below fp32's normal range
WORST = {}


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    yield _lib
    if WORST:
        print("\n[worst |o - o64| / bound per mode]")
        for k, r in sorted(WORST.items()):
            print(f"  {k:<24} {r:.4f}")


def note(k, r):
    WORST[k] = max(WORST.get(k, 0.0), r)


def gamma(k):
    return k * U / (1 - k * U)


def pool(L, x, mode, n_valid=None, p=3.0, use_abs=False, expect=0):
    """x [B, N, D] fp32 (host) -> [B, D] through anyloc_pool, the output NaN-framed"""
    B, N, D = x.shape
    xd = x.cuda()
    nv = None if n_valid is None else torch.tensor(n_valid, dtype=torch.int32, device="cuda")
    buf = torch.full((B * D + 2 * LEAD,), NAN32, dtype=torch.int32, device="cuda")
    rc = L.load().anyloc_pool(dptr(xd), dptr(nv), B, N, D, mode, C.c_float(p), int(use_abs), dptr(buf, LEAD),
                              L.stream_ptr())
    b = buf.cpu()
    assert rc == expect, L.last_error()
    assert bool((b[:LEAD] == NAN32).all() and (b[-LEAD:] == NAN32).all())
    if rc != 0:
        assert bool((b == NAN32).all()), "a refused call wrote"
        return None
    body = b[LEAD:-LEAD]
    assert not bool((body == NAN32).any()), "an output element was not written"
    return body.view(torch.float32).view(B, D).numpy()


def counts(N, n_valid, B):
    return [N] * B if n_valid is None else [min(N, v) for v in n_valid]


def check_avg(x, out, n_valid, fam):
    x64 = x.double().numpy()
    B, N, D = x.shape
    worst = 0.0
    for b, n in enumerate(counts(N, n_valid, B)):
        if n <= 0:
            assert np.isnan(out[b]).all()
            continue
        rows = x64[b, :n]
        o64 = rows.sum(0) / n
        bound = gamma(math.ceil(n / 8) + 8) * np.abs(rows).sum(0) / n + U * np.abs(o64)
        err = np.abs(out[b] - o64)
        assert (err <= bound).all(), (fam, b, float((err / bound).max()))
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    note("average " + fam, worst)


def check_max(x, out, n_valid, fam):
    B, N, D = x.shape
    for b, n in enumerate(counts(N, n_valid, B)):
        if n <= 0:
            assert np.isnan(out[b]).all()
            continue
        ref = x[b, :n].max(dim=0)[0].numpy()           # torch.max propagates NaN
        assert np.array_equal(np.isnan(out[b]), np.isnan(ref)), fam
        ok = ~np.isnan(ref)
        assert np.array_equal(out[b][ok].view(np.uint32), ref[ok].view(np.uint32)), fam
    note("max " + fam, 0.0)


def gem64(rows, p, use_abs):
    """(o64, eps_m, m64) per column, fp64; NaN where a fractional power of a negative value makes the mean NaN"""
    t = np.abs(rows) if use_abs else rows
    with np.errstate(invalid="ignore", divide="ignore"):
        pw = np.power(t, p)
    n = rows.shape[0]
    ip = p == math.floor(p) and 1 <= p <= 16
    k_pow = (p - 1) if ip else 8
    m = pw.mean(0)
    eps = (gamma(math.ceil(n / 8) + 8) + k_pow * U) * np.abs(pw).sum(0) / n + U * np.abs(m) + TINY
    o = np.sign(m) * np.abs(m) ** (1.0 / p)
    return o, eps, m


def check_gem(x, out, n_valid, p, use_abs, fam):
    B, N, D = x.shape
    worst = 0.0
    for b, n in enumerate(counts(N, n_valid, B)):
        if n <= 0:
            assert np.isnan(out[b]).all()
            continue
        o64, eps, m = gem64(x[b, :n].double().numpy(), p, use_abs)
        nan = np.isnan(o64)
        assert np.array_equal(np.isnan(out[b]), nan), (fam, p, use_abs, b)
        o, o64, eps, m = out[b][~nan], o64[~nan], eps[~nan], m[~nan]
        am = np.abs(m)
        clear = am > 2 * eps
        q = 1.0 / p
        with np.errstate(divide="ignore", invalid="ignore"):
            lo, hi = np.maximum(am - eps, 0.0), am + eps
            deriv = np.maximum(np.abs(q) * lo ** (q - 1), np.abs(q) * hi ** (q - 1))
            root = deriv * eps + (8 + np.abs(np.log(am)) / abs(p)) * U * np.abs(o64)
            amb = 2 * (am + eps) ** q
        if p < 0:
            assert clear.all(), "negative p: keep the means clear of zero"
        bound = 2 * np.where(clear, root, amb)
        err = np.abs(o.astype(np.float64) - o64)
        assert np.isfinite(o).all() and (err <= bound).all(), (fam, p, use_abs, b, float((err / bound).max()))
        worst = max(worst, float((err / bound).max(initial=0.0)))
    note(f"gem p={p:g}{' abs' if use_abs else ''} {fam}", worst)


def feats(B, N, D, seed, kind="normal"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, D, generator=g)
    if kind == "offset":                           # mean far from zero relative to the spread
        x = x * 0.1 + 3.0
    elif kind == "positive":
        x = x.abs() + 0.25
    return x


SHAPES = [(3, N, D) for D in (4, 36, 388, 1540) for N in (1, 7, 8, 9, 1369)] + [(2, 5000, 388), (2, 5000, 36)]


@pytest.mark.parametrize("B,N,D", SHAPES)
def test_average_and_max(L, B, N, D):
    for kind in ("normal", "offset"):
        x = feats(B, N, D, N * D + len(kind), kind)
        check_avg(x, pool(L, x, AVG), None, "shapes")
        check_max(x, pool(L, x, MAX), None, "shapes")


P_CASES = [1.0, 2.0, 3.0, 16.0, 17.0, 2.5, 0.5, -1.0]


@pytest.mark.parametrize("p", P_CASES)
@pytest.mark.parametrize("use_abs", [False, True])
def test_gem(L, p, use_abs):
    for B, N, D in ((3, 9, 36), (2, 1369, 388), (2, 7, 1540), (1, 5000, 4)):
        kinds = ("positive",) if p < 0 else ("normal", "offset", "positive")
        for kind in kinds:
            x = feats(B, N, D, N + D + int(4 * p), kind)
            if p >= 16:
                x = x * 0.5                       # keep |x|^17 / N far from fp32 overflow
            check_gem(x, pool(L, x, GEM, p=p, use_abs=use_abs), None, p, use_abs, kind)


def test_gem_fractional_p_on_negative_values(L):
    """NaN exactly where the fp64 reference has a negative value among the image's first n rows"""
    x = feats(3, 9, 36, 21, "positive")
    x[0, 4, 5] = -0.5
    x[1, :, 7] = -1.0
    x[2, 8, 9] = -2.0                              # past n_valid[2] = 8: not read
    for p in (2.5, 0.5):
        out = pool(L, x, GEM, n_valid=[9, 9, 8], p=p)
        check_gem(x, out, [9, 9, 8], p, False, "negative values")
        assert np.isnan(out[0, 5]) and np.isnan(out[1, 7]) and not np.isnan(out[2]).any()
        out = pool(L, x, GEM, n_valid=[9, 9, 8], p=p, use_abs=True)
        assert not np.isnan(out).any()


@pytest.mark.parametrize("D", [4, 388])
def test_n_valid(L, D):
    """n_valid > N clamps to N, 1 takes one row, <= 0 is empty (NaN); rows past n_valid hold NaN / +-Inf and are never
    read"""
    N = 37
    x = feats(6, N, D, D)
    nv = [N + 5, 1, 20, 9, 0, -3]
    for b, n in enumerate(nv):
        if 0 < n < N:
            x[b, n::3] = float("nan")
            x[b, n + 1::3] = float("inf")
            x[b, n + 2::3] = -float("inf")
    check_avg(x, pool(L, x, AVG, n_valid=nv), nv, "n_valid")
    check_max(x, pool(L, x, MAX, n_valid=nv), nv, "n_valid")
    for p, use_abs in ((3.0, False), (2.5, True), (17.0, False)):
        check_gem(x, pool(L, x, GEM, n_valid=nv, p=p, use_abs=use_abs), nv, p, use_abs, "n_valid")
    for mode in (AVG, MAX, GEM):
        assert np.isnan(pool(L, x, mode, n_valid=nv)[4:]).all()     # empty images
    # a NaN among the first n rows propagates in max and average
    x[2, 3, 1] = float("nan")
    assert np.isnan(pool(L, x, MAX, n_valid=nv)[2, 1]) and np.isnan(pool(L, x, AVG, n_valid=nv)[2, 1])


def test_grid_limit(L):
    B = 65535
    x = feats(B, 2, 4, 3)
    nv = [1 + (b % 3) for b in range(B)]          # 1, 2 and (clamped) 3
    out = pool(L, x, AVG, n_valid=nv)
    xs = x.double().numpy()
    n = np.minimum(np.array(nv), 2)
    o64 = np.where((n == 1)[:, None], xs[:, 0], (xs[:, 0] + xs[:, 1]) / 2)
    assert np.abs(out - o64).max() <= gamma(9) * np.abs(xs).sum(1).max()
    m = pool(L, x, MAX)
    assert np.array_equal(m.view(np.uint32), x.max(dim=1)[0].numpy().view(np.uint32))
    pool(L, feats(65536, 1, 4, 4), AVG, expect=ARG)


def test_independence(L):
    """reruns are bit-identical; an image's output is the same alone as inside a batch"""
    x = feats(5, 1369, 388, 22)
    nv = [1369, 700, 1, 1369, 9]
    for mode, p in ((AVG, 3.0), (MAX, 3.0), (GEM, 3.0), (GEM, 2.5)):
        a = pool(L, x, mode, n_valid=nv, p=p, use_abs=p == 2.5)
        assert np.array_equal(a.view(np.uint32), pool(L, x, mode, n_valid=nv, p=p, use_abs=p == 2.5).view(np.uint32))
        for b in (0, 2, 4):
            alone = pool(L, x[b:b + 1].contiguous(), mode, n_valid=[nv[b]], p=p, use_abs=p == 2.5)
            assert np.array_equal(alone[0].view(np.uint32), a[b].view(np.uint32)), (mode, b)


# ------------------------------------------------------------------ the Python entry points on offset views
def offset_view(t, off):
    """a contiguous CUDA view of t's values starting `off` floats into its storage (misaligned for off = 1, 2, 3)"""
    buf = torch.empty(t.numel() + off, device="cuda")
    buf[off:] = t.reshape(-1).cuda()
    v = buf[off:].view(t.shape)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4 * off % 16
    return v


def same(a, b):
    if isinstance(a, (tuple, list)):
        return all(same(p, q) for p, q in zip(a, b))
    a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
    return a.dtype == b.dtype and a.shape == b.shape and bool((a.view(-1).view(torch.uint8) ==
                                                               b.view(-1).view(torch.uint8)).all())


@pytest.mark.parametrize("off", [1, 2, 3])
def test_offset_views_reach_the_kernels_aligned(L, off):
    """every wrapper that funnels rows through _as_device_f32 gives a view at an odd storage offset the result of an
    aligned copy, bit for bit"""
    from anyloc_b200 import utilities as u
    from tests.util import make_vlad
    x = feats(3, 50, 36, 30 + off)
    xv = offset_view(x, off)
    for method, kw in (("average", {}), ("max", {}), ("gem", dict(gem_p=3.0))):
        assert same(u.pool_descriptors(xv, method, **kw), u.pool_descriptors(x.cuda(), method, **kw))
    K, D = 8, 36
    centers = torch.nn.functional.normalize(feats(1, K, D, 31)[0], dim=-1)
    v = make_vlad(u, K, centers)
    q = feats(1, 90, D, 32)[0]
    assert same(v.generate(offset_view(q, off)), v.generate(q.cuda()))
    assert same(v.generate_multi(offset_view(x, off)), v.generate_multi(x.cuda()))
    db, qu = feats(1, 300, 64, 33)[0], feats(1, 7, 64, 34)[0]
    assert same(u.top_k_search(offset_view(db, off), offset_view(qu, off), 5), u.top_k_search(db.cuda(), qu.cuda(), 5))
    ix_v, ix_a = u.FlatIndex(64, "cosine", True, device="cuda"), u.FlatIndex(64, "cosine", True, device="cuda")
    ix_v.add(offset_view(db, off))
    ix_a.add(db.cuda())
    assert same(ix_v.search(offset_view(qu, off), 5), ix_a.search(qu.cuda(), 5))
    tr, te = feats(1, 120, 40, 35)[0], feats(1, 9, 40, 36)[0]
    assert same(u.reduce_pca(offset_view(tr, off), offset_view(te, off), 8), u.reduce_pca(tr.cuda(), te.cuda(), 8))
