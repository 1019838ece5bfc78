"""reduce_pca(svd_solver="randomized") on the GPU.  The "sketch" layout of anyloc_pca_accumulate element by element
against numpy fp64; the route against sklearn's own randomized PCA (oracle restatement) from the same draw of numpy's
global generator; and a 40 000 x 49 152 fit, beyond the exact solver's limit, against the planted factors of rows of
known rank, with the rows on the device, uploaded once and streamed."""
import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from oracle import anyloc_oracle as ao
from tests.test_pca_gpu import spectrum_data
from tests.test_pca_stream_gpu import accumulate, canvas, check_frame, rows_data, vp
from tests.util import rel_inf

pytestmark = pytest.mark.gpu

NAN = float("nan")


# ------------------------------------------------------------------ the sketch kernel
@pytest.mark.parametrize("n,d,k", [(1, 7, 1), (7, 1, 3), (129, 1000, 37), (1000, 129, 70), (197, 3 * 64 + 5, 64),
                                   (64, 64, 16), (300, 49, 130)])
def test_sketch_matches_fp64(cuda, n, d, k):
    x, mu = rows_data(n, d, seed=n * 5 + d)
    w = np.random.default_rng(n + k).standard_normal((d, k + 3))
    ref = (x.astype(np.float64) - mu) @ w[:, :k]
    xs = torch.full((n, d + 5), NAN, device=cuda)          # ld = d + 5
    xs[:, :d] = torch.from_numpy(x).to(cuda)
    xv, mud = xs[:, :d], torch.from_numpy(mu).to(cuda)
    wd = torch.from_numpy(w).to(cuda)[:, :k]                # ld_u = k + 3
    frame, out = canvas(n, k, cuda)
    accumulate("sketch", xv, mud, out, wd)
    torch.cuda.synchronize()
    check_frame(frame, n, k)
    first = out.clone()
    assert rel_inf(first.cpu().numpy(), ref) < 1e-12
    accumulate("sketch", xv, mud, out, wd)                  # += across calls
    assert rel_inf(out.cpu().numpy(), 2 * ref) < 1e-12
    frame2, again = canvas(n, k, cuda)
    accumulate("sketch", xv, mud, again, wd)
    assert torch.equal(again, first)                        # bit-identical rerun
    check_frame(frame, n, k)


@pytest.mark.parametrize("n,d,k,cuts", [(1000, 197, 40, [0, 1, 300, 301, 999, 1000]), (129, 64, 16, [0, 64, 129])])
def test_sketch_row_pieces_equal_one_piece(cuda, n, d, k, cuts):
    x, mu = rows_data(n, d, seed=11)
    xd, mud = torch.from_numpy(x).to(cuda), torch.from_numpy(mu).to(cuda)
    w = torch.from_numpy(np.random.default_rng(2).standard_normal((d, k))).to(cuda)
    whole = torch.zeros(n, k, dtype=torch.float64, device=cuda)
    accumulate("sketch", xd, mud, whole, w)
    parts = torch.zeros_like(whole)
    for a, b in zip(cuts[:-1], cuts[1:]):
        accumulate("sketch", xd[a:b], mud, parts[a:b], w)
    assert torch.equal(parts, whole)                        # each output row sums its columns in one fixed order
    cols = torch.zeros_like(whole)                          # and pieces of the columns add up to the whole
    for a, b in ((0, 5), (5, d // 2), (d // 2, d)):
        accumulate("sketch", xd[:, a:b], mud[a:b], cols, w[a:b])
    assert rel_inf(cols, whole) < 1e-12


def test_sketch_abi_refusals(cuda):
    lib = _lib.load()
    x = torch.zeros(8, 8, device=cuda)
    mu = torch.zeros(8, dtype=torch.float64, device=cuda)
    w = torch.zeros(8, 4, dtype=torch.float64, device=cuda)
    out = torch.full((8, 4), NAN, dtype=torch.float64, device=cuda)
    st, S = _lib.stream_ptr(), _lib.PCA["sketch"]
    assert lib.anyloc_pca_accumulate(S, vp(x), 8, 8, 8, vp(mu), None, 4, 4, vp(out), 4, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(S, vp(x), 8, 8, 8, vp(mu), vp(w), 3, 4, vp(out), 4, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(S, vp(x), 8, 8, 8, vp(mu), vp(w), 4, 4, vp(out), 3, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(S, vp(x), 8, 8, 8, vp(mu), None, 0, 0, vp(out), 4, st) == 0
    torch.cuda.synchronize()
    assert torch.isnan(out).all()                           # a refusal, or k = 0, writes nothing


# ------------------------------------------------------------------ the route against sklearn
def noisy_rows(n, d, seed, n_test=37):
    """fp32-representable float64 rows with a slowly decaying full-rank spectrum and a non-zero mean: the randomized
    and exact fits differ well above rounding"""
    g = np.random.default_rng(seed)
    scales = 0.99 ** np.arange(d)
    offset = 0.3 * g.standard_normal(d)
    make = lambda m: (g.standard_normal((m, d)) * scales + offset).astype(np.float32).astype(np.float64)
    return make(n), make(n_test)


def rng_state():
    s = np.random.get_state()
    return s[1].copy(), s[2:]


def same_state(a, b):
    return np.array_equal(a[0], b[0]) and a[1] == b[1]


def both(fn_ours, fn_ref, seed=123):
    """ours and the oracle's outputs from the same global generator state, and whether they leave it the same"""
    np.random.seed(seed)
    ref = fn_ref()
    after_ref = rng_state()
    np.random.seed(seed)
    ours = fn_ours()
    return ours, ref, same_state(rng_state(), after_ref)


# n_iter = 7 where k < 0.1 min(n, d), else 4
@pytest.mark.parametrize("n,d,k,whiten", [(300, 1000, 20, False), (300, 1000, 40, True), (1500, 400, 32, True),
                                          (1500, 400, 48, False), (2000, 64, 40, True)])
def test_route_matches_sklearn(cuda, n, d, k, whiten):
    tr, te = noisy_rows(n, d, seed=n + d + k)
    kw = dict(svd_solver="randomized", whitening=whiten)
    (o_tr, o_te), (r_tr, r_te), rng_same = both(lambda: u.reduce_pca(tr, te, k, **kw),
                                                lambda: ao.reduce_pca(tr, te, k, **kw))
    assert rng_same
    assert type(o_tr) == np.ndarray and o_tr.dtype == np.float32 and o_tr.shape == (n, k) and o_te.shape == (37, k)
    e_tr, e_te = ao.reduce_pca(tr, te, k, whitening=whiten)                 # the exact fit
    err = max(rel_inf(o_tr, r_tr), rel_inf(o_te, r_te))
    gap = min(rel_inf(e_tr, r_tr), rel_inf(e_te, r_te))
    assert err < 5e-6 and gap > 1e-3, (err, gap)


def test_route_low_factor_fallback_matches_sklearn(cuda):
    tr, te = noisy_rows(120, 512, seed=5)
    kw = dict(low_factor=0.3, fallback=64, svd_solver="randomized")
    (o_tr, o_te), (r_tr, r_te), rng_same = both(lambda: u.reduce_pca(tr, te, 20, **kw),
                                                lambda: ao.reduce_pca(tr, te, 20, **kw))
    assert rng_same
    assert o_tr.shape == r_tr.shape == (120, 20) and o_te.shape == r_te.shape == (37, 20)
    assert rel_inf(o_tr, r_tr) < 5e-6 and rel_inf(o_te, r_te) < 5e-6
    e_tr, _ = ao.reduce_pca(tr, te, 20, low_factor=0.3, fallback=64)
    assert rel_inf(e_tr, r_tr) > 1e-3


def test_route_low_factor_full_basis_keeps_the_generator_in_step(cuda):
    tr, te = noisy_rows(400, 40, seed=6)
    kw = dict(low_factor=0.3, svd_solver="randomized")
    (o_tr, o_te), (r_tr, r_te), rng_same = both(lambda: u.reduce_pca(tr, te, 10, **kw),
                                                lambda: ao.reduce_pca(tr, te, 10, **kw))
    assert rng_same
    assert rel_inf(o_tr, r_tr) < 1e-4 and rel_inf(o_te, r_te) < 1e-4


@pytest.mark.parametrize("n,d,k", [(600, 4096, 32), (3000, 256, 16)])
def test_route_float32_matches_sklearns_float32_run(cuda, n, d, k):
    """sklearn computes in fp32 on fp32 rows, from the fp32-rounded test matrix; this route rounds the test matrix the
    same way and computes in fp64, so the gap is sklearn's own fp32 rounding"""
    tr, te = spectrum_data(n, d, 48, 0.88, seed=n + d)
    kw = dict(svd_solver="randomized")
    (o_tr, o_te), (r_tr, r_te), rng_same = both(lambda: u.reduce_pca(tr, te, k, **kw),
                                                lambda: ao.reduce_pca(tr, te, k, **kw))
    assert rng_same and r_tr.dtype == np.float32
    assert rel_inf(o_tr, r_tr) < 8e-6 and rel_inf(o_te, r_te) < 8e-6


def test_route_torch_inputs_and_errors(cuda):
    tr, te = spectrum_data(300, 200, 48, 0.9, seed=8)
    np.random.seed(1)
    a_tr, a_te = u.reduce_pca(tr, te, 16, svd_solver="randomized")
    for dev in ("cpu", cuda):
        np.random.seed(1)
        o_tr, o_te = u.reduce_pca(torch.from_numpy(tr).to(dev), torch.from_numpy(te).to(dev), 16,
                                  svd_solver="randomized")
        assert isinstance(o_tr, torch.Tensor) and not o_tr.is_cuda and o_tr.dtype == torch.float32
        # the same fp32 rows read in place, or uploaded: the same bits
        assert np.array_equal(o_tr.numpy(), a_tr) and np.array_equal(o_te.numpy(), a_te)
    for k in (0, 201):
        with pytest.raises(ValueError, match="svd_solver='randomized'"):
            u.reduce_pca(tr, te, k, svd_solver="randomized")


# ------------------------------------------------------------------ beyond the exact solver's limit
N_BIG, D_BIG, K_BIG, R_BIG = 40_000, 49_152, 256, 256


@pytest.fixture(scope="module")
def planted(cuda):
    """rows X = U diag(s) V^T + mean of exact rank 256 (U [n, r] zero-mean orthonormal, V [d, r] orthonormal, s
    distinct and decaying), device fp32, and 64 test rows T = A V^T + mean with known coordinates A"""
    g = torch.Generator(device=cuda).manual_seed(17)
    n, d, r = N_BIG, D_BIG, R_BIG
    left = torch.randn(n, r, device=cuda, dtype=torch.float64, generator=g)
    left = torch.linalg.qr(left - left.mean(0)).Q
    v = torch.linalg.qr(torch.randn(d, r, device=cuda, dtype=torch.float64, generator=g)).Q
    s = 1000.0 * 0.97 ** torch.arange(r, device=cuda, dtype=torch.float64)
    mean = 0.01 * torch.randn(d, device=cuda, dtype=torch.float64, generator=g)
    x = torch.empty(n, d, device=cuda)
    for r0 in range(0, n, 4096):
        x[r0:r0 + 4096] = ((left[r0:r0 + 4096] * s) @ v.T + mean).float()
    a = torch.randn(64, r, device=cuda, dtype=torch.float64, generator=g) * s / np.sqrt(n)
    t = (a @ v.T + mean).float()
    return x, t, v, s, a


def fit_planted(x, t):
    np.random.seed(99)
    o_tr, o_te = u.reduce_pca(x, t, K_BIG, svd_solver="randomized")
    return tuple(o if type(o) == np.ndarray else o.numpy() for o in (o_tr, o_te))


def check_planted(pca_like, o_te, v, s, a):
    comps, sv = pca_like
    c = comps.double() @ v                                  # [k, r]: +-1 on the diagonal
    dots = c.diagonal().abs()
    assert float((1 - dots).abs().max()) < 1e-6, float((1 - dots).abs().max())
    assert rel_inf(sv.cpu(), s.cpu()) < 1e-5
    sign = torch.sign(c.diagonal()).cpu().numpy()
    assert rel_inf(o_te, (a.cpu().numpy() * sign)) < 1e-4


def test_beyond_the_exact_limit(cuda, monkeypatch, planted):
    x, t, v, s, a = planted
    n, d = N_BIG, D_BIG
    with pytest.raises(MemoryError, match=f"{n} is beyond the 26733"):
        u.reduce_pca(x, t, K_BIG)                           # the exact route still refuses this size
    fits = []
    real = u._PcaDev.fit_randomized

    def spy(pca, rows, w, P, dev):
        out = real(pca, rows, w, P, dev)
        fits.append((rows.is_cuda, P, pca.components_.clone(), pca.singular_values_.clone()))
        return out
    monkeypatch.setattr(u._PcaDev, "fit_randomized", spy)

    d_tr, d_te = fit_planted(x, t)                          # device rows, read in place
    assert fits[-1][0] and fits[-1][2].shape == (K_BIG, d)
    check_planted(fits[-1][2:], d_te, v, s, a)
    assert np.isfinite(d_tr).all() and d_tr.shape == (n, K_BIG)

    xh, th = x.cpu().numpy(), t.cpu().numpy()
    h_tr, h_te = fit_planted(xh, th)                        # host rows, uploaded once
    assert fits[-1][0] and fits[-1][1] == n
    check_planted(fits[-1][2:], h_te, v, s, a)
    assert np.array_equal(h_tr, d_tr) and np.array_equal(h_te, d_te)    # the same rows on the device: the same bits

    l = K_BIG + 10
    with monkeypatch.context() as mp:                       # host rows streamed in pieces of 4096 rows
        mp.setattr(u, "_device_budget", lambda dev, release_cache=True: u._pca_randomized_bytes(n, d, l) + 4 * n * d - 1)
        mp.setattr(u, "_STAGE_BYTES", 4 * d * 4096)
        s_tr, s_te = fit_planted(xh, th)
        assert not fits[-1][0] and fits[-1][1] == 4096
        s_tr2, s_te2 = fit_planted(xh, th)
    assert np.array_equal(s_tr, s_tr2) and np.array_equal(s_te, s_te2)  # bit-identical rerun
    check_planted(fits[-1][2:], s_te, v, s, a)
    assert rel_inf(s_tr, d_tr) < 1e-6 and rel_inf(s_te, d_te) < 1e-6


# ------------------------------------------------------------------ the exact route is untouched
@pytest.mark.parametrize("n,d,k,whiten", [(300, 96, 16, True), (120, 512, 24, False)])
def test_full_and_auto_unchanged(cuda, n, d, k, whiten):
    tr, te = spectrum_data(n, d, min(n, d, 48), 0.88, seed=n + d)
    state = rng_state()
    base_tr, base_te = u.reduce_pca(tr, te, k, whitening=whiten)
    for solver in ("full", "auto", "arpack", "covariance_eigh"):
        o_tr, o_te = u.reduce_pca(tr, te, k, svd_solver=solver, whitening=whiten)
        assert np.array_equal(o_tr, base_tr) and np.array_equal(o_te, base_te)
    assert same_state(rng_state(), state)                   # the exact route draws nothing
    b_tr, b_te = u.reduce_pca(tr, te, 10, low_factor=0.3, fallback=64)
    o_tr, o_te = u.reduce_pca(tr, te, 10, low_factor=0.3, fallback=64, svd_solver="full")
    assert np.array_equal(o_tr, b_tr) and np.array_equal(o_te, b_te)
