"""reduce_pca_dims' host logic without a GPU: its refusals (made before any work, with numpy's generator untouched),
the draws it takes from that generator against the sequential reduce_pca calls', the pass schedule of randomized fits
with mixed n_iter, and the grouping plans by hand-computed bytes."""
import numpy as np
import pytest
import torch

from anyloc_b200 import utilities as u

GiB = 1 << 30


def rng_state():
    s = np.random.get_state()
    return s[1].copy(), s[2:]


def same_state(a, b):
    return np.array_equal(a[0], b[0]) and a[1] == b[1]


@pytest.mark.parametrize("dims,kw,match", [
    ([], {}, "lower_dims is empty"),
    ([8, 41, 4], {}, r"n_components=41 must be between 0 and min\(n_samples, n_features\)=40 with svd_solver='full'"),
    ([8, -1], {}, "n_components=-1 must be between 0"),
    ([8, 0], dict(svd_solver="randomized"), "n_components=0 must be between 1 and min.*=40 with svd_solver='randomized'"),
    ([41], dict(svd_solver="randomized"), "n_components=41 must be between 1"),
])
def test_refusals_before_any_work(dims, kw, match):
    tr, te = np.zeros((300, 40), np.float32), np.zeros((7, 40), np.float32)
    np.random.seed(5)
    before = rng_state()
    with pytest.raises(ValueError, match=match):
        u.reduce_pca_dims(tr, te, dims, **kw)
    assert same_state(rng_state(), before)


def test_fallback_refusals():
    # n < d with low_factor: the fallback pre-reduction's k, then the full basis of the [n, fallback] rows
    tr, te = torch.zeros(30, 100), torch.zeros(5, 100)
    np.random.seed(5)
    before = rng_state()
    with pytest.raises(ValueError, match="n_components=36 must be between 1 and .*=35 with svd_solver='randomized'"):
        u.reduce_pca_dims(tr, te, [4, 8], low_factor=0.5, fallback=36, svd_solver="randomized")
    with pytest.raises(ValueError, match="n_components=36 must be between 0 and .*=35 with svd_solver='full'"):
        u.reduce_pca_dims(tr, te, [4, 8], low_factor=0.5, fallback=36)
    with pytest.raises(ValueError, match="n_components=32 must be between 0 and .*=30 with svd_solver='full'"):
        u.reduce_pca_dims(tr, te, [4, 8], low_factor=0.5, fallback=32, svd_solver="randomized")
    assert same_state(rng_state(), before)


class Shape:
    """stands for rows of a given shape: the refusals read nothing else"""

    def __init__(self, *shape):
        self.shape = shape


@pytest.mark.parametrize("n,d,kw,m", [(30_000, 49_152, {}, 30_000), (26_734, 26_734, {}, 26_734),
                                      (26_800, 30_000, dict(low_factor=0.2, fallback=64), 26_810),
                                      (40_000, 30_000, dict(low_factor=0.2, svd_solver="randomized"), 30_000)])
def test_exact_limit_refused(n, d, kw, m):
    np.random.seed(5)
    before = rng_state()
    with pytest.raises(ValueError, match=f"m = min\\(n_samples, n_features\\) = {m} is beyond the 26733"):
        u.reduce_pca_dims(Shape(n, d), Shape(10, d), [16, 8], **kw)
    assert same_state(rng_state(), before)


def test_randomized_beyond_the_exact_limit_is_not_refused():
    u._pca_dims_check(40_000, 49_152, 10, [1024, 16], 0.0, 256, "randomized")
    u._pca_dims_check(1000, 49_152, 10, [1024, 16], 0.5, 256, "randomized")


def sequential_draws(n, d, n_te, dims, low_factor, fallback, f32):
    """the draws reduce_pca's randomized routes make, call after call, restated from their code"""
    for k in dims:
        if low_factor == 0.0:
            u._pca_test_matrix(n, d, k, f32)                         # _reduce_pca_randomized -> _pca_fit_randomized
        elif n < d:
            u._pca_test_matrix(n + n_te, d, fallback, f32)           # the fallback pre-reduction
            u._pca_skip_test_matrix(n, fallback, fallback)           # the exact full-basis fit
        else:
            u._pca_skip_test_matrix(n, d, d)                         # reduce_pca's exact fit, then the skip


@pytest.mark.parametrize("n,d,low_factor", [(300, 40, 0.0), (40, 300, 0.0), (40, 300, 0.3), (300, 40, 0.3)])
@pytest.mark.parametrize("dims", [[16], [4, 16, 4, 1, 40], [40, 2, 7]])
@pytest.mark.parametrize("cut", [0, 1, 2])
def test_draws_match_the_sequential_calls(n, d, low_factor, dims, cut):
    """the sweep's draws, taken group by group (any consecutive split), leave the generator where the calls do, and
    each member's test matrix is the one its own call draws"""
    n_te, fallback = 9, 32
    np.random.seed(11)
    np.random.normal()                                      # leave a cached Gaussian in the legacy sampler
    sequential_draws(n, d, n_te, dims, low_factor, fallback, True)
    after = rng_state()
    np.random.seed(11)
    np.random.normal()
    own = []
    for k in dims:
        own += u._pca_draw(u._pca_member_draws(n, d, n_te, k, low_factor, fallback, "randomized"), True)

    np.random.seed(11)
    np.random.normal()
    draws = [u._pca_member_draws(n, d, n_te, k, low_factor, fallback, "randomized") for k in dims]
    cut = min(cut, len(dims))
    ws = u._pca_draw(sum(draws[:cut], []), True) + u._pca_draw(sum(draws[cut:], []), True)
    assert same_state(rng_state(), after)
    assert len(ws) == len(own) == (len(dims) if low_factor == 0.0 or n < d else 0)
    for a, b in zip(ws, own):
        assert a.dtype == np.float32 and np.array_equal(a, b)
    assert all(u._pca_member_draws(n, d, n_te, k, low_factor, fallback, "full") == [] for k in dims)


def test_equal_dimensions_draw_twice():
    np.random.seed(3)
    a, b = u._pca_draw(sum((u._pca_member_draws(200, 50, 5, 8, 0.0, 256, "randomized") for _ in range(2)), []), False)
    assert a.shape == b.shape == (50, 18) and not np.array_equal(a, b)


def test_schedule_with_mixed_n_iter():
    n, d = 1000, 400                                        # n_iter = 7 where k < 40, else 4
    ks = [64, 16, 40, 39]
    assert [u._pca_randomized_params(n, d, k)[1] for k in ks] == [4, 7, 4, 7]
    sched = u._pca_randomized_schedule(n, d, ks)
    assert len(sched) == 16
    assert [f for f, _ in sched] == [True, False] * 8      # A, A^T, ... for every member alike
    for p, (_, live) in enumerate(sched):
        expect = []
        for i, k in enumerate(ks):
            steps = 2 * u._pca_randomized_params(n, d, k)[1] + 2
            if p < steps - 2:
                expect.append((i, "lu"))
            elif p == steps - 2:
                expect.append((i, "qr"))
            elif p == steps - 1:
                expect.append((i, "svd"))
        assert live == expect
    assert sched[8][1] == [(0, "qr"), (1, "lu"), (2, "qr"), (3, "lu")]
    assert sched[9][1] == [(0, "svd"), (1, "lu"), (2, "svd"), (3, "lu")]
    assert sched[10][1] == [(1, "lu"), (3, "lu")]
    assert sched[15][1] == [(1, "svd"), (3, "svd")]
    # a single member: the lone fit's schedule
    assert [live for _, live in u._pca_randomized_schedule(n, d, [64])] == [[(0, "lu")]] * 8 + [[(0, "qr")], [(0, "svd")]]


def test_exact_groups_by_hand():
    m, d = 10_000, 49_152
    ks = [1024, 512, 256, 128, 64, 32, 16]
    per = [8 * k * (m + d) + 4 * k * d for k in ks]
    assert [u._pca_member_bytes(m, d, k) for k in ks] == per
    fixed = 48 * m * m
    assert u._pca_exact_groups(m, d, ks, fixed, fixed + sum(per)) == [list(range(7))]
    # a byte short: the last member starts a group of its own
    assert u._pca_exact_groups(m, d, ks, fixed, fixed + sum(per) - 1) == [list(range(6)), [6]]
    # room for 1024 alone, then for all the rest
    assert u._pca_exact_groups(m, d, ks, fixed, fixed + per[0]) == [[0], [1, 2, 3, 4, 5, 6]]
    # room for 512 + 256: 1024 runs alone, beyond the room, then 512 + 256, then 128 + 64 + 32 + 16
    assert u._pca_exact_groups(m, d, ks, fixed, fixed + per[1] + per[2]) == [[0], [1, 2], [3, 4, 5, 6]]
    # a member that does not fit even alone still runs, alone
    assert u._pca_exact_groups(m, d, [16, 2048, 16], fixed, fixed + per[0]) == [[0], [1], [2]]


def test_randomized_groups_by_hand():
    n, d = 100_000, 49_152
    ks = [1024, 512, 256, 128, 64, 32, 16]
    ls = [k + 10 for k in ks]
    mats = [8 * l * (3 * n + 3 * d) + 4 * l * (n + d) for l in ls]
    assert [u._pca_randomized_bytes(n, d, l) for l in ls] == mats
    rows = 4 * n * d
    piece = 4 * d * (GiB // (4 * d))
    P_up = n                                                # min(n, 2^20)
    # in place: only the matrices count
    assert u._pca_randomized_groups(n, d, ls, [None] * 7, True, sum(mats), GiB) == [(list(range(7)), P_up, False)]
    assert u._pca_randomized_groups(n, d, ls, [None] * 7, True, sum(mats) - 1, GiB) == \
        [(list(range(6)), P_up, False), ([6], P_up, False)]
    # uploaded: the rows once beside every member's matrices
    budget = rows + sum(mats)
    assert u._pca_randomized_groups(n, d, ls, [None] * 7, False, budget, GiB) == [(list(range(7)), P_up, True)]
    budget = rows + mats[0] + mats[1]
    assert u._pca_randomized_groups(n, d, ls, [None] * 7, False, budget, GiB) == \
        [([0, 1], P_up, True), ([2, 3, 4, 5, 6], P_up, True)]
    assert mats[2] + mats[3] + mats[4] + mats[5] + mats[6] <= mats[0] + mats[1]
    # streamed in pieces of P: two device copies of a piece beside the matrices
    P = GiB // (4 * d)
    budget = sum(mats[:4]) + 8 * d * P
    assert u._pca_randomized_groups(n, d, ls, [P] * 7, False, budget, GiB) == \
        [([0, 1, 2, 3], P, False), ([4, 5, 6], P, False)]
    # members whose own calls read the rows in other pieces never share a group
    plans = [P, None, None, P, P - 1, P - 1, None]
    groups = u._pca_randomized_groups(n, d, ls, plans, False, 1 << 50, GiB)
    assert groups == [([0], P, False), ([1, 2], P_up, True), ([3], P, False), ([4, 5], P - 1, False),
                      ([6], P_up, True)]
    assert 2 * piece < mats[0]


def test_lone_plans_always_fit_their_own_group():
    """a member alone is in a group the budget admits whenever its own call's plan does"""
    n, d = 100_000, 49_152
    for budget in (25e9, 30e9, 60e9):
        budget = int(budget)
        for k in (1024, 16):
            l = k + 10
            plan = u._pca_randomized_plan(n, d, l, budget, GiB)
            mats = u._pca_randomized_bytes(n, d, l)
            need = 4 * n * d + max(mats, 2 * 4 * d * (GiB // (4 * d))) if plan is None else mats + 8 * d * plan
            assert need <= budget
