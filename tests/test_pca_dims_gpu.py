"""Several PCA dimensions from one fit (reduce_pca_dims) against one reduce_pca call per dimension, bit for bit: every
member's outputs, their types and dtypes, numpy's generator state afterwards and the printed lines, on every route
(exact Gram and covariance, in memory and streamed; randomized in place, uploaded and streamed; the low_factor
branches), and the number of times the rows are staged."""
import numpy as np
import pytest
import torch

from anyloc_b200 import utilities as u
from tests.test_pca_gpu import spectrum_data
from tests.test_pca_randomized_gpu import noisy_rows

pytestmark = pytest.mark.gpu

GiB = 1 << 30


def rng_state():
    s = np.random.get_state()
    return s[1].copy(), s[2:]


class Staged:
    """counts the calls of _pca_staged, i.e. the passes over rows, and the pieces they stage"""

    def __init__(self, mp):
        self.calls = self.pieces = 0
        real = u._pca_staged

        def counted(rows, boxes, dev):
            self.calls += 1
            self.pieces += len(boxes)
            return real(rows, boxes, dev)
        mp.setattr(u, "_pca_staged", counted)


def check(capsys, tr, te, dims, **kw):
    """reduce_pca_dims against reduce_pca per dimension from np.random.seed(21) -> (sequential stagings, sweep's)"""
    capsys.readouterr()
    with pytest.MonkeyPatch.context() as mp:
        count = Staged(mp)
        np.random.seed(21)
        seq = [u.reduce_pca(tr, te, k, **kw) for k in dims]
        after_seq, seq_n = rng_state(), count.calls
        printed_seq = capsys.readouterr().out
        count.calls = 0
        np.random.seed(21)
        out = u.reduce_pca_dims(tr, te, dims, **kw)
        after, sweep_n = rng_state(), count.calls
    assert capsys.readouterr().out == printed_seq
    assert np.array_equal(after[0], after_seq[0]) and after[1] == after_seq[1]
    assert type(out) == list and len(out) == len(dims)
    for (o_tr, o_te), (r_tr, r_te) in zip(out, seq):
        for o, r in ((o_tr, r_tr), (o_te, r_te)):
            assert type(o) == type(r) and o.dtype == r.dtype and o.shape == r.shape
            if isinstance(o, torch.Tensor):
                assert not o.is_cuda
                o, r = o.numpy(), r.numpy()
            assert np.array_equal(o.view(np.uint32), r.view(np.uint32))     # bits, NaN included
    return seq_n, sweep_n


def inputs(tr, te, kind, cuda):
    """the rows as given (numpy), as CPU tensors, or as device fp32 tensors (read in place where a route can)"""
    if kind == "numpy":
        return tr, te
    if kind == "cpu":
        return torch.from_numpy(tr), torch.from_numpy(te)
    return torch.from_numpy(tr).to(cuda, torch.float32), torch.from_numpy(te).to(cuda, torch.float32)


# ------------------------------------------------------------------ exact, in memory
@pytest.mark.parametrize("n,d,dims", [(120, 512, [24, 1, 120, 24, 7]), (600, 96, [16, 96, 1, 16, 40])])
@pytest.mark.parametrize("whiten", [False, True])
@pytest.mark.parametrize("kind", ["numpy", "cpu", "cuda"])
def test_exact_in_memory(cuda, capsys, n, d, dims, whiten, kind):
    tr, te = inputs(*spectrum_data(n, d, min(n, d, 48), 0.88, seed=n + d), kind, cuda)
    check(capsys, tr, te, dims, whitening=whiten)


def test_exact_in_memory_groups(cuda, capsys, monkeypatch):
    """a budget with room for two members beside the fit: three groups, each its own fit, the same bits"""
    n, d, dims = 200, 700, [64, 32, 64, 8, 16]
    tr, te = spectrum_data(n, d, 48, 0.9, seed=4)
    budget = u._pca_in_memory_bytes(n, d, 37) + 2 * u._pca_member_bytes(n, d, 64)
    assert u._pca_exact_groups(n, d, dims, u._pca_in_memory_bytes(n, d, 37), budget) == [[0, 1], [2, 3, 4]]
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    fits = []
    real = u._pca_decompose
    monkeypatch.setattr(u, "_pca_decompose", lambda x: fits.append(1) or real(x))
    check(capsys, tr, te, dims, whitening=True)
    assert len(fits) == len(dims) + 2                      # one fit per call, one per group


# ------------------------------------------------------------------ exact, streamed
def force_streamed(mp, n_fit, d, width):
    """reduce_pca's exact route forced onto the streamed one, with pieces (or column slabs) of `width`"""
    mp.setattr(u, "_pca_plan", lambda n, d_, n_held, budget, stage: ("cov", width) if n > d_ else ("gram", width))
    mp.setattr(u, "_STAGE_BYTES", 4 * width * min(n_fit, d))


@pytest.mark.parametrize("n,d,dims,width", [(150, 1000, [16, 150, 1, 16, 40], 300), (2000, 96, [8, 96, 1, 8, 33], 450)])
@pytest.mark.parametrize("whiten", [False, True])
def test_exact_streamed(cuda, capsys, monkeypatch, n, d, dims, width, whiten):
    tr, te = spectrum_data(n, d, min(n, d, 48), 0.88, seed=n * 3 + d)
    force_streamed(monkeypatch, n, d, width)
    seq_n, sweep_n = check(capsys, tr, te, dims, whitening=whiten)
    # per call: the mean and matrix passes (one on the Gram route), the vt pass (Gram), and the two projections
    per_call = 4
    assert seq_n == per_call * len(dims) and sweep_n == per_call


def test_exact_streamed_groups(cuda, capsys, monkeypatch):
    n, d, dims = 150, 1000, [16, 150, 16, 40]
    tr, te = spectrum_data(n, d, 48, 0.88, seed=12)
    force_streamed(monkeypatch, n, d, 300)
    fixed = 8 * u._PCA_EIGH_MATRICES * n * n
    budget = fixed + u._pca_member_bytes(n, d, 150)
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    assert u._pca_exact_groups(n, d, dims, fixed, budget) == [[0], [1], [2, 3]]
    seq_n, sweep_n = check(capsys, tr, te, dims)
    assert sweep_n == 4 * 3


# ------------------------------------------------------------------ low_factor
@pytest.mark.parametrize("n,d,dims,fallback", [(120, 512, [10, 20, 1, 10], 32), (400, 40, [10, 40, 3, 10], 256)])
@pytest.mark.parametrize("streamed", [False, True])
def test_low_factor(cuda, capsys, monkeypatch, n, d, dims, fallback, streamed):
    tr, te = spectrum_data(n, d, min(n, d, 48), 0.88 if n < d else 0.9, seed=9 + n)
    if streamed:
        force_streamed(monkeypatch, n + 37 if n < d else n, d, 50)
    check(capsys, tr, te, dims, low_factor=0.3, fallback=fallback)


@pytest.mark.parametrize("n,d,fallback", [(120, 512, 64), (400, 40, 256)])
@pytest.mark.parametrize("kind", ["numpy", "cuda"])
def test_randomized_low_factor(cuda, capsys, n, d, fallback, kind):
    """n < d: every member's own randomized fallback fit, from its own draw; n >= d: the exact fit and its skips"""
    tr, te = inputs(*noisy_rows(n, d, seed=5), kind, cuda)
    check(capsys, tr, te, [20, 5, 20, 33], low_factor=0.3, fallback=fallback, svd_solver="randomized")


# ------------------------------------------------------------------ randomized
@pytest.mark.parametrize("n,d,dims", [(300, 1000, [20, 40, 1, 20, 300, 29]), (1500, 400, [32, 48, 39, 40, 400, 1])])
@pytest.mark.parametrize("whiten", [False, True])
@pytest.mark.parametrize("kind", ["numpy", "cpu", "cuda"])
def test_randomized(cuda, capsys, n, d, dims, whiten, kind):
    """in place (device fp32) or uploaded once; dims with n_iter = 7 and 4 mixed, duplicates, 1 and min(n, d)"""
    tr, te = inputs(*noisy_rows(n, d, seed=n + d), kind, cuda)
    assert {u._pca_randomized_params(n, d, k)[1] for k in dims} == {4, 7}
    seq_n, sweep_n = check(capsys, tr, te, dims, svd_solver="randomized", whitening=whiten)
    passes = 1 + max(2 * u._pca_randomized_params(n, d, k)[1] + 2 for k in dims) + 1      # mean, schedule, test rows
    uploads = 0 if kind == "cuda" else 1
    assert sweep_n == uploads + passes
    assert seq_n == sum(uploads + 1 + 2 * u._pca_randomized_params(n, d, k)[1] + 2 + 1 for k in dims)


def streamed_budget(n, d, dims, P):
    """a budget under which every member's own call streams the rows in pieces of P rows"""
    ls = [k + 10 for k in dims]
    budget = min(4 * n * d + max(u._pca_randomized_bytes(n, d, l), 8 * d * P) for l in ls) - 1
    assert budget >= max(u._pca_randomized_bytes(n, d, l) for l in ls) + 8 * d * P
    assert all(u._pca_randomized_plan(n, d, l, budget, 4 * d * P) == P for l in ls)
    return budget


@pytest.mark.parametrize("whiten", [False, True])
def test_randomized_streamed(cuda, capsys, monkeypatch, whiten):
    n, d, dims, P = 3000, 2048, [16, 64, 1, 16, 120], 400
    tr, te = noisy_rows(n, d, seed=3)
    budget = streamed_budget(n, d, dims, P)
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    monkeypatch.setattr(u, "_STAGE_BYTES", 4 * d * P)
    groups = u._pca_randomized_groups(n, d, [k + 10 for k in dims], [P] * len(dims), False, budget, 4 * d * P)
    assert [g for g, _, _ in groups] == [[0, 1, 2, 3], [4]]
    seq_n, sweep_n = check(capsys, tr, te, dims, svd_solver="randomized", whitening=whiten)
    schedule = [2 * u._pca_randomized_params(n, d, k)[1] + 2 for k in dims]
    assert sweep_n == sum(1 + max(schedule[i] for i in g) + 1 for g, _, _ in groups)
    assert seq_n == sum(1 + s + 1 for s in schedule)


def test_randomized_mixed_plans_and_groups(cuda, capsys, monkeypatch):
    """a budget under which the large members stream and the small ones upload: they never share a group (their mean
    passes sum different pieces), and the bits are still each call's"""
    n, d, P = 3000, 2048, 400
    dims = [120, 8, 1, 120, 4]
    ls = [k + 10 for k in dims]
    budget = 4 * n * d + 8 * d * P                          # the rows beside two staging copies
    plans = [u._pca_randomized_plan(n, d, l, budget, 4 * d * P) for l in ls]
    assert plans[0] == plans[3] == P and plans[1] is None and plans[2] is None and plans[4] is None
    groups = u._pca_randomized_groups(n, d, ls, plans, False, budget, 4 * d * P)
    assert groups == [([0], P, False), ([1, 2], n, True), ([3], P, False), ([4], n, True)]
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    monkeypatch.setattr(u, "_STAGE_BYTES", 4 * d * P)
    tr, te = noisy_rows(n, d, seed=8)
    check(capsys, tr, te, dims, svd_solver="randomized")


def test_randomized_in_place_groups(cuda, capsys, monkeypatch):
    n, d, dims = 300, 1000, [40, 20, 60, 20, 5]
    tr, te = inputs(*noisy_rows(n, d, seed=2), "cuda", cuda)
    ls = [k + 10 for k in dims]
    budget = u._pca_randomized_bytes(n, d, 50) + u._pca_randomized_bytes(n, d, 30)
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    groups = u._pca_randomized_groups(n, d, ls, [None] * 5, True, budget, GiB)
    assert [g for g, _, _ in groups] == [[0, 1], [2], [3, 4]]
    seq_n, sweep_n = check(capsys, tr, te, dims, svd_solver="randomized")
    schedule = [2 * u._pca_randomized_params(n, d, k)[1] + 2 for k in dims]
    assert sweep_n == sum(1 + max(schedule[i] for i in g) + 1 for g, _, _ in groups)


def test_single_dimension_is_reduce_pca(cuda, capsys):
    tr, te = spectrum_data(300, 200, 48, 0.9, seed=8)
    for kw in ({}, dict(svd_solver="randomized"), dict(low_factor=0.5)):
        check(capsys, tr, te, [16], **kw)


def test_dropin_exports_it(cuda):
    from anyloc_b200.dropin import utilities as shim
    assert shim.reduce_pca_dims is u.reduce_pca_dims
