"""reduce_pca(svd_solver="randomized") without a device: its parameters and test matrix against what sklearn's own
randomized PCA uses (observed through its range finder), the LU normaliser against scipy's, and where the fit reads its
rows (_pca_randomized_plan) by hand-computed bytes."""
import numpy as np
import pytest
import scipy.linalg
import torch
from sklearn.decomposition import PCA
from sklearn.utils import extmath

from anyloc_b200 import utilities as u

GiB = 1 << 30


@pytest.mark.parametrize("n,d", [(40, 300), (300, 40), (120, 120), (500, 31), (31, 500)])
@pytest.mark.parametrize("k_frac", [0.02, 0.099, 0.1, 0.5, 1.0])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_params_and_test_matrix_match_sklearn(monkeypatch, n, d, k_frac, dtype):
    k = max(1, int(k_frac * min(n, d)))
    seen = {}
    real = extmath._randomized_range_finder

    def spy(A, *, size, n_iter, power_iteration_normalizer="auto", random_state=None):
        seen.update(shape=A.shape, size=size, n_iter=n_iter, state=np.random.get_state())
        return real(A, size=size, n_iter=n_iter, power_iteration_normalizer=power_iteration_normalizer,
                    random_state=random_state)
    monkeypatch.setattr(extmath, "_randomized_range_finder", spy)
    x = np.random.default_rng(n * d).standard_normal((n, d)).astype(dtype)
    np.random.seed(7)
    PCA(k, svd_solver="randomized").fit(x)
    after_sklearn = np.random.get_state()

    l, n_iter, transpose = u._pca_randomized_params(n, d, k)
    assert (l, n_iter) == (seen["size"], seen["n_iter"])
    assert seen["shape"] == ((d, n) if transpose else (n, d))
    np.random.set_state(seen["state"])                      # the generator as sklearn's range finder found it
    expect = np.random.normal(size=(seen["shape"][1], l))
    np.random.set_state(seen["state"])
    w = u._pca_test_matrix(n, d, k, dtype == np.float32)
    assert w.shape == (seen["shape"][1], l) and w.dtype == dtype
    np.testing.assert_array_equal(w, expect.astype(dtype))
    after = np.random.get_state()
    assert np.array_equal(after[1], after_sklearn[1]) and after[2:] == after_sklearn[2:]


@pytest.mark.parametrize("n,d,k", [(3, 5, 2), (1000, 64, 64), (64, 1000, 7), (997, 13, 13)])
def test_skip_leaves_the_generator_where_the_draw_does(n, d, k):
    np.random.seed(3)
    np.random.normal()                                      # leave a cached Gaussian in the legacy sampler
    u._pca_test_matrix(n, d, k, False)
    a = np.random.get_state()
    np.random.seed(3)
    np.random.normal()
    u._pca_skip_test_matrix(n, d, k, chunk=101)
    b = np.random.get_state()
    assert np.array_equal(a[1], b[1]) and a[2:] == b[2:]


@pytest.mark.parametrize("m,w", [(500, 40), (40, 40), (7, 19), (1, 5), (300, 1)])
def test_lu_pl_is_scipys_permuted_l(m, w):
    y = np.random.default_rng(m + w).standard_normal((m, w))
    pl = scipy.linalg.lu(y, permute_l=True, check_finite=False)[0]
    got = u._lu_pl(torch.from_numpy(y)).numpy()
    assert got.shape == pl.shape
    np.testing.assert_allclose(got, pl, rtol=0, atol=1e-12 * np.abs(pl).max())


def test_footprint_by_hand():
    n, d, l = 100_000, 49_152, 522
    tall = 8 * 100_000 * 522                               # fp64 [max(n, d), l]
    short = 8 * 49_152 * 522                               # fp64 [min(n, d), l]
    outputs = 4 * 522 * (100_000 + 49_152)                 # fp32 fit rows and components, at most l wide
    assert u._pca_randomized_bytes(n, d, l) == 3 * tall + 3 * short + outputs
    assert u._pca_randomized_bytes(d, n, l) == u._pca_randomized_bytes(n, d, l)


@pytest.mark.parametrize("n,d", [(40_000, 49_152), (100_000, 49_152), (26_000, 196_608)])
def test_plan_at_issue_sizes(n, d):
    l = 512 + 10
    rows = 4 * n * d
    mats = 8 * l * (3 * max(n, d) + 3 * min(n, d)) + 4 * l * (n + d)
    assert mats < 4e9                                      # the fit's own matrices are small at every size
    stages = 2 * 4 * d * (GiB // (4 * d))                  # the upload's two device copies of a staging buffer
    # 80 GB: the rows (7.9, 19.7 and 20.4 GB) are uploaded once
    assert u._pca_randomized_plan(n, d, l, 80e9, GiB) is None
    assert u._pca_randomized_plan(n, d, l, rows + max(mats, stages), GiB) is None
    # a byte less: every pass streams the rows, two staging copies of a piece beside the matrices
    P = u._pca_randomized_plan(n, d, l, rows + max(mats, stages) - 1, GiB)
    assert P == min(GiB // (4 * d), n)
    budget = mats + 2 * 4 * d * 100
    assert u._pca_randomized_plan(n, d, l, budget, GiB) == 100
    assert u._pca_randomized_plan(n, d, l, mats + 8 * d, GiB) == 1
    with pytest.raises(MemoryError, match=rf"\[{max(n, d)}, {l}\] and \[{min(n, d)}, {l}\].*{mats} bytes.*"
                                          rf"{8 * d} more, {mats + 8 * d - 1} are free"):
        u._pca_randomized_plan(n, d, l, mats + 8 * d - 1, GiB)


def test_plan_memory_error_for_huge_k():
    # 26 k x 196 608 with k = 26 000: the [196 608, 26 010] fp64 matrices alone are over 80 GB
    n, d, l = 26_000, 196_608, 26_010
    need = 8 * l * (3 * d + 3 * n) + 4 * l * (n + d)
    assert need > 80e9
    with pytest.raises(MemoryError, match=f"{need} bytes"):
        u._pca_randomized_plan(n, d, l, 80e9, GiB)


def test_plan_pieces_stay_within_the_sketch_limit():
    n, d, l = 3_000_000, 8, 18
    P = u._pca_randomized_plan(n, d, l, u._pca_randomized_bytes(n, d, l) + 4 * n * d - 1, 10 * GiB)
    assert P == u._PCA_PIECE_MAX_ROWS == 1 << 20


def test_full_route_still_refuses_beyond_the_eigensolver():
    with pytest.raises(MemoryError, match="40000 is beyond the 26733.*randomized"):
        u._pca_plan(40_000, 49_152, 0, 80e9, GiB)
    m = 600
    with pytest.raises(MemoryError, match=rf"{m} x {m}.*randomized"):
        u._pca_plan(m, 4096, 0, 48 * m * m - 1, GiB)
