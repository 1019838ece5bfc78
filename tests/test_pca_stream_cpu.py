"""Where reduce_pca runs (utilities.py:522-586; scripts/dino_v2_vlad.py:357-369): the in-memory route while its
footprint fits the device, else the rows streamed through the fp64 Gram / covariance accumulation, else MemoryError.
Plan logic and piece layout only: no device."""
import numpy as np
import pytest
import torch

from anyloc_b200 import utilities as u

GiB = 1 << 30


@pytest.mark.parametrize("n,d,n_held", [(10_000, 49_152, 1000), (40_000, 49_152, 0), (5000, 768, 37),
                                        (600, 4096, 600), (1, 1, 0)])
def test_footprint_by_hand(n, d, n_held):
    m = min(n, d)
    rows = 4 * n * d + 4 * n * d + 8 * n * d          # the fp32 rows, their centred fp32 copy, its fp64 copy
    held = 4 * n_held * d
    eig = 6 * 8 * m * m                                # the m x m matrix, eigh's eigenvectors and 4 matrices of workspace
    assert u._pca_in_memory_bytes(n, d, n_held) == rows + held + eig


def test_issue_sizes():
    # 26 k x 196 608 (ViT-G, K = 128): more than 80 GB in memory; the 5.4 GB Gram matrix and its eigh fit
    assert u._pca_in_memory_bytes(26_000, 196_608, 0) > 80e9
    assert u._pca_plan(26_000, 196_608, 0, 80e9, GiB)[0] == "gram"
    # 40 k x 49 152 (K = 32) and 30 k x 196 608: m is beyond what the eigensolver takes
    for n, d in ((40_000, 49_152), (30_000, 196_608)):
        assert u._pca_in_memory_bytes(n, d, 0) > 80e9
        with pytest.raises(MemoryError, match=f"{n} is beyond the 26733"):
            u._pca_plan(n, d, 0, 80e9, GiB)
    # c3's 10 k database fits in memory
    assert u._pca_plan(10_000, 49_152, 1000, 80e9, GiB) is None


@pytest.mark.parametrize("n,d", [(5000, 768), (600, 4096), (20_000, 20_000), (3000, 49_152), (1, 7)])
def test_route_choice_and_memory_error(n, d):
    need = u._pca_in_memory_bytes(n, d, 0)
    m = min(n, d)
    eig = 48 * m * m
    assert u._pca_plan(n, d, 0, need, GiB) is None                        # in memory whenever it fits
    assert u._pca_plan(n, d, 0, need + 10 * GiB, GiB) is None
    if eig < need:
        route, _ = u._pca_plan(n, d, 0, need - 1, GiB)                    # streamed otherwise
        assert route == ("cov" if n > d else "gram")
        assert u._pca_plan(n, d, 0, eig, GiB)[0] == route                 # down to exactly the matrix and its eigh
    with pytest.raises(MemoryError, match=rf"{m} x {m}.*{eig} bytes.*{eig - 1} are free"):
        u._pca_plan(n, d, 0, eig - 1, GiB)                                # and no further


def test_eigh_size_limit():
    m = u._PCA_EIGH_MAX_M
    assert u._pca_plan(m, 10 * m, 0, 60 * m * m, GiB)[0] == "gram"
    assert u._pca_plan(10 * m, m, 0, 60 * m * m, GiB)[0] == "cov"
    for n, d in ((m + 1, 10 * m), (10 * m, m + 1)):
        with pytest.raises(MemoryError, match="beyond"):
            u._pca_plan(n, d, 0, 60 * m * m, GiB)


def test_piece_sizes():
    n, d = 5000, 768
    eig = 48 * d * d
    _, P = u._pca_plan(n, d, 0, u._pca_in_memory_bytes(n, d, 0) - 1, 1000 * 4 * d)
    assert P == 1000                                                      # one staging buffer
    _, P = u._pca_plan(n, d, 0, u._pca_in_memory_bytes(n, d, 0) - 1, 10 * GiB)
    assert P == n                                                         # never more than the rows
    budget = eig
    _, P = u._pca_plan(n, d, 0, budget, 10 * GiB)
    assert 2 * P * 4 * d + 8 * d * d <= budget                           # two device copies beside the matrix
    _, W = u._pca_plan(600, 4096, 0, 48 * 600 * 600, 10 * GiB)
    assert 2 * W * 4 * 600 + 8 * 600 * 600 <= 48 * 600 * 600 and W >= 1


@pytest.mark.parametrize("n,d,plan", [(5000, 768, ("cov", 1000)), (5001, 768, ("cov", 1000)), (7, 3, ("cov", 1)),
                                      (129, 100, ("cov", 200)), (600, 4096, ("gram", 1000)), (1, 7, ("gram", 3)),
                                      (197, 197, ("gram", 64))])
def test_boxes_cover_once_in_order(n, d, plan):
    boxes = u._pca_boxes(n, d, plan)
    seen = np.zeros((n, d), np.int32)
    for r0, r1, c0, c1 in boxes:
        assert r0 < r1 and c0 < c1
        seen[r0:r1, c0:c1] += 1
    assert (seen == 1).all()
    if plan[0] == "cov":
        assert all(c0 == 0 and c1 == d for _, _, c0, c1 in boxes)
        assert [b[0] for b in boxes] == sorted(b[0] for b in boxes)
        assert all(r1 - r0 == plan[1] for r0, r1, _, _ in boxes[:-1])
    else:
        assert all(r0 == 0 and r1 == n for r0, r1, _, _ in boxes)
        assert [b[2] for b in boxes] == sorted(b[2] for b in boxes)
        assert all(c1 - c0 == plan[1] for _, _, c0, c1 in boxes[:-1])


def test_rows_gather_any_input():
    g = np.random.default_rng(0)
    a = g.standard_normal((9, 12))                                        # fp64
    b = np.asfortranarray(g.standard_normal((5, 12)).astype(np.float16))  # non-contiguous rows, fp16
    c = torch.from_numpy(g.standard_normal((30, 12)).astype(np.float32))[::3]
    rows = u._PcaRows([a, b, c])
    full = np.concatenate([a, b.astype(np.float64), c.double().numpy()]).astype(np.float32)
    assert rows.shape == (24, 12) and not rows.is_cuda
    for box in [(0, 24, 0, 12), (7, 16, 0, 12), (0, 24, 5, 9), (13, 14, 11, 12)]:
        r0, r1, c0, c1 = box
        dst = torch.full((r1 - r0, c1 - c0), float("nan"))
        rows.gather(dst, box)
        np.testing.assert_array_equal(dst.numpy(), full[r0:r1, c0:c1])
    # the caller's arrays are read, never converted or pinned in place
    assert a.dtype == np.float64 and not c.is_pinned()
