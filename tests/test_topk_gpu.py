"""GPU parity of the retrieval path (anyloc_topk via get_top_k_recall) against golden vectors
from the reference's get_top_k_recall and against the oracle.  Indices exact outside the
fp64-ambiguous set (adjacent score gap < 1e-6), distances 1e-4 relative."""
import numpy as np
import pytest
import torch

from oracle import anyloc_oracle as ao
from tests.util import load_cases, rel_inf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def _gt(arr):
    gt = np.empty(len(arr), dtype=object)
    for i, row in enumerate(arr):
        gt[i] = np.asarray(row)
    return gt


def test_topk_golden(u):
    g = load_cases("topk.npz")
    db, qu, gt = torch.from_numpy(g[""]["db"]), torch.from_numpy(g[""]["qu"]), _gt(g[""]["gt"])
    for method in ("cosine", "l2"):
        d, i, r = u.get_top_k_recall([1, 3, 5], db, qu, gt, method=method)
        assert d.device.type == "cpu" and i.dtype == torch.int64 and d.dtype == torch.float32
        assert torch.equal(i, torch.from_numpy(g[method]["idx"])), method
        assert torch.allclose(d, torch.from_numpy(g[method]["dist"]), rtol=1e-4, atol=1e-5)
        assert np.allclose([r[k] for k in (1, 3, 5)], g[method]["recalls"])
    d, i, r = u.get_top_k_recall([2], db, qu[0], gt, norm_descs=False, use_percentage=False)
    assert torch.equal(i, torch.from_numpy(g["single"]["idx"])) and r[2] == g["single"]["recalls"][0]
    dn, inn, _ = u.get_top_k_recall([1, 3], db.numpy(), qu.numpy(), gt)
    assert isinstance(inn, np.ndarray) and np.array_equal(inn, g["cosine"]["idx"][:, :3])
    with pytest.raises(NotImplementedError):
        u.get_top_k_recall([1], db, qu, gt, method="hamming")     # utilities.py:444


@pytest.mark.parametrize("n_db,n_q,Dv,k", [(500, 33, 3072, 5), (2000, 100, 1024, 20), (64, 7, 130, 10), (3, 2, 64, 5)])
@pytest.mark.parametrize("method", ["cosine", "l2"])
def test_topk_vs_oracle(u, n_db, n_q, Dv, k, method):
    g = torch.Generator().manual_seed(n_db + k)
    db = torch.randn(n_db, Dv, generator=g)
    qu = db[torch.randint(0, n_db, (n_q,), generator=g)] + 0.5 * torch.randn(n_q, Dv, generator=g)
    dist, idx = u.top_k_search(db.cuda(), qu.cuda(), k, method)
    dist, idx = dist.cpu(), idx.cpu()
    kk = min(k, n_db)
    d64, i64 = ao.top_k(db, qu, kk + 1 if n_db > kk else kk, method, dtype=torch.float64)
    if k > n_db:
        assert bool((idx[:, n_db:] == -1).all())          # faiss pads with -1
    for q in range(n_q):
        gaps = (d64[q, 1:] - d64[q, :-1]).abs()
        amb = bool((gaps[:kk] < 1e-6).any()) if gaps.numel() else False
        if not amb:
            assert torch.equal(idx[q, :kk], i64[q, :kk]), (q, idx[q], i64[q])
    assert rel_inf(dist[:, :kk], d64[:, :kk]) < 1e-4


def test_topk_config3_shape_properties(u):
    """BASELINE config 3 shape, scaled to fit test time (2000 x 49152 DB, 64 queries, top-5):
    every query is a noisy copy of a known DB row -> rank-1 must be that row; scores sorted."""
    g = torch.Generator(device="cuda").manual_seed(7)
    db = torch.nn.functional.normalize(torch.randn(2000, 49152, device="cuda", generator=g), dim=1)
    src = torch.randint(0, 2000, (64,), device="cuda", generator=g)
    qu = db[src] + 0.1 * torch.nn.functional.normalize(torch.randn(64, 49152, device="cuda", generator=g), dim=1)
    dist, idx = u.top_k_search(db, qu, 5)
    assert torch.equal(idx[:, 0], src)
    assert bool((dist[:, :-1] >= dist[:, 1:]).all())
    ref = (torch.nn.functional.normalize(qu).double() @ db.double().T).topk(5, dim=1)
    assert torch.equal(idx, ref.indices) and rel_inf(dist.cpu(), ref.values.cpu()) < 1e-5


def _check_vs_fp64(db, qu, dist, idx, k):
    d64, i64 = ao.top_k(db.cpu(), qu.cpu(), k + 1, "cosine", dtype=torch.float64)
    dist, idx = dist.cpu(), idx.cpu()
    for q in range(qu.shape[0]):
        gaps = (d64[q, 1:] - d64[q, :-1]).abs()
        if not bool((gaps[:k] < 1e-6).any()):
            assert torch.equal(idx[q], i64[q, :k]), (q, idx[q], i64[q, :k])
    assert rel_inf(dist, d64[:, :k]) < 1e-4


def test_topk_coarse_pass_and_fallback(u):
    """The inner-product search on an fp16-pair index: hi-only pass of the wgmma GEMM (640 queries) + exact
    re-scoring of the candidates, and the device-gated 3-term fallback when a candidate list overflows (here: 400
    identical database rows next to the query -> 400 candidates > CAND_MAX; ties must still come out lowest index first)."""
    g = torch.Generator(device="cuda").manual_seed(5)
    db = torch.randn(4096, 256, device="cuda", generator=g)
    qu = db[torch.randint(0, 4096, (640,), device="cuda", generator=g)] + 0.7 * torch.randn(640, 256, device="cuda", generator=g)
    dist, idx = u.top_k_search(db, qu, 10)
    _check_vs_fp64(db, qu, dist, idx, 10)
    # clustered database: many near-equal scores around the k-th best
    centre = torch.randn(1, 256, device="cuda", generator=g)
    db2 = centre + 0.02 * torch.randn(3000, 256, device="cuda", generator=g)
    qu2 = centre + 0.02 * torch.randn(64, 256, device="cuda", generator=g)
    dist, idx = u.top_k_search(db2, qu2, 5)
    _check_vs_fp64(db2, qu2, dist, idx, 5)
    # overflow -> fallback
    db3 = db.clone()
    db3[100:500] = db3[100]
    qu3 = db3[100][None] + 0.05 * torch.randn(40, 256, device="cuda", generator=g)
    dist, idx = u.top_k_search(db3, qu3, 8)
    assert torch.equal(idx.cpu(), torch.arange(100, 108).expand(40, 8))
    assert bool((dist[:, :1] == dist[:, 1:]).all())
    # growth of a FlatIndex keeps what the coarse pass needs (per-row norms, header)
    ix = u.FlatIndex(256, "cosine", True, device="cuda")
    for c0 in range(0, 4096, 1000):
        ix.add(db[c0:c0 + 1000])
    d2, i2 = ix.search(qu, 10)
    d1, i1 = u.top_k_search(db, qu, 10)
    assert torch.equal(i1, i2) and torch.equal(d1, d2)
