"""Several VLAD vocabularies fitted in one pass (fit_vocabularies) against one VLAD.fit per vocabulary, bit for bit:
the shared assignment (anyloc_vlad_assign_multi) against anyloc_vlad_assign per vocabulary, the fused k-means sums
(anyloc_kmeans_accumulate_round_multi) against anyloc_kmeans_accumulate_round per vocabulary, and the whole fit --
centres, desc_dim, kmeans.centroids, c_centers.pt and the numpy RNG state -- in memory, partly resident and fully
streamed.  Every comparison is torch.equal."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from oracle import dinov2_restated as dr
from tests import dropin_harness as H
from tests.util import ROOT

pytestmark = pytest.mark.gpu


def rows(R, D, seed, centres=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, D, generator=g)
    if centres is not None:                         # some rows equal to centres: exact scores at the tie points
        n = min(R, centres.shape[0])
        x[:n] = centres[:n]
    return x


def centre_sets(Ks, D, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for K in Ks:
        c = torch.randn(K, D, generator=g)
        if K >= 4:
            c[K // 2] = c[1]                         # a duplicated centre row: an exact tie, lowest index wins
        out.append(c)
    return out


# (Ks, D, R): K in {1, 8, 32, 256, 437, 1000}; D in {384, 1024, 1536, 2560}; R in {1, 255, 256, 10 000}.  R < 256 and
# D > 2048 take the FFMA kernel, like anyloc_vlad_assign; 60 000 rows at sum K = 1725 span two coarse slices.
ASSIGN = [([8], 384, 10_000), ([1, 8], 384, 256), ([32, 256, 8, 1], 1024, 10_000), ([437, 32], 1536, 10_000),
          ([1000, 8], 384, 255), ([256, 32, 8, 1], 2560, 10_000), ([8, 32], 1536, 1), ([1000, 437, 256, 32], 384, 60_000),
          ([256, 1], 1536, 256), ([32, 8], 2560, 255)]


@pytest.mark.parametrize("mode", ["cosine", "euclidean"])
@pytest.mark.parametrize("Ks,D,R", ASSIGN)
def test_assign_multi_equals_assign(cuda, Ks, D, R, mode):
    cs = [c.to(cuda) for c in centre_sets(Ks, D, seed=D + R)]
    x = rows(R, D, seed=R, centres=cs[0].cpu()).to(cuda)
    if mode == "cosine":
        x[-1] = 3.0 * cs[-1][0]                      # a scaled centre: its cosine ties with the centre's own
    got = u._assign_multi(x, cs, mode)
    assert got.shape == (len(Ks), R) and got.dtype == torch.int32
    for v, c in enumerate(cs):
        want = u._KMeans(Ks[v], mode=mode)._assign(x, c)
        assert torch.equal(got[v], want), (v, Ks[v])
    if Ks[0] >= 4 and R > Ks[0] // 2:
        assert got[0][Ks[0] // 2] == 1               # a row equal to a duplicated centre: the lower index


def test_assign_multi_refusals(cuda):
    lib = _lib.load()
    x = torch.zeros(300, 64, device=cuda)
    c = torch.zeros(4, 64, device=cuda)
    labels = torch.empty(2, 300, dtype=torch.int32, device=cuda)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda)
    ptrs = (C.c_void_p * 2)(c.data_ptr(), c.data_ptr())
    for Ks, D, mode in [((4, 0), 64, 0), ((4, 4), 62, 0), ((4, 4), 64, 7)]:
        rc = lib.anyloc_vlad_assign_multi(_lib.ptr(x), 300, D, 2, ptrs, (C.c_int * 2)(*Ks), mode, _lib.ptr(labels),
                                          _lib.ptr(ws), ws.numel(), None)
        assert rc == _lib.ERR["arg"]
    rc = lib.anyloc_vlad_assign_multi(_lib.ptr(x), 300, 64, 2, ptrs, (C.c_int * 2)(4, 4), 0, _lib.ptr(labels),
                                      _lib.ptr(ws), 1000, None)
    assert rc == _lib.ERR["workspace"]


def run_rounds(x, labels, Ks, fused, rounds_at):
    """the k-means sums of every vocabulary over the rounds of `rounds_at` = (round_rows, piece) -> workspaces"""
    R, D = x.shape
    lib = _lib.load()
    ws = [torch.full((lib.anyloc_kmeans_round_workspace_bytes(R, D, K),), 0x7f, dtype=torch.uint8, device=x.device)
          for K in Ks]
    for j, (x_r, l_r, rr, piece) in enumerate(rounds_at):
        if fused:
            u._accumulate_round_multi(x_r, l_r, Ks, ws, R, rr, piece, int(j > 0))
        else:
            for v, K in enumerate(Ks):
                u._accumulate_round(x_r, l_r[v], R, rr, piece, K, int(j > 0), ws[v])
    return ws


def round_views(x, labels, P):
    """_stream_rounds' round buffers of rows x and labels [V, R] for P rows per chunk"""
    R, D = x.shape
    chunks, rows_per = u._kmeans_partition(R, D)
    out = []
    for pcs in u._stream_rounds(R, chunks, rows_per, P):
        idx = torch.cat([torch.arange(lo, lo + m) for lo, m in pcs]).to(x.device)
        out.append((x[idx].contiguous(), labels[:, idx].contiguous(), idx.numel(), pcs[0][1]))
    return out


@pytest.mark.parametrize("Ks,D,R,P", [([1, 8, 32, 256], 384, 20_000, 10**9), ([256, 128, 64, 32], 1536, 30_001, 97),
                                      ([437, 8, 2], 256, 5_000, 13), ([3, 5], 100 * 4, 257, 1)])
def test_fused_accumulate_equals_per_vocabulary(cuda, Ks, D, R, P):
    x = rows(R, D, seed=R).to(cuda)
    g = torch.Generator().manual_seed(D)
    labels = torch.stack([torch.randint(-1, max(1, K // 2), (R,), generator=g, dtype=torch.int32) for K in Ks])
    labels = labels.to(cuda)                         # clusters K // 2 .. K - 1 stay empty; -1 rows are skipped
    rounds_at = round_views(x, labels, P)
    a = run_rounds(x, labels, Ks, True, rounds_at)
    b = run_rounds(x, labels, Ks, False, rounds_at)
    for v, K in enumerate(Ks):
        assert torch.equal(a[v], b[v]), (v, K)
        c = torch.randn(K, D, device=cuda)
        outs = []
        for ws in (a[v], b[v]):
            nxt, err = torch.empty_like(c), torch.zeros(1, device=cuda)
            u._finalize(c, R, nxt, err, ws)
            outs.append((nxt, err))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        if K > 1:
            assert (outs[0][0][K - 1] == 0).all()   # an empty cluster's centre is 0


def test_fused_accumulate_refuses_tiled_k(cuda):
    lib = _lib.load()
    x = torch.zeros(300, 128, device=cuda)
    labels = torch.zeros(300, dtype=torch.int32, device=cuda)
    ws = torch.empty(lib.anyloc_kmeans_round_workspace_bytes(300, 128, 437), dtype=torch.uint8, device=cuda)
    rc = lib.anyloc_kmeans_accumulate_round_multi(_lib.ptr(x), 1, (C.c_void_p * 1)(labels.data_ptr()),
                                                  (C.c_int * 1)(437), 300, 300, 300, 128, 0,
                                                  (C.c_void_p * 1)(ws.data_ptr()), (C.c_size_t * 1)(ws.numel()), None)
    assert rc == _lib.ERR["arg"]


# ------------------------------------------------------------------ end to end
def clustered(R, D, K, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn(K, D, generator=g, dtype=torch.float64)
    x = centres[torch.randint(0, K, (R,), generator=g)] + 0.6 * torch.randn(R, D, generator=g, dtype=torch.float64)
    return x.to(dtype)


def state(vlads, dirs):
    out = []
    for v, d in zip(vlads, dirs):
        f = None if d is None else torch.load(os.path.join(d, "c_centers.pt"))
        out.append((v.c_centers, v.kmeans.centroids, v.desc_dim, f))
    return out


def fit_both(tmp_path, X, specs, cached=None, **kw):
    """specs: (K, uses a cache dir) per member; cached: member whose directory already holds centres.  -> the
    (state, RNG state) of sequential VLAD.fit and of fit_vocabularies from np.random.seed(7)"""
    res = []
    for arm in ("seq", "multi"):
        dirs = [str(tmp_path / arm / f"m{i}") if c else None for i, (K, c) in enumerate(specs)]
        vl = [u.VLAD(K, cache_dir=d, **kw) for (K, _), d in zip(specs, dirs)]
        if cached is not None:
            torch.save(torch.arange(specs[cached][0] * 4, dtype=torch.float32).reshape(-1, 4) / 7,
                       os.path.join(dirs[cached], "c_centers.pt"))
        np.random.seed(7)
        if arm == "seq":
            for v in vl:
                v.fit(X)
        else:
            u.fit_vocabularies(vl, X)
        res.append((state(vl, dirs), np.random.get_state()))
    return res


def check_same(res):
    (s0, r0), (s1, r1) = res
    for a, b in zip(s0, s1):
        assert a[0].device == b[0].device and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        assert a[2] == b[2]
        assert (a[3] is None) == (b[3] is None) and (a[3] is None or torch.equal(a[3], b[3]))
    assert r0[0] == r1[0] and np.array_equal(r0[1], r1[1]) and r0[2:] == r1[2:]


class Spy:
    """counts the passes of the shared fit and the members of each, and records the plan it took"""

    def __init__(self, m):
        self.active, self.plans = [], []
        am, ls = u._assign_multi, u._lloyd_streamed

        def assign_multi(x, cs, mode):
            self.active.append(len(cs))
            return am(x, cs, mode)

        def lloyd_streamed(kms, X, normalize, plan, dev):
            self.plans.append(plan)
            return ls(kms, X, normalize, plan, dev)
        m.setattr(u, "_assign_multi", assign_multi)
        m.setattr(u, "_lloyd_streamed", lloyd_streamed)


@pytest.mark.parametrize("kind", ["numpy", "cpu", "cuda"])
def test_in_memory_inputs(cuda, tmp_path, monkeypatch, kind):
    X = clustered(6000, 384, 16, seed=1)
    X = {"numpy": X.double().numpy(), "cpu": X, "cuda": X.to(cuda)}[kind]
    spy = Spy(monkeypatch)
    res = fit_both(tmp_path, X, [(2, True), (256, False), (16, True)])
    check_same(res)
    assert not spy.plans and spy.active[0] == 3 and min(spy.active) < 3      # members converge at different passes
    assert res[1][0][0][0].is_cuda == (kind == "cuda")


def test_cached_member_large_k_and_shared_cache_dir(cuda, tmp_path):
    X = clustered(5000, 128, 8, seed=2)
    check_same(fit_both(tmp_path, X, [(8, True), (500, False), (4, True), (12, True)], cached=2))
    # two members writing one directory: the second loads what the first wrote, as its own fit would
    res = []
    for arm in ("seq", "multi"):
        d = str(tmp_path / f"shared_{arm}")
        vl = [u.VLAD(6, cache_dir=d), u.VLAD(9, cache_dir=d), u.VLAD(3)]
        np.random.seed(11)
        if arm == "seq":
            for v in vl:
                v.fit(X)
        else:
            u.fit_vocabularies(vl, X)
        res.append((state(vl, [d, d, None]), np.random.get_state()))
    check_same(res)


def test_no_norm_euclidean(cuda, tmp_path):
    X = clustered(4000, 256, 10, seed=3)
    check_same(fit_both(tmp_path, X, [(10, False), (3, True), (40, False)], norm_descs=False, dist_mode="euclidean"))


@pytest.mark.parametrize("resident", ["zero", "some"])
def test_streamed(cuda, tmp_path, monkeypatch, resident):
    X = clustered(9001, 384, 16, seed=4)
    R, D = X.shape
    Ks = [2, 256, 16, 500]
    with torch.cuda.device(cuda):
        chunks, rows_per = u._kmeans_partition(R, D)
    P, row = 17, 4 * D
    lib = _lib.load()
    arr = (C.c_int * len(Ks))(*Ks)
    ws = u._fit_ws_bytes(lambda n: lib.anyloc_vlad_assign_multi_workspace_bytes(n, D, len(Ks), arr),
                         sum(lib.anyloc_kmeans_round_workspace_bytes(R, D, K) for K in Ks), len(Ks))
    fixed = u._kmeans_stream_bytes(R, D, chunks, P, 2, ws)
    monkeypatch.setattr(u, "_STAGE_BYTES", P * chunks * row)
    budget = 0 if resident == "zero" else fixed + 3 * chunks * P * row
    monkeypatch.setattr(u, "_device_budget", lambda dev: budget)
    spy = Spy(monkeypatch)
    check_same(fit_both(tmp_path, X, [(K, i % 2 == 0) for i, K in enumerate(Ks)]))
    n_rounds = -(-rows_per // P)
    assert spy.plans and spy.plans[0][0] == P
    kept = spy.plans[0][1]
    assert kept == 0 if resident == "zero" else 0 < kept < n_rounds
    assert spy.active[0] == len(Ks) and min(spy.active) < len(Ks)


def test_streamed_round_crosses_link_once(cuda, monkeypatch):
    """with four members active, each staged round is copied once per iteration"""
    X = clustered(3001, 128, 8, seed=5)
    R, D = X.shape
    with torch.cuda.device(cuda):
        chunks, rows_per = u._kmeans_partition(R, D)
    monkeypatch.setattr(u, "_STAGE_BYTES", 7 * chunks * 4 * D)
    monkeypatch.setattr(u, "_device_budget", lambda dev: 0)
    staged = []
    st = u._RoundFeed._stage
    monkeypatch.setattr(u._RoundFeed, "_stage", lambda self: staged.append(len(self.staged)) or st(self))
    iters = []
    fin = u._finalize_multi
    monkeypatch.setattr(u, "_finalize_multi", lambda c, R, ws: iters.append(len(c)) or fin(c, R, ws))
    vl = [u.VLAD(K) for K in (3, 8, 16, 4)]
    np.random.seed(3)
    u.fit_vocabularies(vl, X)
    n_rounds = -(-rows_per // 7)
    # one staging call per round taken, and the first one before the loop
    assert len(iters) > 1 and len(staged) == len(iters) * n_rounds + 1


def test_refusals(cuda):
    a, b = u.VLAD(4), u.VLAD(8, norm_descs=False)
    with pytest.raises(ValueError, match="no VLAD"):
        u.fit_vocabularies([], torch.zeros(10, 8))
    with pytest.raises(ValueError, match=r"members 0 and 2"):
        u.fit_vocabularies([a, u.VLAD(2), a], torch.zeros(10, 8))
    with pytest.raises(ValueError, match=r"members \[1\]"):
        u.fit_vocabularies([a, b], torch.zeros(10, 8))
    with pytest.raises(ValueError, match=r"members \[2\]"):
        u.fit_vocabularies([a, u.VLAD(3), u.VLAD(3, dist_mode="euclidean")], torch.zeros(10, 8))


def test_dropin_replay(cuda, tmp_path):
    """the driver's calling pattern (tests/test_dropin_gpu.py) through the drop-in module, once per K with one cache
    directory per K and the RNG running on from one seed: every c_centers.pt it writes equals the centres
    fit_vocabularies gives for that K from the same seed and the same database rows"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_anyloc_shim_utilities_fitv",
                                                  os.path.join(ROOT, "anyloc_b200", "dropin", "utilities.py"))
    shim = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(shim)
    ds = H.SyntheticVprDataset()
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=3), seed=3).state_dict()
    dino = shim.DinoV2ExtractFeatures("dinov2_vits14", 2, "value", device=cuda, weights=sd)
    descs = []
    for i in range(ds.database_num):
        img = ds[i][0].to(cuda)
        c, h, w = img.shape
        hn, wn = (h // 14) * 14, (w // 14) * 14
        top, left = int(round((h - hn) / 2.0)), int(round((w - wn) / 2.0))
        descs.append(dino(img[None, :, top:top + hn, left:left + wn]).cpu())
    flat = torch.cat(descs).reshape(-1, descs[0].shape[2])
    Ks = [32, 16, 8, 4]
    np.random.seed(42)
    for K in Ks:
        vlad = shim.VLAD(K, None, cache_dir=str(tmp_path / f"k{K}"))
        vlad.fit(flat)
    np.random.seed(42)
    vl = [shim.VLAD(K, None) for K in Ks]
    shim.fit_vocabularies(vl, flat)
    for K, v in zip(Ks, vl):
        assert torch.equal(torch.load(str(tmp_path / f"k{K}" / "c_centers.pt")), v.c_centers)
