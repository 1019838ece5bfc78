"""The streamed search (a FlatIndex over host rows larger than the device) against the resident one.  The device budget
and the staging size are monkeypatched so that small databases stream in pieces of P rows with r of them kept on the
device; (dist, idx) must equal the resident search's bit for bit, except where the coarse route's 3-term fallback
fires, which answers per piece and is held to the fp64 bound of tests/test_retrieval_engine_gpu.py."""
import os

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from oracle import dinov2_restated as dr
from tests import dropin_harness as H
from tests.test_retrieval_engine_gpu import IP, L2, check, make_rows, query_sections, reference, route_of
from tests.util import ROOT, load_cases

pytestmark = pytest.mark.gpu


def byte_fns(dp, norm):
    lib = _lib.load()
    return (lambda n: lib.anyloc_index_bytes(n, dp, norm),
            lambda n, q=u._SEARCH_Q_CHUNK: lib.anyloc_index_search_workspace_bytes(n, q, dp, norm))


def force(m, n_db, d, norm, P, r, extra=0):
    """make an index of n_db host rows of dimension d stream in pieces of P rows, r of them resident; extra: device
    bytes the index already holds (they count as free)"""
    dp = d + (-d) % 4
    ib, wb = byte_fns(dp, int(norm))
    budget = u._stream_fixed_bytes(P, 4 * dp, ib, wb) + r * ib(P) - extra
    m.setattr(u, "_STAGE_BYTES", P * 4 * dp)
    m.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    assert u._search_plan(n_db, dp, u._SEARCH_Q_CHUNK, budget + extra, P * 4 * dp, ib, wb) == (P, r)
    return budget


class Spy:
    """counts the continuation calls and reads the overflow flag each coarse piece left in the search workspace"""

    def __init__(self, m):
        self.calls, self.flags, self.cands = 0, [], []
        lib = _lib.load()
        cont = lib.anyloc_index_search_continue

        def wrapped(*a):
            rc = cont(*a)
            self.calls += 1
            n_rows, n_total, n_q, dp, k, metric, norm = a[4], a[6], a[8], a[9], a[10], a[11], a[12]
            flag, cand = 0, None
            if route_of(n_total, n_q, dp, k, metric, norm)[0] == "coarse":     # the only route that writes the flag
                ws = _lib.workspaces._bufs[(torch.cuda.current_device(), "topk")]
                torch.cuda.synchronize()
                w = query_sections(ws, n_rows, n_q, dp, norm)
                flag, cand = int(w["flag"][0]), float(w["cand_n"].float().mean())
            self.flags.append(flag)
            self.cands.append(cand)
            return rc
        m.setattr(lib, "anyloc_index_search_continue", wrapped)


def resident(db, qu, k, method, norm):
    ix = u.FlatIndex(db.shape[1], method, norm, device="cuda")
    ix.add(db)                                        # device rows: never streams
    assert ix._stream is None
    return ix.search(qu, k)


def streamed(m, db, qu, k, method, norm, P, r):
    force(m, db.shape[0], db.shape[1], norm, P, r)
    spy = Spy(m)
    ix = u.FlatIndex(db.shape[1], method, norm, device="cuda")
    ix.add(db.cpu())
    assert ix._stream is not None and ix._stream["P"] == P and ix.capacity == min(P * r, db.shape[0])
    d, i = ix.search(qu, k)
    n_pieces = -(-db.shape[0] // P)
    assert spy.calls == n_pieces * -(-qu.shape[0] // u._SEARCH_Q_CHUNK)
    return d, i, spy


def same(a, b):
    return torch.equal(a[0].cpu(), b[0].cpu()) and torch.equal(a[1].cpu(), b[1].cpu())


# (family, n_db, n_q, d, k, method, norm, P, r)
CASES = [(fam, 2100, 64, 256, 10, "cosine", True, 300, 2) for fam in ["random", "positive", "spiky", "near_dup",
                                                                      "clustered"]] + [
    ("random", 2100, 64, 256, 1, "cosine", True, 300, 0),          # coarse, k = 1, nothing resident
    ("random", 2100, 64, 256, 64, "cosine", True, 299, 7),         # coarse, k = 64, all pieces but one resident
    ("clustered", 2100, 40, 256, 65, "cosine", True, 300, 3),      # exact tensor-core route (k > 64)
    ("random", 2100, 8, 256, 5, "cosine", True, 300, 3),           # exact SIMT route (n_q < 32)
    ("near_dup", 2100, 40, 256, 5, "l2", True, 300, 2),            # L2, tensor cores
    ("clustered", 2100, 8, 256, 64, "l2", True, 256, 0),           # L2, SIMT
    ("random", 2100, 40, 256, 5, "cosine", False, 300, 1),         # tf32 pairs (raw rows)
    ("spiky", 2100, 8, 258, 5, "cosine", False, 300, 0),           # tf32 pairs, SIMT, d padded to 260
    ("clustered", 1500, 40, 258, 5, "cosine", True, 400, 1),       # normalised tf32 pairs (Dv % 8 != 0)
    ("random", 900, 40, 256, 10, "cosine", True, 250, 1),          # below 1024 rows: the exact route throughout
    ("random", 1500, 40, 3072, 5, "cosine", True, 400, 0),
    ("clustered", 1500, 8, 3072, 5, "l2", True, 400, 1),
    ("random", 1100, 33, 49152, 5, "cosine", True, 200, 2),
    ("near_dup", 1100, 33, 49152, 5, "cosine", True, 250, 0),
]


@pytest.mark.parametrize("fam,n_db,n_q,d,k,method,norm,P,r", CASES)
def test_streamed_equals_resident(cuda, monkeypatch, fam, n_db, n_q, d, k, method, norm, P, r):
    db, qu = make_rows(fam, n_db, n_q, d, seed=n_db + d + k + P, raw=not norm)
    want = resident(db, qu, k, method, norm)
    with monkeypatch.context() as m:
        d1, i1, spy = streamed(m, db, qu, k, method, norm, P, r)
    assert not any(spy.flags[j] for j in range(len(spy.flags))), "the coarse route fell back to the 3-term product"
    assert same((d1, i1), want)
    metric = IP if method == "cosine" else L2
    ref, B = reference(db, qu, int(norm), metric)
    check(d1, i1, ref, B, metric)


def test_threshold_keeps_the_coarse_route(cuda, monkeypatch):
    """random rows: no piece of the streamed search overflows its candidate lists where the resident search does not.
    The running k-th exact score is what bounds them: with tau alone every 128-row piece would keep at least k = 32
    candidates per query, while about k * 128 / 4096 = 1 row of a late piece belongs to the final top-32"""
    db, qu = make_rows("random", 4096, 128, 1024, seed=3)
    ix = u.FlatIndex(1024, "cosine", True, device="cuda")
    ix.add(db)
    want = ix.search(qu, 32)
    ws = _lib.workspaces._bufs[(torch.cuda.current_device(), "topk")]
    assert int(query_sections(ws, 4096, 128, 1024, 1)["flag"][0]) == 0
    with monkeypatch.context() as m:
        d1, i1, spy = streamed(m, db, qu, 32, "cosine", True, 128, 0)       # 32 pieces of 128 rows
    assert spy.flags == [0] * 32
    assert spy.cands[0] >= 32 and max(spy.cands[16:]) < 8, spy.cands
    assert same((d1, i1), want)


def test_fallback_stays_in_the_bound(cuda, monkeypatch):
    """test_topk_gpu's overflow database: 400 identical rows next to the queries overflow the candidate lists"""
    g = torch.Generator(device="cuda").manual_seed(5)
    db = torch.randn(4096, 256, device="cuda", generator=g)
    db[100:500] = db[100]
    qu = db[100][None] + 0.05 * torch.randn(40, 256, device="cuda", generator=g)
    with monkeypatch.context() as m:
        d1, i1, spy = streamed(m, db, qu, 8, "cosine", True, 512, 1)
    assert any(spy.flags)
    ref, B = reference(db, qu, 1, IP)
    check(d1, i1, ref, B, IP, dup_groups=[torch.arange(100, 500)])
    assert torch.equal(i1.cpu(), torch.arange(100, 108).expand(40, 8))


@pytest.mark.parametrize("method", ["cosine", "l2"])
def test_nonfinite_rows_and_queries(cuda, monkeypatch, method):
    db, qu = make_rows("random", 2100, 40, 256, seed=9)
    db[700, 3] = float("nan")                          # inside the third piece
    db[1500, 0] = float("inf")                         # inside a streamed piece
    db[50, 7] = float("nan")                           # inside a resident piece
    qu[5, 2] = float("nan")
    want = resident(db, qu, 10, method, True)
    with monkeypatch.context() as m:
        d1, i1, _ = streamed(m, db, qu, 10, method, True, 300, 1)
    assert same((d1, i1), want)
    assert not bool(torch.isin(i1.cpu(), torch.tensor([50, 700, 1500])).any())
    pad = float("inf") if method == "l2" else -float("inf")
    assert bool((i1[5] == -1).all()) and bool((d1[5] == pad).all())


def test_chunked_add_crosses_into_streaming_and_reset(cuda, monkeypatch):
    """Host chunks of 250 rows on a device of B bytes: the budget of every add is B less what has been allocated since,
    so it shrinks as the index's blob grows.  The blob doubles while that fits (old and new blob during the copy,
    then the new blob and a search workspace), and the index streams once neither the doubled nor an exact blob
    fits.  The device memory allocated while adding never exceeds B (plus one chunk's rows on their way in)."""
    Dv = 1024
    db, qu = make_rows("clustered", 3000, 48, Dv, seed=11)
    want = resident(db, qu, 10, "cosine", True)
    h = db.cpu()
    ib, wb = byte_fns(Dv, 1)
    chunk_bytes = 250 * Dv * 4
    with monkeypatch.context() as m:
        torch.cuda.synchronize()
        base, B = torch.cuda.memory_allocated(), ib(1200) + wb(1200)
        m.setattr(u, "_device_budget", lambda dev, release_cache=True: B - (torch.cuda.memory_allocated() - base))
        m.setattr(u, "_STAGE_BYTES", 350 * 4 * Dv)
        ix = u.FlatIndex(Dv, "cosine", True, device="cuda")
        torch.cuda.reset_peak_memory_stats()
        caps = []
        for c in range(0, 3000, 250):
            ix.add(h[c:c + 250].numpy() if c % 500 else h[c:c + 250])
            caps.append((ix.capacity, ix._stream is not None))
        assert torch.cuda.max_memory_allocated() - base <= B + chunk_bytes, caps
        # 250 -> 500 -> 1000 rows doubling; at 1250 rows neither 2000 nor 1250 fits beside the workspace: streams
        assert caps == [(250, False), (500, False), (1000, False), (1000, False)] + [(1000, True)] * 8, caps
        assert ix.ntotal == 3000 and ix._stream["P"] == 350
        assert same(ix.search(qu, 10), want)
        ix.reset()
        assert ix._stream is None and ix.ntotal == 0
        kept = ix.capacity
        torch.cuda.reset_peak_memory_stats()
        ix.add(h)                                      # the whole database at once: streams beside the kept blob
        assert ix._stream is not None and ix.ntotal == 3000 and ix.capacity == kept
        assert torch.cuda.max_memory_allocated() - base <= B + kept * Dv * 4      # the kept rows on their way in
        assert same(ix.search(qu, 10), want)
        with pytest.raises(ValueError):
            ix.add_at(db[:10], 0)
        with pytest.raises(ValueError):
            ix.search(qu, 4097)


def test_device_rows_join_a_streamed_index(cuda, monkeypatch):
    """device rows added to an index that already streams go to its host copy, as documented, and the answer stays
    the resident one"""
    db, qu = make_rows("random", 2100, 40, 256, seed=17)
    want = resident(db, qu, 10, "cosine", True)
    with monkeypatch.context() as m:
        force(m, 1500, 256, True, 300, 1)
        ix = u.FlatIndex(256, "cosine", True, device="cuda")
        ix.add(db[:1500].cpu())
        assert ix._stream is not None and ix.capacity == 300
        ix.add(db[1500:])
        assert ix.ntotal == 2100 and ix._stream["host"][-1][0] == 1500
        assert same(ix.search(qu, 10), want)


@pytest.mark.parametrize("as_numpy", [True, False])
def test_get_top_k_recall_streamed(cuda, monkeypatch, as_numpy):
    db, qu = make_rows("clustered", 1800, 50, 512, seed=13)
    rng = np.random.default_rng(0)
    gt = [rng.choice(1800, size=5, replace=False) for _ in range(50)]
    h_db, h_qu = db.cpu(), qu.cpu()
    if as_numpy:
        h_db, h_qu = h_db.numpy(), h_qu.numpy()
    want = u.get_top_k_recall([1, 5, 10], db, qu, gt)
    with monkeypatch.context() as m:
        force(m, 1800, 512, True, 256, 2)
        spy = Spy(m)
        got = u.get_top_k_recall([1, 5, 10], h_db, h_qu, gt)
    assert spy.calls == 8
    assert type(got[0]) == type(h_db)
    assert np.array_equal(np.asarray(got[0]), want[0].cpu().numpy())
    assert np.array_equal(np.asarray(got[1]), want[1].cpu().numpy())
    assert got[2] == want[2]


def test_device_database_never_streams(cuda, monkeypatch):
    db, qu = make_rows("random", 1200, 40, 256, seed=15)
    m = monkeypatch
    m.setattr(u, "_device_budget", lambda dev, release_cache=True: 0)
    m.setattr(u, "_STAGE_BYTES", 100 * 4 * 256)
    spy = Spy(m)
    ix = u.FlatIndex(256, "cosine", True, device="cuda")
    ix.add(db)
    assert ix._stream is None
    d0, i0 = ix.search(qu, 5)
    d1, i1 = u.top_k_search(db, qu, 5)
    d2, i2, _ = u.get_top_k_recall([1, 5], db, qu, [np.array([0])] * 40)
    assert spy.calls == 0
    assert same((d0, i0), (d1, i1)) and same((d0, i0), (d2, i2))
    ix2 = u.FlatIndex(256, "cosine", True, device="cuda")
    ix2.add(db.cpu())                                  # the same rows from the host stream under this budget
    assert ix2._stream is not None
    assert same(ix2.search(qu, 5), (d0, i0))


def test_dropin_replay_streamed(cuda, monkeypatch, tmp_path):
    """tests/test_dropin_gpu.py's driver loop with the retrieval forced to stream (pieces of 3 rows, none resident):
    the committed golden top-k and recalls of the reference run"""
    import importlib.util
    g = load_cases("build_vlads.npz")["hard"]
    spec = importlib.util.spec_from_file_location("_anyloc_shim_utilities_search_stream",
                                                  os.path.join(ROOT, "anyloc_b200", "dropin", "utilities.py"))
    shim = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(shim)
    ds = H.SyntheticVprDataset()
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=3), seed=3).state_dict()
    dino = shim.DinoV2ExtractFeatures("dinov2_vits14", 2, "value", device=cuda, weights=sd)

    def extract(indices):
        descs = []
        for i in indices:
            img = ds[i][0].to(cuda)
            c, h, w = img.shape
            hn, wn = (h // 14) * 14, (w // 14) * 14
            top, left = int(round((h - hn) / 2.0)), int(round((w - wn) / 2.0))
            descs.append(dino(img[None, :, top:top + hn, left:left + wn]).cpu())
        return torch.cat(descs)
    num_db = ds.database_num
    full_db = extract(np.arange(0, num_db))
    vlad = shim.VLAD(4, None, cache_dir=str(tmp_path / "cache"))
    np.random.seed(42)
    vlad.fit(full_db.reshape(-1, full_db.shape[2]))
    db_vlads = vlad.generate_multi(full_db, ds.get_image_relpaths(np.arange(0, num_db)))
    qu_vlads = vlad.generate_multi(extract(np.arange(num_db, len(ds))), ds.get_image_relpaths(np.arange(num_db, len(ds))))
    with monkeypatch.context() as m:
        force(m, db_vlads.shape[0], db_vlads.shape[1], True, 3, 0)
        spy = Spy(m)
        dists, indices, recalls = shim.get_top_k_recall([1, 2, 3], db_vlads, qu_vlads, ds.soft_positives_per_query)
    assert spy.calls == -(-db_vlads.shape[0] // 3)
    assert np.array_equal(indices.numpy(), g["idx"])
    assert np.allclose(dists.numpy(), g["dist"], atol=1e-5)
    assert [recalls[1], recalls[2], recalls[3]] == list(g["recalls"])
