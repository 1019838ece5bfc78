"""The split index (FlatIndex(placement="split"): hi, |y|^2, dn and the header on the device, the fp16 lo halves in
page-locked host memory) against the resident index over the same rows.  (dist, idx) must be torch.equal on every
route: the coarse route, which reads only the candidates' lo rows from host memory, and the exact route over pieces,
which also answers a batch whose candidate lists overflow."""
import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from tests.test_retrieval_engine_gpu import make_rows

pytestmark = pytest.mark.gpu


def resident(db, qu, k):
    ix = u.FlatIndex(db.shape[1], device="cuda")
    ix.add(db)
    return ix.search(qu, k)


def same(a, b):
    return torch.equal(a[0].cpu(), b[0].cpu()) and torch.equal(a[1].cpu(), b[1].cpu())


class Spy:
    """counts the pieces the exact route searches (one continuation call per piece and query chunk)"""

    def __init__(self, m):
        self.calls = 0
        lib = _lib.load()
        cont = lib.anyloc_index_search_continue

        def wrapped(*a):
            self.calls += 1
            return cont(*a)
        m.setattr(lib, "anyloc_index_search_continue", wrapped)


def check_blob(ix):
    """the device part is half the resident index, plus half of |y|^2 and dn (4 bytes a row) and a header"""
    lib = _lib.load()
    assert ix._blob.numel() == lib.anyloc_index_split_bytes(ix.capacity, ix.dp)
    assert ix._blob.numel() <= lib.anyloc_index_bytes(ix.capacity, ix.dp, 1) // 2 + 4 * ix.capacity + 512
    lo = ix._lo.t
    assert lo.is_pinned() and lo.dtype == torch.float16 and lo.shape == (ix.capacity, ix.dp)
    assert ix._lo.nbytes == ix.capacity * ix.dp * 2                  # locked to the byte, not rounded up


# (family, n_db, n_q, d, k, rows per piece of the exact route)
CASES = [(fam, 2100, 64, 256, 10, 300) for fam in ["random", "positive", "spiky", "near_dup"]] + [
    ("random", 2100, 64, 256, 1, 300),             # coarse, k = 1
    ("random", 2100, 64, 256, 64, 300),            # coarse, k = 64
    ("clustered", 2100, 40, 256, 65, 300),         # exact, tensor cores (k > 64), 7 pieces
    ("random", 2100, 1, 256, 5, 300),              # exact, SIMT (n_q < 32)
    ("near_dup", 2100, 31, 256, 5, 700),
    ("positive", 2100, 32, 256, 5, 300),           # the smallest coarse batch
    ("random", 900, 40, 256, 5, 250),              # below 1024 rows: exact
    ("random", 1500, 40, 3072, 5, 400),
    ("spiky", 1500, 31, 3072, 64, 400),
    ("near_dup", 1500, 40, 3072, 65, 1500),        # exact, one piece
    ("random", 1100, 33, 49152, 5, 200),
    ("spiky", 1100, 33, 49152, 1, 200),
    ("near_dup", 1100, 8, 49152, 5, 300),
    ("positive", 1100, 40, 49152, 65, 250),
    ("random", 1100, 4100, 256, 5, 300),           # a coarse chunk of 4096 queries, then an exact one of 4
    ("clustered", 1100, 4100, 256, 65, 500),
]


@pytest.mark.parametrize("fam,n_db,n_q,d,k,P", CASES)
def test_split_equals_resident(cuda, monkeypatch, fam, n_db, n_q, d, k, P):
    db, qu = make_rows(fam, n_db, n_q, d, seed=n_db + d + k + n_q)
    want = resident(db, qu, k)
    monkeypatch.setattr(u, "_STAGE_BYTES", P * 4 * d)
    spy = Spy(monkeypatch)
    ix = u.FlatIndex(d, placement="split", device="cuda")
    ix.add(db.cpu())
    check_blob(ix)
    got = ix.search(qu, k)
    assert same(got, want)
    ix._split_stage = lambda nbytes, dev: None                       # the re-scoring reads lo from host memory
    assert same(ix.search(qu, k), want)
    exact = [not (k <= 64 and n_db >= 1024 and c >= 32) for c in (min(4096, n_q - i) for i in range(0, n_q, 4096))]
    assert spy.calls == 2 * -(-n_db // P) * sum(exact)       # every piece once per query chunk left to the exact route
    assert len(ix._split_counts) == len(exact) - sum(exact)
    for uniq, total in ix._split_counts:
        assert 0 < uniq <= min(total, n_db) and total <= n_q * 256
    assert got[0].is_cuda and got[1].is_cuda


def test_overflow_takes_the_exact_route(cuda, monkeypatch):
    """test_topk_gpu's overflow database: 400 identical rows next to the queries overflow the candidate lists.  The
    resident index answers by its device-gated 3-term fallback, the split one by the exact route over pieces"""
    g = torch.Generator(device="cuda").manual_seed(5)
    db = torch.randn(4096, 256, device="cuda", generator=g)
    db[100:500] = db[100]
    qu = db[100][None] + 0.05 * torch.randn(40, 256, device="cuda", generator=g)
    want = resident(db, qu, 8)
    monkeypatch.setattr(u, "_STAGE_BYTES", 1000 * 4 * 256)
    spy = Spy(monkeypatch)
    ix = u.FlatIndex(256, placement="split", device="cuda")
    ix.add(db)
    got = ix.search(qu, 8)
    assert spy.calls == 5                          # the coarse pass overflowed: 5 pieces of 1000 rows
    assert same(got, want)
    assert torch.equal(got[1].cpu(), torch.arange(100, 108).expand(40, 8))


def test_nonfinite_rows_and_queries(cuda):
    db, qu = make_rows("random", 2100, 40, 256, seed=9)
    db[700, 3] = float("nan")
    db[1500, 0] = float("inf")
    qu[5, 2] = float("nan")
    for k in (10, 65):
        want = resident(db, qu, k)
        ix = u.FlatIndex(256, placement="split", device="cuda")
        ix.add(db.cpu())
        got = ix.search(qu, k)
        assert same(got, want)
        assert not bool(torch.isin(got[1].cpu(), torch.tensor([700, 1500])).any())
        assert bool((got[1][5] == -1).all()) and bool((got[0][5] == -float("inf")).all())


def test_chunked_adds_growth_and_reset(cuda):
    """host and device rows added in chunks: the device blob and the pinned lo array grow by doubling and keep the
    rows already added; reset forgets the rows and keeps the allocation"""
    db, qu = make_rows("clustered", 3000, 48, 512, seed=11)
    want = resident(db, qu, 10)
    ix = u.FlatIndex(512, placement="split", device="cuda")
    caps = []
    for c in range(0, 3000, 250):
        rows = db[c:c + 250]
        ix.add(rows if c % 500 else rows.cpu().numpy())
        caps.append(ix.capacity)
    assert caps == [250, 500, 1000, 1000, 2000, 2000, 2000, 2000, 4000, 4000, 4000, 4000], caps
    check_blob(ix)
    assert same(ix.search(qu, 10), want)
    assert same(ix.search(qu[:5], 10), resident(db, qu[:5], 10))
    ix.reset()
    assert ix.ntotal == 0 and ix.capacity == 4000
    ix.add(db[:1500].cpu())
    ix.add(db[1500:])
    assert ix.capacity == 4000
    assert same(ix.search(qu, 10), want)
    with pytest.raises(ValueError):
        ix.add_at(db[:10], 0)
    with pytest.raises(ValueError):
        ix.search(qu, 4097)


def test_device_part_must_fit(cuda, monkeypatch):
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: 1 << 20)
    ix = u.FlatIndex(1024, placement="split", device="cuda")
    with pytest.raises(MemoryError, match="does not fit"):
        ix.add(torch.randn(600, 1024))
    ix.add(torch.randn(100, 1024))                 # 100 rows of hi: 200 KB


@pytest.mark.parametrize("as_numpy", [True, False])
def test_get_top_k_recall_split(cuda, monkeypatch, as_numpy):
    db, qu = make_rows("clustered", 1800, 50, 512, seed=13)
    rng = np.random.default_rng(0)
    gt = [rng.choice(1800, size=5, replace=False) for _ in range(50)]
    h_db, h_qu = db.cpu(), qu.cpu()
    if as_numpy:
        h_db, h_qu = h_db.numpy(), h_qu.numpy()
    want = u.get_top_k_recall([1, 5, 10], db, qu, gt)
    made = []
    real = u.FlatIndex.__init__

    def spy_init(self, *a, **kw):
        real(self, *a, **kw)
        made.append(self._split)
    monkeypatch.setattr(u.FlatIndex, "__init__", spy_init)
    d, i = u.top_k_search(db, qu, 10, placement="split")
    monkeypatch.setenv("ANYLOC_B200_INDEX_PLACEMENT", "split")
    got = u.get_top_k_recall([1, 5, 10], h_db, h_qu, gt)
    got_dev = u.get_top_k_recall([1, 5, 10], db, qu, gt)
    d_env, i_env = u.top_k_search(h_db if not as_numpy else db, qu, 10)
    assert made == [True, True, True, True]
    assert same((d_env, i_env), (want[0], want[1]))
    host = lambda t: t.cpu().numpy() if torch.is_tensor(t) else t
    for g in (got, got_dev):
        assert np.array_equal(host(g[0]), host(want[0]))
        assert np.array_equal(host(g[1]), host(want[1]))
        assert g[2] == want[2]
    assert type(got[0]) == type(h_db)
    assert same((d, i), (want[0], want[1]))


def test_growth_takes_what_fits(cuda, monkeypatch):
    """chunked adds without a reserved capacity: when the doubled device part does not fit beside the old one, the
    largest part that fits is taken; the pinned lo array follows it exactly and the old one is unlocked"""
    lib = _lib.load()
    db, qu = make_rows("random", 1500, 40, 256, seed=21)
    want = resident(db, qu, 5)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    B = lib.anyloc_index_split_bytes(1000, 256) + lib.anyloc_index_split_bytes(1800, 256) + 2048
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: B - (torch.cuda.memory_allocated() - base))
    ix = u.FlatIndex(256, placement="split", device="cuda")
    ix.add(db[:1000].cpu())
    assert ix.capacity == 1000
    ix.add(db[1000:].cpu())                         # 2000 rows do not fit beside the 1000-row part: about 1800 do
    assert 1500 <= ix.capacity < 2000
    check_blob(ix)
    monkeypatch.undo()
    assert same(ix.search(qu, 5), want)
    with monkeypatch.context() as m:
        m.setattr(u, "_device_budget", lambda dev, release_cache=True: lib.anyloc_index_split_bytes(1600, 256))
        with pytest.raises(MemoryError, match="does not fit"):
            ix.add(db[:400].cpu())                  # 1900 rows: not even those fit
