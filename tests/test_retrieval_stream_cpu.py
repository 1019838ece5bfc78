"""The host schedule of the streamed search (a FlatIndex over host rows larger than the device), as pure functions: the
plan must pick the resident index whenever it fits, keep the buffers of a streamed search inside the budget and the
staging buffer, and the pieces must cover every row once, in row order."""
import pytest

from anyloc_b200 import utilities as u


def index_bytes(n):                 # the shape of anyloc_index_bytes: two pair arrays + two per-row floats + header
    return 2 * 2 * 64 * n + 8 * n + 512


def ws_bytes(n, n_q):               # the shape of anyloc_index_search_workspace_bytes
    return 2 * 2 * 64 * n_q + 4 * n_q * n + 4096


D, NQ = 64, 100
ROW = 4 * D


def plan(n_db, budget, stage):
    return u._search_plan(n_db, D, NQ, budget, stage, index_bytes, ws_bytes)


def fixed(P):
    return u._stream_fixed_bytes(P, ROW, index_bytes, lambda n: ws_bytes(n, NQ))


def test_resident_when_it_fits():
    n = 10_000
    need = index_bytes(n) + ws_bytes(n, NQ)
    assert plan(n, need, 1 << 30) is None
    assert plan(n, need - 1, 1 << 30) is not None


@pytest.mark.parametrize("n_db", [10_000, 10_007, 1, 999])
@pytest.mark.parametrize("P_stage", [1, 37, 500, 10**6])
@pytest.mark.parametrize("extra", [0, 1, 3, 10**9])
def test_streamed_plan_stays_in_budget_and_staging(n_db, P_stage, extra):
    """budget = one piece's buffers plus `extra` pieces' worth: the pieces are the staging size (clipped to the
    database), `extra` of them stay resident (all, at most), and the total stays under the budget"""
    stage = P_stage * ROW + ROW - 1
    P0 = min(P_stage, n_db)
    n_pieces = -(-n_db // P0)
    budget = fixed(P0) + min(extra, n_pieces) * index_bytes(P0)
    if index_bytes(n_db) + ws_bytes(n_db, NQ) <= budget:
        assert plan(n_db, budget, stage) is None
        return
    P, r = plan(n_db, budget, stage)
    assert P == P0 and P * ROW <= stage                     # a piece fits the staging buffer
    assert r == min(extra, n_pieces)
    assert r * index_bytes(P) + fixed(P) <= budget


def test_piece_shrinks_to_the_budget():
    n_db, stage = 10_000, 2000 * ROW
    for budget in (fixed(1), fixed(7) + 5, fixed(1999), fixed(2000) - 1):
        P, r = plan(n_db, budget, stage)
        assert fixed(P) <= budget and (P == 2000 or fixed(P + 1) > budget) and r == 0
    assert plan(n_db, 0, stage) == (1, 0)                   # nothing fits: one row at a time
    assert plan(n_db, 0, 0) == (1, 0)                       # a staging buffer below one row still moves one


def test_resident_count_is_monotone():
    n_db, stage = 10_000, 500 * ROW
    prev = -1
    for extra in range(0, 21):
        P, r = plan(n_db, fixed(500) + extra * index_bytes(500) + index_bytes(500) // 2, stage)
        assert P == 500 and r == extra >= prev
        prev = r


def add_plan(ntotal, n, capacity, budget, stage=500 * ROW):
    held = index_bytes(capacity) if capacity else 0
    grow = max(ntotal + n, 2 * capacity if ntotal else 0)
    return u._add_plan(ntotal, n, capacity, held, grow, D, NQ, budget, stage, index_bytes, ws_bytes)


def test_add_plan_fresh_index_is_the_search_plan():
    for budget in (0, fixed(500), fixed(500) + 3 * index_bytes(500), index_bytes(10_000) + ws_bytes(10_000, NQ)):
        p = plan(10_000, budget, 500 * ROW)
        assert add_plan(0, 10_000, 0, budget) == (("resident", 10_000) if p is None else ("stream",) + p)


def test_add_plan_growth_peaks():
    """the old blob is held (outside the budget) while the new one is filled; the search then holds the new blob
    and its workspace, with the old one released"""
    old, total = 1000, 1500
    held, ws = index_bytes(old), ws_bytes(total, NQ)
    doubled, exact = index_bytes(2 * old), index_bytes(total)
    assert add_plan(old, 500, old, max(doubled, doubled + ws - held)) == ("resident", 2000)
    b = max(exact, exact + ws - held)
    assert b < max(doubled, doubled + ws - held)
    assert add_plan(old, 500, old, b) == ("resident", 1500)          # the doubled blob does not fit: exactly the rows
    s = add_plan(old, 500, old, b - 1)
    assert s[0] == "stream" and s[2] == 0 and fixed(s[1]) <= b - 1   # the kept blob counts as used
    assert add_plan(old, 200, 1500, ws_bytes(1200, NQ)) == ("resident", 1500)     # no growth: the workspace must fit
    s = add_plan(old, 200, 1500, ws_bytes(1200, NQ) - 1)
    assert s[0] == "stream" and s[2] == 0 and fixed(s[1]) <= ws_bytes(1200, NQ) - 1


@pytest.mark.parametrize("Dv,chunk", [(49152, 5461), (49152, 1000), (196608, 1365), (3072, 87381)])
def test_chunked_adds_never_exceed_the_device(Dv, chunk):
    """An 80 GB card fed host chunks: the budget of every add is the card less what the index already holds, as
    _device_budget sees it.  Every resident growth (old + new blob, then new blob + workspace) and the streamed
    buffers beside a kept blob must fit the card, and the index must end up streaming."""
    from anyloc_b200 import _lib
    lib = _lib.load()
    ib = lambda n: lib.anyloc_index_bytes(n, Dv, 1)
    wb = lambda n, q: lib.anyloc_index_search_workspace_bytes(n, q, Dv, 1)
    card = 79 << 30                                  # 80 GB less _device_budget's margin
    ntotal = cap = held = 0
    P = None
    for _ in range(-(-(160 << 30) // (chunk * 4 * Dv))):           # 160 GB of rows in all
        grow = max(ntotal + chunk, 2 * cap if ntotal else 0)
        p = u._add_plan(ntotal, chunk, cap, held, grow, Dv, u._SEARCH_Q_CHUNK, card - held, u._STAGE_BYTES, ib, wb)
        if p[0] == "resident":
            if ntotal + chunk > cap:
                assert held + ib(p[1]) <= card               # both blobs during the copy
                held, cap = ib(p[1]), p[1]
            assert held + wb(ntotal + chunk, u._SEARCH_Q_CHUNK) <= card
        else:
            P = p[1]
            assert held + u._stream_fixed_bytes(P, 4 * Dv, ib, lambda n: wb(n, u._SEARCH_Q_CHUNK)) <= card
            assert P * 4 * Dv <= u._STAGE_BYTES
            break
        ntotal += chunk
    assert P is not None, "160 GB of rows never streamed"


@pytest.mark.parametrize("n_db,n_res,P",[(10, 0, 3), (10, 10, 3), (10, 4, 3), (10, 6, 3), (1, 0, 5), (1000, 999, 7),
                                          (1000, 1000, 1000), (12, 12, 4), (12, 5, 100)])
def test_pieces_cover_every_row_in_order(n_db, n_res, P):
    pieces = u._search_pieces(n_db, n_res, P)
    rows = []
    for r0, m, resident in pieces:
        assert 1 <= m <= P
        assert resident == (r0 < n_res) and (not resident or r0 + m <= n_res)
        rows += range(r0, r0 + m)
    assert rows == list(range(n_db))                        # every row exactly once, in row order
    assert [p[2] for p in pieces] == sorted((p[2] for p in pieces), reverse=True)    # resident pieces first
