"""The host schedule of the streamed k-means fit (VLAD.fit on host descriptors larger than the device), as pure
functions: the rounds must hand every chunk of the in-memory update its rows in row order, and the plan must pick
the in-memory fit whenever it fits and keep as many leading rounds resident as the budget allows."""
import pytest

from anyloc_b200 import utilities as u


def partition(R, chunks):
    """anyloc_kmeans_partition's rows_per for a given chunk count"""
    return -(-R // chunks)


@pytest.mark.parametrize("R,chunks", [(1000, 7), (257, 2), (300, 1), (64 * 300 - 5, 64), (10_001, 13)])
@pytest.mark.parametrize("P", [1, 7, 13, 10**9])
def test_rounds_cover_every_row_in_chunk_order(R, chunks, P):
    rows_per = partition(R, chunks)
    rounds = u._stream_rounds(R, chunks, rows_per, P)
    assert len(rounds) == -(-rows_per // min(P, rows_per))
    seen = {c: [] for c in range(chunks)}
    for pieces in rounds:
        assert len(pieces) == chunks
        full = pieces[0][1]
        assert 1 <= full <= P
        for c, (lo, m) in enumerate(pieces):
            # the round buffer layout anyloc_kmeans_accumulate_round reads: all pieces but the last are `full` rows
            assert m == full if c < chunks - 1 else 0 <= m <= full
            seen[c].extend(range(lo, lo + m))
    flat = []
    for c in range(chunks):
        assert seen[c] == list(range(c * rows_per, min(R, (c + 1) * rows_per)))       # row order within each chunk
        flat += seen[c]
    assert flat == list(range(R))                                                     # every row exactly once


def test_short_last_chunk():
    R, chunks = 4 * 100 + 37, 5                # rows_per 88, last chunk 85 rows
    rounds = u._stream_rounds(R, chunks, partition(R, chunks), 10)
    assert [p[-1][1] for p in rounds] == [10] * 8 + [5]
    assert [p[0][1] for p in rounds] == [10] * 8 + [8]


def ws_bytes(n):
    return 1000 + 12 * n


@pytest.mark.parametrize("copies", [1, 2])
def test_plan_selects_in_memory_when_it_fits(copies):
    R, D = 10_000, 64
    need = copies * R * 4 * D + ws_bytes(R)
    assert u._kmeans_plan(R, D, 8, partition(R, 8), need, copies, ws_bytes, 1 << 30) is None
    assert u._kmeans_plan(R, D, 8, partition(R, 8), need - 1, copies, ws_bytes, 1 << 30) is not None


@pytest.mark.parametrize("copies", [1, 2])
def test_plan_resident_rounds(copies):
    R, D, chunks = 10_000, 64, 8
    rows_per, row = partition(R, chunks), 4 * D
    stage = 50 * chunks * row                   # P = 50 -> 25 rounds of 400 rows
    rr = 50 * chunks
    fixed = ws_bytes(rr) + 4 * R + (1 + copies) * rr * row
    plan = lambda budget: u._kmeans_plan(R, D, chunks, rows_per, budget, copies, ws_bytes, stage)
    assert plan(0) == (50, 0)
    assert plan(fixed - 1) == (50, 0)
    assert plan(fixed + rr * row - 1) == (50, 0)
    assert plan(fixed + rr * row) == (50, 1)
    assert plan(fixed + 7 * rr * row + 5) == (50, 7)
    if copies == 2:                             # all rounds resident while the in-memory fit (two copies) does not fit
        assert plan(fixed + 25 * rr * row) == (50, 25)
        assert plan(2 * R * row + ws_bytes(R) - 1) == (50, 25)
    else:                                       # one copy: the in-memory fit needs less than all rounds plus buffers
        assert plan(fixed + 25 * rr * row) is None


def test_plan_piece_length():
    R, D, chunks = 10_000, 64, 8
    rows_per, row = partition(R, chunks), 4 * D
    plan = lambda stage: u._kmeans_plan(R, D, chunks, rows_per, 0, 2, ws_bytes, stage)[0]
    assert plan(0) == 1                          # a staging buffer below one row per chunk still moves one
    assert plan(chunks * row) == 1
    assert plan(13 * chunks * row + chunks * row - 1) == 13
    assert plan(1 << 40) == rows_per             # one round of whole chunks
