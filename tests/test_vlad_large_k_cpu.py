"""Host side of hard VLAD and the k-means fit at any vocabulary size, with no GPU: the route predicate VLAD uses to
send a call to anyloc_vlad_generate_sorted (only where the shared-memory routes refuse), the sorted route's workspace,
the switch to the cluster-tiled k-means update and the streamed fit's plan at large K."""
import pytest

from anyloc_b200 import _lib, utilities as u
from tests.test_vlad_engine_gpu import accumulate_route

ROUTE = {"accumulate3": 0, "accumulate2": 1, "error": _lib.VLAD_ROUTE_SORTED}


def a256(n):
    return -(-n // 256) * 256


@pytest.mark.parametrize("B,N,D,K", [
    (32, 529, 1536, 32), (32, 1369, 1024, 128), (1, 300, 64, 1000), (1, 1369, 1024, 1024),      # accumulate3
    (2, 3942, 1536, 32), (2, 5329, 1536, 32), (2, 3000, 1024, 200),                             # accumulate2
    (1, 4000, 128, 256), (1, 2000, 64, 1000), (2, 5329, 1536, 256), (1, 1369, 1024, 2048),       # sorted
    (8, 3942, 1536, 256), (1, 2000, 1024, 1024), (1, 2815, 128, 201), (1, 2816, 128, 201)])
def test_route_predicate(lib, B, N, D, K):
    """the ABI's route agrees with the dispatch read off vlad_generate_impl, shape for shape"""
    assert lib.anyloc_vlad_generate_route(B, N, D, K) == ROUTE[accumulate_route(N, D, K)]


def test_route_edges(lib):
    """accumulate3's limit at K = 201 is 2815 rows, at K = 256 2739 rows; above K = 200 nothing else runs there"""
    for K, n_max in ((201, 2815), (256, 2739), (1000, 1420)):
        assert lib.anyloc_vlad_generate_route(1, n_max, 128, K) == 0
        assert lib.anyloc_vlad_generate_route(1, n_max + 1, 128, K) == _lib.VLAD_ROUTE_SORTED
    assert lib.anyloc_vlad_generate_route(1, 5000, 128, 200) == 1


@pytest.mark.parametrize("B,N,D,K", [(1, 4000, 128, 256), (1, 2000, 64, 1000), (2, 5329, 1536, 256),
                                     (1, 1369, 1024, 2048), (32, 529, 1536, 32)])
def test_sorted_workspace_bytes(lib, B, N, D, K):
    """anyloc_generate's buffers without the tickets, then the per-image tables, each 256-byte aligned"""
    R, ns = B * N, -(-D // 128)
    hard = [4 * R, 4 * R, 4 * B * K * ns, 4 * K * D, 4 * K * D, 4 * K, 4 * K, 4 * R * K]
    tables = [8 * R, 4 * R, 4 * B * 8 * K] + [4 * B * (K + 1)] * 3 + [4 * B * (N // 64 + K + 1),
                                                                      4 * B * (2 * (N // 64) + 2) * D]
    assert lib.anyloc_vlad_sorted_workspace_bytes(B, N, D, K) == sum(a256(n) for n in hard + tables)
    assert lib.anyloc_vlad_sorted_workspace_bytes(B, N, D, K) > lib.anyloc_vlad_workspace_bytes(B, N, D, K)


def test_tiled_switch():
    assert not u._kmeans_tiled(436) and u._kmeans_tiled(437)
    assert (436 * 128 + 436) * 4 <= 220 * 1024 < (437 * 128 + 437) * 4


def test_stream_plan_large_k():
    """K = 1024, D = 1536, 64 chunks: the partial sums alone are 403 MB; the streamed fit counts them whatever the
    round, and raises MemoryError naming its bytes when they do not fit"""
    R, D, K, chunks = 2_000_000, 1536, 1024, 64
    rows_per = -(-R // chunks)
    psums = chunks * K * D * 4
    assert psums == 402_653_184

    def ws_bytes(n):                                  # assignment buffers of an n-row pass + the update's partials
        return 4 * n * (K + 2) + 8 * K * D + psums

    stage = 1 << 30
    P = stage // (chunks * 4 * D)
    need = u._kmeans_stream_bytes(R, D, chunks, P, 2, ws_bytes)
    rr = chunks * P
    assert need == ws_bytes(rr) + 4 * R + 3 * rr * 4 * D
    assert u._kmeans_fit_plan(R, D, chunks, rows_per, 0, need, 2, ws_bytes, stage) == (P, 0)
    with pytest.raises(MemoryError, match=str(need)):
        u._kmeans_fit_plan(R, D, chunks, rows_per, 0, need - 1, 2, ws_bytes, stage)
    assert u._kmeans_fit_plan(R, D, chunks, rows_per, need + 5 * rr * 4 * D, need + 5 * rr * 4 * D, 2, ws_bytes,
                              stage) == (P, 5)
    assert u._kmeans_fit_plan(1000, D, 4, 250, 1 << 40, 1 << 40, 2, ws_bytes, stage) is None
