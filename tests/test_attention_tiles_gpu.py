"""The 2-byte attention kernel works on 128-query tiles of two 64-row halves, one per consumer warpgroup; a half whose
rows all lie at or beyond T does no work.  Sequence lengths around those edges (one half active or both, the second
half with one row, several key blocks behind a partial tile, the c2 and c1 lengths), fp16 pairs against fp64 under
the bound of test_attention_edges_gpu, bf16 and single fp16 against fp64 under the bounds of test_bf16_kernels_gpu
and test_f16x1_kernels_gpu (the bf16 pairs' tile edges are test_bf16x3_edges_gpu's).  The fp16-pair
and tf32 outputs, hi and lo, are written inside NaN canaries that must stay intact."""
import pytest
import torch

from tests.test_attention_edges_gpu import check, structured, to_qkv

pytestmark = pytest.mark.gpu

TS = [65, 128, 129, 191, 192, 193, 257, 530]


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


@pytest.mark.parametrize("kind", ["flat", "dominant_last"])
@pytest.mark.parametrize("T", TS)
def test_f16_pairs_at_tile_edges(L, T, kind):
    B, heads = 3, 2
    q, k, v = structured(kind, B, heads, T, seed=T * 7 + len(kind))
    check(L, to_qkv(q, k, v), heads, "f16", "tc3", what=f"{kind} T={T}")


@pytest.mark.parametrize("T", TS)
def test_bf16_at_tile_edges(L, T):
    from tests.test_bf16_kernels_gpu import test_attention_against_fp64
    test_attention_against_fp64(L, T)


@pytest.mark.parametrize("T", TS)
def test_f16x1_at_tile_edges(L, T):
    from tests.test_f16x1_kernels_gpu import test_attention_against_fp64
    test_attention_against_fp64(L, T)


@pytest.mark.parametrize("pair", ["f16", "tf32"])
@pytest.mark.parametrize("T", TS)
def test_pairs_write_nothing_outside_the_output(L, T, pair):
    """the pair outputs (hi and lo) inside NaN canaries: every row below T written, nothing around them"""
    from tests.test_attention_varlen_gpu import LEAD, canaries_intact, canary_buf, rows_of
    from tests.util import dptr, split_tf32
    B, heads = 3, 2
    D = 64 * heads
    q_hi, q_lo = split_tf32(L, to_qkv(*structured("flat", B, heads, T, seed=T)).reshape(B * T, 3 * D))
    dt = torch.float16 if pair == "f16" else torch.float32
    o_hi, o_lo = canary_buf(B * T, D, dt), canary_buf(B * T, D, dt)
    L.check(L.load().anyloc_attention(dptr(q_hi), dptr(q_lo), B, T, D, heads, dptr(o_hi, LEAD), dptr(o_lo, LEAD),
                                      L.PAIR[pair], L.ENGINE["tc3"], L.stream_ptr()), "attention")
    torch.cuda.synchronize()
    for buf in (o_hi, o_lo):
        assert canaries_intact(buf, B * T, D, [0], [B * T]), (pair, T)
    assert bool(torch.isfinite(rows_of(o_hi, B * T, D)).all() and torch.isfinite(rows_of(o_lo, B * T, D)).all())
