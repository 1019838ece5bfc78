"""The 2-byte attention kernel works on 128-query tiles of two 64-row halves, one per consumer warpgroup; a half whose
rows all lie at or beyond T does no work.  Sequence lengths around those edges (one half active or both, the second
half with one row, several key blocks behind a partial tile, the c2 and c1 lengths), fp16 pairs against fp64 under
the bound of test_attention_edges_gpu, and bf16 against fp64 under the bound of test_bf16_kernels_gpu."""
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
