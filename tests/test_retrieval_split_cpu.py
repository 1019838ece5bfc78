"""The split index's arguments, its opt-in and its C ABI without a GPU: FlatIndex(placement=...) validation,
$ANYLOC_B200_INDEX_PLACEMENT, the device-blob size and the entries' argument checks."""
import re

import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from tests.util import ROOT


def test_placement_default_and_validation():
    assert not u.FlatIndex(256)._split
    assert u.FlatIndex(256, placement="split")._split
    with pytest.raises(ValueError, match="'device' or 'split'"):
        u.FlatIndex(256, placement="host")


@pytest.mark.parametrize("kw", [dict(method="l2"), dict(norm_descs=False), dict(d=260), dict(d=250)])
def test_split_needs_an_fp16_pair_inner_product_index(kw):
    args = dict(d=256, method="cosine", norm_descs=True) | kw
    with pytest.raises(ValueError, match=r"method='cosine', norm_descs=True and d % 8 == 0"):
        u.FlatIndex(args.pop("d"), **args, placement="split")


def test_placement_positional_arguments_unchanged():
    with pytest.raises(TypeError):
        u.FlatIndex(256, "cosine", True, 0, None, "split")


def test_env_opt_in(monkeypatch):
    monkeypatch.delenv("ANYLOC_B200_INDEX_PLACEMENT", raising=False)
    assert u.resolve_placement() == "device"
    assert u.resolve_placement("split") == "split"
    monkeypatch.setenv("ANYLOC_B200_INDEX_PLACEMENT", "split")
    assert u.resolve_placement() == "split"
    assert u.resolve_placement("device") == "device"           # the argument wins
    monkeypatch.setenv("ANYLOC_B200_INDEX_PLACEMENT", "hbm")
    with pytest.raises(ValueError, match="'device' or 'split'"):
        u.resolve_placement()
    # checked before any device work: a bad opt-in fails the same way on a machine without a GPU
    with pytest.raises(ValueError, match="'device' or 'split'"):
        u.get_top_k_recall([1], torch.zeros(4, 8), torch.zeros(1, 8), [[0]])
    with pytest.raises(ValueError, match="'device' or 'split'"):
        u.top_k_search(torch.zeros(4, 8), torch.zeros(1, 8), 1)


@pytest.mark.parametrize("cap,Dv", [(1, 8), (1000, 256), (100_000, 49152), (100_000, 393216)])
def test_device_blob_is_half_the_index(cap, Dv):
    lib = _lib.load()
    full, split = lib.anyloc_index_bytes(cap, Dv, 1), lib.anyloc_index_split_bytes(cap, Dv)
    hi = -(-cap * Dv * 2 // 256) * 256
    assert split == full - hi                      # the resident layout less its lo region
    assert split <= full // 2 + 4 * cap + 512


def test_entries_check_their_arguments():
    lib = _lib.load()
    fake = 256                                     # never dereferenced: every call below fails its checks first
    assert lib.anyloc_index_split_init(fake, 1 << 20, 10, 12, None) == _lib.ERR["arg"]
    assert "multiple of 8" in _lib.last_error()
    assert lib.anyloc_index_split_add(fake, 1 << 20, 10, fake, 5, fake, 6, 256, None) == _lib.ERR["arg"]
    assert lib.anyloc_index_split_piece(fake, 1 << 20, 10, fake, 1 << 20, 10, fake, 5, 6, 256, None) == _lib.ERR["arg"]
    assert lib.anyloc_index_split_copy(fake, 1 << 20, 10, fake, 1 << 20, 5, 6, 256, None) == _lib.ERR["arg"]
    counts = (_lib.C.c_int64 * 2)(7, 7)
    assert lib.anyloc_index_split_search(fake, 1 << 20, 10, 11, fake, 40, 256, 5, fake, 1 << 20, counts,
                                         None) == _lib.ERR["arg"]         # n_db > capacity
    assert list(counts) == [-1, 0]
    # n_unique above what n_q candidate lists can hold, and k above the coarse route's
    assert lib.anyloc_index_split_rescore(fake, 1 << 20, 2000, fake, 2000, 40, 256, 5, fake, 1 << 20, 40 * 256 + 1,
                                          fake, 1 << 20, fake, fake, None) == _lib.ERR["arg"]
    assert lib.anyloc_index_split_rescore(fake, 1 << 20, 2000, fake, 2000, 40, 256, 65, fake, 1 << 20, 10,
                                          fake, 1 << 20, fake, fake, None) == _lib.ERR["arg"]
    assert lib.anyloc_index_split_init(fake, 100, 10, 256, None) == _lib.ERR["workspace"]


def test_header_documents_every_split_entry():
    text = open(f"{ROOT}/include/anyloc_b200.h").read()
    names = set(re.findall(r"\b(anyloc_index_split_\w+)\(", text))
    assert names == {"anyloc_index_split_bytes", "anyloc_index_split_init", "anyloc_index_split_copy",
                     "anyloc_index_split_add", "anyloc_index_split_search_workspace_bytes",
                     "anyloc_index_split_stage_bytes", "anyloc_index_split_search", "anyloc_index_split_rescore",
                     "anyloc_index_split_piece"}
    assert names <= set(_lib.EXPORTS)


def test_stage_and_workspace_sizes():
    lib = _lib.load()
    assert lib.anyloc_index_split_stage_bytes(10558, 49152) == 2 * 10558 * 49152 * 2       # hi and lo of each row
    assert lib.anyloc_index_split_stage_bytes(0, 256) == 0
    # the search workspace, then one slot per row and one row per candidate-list entry
    assert (lib.anyloc_index_split_search_workspace_bytes(100_000, 1000, 49152) ==
            lib.anyloc_index_search_workspace_bytes(100_000, 1000, 49152, 1) + 400_128 + 1000 * 256 * 4)   # 256-aligned
