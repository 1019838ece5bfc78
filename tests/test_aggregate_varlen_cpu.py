"""The packed list route of pool_descriptors and VLAD.generate_multi without a GPU: the row table built from a list,
the zero-copy detection of consecutive views of one buffer (and every layout it must refuse, which is packed by one
copy with the same rows), and the refusal of both entry points without a device."""
import pytest
import torch

from anyloc_b200 import _lib
from anyloc_b200 import utilities as u


def _buf(R=20, D=8, seed=0):
    return torch.randn(R, D, generator=torch.Generator().manual_seed(seed))


def test_table_from_list():
    items = [torch.randn(5, 8), torch.randn(0, 8), torch.randn(1, 8), torch.randn(7, 8)]
    feats, row0, lens = u._pack_list(items, "cpu")
    assert lens == [5, 0, 1, 7] and row0 == [0, 5, 5, 6]
    assert feats.shape == (13, 8) and feats.dtype == torch.float32 and feats.is_contiguous()
    for q, r, n in zip(items, row0, lens):
        assert torch.equal(feats[r:r + n], q)


def test_table_from_views_of_one_buffer():
    buf = _buf()
    items = list(buf.split([4, 0, 9, 1, 6]))
    view = u._packed_rows(items)
    assert view is not None and view.data_ptr() == buf.data_ptr() and view.shape == (20, 8)
    feats, row0, lens = u._pack_list(items, "cpu")
    assert feats.data_ptr() == buf.data_ptr()            # no copy
    assert row0 == [0, 4, 4, 13, 14] and lens == [4, 0, 9, 1, 6]


def test_views_inside_a_larger_buffer():
    # ext(list) of a *_reg model or with use_cls returns views that start past row 0 of its output
    buf = _buf(24)
    items = [buf[4:9], buf[9:17]]
    view = u._packed_rows(items)
    assert view is not None and view.data_ptr() == buf[4].data_ptr() and view.shape == (13, 8)
    assert torch.equal(view, buf[4:17])


@pytest.mark.parametrize("case", ["overlap", "gap", "order", "strided", "transposed", "fp64", "fp16", "two_buffers",
                                  "misaligned"])
def test_refused_layouts_pack_by_copy(case):
    buf = _buf(40)
    if case == "overlap":
        items = [buf[0:6], buf[4:10]]
    elif case == "gap":
        items = [buf[0:6], buf[7:10]]
    elif case == "order":
        items = [buf[6:10], buf[0:6]]
    elif case == "strided":
        items = [buf[0:12:2], buf[12:20]]
    elif case == "transposed":
        sq = _buf(8, 8, seed=1)
        items = [sq.t(), _buf(3, 8, seed=2)]
    elif case == "fp64":
        items = [buf[0:6].double(), buf[6:10].double()]
    elif case == "fp16":
        items = [buf[0:6].half(), buf[6:10].half()]
    elif case == "two_buffers":
        items = [buf[0:6], _buf(4, 8, seed=3)]
    else:
        flat = _buf(41).flatten()[1:321].view(40, 8)       # rows start 4 bytes past a 16-byte boundary
        items = [flat[0:6], flat[6:10]]
    assert u._packed_rows(items) is None
    feats, row0, lens = u._pack_list(items, "cpu")
    assert feats.dtype == torch.float32 and feats.is_contiguous() and feats.data_ptr() % 16 == 0
    assert feats.data_ptr() != items[0].data_ptr()
    for q, r, n in zip(items, row0, lens):
        assert torch.equal(feats[r:r + n], q.float())
    assert sum(lens) == feats.shape[0]


def test_no_device_raises():
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    items = [torch.randn(5, 8), torch.randn(3, 8)]
    with pytest.raises(_lib.AnylocError):
        u.pool_descriptors(items, "gem")
    v = u.VLAD(2)
    v.kmeans = u._KMeans(2, mode="cosine")
    v.kmeans.centroids = v.c_centers = torch.randn(2, 8)
    v.desc_dim = 8
    with pytest.raises(_lib.AnylocError):
        v.generate_multi(items)


def test_pool_list_checks_method_and_emptiness():
    with pytest.raises(NotImplementedError):
        u.pool_descriptors([torch.randn(3, 8)], "median")
    if torch.cuda.is_available():
        with pytest.raises(ValueError):
            u.pool_descriptors([], "gem")
