"""The packed list route of VLAD.generate_multi and pool_descriptors on the GPU.

Every packed output is compared bit for bit (torch.equal) with the padded call it replaces -- VLAD._run on the
zero-padded [B, max len, D] batch with n_valid, anyloc_pool with n_valid -- labels and soft assignments included:
hard VLAD on each accumulation route (accumulate3, accumulate2, sorted), soft VLAD and the three pool modes, with empty
and single-row items, one item and 300 items.  Packed buffers hold the images in shuffled order with NaN rows between
them and after the last, so a descriptor that read outside its own rows would be NaN or differ.  The list pooling is
also checked against fp64 (the tolerance of tests/test_pool_gpu.py), the chain preprocess_images(list) -> ext(list) ->
generate_multi / pool_descriptors is checked to hand the extractor's own buffer to the kernels, and the table and
pointer refusals are checked to return ANYLOC_ERR_ARG without a launch."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import anyloc_oracle as ao
from tests.util import rel_inf

pytestmark = pytest.mark.gpu
NAN = float("nan")


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    return _lib


def make_vlad(u, K, D, mode="hard", seed=0, dist="cosine"):
    g = torch.Generator().manual_seed(seed)
    v = u.VLAD(K, vlad_mode=mode, dist_mode=dist)
    v.kmeans = u._KMeans(K, mode=dist)
    v.kmeans.centroids = v.c_centers = torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1)
    v.desc_dim = D
    return v


def make_items(lens, D, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, D, generator=g) for n in lens]


def padded(items, D):
    n_max = max(max(q.shape[0] for q in items), 1)
    x = torch.zeros(len(items), n_max, D)
    for i, q in enumerate(items):
        x[i, :q.shape[0]] = q
    return x.cuda(), torch.tensor([q.shape[0] for q in items], dtype=torch.int32, device="cuda")


def scattered(items, D, seed):
    """the items in shuffled order inside one buffer, 0-3 NaN rows before each and 2 after the last -> (buf, row0)"""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(items))
    gaps = rng.integers(0, 4, len(items))
    rows, row0, r = [], [0] * len(items), 0
    for j, i in enumerate(order):
        rows.append(torch.full((int(gaps[j]), D), NAN)); r += int(gaps[j])
        row0[i] = r
        rows.append(items[i]); r += items[i].shape[0]
    rows.append(torch.full((2, D), NAN))
    return torch.cat(rows).cuda(), row0


def check_vlad(u, v, items, D, seed):
    dev = torch.device("cuda", 0)
    x, n_valid = padded(items, D)
    ref, ref_lab = v._run(x, n_valid, dev, want_labels=True)
    lens = [q.shape[0] for q in items]
    # consecutive, and scattered with NaN rows around every image
    feats, row0, _ = u._pack_list([q.cuda() for q in items], dev)
    for buf, r0 in ((feats, row0), scattered(items, D, seed)):
        out, lab = v._run_varlen(buf, r0, lens, dev, want_labels=True)
        assert torch.equal(out, ref)
        assert not torch.isnan(out).any()
        inside = torch.zeros(buf.shape[0], dtype=torch.bool, device=dev)
        for i, (r, n) in enumerate(zip(r0, lens)):
            assert torch.equal(lab[r:r + n], ref_lab[i, :n])
            inside[r:r + n] = True
        if v.vlad_mode == "hard":
            assert bool((lab[~inside] == -1).all())
        else:
            assert bool((lab[~inside] == 0).all())
    return ref


def route(L, B, N, D, K):
    return L.load().anyloc_vlad_generate_route(B, N, D, K)


@pytest.mark.parametrize("K,D,lens,want", [
    (32, 384, [517, 0, 1, 233, 600, 64, 65], 0),             # accumulate3
    (32, 128, [5000, 17, 0, 4096], 1),                       # accumulate2: 5000 rows exceed its 100 KB
    (256, 384, [3000, 1, 0, 1777], 2),                       # sorted: K = 256 at 3000 rows
    (8, 64, [300], 0),                                       # one item
    (8, 64, [1, 1, 1], 0),                                   # single rows, fewer than the coarse GEMM's 256
])
def test_hard_packed_equals_padded(u, L, K, D, lens, want):
    assert route(L, len(lens), max(lens), D, K) == want
    v = make_vlad(u, K, D, seed=K + D)
    check_vlad(u, v, make_items(lens, D, seed=len(lens)), D, seed=K)


def test_hard_euclidean_and_flags(u, L):
    v = make_vlad(u, 16, 256, dist="euclidean", seed=3)
    v.intra_norm, v.norm_descs = False, False
    check_vlad(u, v, make_items([40, 0, 700, 3], 256, seed=4), 256, seed=5)


def test_hard_300_items(u, L):
    rng = np.random.default_rng(7)
    lens = [int(n) for n in rng.integers(0, 40, 300)]
    lens[5] = 0
    lens[9] = 1
    v = make_vlad(u, 8, 64, seed=8)
    check_vlad(u, v, make_items(lens, 64, seed=9), 64, seed=10)


@pytest.mark.parametrize("K,D,lens", [(32, 384, [517, 0, 1, 233, 600]), (64, 128, [1]), (8, 64, None)])
def test_soft_packed_equals_padded(u, K, D, lens):
    if lens is None:
        lens = [int(n) for n in np.random.default_rng(11).integers(0, 30, 300)]
    v = make_vlad(u, K, D, mode="soft", seed=K)
    check_vlad(u, v, make_items(lens, D, seed=12), D, seed=13)


def test_packed_equals_each_images_own_generate(u):
    # accumulate3 (and the sorted route) sum in an order of the image's own rows, so where the list and each image
    # alone take accumulate3 and the coarse-pass assignment (>= 256 rows) a list's descriptors are also the per-image
    # generate's; the soft route's sums never depend on the batch
    for mode in ("hard", "soft"):
        v = make_vlad(u, 32, 384, mode=mode, seed=14)
        items = [q.cuda() for q in make_items([300, 256, 999, 517], 384, seed=15)]
        out = v.generate_multi(items)
        for i, q in enumerate(items):
            assert torch.equal(out[i], v.generate(q))


def pool_padded(L, items, D, mode, p=3.0, use_abs=False):
    x, n_valid = padded(items, D)
    out = torch.empty(len(items), D, device="cuda")
    L.check(L.load().anyloc_pool(L.ptr(x), L.ptr(n_valid), len(items), x.shape[1], D, mode, float(p), int(use_abs),
                                 L.ptr(out), L.stream_ptr()), "anyloc_pool")
    return out


def pool_packed(L, buf, row0, lens, D, mode, p=3.0, use_abs=False):
    r0 = torch.tensor(row0, dtype=torch.int64, device="cuda")
    ln = torch.tensor(lens, dtype=torch.int32, device="cuda")
    out = torch.empty(len(lens), D, device="cuda")
    L.check(L.load().anyloc_pool_varlen(L.ptr(buf), buf.shape[0], L.ptr(r0), L.ptr(ln), len(lens), D, mode, float(p),
                                        int(use_abs), L.ptr(out), L.stream_ptr()), "anyloc_pool_varlen")
    return out


@pytest.mark.parametrize("lens,D", [([529, 0, 1, 1369, 7], 1536), ([1], 36), (None, 388)])
def test_pool_packed_equals_padded(u, L, lens, D):
    if lens is None:
        lens = [int(n) for n in np.random.default_rng(16).integers(0, 20, 300)]
    items = make_items(lens, D, seed=17)
    for mode, p, use_abs in ((0, 3.0, False), (1, 3.0, False), (2, 3.0, False), (2, 2.5, True)):
        ref = pool_padded(L, items, D, mode, p, use_abs)
        for buf, r0 in (u._pack_list([q.cuda() for q in items], "cuda:0")[:2], scattered(items, D, seed=18)):
            out = pool_packed(L, buf, r0, lens, D, mode, p, use_abs)
            assert torch.equal(out.isnan(), ref.isnan())
            assert torch.equal(torch.nan_to_num(out), torch.nan_to_num(ref))
            empty = torch.tensor([n == 0 for n in lens], device="cuda")
            assert bool(out[empty].isnan().all()) and not out[~empty].isnan().any()


def test_pool_list_against_fp64(u):
    D = 1536
    items = [torch.nn.functional.normalize(q, dim=-1) for q in make_items([529, 1, 1369, 88], D, seed=19)]
    for on_dev in (False, True):
        lst = [q.cuda() for q in items] if on_dev else items
        for method in ("average", "max"):
            out = u.pool_descriptors(lst, method)
            assert out.is_cuda == on_dev and out.shape == (len(items), D)
            for i, q in enumerate(items):
                ref = ao.pool_descriptors(q[None].double(), method)[0]
                if method == "max":
                    assert torch.equal(out[i].cpu(), ref.float())
                else:
                    assert rel_inf(out[i].cpu(), ref) < 1e-4
        for p, use_abs in ((3, False), (3, True), (2.5, True), (5, False)):
            out = u.pool_descriptors(lst, "gem", gem_p=p, gem_use_abs=use_abs)
            for i, q in enumerate(items):
                assert rel_inf(out[i].cpu(), ao.gem_descriptors(q[None].double(), p, use_abs)[0]) < 1e-4


def test_end_to_end_reads_the_extractors_buffer(u, L, monkeypatch):
    from oracle import dinov2_restated as dr
    model = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=3), seed=1)
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 2, "value", device="cuda:0", weights=model.state_dict())
    rng = np.random.default_rng(20)
    photos = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((150, 220), (300, 120), (98, 400))]
    feats = ext(u.preprocess_images(photos, max_side=224))
    assert u._packed_rows(feats) is not None
    seen = []
    lib = L.load()
    for name in ("anyloc_vlad_generate_varlen", "anyloc_pool_varlen"):
        fn = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *a, _fn=fn: (seen.append(a[0].value), _fn(*a))[1])
    v = make_vlad(u, 8, 384, seed=21)
    out = v.generate_multi(feats)
    pooled = u.pool_descriptors(feats, "gem")
    assert seen == [feats[0].data_ptr()] * 2
    x, n_valid = padded([q.cpu() for q in feats], 384)
    assert torch.equal(out, v._run(x, n_valid, torch.device("cuda", 0))[0])
    assert torch.equal(pooled, pool_padded(L, [q.cpu() for q in feats], 384, 2))


def test_refusals_launch_nothing(u, L):
    lib = L.load()
    D, K = 64, 8
    buf = torch.randn(40, D, device="cuda")
    v = make_vlad(u, K, D, seed=22)
    centers = v._centers_on(torch.device("cuda", 0))
    out = torch.empty(3, K * D, device="cuda")
    pout = torch.empty(3, D, device="cuda")
    ws = torch.empty(lib.anyloc_vlad_varlen_workspace_bytes(40, 3, 40, D, K), dtype=torch.uint8, device="cuda")
    sws = torch.empty(lib.anyloc_vlad_soft_varlen_workspace_bytes(40, 3, D, K), dtype=torch.uint8, device="cuda")
    r64 = torch.zeros(8, dtype=torch.int64, device="cuda")
    l32 = torch.zeros(8, dtype=torch.int32, device="cuda")

    def calls(feats_p, r0_p, len_p, R=40):
        yield lib.anyloc_vlad_generate_varlen(feats_p, R, r0_p, len_p, 3, L.ptr(centers), None, 0, D, K, 0, 1, 1,
                                              L.ptr(out), None, L.ptr(ws), ws.numel(), L.stream_ptr())
        yield lib.anyloc_vlad_generate_soft_varlen(feats_p, R, r0_p, len_p, 3, L.ptr(centers), D, K, 100.0, 1, 1,
                                                   L.ptr(out), None, L.ptr(sws), sws.numel(), L.stream_ptr())
        yield lib.anyloc_pool_varlen(feats_p, R, r0_p, len_p, 3, D, 2, 3.0, 0, L.ptr(pout), L.stream_ptr())

    def table(row0, lens):
        r64[:3] = torch.tensor(row0)
        l32[:3] = torch.tensor(lens)
        return C.c_void_p(r64.data_ptr()), C.c_void_p(l32.data_ptr())

    good = table([0, 10, 20], [10, 10, 20])
    assert list(calls(L.ptr(buf), *good)) == [0, 0, 0]
    torch.cuda.synchronize()
    cases = [
        (C.c_void_p(buf.data_ptr() + 4), *good),                                   # misaligned feats
        (L.ptr(buf), C.c_void_p(r64.data_ptr() + 4), good[1]),                     # misaligned row0
        (L.ptr(buf), good[0], C.c_void_p(l32.data_ptr() + 2)),                     # misaligned len
    ]
    for row0, lens in (([0, 5, 20], [10, 10, 20]), ([0, 10, 21], [10, 10, 20]), ([0, 10, 20], [10, -1, 20]),
                       ([0, -1, 20], [10, 1, 5])):                                 # overlap, past R, len < 0, row0 < 0
        cases.append((L.ptr(buf), *table(row0, lens)))
    for args in cases:
        before = L.launch_count()
        assert list(calls(*args)) == [L.ERR["arg"]] * 3
        assert L.launch_count() == before
    # empty images may sit anywhere, even inside another image's rows
    assert list(calls(L.ptr(buf), *table([0, 5, 20], [10, 0, 20]))) == [0, 0, 0]
    torch.cuda.synchronize()
