"""generate_vocabularies and its C entries against each member's own call, bit for bit: the shared labels and 1/|x|
against anyloc_vlad_generate_prepared / _sorted / _varlen's labels and the 1/|x| in their workspaces, the shared soft
assignment against anyloc_vlad_generate_soft(_varlen)'s, the accumulations from given labels against the generate
calls' descriptors, and whole sweeps against VLAD.generate_multi for device, host and numpy [n, N, D] input and lists."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def up(n):
    return -(-n // 256) * 256


def bits(t):
    return t.contiguous().view(torch.int32)


def st():
    return _lib.stream_ptr()


def centres(K, D, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(K, D, generator=g)
    if ties and K >= 4:
        c[2] = c[1]                                   # an exact tie: the lower index wins
        c[K - 1] = 50.0 + c[K - 1]                    # a far centre, an empty cluster
    return c.to(DEV)


def features(B, N, D, seed, c=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, D, generator=g)
    if c is not None:                                 # rows on top of centres: exact ties in the scores
        x.view(-1, D)[::7] = c[torch.arange(0, B * N, 7) % c.shape[0]].cpu()
    return x.to(DEV).contiguous()


def prepare(c, mode):
    lib = _lib.load()
    K, D = c.shape
    blob = torch.empty(lib.anyloc_vlad_prepared_bytes(D, K), dtype=torch.uint8, device=DEV)
    _lib.check(lib.anyloc_vlad_prepare(_lib.ptr(c), D, K, mode, _lib.ptr(blob), blob.numel(), st()), "prepare")
    return blob


def own_hard(x, n_valid, c, mode, nd=1, intra=1):
    """the member's own padded call: (vlad, labels, 1/|x| from its workspace)"""
    lib = _lib.load()
    B, N, D = x.shape
    K = c.shape[0]
    R = B * N
    srt = lib.anyloc_vlad_generate_route(B, N, D, K) == _lib.VLAD_ROUTE_SORTED
    fn, wsb = ((lib.anyloc_vlad_generate_sorted, lib.anyloc_vlad_sorted_workspace_bytes) if srt else
               (lib.anyloc_vlad_generate_prepared, lib.anyloc_vlad_workspace_bytes))
    ws = torch.empty(wsb(B, N, D, K), dtype=torch.uint8, device=DEV)
    blob = prepare(c, mode)
    vl = torch.empty(B, K * D, device=DEV)
    lab = torch.empty(R, dtype=torch.int32, device=DEV)
    _lib.check(fn(_lib.ptr(x), _lib.ptr(n_valid), _lib.ptr(c), _lib.ptr(blob), blob.numel(), B, N, D, K, mode, nd,
                  intra, _lib.ptr(vl), _lib.ptr(lab), _lib.ptr(ws), ws.numel(), st()), "own generate")
    inv = ws[up(4 * R):up(4 * R) + 4 * R].view(torch.float32).clone()
    return vl, lab, inv


def own_hard_varlen(feats, row0, lens, c, mode, nd=1, intra=1):
    lib = _lib.load()
    R, D = feats.shape
    K, B = c.shape[0], len(lens)
    r0, ln = u._table_dev(row0, lens, torch.device(DEV))
    ws = torch.empty(lib.anyloc_vlad_varlen_workspace_bytes(R, B, max(lens), D, K), dtype=torch.uint8, device=DEV)
    blob = prepare(c, mode)
    vl = torch.empty(B, K * D, device=DEV)
    lab = torch.empty(R, dtype=torch.int32, device=DEV)
    _lib.check(lib.anyloc_vlad_generate_varlen(_lib.ptr(feats), R, _lib.ptr(r0), _lib.ptr(ln), B, _lib.ptr(c),
                                               _lib.ptr(blob), blob.numel(), D, K, mode, nd, intra, _lib.ptr(vl),
                                               _lib.ptr(lab), _lib.ptr(ws), ws.numel(), st()), "own varlen")
    inv = ws[up(4 * R):up(4 * R) + 4 * R].view(torch.float32).clone()
    return vl, lab, inv


def own_soft(x, n_valid, c, temp, nd=1, intra=1):
    lib = _lib.load()
    B, N, D = x.shape
    K = c.shape[0]
    ws = torch.empty(lib.anyloc_vlad_workspace_bytes(B, N, D, K), dtype=torch.uint8, device=DEV)
    vl = torch.empty(B, K * D, device=DEV)
    a = torch.empty(B * N, K, device=DEV)
    _lib.check(lib.anyloc_vlad_generate_soft(_lib.ptr(x), _lib.ptr(n_valid), _lib.ptr(c), B, N, D, K, C.c_float(temp),
                                             nd, intra, _lib.ptr(vl), _lib.ptr(a), _lib.ptr(ws), ws.numel(), st()),
               "own soft")
    return vl, a, ws[:4 * B * N].view(torch.float32).clone()


def own_soft_varlen(feats, row0, lens, c, temp, nd=1, intra=1):
    lib = _lib.load()
    R, D = feats.shape
    K, B = c.shape[0], len(lens)
    r0, ln = u._table_dev(row0, lens, torch.device(DEV))
    ws = torch.empty(lib.anyloc_vlad_soft_varlen_workspace_bytes(R, B, D, K), dtype=torch.uint8, device=DEV)
    vl = torch.empty(B, K * D, device=DEV)
    a = torch.empty(R, K, device=DEV)
    _lib.check(lib.anyloc_vlad_generate_soft_varlen(_lib.ptr(feats), R, _lib.ptr(r0), _lib.ptr(ln), B, _lib.ptr(c), D,
                                                    K, C.c_float(temp), nd, intra, _lib.ptr(vl), _lib.ptr(a),
                                                    _lib.ptr(ws), ws.numel(), st()), "own soft varlen")
    return vl, a, ws[:4 * R].view(torch.float32).clone()


def label_multi(x, n_valid, N, cs, mode, route_rows, prepared=True):
    lib = _lib.load()
    D = x.shape[-1]
    R = x.numel() // D
    V = len(cs)
    Ks = (C.c_int * V)(*[c.shape[0] for c in cs])
    blobs = [prepare(c, mode) for c in cs] if prepared else None
    labels = torch.full((V, R), -7, dtype=torch.int32, device=DEV)
    inv = torch.empty(R, device=DEV)
    ws = torch.empty(lib.anyloc_vlad_label_multi_workspace_bytes(R, D, V, Ks), dtype=torch.uint8, device=DEV)
    _lib.check(lib.anyloc_vlad_label_multi(
        _lib.ptr(x), _lib.ptr(n_valid), N, R, (C.c_int64 * V)(*route_rows), D, V,
        (C.c_void_p * V)(*[c.data_ptr() for c in cs]),
        (C.c_void_p * V)(*[b.data_ptr() for b in blobs]) if prepared else None,
        (C.c_size_t * V)(*[b.numel() for b in blobs]) if prepared else None, Ks, mode, _lib.ptr(labels),
        _lib.ptr(inv), _lib.ptr(ws), ws.numel(), st()), "label_multi")
    return labels, inv


def soft_multi(x, n_valid, N, cs, temps):
    lib = _lib.load()
    D = x.shape[-1]
    R = x.numel() // D
    V = len(cs)
    Ks = (C.c_int * V)(*[c.shape[0] for c in cs])
    assign = [torch.full((R, c.shape[0]), 7.0, device=DEV) for c in cs]
    inv = torch.empty(R, device=DEV)
    ws = torch.empty(lib.anyloc_vlad_soft_assign_multi_workspace_bytes(D, V, Ks), dtype=torch.uint8, device=DEV)
    _lib.check(lib.anyloc_vlad_soft_assign_multi(
        _lib.ptr(x), _lib.ptr(n_valid), N, R, D, V, (C.c_void_p * V)(*[c.data_ptr() for c in cs]), Ks,
        (C.c_float * V)(*temps), (C.c_void_p * V)(*[a.data_ptr() for a in assign]), _lib.ptr(inv), _lib.ptr(ws),
        ws.numel(), st()), "soft_multi")
    return assign, inv


def accumulate(x, n_valid, labels, assign, inv, c, nd=1, intra=1):
    lib = _lib.load()
    B, N, D = x.shape
    K = c.shape[0]
    ws = torch.empty(lib.anyloc_vlad_accumulate_workspace_bytes(B, N, D, K, int(assign is not None)),
                     dtype=torch.uint8, device=DEV)
    vl = torch.full((B, K * D), 7.0, device=DEV)
    _lib.check(lib.anyloc_vlad_accumulate(_lib.ptr(x), _lib.ptr(n_valid), _lib.ptr(labels), _lib.ptr(assign),
                                          _lib.ptr(inv), _lib.ptr(c), B, N, D, K, nd, intra, _lib.ptr(vl), _lib.ptr(ws),
                                          ws.numel(), st()), "accumulate")
    return vl


def accumulate_varlen(feats, row0, lens, labels, assign, inv, c, nd=1, intra=1):
    lib = _lib.load()
    R, D = feats.shape
    K, B = c.shape[0], len(lens)
    r0, ln = u._table_dev(row0, lens, torch.device(DEV))
    ws = torch.empty(lib.anyloc_vlad_accumulate_workspace_bytes(B, max(lens), D, K, int(assign is not None)),
                     dtype=torch.uint8, device=DEV)
    vl = torch.full((B, K * D), 7.0, device=DEV)
    _lib.check(lib.anyloc_vlad_accumulate_varlen(_lib.ptr(feats), R, _lib.ptr(r0), _lib.ptr(ln), B, _lib.ptr(labels),
                                                 _lib.ptr(assign), _lib.ptr(inv), _lib.ptr(c), D, K, nd, intra,
                                                 _lib.ptr(vl), _lib.ptr(ws), ws.numel(), st()), "accumulate_varlen")
    return vl


# --------------------------------------------------------------------------------------------------- the C entries
HARD_CASES = [  # B, N, D, Ks: R = B * N around the 256-row route switch, D = 2560 on the FFMA route, K up to 1000
    (1, 255, 64, [1, 7, 32]), (1, 256, 64, [1, 7, 32]), (3, 100, 1536, [32, 64, 128, 256]), (2, 130, 2560, [8, 1]),
    (4, 300, 384, [1000]), (2, 3942, 1536, [256]), (1, 20, 1536, [5, 64]), (8, 529, 1536, [32, 64, 128, 256]),
    (2, 3942, 1536, [32, 64, 128]),           # accumulate3's shared memory exceeded, K <= 200: ACC2
]
ACC3, ACC2, SORTED = 0, 1, 2


def route(B, N, D, K):
    return _lib.load().anyloc_vlad_generate_route(B, N, D, K)


def test_cases_reach_every_accumulation_route():
    padded = {route(B, N, D, K) for B, N, D, Ks in HARD_CASES for K in Ks}
    packed = {route(len(lens), max(lens), D, K) for lens, D, Ks in PACKED_CASES for K in Ks}
    assert padded == packed == {ACC3, ACC2, SORTED}
    assert {route(2, 3942, 1536, K) for K in (32, 64, 128)} == {ACC2} and route(2, 3942, 1536, 256) == SORTED


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("B,N,D,Ks", HARD_CASES)
def test_labels_norms_and_descriptors_equal_each_members_call(B, N, D, Ks, mode):
    cs = [centres(K, D, 10 + i, ties=True) for i, K in enumerate(Ks)]
    x = features(B, N, D, 1, cs[-1])
    n_valid = torch.tensor([N - (b % 3) * (N // 4) for b in range(B)], dtype=torch.int32, device=DEV)
    for b in range(B):                                # ragged padded rows holding NaN
        x[b, int(n_valid[b]):] = float("nan")
    for prepared in (True, False):
        labels, inv = label_multi(x, n_valid, N, cs, mode, [B * N] * len(cs), prepared)
        for v, c in enumerate(cs):
            for intra in (0, 1):
                vl, lab, own_inv = own_hard(x, n_valid, c, mode, intra=intra)
                assert torch.equal(labels[v], lab), (v, prepared)
                assert torch.equal(bits(inv), bits(own_inv)), (v, prepared)
                assert torch.equal(bits(accumulate(x, None, labels[v], None, inv, c, intra=intra)), bits(vl)), v


def test_each_member_keeps_its_own_route():
    # member 0's own call has 300 rows (coarse route), member 1's 150 (FFMA): labels equal each member's own call
    D = 384
    cs = [centres(64, D, 3), centres(40, D, 4)]
    x = features(1, 150, D, 5)
    labels, inv = label_multi(x, None, 1, cs, 0, [300, 150])
    big = torch.cat([x, features(1, 150, D, 6)], 1)
    _, lab0, inv0 = own_hard(big, None, cs[0], 0)
    _, lab1, inv1 = own_hard(x, None, cs[1], 0)
    assert torch.equal(labels[0], lab0[:150]) and torch.equal(labels[1], lab1)
    assert torch.equal(bits(inv), bits(inv1)) and torch.equal(bits(inv), bits(inv0[:150]))


def _packed(lens, D, seed, canary=True):
    """rows of len[i] per image with a NaN canary row before each image -> (feats [R, D], row0)"""
    g = torch.Generator().manual_seed(seed)
    rows, row0, r = [], [], 0
    for n in lens:
        if canary:
            rows.append(torch.full((1, D), float("nan")))
            r += 1
        row0.append(r)
        rows.append(torch.randn(n, D, generator=g))
        r += n
    return torch.cat(rows).to(DEV).contiguous(), row0


PACKED_CASES = [
    ([100, 0, 1, 90], 384, [8, 64]),          # R < 256 <= B * max len: the padded shape's (coarse) route
    ([40, 3], 64, [1, 5]),                    # B * max len < 256: FFMA
    ([529] * 5 + [1, 0, 300], 1536, [32, 64, 128, 256]),
    ([3942, 10], 1536, [256]),                # the sorted route
    ([3942, 10], 1536, [32, 128]),            # ACC2
    ([60, 70], 2560, [16, 3]),
]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("lens,D,Ks", PACKED_CASES)
def test_packed_labels_and_descriptors(lens, D, Ks, mode):
    cs = [centres(K, D, 20 + i, ties=True) for i, K in enumerate(Ks)]
    feats, row0 = _packed(lens, D, 2)
    labels, inv = label_multi(feats, None, 1, cs, mode, [len(lens) * max(lens)] * len(cs))
    rows = torch.cat([torch.arange(r, r + n) for r, n in zip(row0, lens)]).to(DEV)
    for v, c in enumerate(cs):
        vl, lab, own_inv = own_hard_varlen(feats, row0, lens, c, mode)
        assert torch.equal(labels[v][rows], lab[rows]), v
        assert torch.equal(bits(inv[rows]), bits(own_inv[rows])), v
        got = accumulate_varlen(feats, row0, lens, labels[v], None, inv, c)
        assert torch.equal(bits(got), bits(vl)), v


@pytest.mark.parametrize("B,N,D,Ks,temps", [
    (2, 100, 64, [1, 7, 32], [1.0, 0.3, 25.0]), (1, 300, 1536, [32, 64, 128, 256], [1.0, 2.0, 0.5, 10.0]),
    (3, 50, 2560, [2048, 5], [1.0, 4.0]), (1, 8, 64, [2048] * 15, [float(i + 1) for i in range(15)]),
])
def test_soft_assignments_equal_each_members_call(B, N, D, Ks, temps):
    cs = [centres(K, D, 30 + i, ties=True) for i, K in enumerate(Ks)]
    x = features(B, N, D, 3, cs[0])
    n_valid = torch.tensor([N - b * (N // 3) for b in range(B)], dtype=torch.int32, device=DEV)
    for b in range(B):
        x[b, int(n_valid[b]):] = float("nan")
    assign, inv = soft_multi(x, n_valid, N, cs, temps)
    for v, (c, t) in enumerate(zip(cs, temps)):
        vl, a, own_inv = own_soft(x, n_valid, c, t)
        assert torch.equal(bits(assign[v]), bits(a)), v                # padded rows exactly 0 in both
        assert torch.equal(bits(inv), bits(own_inv)), v
        assert torch.equal(bits(accumulate(x, n_valid, None, assign[v], inv, c)), bits(vl)), v
    # packed rows, NaN canaries between images
    lens = [N, 0, 1, max(1, N // 2)]
    feats, row0 = _packed(lens, D, 4)
    assign, inv = soft_multi(feats, None, 1, cs, temps)
    rows = torch.cat([torch.arange(r, r + n) for r, n in zip(row0, lens)]).to(DEV)
    for v, (c, t) in enumerate(zip(cs, temps)):
        vl, a, own_inv = own_soft_varlen(feats, row0, lens, c, t)
        assert torch.equal(bits(assign[v][rows]), bits(a[rows])), v
        assert torch.equal(bits(inv[rows]), bits(own_inv[rows])), v
        assert torch.equal(bits(accumulate_varlen(feats, row0, lens, None, assign[v], inv, c)), bits(vl)), v


def test_packed_table_refusals():
    lib = _lib.load()
    feats = torch.zeros(10, 8, device=DEV)
    c = torch.zeros(4, 8, device=DEV)
    lab = torch.zeros(10, dtype=torch.int32, device=DEV)
    vl = torch.zeros(2, 32, device=DEV)
    ws = torch.empty(1 << 16, dtype=torch.uint8, device=DEV)
    for row0, lens in (([0, 4], [5, 2]), ([0, 8], [4, 3]), ([-1, 4], [1, 1]), ([0, 4], [-1, 1])):
        r0, ln = u._table_dev(row0, lens, torch.device(DEV))
        rc = lib.anyloc_vlad_accumulate_varlen(_lib.ptr(feats), 10, _lib.ptr(r0), _lib.ptr(ln), 2, _lib.ptr(lab), None,
                                               _lib.ptr(feats), _lib.ptr(c), 8, 4, 1, 1, _lib.ptr(vl), _lib.ptr(ws),
                                               ws.numel(), st())
        assert rc == _lib.ERR["arg"], (row0, lens)
    torch.cuda.synchronize()


# --------------------------------------------------------------------------------------------- generate_vocabularies
def _members(D, specs, mode="cosine", nd=True):
    out = []
    for i, (K, vm, t, intra) in enumerate(specs):
        v = u.VLAD(K, dist_mode=mode, norm_descs=nd, vlad_mode=vm, soft_temp=t, intra_norm=intra)
        v.kmeans = u._KMeans(K, mode=mode)
        v.kmeans.centroids = v.c_centers = centres(K, D, 40 + i, ties=True).cpu()
        v.desc_dim = D
        out.append(v)
    return out


def _same(got, vlads, x):
    assert len(got) == len(vlads)
    for v, g in zip(vlads, got):
        want = v.generate_multi(x)
        assert g.device == want.device and g.dtype == want.dtype and g.shape == want.shape
        assert torch.equal(bits(g), bits(want)), v.num_clusters


SPECS = [(32, "hard", 1.0, True), (64, "soft", 0.5, False), (128, "hard", 1.0, False), (7, "soft", 20.0, True)]


@pytest.mark.parametrize("mode,nd", [("cosine", True), ("euclidean", False)])
def test_device_host_and_numpy_inputs(mode, nd, monkeypatch):
    D = 384
    vlads = _members(D, SPECS, mode, nd)
    x = features(9, 70, D, 7).cpu()
    _same(u.generate_vocabularies(vlads, x.to(DEV)), vlads, x.to(DEV))
    _same(u.generate_vocabularies(vlads, x.numpy()), vlads, x.numpy())
    _same(u.generate_vocabularies(vlads, x), vlads, x)
    # host features through several chunks: a budget of about three images
    budget = u._generate_chunk_bytes(3, 70, D, [32, 128], [64, 7], True)
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    _same(u.generate_vocabularies(vlads, x), vlads, x)
    _same(u.generate_vocabularies(vlads, x.double()), vlads, x.double())
    _same(u.generate_vocabularies(vlads, x.to(DEV)), vlads, x.to(DEV))
    _same(u.generate_vocabularies(vlads[:1], x), vlads[:1], x)                         # V = 1


def test_members_whose_generate_multi_chunks_differently(monkeypatch):
    # member 1 streams host features in calls of 2 images (140 rows, FFMA), member 0 in one call (coarse route)
    D = 1536
    vlads = _members(D, [(64, "hard", 1.0, True), (32, "hard", 1.0, True), (16, "soft", 2.0, True)])
    vlads[1]._host_chunk_bytes = 2 * 70 * D * 4 + 5
    x = features(7, 70, D, 8).cpu()
    _same(u.generate_vocabularies(vlads, x), vlads, x)
    budget = u._generate_chunk_bytes(3, 70, D, [64, 32], [16], True)
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    _same(u.generate_vocabularies(vlads, x), vlads, x)


@pytest.mark.parametrize("mode", ["cosine", "euclidean"])
def test_ablation_sweep_on_long_images(mode, monkeypatch):
    # the reference ablation's num_clusters = (256, 128, 64, 32) on 3942-patch images: K <= 128 take ACC2, 256 sorted
    D = 1536
    vlads = _members(D, [(256, "hard", 1.0, True), (128, "hard", 1.0, False), (64, "soft", 2.0, True),
                         (32, "hard", 1.0, True)], mode)
    assert [route(3, 3942, D, K) for K in (256, 128, 32)] == [SORTED, ACC2, ACC2]
    x = features(3, 3942, D, 12)
    _same(u.generate_vocabularies(vlads, x), vlads, x)
    budget = u._generate_chunk_bytes(1, 3942, D, [256, 128, 32], [64], True)
    monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: budget)
    _same(u.generate_vocabularies(vlads, x.cpu()), vlads, x.cpu())         # one image per staged chunk


def test_sorted_route_and_large_k():
    D = 1536
    vlads = _members(D, [(256, "hard", 1.0, True), (1000, "hard", 1.0, False), (2048, "soft", 1.0, True)])
    x = features(2, 3942, D, 9)
    assert _lib.load().anyloc_vlad_generate_route(2, 3942, D, 256) == _lib.VLAD_ROUTE_SORTED
    _same(u.generate_vocabularies(vlads, x), vlads, x)


@pytest.mark.parametrize("D", [64, 2560])
def test_lists(D):
    vlads = _members(D, SPECS)
    g = torch.Generator().manual_seed(11)
    lens = [100, 0, 1, 90, 37]
    buf = torch.randn(sum(lens), D, generator=g).to(DEV)
    views = list(torch.split(buf, lens))              # ext(list)'s consecutive views of one buffer: read in place
    assert u._packed_rows(views) is not None
    _same(u.generate_vocabularies(vlads, views), vlads, views)
    _same(u.generate_vocabularies(vlads, [q.cpu() for q in views]), vlads, [q.cpu() for q in views])
    _same(u.generate_vocabularies(vlads, [views[3], views[0].clone()]), vlads, [views[3], views[0].clone()])
    _same(u.generate_vocabularies(vlads, views[2:3]), vlads, views[2:3])


def test_empty_and_zero_row_inputs():
    # generate_multi refuses both empty shapes (the empty tensor's null data pointer); the sweep gives what the shape
    # says: no descriptors for [0, N, D], zero descriptors for [n, 0, D]
    vlads = _members(64, SPECS[:2])
    for x in (torch.zeros(0, 5, 64), torch.zeros(3, 0, 64), torch.zeros(3, 0, 64, device=DEV)):
        for v in vlads:
            with pytest.raises(_lib.AnylocError, match="null pointer"):
                v.generate_multi(x)
        got = u.generate_vocabularies(vlads, x)
        for v, g in zip(vlads, got):
            assert g.device == x.device and g.shape == (x.shape[0], v.num_clusters * 64) and not g.any()
