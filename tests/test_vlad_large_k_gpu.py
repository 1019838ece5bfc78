"""Hard VLAD and the k-means update at any vocabulary size.

anyloc_vlad_generate_sorted keeps accumulate3's summation order with its per-image tables in the workspace: inside
accumulate3's envelope it must equal anyloc_vlad_generate_prepared bit for bit (descriptors and labels), and outside
it the descriptors must satisfy the element-wise fp64 bound of tests/test_vlad_engine_gpu.py.  The cluster-tiled
k-means update must equal the untiled one bit for bit where that runs, stay within the fp64 bound of the mean beyond
it, and give the same bits streamed in rounds.  Through the public API, VLAD picks the sorted route only where the
shared-memory routes refuse."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from oracle import anyloc_oracle as ao
from tests.test_kmeans_stream_gpu import check_equal, clustered, vlad_fit
from tests.test_vlad_engine_gpu import (C_ACC, COS, EUC, LEAD, U, L, accumulate_route, assert_canaries, canary,  # noqa: F401
                                        check_labels, generate, hard_reference, inner, make_inputs, permuted_targets,
                                        prepare, ratio, sms, workspace)
from tests.util import dptr, make_vlad, rel_inf

pytestmark = pytest.mark.gpu
ERR_WORKSPACE = -3
TOL = 1e-4


def generate_sorted(L, x, centers, B, N, D, K, *, dist=COS, norm=1, intra=1, n_valid=None, blob=None, ws=None,
                    expect_rc=0):
    """one anyloc_vlad_generate_sorted call -> (vlad [B,K,D], labels [B,N])"""
    lib = L.load()
    blob = prepare(L, centers, D, K, dist) if blob is None else blob
    out, lab = canary(B * K * D), canary(B * N, torch.int32)
    ws = workspace(lib.anyloc_vlad_sorted_workspace_bytes(B, N, D, K)) if ws is None else ws
    rc = lib.anyloc_vlad_generate_sorted(dptr(x), dptr(n_valid), dptr(centers), dptr(blob), blob.numel(), B, N, D, K,
                                         dist, norm, intra, dptr(out, LEAD), dptr(lab, LEAD), dptr(ws), ws.numel(),
                                         L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == expect_rc, (rc, L.last_error())
    assert_canaries(out, B * K * D, "vlad", written=rc == 0)
    assert_canaries(lab, B * N, "labels", written=rc == 0)
    return inner(out, B * K * D).view(B, K, D), inner(lab, B * N).view(B, N)


def route(L, B, N, D, K):
    return L.load().anyloc_vlad_generate_route(B, N, D, K)


# ------------------------------------------------------------------------------ bitwise equal to accumulate3
ENVELOPE = {
    # name: (B, N, D, K, family, kwargs)
    "c2": (4, 529, 1536, 32, "clustered", {}),
    "c5": (2, 1369, 1024, 128, "random", {}),
    "euclidean": (3, 400, 256, 12, "random", {"dist": EUC}),
    "euclidean_no_norm": (2, 300, 384, 16, "clustered", {"dist": EUC, "norm": 0}),
    "intra_off": (3, 400, 256, 12, "random", {"intra": 0}),
    "norm_descs_off": (3, 400, 256, 12, "spread", {"norm": 0}),
    "K1": (2, 300, 128, 1, "random", {}),
    "K201": (2, 400, 128, 201, "random", {}),
    "K1000": (1, 300, 64, 1000, "random", {}),
    "D36": (3, 300, 36, 8, "random", {}),
    "D1028": (2, 400, 1028, 16, "random", {}),
    "ffma_assign": (1, 200, 384, 8, "clustered", {}),
}


def check_bitwise(L, x, centers, B, N, D, K, n_valid=None, **kw):
    dist = kw.get("dist", COS)
    blob = prepare(L, centers, D, K, dist)
    v3, l3, _ = generate(L, x, centers, B, N, D, K, n_valid=n_valid, blob=blob, **kw)
    vs, ls = generate_sorted(L, x, centers, B, N, D, K, n_valid=n_valid, blob=blob, **kw)
    assert torch.equal(ls, l3), "labels differ from accumulate3's"
    assert torch.equal(vs.view(torch.int32), v3.view(torch.int32)), "descriptors differ from accumulate3's"
    return vs, ls


@pytest.mark.parametrize("name", sorted(ENVELOPE))
def test_sorted_equals_accumulate3(L, name):
    B, N, D, K, fam, kw = ENVELOPE[name]
    assert accumulate_route(N, D, K) == "accumulate3" and route(L, B, N, D, K) == 0
    x, centers = make_inputs(fam, B, N, D, K, seed=len(name))
    check_bitwise(L, x, centers, B, N, D, K, **kw)


@pytest.mark.parametrize("layout", ["one_cluster", "exact65", "empty_clusters"])
def test_sorted_equals_accumulate3_structure(L, layout):
    """one cluster of 3000 rows (47 tasks combined from slots), every cluster 65 rows (two tasks each), half the
    clusters empty (exactly 0)"""
    D = 256
    if layout == "one_cluster":
        K, counts = 8, [3000, 0, 0, 0, 0, 0, 0, 0]
    elif layout == "exact65":
        K, counts = 16, [65] * 16
    else:
        K, counts = 32, [37 if k % 2 else 0 for k in range(32)]
    B, N = 2, sum(counts)
    target = permuted_targets(B, counts, seed=K)
    x, centers = make_inputs("clustered", B, N, D, K, seed=N, target=target)
    v, lab = check_bitwise(L, x, centers, B, N, D, K)
    assert torch.equal(lab.long(), target)
    cnt = torch.tensor(counts, device="cuda")
    assert bool((v[:, cnt == 0] == 0).all()) and bool((v[:, cnt > 0].norm(dim=2) > 0).all())


def test_sorted_equals_accumulate3_ragged_nan(L):
    """rows at or beyond n_valid[b] hold NaN (an image with no valid row included): labels -1 there, same bits"""
    B, N, D, K = 5, 411, 384, 16
    nv = [300, 257, 1, 411, 0]
    x, centers = make_inputs("clustered", B, N, D, K, seed=21)
    for b, n in enumerate(nv):
        x[b, n:] = float("nan")
    n_valid = torch.tensor(nv, dtype=torch.int32, device="cuda")
    v, lab = check_bitwise(L, x, centers, B, N, D, K, n_valid=n_valid)
    for b, n in enumerate(nv):
        assert bool((lab[b, n:] == -1).all()) and bool((lab[b, :n] >= 0).all())
    assert bool((v[4] == 0).all()) and bool(torch.isfinite(v).all())


def test_sorted_equals_accumulate3_last_cta(L, sms):
    """more CTAs than can be co-resident, so accumulate3 normalises each image in its last CTA instead of the
    distributed normalise the shapes above take: the sorted route still gives the same bits"""
    B, N, D, K = 8 * sms + 144, 300, 128, 16
    assert (D + 127) // 128 * B > 8 * sms
    x, centers = make_inputs("random", B, N, D, K, seed=B)
    check_bitwise(L, x, centers, B, N, D, K)


# ------------------------------------------------------------------------------ outside the envelope
OUTSIDE = [(1, 4000, 128, 256), (1, 2000, 64, 1000), (2, 5329, 1536, 256), (1, 1369, 1024, 2048)]


@pytest.mark.parametrize("B,N,D,K", OUTSIDE)
def test_sorted_outside_envelope(L, B, N, D, K):
    assert accumulate_route(N, D, K) == "error" and route(L, B, N, D, K) == _lib.VLAD_ROUTE_SORTED
    x, centers = make_inputs("random", B, N, D, K, seed=N + K)
    blob = prepare(L, centers, D, K)
    v, lab = generate_sorted(L, x, centers, B, N, D, K, blob=blob)
    assert int(lab.min()) >= 0 and int(lab.max()) < K
    check_labels(x, centers, lab, COS, f"sorted N{N} K{K}")
    v64, bound, _ = hard_reference(x, centers, lab)
    r = ratio(v, v64, bound)
    print(f"sorted B{B} N{N} D{D} K{K}: worst ratio {r:.3f}")
    assert r <= 1.0
    for b in range(B):
        vs, ls = generate_sorted(L, x[b:b + 1].contiguous(), centers, 1, N, D, K, blob=blob)
        assert torch.equal(vs[0], v[b]) and torch.equal(ls[0], lab[b]), f"image {b}: batch != single image"
    short = workspace(L.load().anyloc_vlad_sorted_workspace_bytes(B, N, D, K) - 1)
    generate_sorted(L, x, centers, B, N, D, K, blob=blob, ws=short, expect_rc=ERR_WORKSPACE)


# ------------------------------------------------------------------------------ tiled k-means
def kmeans_call(L, x, labels, old, K, k_tile=None):
    """anyloc_kmeans_update (k_tile None) or _tiled -> (centres, err, partial sums, partial counts)"""
    lib = L.load()
    R, D = x.shape
    chunks, rows_per = C.c_int(0), C.c_int64(0)
    L.check(lib.anyloc_kmeans_partition(R, D, C.byref(chunks), C.byref(rows_per)), "partition")
    new, err = canary(K * D), canary(1)
    ws = workspace(lib.anyloc_kmeans_workspace_bytes(R, D, K))
    args = (dptr(new, LEAD), dptr(err, LEAD), dptr(ws), ws.numel(), L.stream_ptr())
    if k_tile is None:
        L.check(lib.anyloc_kmeans_update(dptr(x), dptr(labels), dptr(old), R, D, K, *args), "kmeans_update")
    else:
        L.check(lib.anyloc_kmeans_update_tiled(dptr(x), dptr(labels), dptr(old), R, D, K, k_tile, *args),
                "kmeans_update_tiled")
    torch.cuda.synchronize()
    assert_canaries(new, K * D, "kmeans centres")
    assert_canaries(err, 1, "kmeans err")
    n_sums = chunks.value * K * D
    off = -(-n_sums * 4 // 256) * 256
    psums = ws[:n_sums * 4].view(torch.float32)
    pcounts = ws[off:off + chunks.value * K * 4].view(torch.float32)
    return inner(new, K * D).view(K, D), inner(err, 1), psums, pcounts


def kmeans_inputs(R, D, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(R, D, device="cuda", generator=g) * 10.0 ** (2 * torch.rand(R, 1, device="cuda", generator=g) - 1)
    labels = torch.randint(0, K - 3, (R,), device="cuda", generator=g, dtype=torch.int32)     # K-3.. stay empty
    labels[::7] = -1
    old = torch.randn(K, D, device="cuda", generator=g)
    return x, labels, old


@pytest.mark.parametrize("R,D,K,k_tile", [(20_000, 132, 100, 37), (20_000, 132, 436, 37), (3001, 384, 436, 0),
                                          (257, 128, 8, 3)])
def test_kmeans_tiled_equals_untiled(L, R, D, K, k_tile):
    x, labels, old = kmeans_inputs(R, D, K, seed=R + K)
    a = kmeans_call(L, x, labels, old, K)
    b = kmeans_call(L, x, labels, old, K, k_tile)
    for p, q, what in zip(a, b, ("centres", "err", "partial sums", "counts")):
        assert torch.equal(p.view(torch.int32), q.view(torch.int32)), f"{what} differ"


@pytest.mark.parametrize("K", [437, 1024, 2048])
def test_kmeans_tiled_fp64(L, K):
    R, D = 30_000, 128
    x, labels, old = kmeans_inputs(R, D, K, seed=K)
    x[:, 0] = 1.0
    chunks, rows_per = C.c_int(0), C.c_int64(0)
    L.check(L.load().anyloc_kmeans_partition(R, D, C.byref(chunks), C.byref(rows_per)), "partition")
    c, err, _, _ = kmeans_call(L, x, labels, old, K, 0)
    keep = labels >= 0
    lab = labels[keep].long()
    n = torch.bincount(lab, minlength=K).double()
    s64 = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, lab, x[keep].double())
    a64 = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, lab, x[keep].double().abs())
    c64 = torch.where(n[:, None] > 0, s64 / n.clamp_min(1)[:, None], torch.zeros((), dtype=torch.float64, device="cuda"))
    bound = C_ACC * U * ((n + chunks.value + 2).sqrt()[:, None] * a64 / n.clamp_min(1)[:, None] + c64.abs())
    empty = n == 0
    assert bool((c[empty] == 0).all()) and bool((c[~empty, 0] == 1.0).all())
    r = float(((c.double() - c64).abs()[~empty] / bound[~empty]).max())
    print(f"kmeans tiled K={K}: worst ratio {r:.3f}")
    assert r <= 1.0


def test_kmeans_tiled_rounds_equal_in_memory(L):
    """anyloc_kmeans_accumulate_round_tiled over several rounds (resume) + finalize == anyloc_kmeans_update_tiled"""
    lib = L.load()
    R, D, K = 10_007, 128, 1024
    x, labels, old = kmeans_inputs(R, D, K, seed=5)
    c_ref, e_ref, _, _ = kmeans_call(L, x, labels, old, K, 0)
    with torch.cuda.device(0):
        chunks, rows_per = u._kmeans_partition(R, D)
    ws = workspace(lib.anyloc_kmeans_round_workspace_bytes(R, D, K))
    rounds = u._stream_rounds(R, chunks, rows_per, 13)
    assert len(rounds) > 1
    for j, pcs in enumerate(rounds):
        idx = torch.cat([torch.arange(lo, lo + m) for lo, m in pcs]).cuda()
        xr, lr = x[idx].contiguous(), labels[idx].contiguous()
        L.check(lib.anyloc_kmeans_accumulate_round_tiled(dptr(xr), dptr(lr), R, idx.numel(), pcs[0][1], D, K, 0,
                                                         int(j > 0), dptr(ws), ws.numel(), L.stream_ptr()), "round")
    c, e = torch.empty(K, D, device="cuda"), torch.zeros(1, device="cuda")
    L.check(lib.anyloc_kmeans_finalize(dptr(old), R, D, K, dptr(c), dptr(e), dptr(ws), ws.numel(), L.stream_ptr()),
            "finalize")
    torch.cuda.synchronize()
    assert torch.equal(c, c_ref) and torch.equal(e, e_ref)


def test_vlad_fit_streamed_tiled(cuda, monkeypatch):
    """VLAD(1024).fit on host rows, streamed in rounds, equals the in-memory tiled fit bit for bit"""
    X = clustered(6000, 64, 1024, seed=7)
    check_equal(vlad_fit(X, 1024), monkeypatch, (X, 1024, 2, 17, "zero"))


# ------------------------------------------------------------------------------ public API
def test_vlad_256_demo_photo_list(cuda):
    """VLAD(256).generate_multi on the demo's 1024-px photos' ViT-G patch features (73 x 54 and 73 x 73 patches)"""
    D, K = 1536, 256
    g = torch.Generator().manual_seed(3)
    centers = 0.5 * torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1) * (1 + 0.3 * torch.rand(K, 1, generator=g))
    qs = [torch.randn(n, D, generator=g) * (0.3 + torch.rand(n, 1, generator=g)) for n in (3942, 5329, 3942)]
    v = make_vlad(u, K, centers)
    outs = v.generate_multi(qs)
    assert outs.shape == (3, K * D) and not outs.is_cuda
    for q, o in zip(qs, outs):
        lab = v.kmeans.predict(q)
        gap, lab64 = ao.label_margins(q, centers)
        assert torch.equal(lab[gap > 1e-5], lab64[gap > 1e-5])
        assert rel_inf(o, ao.vlad_generate(q, centers, labels=lab, dtype=torch.float64)) < TOL
        assert torch.equal(v.generate(q), o)
    dev = v.generate_multi(torch.stack(qs[::2]).cuda())
    assert torch.equal(dev.cpu(), outs[::2])
    v._host_chunk_bytes = qs[0].numel() * 4                          # one image per host chunk
    assert torch.equal(v.generate_multi(torch.stack(qs[::2])), outs[::2])


def test_vlad_1024_fit_and_generate(cuda, tmp_path):
    """VLAD(1024).fit (the tiled update) against fpk's Lloyd loop from the same draw, then generate on rows that were
    not in the fit (a query equal to a singleton cluster's centre leaves a residual of rounding noise, which intra
    normalisation blows up in any precision) against the oracle, directly and through the `<id>_l.pt` cache"""
    xall, _, _ = ao.clustered_features(24_000, 128, 1024, seed=4)
    x, q, q2 = xall[:20_000], xall[20_000:22_000], xall[22_000:].reshape(2, 1000, 128)
    np.random.seed(42)
    v = u.VLAD(1024, cache_dir=str(tmp_path / "c"))
    v.fit(x)
    assert v.c_centers.shape == (1024, 128)
    from oracle import fpk_restated as fpk
    np.random.seed(42)
    km = fpk.KMeans(1024, mode="cosine")
    km.fit(torch.nn.functional.normalize(x))
    assert rel_inf(v.c_centers, km.centroids) < 1e-4
    assert route(_lib, 1, 2000, 128, 1024) == _lib.VLAD_ROUTE_SORTED   # N = 1369 still fits accumulate3 at D = 128
    out = v.generate(q)
    lab = v.kmeans.predict(q)
    ref = ao.vlad_generate(q, v.c_centers, labels=lab, dtype=torch.float64)
    assert rel_inf(out, ref) < TOL
    o1 = v.generate(q, cache_id="img0")                             # labels computed and saved ...
    assert torch.equal(torch.load(tmp_path / "c" / "img0_l.pt"), lab)
    o2 = v.generate(q, cache_id="img0")                             # ... then read back (residual kernels)
    assert rel_inf(o1, ref) < TOL and rel_inf(o2, ref) < TOL
    np.random.seed(7)
    v2 = u.VLAD(1024)
    outs = v2.fit_and_generate(torch.cat([x[:4000].reshape(2, 2000, 128), q[None]]))
    assert outs.shape == (3, 1024 * 128)
    assert torch.equal(outs, v2.generate_multi(torch.cat([x[:4000].reshape(2, 2000, 128), q[None]])))
    for w in (v, v2):                                                # rows neither vocabulary was fitted on
        outs = w.generate_multi(q2)
        for b in range(2):
            lab = w.kmeans.predict(q2[b])
            assert rel_inf(outs[b], ao.vlad_generate(q2[b], w.c_centers, labels=lab, dtype=torch.float64)) < TOL


def test_envelope_keeps_its_kernels(cuda):
    """a shape accumulate3 serves launches what it launched before (prep is cached: GEMM + rescore + accumulate3) and
    gives the ABI call's bits"""
    B, N, D, K = 2, 529, 1536, 32
    g = torch.Generator().manual_seed(8)
    x = torch.randn(B, N, D, generator=g).cuda()
    centers = 0.5 * torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1)
    v = make_vlad(u, K, centers)
    v.generate_multi(x)
    n0 = _lib.launch_count()
    out = v.generate_multi(x)
    assert _lib.launch_count() - n0 == 3
    lib = _lib.load()
    ref = torch.empty(B, K * D, device="cuda")
    ws = torch.empty(lib.anyloc_vlad_workspace_bytes(B, N, D, K), dtype=torch.uint8, device="cuda")
    cc = centers.cuda()
    _lib.check(lib.anyloc_vlad_generate(_lib.ptr(x), None, _lib.ptr(cc), B, N, D, K, 0, 1, 1, _lib.ptr(ref), None,
                                        _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "generate")
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
