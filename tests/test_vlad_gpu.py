"""GPU parity: anyloc_vlad_generate (through the utilities mirror -> ctypes -> C ABI) against the
golden vectors produced by the reference's own code, and against the oracle on seeded inputs.
Tolerance: labels exact outside the fp64-ambiguous set (top1-top2 gap < 1e-5); descriptors
1e-4 relative (inf-norm) as BASELINE.json's north_star states."""
import numpy as np
import pytest
import torch

from oracle import anyloc_oracle as ao
from tests.util import load_cases, case_kwargs, rel_inf, make_vlad

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


@pytest.mark.parametrize("name", sorted(n for n in load_cases("vlad.npz") if not n.startswith("multi")))
def test_vlad_golden(u, name):
    c = load_cases("vlad.npz")[name]
    kw = case_kwargs(c)
    x, centers = torch.from_numpy(c["x"]), torch.from_numpy(c["centers"])
    v = make_vlad(u, centers.shape[0], centers, **kw)
    out = v.generate(x)
    assert out.device.type == "cpu" and out.shape == (centers.numel(),)
    lab = v.kmeans.predict(x)
    gap, _ = ao.label_margins(x, centers, kw.get("dist_mode", "cosine"))
    safe = gap > 1e-5
    if name.startswith("ties"):
        safe[:] = True          # exact ties / zero rows must resolve like the reference
    assert torch.equal(lab[safe], torch.from_numpy(c["labels"])[safe])
    if bool(safe.all()) or torch.equal(lab, torch.from_numpy(c["labels"])):
        assert rel_inf(out, c["out"]) < TOL
    else:   # a near-tie flipped: compare conditioned on the product's own labels
        ref = ao.vlad_generate(x, centers, labels=lab, **kw)
        assert rel_inf(out, ref) < TOL


def test_vlad_multi_golden_and_ragged(u):
    c = load_cases("vlad.npz")["multi_b4_n50_d32_k6"]
    x, centers = torch.from_numpy(c["x"]), torch.from_numpy(c["centers"])
    v = make_vlad(u, 6, centers)
    out = v.generate_multi(x)
    assert out.shape == (4, 6 * 32) and rel_inf(out, c["out"]) < TOL
    # numpy input, list input (ragged), device input
    assert rel_inf(v.generate_multi(x.numpy()), c["out"]) < TOL
    ragged = [x[0], x[1][:37], x[2][:1], x[3][:49]]
    outs = v.generate_multi(ragged)
    for o, q in zip(outs, ragged):
        assert rel_inf(o, ao.vlad_generate(q, centers)) < TOL
    dev_out = v.generate_multi(x.cuda())
    assert dev_out.is_cuda and rel_inf(dev_out.cpu(), c["out"]) < TOL


@pytest.mark.parametrize("N,D,K", [(1, 384, 8), (255, 384, 8), (256, 384, 8), (529, 1536, 32), (1369, 1024, 128),
                                   (530, 768, 1)])
@pytest.mark.parametrize("kind", ["clustered", "random"])
def test_vlad_vs_oracle(u, N, D, K, kind):
    if kind == "clustered":
        x, centers, _ = ao.clustered_features(N, D, K, seed=N + K)
    else:
        g = torch.Generator().manual_seed(N * 7 + K)
        x = torch.nn.functional.normalize(torch.randn(N, D, generator=g), dim=1)
        centers = 0.5 * torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1) * \
            (1 + 0.2 * torch.rand(K, 1, generator=g))
    v = make_vlad(u, K, centers)
    out = v.generate(x)
    lab = v.kmeans.predict(x)
    gap, lab64 = ao.label_margins(x, centers)
    safe = gap > 1e-5
    assert torch.equal(lab[safe], lab64[safe])
    ref = ao.vlad_generate(x, centers, labels=lab, dtype=torch.float64)
    assert rel_inf(out, ref) < TOL
    if kind == "clustered":     # large margins: unconditional end-to-end parity with the fp32 oracle
        assert rel_inf(out, ao.vlad_generate(x, centers)) < TOL
    assert abs(float(out.norm()) - 1.0) < 1e-5


def test_vlad_full_size_properties(u):
    """BASELINE config 2 size (B=32, N=529, D=1536, K=32): size-independent properties --
    unit global norm, per-block norm 1/sqrt(#non-empty), empty blocks exactly zero, batch result ==
    per-image result, permutation invariance over patches."""
    B, N, D, K = 32, 529, 1536, 32
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.nn.functional.normalize(torch.randn(B, N, D, device="cuda", generator=g), dim=-1)
    centers = 0.6 * torch.nn.functional.normalize(torch.randn(K, D, device="cuda", generator=g), dim=-1)
    centers[5] = 100.0 * centers[5]      # norm does not matter for cosine assignment
    v = make_vlad(u, K, centers.cpu())
    out = v.generate_multi(x)
    assert out.is_cuda and out.shape == (B, K * D)
    assert torch.allclose(out.norm(dim=1), torch.ones(B, device="cuda"), atol=1e-5)
    blocks = out.reshape(B, K, D).norm(dim=2)
    nonempty = (blocks > 0).sum(1, keepdim=True).float()
    expected = torch.where(blocks > 0, 1.0 / nonempty.sqrt(), torch.zeros_like(blocks))
    assert torch.allclose(blocks, expected, atol=1e-5)
    single = v.generate(x[3])
    assert torch.equal(single, out[3])
    perm = torch.randperm(N, device="cuda")
    assert rel_inf(v.generate(x[3][perm]).cpu(), out[3].cpu()) < 1e-5


def test_vlad_c5_shape_properties(u):
    """BASELINE config 5 VLAD shape (N=1369, D=1024, K=128; 8 images here): exactness against the oracle on the
    first image plus the size-independent properties on all."""
    B, N, D, K = 8, 1369, 1024, 128
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.nn.functional.normalize(torch.randn(B, N, D, device="cuda", generator=g), dim=-1)
    centers = 0.6 * x.reshape(-1, D)[torch.randperm(B * N, device="cuda", generator=g)[:K]].contiguous()
    v = make_vlad(u, K, centers.cpu())
    out = v.generate_multi(x)
    assert torch.allclose(out.norm(dim=1), torch.ones(B, device="cuda"), atol=1e-5)
    lab = v.kmeans.predict(x[0])
    gap, lab64 = ao.label_margins(x[0].cpu(), centers.cpu())
    assert torch.equal(lab.cpu()[gap > 1e-5], lab64[gap > 1e-5])
    ref = ao.vlad_generate(x[0].cpu(), centers.cpu(), labels=lab.cpu(), dtype=torch.float64)
    assert rel_inf(out[0].cpu(), ref) < TOL


@pytest.mark.parametrize("B,N,D,K", [(48, 1369, 256, 128), (64, 1369, 1024, 128), (200, 529, 64, 16)])
def test_vlad_many_tiles_per_cta(u, B, N, D, K):
    """More 128-row tiles of the coarse-score GEMM than SMs (the full BASELINE config 5 batch: 87 616 rows = 4-5 tiles
    per persistent CTA), and many images for the rescoring and accumulate3 passes.  Labels exact outside the
    fp64-ambiguous set on two images, descriptors against the oracle, batch == single image (bitwise)."""
    g = torch.Generator(device="cuda").manual_seed(B + D)
    x = torch.nn.functional.normalize(torch.randn(B, N, D, device="cuda", generator=g), dim=-1)
    centers = 0.6 * x.reshape(-1, D)[torch.randperm(B * N, device="cuda", generator=g)[:K]].contiguous()
    v = make_vlad(u, K, centers.cpu())
    out = v.generate_multi(x)
    assert torch.allclose(out.norm(dim=1), torch.ones(B, device="cuda"), atol=1e-5)
    lab_all = v.kmeans.predict(x.reshape(-1, D)).reshape(B, N)
    assert int(lab_all.min()) >= 0 and int(lab_all.max()) < K
    for b in (0, B - 1):
        gap, lab64 = ao.label_margins(x[b].cpu(), centers.cpu())
        assert torch.equal(lab_all[b].cpu()[gap > 1e-5], lab64[gap > 1e-5])
        ref = ao.vlad_generate(x[b].cpu(), centers.cpu(), labels=lab_all[b].cpu(), dtype=torch.float64)
        assert rel_inf(out[b].cpu(), ref) < TOL
        assert torch.equal(v.generate(x[b]), out[b])


def test_vlad_generate_multi_host_chunks(u):
    """The driver hands VLAD.generate_multi a CPU [n_imgs, n_patches, D] tensor (scripts/dino_v2_vlad.py:233-237: 32 GB for the
    10k-image database of c3); large host batches are streamed in chunks -- same result as one pass, and numpy in ->
    numpy-compatible tensor out (utilities.py:892-926)."""
    x, centers, _ = ao.clustered_features(12 * 300, 64, 8, seed=9)
    xb = x.reshape(12, 300, 64)
    v = make_vlad(u, 8, centers)
    whole = v.generate_multi(xb)
    v._host_chunk_bytes = 5 * 300 * 64 * 4 - 1            # forces chunks of 4 images
    chunked = v.generate_multi(xb)
    assert not chunked.is_cuda and torch.equal(whole, chunked)
    assert torch.equal(torch.as_tensor(v.generate_multi(xb.numpy())), whole)


def test_vlad_switches_and_errors(u):
    x, centers, _ = ao.clustered_features(64, 64, 4, seed=2)
    for kw in ({"intra_norm": False}, {"norm_descs": False}, {"dist_mode": "euclidean"}):
        v = make_vlad(u, 4, centers, **kw)
        assert rel_inf(v.generate(x * 1.7), ao.vlad_generate(x * 1.7, centers, **kw)) < TOL
    v = u.VLAD(4)
    with pytest.raises(AssertionError):
        v.generate(x)                                   # fit not called (utilities.py:948-949)
    with pytest.raises(ValueError):
        u.VLAD(4).fit(None)                             # utilities.py:778


@pytest.mark.parametrize("name", sorted(load_cases("vlad_soft.npz")))
def test_vlad_soft_golden(u, name):
    """vlad_mode="soft" against the reference's own outputs (tests/golden/vlad_soft.npz)."""
    c = load_cases("vlad_soft.npz")[name]
    kw = case_kwargs(c)
    x, centers = torch.from_numpy(c["x"]), torch.from_numpy(c["centers"])
    v = make_vlad(u, centers.shape[0], centers, vlad_mode="soft", **kw)
    out = v.generate_multi(x) if x.dim() == 3 else v.generate(x)
    assert out.device.type == "cpu" and out.shape == c["out"].shape
    assert rel_inf(out, torch.from_numpy(c["out"])) < TOL


@pytest.mark.parametrize("B,N,D,K,temp", [(3, 529, 1536, 32, 1.0), (2, 1369, 1024, 128, 30.0), (2, 77, 384, 200, 4.0)])
def test_vlad_soft_sizes(u, B, N, D, K, temp):
    """Pipeline-sized soft VLAD against the fp64 oracle, the assignment probabilities, and a ragged batch."""
    g = torch.Generator().manual_seed(B * N + K)
    x = torch.randn(B, N, D, generator=g) * (0.5 + torch.rand(B, N, 1, generator=g))
    centers = 0.7 * torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1)
    v = make_vlad(u, K, centers, vlad_mode="soft", soft_temp=temp)
    out, assign = v._run(x.cuda(), None, torch.device("cuda", 0), want_labels=True)
    for b in range(B):
        ref = ao.vlad_generate_soft_closed(x[b], centers, soft_temp=temp)
        assert rel_inf(out[b].cpu(), ref) < TOL
        a_ref = ao.vlad_soft_assign(x[b].double(), centers.double(), temp)
        assert float((assign[b].cpu().double() - a_ref).abs().max()) < 1e-5
    ragged = [x[0, :N - 7], x[1, :max(1, N // 3)]]
    outs = v.generate_multi(ragged)
    for q, o in zip(ragged, outs):
        assert rel_inf(o, ao.vlad_generate_soft_closed(q, centers, soft_temp=temp)) < TOL


def test_vlad_fit_cache_roundtrip(u, tmp_path):
    x, _, _ = ao.clustered_features(600, 64, 5, seed=3, kappa_noise=0.8)
    np.random.seed(42)
    v = u.VLAD(5, cache_dir=str(tmp_path / "c"))
    v.fit(x)
    assert v.desc_dim == 64 and v.c_centers.shape == (5, 64)
    assert (tmp_path / "c" / "c_centers.pt").exists() and v.can_use_cache_vlad()
    # oracle Lloyd from the same init reaches the same vocabulary (well separated data)
    from oracle import fpk_restated as fpk
    np.random.seed(42)
    km = fpk.KMeans(5, mode="cosine"); km.fit(torch.nn.functional.normalize(x))
    assert rel_inf(v.c_centers, km.centroids) < 1e-4
    v2 = u.VLAD(5, cache_dir=str(tmp_path / "c"))
    v2.fit(None)
    assert v2.desc_dim == 64 and torch.equal(v2.c_centers, v.c_centers.cpu())
    assert rel_inf(v2.generate(x[:100]), ao.vlad_generate(x[:100], v.c_centers.cpu())) < TOL


def test_vlad_prepared_equals_plain(u):
    """anyloc_vlad_prepare + anyloc_vlad_generate_prepared (centre prep once per vocabulary, the path VLAD.generate*
    takes) is bitwise identical to the plain anyloc_vlad_generate call, and the blob is reusable across calls: they
    leave it byte for byte as anyloc_vlad_prepare wrote it."""
    from anyloc_b200 import _lib
    lib = _lib.load()
    B, N, D, K = 3, 300, 384, 16
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(B, N, D, generator=g) * (0.5 + torch.rand(B, N, 1, generator=g))).cuda()
    centers = (0.5 * torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1)).cuda()
    res = []
    for prepared in (False, True):
        out = torch.empty(B, K * D, device="cuda")
        labels = torch.empty(B, N, dtype=torch.int32, device="cuda")
        ws = torch.empty(lib.anyloc_vlad_workspace_bytes(B, N, D, K), dtype=torch.uint8, device="cuda")
        if prepared:
            blob = torch.empty(lib.anyloc_vlad_prepared_bytes(D, K), dtype=torch.uint8, device="cuda")
            _lib.check(lib.anyloc_vlad_prepare(_lib.ptr(centers), D, K, 0, _lib.ptr(blob), blob.numel(), _lib.stream_ptr()),
                       "anyloc_vlad_prepare")
            torch.cuda.synchronize()
            blob0 = blob.clone()
            for _ in range(2):
                _lib.check(lib.anyloc_vlad_generate_prepared(_lib.ptr(x), None, _lib.ptr(centers), _lib.ptr(blob), blob.numel(),
                                                             B, N, D, K, 0, 1, 1, _lib.ptr(out), _lib.ptr(labels),
                                                             _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                           "anyloc_vlad_generate_prepared")
            torch.cuda.synchronize()
            assert torch.equal(blob, blob0), "generate_prepared changed the prepared blob"
        else:
            _lib.check(lib.anyloc_vlad_generate(_lib.ptr(x), None, _lib.ptr(centers), B, N, D, K, 0, 1, 1, _lib.ptr(out),
                                                _lib.ptr(labels), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                       "anyloc_vlad_generate")
        torch.cuda.synchronize()
        res.append((out.cpu(), labels.cpu()))
    assert torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][0], res[1][0])
    ref = ao.vlad_generate(x[1].cpu(), centers.cpu(), labels=res[0][1][1].long(), dtype=torch.float64)
    assert rel_inf(res[0][0][1], ref) < TOL


# ---- v3 pipeline corners (tensor-core assignment needs >= 256 rows per call; these shapes take that route or, for
# K > 128, the v2 assignment in front of the v3 accumulate kernel)
def _check_against_oracle(v, x, centers, dist_mode="cosine", **kw):
    out = v.generate(x)
    lab = v.kmeans.predict(x)
    gap, lab64 = ao.label_margins(x, centers, dist_mode)
    safe = gap > 1e-5
    assert torch.equal(lab[safe], lab64[safe])
    ref = ao.vlad_generate(x, centers, labels=lab, dtype=torch.float64, dist_mode=dist_mode, **kw)
    assert rel_inf(out, ref) < TOL
    return out


def test_vlad_v3_ragged_large(u):
    g = torch.Generator().manual_seed(21)
    centers = 0.6 * torch.nn.functional.normalize(torch.randn(16, 384, generator=g), dim=1)
    qs = [torch.randn(n, 384, generator=g) for n in (300, 257, 1, 411)]
    v = make_vlad(u, 16, centers)
    outs = v.generate_multi(qs)                     # padded to [4, 411, 384] with n_valid
    for q, o in zip(qs, outs):
        lab = v.kmeans.predict(q)
        ref = ao.vlad_generate(q, centers, labels=lab, dtype=torch.float64)
        assert rel_inf(o, ref) < TOL


@pytest.mark.parametrize("N,D,K", [(300, 384, 200), (300, 100, 8), (700, 36, 5), (260, 2048, 128)])
def test_vlad_v3_odd_shapes(u, N, D, K):
    g = torch.Generator().manual_seed(N + D + K)
    x = torch.randn(N, D, generator=g) * (0.3 + torch.rand(N, 1, generator=g))
    centers = 0.5 * torch.nn.functional.normalize(torch.randn(K, D, generator=g), dim=1) * (1 + 0.3 * torch.rand(K, 1, generator=g))
    _check_against_oracle(make_vlad(u, K, centers), x, centers)


def test_vlad_v3_euclidean_and_switches_large(u):
    g = torch.Generator().manual_seed(33)
    x = torch.randn(400, 256, generator=g) * 1.3
    centers = torch.randn(12, 256, generator=g) * 0.4
    for kw in ({"dist_mode": "euclidean"}, {"intra_norm": False}, {"norm_descs": False}):
        v = make_vlad(u, 12, centers, **kw)
        dm = kw.get("dist_mode", "cosine")
        okw = {k: val for k, val in kw.items() if k != "dist_mode"}
        _check_against_oracle(v, x, centers, dist_mode=dm, **okw)
