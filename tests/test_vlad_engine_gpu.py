"""Every VLAD aggregation route, the soft path, the k-means update and the residual-cache kernels, checked element by
element against fp64 through the C ABI.

Hard VLAD, conditioned on the product's own labels (labels_out).  The fp64 reference is

    x^_q = x_q / max(|x_q|, 1e-12)  (x_q when norm_descs is off)     u_k = sum_{l_q = k} (x^_q - c_k)
    s_k  = 1 / max(|u_k|, 1e-12)    (1 when intra_norm is off)        g = 1 / max(|(s_k u_k)_k|, 1e-12)
    v64  = g s_k u_k

and every element must satisfy, with u = 2^-24 and the sqrt-style constant of test_gemm_engine_gpu.py,

    |v - v64|_kj <= 16 u ( g s_k E_kj + (sqrt(D + K) + rho_k) |v64_kj| ),
    E_kj = sqrt(n_k + 2) sum_{l_q = k} (|x^_qj| + |c_kj|),   rho_k = |E_k| / |u_k|  (intra_norm)  or  |E| / |U|.

Derivation from the kernels' arithmetic (accumulate3 and accumulate2 do the same per element):
  * 1/|x_q| comes from an fp32 sum of D squares (D/128 terms per lane, then a 5-level warp tree), a sqrt and a
    division: a relative error of about (D/256 + 8) u, common to the row.  fl(fl(x_qj s_q) - c_kj) then adds two
    roundings, so each term is off by at most ~(D/256 + 10) u |x^_qj| + u |c_kj|.
  * The n_k terms are summed in one fixed order (rows in tasks of <= 64, tasks combined in order): gamma_{n_k} times
    the sum of the terms' magnitudes, taken in the sqrt form sqrt(n_k) u as for the GEMM.  The "+2" keeps a single-row
    cluster above the row-norm error, and 16 u sqrt(n_k + 2) >= 27 u covers it for D <= 2048.  This gives g s_k E_kj.
  * The block norm |u_k| and the global norm are fp32 sums of D (per slice: 4 per lane + warp tree, then the slices)
    and K squares, a sqrt and a reciprocal each; the two scalings round twice: sqrt(D + K) u |v64|.
  * The block is divided by the norm of the COMPUTED sum, whose relative error is at most |E_k| / |u_k| (or, without
    intra-normalisation, the whole descriptor's |E| / |U| through g): rho_k.
Soft VLAD evaluates the closed form V_k = K sum_q a_qk x^_q - (sum_q a_qk) sum_c c_c (one fma chain over the image's
rows, one sum over the K centres), so E_kj = sqrt(n + K + 2) (K sum_q a_qk |x^_qj| + sum_q a_qk sum_c |c_cj|), with the
product's own assignment a.  The soft assignment is bounded against an fp64 softmax of T cos(x_q, c_k):
    |a - a64|_qk <= a64_qk (2 max_c ds_qc + 16 u (|s_qk - max_c s_qc| + sqrt(K) + 4)) + 1e-37,
    ds_qc = 16 u T sqrt(D + 2) sum_i |x_qi c^_ci| / |x_q|,
i.e. the logits' fp32 dot-product error moves a softmax by at most twice itself, plus the exp argument, the sum of the K
exponentials and the final scaling.  The k-means mean of cluster k is a sum over <= rows_per rows per chunk plus the
chunks in order, then one division: |c - c64|_kj <= 16 u (sqrt(n_k + chunks + 2) sum_{l_q = k} |x_qj| / n_k + |c64_kj|).

Three wrong references must each violate the hard bound on the same kernel output (one row dropped from a cluster of
>= 65 rows, features truncated to tf32 before aggregating, one block not intra-normalised), so the bound is tight
enough to catch them.  Every route of vlad_generate_impl is reached by shape and identified by the number of launches
a call makes (anyloc_launch_count) or, for the two normalisations of accumulate3, by the number of CTAs against the SM
count; NaN canaries surround every output.  The worst bound ratio per (route, input family) is printed at the end."""
import ctypes as C

import pytest
import torch

from tests.util import dptr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ACC = 16
LEAD = 16                                   # canary elements before and after every output (64 B: float4 alignment)
NAN32 = 0x7FC0DEAD                          # a quiet-NaN pattern no kernel writes
COS, EUC = 0, 1
ERR_ARG = -1
WORST = {}                                  # (route, family) -> worst ratio seen


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    yield _lib
    if WORST:
        print("\n[worst |v - v64| / bound per route and family]")
        for (route, fam), r in sorted(WORST.items()):
            print(f"  {route:<28} {fam:<22} {r:.3f}")


@pytest.fixture(scope="module")
def sms(L):
    n = C.c_int(0)
    assert L.load().anyloc_device_info(C.byref(n), None) >= 90
    return n.value


def note(route, fam, r):
    WORST[(route, fam)] = max(WORST.get((route, fam), 0.0), r)
    print(f"{route} / {fam}: worst ratio {r:.3f}")


# ------------------------------------------------------------------------------------------------ dispatch mirror
# vlad_generate_impl, read off vlad.cu: accumulate3 when its shared memory fits 100 KB, else accumulate2 with
# min(4, 200 KB / (K 128 4) - 1) row-splitting warps, else an error.
def acc3_smem(N, K):
    tasks, slots = N // 64 + K + 1, 2 * (N // 64) + 2
    return (4 * N + 3 * (K + 1) + 8 * K + 2 * K + tasks + 4) * 4 + slots * 512


def acc2_warps(K):
    return min(4, (200 * 1024) // (K * 128 * 4) - 1)


def accumulate_route(N, D, K):
    if acc3_smem(N, K) <= 100 * 1024 and N * D < 2 ** 31:
        return "accumulate3"
    return "accumulate2" if acc2_warps(K) >= 1 else "error"


def fast_assign(R, D):
    return D <= 2048 and R >= 256


def expected_launches(B, N, D, K, prepared=False):
    """centre prep (unless the prepared blob is used), coarse GEMM + rescore or the FFMA assignment, then accumulate3
    alone or accumulate2 + normalise"""
    route = accumulate_route(N, D, K)
    prep = 0 if prepared else 1
    assign = 2 if fast_assign(B * N, D) else 1
    return prep + assign + (1 if route == "accumulate3" else 2)


# ------------------------------------------------------------------------------------------------------- buffers
def canary(n, dtype=torch.float32):
    buf = torch.full((LEAD + n + LEAD,), NAN32, dtype=torch.int32, device="cuda")
    return buf if dtype == torch.int32 else buf.view(torch.float32)


def inner(buf, n):
    return buf[LEAD:LEAD + n]


def assert_canaries(buf, n, what, written=True):
    bits = buf.view(torch.int32)
    outside = torch.cat([bits[:LEAD], bits[LEAD + n:]]) if written else bits
    bad = int((outside != NAN32).sum())
    assert bad == 0, f"{what}: {bad} canary words overwritten"


def workspace(nbytes):
    return torch.empty(int(nbytes), dtype=torch.uint8, device="cuda")


def generate(L, x, centers, B, N, D, K, *, dist=COS, norm=1, intra=1, n_valid=None, blob=None, ws=None,
             expect_rc=0):
    """one anyloc_vlad_generate(_prepared) call -> (vlad [B,K,D], labels [B,N], launches)"""
    lib = L.load()
    out, lab = canary(B * K * D), canary(B * N, torch.int32)
    ws = workspace(lib.anyloc_vlad_workspace_bytes(B, N, D, K)) if ws is None else ws
    n0 = L.launch_count()
    if blob is None:
        rc = lib.anyloc_vlad_generate(dptr(x), dptr(n_valid), dptr(centers), B, N, D, K, dist, norm, intra,
                                      dptr(out, LEAD), dptr(lab, LEAD), dptr(ws), ws.numel(), L.stream_ptr())
    else:
        rc = lib.anyloc_vlad_generate_prepared(dptr(x), dptr(n_valid), dptr(centers), dptr(blob), blob.numel(), B, N,
                                               D, K, dist, norm, intra, dptr(out, LEAD), dptr(lab, LEAD), dptr(ws),
                                               ws.numel(), L.stream_ptr())
    launches = L.launch_count() - n0
    torch.cuda.synchronize()
    assert rc == expect_rc, (rc, L.last_error())
    assert_canaries(out, B * K * D, "vlad", written=rc == 0)
    assert_canaries(lab, B * N, "labels", written=rc == 0)
    return inner(out, B * K * D).view(B, K, D), inner(lab, B * N).view(B, N), launches


def prepare(L, centers, D, K, dist=COS):
    lib = L.load()
    blob = workspace(lib.anyloc_vlad_prepared_bytes(D, K))
    L.check(lib.anyloc_vlad_prepare(dptr(centers), D, K, dist, dptr(blob), blob.numel(), L.stream_ptr()), "prepare")
    return blob


def generate_soft(L, x, centers, B, N, D, K, T, *, norm=1, intra=1, n_valid=None):
    lib = L.load()
    out, asg = canary(B * K * D), canary(B * N * K)
    ws = workspace(lib.anyloc_vlad_workspace_bytes(B, N, D, K))
    L.check(lib.anyloc_vlad_generate_soft(dptr(x), dptr(n_valid), dptr(centers), B, N, D, K, C.c_float(T), norm,
                                          intra, dptr(out, LEAD), dptr(asg, LEAD), dptr(ws), ws.numel(),
                                          L.stream_ptr()), "generate_soft")
    torch.cuda.synchronize()
    assert_canaries(out, B * K * D, "soft vlad")
    assert_canaries(asg, B * N * K, "soft assign")
    return inner(out, B * K * D).view(B, K, D), inner(asg, B * N * K).view(B, N, K)


# --------------------------------------------------------------------------------------------------- references
def trunc_tf32(t):
    return (t.contiguous().view(torch.int32) & -8192).view(torch.float32)


def normalise(u64, E, intra, skip_intra_block=None):
    """(v64, bound) from the fp64 block sums u64 [B,K,D] and their error magnitudes E [B,K,D] (see the docstring)"""
    B, K, D = u64.shape
    un = u64.norm(dim=2)                                             # [B,K]
    s = 1.0 / un.clamp_min(1e-12) if intra else torch.ones_like(un)
    if skip_intra_block is not None:
        s[skip_intra_block] = 1.0
    blocks = s[:, :, None] * u64
    g = 1.0 / blocks.reshape(B, -1).norm(dim=1).clamp_min(1e-12)    # [B]
    v64 = g[:, None, None] * blocks
    if intra:
        rho = torch.where(un > 0, E.norm(dim=2) / un.clamp_min(1e-300), torch.zeros_like(un))[:, :, None]
    else:
        Un = u64.reshape(B, -1).norm(dim=1)
        rho = torch.where(Un > 0, E.reshape(B, -1).norm(dim=1) / Un.clamp_min(1e-300), torch.zeros_like(Un))
        rho = rho[:, None, None]
    bound = C_ACC * U * (g[:, None, None] * s[:, :, None] * E + ((D + K) ** 0.5 + rho) * v64.abs())
    return v64, bound


def hard_reference(x, centers, labels, norm=1, intra=1, mutate=None):
    """fp64 descriptor conditioned on `labels` [B,N] (-1: ignored) and its bound.  mutate: None, "drop_row" (one row
    of the first cluster with >= 65 rows left out), "tf32" (features truncated to tf32), "skip_intra" (block of the
    largest cluster of image 0 not intra-normalised)."""
    B, N = labels.shape
    K, D = centers.shape
    x64 = x.reshape(B, N, D).double()
    c64 = centers.double()
    lab = labels.long()
    valid = lab >= 0
    xs = trunc_tf32(x.reshape(B, N, D)).double() if mutate == "tf32" else x64
    xs = torch.where(valid[:, :, None], xs, torch.zeros((), dtype=torch.float64, device=x.device))
    if norm:
        xn = torch.where(valid, x64.nan_to_num(0.0).norm(dim=2), torch.ones((), dtype=torch.float64, device=x.device))
        xs = xs / xn.clamp_min(1e-12)[:, :, None]
    idx = torch.arange(B, device=x.device)[:, None] * K + lab.clamp_min(0)
    cnt = torch.bincount(idx[valid], minlength=B * K)
    skip = None
    if mutate == "drop_row":
        big = int(torch.nonzero(cnt >= 65)[0])
        q = int(torch.nonzero(((idx == big) & valid).reshape(-1))[-1])
        valid = valid.clone()
        valid.view(-1)[q] = False
    if mutate == "skip_intra":
        skip = (0, int(cnt[:K].argmax()))
    vi, vr = idx[valid], xs[valid]
    cl = c64[lab[valid]]
    u64 = torch.zeros(B * K, D, dtype=torch.float64, device=x.device).index_add_(0, vi, vr - cl)
    E = torch.zeros(B * K, D, dtype=torch.float64, device=x.device).index_add_(0, vi, vr.abs() + cl.abs())
    E = E * (torch.bincount(vi, minlength=B * K).double() + 2).sqrt()[:, None]
    v64, bound = normalise(u64.view(B, K, D), E.view(B, K, D), intra, skip)
    return v64, bound, cnt.view(B, K)


def ratio(v, v64, bound):
    """max |v - v64| / bound; where the bound is 0 (empty blocks) v must be exactly 0"""
    d = (v.double() - v64).abs()
    assert bool(torch.isfinite(v).all()), "non-finite output"
    zero = bound == 0
    assert int((d[zero] != 0).sum()) == 0, "an empty block is not exactly 0"
    return float((d[~zero] / bound[~zero]).max()) if bool((~zero).any()) else 0.0


def fp64_labels(x, centers, dist):
    """fp64 argmax labels and the rows whose top-1/top-2 gap exceeds 1e-5 of the score scale"""
    x64, c64 = x.double(), centers.double()
    if dist == COS:
        chat, bias = c64 / (c64.norm(dim=1, keepdim=True) + 1e-8), torch.zeros(c64.shape[0], dtype=torch.float64,
                                                                                device=x.device)
    else:
        chat, bias = c64, -0.5 * (c64 * c64).sum(1)
    s = x64 @ chat.T + bias
    top = s.topk(min(2, s.shape[1]), dim=1).values
    scale = x64.norm(dim=1) * chat.norm(dim=1).max() + bias.abs().max()
    gap = (top[:, 0] - top[:, 1]) if s.shape[1] > 1 else torch.full_like(scale, float("inf"))
    return s.argmax(1), gap > 1e-5 * scale


def check_labels(x, centers, labels, dist, what):
    lab64, safe = fp64_labels(x.reshape(-1, centers.shape[1]), centers, dist)
    lab = labels.reshape(-1).long()
    assert float(safe.double().mean()) > 0.5, f"{what}: fewer than half the rows are unambiguous"
    bad = int((lab[safe] != lab64[safe]).sum())
    assert bad == 0, f"{what}: {bad} labels differ from the fp64 argmax outside the 1e-5 gap set"


# ------------------------------------------------------------------------------------------------------- inputs
def make_inputs(family, B, N, D, K, seed, target=None):
    """x [B,N,D], centres [K,D] on the device.  target [B,N]: rows placed on these clusters with a large margin."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    rand = lambda *s: torch.rand(*s, device="cuda", generator=g)
    base = torch.nn.functional.normalize(rn(K, D), dim=1)
    if target is not None or family == "clustered":
        lab = target if target is not None else torch.randint(0, K, (B, N), device="cuda", generator=g)
        x = base[lab] + (0.1 if target is not None else 0.7) * rn(B, N, D) / D ** 0.5
        centers = 0.6 * base * (1 + 0.2 * rand(K, 1))
    elif family == "random":
        x = rn(B, N, D) * (0.5 + rand(B, N, 1))
        centers = 0.5 * base * (1 + 0.3 * rand(K, 1))
    elif family == "spread":                                          # row norms 1e-3 .. 1e3
        x = rn(B, N, D) / D ** 0.5 * 10.0 ** (6 * rand(B, N, 1) - 3)
        centers = 0.5 * base * (1 + 0.3 * rand(K, 1))
    elif family == "common":                                          # DINOv2-like: a large mean shared by all rows
        m = torch.nn.functional.normalize(rn(1, D), dim=1)
        x = m + 0.15 * rn(B, N, D) / D ** 0.5
        centers = m + 0.15 * rn(K, D) / D ** 0.5
    else:
        raise ValueError(family)
    return x.float().contiguous(), centers.float().contiguous()


def permuted_targets(B, counts, seed):
    """labels [B, sum(counts)]: cluster k repeated counts[k] times, rows shuffled per image"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.repeat_interleave(torch.arange(len(counts), device="cuda"), torch.tensor(counts, device="cuda"))
    return torch.stack([lab[torch.randperm(lab.numel(), device="cuda", generator=g)] for _ in range(B)])


# ----------------------------------------------------------------------------------------- hard VLAD by route
def run_hard(L, route_name, fam, B, N, D, K, *, case="", dist=COS, norm=1, intra=1, target=None, seed=0):
    x, centers = make_inputs(fam, B, N, D, K, seed, target)
    v, lab, launches = generate(L, x, centers, B, N, D, K, dist=dist, norm=norm, intra=intra)
    assert launches == expected_launches(B, N, D, K), (launches, route_name)
    assert int(lab.min()) >= 0 and int(lab.max()) < K
    if target is not None:
        assert torch.equal(lab.long(), target), "rows did not land on the clusters they were built for"
    check_labels(x, centers, lab, dist, route_name)
    v64, bound, cnt = hard_reference(x, centers, lab, norm, intra)
    r = ratio(v, v64, bound)
    note(route_name, f"{fam}:{case}" if case else fam, r)
    assert r <= 1.0, (route_name, fam, case, r)
    return x, centers, v, lab, cnt


HARD_CASES = {
    # name: (B, N, D, K, family, kwargs); accumulate3 with the distributed normalise unless said otherwise
    "c2_width": (4, 529, 1536, 32, "clustered", {}),
    "c5_width": (2, 1369, 1024, 128, "random", {}),
    "D36": (3, 300, 36, 8, "random", {}),
    "D100": (3, 300, 100, 8, "clustered", {}),
    "D1028": (2, 400, 1028, 16, "random", {}),
    "K1": (2, 300, 128, 1, "random", {}),
    "K33": (2, 500, 256, 33, "clustered", {}),
    "K201": (2, 400, 128, 201, "random", {}),
    "K1000": (1, 300, 64, 1000, "random", {}),
    "intra_off": (3, 400, 256, 12, "random", {"intra": 0}),
    "norm_descs_off_spread": (3, 400, 256, 12, "spread", {"norm": 0}),
    "spread": (3, 400, 256, 12, "spread", {}),
    "euclidean": (3, 400, 256, 12, "random", {"dist": EUC}),
    "euclidean_no_norm": (2, 300, 384, 16, "clustered", {"dist": EUC, "norm": 0}),
    "tiny_ffma_assign": (1, 200, 384, 8, "clustered", {}),
}


@pytest.mark.parametrize("name", sorted(HARD_CASES))
def test_hard_bound_accumulate3(L, sms, name):
    B, N, D, K, fam, kw = HARD_CASES[name]
    assert accumulate_route(N, D, K) == "accumulate3"
    if (D + 127) // 128 * B <= sms:
        route = "accumulate3/distributed"
    else:
        route = "accumulate3/unclassified"
    run_hard(L, route, fam, B, N, D, K, case=name, seed=len(name), **kw)


@pytest.mark.parametrize("layout", ["one_cluster", "exact64", "exact65", "empty_clusters"])
def test_hard_accumulate3_structure(L, layout):
    """task boundaries of accumulate3: one cluster of 3000 rows (47 tasks combined from slots), every cluster exactly
    64 rows (one task each) or 65 rows (two tasks each: the most slots), half the clusters empty (exactly 0)"""
    D = 256
    if layout == "one_cluster":
        K, counts = 8, [3000, 0, 0, 0, 0, 0, 0, 0]
    elif layout == "exact64":
        K, counts = 16, [64] * 16
    elif layout == "exact65":
        K, counts = 16, [65] * 16
    else:
        K, counts = 32, [37 if k % 2 else 0 for k in range(32)]
    B, N = 2, sum(counts)
    assert accumulate_route(N, D, K) == "accumulate3"
    target = permuted_targets(B, counts, seed=K)
    _, _, v, _, cnt = run_hard(L, "accumulate3/structure", "targets", B, N, D, K, case=layout, target=target,
                               seed=N)
    empty = cnt == 0
    assert bool((v[empty] == 0).all()) and bool((v[~empty].norm(dim=1) > 0).all())


def test_hard_bound_catches_wrong_references(L):
    """the bound is tight enough to matter: on the same kernel output, a reference with one row dropped from a
    cluster of >= 65 rows, with tf32-truncated features, or with one block not intra-normalised violates it"""
    B, N, D, K = 2, 1040, 256, 16
    target = permuted_targets(B, [65] * K, seed=3)
    x, centers, v, lab, _ = run_hard(L, "accumulate3/structure", "targets", B, N, D, K, case="mutation_base",
                                     target=target, seed=5)
    for mutate in ("drop_row", "tf32", "skip_intra"):
        v64, bound, _ = hard_reference(x, centers, lab, mutate=mutate)
        d = (v.double() - v64).abs()
        r = float((d / bound.clamp_min(1e-300)).max())
        print(f"mutation {mutate}: worst ratio {r:.3g}")
        assert r > 1.0, f"the bound does not catch the {mutate} mutation (worst ratio {r:.3g})"


def test_hard_last_cta_normalise(L, sms):
    """nslices * B > 8 * SMs: more CTAs than can be co-resident (256 threads cap occupancy at 8), so the last CTA of each
    image normalises it.  Two calls on one workspace (the done[b] tickets must be reset), images bitwise equal to
    single-image calls, which take the distributed normalise"""
    for fam, B, N, D, K in (("random", 8 * sms + 144, 300, 128, 16), ("clustered", 8 * sms // 12 + 2, 529, 1536, 32)):
        nslices = (D + 127) // 128
        assert nslices * B > 8 * sms and nslices <= sms
        x, centers = make_inputs(fam, B, N, D, K, seed=B)
        ws = workspace(L.load().anyloc_vlad_workspace_bytes(B, N, D, K))
        v1, lab, n1 = generate(L, x, centers, B, N, D, K, ws=ws)
        v2, lab2, n2 = generate(L, x, centers, B, N, D, K, ws=ws)
        assert n1 == n2 == expected_launches(B, N, D, K)
        assert torch.equal(v1, v2) and torch.equal(lab, lab2), "second call on the same workspace differs"
        v64, bound, _ = hard_reference(x, centers, lab)
        r = ratio(v1, v64, bound)
        note("accumulate3/last_cta", f"{fam}:D{D}", r)
        assert r <= 1.0
        check_labels(x[:8], centers, lab[:8], COS, "last_cta")
        for b in (0, 1, B // 2, B - 1):
            vs, ls, _ = generate(L, x[b:b + 1].contiguous(), centers, 1, N, D, K)
            assert torch.equal(vs[0], v1[b]) and torch.equal(ls[0], lab[b]), f"image {b}: batch != single image"


@pytest.mark.parametrize("N,K", [(3942, 32), (5329, 32), (4096, 128), (3000, 200)])
def test_hard_accumulate2_prepared(L, N, K):
    """N beyond accumulate3's 100 KB (the demo's 1024-px ViT-G images: 73 x 54 and 73 x 73 patches): accumulate2 with
    4, 2 or 1 row-splitting warps + the normalise launch.  Bound, batch == single image, prepared == plain with one
    launch fewer (no centre prep), and the prepared blob is left as it was"""
    D = 1536 if K == 32 else 1024
    B = 2
    assert accumulate_route(N, D, K) == "accumulate2"
    print(f"accumulate2 N={N} K={K}: {acc2_warps(K)} row-splitting warps")
    x, centers = make_inputs("clustered" if K == 32 else "random", B, N, D, K, seed=N)
    v, lab, launches = generate(L, x, centers, B, N, D, K)
    assert launches == expected_launches(B, N, D, K) == 5
    check_labels(x, centers, lab, COS, "accumulate2")
    v64, bound, _ = hard_reference(x, centers, lab)
    r = ratio(v, v64, bound)
    note(f"accumulate2/{acc2_warps(K)}warps", f"N{N}:K{K}", r)
    assert r <= 1.0
    vs, ls, _ = generate(L, x[1:].contiguous(), centers, 1, N, D, K)
    assert torch.equal(vs[0], v[1]) and torch.equal(ls[0], lab[1]), "batch != single image"
    blob = prepare(L, centers, D, K)
    torch.cuda.synchronize()
    blob0 = blob.clone()
    vp, lp, lp_launches = generate(L, x, centers, B, N, D, K, blob=blob)
    assert lp_launches == expected_launches(B, N, D, K, prepared=True) == 4
    assert torch.equal(vp, v) and torch.equal(lp, lab), "prepared != plain"
    assert torch.equal(blob, blob0), "generate_prepared changed the prepared blob"


@pytest.mark.parametrize("D", [512, 516, 1024, 1028, 2048, 2052, 3072])
def test_assign_routes(L, D):
    """anyloc_vlad_assign across the rescore kernel's register tiers (<4>: D <= 512, <8>: <= 1024, <16>: <= 2048) and
    the FFMA kernel above 2048: labels equal the fp64 argmax outside the 1e-5 gap set"""
    lib = L.load()
    R, K = 1000, 64
    for dist in (COS, EUC):
        x, centers = make_inputs("random", 1, R, D, K, seed=D + dist)
        x = x.view(R, D)
        lab = canary(R, torch.int32)
        ws = workspace(lib.anyloc_vlad_workspace_bytes(1, R, D, K))
        n0 = L.launch_count()
        L.check(lib.anyloc_vlad_assign(dptr(x), dptr(centers), R, D, K, dist, dptr(lab, LEAD), dptr(ws), ws.numel(),
                                       L.stream_ptr()), "assign")
        launches = L.launch_count() - n0
        torch.cuda.synchronize()
        assert launches == (3 if fast_assign(R, D) else 2), (D, launches)
        assert_canaries(lab, R, "labels")
        check_labels(x, centers, inner(lab, R), dist, f"assign D={D}")


def test_envelope_errors(L):
    """outside the shared-memory envelope the call returns an error and writes nothing: hard VLAD at K = 256 with
    N = 4000 and at K = 1000 with N = 2000 (too many rows for accumulate3's 100 KB, too many clusters for one
    accumulate2 row-splitting warp), and a k-means update whose K needs more than 220 KB"""
    for B, N, D, K in ((1, 4000, 128, 256), (1, 2000, 64, 1000)):
        assert accumulate_route(N, D, K) == "error"
        x, centers = make_inputs("random", B, N, D, K, seed=K)
        generate(L, x, centers, B, N, D, K, expect_rc=ERR_ARG)
        assert "shared memory" in L.last_error()
    lib = L.load()
    R, D, K = 1000, 128, 437                                         # (K 128 + K) 4 > 220 KB
    x = torch.randn(R, D, device="cuda")
    labels = torch.randint(0, K, (R,), device="cuda", dtype=torch.int32)
    old = torch.randn(K, D, device="cuda")
    new, err = canary(K * D), canary(1)
    ws = workspace(lib.anyloc_kmeans_workspace_bytes(R, D, K))
    rc = lib.anyloc_kmeans_update(dptr(x), dptr(labels), dptr(old), R, D, K, dptr(new, LEAD), dptr(err, LEAD),
                                  dptr(ws), ws.numel(), L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == ERR_ARG, rc
    assert_canaries(new, K * D, "kmeans centres", written=False)
    assert_canaries(err, 1, "kmeans err", written=False)


# ------------------------------------------------------------------------------------------- ragged batches, NaN
def test_hard_ragged_nan_padding(L):
    """rows at or beyond n_valid[b] hold NaN: labels -1 there, and each image bitwise equal to a call on its valid rows"""
    B, N, D, K = 4, 411, 384, 16
    nv = [300, 257, 1, 411]
    x, centers = make_inputs("clustered", B, N, D, K, seed=21)
    for b, n in enumerate(nv):
        x[b, n:] = float("nan")
    n_valid = torch.tensor(nv, dtype=torch.int32, device="cuda")
    v, lab, _ = generate(L, x, centers, B, N, D, K, n_valid=n_valid)
    for b, n in enumerate(nv):
        assert bool((lab[b, n:] == -1).all()) and bool((lab[b, :n] >= 0).all())
        vs, ls, _ = generate(L, x[b, :n].contiguous(), centers, 1, n, D, K)
        assert torch.equal(vs[0], v[b]) and torch.equal(ls[0], lab[b, :n]), f"image {b}: ragged != unpadded"
    v64, bound, _ = hard_reference(x, centers, lab)
    r = ratio(v, v64, bound)
    note("accumulate3/distributed", "ragged_nan", r)
    assert r <= 1.0


# ---------------------------------------------------------------------------------------------------- soft VLAD
def soft_reference(x, centers, a, n_valid, norm=1, intra=1):
    B, N, D = x.shape
    K = centers.shape[0]
    x64, c64, a64 = x.double(), centers.double(), a.double()
    valid = torch.arange(N, device=x.device)[None, :] < n_valid[:, None]
    x64 = torch.where(valid[:, :, None], x64, torch.zeros((), dtype=torch.float64, device=x.device))
    a64 = torch.where(valid[:, :, None], a64, torch.zeros((), dtype=torch.float64, device=x.device))
    if norm:
        x64 = x64 / x64.norm(dim=2, keepdim=True).clamp_min(1e-12)
    w = a64.sum(1)                                                    # [B,K]
    u64 = K * torch.einsum("bnk,bnd->bkd", a64, x64) - w[:, :, None] * c64.sum(0)
    E = K * torch.einsum("bnk,bnd->bkd", a64, x64.abs()) + w[:, :, None] * c64.abs().sum(0)
    E = E * (n_valid.double() + K + 2).sqrt()[:, None, None]
    return normalise(u64, E, intra)


def soft_assign_reference(x, centers, T):
    """fp64 softmax(T cos) and its bound (docstring)"""
    x64, c64 = x.double(), centers.double()
    K, D = c64.shape
    chat = c64 / c64.norm(dim=1, keepdim=True).clamp_min(1e-8)
    xn = x64.norm(dim=1, keepdim=True).clamp_min(1e-8)
    s = T * (x64 @ chat.T) / xn
    a64 = torch.softmax(s, dim=1)
    ds = C_ACC * U * T * (D + 2) ** 0.5 * (x64.abs() @ chat.abs().T) / xn
    m = s.max(1, keepdim=True).values
    bound = a64 * (2 * ds.max(1, keepdim=True).values + C_ACC * U * ((s - m).abs() + K ** 0.5 + 4)) + 1e-37
    return a64, bound


@pytest.mark.parametrize("fam,B,N,D,K,T", [("random", 3, 529, 1536, 32, 1.0), ("clustered", 2, 1369, 1024, 128, 30.0),
                                           ("random", 2, 300, 384, 200, 100.0), ("common", 3, 529, 1536, 32, 1.0),
                                           ("common", 2, 400, 384, 37, 30.0), ("spread", 2, 300, 256, 40, 100.0)])
def test_soft_bound(L, fam, B, N, D, K, T):
    """soft VLAD within the closed-form bound conditioned on the product's assignment, the assignment within its
    bound against the fp64 softmax, and the pipeline's 1e-4 (max|dv| / max|v64|) -- the "common" family (features close
    to the centres' mean, as DINOv2's are) is where the closed form K sum a x^ - (sum a) sum c cancels"""
    x, centers = make_inputs(fam, B, N, D, K, seed=N + K)
    v, a = generate_soft(L, x, centers, B, N, D, K, T)
    n_valid = torch.full((B,), N, device="cuda")
    v64, bound = soft_reference(x, centers, a, n_valid)
    r = ratio(v, v64, bound)
    rel = float((v.double() - v64).abs().max() / v64.abs().max())
    a64, abound = soft_assign_reference(x.view(-1, D), centers, T)
    ra = float(((a.view(-1, K).double() - a64).abs() / abound).max())
    note("soft", f"{fam}:T{T:g}", r)
    note("soft_assign", f"{fam}:T{T:g}", ra)
    print(f"soft {fam} T={T}: max|dv|/max|v64| {rel:.2e}")
    assert r <= 1.0 and ra <= 1.0
    assert rel < 1e-4


def test_soft_ragged_nan_padding(L):
    """padded rows hold NaN: the descriptors stay finite and within the bound, padded assignments are exactly 0, and
    valid rows are bitwise what a batch with zero padding gives"""
    B, N, D, K, T = 3, 300, 384, 37, 30.0
    nv = [300, 123, 1]
    x, centers = make_inputs("random", B, N, D, K, seed=77)
    n_valid = torch.tensor(nv, dtype=torch.int32, device="cuda")
    xz = x.clone()
    for b, n in enumerate(nv):
        x[b, n:] = float("nan")
        xz[b, n:] = 0.0
    v, a = generate_soft(L, x, centers, B, N, D, K, T, n_valid=n_valid)
    vz, az = generate_soft(L, xz, centers, B, N, D, K, T, n_valid=n_valid)
    assert bool(torch.isfinite(v).all()), "NaN padding leaked into the soft descriptors"
    for b, n in enumerate(nv):
        assert bool((a[b, n:] == 0).all()) and not bool(torch.signbit(a[b, n:]).any()), "padded assignment != +0"
    assert torch.equal(v, vz) and torch.equal(a, az)
    v64, bound = soft_reference(x, centers, a, n_valid.long())
    r = ratio(v, v64, bound)
    note("soft", "ragged_nan", r)
    assert r <= 1.0


# -------------------------------------------------------------------------------------------------------- k-means
@pytest.mark.parametrize("R", [255, 256, 257, 16383, 16384, 16385, 100003])
def test_kmeans_update_fp64(L, R):
    """cluster means within the bound, exact counts (through the mean of a constant column), empty clusters exactly 0,
    and the err_out shift within a relative bound, at row counts around the partition's chunk edges"""
    lib = L.load()
    D, K = 132, 37
    chunks, rows_per = C.c_int(0), C.c_int64(0)
    L.check(lib.anyloc_kmeans_partition(R, D, C.byref(chunks), C.byref(rows_per)), "partition")
    print(f"kmeans R={R}: {chunks.value} chunks of {rows_per.value} rows")
    g = torch.Generator(device="cuda").manual_seed(R)
    x = torch.randn(R, D, device="cuda", generator=g) * 10.0 ** (2 * torch.rand(R, 1, device="cuda", generator=g) - 1)
    x[:, 0] = 1.0                                                     # column 0 of every mean is count / count
    labels = torch.randint(0, K - 5, (R,), device="cuda", generator=g, dtype=torch.int32)   # clusters K-5.. are empty
    labels[::7] = -1                                                  # rows the update ignores
    old = torch.randn(K, D, device="cuda", generator=g)
    new, err = canary(K * D), canary(1)
    ws = workspace(lib.anyloc_kmeans_workspace_bytes(R, D, K))
    L.check(lib.anyloc_kmeans_update(dptr(x), dptr(labels), dptr(old), R, D, K, dptr(new, LEAD), dptr(err, LEAD),
                                     dptr(ws), ws.numel(), L.stream_ptr()), "kmeans_update")
    torch.cuda.synchronize()
    assert_canaries(new, K * D, "kmeans centres")
    assert_canaries(err, 1, "kmeans err")
    c = inner(new, K * D).view(K, D)
    keep = labels >= 0
    lab = labels[keep].long()
    n = torch.bincount(lab, minlength=K).double()
    s64 = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, lab, x[keep].double())
    a64 = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, lab, x[keep].double().abs())
    c64 = torch.where(n[:, None] > 0, s64 / n.clamp_min(1)[:, None], torch.zeros((), dtype=torch.float64, device="cuda"))
    bound = C_ACC * U * ((n + chunks.value + 2).sqrt()[:, None] * a64 / n.clamp_min(1)[:, None] + c64.abs())
    empty = n == 0
    assert bool((c[empty] == 0).all()) and not bool(torch.signbit(c[empty]).any())
    assert bool((c[~empty, 0] == 1.0).all()), "a count is not exact"
    r = float(((c.double() - c64).abs()[~empty] / bound[~empty]).max())
    d = c64 - old.double()
    e64 = float((d * d).sum())
    e_bound = C_ACC * U * ((K * D) ** 0.5 * e64 + 2 * float((d.abs() * bound).sum()))
    re = abs(float(inner(err, 1)) - e64) / e_bound
    note("kmeans_update", f"R{R}", r)
    note("kmeans_update err_out", f"R{R}", re)
    assert r <= 1.0 and re <= 1.0


# ------------------------------------------------------------------------------------------- residual cache path
@pytest.mark.parametrize("soft", [False, True])
def test_vlad_from_residuals_fp64(L, soft):
    """anyloc_vlad_residuals against fp64 (x^ - c) and anyloc_vlad_from_residuals (hard labels or soft assignment,
    K = 37: a partial 32-cluster pass) against the fp64 sums of the residuals it is given"""
    lib = L.load()
    N, D, K = 150, 132, 37
    x, centers = make_inputs("random", 1, N, D, K, seed=9 + soft)
    x = x.view(N, D)
    res = canary(N * K * D)
    L.check(lib.anyloc_vlad_residuals(dptr(x), dptr(centers), N, D, K, 1, dptr(res, LEAD), L.stream_ptr()), "residuals")
    torch.cuda.synchronize()
    assert_canaries(res, N * K * D, "residuals")
    Rt = inner(res, N * K * D).view(N, K, D)
    x64 = x.double()
    xh = x64 / x64.norm(dim=1, keepdim=True)
    r64 = xh[:, None, :] - centers.double()[None]
    rb = C_ACC * U * ((D ** 0.5) * xh.abs()[:, None, :] + centers.double().abs()[None])
    rr = float(((Rt.double() - r64).abs() / rb).max())
    note("vlad_residuals", "random", rr)
    assert rr <= 1.0
    R64 = Rt.double()                                                 # the fp32 residuals the kernel is given
    ws = workspace(lib.anyloc_vlad_from_residuals_workspace_bytes(D, K))
    out = canary(K * D)
    if soft:
        T = 30.0
        a = torch.softmax(T * torch.nn.functional.cosine_similarity(x[:, None], centers[None], dim=2), dim=1).contiguous()
        L.check(lib.anyloc_vlad_from_residuals(dptr(Rt), None, dptr(a), N, D, K, 1, dptr(out, LEAD), dptr(ws),
                                               ws.numel(), L.stream_ptr()), "from_residuals soft")
        rs = R64.sum(1)                                               # [N,D]: sum over all centres
        u64 = a.double().T @ rs
        E = a.double().T @ R64.abs().sum(1) * (N + K + 2) ** 0.5
    else:
        lab = torch.randint(0, K - 4, (N,), device="cuda", dtype=torch.int32)   # the last 4 clusters stay empty
        L.check(lib.anyloc_vlad_from_residuals(dptr(Rt), dptr(lab), None, N, D, K, 1, dptr(out, LEAD), dptr(ws),
                                               ws.numel(), L.stream_ptr()), "from_residuals hard")
        sel = R64[torch.arange(N, device="cuda"), lab.long()]           # [N,D]
        u64 = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, lab.long(), sel)
        E = torch.zeros(K, D, dtype=torch.float64, device="cuda").index_add_(0, lab.long(), sel.abs())
        E = E * (torch.bincount(lab.long(), minlength=K).double() + 2).sqrt()[:, None]
    torch.cuda.synchronize()
    assert_canaries(out, K * D, "from_residuals")
    v64, bound = normalise(u64[None], E[None], 1)
    r = ratio(inner(out, K * D).view(1, K, D), v64, bound)
    note("vlad_from_residuals", "soft" if soft else "hard", r)
    assert r <= 1.0
