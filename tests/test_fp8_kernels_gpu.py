"""The single-e4m3 building blocks (ANYLOC_PAIR_FP8) against torch.float8_e4m3fn and fp64 restatements.

Quantisers (LayerNorm -> e4m3, bf16 rows -> e4m3, fp32 weights -> e4m3): bit for bit.  A row (or the tensor) gets
s = 2^ceil(log2(max|x| / 448)) (1 for an all-zero row) and q = e4m3_rn(x / s); dividing by a power of two is exact, so
torch's round-to-nearest-even cast of x / s restates the kernels' cvt.rn.satfinite.e4m3x2.f32 exactly.  The
LayerNorm's fp32 output comes from the tf32-pair LayerNorm of the same input (hi + lo == y exactly).

GEMM (wgmma e4m3, partial sums promoted into a round-to-nearest fp32 accumulator every 128 elements of K): with A = q_a
s_r and B = q_b the dequantised operands (alpha = s_w carries the weight scale) and |A||B|^T the magnitude product,
    |pre - pre64| <= 2^-9 (|A| |B|^T) |alpha| + c u sqrt(K) (|A| |B|^T) |alpha| + 2 u |pre64|,  u = 2^-24, c = 16
The first term is the accumulation inside one 128-element chunk (4 wgmma k-steps): the tensor core keeps only about 14
bits of its partial sum (public reports for Hopper's fp8 MMA) and truncates, so each chunk may lose a few 2^-13 of its
own magnitude; summed over the chunks that stays a fixed fraction of the whole magnitude.  The second is the fp32
promotion (tests/test_gemm_engine_gpu.py's reference()), the third the epilogue.  SPLIT outputs add one bf16 rounding,
2^-8 |v|.  With all-positive operands the partial sums grow with K (test_positive_operands_at_k4096: M = 257, N = 256,
K = 4096).  Observed there on an H100: max relative error 7.0e-4 with the promotion every 128 elements, 2.2e-3 every
256 (ANYLOC_GEMM_CHUNK=2, over the bound), 6.9e-2 with one chunk per tile (ANYLOC_GEMM_CHUNK=64), 126x over the
bound: the accumulator really is short, and the test fails without the promotion."""
import ctypes as C

import pytest
import torch

from tests.test_gemm_engine_gpu import reference

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
R16 = 2.0 ** -8
T_ACC = 2.0 ** -9
LEAD = 64
NAN8, NAN32, NANBF = 0x7F, 0x7FC0DEAD, 0x7FDA     # e4m3fn NaN, quiet-NaN patterns no kernel writes
EPIS = ["bias", "bias_split", "gelu_split", "swiglu_split", "ls_resid"]


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off * t.element_size())


def restate_rows(x):
    """x [M, K] fp32 (CPU) -> (e4m3 bytes [M, K], scales [M]) of the row rule"""
    x = x.float()
    amax = x.abs().amax(dim=1).double()
    k = torch.ceil(torch.log2(amax / 448.0)).clamp_min(-126)
    s = torch.where(amax > 0, 2.0 ** k, torch.ones_like(amax)).float()
    q = (x / s[:, None]).to(torch.float8_e4m3fn)
    return q.view(torch.uint8), s


def nan_bytes(n):
    return torch.full((LEAD + n + LEAD,), NAN8, dtype=torch.uint8, device="cuda")


def nan_f32(n):
    return torch.full((LEAD + n + LEAD,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def untouched(buf, n, nan):
    bits = buf.view(torch.uint8 if buf.dtype == torch.uint8 else torch.int32)
    return bool((bits[:LEAD] == nan).all() and (bits[LEAD + n:] == nan).all())


def special_rows(K, g):
    """rows that exercise the scale rule and e4m3's edges: zeros, powers of two, +-448 after scaling, values in e4m3's
    subnormal range (below 2^-6 s), round-to-even ties, tiny and large magnitudes, random rows"""
    rows = [torch.zeros(K)]
    r = torch.zeros(K); r[::7] = 2.0 ** torch.arange(-20, 20, dtype=torch.float32).repeat(K)[: r[::7].numel()]; rows.append(r)
    for k in (-30, -3, 0, 5, 40):
        r = torch.randn(K, generator=g) * 2.0 ** k
        r[3] = 448.0 * 2.0 ** k; r[5] = -448.0 * 2.0 ** k           # amax exactly at a boundary: q = +-448
        rows.append(r)
        r = torch.randn(K, generator=g) * 2.0 ** k
        r[0] = 449.0 * 2.0 ** k                                     # just above: the next power of two
        rows.append(r)
    r = torch.randn(K, generator=g) * 2.0 ** -10; r[0] = 448.0; rows.append(r)      # subnormal e4m3 range
    r = (torch.arange(K, dtype=torch.float32) % 64 + 0.5) * 2.0 ** -9; r[0] = 448.0; rows.append(r)  # ties
    r = torch.full((K,), 1e-30); r[1] = -3e-31; rows.append(r)
    for _ in range(8):
        rows.append(torch.randn(K, generator=g) * torch.exp(torch.randn(1, generator=g) * 3))
    return torch.stack(rows)


@pytest.mark.parametrize("K", [384, 1024, 1536, 4096, 8])
def test_row_quantiser_bit_exact(L, K):
    g = torch.Generator().manual_seed(K)
    x = special_rows(K, g).to(torch.bfloat16)
    M = x.shape[0]
    xd = x.cuda().contiguous()
    q, s = nan_bytes(M * K), nan_f32(M)
    L.check(L.load().anyloc_quantize_fp8_rows(ptr(xd), M, K, ptr(q, LEAD), ptr(s, LEAD), L.stream_ptr()), "rows")
    torch.cuda.synchronize()
    assert untouched(q, M * K, NAN8) and untouched(s, M, NAN32)
    want_q, want_s = restate_rows(x.float())
    assert torch.equal(s[LEAD:LEAD + M].cpu(), want_s)
    got = q[LEAD:LEAD + M * K].cpu().view(M, K)
    assert torch.equal(got, want_q), int((got != want_q).sum())
    assert (got.view(torch.float8_e4m3fn).float().abs().amax(dim=1)[1:] >= 224).all()     # the scale is the smallest


@pytest.mark.parametrize("D", [384, 768, 1024, 1536])
def test_layernorm_e4m3_bit_exact(L, D):
    g = torch.Generator().manual_seed(D)
    x = special_rows(D, g)
    x[0] = 3.0                                         # a constant row: LayerNorm gives the bias
    M = x.shape[0]
    w = torch.randn(D, generator=g) * 2
    b = torch.randn(D, generator=g) * 0.1
    b_zero = torch.zeros(D)
    lib = L.load()
    for bias in (b, b_zero):
        xd, wd, bd = x.cuda(), w.cuda(), bias.cuda()
        hi, lo = torch.empty(M, D, device="cuda"), torch.empty(M, D, device="cuda")
        L.check(lib.anyloc_layernorm_split(ptr(xd), ptr(wd), ptr(bd), M, D, C.c_float(1e-6), ptr(hi), ptr(lo),
                                           L.PAIR["tf32"], L.stream_ptr()), "ln tf32")
        q, s = nan_bytes(M * D), nan_f32(M)
        L.check(lib.anyloc_layernorm_split(ptr(xd), ptr(wd), ptr(bd), M, D, C.c_float(1e-6), ptr(q, LEAD),
                                           ptr(s, LEAD), L.PAIR["fp8"], L.stream_ptr()), "ln fp8")
        torch.cuda.synchronize()
        assert untouched(q, M * D, NAN8) and untouched(s, M, NAN32)
        want_q, want_s = restate_rows((hi + lo).cpu())
        assert torch.equal(s[LEAD:LEAD + M].cpu(), want_s)
        assert torch.equal(q[LEAD:LEAD + M * D].cpu().view(M, D), want_q)
    assert float(want_s[0]) == 1.0                    # the zero row (constant input, zero bias)


def quantize_tensor(L, w):
    q = torch.empty(w.shape, dtype=torch.float8_e4m3fn, device="cuda")
    s = C.c_float()
    rc = L.load().anyloc_quantize_fp8_tensor(ptr(w), ptr(q), w.numel(), C.byref(s), L.stream_ptr())
    return rc, q, s.value


@pytest.mark.parametrize("scale", [2.0 ** -20, 0.02, 1.0, 448.0, 3.0e4])
def test_weight_quantiser_bit_exact(L, scale):
    g = torch.Generator().manual_seed(5)
    w = torch.randn(1536, 384, generator=g) * scale
    w[7, 7] = 0.0
    rc, q, s = quantize_tensor(L, w.cuda())
    assert rc == 0, L.last_error()
    amax = float(w.abs().max())
    assert s == L.load().anyloc_fp8_scale(amax) and amax / s <= 448 < 2 * amax / s
    assert torch.equal(q.cpu().view(torch.uint8), (w / s).to(torch.float8_e4m3fn).view(torch.uint8))
    rc, q, s = quantize_tensor(L, torch.zeros(64, device="cuda"))
    assert rc == 0 and s == 1.0 and not q.view(torch.uint8).any()
    bad = w.cuda()
    bad[3, 3] = float("nan")
    assert quantize_tensor(L, bad)[0] == L.ERR["arg"]
    bad[3, 3] = float("inf")
    assert quantize_tensor(L, bad)[0] == L.ERR["arg"]


def propagate(epi, extra, ref, pre, gamma):
    """how the epilogue carries an error bound `extra` of pre (the same rules as reference())"""
    if epi in ("bias", "bias_split"):
        return extra
    if epi == "gelu_split":
        return 1.13 * extra
    if epi == "swiglu_split":
        x2 = pre[:, 1::2]
        return 1.1 * extra[:, 0::2] * x2.abs() + torch.nn.functional.silu(pre[:, 0::2]).abs() * extra[:, 1::2]
    return gamma.double().abs() * extra


def run_gemm(L, epi, M, N, K, *, positive=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g) * 0.05
    if positive:
        a, b = a.abs(), b.abs()
    a16 = a.to(torch.bfloat16)
    qa, sa = torch.empty(M, K, dtype=torch.uint8, device="cuda"), torch.empty(M, device="cuda")
    lib = L.load()
    L.check(lib.anyloc_quantize_fp8_rows(ptr(a16), M, K, ptr(qa), ptr(sa), L.stream_ptr()), "rows")
    rc, qb, s_w = quantize_tensor(L, b)
    assert rc == 0
    A = qa.view(torch.float8_e4m3fn).double() * sa.double()[:, None]
    B = qb.double()
    n_out = N // 2 if epi == "swiglu_split" else N
    split = "split" in epi
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    if split:
        out = torch.full((LEAD + M * n_out + LEAD,), NANBF, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    else:
        out = nan_f32(M * n_out)
    resid = None
    if epi == "ls_resid":
        resid = torch.randn(M, n_out, device="cuda", generator=g)
        out[LEAD:LEAD + M * n_out] = resid.reshape(-1)         # in place, as the ViT's residual stream
    rc = lib.anyloc_gemm_nt(ptr(qa), ptr(sa), K, ptr(qb), None, K, M, N, K, L.PAIR["fp8"], C.c_float(s_w), L.EPI[epi],
                            ptr(bias), ptr(gamma) if gamma is not None else None,
                            ptr(out, LEAD) if resid is not None else None, ptr(out, LEAD), None, n_out,
                            L.PAIR["bf16"], L.ENGINE["auto"], L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    bits = out.view(torch.int16 if split else torch.int32)
    nan = NANBF if split else NAN32
    assert bool((bits[:LEAD] == nan).all() and (bits[LEAD + M * n_out:] == nan).all())
    got = out[LEAD:LEAD + M * n_out].view(M, n_out).double()
    ref, err = reference(dict(A=A, B=B), K, epi, s_w, bias, gamma, resid)
    pre = (A @ B.T) * s_w + bias.double()
    err = err + propagate(epi, T_ACC * (A.abs() @ B.abs().T) * s_w, ref, pre, gamma)
    if split:
        err = err + R16 * ref.abs()
    return got, ref, err


def check(got, ref, err, what):
    bad = (got - ref).abs() > err
    assert not bad.any(), f"{what}: {int(bad.sum())} elements over the bound; worst excess " \
                          f"{float(((got - ref).abs() / err)[bad].max()):.3g}x"


SHAPES = [(1, 384), (65, 1024), (257, 1536), (530, 4096), (16960, 384)]


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("M,K", SHAPES)
def test_gemm_against_fp64_of_the_dequantised_operands(L, epi, M, K):
    N = 384 if M < 16960 else 256
    got, ref, err = run_gemm(L, epi, M, N, K, seed=M + K)
    check(got, ref, err, (epi, M, K))


@pytest.mark.parametrize("epi", ["bias", "bias_split"])
def test_positive_operands_at_k4096(L, epi):
    """partial sums that grow with K: the case a short tensor-core accumulator gets wrong without the promotion"""
    got, ref, err = run_gemm(L, epi, 257, 256, 4096, positive=True, seed=3)
    rel = float(((got - ref).abs() / ref.abs()).max())
    print(f"{epi}: max relative error {rel:.3e} (the bound's accumulation term is {T_ACC:.3e})")
    check(got, ref, err, epi)
