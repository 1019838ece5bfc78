"""The single-e4m3 building blocks (ANYLOC_PAIR_FP8) at the edges where kernels go wrong, through the C ABI.

GEMM (anyloc_gemm_nt, every epilogue): every output element against fp64 of the dequantised operands with the bound
of tests/test_fp8_kernels_gpu.py,
    2^-9 (|A| |B|^T) |alpha| + 16 u sqrt(K) (|A| |B|^T) |alpha| + 2 u |v|   (+ 2^-8 |v| for the bf16 SPLIT outputs),
carried through the epilogue as propagate() does, plus an absolute SUB: an output below fp32's (or bf16's) normal range
rounds to a fixed step, 2^-149 (bf16: 2^-133), which no relative term covers; SUB allows eight fp32 steps (a
few roundings of the scale, alpha and the epilogue) or one bf16 step; the rows under 448 2^-126 produce such
outputs.  NaN canaries surround every output.  Shapes: M tails 1, 63, 65, 129; N tails 8, 136, 200 (and the odd
SwiGLU halves 4, 68, 100); K tails 16, 48, 144, 208, 400 (K < 128 is one partial k-block that TMA zero-fills); ldo
of n_out + 40 (staged), n_out + 1 and a bf16 row of 66 or 132 elements (register epilogue), the path asserted against
make_epi_maps' rule; lda / ldb > K with the bytes past K the e4m3 NaN 0x7F; alpha not a power of two and no bias; a
residual apart from the output; SMs - 1 .. 2 SMs + 1 tiles and two column bands.  Per-row scales: rows of magnitude
2^-60 .. 2^60 in shuffled order, so that the 16 rows of every fragment carry 16 different scales and a misapplied one
costs at least 2x, an all-zero row (scale 1) and rows under 448 2^-126 (scale clamped at 2^-126, e4m3 subnormals).
Rows do not depend on M; the refusals return what they return and leave every canary intact.

Quantisers: anyloc_quantize_fp8_rows (K across the 32-lane x 8-element stride and its tails, M around the 8 rows per
CTA, special_rows plus bf16 subnormals, the -126 clamp and -0) and the e4m3 LayerNorm (D across its three templates and
their float4 tails, the LayerNorm rows of test_vit_rows_gpu.py, eps 1e-6 and 1e-3) bit for bit against restate_rows;
anyloc_quantize_fp8_tensor on fp32 subnormals, amax at 448 2^k and one ulp above, n not a multiple of its blocks.

Non-finite rows.  A NaN element becomes an e4m3 NaN and the row's scale comes from its finite elements; a row that
holds an Inf (or whose LayerNorm output overflows) is written as NaN bytes with a NaN scale, so that the GEMM that
consumes it writes a non-finite output row, as the bf16 GEMM does (satfinite would otherwise clamp the Inf to +-448 and
leave the row finite and wrong).  The rows beside it keep their bits.

Measured on an H100 80GB HBM3 (700 W power limit), worst |v - v64| / bound (printed as SHARE|...): SMs-count tiles
0.64 (bf16 output), M / N / K tails 0.55, strided operands 0.46, distinct row scales 0.44, output pitches 0.41.  The
parent commit's kernels fail the four non-finite tests (an Inf row came out of the GEMM with all 256 outputs finite)
and pass the rest.  Deliberately broken kernels, one per build: the
dequantisation applying row r's scale to row r + 8 when r + 8 = M - 1 exceeds the bound 149x .. 368x (caught by the
SM-count tiles, whose K = 48 rows have different scales; the tails' randn rows mostly share one scale, and the
distinct-scale test's M = 131 puts M - 1 in a fragment's lower half); reading the upper half's scale from row r fails
every GEMM test here by 57x .. 5e67x; dropping the last partial k-block (num_k = K / 128, at least 1) fails them by
55x .. 1590x, which no existing fp8 test sees (their K are multiples of 128); a row quantiser taking amax over the
first 256 elements fails the bit-exact tests at K = 264 and 4104 and the non-finite test.  The file runs in about 5 s."""
import ctypes as C

import pytest
import torch

from tests import test_fp8_kernels_gpu as k8
from tests.test_bf16_kernels_gpu import (ARG, LEAD, UNSUPPORTED, all_canary, canaries, sms, to_bf16,  # noqa: F401
                                         untouched_outside, window)
from tests.test_fp8_kernels_gpu import EPIS, NAN8, R16, T_ACC, propagate, quantize_tensor, restate_rows, special_rows
from tests.test_gemm_engine_gpu import reference
from tests.test_vit_rows_gpu import MS, _rows
from tests.util import dptr, gemm_nt

pytestmark = pytest.mark.gpu

SUB = {True: 2.0 ** -133, False: 2.0 ** -146}        # subnormal outputs: one bf16 step (SPLIT), eight fp32 steps
E4M3_NAN = 0x7F                                      # |q| bits of e4m3fn's NaN (0x7F or 0xFF)


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def quantize_rows(L, x16):
    """anyloc_quantize_fp8_rows of bf16 rows [M, K], with NaN canaries around q and the scales -> (q [M, K] uint8,
    s [M]), views into the canary buffers"""
    M, K = x16.shape
    q, s = k8.nan_bytes(M * K), k8.nan_f32(M)
    L.check(L.load().anyloc_quantize_fp8_rows(dptr(x16), M, K, k8.ptr(q, k8.LEAD), k8.ptr(s, k8.LEAD),
                                              L.stream_ptr()), "rows")
    torch.cuda.synchronize()
    assert k8.untouched(q, M * K, NAN8) and k8.untouched(s, M, k8.NAN32)
    return q[k8.LEAD:k8.LEAD + M * K].view(M, K), s[k8.LEAD:k8.LEAD + M]


def pitched(q, ld):
    """e4m3 bytes [R, K] at row pitch ld, the bytes past K the e4m3 NaN: any read past K poisons the result"""
    p = torch.full((q.shape[0], ld), NAN8, dtype=torch.uint8, device="cuda")
    p[:, :q.shape[1]] = q.view(torch.uint8)
    return p


# ---------------------------------------------------------------------------------------------------------- GEMM
def run_gemm(L, epi, M, N, K, *, a=None, ldo=None, alpha=1.0, use_bias=True, lda=None, ldb=None, seed=0):
    """one e4m3 GEMM (A rows from `a` or randn) with NaN canaries around its output -> (value, reference, bound,
    staged); alpha multiplies the weight scale"""
    lda, ldb = lda or K, ldb or K
    g = torch.Generator(device="cuda").manual_seed(seed)
    if a is None:
        a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g) * 0.05
    qa, sa = quantize_rows(L, a.to(torch.bfloat16))
    rc, qb, s_w = quantize_tensor(L, b)
    assert rc == 0, L.last_error()
    A = qa.view(torch.float8_e4m3fn).double() * sa.double()[:, None]
    B = qb.double()
    al = alpha * s_w
    n_out = N // 2 if epi == "swiglu_split" else N
    ldo = ldo or n_out
    split = "split" in epi
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    resid = torch.randn(LEAD + M * ldo, device="cuda", generator=g) if epi == "ls_resid" else None
    out = canaries(M, ldo, split)
    rc = gemm_nt(L, pitched(qa, lda), sa, pitched(qb, ldb), None, M, N, K, pair="fp8", out_dtype="bf16", alpha=al,
                 epi=epi, bias=bias, gamma=gamma, resid=resid, out=out, ldo=ldo, lda=lda, ldb=ldb, out_off=LEAD,
                 engine="auto")
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    staged = L.load().anyloc_gemm_tc_last_staged()
    esz = 2 if split else 4
    assert staged == int((ldo * esz) % 16 == 0 and (n_out * esz) % 16 == 0), (epi, M, N, K, ldo, staged)
    assert untouched_outside(out, M, ldo, n_out) == 0, (epi, M, N, K, ldo)
    got = window(out, M, ldo, n_out).double()
    ref, err = reference(dict(A=A, B=B), K, epi, al, bias, gamma,
                         window(resid, M, ldo, n_out) if resid is not None else None)
    pre = (A @ B.T) * al + (bias.double() if bias is not None else 0.0)
    err = err + propagate(epi, T_ACC * (A.abs() @ B.abs().T) * abs(al), ref, pre, gamma) + SUB[split]
    if split:
        err = err + R16 * ref.abs()
    return got, ref, err, staged


def check(got, ref, err, what):
    """every element within its bound; prints and returns the worst share of the bound"""
    assert torch.isfinite(got).all(), what
    share = float(((got - ref).abs() / err).max())
    print(f"SHARE|{what}|{share:.3f}")
    assert share <= 1.0, f"{what}: {int(((got - ref).abs() > err).sum())} elements over the bound; worst {share:.3g}x"
    return share


TAILS = [(1, 8, 16), (63, 136, 48), (65, 200, 144), (129, 136, 208), (129, 200, 400), (63, 264, 400), (65, 8, 208)]


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_m_n_k_tails(L, epi):
    for M, N, K in TAILS:
        check(*run_gemm(L, epi, M, N, K, seed=M + N + K)[:3], (epi, M, N, K))


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_output_pitch_alpha_and_no_bias(L, epi):
    """staged (ldo = n_out, n_out + 40) and register (ldo = n_out + 1, or a bf16 row of 66 / 132 elements) epilogues,
    alpha = 0.75 s_w, no bias"""
    staged = set()
    for N in (132, 256):
        n_out = N // 2 if epi == "swiglu_split" else N
        for ldo in (n_out, n_out + 40, n_out + 1):
            got, ref, err, st = run_gemm(L, epi, 150, N, 208, ldo=ldo, alpha=0.75, use_bias=False, seed=ldo)
            check(got, ref, err, (epi, N, ldo))
            staged.add(st)
    assert staged == {0, 1}, epi


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_strided_operands_poisoned_past_k(L, epi):
    check(*run_gemm(L, epi, 70, 192, 144, lda=208, ldb=240)[:3], (epi, "strided"))
    check(*run_gemm(L, epi, 33, 136, 48, lda=64, ldb=128, seed=1)[:3], (epi, "strided, one partial k-block"))


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_tiles_around_the_sm_count(L, sms, epi):
    """SMs-1 .. 2 SMs+1 tiles (each persistent CTA carries its pipeline into the next tile), and 17 column blocks:
    two raster bands"""
    for tiles in (sms - 1, sms, sms + 1, 2 * sms + 1):
        check(*run_gemm(L, epi, 128 * tiles, 128, 48, seed=tiles)[:3], (epi, tiles, "tiles"))
    check(*run_gemm(L, epi, 256, 2176, 144, seed=7)[:3], (epi, "two bands"))


def scale_rows(M, K, seed):
    """A rows whose scales differ from row to row: magnitudes 2^-60 .. 2^60 in shuffled order, an all-zero row and rows
    under 448 2^-126 (bf16 normals and subnormals: the scale clamps at 2^-126)"""
    g = torch.Generator().manual_seed(seed)
    e = torch.arange(-60, 61)[torch.randperm(121, generator=g)]
    a = torch.randn(M, K, generator=g)
    a[:121] *= (2.0 ** e.double())[:, None].float()
    a[121] = 0.0
    a[122:126] *= 1e-37
    a[126:M] *= 1e-39
    return a.cuda()


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_a_distinct_scale_on_every_row(L, epi):
    M = 131
    a = scale_rows(M, 208, seed=3)
    _, sa = quantize_rows(L, a.to(torch.bfloat16))
    for r0 in range(0, 112, 16):     # the 16 rows of every fragment: 16 scales, each >= 2x from any other
        assert len(set(sa[r0:r0 + 16].tolist())) == 16, r0
    assert float(sa[121]) == 1.0 and (sa[122:] == 2.0 ** -126).all()
    check(*run_gemm(L, epi, M, 256, 208, a=a, use_bias=False, seed=3)[:3], (epi, "row scales"))


def test_gemm_rows_do_not_depend_on_m(L):
    g = torch.Generator(device="cuda").manual_seed(5)
    qa, sa = quantize_rows(L, torch.randn(300, 384, device="cuda", generator=g).to(torch.bfloat16))
    rc, qb, s_w = quantize_tensor(L, torch.randn(1152, 384, device="cuda", generator=g) * 0.05)
    assert rc == 0
    bias = torch.randn(1152, device="cuda", generator=g)
    outs = []
    for rows in (slice(7, 8), slice(0, 31), slice(0, 300)):
        m = rows.stop - rows.start
        o = torch.empty(m, 1152, dtype=torch.bfloat16, device="cuda")
        assert gemm_nt(L, qa[rows], sa[rows], qb, None, m, 1152, 384, pair="fp8", out_dtype="bf16", alpha=s_w,
                       epi="bias_split", bias=bias, out=o, ldo=1152, engine="auto") == 0, L.last_error()
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][7]) and torch.equal(outs[1], outs[2][:31])


def test_gemm_refusals_leave_the_canaries(L):
    M, N, K = 64, 128, 64
    qa, sa = quantize_rows(L, torch.randn(M, K + 16, device="cuda").to(torch.bfloat16))
    rc, qb, _ = quantize_tensor(L, torch.randn(N, K + 16, device="cuda"))
    assert rc == 0
    out, lo = canaries(M, N, True), canaries(M, N, True)

    def gemm(a_lo=sa, b_lo=None, out_lo=None, out_dtype="bf16", engine="auto", k=K, lda=K, ldb=K):
        return gemm_nt(L, qa, a_lo, qb, b_lo, M, N, k, pair="fp8", out_dtype=out_dtype, epi="bias_split", out=out,
                       out_lo=out_lo, ldo=N, lda=lda, ldb=ldb, engine=engine, out_off=LEAD)

    assert gemm(engine="simt") == UNSUPPORTED and "tensor-core" in L.last_error()
    assert gemm(a_lo=None) == ARG and "row scales" in L.last_error()
    assert gemm(a_lo=sa.view(torch.int16)[1:]) == UNSUPPORTED           # row scales 2 bytes off their alignment
    assert gemm(b_lo=qb) == ARG and gemm(out_lo=lo) == ARG
    for dt in ("tf32", "f16", "fp8", "f16x1"):
        assert gemm(out_dtype=dt) == ARG, dt
    assert gemm(k=56, lda=K + 16, ldb=K + 16) == UNSUPPORTED                   # K not a multiple of 16
    assert gemm(lda=K + 8) == UNSUPPORTED and gemm(ldb=K + 8) == UNSUPPORTED
    torch.cuda.synchronize()
    assert all_canary(out) and all_canary(lo)


# ------------------------------------------------------------------------------------------------------ quantisers
def extra_rows(K, g):
    """bf16 subnormals, rows at and under the -126 clamp, -0"""
    rows = [torch.randn(K, generator=g) * 2.0 ** -130, torch.randn(K, generator=g) * 2.0 ** -128]
    r = torch.randn(K, generator=g) * 2.0 ** -124; r[0] = 448.0 * 2.0 ** -126; rows.append(r)     # k = -126 exactly
    r = torch.randn(K, generator=g) * 2.0 ** -125; r[0] = 448.0 * 2.0 ** -127; rows.append(r)     # clamped
    rows.append(torch.full((K,), -0.0))
    return torch.stack(rows)


@pytest.mark.parametrize("K", [8, 16, 248, 256, 264, 4104])
def test_row_quantiser_tails_bit_exact(L, K):
    g = torch.Generator().manual_seed(K)
    base = torch.cat([special_rows(K, g), extra_rows(K, g)])
    for M in MS:
        rnd = torch.randn(max(M, len(base)), K, generator=g) * torch.exp(torch.randn(max(M, len(base)), 1,
                                                                                     generator=g) * 3)
        x = torch.cat([base, rnd])[torch.randperm(len(base) + len(rnd), generator=g)[:M]].to(torch.bfloat16)
        if M >= len(base):
            x[:len(base)] = base.to(torch.bfloat16)      # every special row at least once
        q, s = quantize_rows(L, x.cuda())
        want_q, want_s = restate_rows(x.float())
        assert torch.equal(s.cpu(), want_s), (K, M)
        assert torch.equal(q.cpu(), want_q), (K, M, int((q.cpu() != want_q).sum()))
    assert (want_q[len(base) - 1] == 0x80).all()          # the -0 row: scale 1, e4m3 -0


@pytest.mark.parametrize("D", [4, 36, 388, 512, 516, 1028, 2044, 2048])
def test_layernorm_e4m3_tails_bit_exact(L, D):
    """the e4m3 rows are restate_rows of the fp32 LayerNorm whose tf32 pair the 3-term path writes (hi + lo == y)"""
    lib = L.load()
    g = torch.Generator().manual_seed(D)
    w = torch.randn(D, generator=g) * 2
    for M in MS:
        x = _rows(M, D, seed=M * D).cuda()
        for eps, b in ((1e-6, torch.randn(D, generator=g) * 0.1), (1e-3, torch.zeros(D))):
            wd, bd = w.cuda(), b.cuda()
            hi, lo = torch.empty(M, D, device="cuda"), torch.empty(M, D, device="cuda")
            L.check(lib.anyloc_layernorm_split(dptr(x), dptr(wd), dptr(bd), M, D, C.c_float(eps), dptr(hi), dptr(lo),
                                               L.PAIR["tf32"], L.stream_ptr()), "ln tf32")
            q, s = k8.nan_bytes(M * D), k8.nan_f32(M)
            L.check(lib.anyloc_layernorm_split(dptr(x), dptr(wd), dptr(bd), M, D, C.c_float(eps), k8.ptr(q, k8.LEAD),
                                               k8.ptr(s, k8.LEAD), L.PAIR["fp8"], L.stream_ptr()), "ln fp8")
            torch.cuda.synchronize()
            assert k8.untouched(q, M * D, NAN8) and k8.untouched(s, M, k8.NAN32)
            want_q, want_s = restate_rows((hi + lo).cpu())
            assert torch.equal(s[k8.LEAD:k8.LEAD + M].cpu(), want_s), (D, M, eps)
            assert torch.equal(q[k8.LEAD:k8.LEAD + M * D].cpu().view(M, D), want_q), (D, M, eps)


def test_tensor_quantiser_edges(L):
    g = torch.Generator().manual_seed(9)
    n = 256 * 37 + 5                                     # not a multiple of the 256-thread blocks
    sub = torch.randn(n, generator=g) * 1e-40            # fp32 subnormals: the scale clamps at 2^-126
    assert (sub.abs() < 2.0 ** -126).all()
    at = torch.randn(n, generator=g)
    at[11] = -448.0 * 2.0 ** -3                          # amax exactly 448 2^-3: s = 2^-3, q = -448
    above = at.clone()
    above[11] = -torch.nextafter(torch.tensor(56.0), torch.tensor(100.0))        # one ulp above: s = 2^-2
    for w, want_s in ((sub, 2.0 ** -126), (at, 2.0 ** -3), (above, 2.0 ** -2)):
        rc, q, s = quantize_tensor(L, w.cuda())
        assert rc == 0 and s == want_s, (rc, s, want_s)
        assert torch.equal(q.cpu().view(torch.uint8), (w / s).to(torch.float8_e4m3fn).view(torch.uint8))
        if w is at:
            assert int(q.view(torch.uint8)[11]) == 0xFE          # -448: e4m3's largest magnitude, reached exactly


# ---------------------------------------------------------------------------------------------- non-finite rows
def is_nan_byte(q):
    return (q & 0x7F) == E4M3_NAN


def test_row_quantiser_non_finite_rows(L):
    """a NaN element: e4m3 NaN, the scale of the finite elements; an Inf element: NaN bytes and a NaN scale"""
    K, M = 264, 9
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(M, K, generator=g) * 3).to(torch.bfloat16)
    nan_at, inf_rows = [(2, 5), (6, 200)], (4, 5, 6)
    clean = x.clone()
    for r, c in nan_at:
        x[r, c] = float("nan")
    x[4, 100], x[5, 263], x[6, 0] = float("inf"), -float("inf"), float("inf")
    q, s = quantize_rows(L, x.cuda())
    q, s = q.cpu(), s.cpu()
    want_q, want_s = restate_rows(clean.float())
    for r in range(M):
        if r in inf_rows:
            assert torch.isnan(s[r]) and is_nan_byte(q[r]).all(), (r, float(s[r]))
        elif r == 2:
            assert s[r] == restate_rows(torch.where(x[r:r + 1].isnan(), 0.0, x[r:r + 1].float()))[1][0]
            assert is_nan_byte(q[r, 5]) and torch.equal(q[r, :5], want_q[r, :5]) and torch.equal(q[r, 6:], want_q[r, 6:])
        else:
            assert s[r] == want_s[r] and torch.equal(q[r], want_q[r]), r


@pytest.mark.parametrize("epi", ["bias", "bias_split"])
def test_gemm_non_finite_rows(L, epi):
    """A rows holding an Inf or a NaN give non-finite output rows, as the bf16 GEMM's; every other row keeps the bits
    it has without them"""
    M, N, K = 40, 256, 208
    g = torch.Generator(device="cuda").manual_seed(2)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g) * 0.05
    bias = torch.randn(N, device="cuda", generator=g)
    bad = {3: float("inf"), 11: -float("inf"), 12: float("nan"), 20: float("inf")}
    poisoned = a.clone()
    for r, v in bad.items():
        poisoned[r, 7 * r % K] = v
    rc, qb, s_w = quantize_tensor(L, b)
    assert rc == 0
    b16 = to_bf16(L, b)
    split = "split" in epi
    outs = []
    for x in (a, poisoned):
        qa, sa = quantize_rows(L, x.to(torch.bfloat16))
        o = canaries(M, N, split)
        assert gemm_nt(L, qa, sa, qb, None, M, N, K, pair="fp8", out_dtype="bf16", alpha=s_w, epi=epi, bias=bias,
                       out=o, ldo=N, engine="auto", out_off=LEAD) == 0, L.last_error()
        o16 = canaries(M, N, split)
        assert gemm_nt(L, to_bf16(L, x), None, b16, None, M, N, K, pair="bf16", epi=epi, bias=bias, out=o16, ldo=N,
                       engine="auto", out_off=LEAD) == 0, L.last_error()
        torch.cuda.synchronize()
        assert untouched_outside(o, M, N, N) == 0 and untouched_outside(o16, M, N, N) == 0
        outs.append((window(o, M, N, N), window(o16, M, N, N)))
    (f8, f16), (p8, p16) = outs
    rows = torch.tensor(sorted(bad))
    keep = torch.ones(M, dtype=torch.bool)
    keep[rows] = False
    assert not torch.isfinite(p16[rows]).any(), "the bf16 GEMM's rows"
    assert not torch.isfinite(p8[rows]).any(), [int(torch.isfinite(p8[r]).sum()) for r in rows]
    assert torch.isfinite(f8).all() and torch.equal(p8[keep], f8[keep])


def test_layernorm_e4m3_non_finite_rows(L):
    """an Inf input gives NaN bytes (every element's x - mean is non-finite), an output that overflows fp32 (a huge
    gain) NaN bytes and a NaN scale; the tf32 pair LayerNorm writes a non-finite row for both"""
    M, D = 12, 388
    g = torch.Generator().manual_seed(4)
    x = torch.randn(M, D, generator=g)
    x[:, 0] = x[:, 1:].mean(dim=1)            # y[:, 0] = (x0 - mean) rstd w0 + b0 stays finite under w0 = 3e38 ...
    x[5, 0] = 10.0                            # ... except in row 5, where it overflows
    x[8, 17] = float("inf")
    w = torch.randn(D, generator=g)
    w[0] = 3e38
    b = torch.randn(D, generator=g) * 0.1
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    lib = L.load()
    hi, lo = torch.empty(M, D, device="cuda"), torch.empty(M, D, device="cuda")
    L.check(lib.anyloc_layernorm_split(dptr(xd), dptr(wd), dptr(bd), M, D, C.c_float(1e-6), dptr(hi), dptr(lo),
                                       L.PAIR["tf32"], L.stream_ptr()), "ln tf32")
    q, s = k8.nan_bytes(M * D), k8.nan_f32(M)
    L.check(lib.anyloc_layernorm_split(dptr(xd), dptr(wd), dptr(bd), M, D, C.c_float(1e-6), k8.ptr(q, k8.LEAD),
                                       k8.ptr(s, k8.LEAD), L.PAIR["fp8"], L.stream_ptr()), "ln fp8")
    torch.cuda.synchronize()
    assert k8.untouched(q, M * D, NAN8) and k8.untouched(s, M, k8.NAN32)
    y = (hi + lo).cpu()
    q, s = q[k8.LEAD:k8.LEAD + M * D].cpu().view(M, D), s[k8.LEAD:k8.LEAD + M].cpu()
    assert not torch.isfinite(y[5, 0]) and not torch.isfinite(y[8]).any()
    assert torch.isnan(s[5]) and is_nan_byte(q[5]).all(), float(s[5])
    assert is_nan_byte(q[8]).all()
    fin = [r for r in range(M) if r not in (5, 8)]
    assert torch.isfinite(y[fin]).all()
    want_q, want_s = restate_rows(y[fin])
    assert torch.equal(s[fin], want_s) and torch.equal(q[fin], want_q)
