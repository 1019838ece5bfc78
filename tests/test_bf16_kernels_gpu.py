"""The single-bf16 building blocks (ANYLOC_PAIR_BF16) element by element against fp64 of the bf16-rounded operands they
consume.

GEMM (wgmma, one bf16 MMA per k-step, fp32 accumulation in round-to-nearest chunks): with A, B the bf16 operands,
    |pre - pre64| <= c u sqrt(K) (|A| |B|^T) |alpha| + 2 u |pre64|,  u = 2^-24, c = 16
-- the accumulation term of tests/test_gemm_engine_gpu.py, whose reference() computes it -- and the SPLIT epilogues add
one round-to-nearest bf16 output rounding, 2^-8 |v| (8 significant bits), to the propagated bound.  BIAS and LS_RESID
write fp32 as before.

Attention (wgmma m64n64k16 with bf16 operands, fp32 accumulators, softmax in fp32): with q, k, v the bf16 operands
and P = softmax(q k^T / 8),
    |o - o64| <= (2^-8 + 2 d_s + 2 (T + 64) u + 2^-20) (P |V|) + 2^-8 |o64|
where 2^-8 (P|V|) is P rounded once to bf16 (p <= 1 after the max subtraction; the denominator sums the unrounded p),
d_s = 2 u 64 |q_i| max_j |k_j| / 8 bounds the fp32 error of a logit (2 u: the tensor core's accumulation need not round
to nearest; each logit error moves p and the denominator by e^d_s), 2 (T + 64) u the fp32 accumulation of P V over
the key blocks, 2^-20 the ex2.approx error, and 2^-8 |o64| the bf16 output rounding.

Also: the bf16 conversion and LayerNorm bit for bit against torch's round-to-nearest cast, NaN canaries around every
output, the staged-epilogue observable, and the refusals (non-NULL lo arrays, the SIMT engine), which leave the
canaries untouched.  attn_bound() is the attention bound; tests/test_attention_varlen_gpu.py applies it to the packed
(varlen) attention, image by image."""
import ctypes as C

import pytest
import torch

from tests.test_gemm_engine_gpu import reference
from tests.util import dptr, gemm_nt

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
R16 = 2.0 ** -8                  # bf16 round-to-nearest: half an ulp of 8 significant bits, relative
LEAD = 16
NAN32, NANBF = 0x7FC0DEAD, 0x7FDA      # quiet-NaN patterns no kernel writes (fp32, bf16)
EPIS = ["bias", "bias_split", "gelu_split", "swiglu_split", "ls_resid"]
ARG, UNSUPPORTED = -1, -4


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


@pytest.fixture(scope="module")
def sms(L):
    n = C.c_int(0)
    assert L.load().anyloc_device_info(C.byref(n), None) >= 90
    return n.value


def to_bf16(L, x):
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    L.check(L.load().anyloc_split_bf16(L.ptr(x.contiguous()), L.ptr(y), x.numel(), L.stream_ptr()), "split_bf16")
    return y


def canaries(rows, ld, bf16):
    n = LEAD + rows * ld + 2 * ld + LEAD
    if bf16:
        return torch.full((n,), NANBF, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return torch.full((n,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def window(buf, rows, ld, cols):
    return buf[LEAD:LEAD + rows * ld].view(rows, ld)[:, :cols]


def untouched_outside(buf, rows, ld, cols):
    """elements of buf outside the [rows, cols] window that no longer hold the NaN pattern"""
    bf = buf.dtype == torch.bfloat16
    bits = buf.view(torch.int16 if bf else torch.int32).clone()
    window(bits, rows, ld, cols).fill_(NANBF if bf else NAN32)
    return int((bits != (NANBF if bf else NAN32)).sum())


def all_canary(buf):
    bf = buf.dtype == torch.bfloat16
    return bool((buf.view(torch.int16 if bf else torch.int32) == (NANBF if bf else NAN32)).all())


# ---------------------------------------------------------------------------------------------------------- GEMM
def run_gemm(L, epi, M, N, K, *, ldo=None, alpha=1.0, use_bias=True, seed=0, lda=None, ldb=None):
    lda, ldb = lda or K, ldb or K
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, lda, device="cuda", generator=g)
    b = torch.randn(N, ldb, device="cuda", generator=g) * 0.05
    a[:, K:], b[:, K:] = 1e30, 1e30             # poisons any result that reads past K
    a16, b16 = to_bf16(L, a), to_bf16(L, b)
    A, B = a16[:, :K].double(), b16[:, :K].double()
    n_out = N // 2 if epi == "swiglu_split" else N
    ldo = ldo or n_out
    split = "split" in epi
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    # a residual apart from the output, laid out like it (element LEAD is row 0)
    resid = torch.randn(LEAD + M * ldo, device="cuda", generator=g) if epi == "ls_resid" else None
    out = canaries(M, ldo, split)
    rc = gemm_nt(L, a16, None, b16, None, M, N, K, pair="bf16", alpha=alpha, epi=epi, bias=bias, gamma=gamma,
                 resid=resid, out=out, ldo=ldo, lda=lda, ldb=ldb, out_off=LEAD, engine="auto")
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    staged = L.load().anyloc_gemm_tc_last_staged()
    esz = 2 if split else 4
    # the staged epilogue (TMA stores) where row pitch and row length are multiples of 16 bytes, else from registers
    assert staged == int((ldo * esz) % 16 == 0 and (n_out * esz) % 16 == 0), (epi, M, N, K, ldo, staged)
    assert untouched_outside(out, M, ldo, n_out) == 0, (epi, M, N, K, ldo)
    got = window(out, M, ldo, n_out).double()
    ref, err = reference(dict(A=A, B=B), K, epi, alpha, bias, gamma,
                         window(resid, M, ldo, N) if resid is not None else None)
    if split:
        err = err + R16 * ref.abs()
    return got, ref, err, staged


def check(got, ref, err, what):
    bad = (got - ref).abs() > err
    assert not bad.any(), f"{what}: {int(bad.sum())} elements over the bound; worst excess " \
                          f"{float(((got - ref).abs() - err).max()):.3g}"
    assert torch.isfinite(got).all(), what


SHAPES = [(1, 200, 72), (37, 136, 264), (100, 264, 1040), (129, 128, 64), (256, 2176, 128)]


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_every_epilogue_against_fp64(L, epi):
    staged = []
    for M, N, K in SHAPES:
        got, ref, err, st = run_gemm(L, epi, M, N, K, seed=M + N)
        check(got, ref, err, (epi, M, N, K))
        staged.append(st)
    assert 1 in staged, epi


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_tiles_around_the_sm_count(L, sms, epi):
    """SMs-1 .. 2 SMs+1 tiles: every persistent CTA carries its pipeline ring (and staging buffers) into the next tile"""
    for tiles in (sms - 1, sms, sms + 1, 2 * sms + 1):
        got, ref, err, _ = run_gemm(L, epi, 128 * tiles, 128, 96, seed=tiles)
        check(got, ref, err, (epi, tiles))


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_wide_and_odd_output_pitch_alpha_and_no_bias(L, epi):
    for N in (136, 256):
        n_out = N // 2 if epi == "swiglu_split" else N
        for ldo in (n_out + 40, n_out + 1):
            got, ref, err, _ = run_gemm(L, epi, 150, N, 200, ldo=ldo, alpha=0.75, use_bias=False, seed=ldo)
            check(got, ref, err, (epi, N, ldo))


def test_gemm_strided_operands(L):
    got, ref, err, _ = run_gemm(L, "gelu_split", 70, 192, 120, lda=136, ldb=160)
    check(got, ref, err, "strided")


def test_coarse_fp16_pass_still_uses_the_register_epilogue(L):
    """the bf16 instantiation is hi-only with the staged epilogue; the hi-only fp16 coarse passes keep their kernel"""
    run_gemm(L, "bias", 256, 256, 128)
    assert L.load().anyloc_gemm_tc_last_staged() == 1
    a = torch.randn(256, 128, device="cuda").half()
    b = torch.randn(256, 128, device="cuda").half()
    out = torch.empty(256, 256, device="cuda")
    assert gemm_nt(L, a, None, b, None, 256, 256, 128, pair="f16", out=out, ldo=256, engine="tc3") == 0
    torch.cuda.synchronize()
    assert L.load().anyloc_gemm_tc_last_staged() == 0


def test_gemm_rows_do_not_depend_on_m(L):
    """no SIMT route at small M: one row alone, or with others, is the same bits"""
    g = torch.Generator(device="cuda").manual_seed(5)
    a = to_bf16(L, torch.randn(300, 384, device="cuda", generator=g))
    b = to_bf16(L, torch.randn(1152, 384, device="cuda", generator=g) * 0.05)
    outs = []
    for rows in (slice(7, 8), slice(0, 31), slice(0, 300)):
        aa = a[rows].contiguous()
        o = torch.empty(aa.shape[0], 1152, dtype=torch.bfloat16, device="cuda")
        assert gemm_nt(L, aa, None, b, None, aa.shape[0], 1152, 384, pair="bf16", epi="bias_split", out=o, ldo=1152,
                       engine="auto") == 0
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][7]) and torch.equal(outs[1], outs[2][:31])


def test_gemm_refusals_leave_the_output_untouched(L):
    M, N, K = 64, 128, 64
    a16 = to_bf16(L, torch.randn(M, K, device="cuda"))
    b16 = to_bf16(L, torch.randn(N, K, device="cuda"))
    out, lo = canaries(M, N, True), canaries(M, N, True)
    kw = dict(pair="bf16", epi="bias_split", out=out, ldo=N, out_off=LEAD)
    assert gemm_nt(L, a16, a16, b16, None, M, N, K, **kw) == ARG
    assert gemm_nt(L, a16, None, b16, b16, M, N, K, **kw) == ARG
    assert gemm_nt(L, a16, None, b16, None, M, N, K, out_lo=lo, **kw) == ARG
    assert gemm_nt(L, a16, None, b16, None, M, N, K, engine="simt", **kw) == UNSUPPORTED
    assert "tensor-core" in L.last_error()
    # bf16 in with a pair format out (and the reverse)
    assert L.load().anyloc_gemm_nt(dptr(a16), None, K, dptr(b16), None, K, M, N, K, L.PAIR["bf16"], C.c_float(1.0),
                                   L.EPI["bias_split"], None, None, None, dptr(out, LEAD), dptr(lo, LEAD), N,
                                   L.PAIR["f16"], L.ENGINE["tc3"], L.stream_ptr()) == ARG
    torch.cuda.synchronize()
    assert all_canary(out) and all_canary(lo)


# ------------------------------------------------------------------------------------------ conversion, LayerNorm
def test_split_bf16_equals_torch_round_to_nearest_cast(L):
    """anyloc_split_bf16 (__float2bfloat16_rn) is torch's fp32 -> bf16 cast bit for bit: ties to even, subnormals,
    overflow to inf, signed zeros"""
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.cat([torch.randn(1 << 20, device="cuda", generator=g) * 10.0 ** torch.randint(-40, 39, (1 << 20,),
                   device="cuda", generator=g).float(),
                   torch.tensor([0.0, -0.0, 1e-45, -1e-45, 3.4e38, -3.4e38, float("inf"), -float("inf")],
                                device="cuda")])
    # exact halfway points between neighbouring bf16 values: low 16 bits = 0x8000
    halves = (torch.randint(0, 1 << 15, (1 << 16,), device="cuda", generator=g, dtype=torch.int32) << 16) | 0x8000
    x = torch.cat([x, halves.view(torch.float32)])
    x = x[torch.isfinite(x) | torch.isinf(x)]
    assert torch.equal(to_bf16(L, x).view(torch.int16), x.to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("D", [384, 1024, 1536])
def test_layernorm_bf16_is_the_rounded_fp32_layernorm(L, D):
    """the bf16 output is bf16_rn of the very fp32 value whose tf32 pair the 3-term path writes (hi + lo is exact)"""
    M = 77
    g = torch.Generator(device="cuda").manual_seed(D)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 1
    w = torch.randn(D, device="cuda", generator=g)
    b = torch.randn(D, device="cuda", generator=g)
    hi, lo = torch.empty(M, D, device="cuda"), torch.empty(M, D, device="cuda")
    lib = L.load()
    L.check(lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), L.ptr(hi), L.ptr(lo),
                                       L.PAIR["tf32"], L.stream_ptr()), "ln tf32")
    y = canaries(M, D, True)
    L.check(lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), dptr(y, LEAD), None,
                                       L.PAIR["bf16"], L.stream_ptr()), "ln bf16")
    torch.cuda.synchronize()
    assert untouched_outside(y, M, D, D) == 0
    assert torch.equal(window(y, M, D, D).view(torch.int16), (hi + lo).to(torch.bfloat16).view(torch.int16))
    y2 = canaries(M, D, True)
    assert lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), dptr(y2, LEAD), L.ptr(lo),
                                      L.PAIR["bf16"], L.stream_ptr()) == ARG
    torch.cuda.synchronize()
    assert all_canary(y2)


# ---------------------------------------------------------------------------------------------------------- attention
def attn_inputs(L, B, T, D, seed, logit=60.0, equal_keys=False):
    """q, k rows of norm sqrt(8 logit) (so |q.k| / 8 <= logit), v ~ N(0,1); returns the bf16 [B*T, 3D] buffer and its
    fp64 values"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    H = D // 64
    qkv = torch.randn(B, T, 3, H, 64, device="cuda", generator=g)
    for i in (0, 1):
        qkv[:, :, i] = qkv[:, :, i] / qkv[:, :, i].norm(dim=-1, keepdim=True) * (8 * logit) ** 0.5
    if equal_keys:
        qkv[:, :, 1] = qkv[:, :1, 1]
    x16 = to_bf16(L, qkv.reshape(B * T, 3 * D))
    return x16, x16.double().reshape(B, T, 3, H, 64)


def attn_reference(X):
    q, k, v = (X[:, :, i].transpose(1, 2) for i in range(3))      # [B, H, T, 64]
    s = q @ k.transpose(-1, -2) / 8
    p = torch.softmax(s, dim=-1)
    o = p @ v
    pv = p @ v.abs()
    qk = q.norm(dim=-1, keepdim=True) * k.norm(dim=-1).amax(dim=-1)[..., None, None]      # |q_i| max_j |k_j|
    return o, pv, qk


def attn_bound(X):
    """fp64 softmax(q k^T / 8) v of the bf16 operands X [B, T, 3, H, 64] (as doubles) and the bound of the module
    docstring, both [B, H, T, 64]"""
    ref, pv, qk = attn_reference(X)
    T = X.shape[1]
    d_s = 2 * 64 * U * qk / 8
    return ref, (R16 + 2 * d_s + 2 * (T + 64) * U + 2.0 ** -20) * pv + R16 * ref.abs()


@pytest.mark.parametrize("T", [1, 2, 63, 64, 127, 1025])
def test_attention_against_fp64(L, T):
    B, D = 2, 384
    for logit, equal in ((60.0, False), (4.0, False), (60.0, True)):
        x16, X = attn_inputs(L, B, T, D, seed=T, logit=logit, equal_keys=equal)
        o = canaries(B * T, D, True)
        L.check(L.load().anyloc_attention(dptr(x16), None, B, T, D, D // 64, dptr(o, LEAD), None, L.PAIR["bf16"],
                                          L.ENGINE["auto"], L.stream_ptr()), "attention bf16")
        torch.cuda.synchronize()
        assert untouched_outside(o, B * T, D, D) == 0, (T, logit, equal)
        got = window(o, B * T, D, D).double().reshape(B, T, D // 64, 64).transpose(1, 2)
        ref, bound = attn_bound(X)
        excess = (got - ref).abs() - bound
        assert float(excess.max()) <= 0, (T, logit, equal, float(excess.max()))
        if equal:         # equal keys: P is uniform (exp(0) = 1 exactly), o is the mean of v in every row
            assert torch.isfinite(got).all()
        print(f"T={T} logit={logit} equal={equal}: max|o-o64| {float((got - ref).abs().max()):.3g}")


def test_attention_refusals_leave_the_output_untouched(L):
    B, T, D = 1, 64, 128
    x16, _ = attn_inputs(L, B, T, D, seed=0)
    o, o_lo = canaries(B * T, D, True), canaries(B * T, D, True)
    lib = L.load()
    args = (B, T, D, 2)
    assert lib.anyloc_attention(dptr(x16), dptr(x16), *args, dptr(o, LEAD), None, L.PAIR["bf16"], L.ENGINE["tc3"],
                                L.stream_ptr()) == ARG
    assert lib.anyloc_attention(dptr(x16), None, *args, dptr(o, LEAD), dptr(o_lo, LEAD), L.PAIR["bf16"],
                                L.ENGINE["tc3"], L.stream_ptr()) == ARG
    assert lib.anyloc_attention(dptr(x16), None, *args, dptr(o, LEAD), None, L.PAIR["bf16"], L.ENGINE["simt"],
                                L.stream_ptr()) == UNSUPPORTED
    torch.cuda.synchronize()
    assert all_canary(o) and all_canary(o_lo)
