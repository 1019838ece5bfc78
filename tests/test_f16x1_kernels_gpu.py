"""The single-fp16 building blocks (ANYLOC_PAIR_F16X1) against the fp16 pairs' hi arrays and against fp64.

Producers: every single-fp16 array is the hi array that the fp16-pair (f16x3) producer writes for the same input, bit
for bit -- LayerNorm, the weight split (the hi of anyloc_split_f16), the GEMM's SPLIT epilogues (the hi of the pair
epilogue), and, through a ViT whose patch embedding is an identity and whose block is a no-op, im2col of padded and
packed batches.  The qkv tap is checked in tests/test_vit_f16x1_gpu.py (a tap call equals the single call, whose
operands come from the GEMM epilogue).  NaN canaries surround every output.

GEMM (wgmma, one fp16 MMA per k-step, fp32 accumulation in round-to-nearest chunks): with A, B the fp16 operands
(A = hi(8 a), B = hi(s_w b)) and alpha = 1 / (8 s_w),
    |pre - pre64| <= c u sqrt(K) (|A| |B|^T) |alpha| + 2 u |pre64|,  u = 2^-24, c = 16
-- the accumulation term of tests/test_gemm_engine_gpu.py, whose reference() computes it.  The SPLIT epilogues round
8 v once more to 11 significant bits (round to nearest: 2^-11 |v|) and, where |8 v| < 2^-14, to fp16's subnormal
spacing 2^-24 (2^-25 / 8 in v).  BIAS and LS_RESID write fp32 as before.

Attention (wgmma m64n64k16 with fp16 operands of 8 x, fp32 accumulators, softmax in fp32), with q, k, v the operands
and P = softmax(q k^T / 8): the bf16 bound of tests/test_bf16_kernels_gpu.py with 2^-11 in place of 2^-8,
    |o - o64| <= (2^-11 + 2 d_s + 2 (T + 64) u + 2^-20) (P |V|) + 2^-11 |o64| + 2^-28
where 2^-11 (P|V|) is P = 1024 p rounded once to 11 bits (1024 p >= 2^-14 unless p < 2^-24, whose share is below
2^-20 (P|V|)), d_s bounds the fp32 error of a logit, 2 (T + 64) u the fp32 accumulation of P V, 2^-20 the ex2.approx
error, 2^-11 |o64| the output's rounding of 8 o and 2^-28 its subnormal spacing.  Each test prints the worst share of
its bound that it measured."""
import ctypes as C

import pytest
import torch

from tests.test_bf16_kernels_gpu import attn_reference
from tests.test_gemm_engine_gpu import reference
from tests.util import dptr, gemm_nt

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
R11 = 2.0 ** -11                 # 11 significant bits, round to nearest: half an ulp, relative
SUB = 2.0 ** -25 / 8             # half fp16's subnormal spacing in 8 v, in v
LEAD = 16
NAN32, NANH = 0x7FC0DEAD, 0x7E5A       # quiet-NaN patterns no kernel writes (fp32, fp16)
EPIS = ["bias", "bias_split", "gelu_split", "swiglu_split", "ls_resid"]
ARG, UNSUPPORTED = -1, -4


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def split_f16(L, x, scale):
    """(hi, lo) of the fp16 pair of scale * x (anyloc_split_f16)"""
    x = x.contiguous()
    hi = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    lo = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    L.check(L.load().anyloc_split_f16(L.ptr(x), L.ptr(hi), L.ptr(lo), x.numel(), C.c_float(scale), L.stream_ptr()),
            "split_f16")
    return hi, lo


def canaries(rows, ld, half):
    n = LEAD + rows * ld + 2 * ld + LEAD
    if half:
        return torch.full((n,), NANH, dtype=torch.int16, device="cuda").view(torch.float16)
    return torch.full((n,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def window(buf, rows, ld, cols):
    return buf[LEAD:LEAD + rows * ld].view(rows, ld)[:, :cols]


def _pat(buf):
    half = buf.dtype == torch.float16
    return buf.view(torch.int16 if half else torch.int32), NANH if half else NAN32


def untouched_outside(buf, rows, ld, cols):
    """elements of buf outside the [rows, cols] window that no longer hold the NaN pattern"""
    bits, nan = _pat(buf)
    bits = bits.clone()
    window(bits, rows, ld, cols).fill_(nan)
    return int((bits != nan).sum())


def all_canary(buf):
    bits, nan = _pat(buf)
    return bool((bits == nan).all())


# ---------------------------------------------------------------------------------------------------------- GEMM
def run_gemm(L, epi, M, N, K, *, ldo=None, use_bias=True, seed=0, lda=None, ldb=None):
    """one f16x1 GEMM with canaries -> (got, fp64 reference, bound, staged); the SPLIT outputs also against the hi of
    the fp16-pair epilogue on the same operands"""
    lda, ldb = lda or K, ldb or K
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, lda, device="cuda", generator=g)
    b = torch.randn(N, ldb, device="cuda", generator=g) * 0.05
    a[:, K:], b[:, K:] = 1e30, 1e30             # poisons any result that reads past K
    s_w = 2.0 ** int(torch.floor(torch.log2(16384.0 / b[:, :K].abs().max())).item())
    alpha = 1.0 / (8.0 * s_w)
    a16, _ = split_f16(L, a, 8.0)
    b16, _ = split_f16(L, b, s_w)
    A, B = a16[:, :K].double(), b16[:, :K].double()
    n_out = N // 2 if epi == "swiglu_split" else N
    ldo = ldo or n_out
    split = "split" in epi
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    resid = torch.randn(LEAD + M * ldo, device="cuda", generator=g) if epi == "ls_resid" else None
    out = canaries(M, ldo, split)
    rc = gemm_nt(L, a16, None, b16, None, M, N, K, pair="f16x1", alpha=alpha, epi=epi, bias=bias, gamma=gamma,
                 resid=resid, out=out, ldo=ldo, lda=lda, ldb=ldb, out_off=LEAD, engine="auto")
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    staged = L.load().anyloc_gemm_tc_last_staged()
    esz = 2 if split else 4
    assert staged == int((ldo * esz) % 16 == 0 and (n_out * esz) % 16 == 0), (epi, M, N, K, ldo, staged)
    assert untouched_outside(out, M, ldo, n_out) == 0, (epi, M, N, K, ldo)
    got = window(out, M, ldo, n_out).double()
    ref, err = reference(dict(A=A, B=B), K, epi, alpha, bias, gamma,
                         window(resid, M, ldo, N) if resid is not None else None)
    if split:
        got = got / 8
        err = err + R11 * ref.abs() + SUB
    return got, ref, err, staged


def check(got, ref, err, what):
    share = float(((got - ref).abs() / err).max())
    assert share <= 1, f"{what}: {share:.3g} of the bound"
    assert torch.isfinite(got).all(), what
    return share


SHAPES = [(1, 200, 384), (37, 136, 392), (100, 264, 1040), (129, 128, 4096), (256, 2176, 768), (16960, 256, 384)]


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_every_epilogue_against_fp64(L, epi):
    staged, worst = [], 0.0
    for M, N, K in SHAPES:
        got, ref, err, st = run_gemm(L, epi, M, N, K, seed=M + N)
        worst = max(worst, check(got, ref, err, (epi, M, N, K)))
        staged.append(st)
    print(f"{epi}: worst share of the bound {worst:.3f}")
    assert 1 in staged, epi


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_output_pitch_and_no_bias(L, epi):
    """N tails, an odd output pitch (register epilogue) and a wide one (staged)"""
    for N in (136, 264):
        n_out = N // 2 if epi == "swiglu_split" else N
        for ldo in (n_out + 40, n_out + 1):
            got, ref, err, _ = run_gemm(L, epi, 150, N, 200, ldo=ldo, use_bias=False, seed=ldo)
            check(got, ref, err, (epi, N, ldo))


def test_gemm_strided_operands(L):
    got, ref, err, _ = run_gemm(L, "gelu_split", 70, 192, 120, lda=136, ldb=160)
    check(got, ref, err, "strided")


@pytest.mark.parametrize("epi", ["bias_split", "gelu_split", "swiglu_split"])
def test_gemm_split_output_is_the_hi_of_the_pair_epilogue(L, epi):
    """the single-fp16 epilogue writes the very bits of the hi array the fp16-pair epilogue writes for the same value:
    with a_lo = b_lo = 0 the pair GEMM's extra products add exact zeros to the same fp32 sums"""
    M, N, K = 300, 512, 384
    g = torch.Generator(device="cuda").manual_seed(3)
    a16, _ = split_f16(L, torch.randn(M, K, device="cuda", generator=g), 8.0)
    b16, _ = split_f16(L, torch.randn(N, K, device="cuda", generator=g) * 0.05, 2.0 ** 16)
    zero_a, zero_b = torch.zeros_like(a16), torch.zeros_like(b16)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    n_out = N // 2 if epi == "swiglu_split" else N
    one, hi, lo = (torch.empty(M, n_out, dtype=torch.float16, device="cuda") for _ in range(3))
    kw = dict(alpha=2.0 ** -19, epi=epi, bias=bias, ldo=n_out, engine="tc3")
    assert gemm_nt(L, a16, None, b16, None, M, N, K, pair="f16x1", out=one, **kw) == 0
    assert gemm_nt(L, a16, zero_a, b16, zero_b, M, N, K, pair="f16", out=hi, out_lo=lo, **kw) == 0
    torch.cuda.synchronize()
    assert torch.equal(one.view(torch.int16), hi.view(torch.int16)), epi


def test_coarse_fp16_pass_still_uses_the_register_epilogue(L):
    """single fp16 is its own staged instantiation; the hi-only fp16 coarse passes keep their kernel"""
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
    a, _ = split_f16(L, torch.randn(300, 384, device="cuda", generator=g), 8.0)
    b, _ = split_f16(L, torch.randn(1152, 384, device="cuda", generator=g) * 0.05, 2.0 ** 16)
    outs = []
    for rows in (slice(7, 8), slice(0, 31), slice(0, 300)):
        aa = a[rows].contiguous()
        o = torch.empty(aa.shape[0], 1152, dtype=torch.float16, device="cuda")
        assert gemm_nt(L, aa, None, b, None, aa.shape[0], 1152, 384, pair="f16x1", alpha=2.0 ** -19,
                       epi="bias_split", out=o, ldo=1152, engine="auto") == 0
        outs.append(o)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][7]) and torch.equal(outs[1], outs[2][:31])


def test_gemm_refusals_leave_the_output_untouched(L):
    M, N, K = 64, 128, 64
    a16, _ = split_f16(L, torch.randn(M, K, device="cuda"), 8.0)
    b16, _ = split_f16(L, torch.randn(N, K, device="cuda"), 8.0)
    out, lo = canaries(M, N, True), canaries(M, N, True)
    kw = dict(pair="f16x1", epi="bias_split", out=out, ldo=N, out_off=LEAD)
    assert gemm_nt(L, a16, a16, b16, None, M, N, K, **kw) == ARG
    assert gemm_nt(L, a16, None, b16, b16, M, N, K, **kw) == ARG
    assert gemm_nt(L, a16, None, b16, None, M, N, K, out_lo=lo, **kw) == ARG
    assert gemm_nt(L, a16, None, b16, None, M, N, K, engine="simt", **kw) == UNSUPPORTED
    torch.cuda.synchronize()
    assert all_canary(out) and all_canary(lo)


# ------------------------------------------------------------------------------------- LayerNorm, weights, im2col
@pytest.mark.parametrize("D", [4, 384, 1024, 1536, 2048])
def test_layernorm_is_the_hi_of_the_fp16_pair(L, D):
    lib = L.load()
    for M in (1, 9, 531):
        g = torch.Generator(device="cuda").manual_seed(D + M)
        x = torch.randn(M, D, device="cuda", generator=g) * 3 + 1
        x[::7] *= 1e-4                         # rows whose 8 y reach fp16's subnormal range
        w = torch.randn(D, device="cuda", generator=g)
        b = torch.randn(D, device="cuda", generator=g)
        hi, lo = torch.empty(M, D, dtype=torch.float16, device="cuda"), torch.empty(M, D, dtype=torch.float16,
                                                                                  device="cuda")
        L.check(lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), L.ptr(hi), L.ptr(lo),
                                           L.PAIR["f16"], L.stream_ptr()), "ln f16")
        y = canaries(M, D, True)
        L.check(lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), dptr(y, LEAD), None,
                                           L.PAIR["f16x1"], L.stream_ptr()), "ln f16x1")
        torch.cuda.synchronize()
        assert untouched_outside(y, M, D, D) == 0, (D, M)
        assert torch.equal(window(y, M, D, D).view(torch.int16), hi.view(torch.int16)), (D, M)


def test_weights_are_the_hi_of_the_fp16_pairs(L):
    from anyloc_b200 import vit
    from oracle import dinov2_restated as dr
    sd = dr.perturb(dr.build("dinov2_vitg14", depth_override=2), 1).state_dict()
    h1, f16 = (vit.VitWeights("dinov2_vitg14", sd, "cuda", pair=p) for p in ("f16x1", "f16"))
    his = [t for t in h1._keep if t is not None and t.dtype == torch.float16]
    pairs = [t for t in f16._keep if t.dtype == torch.float16]
    assert len(pairs) == 2 * len(his) > 0
    for mine, theirs in zip(his, pairs[::2]):
        assert torch.equal(mine.view(torch.int16), theirs.view(torch.int16))
    assert sum(t.numel() * 2 for t in his) * 2 == sum(t.numel() * 2 for t in pairs)
    for b1, b2 in zip(h1.blocks, f16.blocks):
        assert not any(getattr(b1, n) for n in ("qkv_w_lo", "proj_w_lo", "in_w_lo", "out_w_lo"))
        assert (b1.qkv_alpha, b1.proj_alpha, b1.in_alpha, b1.out_alpha) == \
            (b2.qkv_alpha, b2.proj_alpha, b2.in_alpha, b2.out_alpha)
    assert h1.struct.patch_w_lo is None and h1.struct.patch_alpha == f16.struct.patch_alpha


def _identity_patch_model():
    """ViT-L with one block: the patch embedding copies the 588 pixels of a patch into columns 0..587 (identity
    weights, exact in fp16; zero bias, cls and positional table) and the block adds exactly zero (zero matrices, zero
    LayerScale), so the layer-0 token facet of a patch row is the im2col row as the GEMM consumed it (alpha hi / 8)"""
    from oracle import dinov2_restated as dr
    sd = dr.build("dinov2_vitl14", depth_override=1).state_dict()
    for k, t in sd.items():
        if k.startswith("blocks.") or k in ("cls_token", "pos_embed", "patch_embed.proj.bias"):
            sd[k] = torch.zeros_like(t)
    sd["patch_embed.proj.weight"] = torch.eye(1024, 588).reshape(1024, 3, 14, 14)
    return sd


def test_im2col_padded_and_packed_is_the_hi_of_the_fp16_pair(L):
    from anyloc_b200 import vit
    m = vit.VitWeights("dinov2_vitl14", _identity_patch_model(), "cuda", pair="f16x1")
    g = torch.Generator().manual_seed(11)
    sizes = [(42, 28), (14, 70), (56, 56)]
    imgs = [(torch.randn(3, H, W, generator=g) * 10.0 ** torch.randint(-6, 2, (3, H, W), generator=g)).cuda()
            for H, W in sizes]

    def expect(x):       # [3, H, W] -> the hi(8 x) / 8 of its im2col rows, (c, ky, kx) order
        p = x.reshape(3, x.shape[1] // 14, 14, x.shape[2] // 14, 14).permute(1, 3, 0, 2, 4).reshape(-1, 588)
        hi, _ = split_f16(L, p, 8.0)
        return hi.float() / 8

    packed, n = m.extract_varlen(imgs, 0, "token", use_cls=False, norm_descs=False)
    for x, got in zip(imgs, packed.split(n)):
        assert torch.equal(got[:, :588], expect(x))
        assert torch.equal(m.extract(x[None], 0, "token", False, False)[0], got)
    batch = torch.stack([imgs[2], imgs[2] * 3])
    out = m.extract(batch, 0, "token", False, False)
    for i in range(2):
        assert torch.equal(out[i][:, :588], expect(batch[i]))


# ---------------------------------------------------------------------------------------------------------- attention
def attn_inputs(L, B, T, D, seed, logit=60.0, equal_keys=False):
    """q, k rows of norm sqrt(8 logit) (|q.k| / 8 <= logit), v ~ N(0,1) -> the single-fp16 [B*T, 3D] buffer of 8 x and
    its values x as doubles [B, T, 3, H, 64]"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    H = D // 64
    qkv = torch.randn(B, T, 3, H, 64, device="cuda", generator=g)
    for i in (0, 1):
        qkv[:, :, i] = qkv[:, :, i] / qkv[:, :, i].norm(dim=-1, keepdim=True) * (8 * logit) ** 0.5
    if equal_keys:
        qkv[:, :, 1] = qkv[:, :1, 1]
    x16, _ = split_f16(L, qkv.reshape(B * T, 3 * D), 8.0)
    return x16, (x16.double() / 8).reshape(B, T, 3, H, 64)


def attn_bound(X):
    ref, pv, qk = attn_reference(X)
    T = X.shape[1]
    d_s = 2 * 64 * U * qk / 8
    return ref, (R11 + 2 * d_s + 2 * (T + 64) * U + 2.0 ** -20) * pv + R11 * ref.abs() + SUB


@pytest.mark.parametrize("T", [1, 2, 63, 64, 127, 1025])
def test_attention_against_fp64(L, T):
    B, D = 2, 384
    worst = 0.0
    for logit, equal in ((60.0, False), (4.0, False), (60.0, True)):
        x16, X = attn_inputs(L, B, T, D, seed=T, logit=logit, equal_keys=equal)
        o = canaries(B * T, D, True)
        L.check(L.load().anyloc_attention(dptr(x16), None, B, T, D, D // 64, dptr(o, LEAD), None, L.PAIR["f16x1"],
                                          L.ENGINE["auto"], L.stream_ptr()), "attention f16x1")
        torch.cuda.synchronize()
        assert untouched_outside(o, B * T, D, D) == 0, (T, logit, equal)
        got = (window(o, B * T, D, D).double() / 8).reshape(B, T, D // 64, 64).transpose(1, 2)
        ref, bound = attn_bound(X)
        share = float(((got - ref).abs() / bound).max())
        assert share <= 1, (T, logit, equal, share)
        assert torch.isfinite(got).all()
        worst = max(worst, share)
    print(f"T={T}: worst share of the bound {worst:.3f}")


def test_packed_attention_rows_equal_lone_calls_under_nan_neighbours(L):
    """images packed with gaps of NaN rows between them: each image's output rows are the lone call's bits, and the
    rows outside every image keep their canaries"""
    D, H = 384, 6
    lens = [257, 1, 63, 130, 64]
    gap = 5
    row0, r = [], gap
    for n in lens:
        row0.append(r)
        r += n + gap
    rows = r
    buf = torch.full((rows, 3 * D), float("nan"), device="cuda").half()
    alone = []
    for i, (s, n) in enumerate(zip(row0, lens)):
        x16, _ = attn_inputs(L, 1, n, D, seed=100 + i)
        buf[s:s + n] = x16
        o = torch.empty(n, D, dtype=torch.float16, device="cuda")
        L.check(L.load().anyloc_attention(dptr(x16), None, 1, n, D, H, dptr(o), None, L.PAIR["f16x1"],
                                          L.ENGINE["tc3"], L.stream_ptr()), "attention f16x1")
        alone.append(o)
    out = canaries(rows, D, True)
    rc = L.load().anyloc_attention_varlen(dptr(buf), None, len(lens), (C.c_int32 * len(lens))(*row0),
                                          (C.c_int32 * len(lens))(*lens), D, H, dptr(out, LEAD), None,
                                          L.PAIR["f16x1"], L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    got = window(out, rows, D, D)
    bits, nan = _pat(out)
    mask = torch.ones(rows, dtype=torch.bool, device="cuda")
    for s, n, o in zip(row0, lens, alone):
        assert torch.equal(got[s:s + n].view(torch.int16), o.view(torch.int16)), (s, n)
        mask[s:s + n] = False
    assert bool((window(bits, rows, D, D)[mask] == nan).all())


def test_attention_refusals_leave_the_output_untouched(L):
    B, T, D = 1, 64, 128
    x16, _ = attn_inputs(L, B, T, D, seed=0)
    o, o_lo = canaries(B * T, D, True), canaries(B * T, D, True)
    lib = L.load()
    args = (B, T, D, 2)
    h1 = L.PAIR["f16x1"]
    assert lib.anyloc_attention(dptr(x16), dptr(x16), *args, dptr(o, LEAD), None, h1, L.ENGINE["tc3"],
                                L.stream_ptr()) == ARG
    assert lib.anyloc_attention(dptr(x16), None, *args, dptr(o, LEAD), dptr(o_lo, LEAD), h1, L.ENGINE["tc3"],
                                L.stream_ptr()) == ARG
    assert lib.anyloc_attention(dptr(x16), None, *args, dptr(o, LEAD), None, h1, L.ENGINE["simt"],
                                L.stream_ptr()) == UNSUPPORTED
    torch.cuda.synchronize()
    assert all_canary(o) and all_canary(o_lo)
