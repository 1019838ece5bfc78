"""The bf16-pair building blocks (ANYLOC_PAIR_BF16X3) against their definition and against fp64.

Producers: every pair a kernel writes is, bit for bit, hi = x.bfloat16() and lo = (x - hi.float()).bfloat16() of the
fp32 value x it rounds -- LayerNorm (x its fp32 output, the tf32 pair's hi + lo), the weight split (anyloc_split_bf16
of w and of w - hi), the GEMM's BIAS_SPLIT epilogue (x the fp32 value the single-bf16 BIAS epilogue writes for the same
sums; GELU and SwiGLU are held to the pair rounding of their fp64 value), im2col (through a ViT whose patch embedding is
an identity) and the qkv tap (its pairs and the fp32 rows they come from, read from the workspace of a
tap call).  NaN canaries surround every output.

GEMM (wgmma, three bf16 MMAs per k-step, hi.hi + lo.hi + hi.lo, fp32 accumulation in round-to-nearest chunks): with
A = A_hi + A_lo and B = B_hi + B_lo the operand pairs' values, the kernel leaves out A_lo.B_lo, so
    |pre - pre64| <= c u sqrt(K) (|A| |B|^T) + 2 u |pre64| + |A_lo| |B_lo|^T,  u = 2^-24, c = 16
where pre64 = A B^T (+ bias) in fp64 -- the accumulation term of tests/test_gemm_engine_gpu.py plus the dropped term,
computed exactly.  The SPLIT epilogues round v once more into a pair: lo = bf16_rn(v - hi) is off by at most half an
ulp of an 8-bit value below 2^-8 |v|, so |hi + lo - v| <= 2^-16 |v| (bf16 has fp32's exponent range: no subnormal
floor matters at these sizes).

Attention (wgmma m64n64k16 with bf16 pairs, fp32 accumulators, softmax in fp32), with q, k, v the pair values and
P = softmax(q k^T / 8): the bound of tests/test_f16x1_kernels_gpu.py with the pair's terms,
    |o - o64| <= (2^-15 + 2 d_s + 2 (T + 64) u + 2^-20) (P |V|) + 2^-16 |o64|
where d_s = 2 * 64 u |q| |k| / 8 + 2^-16 |q| |k| / 8 bounds a logit's error (fp32 sums and the dropped q_lo.k_lo, at
most 2^-8 |q| 2^-8 |k|), 2^-15 (P|V|) is P split into a pair (2^-16) plus the dropped P_lo.V_lo (2^-16), 2 (T + 64) u
the fp32 accumulation of P V, 2^-20 the ex2.approx error and 2^-16 |o64| the output's pair.  Each test prints the worst
share of its bound that it measured."""
import ctypes as C

import pytest
import torch

from tests.test_bf16_kernels_gpu import attn_reference
from tests.test_gemm_engine_gpu import reference
from tests.util import dptr, gemm_nt

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
R16 = 2.0 ** -16
LEAD = 16
NANB = 0x7FDA                    # a bf16 quiet-NaN pattern no kernel writes
NAN32 = 0x7FC0DEAD
EPIS = ["bias", "bias_split", "gelu_split", "swiglu_split", "ls_resid"]
ARG, UNSUPPORTED = -1, -4


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def pair_of(x):
    """(hi, lo) bf16 of the fp32 tensor x: the definition every producer is held to"""
    hi = x.bfloat16()
    return hi, (x - hi.float()).bfloat16()


def bits(t):
    return t.view(torch.int16)


def split_pair(L, x):
    """the weight split of vit.VitWeights(pair="bf16pair"): anyloc_split_bf16 of x and of x - hi"""
    lib = L.load()
    x = x.contiguous()
    hi, lo = torch.empty(x.shape, dtype=torch.bfloat16, device="cuda"), torch.empty(x.shape, dtype=torch.bfloat16,
                                                                                      device="cuda")
    L.check(lib.anyloc_split_bf16(L.ptr(x), L.ptr(hi), x.numel(), L.stream_ptr()), "split_bf16")
    rem = x - hi.float()
    L.check(lib.anyloc_split_bf16(L.ptr(rem), L.ptr(lo), x.numel(), L.stream_ptr()), "split_bf16")
    return hi, lo


def canaries(rows, ld, half):
    n = LEAD + rows * ld + 2 * ld + LEAD
    if half:
        return torch.full((n,), NANB, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return torch.full((n,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def window(buf, rows, ld, cols):
    return buf[LEAD:LEAD + rows * ld].view(rows, ld)[:, :cols]


def _pat(buf):
    half = buf.dtype == torch.bfloat16
    return buf.view(torch.int16 if half else torch.int32), NANB if half else NAN32


def untouched_outside(buf, rows, ld, cols):
    b, nan = _pat(buf)
    b = b.clone()
    window(b, rows, ld, cols).fill_(nan)
    return int((b != nan).sum())


def all_canary(buf):
    b, nan = _pat(buf)
    return bool((b == nan).all())


def operands(L, M, N, K, seed, lda=None, ldb=None):
    lda, ldb = lda or K, ldb or K
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, lda, device="cuda", generator=g)
    b = torch.randn(N, ldb, device="cuda", generator=g) * 0.05
    a[:, K:], b[:, K:] = 1e30, 1e30             # poisons any result that reads past K
    return split_pair(L, a), split_pair(L, b)


# ---------------------------------------------------------------------------------------------------------- GEMM
def run_gemm(L, epi, M, N, K, *, ldo=None, alpha=1.0, use_bias=True, seed=0, lda=None, ldb=None, engine="auto",
             resid="plain"):
    """one bf16pair GEMM with canaries -> (got, fp64 reference, bound, staged).  The LS_RESID residual is a plain
    buffer of its own ("plain"), one inside canaries ("separate") or the output itself ("in_place", as in the ViT)"""
    (a_hi, a_lo), (b_hi, b_lo) = operands(L, M, N, K, seed, lda, ldb)
    A, B = a_hi[:, :K].double() + a_lo[:, :K].double(), b_hi[:, :K].double() + b_lo[:, :K].double()
    n_out = N // 2 if epi == "swiglu_split" else N
    ldo = ldo or n_out
    split = "split" in epi
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    out = canaries(M, ldo, split)
    out_lo = canaries(M, ldo, True) if split else None
    resid_buf, resid_t = None, None
    if epi == "ls_resid":
        if resid == "plain":
            resid_buf = torch.randn(LEAD + M * ldo, device="cuda", generator=g)
        else:
            resid_buf = out if resid == "in_place" else canaries(M, ldo, False)
            window(resid_buf, M, ldo, N).copy_(torch.randn(M, N, device="cuda", generator=g))
        resid_t = window(resid_buf, M, ldo, N).clone()
    rc = gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, pair="bf16pair", alpha=alpha, epi=epi, bias=bias, gamma=gamma,
                 resid=resid_buf, out=out, out_lo=out_lo, ldo=ldo, lda=lda, ldb=ldb, out_off=LEAD, engine=engine)
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    staged = L.load().anyloc_gemm_tc_last_staged()
    esz = 2 if split else 4
    assert staged == int((ldo * esz) % 16 == 0 and (n_out * esz) % 16 == 0), (epi, M, N, K, ldo, staged)
    assert untouched_outside(out, M, ldo, n_out) == 0, (epi, M, N, K, ldo)
    if resid == "separate" and resid_buf is not None:
        assert untouched_outside(resid_buf, M, ldo, N) == 0, (epi, M, N, K, ldo)
    ref, err = reference(dict(A=A, B=B), K, epi, alpha, bias, gamma, resid_t)
    dropped = abs(alpha) * (a_lo[:, :K].double().abs() @ b_lo[:, :K].double().abs().T)
    if epi == "swiglu_split":       # the dropped term enters through x1 (|silu'| <= 1.1) and x2
        x = A @ B.T * alpha + (bias.double() if bias is not None else 0)
        s1 = torch.nn.functional.silu(x[:, 0::2])
        err = err + 1.1 * dropped[:, 0::2] * x[:, 1::2].abs() + s1.abs() * dropped[:, 1::2] + \
            1.1 * dropped[:, 0::2] * dropped[:, 1::2]
    elif epi == "gelu_split":
        err = err + 1.13 * dropped
    elif epi == "ls_resid":
        err = err + gamma.double().abs() * dropped
    else:
        err = err + dropped
    got = window(out, M, ldo, n_out).double()
    if split:
        assert untouched_outside(out_lo, M, ldo, n_out) == 0, (epi, M, N, K, ldo)
        got = got + window(out_lo, M, ldo, n_out).double()
        err = err + R16 * (ref.abs() + err)
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
def test_gemm_output_pitch_no_bias_and_strides(L, epi):
    """N tails, an odd output pitch (register epilogue) and a wide one (staged), strided operands"""
    for N in (136, 264):
        n_out = N // 2 if epi == "swiglu_split" else N
        for ldo in (n_out + 40, n_out + 1):
            got, ref, err, _ = run_gemm(L, epi, 150, N, 200, ldo=ldo, use_bias=False, seed=ldo)
            check(got, ref, err, (epi, N, ldo))
    got, ref, err, _ = run_gemm(L, epi, 70, 192, 120, lda=136, ldb=160, engine="tc3")
    check(got, ref, err, (epi, "strided"))


@pytest.mark.parametrize("epi", ["bias_split", "gelu_split", "swiglu_split"])
def test_gemm_split_output_is_the_pair_of_its_fp32_value(L, epi):
    """with A_lo = B_lo = 0 the bf16pair GEMM adds exact zeros to the single-bf16 GEMM's fp32 sums, so its BIAS_SPLIT
    pair is pair_of(v) bit for bit, v what the single-bf16 BIAS epilogue writes; GELU and SwiGLU (erff and expf on the
    device, not torch's) are held to v's pair rounding, 2^-16 |v|, plus the fp32 error of erff / expf, a few ulps of
    |pre| (1 + erf(x) cancels for negative x, so that error is not relative to |v|)"""
    M, N, K = 300, 512, 384
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    b = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    za, zb = torch.zeros_like(a), torch.zeros_like(b)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    n_out = N // 2 if epi == "swiglu_split" else N
    hi, lo = (torch.empty(M, n_out, dtype=torch.bfloat16, device="cuda") for _ in range(2))
    assert gemm_nt(L, a, za, b, zb, M, N, K, pair="bf16pair", epi=epi, bias=bias, out=hi, out_lo=lo, ldo=n_out) == 0
    pre = torch.empty(M, N, device="cuda")
    assert gemm_nt(L, a, None, b, None, M, N, K, pair="bf16", epi="bias", bias=bias, out=pre, ldo=N) == 0
    torch.cuda.synchronize()
    if epi == "bias_split":
        want_hi, want_lo = pair_of(pre)
        assert torch.equal(bits(hi), bits(want_hi)) and torch.equal(bits(lo), bits(want_lo))
        return
    p = pre.double()
    v = torch.nn.functional.gelu(p) if epi == "gelu_split" else torch.nn.functional.silu(p[:, 0::2]) * p[:, 1::2]
    got = hi.double() + lo.double()
    share = float(((got - v).abs() / (R16 * v.abs() + 16 * U * p.abs().amax(dim=1, keepdim=True) + 1e-30)).max())
    print(f"{epi}: {share:.3f} of the bound")
    assert share <= 1.0, epi


def test_gemm_rows_do_not_depend_on_m(L):
    """no SIMT route at small M: one row alone, or with others, is the same bits"""
    (a_hi, a_lo), (b_hi, b_lo) = operands(L, 300, 1152, 384, 5)
    outs = []
    for rows in (slice(7, 8), slice(0, 31), slice(0, 300)):
        ah, al = a_hi[rows].contiguous(), a_lo[rows].contiguous()
        o = torch.empty(ah.shape[0], 1152, dtype=torch.bfloat16, device="cuda")
        ol = torch.empty_like(o)
        assert gemm_nt(L, ah, al, b_hi, b_lo, ah.shape[0], 1152, 384, pair="bf16pair", epi="bias_split", out=o,
                       out_lo=ol, ldo=1152, engine="auto") == 0
        outs.append((o, ol))
    torch.cuda.synchronize()
    for i in (0, 1):
        assert torch.equal(bits(outs[0][i][0]), bits(outs[1][i][7])) and torch.equal(bits(outs[1][i]),
                                                                                       bits(outs[2][i][:31]))


def test_gemm_refusals_leave_the_output_untouched(L):
    M, N, K = 64, 128, 64
    (a_hi, a_lo), (b_hi, b_lo) = operands(L, M, N, K, 0)
    out, lo = canaries(M, N, True), canaries(M, N, True)
    kw = dict(pair="bf16pair", epi="bias_split", out=out, ldo=N, out_off=LEAD)
    assert gemm_nt(L, a_hi, None, b_hi, b_lo, M, N, K, out_lo=lo, **kw) == ARG
    assert gemm_nt(L, a_hi, a_lo, b_hi, None, M, N, K, out_lo=lo, **kw) == ARG
    assert gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, **kw) == ARG
    assert gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, out_lo=lo, engine="simt", **kw) == UNSUPPORTED
    assert gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, out_lo=lo, out_dtype="f16", **kw) == ARG
    torch.cuda.synchronize()
    assert all_canary(out) and all_canary(lo)


# --------------------------------------------------------------------------------------------- LayerNorm, weights
@pytest.mark.parametrize("D", [4, 384, 1024, 1536, 2048])
def test_layernorm_is_the_pair_of_its_fp32_output(L, D):
    """the fp32 output y is the tf32 pair's hi + lo (exact), computed by the same statistics"""
    lib = L.load()
    for M in (1, 9, 531):
        g = torch.Generator(device="cuda").manual_seed(D + M)
        x = torch.randn(M, D, device="cuda", generator=g) * 3 + 1
        x[::7] *= 1e-30                        # rows whose variance is far below eps: outputs near 1e-27 |w|
        w = torch.randn(D, device="cuda", generator=g)
        b = torch.randn(D, device="cuda", generator=g)
        b[::3] *= 1e-30
        th, tl = torch.empty(M, D, device="cuda"), torch.empty(M, D, device="cuda")
        L.check(lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), L.ptr(th), L.ptr(tl),
                                           L.PAIR["tf32"], L.stream_ptr()), "ln tf32")
        hi, lo = canaries(M, D, True), canaries(M, D, True)
        L.check(lib.anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), M, D, C.c_float(1e-6), dptr(hi, LEAD),
                                           dptr(lo, LEAD), L.PAIR["bf16pair"], L.stream_ptr()), "ln bf16pair")
        torch.cuda.synchronize()
        assert untouched_outside(hi, M, D, D) == 0 and untouched_outside(lo, M, D, D) == 0, (D, M)
        want_hi, want_lo = pair_of(th + tl)
        assert torch.equal(bits(window(hi, M, D, D)), bits(want_hi)), (D, M)
        assert torch.equal(bits(window(lo, M, D, D)), bits(want_lo)), (D, M)


def test_weights_are_the_pairs_of_the_fp32_weights(L):
    from anyloc_b200 import vit
    from oracle import dinov2_restated as dr
    sd = dr.perturb(dr.build("dinov2_vitg14", depth_override=2), 1).state_dict()
    m = vit.VitWeights("dinov2_vitg14", sd, "cuda", pair="bf16pair")
    pw = sd["patch_embed.proj.weight"].reshape(m.dim, -1).float().cuda()
    pw = torch.nn.functional.pad(pw, (0, m.patch_k - pw.shape[1]))
    hi, lo, alpha = m.patch_w
    want = pair_of(pw)
    assert alpha == 1.0 and torch.equal(bits(hi), bits(want[0])) and torch.equal(bits(lo), bits(want[1]))
    pairs = [t for t in m._keep if t is not None and t.dtype == torch.bfloat16]
    assert len(pairs) == 2 * (1 + 4 * m.depth)
    for blk in m.blocks:
        assert all(getattr(blk, n) for n in ("qkv_w_lo", "proj_w_lo", "in_w_lo", "out_w_lo"))
        assert (blk.qkv_alpha, blk.proj_alpha, blk.in_alpha, blk.out_alpha) == (1.0, 1.0, 1.0, 1.0)
    w = sd["blocks.1.attn.qkv.weight"].float().cuda()
    mine = [t for t in pairs if t.shape == w.shape]
    want = pair_of(w)
    assert any(torch.equal(bits(a), bits(want[0])) and torch.equal(bits(b), bits(want[1]))
               for a, b in zip(mine[::2], mine[1::2]))
    assert m.struct.patch_w_lo is not None and m.struct.patch_alpha == 1.0


def _identity_patch_model():
    """ViT-L with one block: the patch embedding copies the 588 pixels of a patch into columns 0..587 (identity
    weights, exact in bf16; zero bias, cls and positional table) and the block adds exactly zero, so the layer-0 token
    facet of a patch row is the im2col pair's value hi + lo as the GEMM consumed it"""
    from oracle import dinov2_restated as dr
    sd = dr.build("dinov2_vitl14", depth_override=1).state_dict()
    for k, t in sd.items():
        if k.startswith("blocks.") or k in ("cls_token", "pos_embed", "patch_embed.proj.bias"):
            sd[k] = torch.zeros_like(t)
    sd["patch_embed.proj.weight"] = torch.eye(1024, 588).reshape(1024, 3, 14, 14)
    return sd


def test_im2col_padded_and_packed_is_the_pair_of_the_pixels(L):
    from anyloc_b200 import vit
    m = vit.VitWeights("dinov2_vitl14", _identity_patch_model(), "cuda", pair="bf16pair")
    g = torch.Generator().manual_seed(11)
    sizes = [(42, 28), (14, 70), (56, 56)]
    imgs = [(torch.randn(3, H, W, generator=g) * 10.0 ** torch.randint(-6, 2, (3, H, W), generator=g)).cuda()
            for H, W in sizes]

    def expect(x):       # [3, H, W] -> the pair values of its im2col rows, (c, ky, kx) order
        p = x.reshape(3, x.shape[1] // 14, 14, x.shape[2] // 14, 14).permute(1, 3, 0, 2, 4).reshape(-1, 588)
        hi, lo = pair_of(p.contiguous())
        return hi.float() + lo.float()                  # exact: the GEMM's sum of two products with 1.0

    packed, n = m.extract_varlen(imgs, 0, "token", use_cls=False, norm_descs=False)
    for x, got in zip(imgs, packed.split(n)):
        assert torch.equal(got[:, :588], expect(x))
        assert torch.equal(m.extract(x[None], 0, "token", False, False)[0], got)
    batch = torch.stack([imgs[2], imgs[2] * 3])
    out = m.extract(batch, 0, "token", False, False)
    for i in range(2):
        assert torch.equal(out[i][:, :588], expect(batch[i]))


def test_qkv_tap_writes_the_pairs_of_its_fp32_rows(L):
    """a tap call of layer 0's query and token facets keeps layer 0's fp32 qkv rows (the workspace's last buffer) and
    writes the attention's operands from them with the tap kernel (the qkv and qkv_lo buffers, placed by the workspace
    formula of include/anyloc_b200.h); nothing later in the call writes either.  Both must be pair_of(rows), for a
    padded batch and a packed list"""
    from anyloc_b200 import _lib, vit
    from oracle import dinov2_restated as dr
    sd = dr.perturb(dr.build("dinov2_vits14", depth_override=1), 1).state_dict()
    m = vit.VitWeights("dinov2_vits14", sd, "cuda", pair="bf16pair")
    D, Hf, Kp = m.dim, m.hidden, m.patch_k
    A = lambda x: (x + 255) // 256 * 256
    taps = [(0, "query"), (0, "token")]

    def check_ws(n_patch, M):
        off = 2 * A(2 * n_patch * Kp) + A(4 * n_patch * D) + A(4 * M * D) + 2 * A(2 * M * D)
        ws = _lib.workspaces.get(m.device, 0, "vit")
        q_hi = ws[off:off + 6 * M * D].view(torch.bfloat16).view(M, 3 * D)
        off += A(6 * M * D)
        q_lo = ws[off:off + 6 * M * D].view(torch.bfloat16).view(M, 3 * D)
        off += A(6 * M * D) + 2 * A(2 * M * Hf)
        rows = ws[off:off + 12 * M * D].view(torch.float32).view(M, 3 * D)
        want_hi, want_lo = pair_of(rows)
        assert torch.isfinite(rows).all()
        assert torch.equal(bits(q_hi), bits(want_hi)) and torch.equal(bits(q_lo), bits(want_lo))

    _lib.workspaces.clear()
    img = torch.randn(2, 3, 56, 70, generator=torch.Generator().manual_seed(2)).cuda()
    m.extract_taps(img, taps)
    torch.cuda.synchronize()
    check_ws(2 * 20, 2 * 21)
    _lib.workspaces.clear()
    imgs = [torch.randn(3, H, W, generator=torch.Generator().manual_seed(H)).cuda() for H, W in ((42, 28), (98, 70))]
    m.extract_taps_varlen(imgs, taps)
    torch.cuda.synchronize()
    check_ws(6 + 35, 6 + 35 + 2)
    _lib.workspaces.clear()


# ---------------------------------------------------------------------------------------------------------- attention
def attn_inputs(B, T, D, seed, logit=60.0, equal_keys=False):
    """q, k rows of norm sqrt(8 logit) (|q.k| / 8 <= logit), v ~ N(0,1) -> the bf16-pair [B*T, 3D] buffers and their
    values as doubles [B, T, 3, H, 64]"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    H = D // 64
    qkv = torch.randn(B, T, 3, H, 64, device="cuda", generator=g)
    for i in (0, 1):
        qkv[:, :, i] = qkv[:, :, i] / qkv[:, :, i].norm(dim=-1, keepdim=True) * (8 * logit) ** 0.5
    if equal_keys:
        qkv[:, :, 1] = qkv[:, :1, 1]
    hi, lo = pair_of(qkv.reshape(B * T, 3 * D).contiguous())
    return hi, lo, (hi.double() + lo.double()).reshape(B, T, 3, H, 64)


def attn_bound(X):
    ref, pv, qk = attn_reference(X)
    T = X.shape[1]
    d_s = 2 * 64 * U * qk / 8 + R16 * qk / 8
    return ref, (2 * R16 + 2 * d_s + 2 * (T + 64) * U + 2.0 ** -20) * pv + R16 * ref.abs()


@pytest.mark.parametrize("T", [1, 2, 63, 64, 127, 1025])
def test_attention_against_fp64(L, T):
    B, D = 2, 384
    worst = 0.0
    for logit, equal in ((60.0, False), (4.0, False), (60.0, True)):
        hi, lo, X = attn_inputs(B, T, D, seed=T, logit=logit, equal_keys=equal)
        o, o_lo = canaries(B * T, D, True), canaries(B * T, D, True)
        L.check(L.load().anyloc_attention(dptr(hi), dptr(lo), B, T, D, D // 64, dptr(o, LEAD), dptr(o_lo, LEAD),
                                          L.PAIR["bf16pair"], L.ENGINE["auto"], L.stream_ptr()), "attention bf16pair")
        torch.cuda.synchronize()
        assert untouched_outside(o, B * T, D, D) == 0 and untouched_outside(o_lo, B * T, D, D) == 0, (T, logit)
        got = (window(o, B * T, D, D).double() + window(o_lo, B * T, D, D).double())
        got = got.reshape(B, T, D // 64, 64).transpose(1, 2)
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
    buf = torch.full((rows, 3 * D), float("nan"), device="cuda").bfloat16()
    buf_lo = torch.full((rows, 3 * D), float("nan"), device="cuda").bfloat16()
    alone = []
    for i, (s, n) in enumerate(zip(row0, lens)):
        hi, lo, _ = attn_inputs(1, n, D, seed=100 + i)
        buf[s:s + n], buf_lo[s:s + n] = hi, lo
        o, ol = (torch.empty(n, D, dtype=torch.bfloat16, device="cuda") for _ in range(2))
        L.check(L.load().anyloc_attention(dptr(hi), dptr(lo), 1, n, D, H, dptr(o), dptr(ol), L.PAIR["bf16pair"],
                                          L.ENGINE["tc3"], L.stream_ptr()), "attention bf16pair")
        alone.append((o, ol))
    out, out_lo = canaries(rows, D, True), canaries(rows, D, True)
    rc = L.load().anyloc_attention_varlen(dptr(buf), dptr(buf_lo), len(lens), (C.c_int32 * len(lens))(*row0),
                                          (C.c_int32 * len(lens))(*lens), D, H, dptr(out, LEAD), dptr(out_lo, LEAD),
                                          L.PAIR["bf16pair"], L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, L.last_error()
    mask = torch.ones(rows, dtype=torch.bool, device="cuda")
    for s, n, (o, ol) in zip(row0, lens, alone):
        assert torch.equal(bits(window(out, rows, D, D)[s:s + n]), bits(o)), (s, n)
        assert torch.equal(bits(window(out_lo, rows, D, D)[s:s + n]), bits(ol)), (s, n)
        mask[s:s + n] = False
    for b in (out, out_lo):
        bb, nan = _pat(b)
        assert bool((window(bb, rows, D, D)[mask] == nan).all())
        assert untouched_outside(b, rows, D, D) == 0


def test_attention_refusals_leave_the_output_untouched(L):
    B, T, D = 1, 64, 128
    hi, lo, _ = attn_inputs(B, T, D, seed=0)
    o, o_lo = canaries(B * T, D, True), canaries(B * T, D, True)
    lib = L.load()
    args = (B, T, D, 2)
    x3 = L.PAIR["bf16pair"]
    assert lib.anyloc_attention(dptr(hi), None, *args, dptr(o, LEAD), dptr(o_lo, LEAD), x3, L.ENGINE["tc3"],
                                L.stream_ptr()) == ARG
    assert lib.anyloc_attention(dptr(hi), dptr(lo), *args, dptr(o, LEAD), None, x3, L.ENGINE["tc3"],
                                L.stream_ptr()) == ARG
    assert lib.anyloc_attention(dptr(hi), dptr(lo), *args, dptr(o, LEAD), dptr(o_lo, LEAD), x3, L.ENGINE["simt"],
                                L.stream_ptr()) == UNSUPPORTED
    torch.cuda.synchronize()
    assert all_canary(o) and all_canary(o_lo)
