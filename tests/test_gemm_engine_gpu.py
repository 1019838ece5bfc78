"""The GEMM engine contract of anyloc_gemm_nt, checked element by element against an fp64 product of the operands the
engine actually multiplies:

    |C - C64|_ij <= c u sqrt(K) (|A| |B|^T)_ij |alpha|  (+ rounding of the epilogue),   u = 2^-24, c = C_ACC = 16,

with A, B the consumed operands: hi + lo (tf32 pairs: each word truncated to tf32 by the tensor core, kept whole by the
SIMT engine; fp16 pairs: (hi + lo) / s).  The same metric holds for both engines.  Covered: N and K tails, M below one
tile, more tiles than SMs (so every CTA carries its pipeline ring into a second tile), two column bands, every lo-operand
variant (LOM 0..3), strided operands, wide and odd output leading dimensions, alpha != 1, no bias, a residual that does
not alias the output, NaN canaries around every output, shapes outside the tensor-core contract, the round-to-nearest
chunk accumulation (with a mutation run that switches it off), and batch invariance of rows."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.test_vlad_bound_cpu import trunc_tf32 as trunc_tf32_np
from tests.util import ROOT, gemm, gemm_nt, split_f16, split_tf32

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ACC = 16                       # c of the per-element bound above
LEAD = 16                        # canary elements before every output (64 B fp32 / 32 B fp16: alignment kept)
NAN32, NAN16 = 0x7FC0DEAD, 0x7E5A   # quiet-NaN bit patterns no epilogue writes
EPIS = ["bias", "bias_split", "gelu_split", "swiglu_split", "ls_resid"]
UNSUPPORTED = -4                 # ANYLOC_ERR_UNSUPPORTED


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


def trunc_tf32(t):
    """what the tensor core reads of an fp32 word: the low 13 mantissa bits dropped (same mask as the CPU model)"""
    return (t.contiguous().view(torch.int32) & -8192).view(torch.float32)


# ----------------------------------------------------------------------------------------------------- operands
def operands(L, M, N, K, pair, engine, lom=3, lda=None, ldb=None, seed=0, dist="randn"):
    """(hi, lo) operands in buffers of leading dimension lda / ldb (columns >= K hold 1e30, which poisons any result
    that reads them) and the fp64 values the engine multiplies."""
    lda, ldb = lda or K, ldb or K
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rand(rows, ld, s):
        x = torch.randn(rows, ld, device="cuda", generator=g) if dist == "randn" else \
            torch.rand(rows, ld, device="cuda", generator=g)
        x = x * s
        x[:, K:] = 1e30
        return x

    a, b = rand(M, lda, 1.0), rand(N, ldb, 0.05 if dist == "randn" else 1.0)
    has_a_lo, has_b_lo = bool(lom & 1), bool(lom & 2)
    if pair == "tf32":
        take = trunc_tf32 if engine == "tc3" else (lambda t: t)
        a_hi, a_lo = split_tf32(L, a) if has_a_lo else (a, None)     # hi-only: raw fp32 words, as the coarse passes
        b_hi, b_lo = split_tf32(L, b) if has_b_lo else (b, None)
        A = take(a_hi).double() + (take(a_lo).double() if has_a_lo else 0)
        B = take(b_hi).double() + (take(b_lo).double() if has_b_lo else 0)
        scale = 1.0
    else:
        s_a = L.ACT_SCALE
        s_b = 2.0 ** int(torch.floor(torch.log2(16384.0 / b[:, :K].abs().max())).item())
        a_hi, a_lo = split_f16(L, a, s_a)
        b_hi, b_lo = split_f16(L, b, s_b)
        a_lo, b_lo = (a_lo if has_a_lo else None), (b_lo if has_b_lo else None)
        A = (a_hi.double() + (a_lo.double() if has_a_lo else 0)) / s_a
        B = (b_hi.double() + (b_lo.double() if has_b_lo else 0)) / s_b
        scale = 1.0 / (s_a * s_b)
    return dict(a_hi=a_hi, a_lo=a_lo, b_hi=b_hi, b_lo=b_lo, A=A[:, :K], B=B[:, :K], scale=scale, lda=lda, ldb=ldb)


def canary_buffer(rows, ldo, dtype):
    n = LEAD + rows * ldo + 2 * ldo + LEAD
    idt = torch.int32 if dtype == torch.float32 else torch.int16
    return torch.full((n,), NAN32 if dtype == torch.float32 else NAN16, dtype=idt, device="cuda").view(dtype)


def window(buf, rows, ldo, cols):
    return buf[LEAD:LEAD + rows * ldo].view(rows, ldo)[:, :cols]


def assert_canaries(buf, rows, ldo, cols, what):
    """every element outside the [rows, cols] window of `buf` still holds the NaN pattern"""
    idt = torch.int32 if buf.dtype == torch.float32 else torch.int16
    bits = buf.view(idt).clone()
    window(bits, rows, ldo, cols).fill_(NAN32 if idt == torch.int32 else NAN16)
    bad = int((bits != (NAN32 if idt == torch.int32 else NAN16)).sum())
    assert bad == 0, f"{what}: {bad} elements written outside [M, n_out]"


# ---------------------------------------------------------------------------------------------------- reference
def reference(ops, K, epi, alpha, bias, gamma, resid):
    """(value, bound) in fp64 for every output element; A and B hold unscaled values (the kernel's alpha also undoes
    the fp16 pair scales)"""
    al = alpha
    A, B = ops["A"], ops["B"]
    pre = (A @ B.T) * al
    if bias is not None:
        pre = pre + bias.double()
    err = C_ACC * U * K ** 0.5 * (A.abs() @ B.abs().T) * abs(al) + 2 * U * pre.abs()
    if epi == "bias":
        return pre, err
    if epi == "bias_split":
        return pre, err + 8 * U * pre.abs()                 # fp16 pair of 8x: 22 significant bits
    if epi == "gelu_split":
        ref = torch.nn.functional.gelu(pre)
        return ref, 1.13 * err + 8 * U * (ref.abs() + pre.abs())      # |gelu'| <= 1.13, erff to a few ulp
    if epi == "swiglu_split":
        x1, x2, e1, e2 = pre[:, 0::2], pre[:, 1::2], err[:, 0::2], err[:, 1::2]
        s1 = torch.nn.functional.silu(x1)
        ref = s1 * x2
        return ref, 1.1 * e1 * x2.abs() + s1.abs() * e2 + 16 * U * ref.abs()   # |silu'| <= 1.1
    if epi == "ls_resid":
        gx = gamma.double() * pre
        ref = resid.double() + gx
        return ref, gamma.double().abs() * err + 2 * U * (resid.double().abs() + gx.abs() + ref.abs())
    raise ValueError(epi)


def run(L, pair, engine, epi, M, N, K, *, lom=3, lda=None, ldb=None, ldo=None, alpha=1.0, use_bias=True,
        resid_alias=True, seed=0, dist="randn", expect_rc=0):
    """one anyloc_gemm_nt call with NaN canaries around every output -> (value, reference, bound) in fp64"""
    ops = operands(L, M, N, K, pair, engine, lom, lda, ldb, seed, dist)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    n_out = N // 2 if epi == "swiglu_split" else N
    ldo = ldo or n_out
    bias = torch.randn(N, device="cuda", generator=g) if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    is_split = "split" in epi
    odt = torch.float16 if (is_split and pair == "f16") else torch.float32
    out = canary_buffer(M, ldo, odt)
    out_lo = canary_buffer(M, ldo, odt) if is_split else None
    resid_t, resid_buf = None, None
    if epi == "ls_resid":
        resid_t = torch.randn(M, n_out, device="cuda", generator=g)
        if resid_alias:                                     # in place, as the ViT's residual stream
            window(out, M, ldo, n_out).copy_(resid_t)
            resid_buf = out
        else:
            resid_buf = canary_buffer(M, ldo, torch.float32)
            window(resid_buf, M, ldo, n_out).copy_(resid_t)
    rc = gemm_nt(L, ops["a_hi"], ops["a_lo"], ops["b_hi"], ops["b_lo"], M, N, K, pair=pair, alpha=alpha * ops["scale"],
                 epi=epi, bias=bias, gamma=gamma, resid=resid_buf, out=out, out_lo=out_lo, ldo=ldo, lda=ops["lda"],
                 ldb=ops["ldb"], engine=engine, out_off=LEAD)
    torch.cuda.synchronize()
    assert rc == expect_rc, (rc, L.last_error())
    assert_canaries(out, M, ldo, n_out, "out")
    if out_lo is not None:
        assert_canaries(out_lo, M, ldo, n_out, "out_lo")
    if resid_buf is not None and not resid_alias:
        assert_canaries(resid_buf, M, ldo, n_out, "resid")
    if rc:
        return None
    val = window(out, M, ldo, n_out).double()
    if is_split:
        val = val + window(out_lo, M, ldo, n_out).double()
        if pair == "f16":
            val = val / L.ACT_SCALE
    ref, bound = reference(ops, K, epi, alpha, bias, gamma, resid_t)
    return val, ref, bound


def check(res, what):
    val, ref, bound = res
    excess = (val - ref).abs() / bound
    worst = float(excess.max())
    assert torch.isfinite(val).all() and worst <= 1.0, (what, f"max |C-C64|/bound = {worst:.3f}",
                                                        tuple(int(i) for i in divmod(int(excess.argmax()), ref.shape[1])))
    return worst


# -------------------------------------------------------------------------------------------- shapes x epilogues
# K = 72 is a whole number of 16-byte groups in both formats and ends in a partial 128-byte k-block in both
SHAPES = {
    # N tails (N % 128 != 0), odd N where the epilogue allows it
    "N1": (200, 1, 72), "N2": (200, 2, 72), "N3": (200, 3, 72), "N8": (200, 8, 72), "N129": (200, 129, 72),
    "N130": (200, 130, 72), "N200": (200, 200, 72), "N254": (200, 254, 72), "N255": (200, 255, 72),
    # K tails: tf32 K % 32 != 0 (4, 36, 100, 4084 = 4 * 1021), fp16 K % 64 != 0 (8, 72, 600)
    "K4": (150, 136, 4), "K36": (150, 136, 36), "K100": (150, 136, 100), "K4084": (150, 136, 4084),
    "K8": (150, 136, 8), "K600": (150, 136, 600),
    # M below one tile: the second consumer warpgroup has no valid rows for M <= 64
    "M1": (1, 136, 72), "M31": (31, 136, 72), "M64": (64, 136, 72), "M65": (65, 136, 72), "M127": (127, 136, 72),
    # two column bands of 16 and 3 column blocks (N = 2048 + 384 - 8), 190 tiles
    "bands": (1260, 2424, 200),
}
TILE_CASES = {"tiles=SMs-1": -1, "tiles=SMs": 0, "tiles=SMs+1": 1, "tiles=2SMs+1": None}


def tile_shape(sms, case):
    """(M, N) with exactly the requested number of 128x128 tiles, tails in both M and N"""
    t = 2 * sms + 1 if TILE_CASES[case] is None else sms + TILE_CASES[case]
    num_n = next((d for d in range(5, 1, -1) if t % d == 0), 1)
    num_m = t // num_n
    return 128 * (num_m - 1) + 77, 128 * (num_n - 1) + 100


def shape_ok(pair, epi, N, K):
    q = 8 if pair == "f16" else 4
    return K % q == 0 and not (epi == "swiglu_split" and N % 2)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("engine", ["simt", "tc3"])
@pytest.mark.parametrize("pair", ["tf32", "f16"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_gemm_shapes(L, shape, pair, engine, epi):
    M, N, K = SHAPES[shape]
    if not shape_ok(pair, epi, N, K):
        pytest.skip("K not a multiple of 16 bytes in this format, or odd N for SwiGLU")
    check(run(L, pair, engine, epi, M, N, K, seed=M + N + K), (shape, pair, engine, epi))


@pytest.mark.parametrize("epi", ["bias", "bias_split", "swiglu_split", "ls_resid"])
@pytest.mark.parametrize("pair", ["tf32", "f16"])
@pytest.mark.parametrize("case", list(TILE_CASES))
def test_gemm_persistent_tiles(L, sms, case, pair, epi):
    """more tiles than SMs: a CTA runs its second tile on the stage/phase ring state the first one left; K = 1088 spans
    17 tf32 chunks (3 fp16 chunks, the last one partial)"""
    M, N = tile_shape(sms, case)
    check(run(L, pair, "tc3", epi, M, N, 1088, seed=M), (case, pair, epi, M, N))


# ------------------------------------------------------------------------------------------------------ variants
LAYOUTS = {
    # name: (lda pad, ldb pad, ldo pad, alpha, bias, resid aliases out)
    "dense": (0, 0, 0, 1.0, True, True),
    "strided": (8, 16, 0, 1.0, True, False),     # lda, ldb > K; pads keep 16-byte rows in both formats
    "wide_ldo": (0, 0, 6, -0.3, False, False),    # ldo > n_out (even: the vector store path), alpha != 1, no bias
    "odd_ldo": (0, 8, 3, 0.7, True, False),       # odd ldo: the scalar store path
}


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("lom", [0, 1, 2, 3], ids=["hi_only", "a_lo", "b_lo", "a_lo+b_lo"])
@pytest.mark.parametrize("engine", ["simt", "tc3"])
@pytest.mark.parametrize("pair", ["tf32", "f16"])
def test_gemm_variants(L, pair, engine, lom, layout, epi):
    """every lo-operand variant (a_lo / b_lo nullable) with strided operands, wide / odd ldo, alpha != 1, bias=None,
    and a residual that is not the output; M = 200 and N = 136 leave tails in both"""
    M, N, K = 200, 136, 104
    pa, pb, po, alpha, use_bias, alias = LAYOUTS[layout]
    n_out = N // 2 if epi == "swiglu_split" else N
    check(run(L, pair, engine, epi, M, N, K, lom=lom, lda=K + pa, ldb=K + pb, ldo=n_out + po, alpha=alpha,
              use_bias=use_bias, resid_alias=alias, seed=lom * 7 + len(layout)), (pair, engine, lom, layout, epi))


def test_trunc_tf32_matches_cpu_model(L):
    x = torch.randn(4099, device="cuda") * torch.logspace(-30, 30, 4099, device="cuda")
    assert np.array_equal(trunc_tf32(x).cpu().numpy(), trunc_tf32_np(x.cpu().numpy()))


def test_hi_only_tf32_reads_truncated_words(L):
    """a raw fp32 a_hi is consumed truncated to tf32: the truncated reference passes the per-element bound, the
    round-to-nearest one (2^-11 relative away) does not"""
    M, N, K = 256, 136, 256
    ops = operands(L, M, N, K, "tf32", "tc3", lom=0, seed=3)
    val, ref, bound = run(L, "tf32", "tc3", "bias", M, N, K, lom=0, use_bias=False, seed=3)
    assert float(((val - ref).abs() / bound).max()) <= 1.0
    a_rn = ops["a_hi"].double()                           # the word as stored (closer to round-to-nearest)
    ref_rn = a_rn @ ops["B"].T
    assert float(((val - ref_rn).abs() / bound).max()) > 10.0


# --------------------------------------------------------------------------------------------- contract edges
EDGES = {
    # name: (pair, K, lda, a offset [elements], out offset [elements], bias offset, auto falls back to SIMT)
    "tf32_K%4": ("tf32", 34, 36, 0, 0, 0, False),
    "f16_K%8": ("f16", 36, 40, 0, 0, 0, True),
    "f16_lda%8": ("f16", 64, 68, 0, 0, 0, True),
    "f16_a+8B": ("f16", 64, 64, 4, 0, 0, True),
    "tf32_a+4B": ("tf32", 64, 64, 1, 0, 0, False),
    "tf32_out+4B": ("tf32", 64, 64, 0, 1, 0, True),
    "f16_out+4B": ("f16", 64, 64, 0, 1, 0, True),
    "tf32_bias+4B": ("tf32", 64, 64, 0, 0, 1, True),
}


@pytest.mark.parametrize("edge", list(EDGES))
def test_gemm_contract_edges(L, edge):
    """outside gemm_tc_supported the tensor-core engine returns ANYLOC_ERR_UNSUPPORTED and writes nothing; "auto" falls
    back to the SIMT engine and matches, or -- where SIMT cannot take the operands either -- returns an error"""
    pair, K, lda, a_off, o_off, b_off, falls_back = EDGES[edge]
    M, N = 100, 72
    g = torch.Generator(device="cuda").manual_seed(len(edge))
    a = torch.randn(M * lda + 16, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g) * 0.05
    bias_buf = torch.randn(N + 4, device="cuda", generator=g)
    bias = bias_buf[b_off:b_off + N]
    if pair == "tf32":
        a_hi, a_lo = split_tf32(L, a)
        b_hi, b_lo = split_tf32(L, b)
        A = a.double()[a_off:a_off + M * lda].view(M, lda)[:, :K]
        B, scale = b.double(), 1.0
    else:
        a_hi, a_lo = split_f16(L, a, L.ACT_SCALE)
        b_hi, b_lo = split_f16(L, b, 256.0)
        A = ((a_hi.double() + a_lo.double()) / L.ACT_SCALE)[a_off:a_off + M * lda].view(M, lda)[:, :K]
        B, scale = (b_hi.double() + b_lo.double()) / 256.0, 1.0 / (L.ACT_SCALE * 256.0)
    outs = {}
    for engine in ("tc3", "auto"):
        out = canary_buffer(M, N + o_off, torch.float32)
        ldo = N + o_off
        rc = L.load().anyloc_gemm_nt(
            C.c_void_p(a_hi.data_ptr() + a_off * a_hi.element_size()),
            C.c_void_p(a_lo.data_ptr() + a_off * a_lo.element_size()), lda, L.ptr(b_hi), L.ptr(b_lo), K, M, N, K,
            L.PAIR[pair], C.c_float(scale), L.EPI["bias"], C.c_void_p(bias.data_ptr()), None, None,
            C.c_void_p(out.data_ptr() + (LEAD + o_off) * 4), None, ldo, L.PAIR[pair], L.ENGINE[engine],
            L.stream_ptr())
        torch.cuda.synchronize()
        outs[engine] = (rc, out)
    rc, out = outs["tc3"]
    assert rc == UNSUPPORTED, (rc, L.last_error())
    assert bool((out.view(torch.int32) == NAN32).all()), "the refused call wrote its output"
    rc, out = outs["auto"]
    if not falls_back:
        assert rc != 0 and bool((out.view(torch.int32) == NAN32).all())
        return
    assert rc == 0, L.last_error()
    val = out[LEAD + o_off:LEAD + o_off + M * (N + o_off)].view(M, N + o_off)[:, :N].double()
    ref = A @ B.T + bias.double()                           # A, B hold the unscaled values; alpha undid the scales
    bound = C_ACC * U * K ** 0.5 * (A.abs() @ B.abs().T) + 2 * U * ref.abs()
    assert float(((val - ref).abs() / bound).max()) <= 1.0


# --------------------------------------------------------------------------------- round-to-nearest chunk adds
# The tensor core accumulates a chunk's wgmma k-steps in fp32 without rounding to nearest: each step drops less than one
# ulp (<= 2u |partial|) of the running partial sum, always toward zero.  With all-positive operands every partial is at
# most the chunk's total, so one chunk of n steps loses at most 2 n u of its value; the chunks themselves are added with
# round-to-nearest fp32 adds, which carry no bias.  n is 3 wgmmas (hi.hi, lo.hi, hi.lo) x 4 k-steps per 128-byte k-block
# x the k-blocks per chunk of gemm_tc.cu: CHUNK_KB_TF32 = 2 -> 24 steps, CHUNK_KB_F16 = 8 -> 96 steps.  Without chunks n
# is 3 K / 8 (tf32) or 3 K / 16 (fp16): at K = 16384, 6144 and 3072 steps.
TRUNC_STEPS = {"tf32": 24, "f16": 96}
RN_KS = (4096, 16384)


def rn_bias_threshold(pair):
    return 2 * TRUNC_STEPS[pair] * U


def rn_bias(L, pair, K):
    """signed relative bias mean((C - C64) sign(C64)) / mean|C64| of the 3-term tensor-core GEMM on uniform [0, 1)"""
    ops = operands(L, 256, 256, K, pair, "tc3", seed=K, dist="uniform")
    out = torch.empty(256, 256, device="cuda")
    L.check(gemm_nt(L, ops["a_hi"], ops["a_lo"], ops["b_hi"], ops["b_lo"], 256, 256, K, pair=pair, alpha=ops["scale"],
                    out=out, ldo=256), "gemm")
    ref = ops["A"] @ ops["B"].T
    return float(((out.double() - ref) * ref.sign()).mean() / ref.abs().mean())


def _rn_bias_main():
    """entry point of the mutation run (a separate process, so that ANYLOC_GEMM_CHUNK is read afresh)"""
    from anyloc_b200 import _lib
    _lib.load()
    print(json.dumps({f"{p}/{K}": rn_bias(_lib, p, K) for p in ("tf32", "f16") for K in RN_KS}))


def test_rn_chunk_bias(L):
    """Measured on one H100 SXM (80 GB HBM3, 700 W power limit), uniform [0, 1) operands, 256 x 256 outputs:
        chunked (default)  tf32: K=4096 -5.5e-7, K=16384 -5.5e-7   fp16: K=4096 -3.5e-6, K=16384 -3.6e-6
        one chunk          tf32: K=4096 -4.3e-5, K=16384 -1.7e-4   fp16: K=4096 -3.1e-5, K=16384 -1.3e-4
    against thresholds of 2.9e-6 (tf32) and 1.1e-5 (fp16): the chunked bias does not grow with K, the unchunked one
    grows linearly and clears the threshold by 2.8x (fp16, K=4096) to 60x (tf32, K=16384)."""
    for pair in ("tf32", "f16"):
        for K in RN_KS:
            b = rn_bias(L, pair, K)
            print(f"RN-chunk bias {pair} K={K}: chunked {b:+.2e} (threshold {rn_bias_threshold(pair):.1e})")
            assert abs(b) <= rn_bias_threshold(pair), (pair, K, b)


def test_rn_chunk_bias_mutation(L):
    """the same measurement with chunking switched off (ANYLOC_GEMM_CHUNK=100000: one chunk for the whole K) must exceed
    the threshold -- so the check above would catch a chunk length that silently stopped applying"""
    env = dict(os.environ, ANYLOC_GEMM_CHUNK="100000", PYTHONPATH=ROOT)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", "from tests.test_gemm_engine_gpu import _rn_bias_main; _rn_bias_main()"]
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    for key, b in sorted(res.items()):
        pair = key.split("/")[0]
        print(f"RN-chunk bias {key}: one chunk {b:+.2e} (threshold {rn_bias_threshold(pair):.1e})")
    for key, b in res.items():
        assert abs(b) > rn_bias_threshold(key.split("/")[0]), (key, b)


# ------------------------------------------------------------------------------------------------ batch invariance
@pytest.mark.parametrize("pair", ["tf32", "f16"])
def test_gemm_rows_batch_invariant(L, pair):
    """rows of A[:m] . B^T are bit-identical to the same rows of A . B^T, m cutting tiles anywhere"""
    g = torch.Generator(device="cuda").manual_seed(11)
    a = torch.randn(700, 264, device="cuda", generator=g)
    b = torch.randn(392, 264, device="cuda", generator=g) * 0.05
    bias = torch.randn(392, device="cuda", generator=g)
    full = gemm(L, a, b, "bias", bias, engine="tc3", pair=pair)
    for m in (32, 33, 64, 100, 128, 191, 256, 321, 699):
        part = gemm(L, a[:m].contiguous(), b, "bias", bias, engine="tc3", pair=pair)
        assert torch.equal(part, full[:m]), (pair, m)


@pytest.mark.parametrize("precision", ["tf32x3", "f16x3"])
def test_vit_batch_invariant(cuda, precision):
    """DinoV2ExtractFeatures(img)[i] == DinoV2ExtractFeatures(img[i:i+1])[0] bit for bit (T = 257): what the multi-GPU
    descriptors' equality with the single-GPU ones rests on"""
    from anyloc_b200 import utilities as u
    from anyloc_b200.vit import random_state_dict
    sd = random_state_dict("dinov2_vits14", seed=0, device="cuda", depth=3)
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 2, "value", device="cuda", weights=sd, precision=precision)
    img = torch.randn(3, 3, 224, 224, generator=torch.Generator().manual_seed(7)).cuda()
    full = ext(img)
    for i in range(3):
        assert torch.equal(ext(img[i:i + 1])[0], full[i]), (precision, i)
