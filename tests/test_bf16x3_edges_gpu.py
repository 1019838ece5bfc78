"""The bf16-pair GEMM and attention (ANYLOC_PAIR_BF16X3) at the edges the tf32 and fp16 pairs are tested at in
tests/test_gemm_engine_gpu.py, tests/test_gemm_epilogue_stage_gpu.py, tests/test_attention_edges_gpu.py and
tests/test_attention_tiles_gpu.py, under the bounds of tests/test_bf16x3_kernels_gpu.py (whose helpers run every case):

GEMM, element by element against fp64: the engine suite's N, K and M tails (K a multiple of 8, the format's 16 bytes),
every epilogue, on the tensor-core engine and on "auto", which must take the same route (the format has no SIMT
kernel); tiles around the SM count with K = 1088 (17 k-blocks of 64: two full round-to-nearest chunks of 8 and a
partial one); strided operands, wide and odd output pitches, alpha != 1 and no bias, and the LS_RESID residual in
place and in a canaried buffer of its own.  Outside the tensor-core contract both engines refuse and write nothing.
Rows do not depend on how many rows share the call.  The staged (TMA) epilogue and the register epilogue write the
same bits, hi and lo, and the canaries in the ldo padding survive both.  The round-to-nearest chunks keep the
accumulation unbiased, and a mutation run that switches them off shows the check would notice.

Attention, element by element against fp64 on the pair values: logits up to +-60 (a dominant key in the last, partial
key block, a ramp that raises the running maximum block after block, all keys equal), sequence lengths around the
64-key blocks and the 128-query tiles, and a 40-image x 24-head grid whose images, permuted, permute both output arrays
bit for bit.  Every output, hi and lo, lies inside NaN canaries that must survive, and every row below T is written.
Each bound test prints the worst share of its bound that it measured."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from tests.test_attention_edges_gpu import structured, to_qkv
from tests.test_attention_tiles_gpu import TS
from tests.test_bf16x3_kernels_gpu import (EPIS, LEAD, U, UNSUPPORTED, all_canary, attn_bound, bits, canaries, check,
                                           operands, pair_of, run_gemm, split_pair, untouched_outside, window)
from tests.test_gemm_engine_gpu import LAYOUTS, SHAPES, TILE_CASES, tile_shape
from tests.test_gemm_epilogue_stage_gpu import SHAPES as STAGE_SHAPES, staged_ldo
from tests.util import ROOT, dptr, gemm_nt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


@pytest.fixture(scope="module")
def sms(L):
    return torch.cuda.get_device_properties(0).multi_processor_count


def same_bits(a, b):
    idt = torch.int32 if a.dtype == torch.float32 else torch.int16
    return torch.equal(a.contiguous().view(idt), b.contiguous().view(idt))


# ------------------------------------------------------------------------------------------- shapes x epilogues
GEMM_SHAPES = sorted(s for s in SHAPES if SHAPES[s][2] % 8 == 0)       # K a whole number of 16 bytes


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("shape", GEMM_SHAPES)
def test_gemm_shapes(L, shape, epi):
    """odd N with the SPLIT epilogues: 2-byte pair words at an odd column count (register epilogue)"""
    M, N, K = SHAPES[shape]
    if epi == "swiglu_split" and N % 2:
        pytest.skip("SwiGLU needs even N")
    res = {}
    for engine in ("tc3", "auto"):
        got, ref, err, staged = run_gemm(L, epi, M, N, K, seed=M + N + K, engine=engine)
        res[engine] = (check(got, ref, err, (shape, engine, epi)), got, staged)
    print(f"{shape} {epi}: worst share of the bound {max(r[0] for r in res.values()):.3f}")
    assert torch.equal(res["tc3"][1], res["auto"][1]) and res["tc3"][2] == res["auto"][2], (shape, epi)


@pytest.mark.parametrize("epi", ["bias", "bias_split", "swiglu_split", "ls_resid"])
@pytest.mark.parametrize("case", list(TILE_CASES))
def test_gemm_persistent_tiles(L, sms, case, epi):
    """more tiles than SMs: a CTA runs its next tile on the stage/phase ring state the last one left"""
    M, N = tile_shape(sms, case)
    got, ref, err, _ = run_gemm(L, epi, M, N, 1088, seed=M, engine="tc3")
    print(f"{case} {epi}: worst share of the bound {check(got, ref, err, (case, epi, M, N)):.3f}")


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_gemm_layouts(L, layout, epi):
    """M = 200 and N = 136 leave tails in both; "dense" runs LS_RESID in place, the others on a canaried residual"""
    M, N, K = 200, 136, 104
    pa, pb, po, alpha, use_bias, alias = LAYOUTS[layout]
    n_out = N // 2 if epi == "swiglu_split" else N
    got, ref, err, _ = run_gemm(L, epi, M, N, K, lda=K + pa, ldb=K + pb, ldo=n_out + po, alpha=alpha,
                                use_bias=use_bias, resid="in_place" if alias else "separate", seed=len(layout),
                                engine="tc3")
    print(f"{layout} {epi}: worst share of the bound {check(got, ref, err, (layout, epi)):.3f}")


# --------------------------------------------------------------------------------------------- contract edges
EDGES = {
    # name: (epilogue, K, lda, {pointer: byte offset})
    "K36": ("bias_split", 36, 40, {}),
    "lda68": ("bias_split", 64, 68, {}),
    "a_hi+8B": ("bias_split", 64, 64, {"a_hi": 8}),
    "a_lo+8B": ("bias_split", 64, 64, {"a_lo": 8}),
    "b_lo+8B": ("bias_split", 64, 64, {"b_lo": 8}),
    "out+4B": ("bias_split", 64, 64, {"out": 4}),
    "out_lo+4B": ("bias_split", 64, 64, {"out_lo": 4}),
    "bias+4B": ("bias_split", 64, 64, {"bias": 4}),
    "gamma+4B": ("ls_resid", 64, 64, {"gamma": 4}),
}


@pytest.mark.parametrize("edge", list(EDGES))
def test_gemm_contract_edges(L, edge):
    """outside gemm_tc_supported both the tensor-core engine and "auto" return ANYLOC_ERR_UNSUPPORTED (the format has
    no SIMT kernel to fall back to) and write nothing"""
    epi, K, lda, offs = EDGES[edge]
    M, N = 100, 72
    g = torch.Generator(device="cuda").manual_seed(len(edge))
    a_hi, a_lo = split_pair(L, torch.randn(M * lda + 16, device="cuda", generator=g))
    b_hi, b_lo = split_pair(L, torch.randn(N * K + 16, device="cuda", generator=g) * 0.05)
    bias = torch.randn(N + 4, device="cuda", generator=g)
    gamma = torch.randn(N + 4, device="cuda", generator=g) if epi == "ls_resid" else None
    split = "split" in epi
    lib = L.load()
    for engine in ("tc3", "auto"):
        out = canaries(M, N, split)
        out_lo = canaries(M, N, True) if split else None
        resid = canaries(M, N, False) if epi == "ls_resid" else None
        if resid is not None:
            window(resid, M, N, N).copy_(torch.randn(M, N, device="cuda", generator=g))

        def p(name, t, lead=0):
            return None if t is None else C.c_void_p(t.data_ptr() + lead * t.element_size() + offs.get(name, 0))
        rc = lib.anyloc_gemm_nt(p("a_hi", a_hi), p("a_lo", a_lo), lda, p("b_hi", b_hi), p("b_lo", b_lo), K, M, N, K,
                                L.PAIR["bf16pair"], C.c_float(1.0), L.EPI[epi], p("bias", bias), p("gamma", gamma),
                                p("resid", resid, LEAD), p("out", out, LEAD), p("out_lo", out_lo, LEAD), N,
                                L.PAIR["bf16pair"], L.ENGINE[engine], L.stream_ptr())
        torch.cuda.synchronize()
        assert rc == UNSUPPORTED, (edge, engine, rc, L.last_error())
        assert all_canary(out), (edge, engine, "the refused call wrote its output")
        assert out_lo is None or all_canary(out_lo), (edge, engine, "the refused call wrote out_lo")
        assert resid is None or untouched_outside(resid, M, N, N) == 0, (edge, engine)


# ------------------------------------------------------------------------------------------------ batch invariance
@pytest.mark.parametrize("epi", ["bias", "bias_split"])
def test_gemm_rows_batch_invariant(L, epi):
    """rows of A[:m] . B^T are bit-identical (hi and lo) to the same rows of A . B^T, m cutting tiles anywhere"""
    M, N, K = 700, 392, 264
    (a_hi, a_lo), (b_hi, b_lo) = operands(L, M, N, K, 11)
    bias = torch.randn(N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(12))
    split = "split" in epi

    def run(m):
        dt = torch.bfloat16 if split else torch.float32
        out = torch.empty(m, N, dtype=dt, device="cuda")
        out_lo = torch.empty(m, N, dtype=dt, device="cuda") if split else None
        assert gemm_nt(L, a_hi[:m].contiguous(), a_lo[:m].contiguous(), b_hi, b_lo, m, N, K, pair="bf16pair", epi=epi,
                       bias=bias, out=out, out_lo=out_lo, ldo=N, engine="auto") == 0, L.last_error()
        return [t for t in (out, out_lo) if t is not None]

    full = run(M)
    for m in (1, 31, 32, 33, 64, 65, 100, 128, 191, 256, 321, 699):
        part = run(m)
        torch.cuda.synchronize()
        for i, (p, f) in enumerate(zip(part, full)):
            assert same_bits(p, f[:m]), (epi, m, ("hi", "lo")[i])


# -------------------------------------------------------------------------------------- staged vs register epilogue
def run_once(L, ops, epi, M, N, K, ldo, alpha, bias, gamma, resid_t, resid_alias):
    """one tc3 call into NaN-canaried buffers of pitch ldo -> the [M, n_out] outputs (out and out_lo), staged"""
    (a_hi, a_lo), (b_hi, b_lo) = ops
    n_out = N // 2 if epi == "swiglu_split" else N
    split = "split" in epi
    out = canaries(M, ldo, split)
    out_lo = canaries(M, ldo, True) if split else None
    resid_buf = None
    if epi == "ls_resid":
        resid_buf = out if resid_alias else canaries(M, ldo, False)
        window(resid_buf, M, ldo, n_out).copy_(resid_t)
    rc = gemm_nt(L, a_hi, a_lo, b_hi, b_lo, M, N, K, pair="bf16pair", alpha=alpha, epi=epi, bias=bias, gamma=gamma,
                 resid=resid_buf, out=out, out_lo=out_lo, ldo=ldo, engine="tc3", out_off=LEAD)
    torch.cuda.synchronize()
    assert rc == 0, (rc, L.last_error())
    staged = L.load().anyloc_gemm_tc_last_staged()
    res = []
    for name, buf in (("out", out), ("out_lo", out_lo)):
        if buf is not None:
            assert untouched_outside(buf, M, ldo, n_out) == 0, (name, f"ldo={ldo}", "written outside [M, n_out]")
            res.append(window(buf, M, ldo, n_out).contiguous())
    if resid_buf is not None and not resid_alias:
        assert untouched_outside(resid_buf, M, ldo, n_out) == 0, ("resid", f"ldo={ldo}")
    return res, staged


def compare(L, epi, M, N, K, *, pad=0, alpha=1.0, use_bias=True, resid_alias=True, seed=0):
    """staged (pitch staged_ldo(n_out, pad)) vs register path (that pitch + 1) on the same operands: bit-identical;
    the staged call must have staged wherever the output row is a whole number of 16-byte units (2-byte pair words
    for the SPLIT outputs, fp32 for BIAS and LS_RESID)"""
    ops = operands(L, M, N, K, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    n_out = N // 2 if epi == "swiglu_split" else N
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    resid_t = torch.randn(M, n_out, device="cuda", generator=g) if epi == "ls_resid" else None
    ldo = staged_ldo(n_out, pad)
    staged, path_s = run_once(L, ops, epi, M, N, K, ldo, alpha, bias, gamma, resid_t, resid_alias)
    regs, path_r = run_once(L, ops, epi, M, N, K, ldo + 1, alpha, bias, gamma, resid_t, resid_alias)
    esz = 2 if "split" in epi else 4
    assert (path_s, path_r) == (int((n_out * esz) % 16 == 0), 0), (path_s, path_r)
    for name, s, r in zip(("out", "out_lo"), staged, regs):
        assert same_bits(s, r), (name, "the staged and the register path differ")


@pytest.mark.parametrize("epi", EPIS)
def test_staged_modes(L, epi):
    """M = 200, N = 144: tails in both; the second warpgroup of the last row block holds 8 rows"""
    compare(L, epi, 200, 144, 104, seed=len(epi))


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("shape", list(STAGE_SHAPES))
def test_staged_shapes(L, shape, epi):
    M, N = STAGE_SHAPES[shape]
    compare(L, epi, M, N, 256, seed=M + N)


@pytest.mark.parametrize("epi", EPIS)
def test_staged_many_tiles(L, sms, epi):
    """2 x SMs + 1 tiles: every CTA reuses its staging buffers (and LS_RESID its residual barriers) across tiles"""
    M, N = tile_shape(sms, "tiles=2SMs+1")
    compare(L, epi, M, N + 12, 320, seed=M)


@pytest.mark.parametrize("resid_alias", [True, False], ids=["in_place", "separate"])
def test_staged_residual(L, resid_alias):
    compare(L, "ls_resid", 1088, 392, 264, resid_alias=resid_alias, seed=7)


@pytest.mark.parametrize("epi", EPIS)
def test_staged_alpha_no_bias_wide_ldo(L, epi):
    compare(L, epi, 300, 272, 104, pad=16, alpha=-0.3, use_bias=False, resid_alias=False, seed=3)


# --------------------------------------------------------------------------------- round-to-nearest chunk adds
# As for the fp16 pairs (tests/test_gemm_engine_gpu.py): the tensor core truncates within a chunk of n wgmma k-steps,
# at most 2 n u of the chunk's value with all-positive operands, and the chunks are added with round-to-nearest.  The
# bf16 pairs take CHUNK_KB_F16 = 8 k-blocks per chunk: 3 wgmmas x 4 k-steps x 8 = 96 steps, threshold 2 * 96 u.  The
# reference is the three products the kernel computes, A_hi B_hi^T + A_lo B_hi^T + A_hi B_lo^T, in fp64, so the dropped
# A_lo B_lo^T can neither hide a bias nor fake one.
RN_KS = (4096, 16384)
RN_THRESHOLD = 2 * 96 * U


def rn_bias(L, K):
    """signed relative bias mean((C - C64) sign(C64)) / mean|C64| on uniform [0, 1) operands, 256 x 256 outputs"""
    g = torch.Generator(device="cuda").manual_seed(K)
    (a_hi, a_lo), (b_hi, b_lo) = (split_pair(L, torch.rand(256, K, device="cuda", generator=g)) for _ in range(2))
    out = torch.empty(256, 256, device="cuda")
    L.check(gemm_nt(L, a_hi, a_lo, b_hi, b_lo, 256, 256, K, pair="bf16pair", out=out, ldo=256), "gemm bf16pair")
    ah, al, bh, bl = (t.double() for t in (a_hi, a_lo, b_hi, b_lo))
    ref = ah @ bh.T + al @ bh.T + ah @ bl.T
    return float(((out.double() - ref) * ref.sign()).mean() / ref.abs().mean())


def _rn_bias_main():
    """entry point of the mutation run (a separate process, so that ANYLOC_GEMM_CHUNK is read afresh)"""
    from anyloc_b200 import _lib
    _lib.load()
    print(json.dumps({str(K): rn_bias(_lib, K) for K in RN_KS}))


def test_rn_chunk_bias(L):
    """Measured on one H100 SXM (80 GB HBM3, 700 W power limit), uniform [0, 1) operands, 256 x 256 outputs:
        chunked (default)  K=4096 -1.7e-6, K=16384 -1.7e-6
        one chunk          K=4096 -1.9e-5, K=16384 -1.0e-4
    against a threshold of 1.1e-5: the chunked bias does not grow with K and stays 6x below it; the unchunked one grows
    linearly and clears it by 1.7x at K=4096 and 8.9x at K=16384."""
    for K in RN_KS:
        b = rn_bias(L, K)
        print(f"RN-chunk bias bf16pair K={K}: chunked {b:+.2e} (threshold {RN_THRESHOLD:.1e})")
        assert abs(b) <= RN_THRESHOLD, (K, b)


def test_rn_chunk_bias_mutation(L):
    """the same measurement with chunking switched off (ANYLOC_GEMM_CHUNK=100000: one chunk for the whole K) must exceed
    the threshold -- so the check above would catch a chunk length that silently stopped applying"""
    env = dict(os.environ, ANYLOC_GEMM_CHUNK="100000", PYTHONPATH=ROOT)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", "from tests.test_bf16x3_edges_gpu import _rn_bias_main; _rn_bias_main()"]
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    for K, b in sorted(res.items()):
        print(f"RN-chunk bias bf16pair K={K}: one chunk {b:+.2e} ({abs(b) / RN_THRESHOLD:.1f}x the threshold)")
    for K, b in res.items():
        assert abs(b) > RN_THRESHOLD, (K, b)


# ---------------------------------------------------------------------------------------------------------- attention
def attention(L, qkv, heads):
    """fp32 qkv [B, T, 3D] -> its pairs' values [B, T, 3, H, 64] (doubles) and the attention's (hi, lo) [B*T, D],
    written inside NaN canaries that must survive"""
    B, T, D3 = qkv.shape
    D = D3 // 3
    hi, lo = pair_of(qkv.reshape(B * T, D3).contiguous())
    o, o_lo = canaries(B * T, D, True), canaries(B * T, D, True)
    L.check(L.load().anyloc_attention(dptr(hi), dptr(lo), B, T, D, heads, dptr(o, LEAD), dptr(o_lo, LEAD),
                                      L.PAIR["bf16pair"], L.ENGINE["tc3"], L.stream_ptr()), "attention bf16pair")
    torch.cuda.synchronize()
    assert untouched_outside(o, B * T, D, D) == 0 and untouched_outside(o_lo, B * T, D, D) == 0, (B, T, heads)
    X = (hi.double() + lo.double()).reshape(B, T, 3, heads, 64)
    return X, window(o, B * T, D, D), window(o_lo, B * T, D, D)


def share(X, o, o_lo):
    """max |o - o64| / attn_bound over every element; every row below T written (no NaN canary left, none made)"""
    B, T, _, H, _ = X.shape
    got = (o.double() + o_lo.double()).reshape(B, T, H, 64).transpose(1, 2)
    assert bool(torch.isfinite(got).all())
    ref, bound = attn_bound(X)
    return float(((got - ref).abs() / bound).max())


@pytest.mark.parametrize("kind", ["flat", "dominant_last", "ramp", "equal"])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 127, 1025])
def test_attention_edges(L, T, kind):
    B, heads = 2, 3
    X, o, o_lo = attention(L, to_qkv(*structured(kind, B, heads, T, seed=T * 10 + len(kind))), heads)
    if kind in ("dominant_last", "ramp") and T > 1:     # the construction does what it claims, on the pair values
        logits = X[:, :, 0].transpose(1, 2) @ X[:, :, 1].transpose(1, 2).transpose(-1, -2) / 8
        assert float(logits.abs().max()) > 50.0
        if kind == "dominant_last":
            assert bool((logits.argmax(-1) == T - 1).all())
    s = share(X, o, o_lo)
    print(f"attention bf16pair {kind} T={T}: worst share of the bound {s:.3f}")
    assert s <= 1.0, (kind, T, s)


@pytest.mark.parametrize("kind", ["flat", "dominant_last"])
@pytest.mark.parametrize("T", TS)
def test_attention_at_tile_edges(L, T, kind):
    B, heads = 3, 2
    X, o, o_lo = attention(L, to_qkv(*structured(kind, B, heads, T, seed=T * 7 + len(kind))), heads)
    s = share(X, o, o_lo)
    print(f"attention bf16pair {kind} T={T}: worst share of the bound {s:.3f}")
    assert s <= 1.0, (kind, T, s)


def test_attention_large_grid_permutation(L):
    """B = 40 images x 24 heads with different data each: correct everywhere, and permuting the images permutes both
    output arrays bit for bit (no state leaks between (image, head) CTAs)"""
    B, heads, T = 40, 24, 130
    D = 64 * heads
    g = torch.Generator(device="cuda").manual_seed(40)
    qkv = torch.randn(B, T, 3 * D, device="cuda", generator=g) * \
        torch.rand(B, 1, 1, device="cuda", generator=g).add(0.5) * 1.5
    X, o, o_lo = attention(L, qkv, heads)
    s = share(X, o, o_lo)
    print(f"attention bf16pair grid 40x24: worst share of the bound {s:.3f}")
    assert s <= 1.0, s
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(3)).cuda()
    _, o_p, o_lo_p = attention(L, qkv[perm].contiguous(), heads)
    for a, b in ((o, o_p), (o_lo, o_lo_p)):
        assert torch.equal(bits(b.reshape(B, T, D)), bits(a.reshape(B, T, D)[perm]))
