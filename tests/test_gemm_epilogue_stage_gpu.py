"""The tensor-core GEMM stores its epilogue in two ways: staged through shared memory and TMA when the output's row pitch
and row length are multiples of 16 bytes, pair by pair from registers otherwise.  Both apply the same arithmetic, so
every case here runs twice on the same operands -- once with a TMA-storable ldo, once with an odd ldo that forces the
register path -- and the valid outputs must agree bit for bit, while NaN canaries in the ldo padding and in the rows
past M survive.  Each launch also reports which epilogue it ran (anyloc_gemm_tc_last_staged), so a case that meant to
stage cannot silently compare the register path with itself.  The hi-only passes (no lo operand) always use the
register epilogue.
Covered: every epilogue mode x both pair formats x the three lo-operand variants, M and N tails, M <= 64 (the second
consumer warpgroup has no rows), half tiles in M, more than 2 x SMs tiles (staging buffers reused across tiles), an
in-place and a separate residual, alpha != 1 and no bias."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests.test_gemm_engine_gpu import EPIS, LEAD, assert_canaries, canary_buffer, operands, tile_shape, window
from tests.util import ROOT, gemm_nt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


@pytest.fixture(scope="module")
def sms(L):
    return torch.cuda.get_device_properties(0).multi_processor_count


def staged_ldo(n_out, pad=0):
    """a row pitch TMA can store in both output element sizes (a multiple of 8 elements)"""
    return (n_out + 7) // 8 * 8 + pad


def run_once(L, ops, pair, epi, M, N, K, ldo, alpha, bias, gamma, resid_t, resid_alias):
    """one tc3 call into NaN-canaried buffers of pitch ldo -> the [M, n_out] bit patterns of out (and out_lo)"""
    n_out = N // 2 if epi == "swiglu_split" else N
    is_split = "split" in epi
    odt = torch.float16 if (is_split and pair == "f16") else torch.float32
    idt = torch.int16 if odt == torch.float16 else torch.int32
    out = canary_buffer(M, ldo, odt)
    out_lo = canary_buffer(M, ldo, odt) if is_split else None
    resid_buf = None
    if epi == "ls_resid":
        if resid_alias:
            window(out, M, ldo, n_out).copy_(resid_t)
            resid_buf = out
        else:
            resid_buf = canary_buffer(M, ldo, torch.float32)
            window(resid_buf, M, ldo, n_out).copy_(resid_t)
    rc = gemm_nt(L, ops["a_hi"], ops["a_lo"], ops["b_hi"], ops["b_lo"], M, N, K, pair=pair, alpha=alpha * ops["scale"],
                 epi=epi, bias=bias, gamma=gamma, resid=resid_buf, out=out, out_lo=out_lo, ldo=ldo, lda=ops["lda"],
                 ldb=ops["ldb"], engine="tc3", out_off=LEAD)
    torch.cuda.synchronize()
    assert rc == 0, (rc, L.last_error())
    staged = L.load().anyloc_gemm_tc_last_staged()
    assert_canaries(out, M, ldo, n_out, f"out (ldo={ldo})")
    res = [window(out, M, ldo, n_out).contiguous().view(idt)]
    if out_lo is not None:
        assert_canaries(out_lo, M, ldo, n_out, f"out_lo (ldo={ldo})")
        res.append(window(out_lo, M, ldo, n_out).contiguous().view(idt))
    if resid_buf is not None and not resid_alias:
        assert_canaries(resid_buf, M, ldo, n_out, f"resid (ldo={ldo})")
    return res, staged


def stages(pair, epi, N, lom):
    """whether the tensor-core GEMM takes the staged epilogue at a TMA-storable ldo: 3-term passes whose rows are a
    whole number of 16-byte units"""
    n_out = N // 2 if epi == "swiglu_split" else N
    esz = 2 if ("split" in epi and pair == "f16") else 4
    return lom != 0 and (n_out * esz) % 16 == 0


def compare(L, pair, epi, M, N, K, *, lom=3, pad=0, alpha=1.0, use_bias=True, resid_alias=True, seed=0):
    """staged (pitch staged_ldo(n_out, pad)) vs register path (that pitch + 1) on the same operands: bit-identical"""
    ops = operands(L, M, N, K, pair, "tc3", lom, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    n_out = N // 2 if epi == "swiglu_split" else N
    bias = torch.randn(N, device="cuda", generator=g) if use_bias else None
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    resid_t = torch.randn(M, n_out, device="cuda", generator=g) if epi == "ls_resid" else None
    ldo = staged_ldo(n_out, pad)
    staged, path_s = run_once(L, ops, pair, epi, M, N, K, ldo, alpha, bias, gamma, resid_t, resid_alias)
    regs, path_r = run_once(L, ops, pair, epi, M, N, K, ldo + 1, alpha, bias, gamma, resid_t, resid_alias)
    assert (path_s, path_r) == (int(stages(pair, epi, N, lom)), 0), (path_s, path_r)
    for name, s, r in zip(("out", "out_lo"), staged, regs):
        diff = int((s != r).sum())
        assert diff == 0, (name, f"{diff} of {s.numel()} elements differ between the staged and the register path")


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("lom", [1, 2, 3], ids=["a_lo", "b_lo", "a_lo+b_lo"])
@pytest.mark.parametrize("pair", ["tf32", "f16"])
def test_staged_modes(L, pair, lom, epi):
    """M = 200, N = 144: tails in both; the second warpgroup of the last row block holds 8 rows"""
    compare(L, pair, epi, 200, 144, 104, lom=lom, seed=lom * 5 + len(epi))


# (M, N): M <= 64, half row blocks, N tails (N = 2 and 254 leave rows the register path stores in every format, N = 100
# in the fp16 formats)
SHAPES = {"M1": (1, 256), "M40": (40, 144), "M64": (64, 256), "M65": (65, 208), "half_tiles": (1088, 1536),
          "N2": (300, 2), "N16": (300, 16), "N100": (300, 100), "N176": (300, 176), "N254": (300, 254)}


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("pair", ["tf32", "f16"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_staged_shapes(L, shape, pair, epi):
    M, N = SHAPES[shape]
    compare(L, pair, epi, M, N, 256, seed=M + N)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("pair", ["tf32", "f16"])
def test_staged_many_tiles(L, sms, pair, epi):
    """2 x SMs + 1 tiles: every CTA reuses its staging buffers (and LS_RESID its residual barriers) across tiles"""
    M, N = tile_shape(sms, "tiles=2SMs+1")
    N += 12                               # a 112-column tail: rows of 16-byte multiples in every output format
    compare(L, pair, epi, M, N, 320, seed=M)


@pytest.mark.parametrize("resid_alias", [True, False], ids=["in_place", "separate"])
@pytest.mark.parametrize("pair", ["tf32", "f16"])
def test_staged_residual(L, pair, resid_alias):
    """LS_RESID with the residual aliasing the output (the ViT's residual stream) or in a buffer of its own"""
    compare(L, pair, "ls_resid", 1088, 392, 264, resid_alias=resid_alias, seed=7)


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("pair", ["tf32", "f16"])
def test_staged_alpha_no_bias_wide_ldo(L, pair, epi):
    compare(L, pair, epi, 300, 272, 104, lom=1, pad=16, alpha=-0.3, use_bias=False, resid_alias=False, seed=3)


def _skip_epi_main():
    """entry point of the discard run (a separate process, so that ANYLOC_GEMM_DEBUG_SKIP_EPI is read afresh)"""
    from anyloc_b200 import _lib
    _lib.load()
    ops = operands(_lib, 300, 256, 128, "f16", "tc3")
    out = canary_buffer(300, 256, torch.float32)
    rc = gemm_nt(_lib, ops["a_hi"], ops["a_lo"], ops["b_hi"], ops["b_lo"], 300, 256, 128, pair="f16",
                 alpha=ops["scale"], epi="bias", out=out, ldo=256, engine="tc3", out_off=LEAD)
    torch.cuda.synchronize()
    print(json.dumps({"rc": rc, "staged": _lib.load().anyloc_gemm_tc_last_staged(),
                      "written": int((out.view(torch.int32) != 0x7FC0DEAD).sum())}))


def test_debug_skip_epilogue_discards(L):
    """ANYLOC_GEMM_DEBUG_SKIP_EPI (the no-epilogue timing of tools/diag_gemm.py) stores nothing and stages nothing"""
    env = dict(os.environ, ANYLOC_GEMM_DEBUG_SKIP_EPI="1", PYTHONPATH=ROOT)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", "from tests.test_gemm_epilogue_stage_gpu import _skip_epi_main; _skip_epi_main()"]
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert res == {"rc": 0, "staged": 0, "written": 0}, res
