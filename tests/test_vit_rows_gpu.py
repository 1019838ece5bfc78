"""The ViT's row kernels element by element against fp64: anyloc_layernorm_split (tf32 and fp16 pairs; the single bf16
and e4m3 outputs are rounded from the same fp32 value, which test_bf16_kernels_gpu / test_fp8_kernels_gpu pin) and
anyloc_l2_normalize_rows (VLAD.fit's F.normalize).  Every output carries NaN canaries before and after it.

LayerNorm bound.  One warp per row; lane l sums its float4s d = l, l + 32, ... (2 adds inside a float4, at most MAXV
steps: MAXV = 4, 8, 16 for D <= 512, 1024, 2048), then 5 butterfly levels, so every fp32 sum has depth
k = MAXV + 7 + 1 (the division by D).  With u = 2^-24, mu64, r64 = 1/sqrt(var64 + eps) and yhat64 = (x - mu64) r64 the
fp64 statistics of the fp32 row:
  |mu - mu64|    <= k u mean|x|                      (recursive summation)
  (x - mu)       =  (x - mu64)(1 + u) + O(k u mean|x|)
  rstd           =  r64 (1 + O(k u))                  (the squared deviations sum at depth k; the mean's error enters
                                                       only at second order; rsqrtf adds 2 ulp)
  y = ((x - mu) rstd) w + b  adds 3 roundings, so
  |y - y64| <= c u ( r64 |w| (|x - mu64| + k mean|x|) + k |yhat64 w| + |b| ).
tf32 pairs hold y exactly (hi + lo == y).  fp16 pairs of 8 y add two terms to the bracket: 2^-22 |y| (the lo half
keeps 11 bits of a value below 2^-11 |8 y|) and an absolute floor: lo rounds to the fp16 subnormal spacing 2^-24, and
so does hi once |8 y| < 2^-14, which is 2 * 2^-25 / 8 = 2^-27 in y.  Rows of constant value (variance 0,
rstd = 1/sqrt(eps)), a large common offset (a one-pass variance E[x^2] - mu^2 cancels catastrophically there), a
DINOv2-like high-norm element, zeros and rows of 1e-20 (eps dominates; bias 0 so the output is not swamped by b) are
covered, and one eps other than 1e-6.  Measured worst |y - y64| / (u bracket) on an H100 80GB HBM3 (700 W): 0.94
(tf32 pairs, D = 2048), 0.74 (fp16 pairs); C_LN is 1.5x the worst, rounded up to a power of two.

l2 bound.  Lane sums of x^2 at depth D/128 + 3, 5 butterfly levels, sqrt and one division: |y - y64| <= c u k |y64|
with k = ceil(D / 128) + 10; rows of norm below 1e-12 are divided by 1e-12, zero rows stay 0.  Measured worst
|y - y64| / (u k |y64|) on an H100 80GB HBM3 (700 W): 0.26 (D = 128); C_L2 as C_LN."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LEAD = 16                   # canary elements before and after every output (64 B fp32, 32 B fp16, 16 B e4m3)
C_LN = 2.0
C_L2 = 0.5
F16_FLOOR = 2.0 ** -27
EPS32 = float(np.float32(1e-6))
DS = [4, 36, 128, 508, 512, 516, 1020, 1024, 1028, 1536, 2044, 2048]
MS = [1, 7, 8, 9, 531]
KINDS = ["random", "offset", "constant", "spike", "zeros", "tiny"]


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def _rows(M, D, seed):
    """M rows of width D, row r of kind KINDS[r % 6] (M >= 6 holds every kind)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.empty(M, D)
    for r in range(M):
        kind = KINDS[r % len(KINDS)]
        z = torch.randn(D, generator=g)
        if kind == "random":
            x[r] = z * (0.5 + torch.rand(1, generator=g)) + 0.3 * torch.randn(1, generator=g)
        elif kind == "offset":
            x[r] = 1e3 + z
        elif kind == "constant":
            x[r] = torch.randn(1, generator=g).expand(D)
        elif kind == "spike":
            x[r] = z
            x[r, int(torch.randint(D, (1,), generator=g))] = 1e4
        elif kind == "zeros":
            x[r] = 0.0
        else:
            x[r] = z * 1e-20
    return x


def _guarded(n, dtype, fill):
    """a device buffer of n elements with LEAD canary elements on both sides, filled with `fill` (a NaN pattern)"""
    buf = torch.empty(n + 2 * LEAD, dtype=dtype, device="cuda")
    if dtype == torch.uint8:
        buf.fill_(fill)
    else:
        buf.view(torch.int32 if dtype == torch.float32 else torch.int16).fill_(fill)
    return buf


def _dptr(buf):
    return C.c_void_p(buf.data_ptr() + LEAD * buf.element_size())


def _canaries_intact(buf, n):
    edges = torch.cat([buf[:LEAD], buf[LEAD + n:]])
    if buf.dtype == torch.uint8:
        return bool((edges == 0x7F).all())
    return bool(torch.isnan(edges.float()).all())


def _ln_ref(x, w, b, eps):
    """fp64 LayerNorm of the fp32 inputs, and the bound's scale (the bracket of the module docstring, times u)"""
    x64, w64, b64 = x.double(), w.double(), b.double()
    mu = x64.mean(dim=1, keepdim=True)
    r = 1.0 / torch.sqrt(((x64 - mu) ** 2).mean(dim=1, keepdim=True) + eps)
    yhat = (x64 - mu) * r
    y = yhat * w64 + b64
    D = x.shape[1]
    k = (4 if D <= 512 else 8 if D <= 1024 else 16) + 8
    scale = U * (r * w64.abs() * ((x64 - mu).abs() + k * x64.abs().mean(dim=1, keepdim=True)) +
                 k * (yhat * w64).abs() + b64.abs())
    return y, scale


def _layernorm(L, x, w, b, eps, fmt):
    """anyloc_layernorm_split into canary-guarded outputs -> the outputs (without canaries) after checking them"""
    M, D = x.shape
    n = M * D
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    if fmt == "fp8":
        hi, lo = _guarded(n, torch.uint8, 0x7F), _guarded(M, torch.float32, 0x7FC0DEAD)
    else:
        dt = torch.float16 if fmt == "f16" else torch.float32
        fill = 0x7E5A if fmt == "f16" else 0x7FC0DEAD
        hi, lo = _guarded(n, dt, fill), _guarded(n, dt, fill)
    L.check(L.load().anyloc_layernorm_split(L.ptr(xd), L.ptr(wd), L.ptr(bd), M, D, C.c_float(eps), _dptr(hi), _dptr(lo),
                                            L.PAIR[fmt], L.stream_ptr()), "layernorm")
    torch.cuda.synchronize()
    assert _canaries_intact(hi, n) and _canaries_intact(lo, M if fmt == "fp8" else n), (fmt, M, D)
    return hi[LEAD:LEAD + n].view(M, D), lo[LEAD:LEAD + (M if fmt == "fp8" else n)]


def _ln_check(L, x, w, b, eps, fmt):
    """worst |y - y64| / (u-scaled bound) of one call"""
    M, D = x.shape
    hi, lo = _layernorm(L, x, w, b, eps, fmt)
    y = (hi.double() + lo.view(M, D).double()).cpu()
    if fmt == "f16":
        y = y / L.ACT_SCALE
    ref, scale = _ln_ref(x, w, b, eps)
    if fmt == "f16":
        scale = scale + 2.0 ** -22 * ref.abs() + F16_FLOOR
    assert bool(torch.isfinite(y).all()), (fmt, M, D)
    return float(((y - ref).abs() / scale).max())


def _gains(D, seed):
    g = torch.Generator().manual_seed(seed)
    return 1.0 + 0.5 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)


@pytest.mark.parametrize("fmt", ["tf32", "f16"])
@pytest.mark.parametrize("D", DS)
def test_layernorm_elementwise(L, fmt, D):
    w, b = _gains(D, D)
    worst = {}
    for M in MS:
        x = _rows(M, D, seed=1000 * D + M)
        worst[M] = max(_ln_check(L, x, w, b, EPS32, fmt), _ln_check(L, x, w, torch.zeros(D), EPS32, fmt))
    print(f"layernorm {fmt} D={D}: worst |y - y64| / (u bound) by M {worst}")
    assert max(worst.values()) <= C_LN, (fmt, D, worst)


@pytest.mark.parametrize("fmt", ["tf32", "f16"])
def test_layernorm_honours_eps(L, fmt):
    """eps 1e-3 next to rows of variance 1e-4 .. 1e-2: a kernel that ignored the argument would miss by ~10 %"""
    D, M = 384, 64
    g = torch.Generator().manual_seed(7)
    x = torch.randn(M, D, generator=g) * torch.logspace(-2, -1, M)[:, None]
    w, b = _gains(D, 3)
    eps = float(np.float32(1e-3))
    assert _ln_check(L, x, w, b, eps, fmt) <= C_LN
    y_hi, y_lo = _layernorm(L, x, w, b, eps, fmt)
    y = (y_hi.double() + y_lo.view(M, D).double()).cpu() / (L.ACT_SCALE if fmt == "f16" else 1.0)
    wrong, _ = _ln_ref(x, w, b, EPS32)
    assert float((y - wrong).abs().max()) > 0.05


def test_layernorm_fp8_canaries(L):
    """the single-e4m3 output's rows and its [M] row scales stay inside their buffers at every width class"""
    for D in (36, 516, 2044):
        w, b = _gains(D, D)
        for M in (1, 9, 531):
            q, s = _layernorm(L, _rows(M, D, seed=M + D), w, b, EPS32, "fp8")
            assert bool(torch.isfinite(s).all()) and bool((s > 0).all())


def _l2(L, x, D, ld):
    rows = x.shape[0]
    y = _guarded(rows * D, torch.float32, 0x7FC0DEAD)
    xd = x.cuda()
    L.check(L.load().anyloc_l2_normalize_rows(L.ptr(xd), rows, D, ld, _dptr(y), L.stream_ptr()), "l2_normalize_rows")
    torch.cuda.synchronize()
    assert _canaries_intact(y, rows * D), (rows, D, ld)
    return y[LEAD:LEAD + rows * D].view(rows, D).cpu()


@pytest.mark.parametrize("D", [4, 36, 128, 384, 516, 1028, 2044, 8192])
def test_l2_normalize_rows(L, D):
    g = torch.Generator().manual_seed(D)
    worst = 0.0
    for rows in MS:
        for ld in (D, D + 4, D + 132):
            x = torch.randn(rows, ld, generator=g) * torch.logspace(-3, 3, rows)[:, None]
            if rows > 2:
                x[1] = 0.0                                     # zero row: 0 / 1e-12 = 0
                x[2, :D] = x[2, :D] / x[2, :D].norm() * 1e-14   # norm 1e-14: divided by 1e-12, not by its norm
            y = _l2(L, x.contiguous(), D, ld)
            x64 = x[:, :D].double()
            ref = x64 / x64.norm(dim=1, keepdim=True).clamp_min(float(np.float32(1e-12)))
            k = math.ceil(D / 128) + 10
            ratio = float(((y.double() - ref).abs() / (U * k * ref.abs()).clamp_min(1e-300)).max())
            worst = max(worst, ratio)
            assert ratio <= C_L2, (D, rows, ld, ratio)
            if rows > 2:
                assert bool((y[1] == 0).all())
                assert float(x64[2].norm()) < 1e-12 and torch.allclose(y[2].double(), x64[2] / float(np.float32(1e-12)),
                                                                        rtol=4 * U, atol=0)
    print(f"l2_normalize_rows D={D}: worst |y - y64| / (u k |y64|) {worst:.3f}")
