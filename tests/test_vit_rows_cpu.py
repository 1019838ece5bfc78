"""Argument checks of the row kernels' entry points (anyloc_layernorm_split, anyloc_l2_normalize_rows), without a GPU:
both read and write with float4-wide accesses, so a bad size or a misaligned pointer is refused before any CUDA call
and the placeholder device pointers here are never touched."""
import ctypes as C

from anyloc_b200 import _lib

P = 4096                    # placeholder device address, 16-byte aligned
ARG = _lib.ERR["arg"]
EPS = C.c_float(1e-6)


def _ln(lib, fmt="tf32", M=8, D=384, x=P, w=P, b=P, y_hi=P, y_lo="fit"):
    y_lo = (None if fmt == "bf16" else P) if y_lo == "fit" else y_lo
    return lib.anyloc_layernorm_split(C.c_void_p(x), C.c_void_p(w), C.c_void_p(b), M, D, EPS, C.c_void_p(y_hi),
                                      C.c_void_p(y_lo), _lib.PAIR[fmt], None)


def _l2(lib, rows=8, D=384, ld_in=384, x=P, y=P):
    return lib.anyloc_l2_normalize_rows(C.c_void_p(x), rows, D, ld_in, C.c_void_p(y), None)


def test_layernorm_sizes(lib):
    for fmt in ("tf32", "f16", "bf16", "fp8"):
        for M, D in ((-1, 384), (-(2 ** 31), 384), (8, 0), (8, -4), (8, 386), (8, 2052), (0, 0), (0, 4096)):
            assert _ln(lib, fmt, M=M, D=D) == ARG, (fmt, M, D)
        assert "D a multiple of 4" in _lib.last_error()
        assert _ln(lib, fmt, M=0) == 0                 # nothing to do, nothing launched


def test_layernorm_alignment(lib):
    for fmt in ("tf32", "f16", "bf16", "fp8"):
        for kw in (dict(x=P + 4), dict(x=P + 8), dict(w=P + 4), dict(b=P + 12)):
            assert _ln(lib, fmt, M=0, **kw) == ARG, (fmt, kw)
            assert "16-byte aligned" in _lib.last_error()
    # the outputs are stored 4 elements at a time: 16 bytes (tf32 pairs), 8 (fp16 pairs, bf16), 4 (e4m3)
    for fmt, step in (("tf32", 16), ("f16", 8), ("bf16", 8), ("fp8", 4)):
        for off in range(1, step):
            assert _ln(lib, fmt, M=0, y_hi=P + off) == ARG, (fmt, off)
        assert _ln(lib, fmt, M=0, y_hi=P + step) == 0, fmt
    for fmt, step in (("tf32", 16), ("f16", 8), ("fp8", 4)):       # fp8: y_lo holds the fp32 row scales
        for off in range(1, step):
            assert _ln(lib, fmt, M=0, y_lo=P + off) == ARG, (fmt, off)
        assert _ln(lib, fmt, M=0, y_lo=P + step) == 0, fmt


def test_layernorm_null_pointers(lib):
    for fmt in ("tf32", "f16", "fp8"):
        for kw in (dict(x=None), dict(w=None), dict(b=None), dict(y_hi=None), dict(y_lo=None)):
            assert _ln(lib, fmt, **kw) == ARG, (fmt, kw)
    assert _ln(lib, "bf16", y_lo=P) == ARG and "no lo array" in _lib.last_error()


def test_l2_normalize_sizes(lib):
    for rows, D, ld in ((-1, 384, 384), (8, 0, 0), (8, -4, 384), (8, 386, 388), (8, 384, 382), (8, 384, 380),
                        (0, 0, 0), (0, 384, 256)):
        assert _l2(lib, rows, D, ld) == ARG, (rows, D, ld)
    assert _l2(lib, 0) == 0 and _l2(lib, 0, 4, 8) == 0      # nothing to do, nothing launched


def test_l2_normalize_alignment_and_nulls(lib):
    for kw in (dict(x=P + 4), dict(x=P + 8), dict(y=P + 4), dict(y=P + 12)):
        assert _l2(lib, 0, **kw) == ARG, kw
        assert "16-byte aligned" in _lib.last_error()
    assert _l2(lib, x=None) == ARG and _l2(lib, y=None) == ARG
