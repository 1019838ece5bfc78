"""Argument checks of the packed attention entry point (anyloc_attention_varlen), without a GPU: every refusal returns
before any CUDA call, so placeholder device pointers are never touched."""
import ctypes as C

from anyloc_b200 import _lib

P = 4096                    # placeholder device address, 16-byte aligned
ARG, UNSUPPORTED = _lib.ERR["arg"], _lib.ERR["unsupported"]


def _call(lib, row0=(0, 70), lens=(65, 130), *, fmt="f16", qkv_hi=P, qkv_lo="fit", o_hi=P, o_lo="fit", D=128,
          heads=2, n=None, host=True):
    """lo pointers "fit" the format unless given: a placeholder for the pair formats, NULL for bf16"""
    n = len(lens) if n is None else n
    arr = lambda v: (C.c_int32 * max(len(v), 1))(*v) if host else None
    fit = None if fmt == "bf16" else P
    qkv_lo, o_lo = (fit if v == "fit" else v for v in (qkv_lo, o_lo))
    return lib.anyloc_attention_varlen(C.c_void_p(qkv_hi), C.c_void_p(qkv_lo), n, arr(row0), arr(lens), D, heads,
                                       C.c_void_p(o_hi), C.c_void_p(o_lo), _lib.PAIR.get(fmt, fmt), None)


def test_null_pointers(lib):
    for fmt in ("tf32", "f16", "bf16"):
        for kw in (dict(qkv_hi=None), dict(o_hi=None), dict(host=False)):
            assert _call(lib, fmt=fmt, **kw) == ARG, (fmt, kw)
    for fmt in ("tf32", "f16"):
        assert _call(lib, fmt=fmt, qkv_lo=None) == ARG and "need qkv_lo and o_lo" in _lib.last_error()
        assert _call(lib, fmt=fmt, o_lo=None) == ARG


def test_lo_arrays_with_single_bf16(lib):
    assert _call(lib, fmt="bf16", qkv_lo=P, o_lo=None) == ARG and "no lo arrays" in _lib.last_error()
    assert _call(lib, fmt="bf16", qkv_lo=None, o_lo=P) == ARG


def test_image_count(lib):
    assert _call(lib, row0=(), lens=()) == ARG and "out of range" in _lib.last_error()
    assert _call(lib, n=-1) == ARG
    many = _lib.VIT_VARLEN_MAX_B + 1
    assert _call(lib, row0=range(0, 2 * many, 2), lens=[1] * many) == ARG and "out of range" in _lib.last_error()


def test_lengths_offsets_and_overlaps(lib):
    for row0, lens in [((0, 70), (0, 130)), ((0, 70), (65, -3)), ((-1, 70), (65, 130)),
                       ((0, 2 ** 31 - 10), (65, 20)),          # the last row past the 32-bit row index
                       ((0, 64), (65, 130)),                   # image 1 starts on image 0's last row
                       ((200, 0), (65, 201)),                  # listed out of row order, image 1 runs into image 0
                       ((0, 300, 10), (5, 5, 400))]:           # image 2 covers image 1
        assert _call(lib, row0=row0, lens=lens) == ARG, (row0, lens)
    assert "overlap" in _lib.last_error()


def test_head_dim_and_format(lib):
    assert _call(lib, D=192) == ARG and "head_dim must be 64" in _lib.last_error()
    assert _call(lib, D=0, heads=0) == ARG
    for fmt in (3, -1):
        assert _call(lib, fmt=fmt) == ARG and "bad fmt" in _lib.last_error()


def test_unaligned_qkv_is_unsupported(lib):
    for kw in (dict(qkv_hi=P + 8), dict(qkv_lo=P + 4)):
        assert _call(lib, **kw) == UNSUPPORTED and "16-byte aligned" in _lib.last_error()
    assert _call(lib, fmt="bf16", qkv_hi=P + 2) == UNSUPPORTED
