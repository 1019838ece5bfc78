"""Alignment checks of the pooling and pre-processing entry points, without a GPU.  anyloc_pool reads the features and
writes the output with float4 accesses, anyloc_preprocess_u8 stores pairs of columns as float2 when Wc is even, and
every pre-processing kernel stores fp32 elements, so a pointer those accesses would fault on is refused before any
CUDA call: the placeholder device pointers here are never touched.  Calls with nothing to do (B = 0, n = 0) and
aligned pointers still return OK without launching."""
import ctypes as C

from anyloc_b200 import _lib

P = 4096                    # placeholder device address, 16-byte aligned
ARG = _lib.ERR["arg"]
AVG, MAX, GEM = 0, 1, 2
M3 = (C.c_float * 3)(0.485, 0.456, 0.406)
S3 = (C.c_float * 3)(0.229, 0.224, 0.225)


def _pool(lib, B=2, N=9, D=36, mode=AVG, feats=P, out=P, n_valid=None, p=3.0):
    return lib.anyloc_pool(C.c_void_p(feats), C.c_void_p(n_valid), B, N, D, mode, C.c_float(p), 0, C.c_void_p(out),
                           None)


def _crop(lib, B=1, Wc=28, out=P):
    return lib.anyloc_preprocess_u8(C.c_void_p(P), B, 56, 57, 0, 0, 28, Wc, M3, S3, C.c_void_p(out), None)


def _resize(lib, B=1, Wc=28, out=P):
    return lib.anyloc_preprocess_resize_u8(C.c_void_p(P), B, 100, 90, 56, 57, 1, 0, 0, 28, Wc, M3, S3,
                                           C.c_void_p(out), None)


def _varlen(lib, n=1, interp=-1, out=P):
    def ints(v):
        return (C.c_int * 1)(v)
    return lib.anyloc_preprocess_u8_varlen(n, (C.c_void_p * 1)(P), ints(56), ints(57), ints(56), ints(57), interp,
                                           ints(0), ints(0), ints(28), ints(27), M3, S3, C.c_void_p(out),
                                           (C.c_int64 * 1)(0), None)


def test_pool_refuses_misaligned_pointers(lib):
    for mode in (AVG, MAX, GEM):
        for B in (0, 2):
            for kw in (dict(feats=P + 4), dict(feats=P + 8), dict(feats=P + 12), dict(feats=P + 1),
                       dict(out=P + 4), dict(out=P + 8), dict(out=P + 12), dict(out=P + 2)):
                assert _pool(lib, B=B, mode=mode, **kw) == ARG, (mode, B, kw)
                assert "16-byte aligned" in _lib.last_error()
        assert _pool(lib, B=0, mode=mode) == 0                  # nothing to do, nothing launched
        assert _pool(lib, B=0, mode=mode, feats=P + 16, out=P + 32, n_valid=P + 4) == 0


def test_pool_other_refusals_unchanged(lib):
    assert _pool(lib, feats=0) == ARG and "null pointer" in _lib.last_error()
    for B, N, D in ((-1, 9, 36), (2, 0, 36), (2, 9, 0), (2, 9, 38), (65536, 1, 4)):
        assert _pool(lib, B=B, N=N, D=D) == ARG, (B, N, D)
    assert _pool(lib, B=0, mode=3) == ARG and "unknown mode" in _lib.last_error()
    assert _pool(lib, B=0, mode=GEM, p=0.0) == ARG and "non-zero" in _lib.last_error()


def test_preprocess_u8_alignment(lib):
    # odd Wc: the kernel stores one float at a time, 4-byte alignment is enough
    for off in (1, 2, 3):
        assert _crop(lib, B=0, Wc=27, out=P + off) == ARG, off
        assert "4-byte aligned" in _lib.last_error()
    assert _crop(lib, B=0, Wc=27, out=P + 4) == 0
    # even Wc: pairs of columns are float2 stores
    for off in (1, 2, 3, 4, 5, 6, 7, 12):
        assert _crop(lib, B=0, Wc=28, out=P + off) == ARG, off
        assert "8-byte aligned when Wc is even" in _lib.last_error()
    assert _crop(lib, B=0, Wc=28, out=P + 8) == 0
    assert _crop(lib, B=3, Wc=28, out=P + 4) == ARG             # refused before the launch, whatever B


def test_preprocess_resize_and_list_alignment(lib):
    for Wc in (27, 28):
        for off in (1, 2, 3):
            assert _resize(lib, B=0, Wc=Wc, out=P + off) == ARG, (Wc, off)
            assert "4-byte aligned" in _lib.last_error()
            assert _resize(lib, B=1, Wc=Wc, out=P + off) == ARG, (Wc, off)
        assert _resize(lib, B=0, Wc=Wc, out=P + 4) == 0         # fp32 stores only
    for interp in (-1, 0, 1):
        for off in (1, 2, 3):
            assert _varlen(lib, n=1, interp=interp, out=P + off) == ARG, (interp, off)
            assert "4-byte aligned" in _lib.last_error()
            assert _varlen(lib, n=0, interp=interp, out=P + off) == ARG, (interp, off)
        assert _varlen(lib, n=0, interp=interp, out=P + 4) == 0
