"""List pre-processing without a GPU: the demo's `max_side` sizing against a verbatim transcription of the demo's
arithmetic, the argument errors `preprocess_images` raises on a list before any device work, the C ABI's refusals
(which return before anything touches the device) and the header's declaration of the new entry."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib
from anyloc_b200 import utilities as u

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARG = _lib.ERR["arg"]
FAKE = 4096                      # placeholder device pointer; every checked error returns before a launch


def demo_size(h, w, max_img_size):
    """demo/anyloc_vlad_generate.py:165-173, transcribed verbatim on a [c, h, w] shape"""
    shape = (3, h, w)
    if max(shape[-2:]) > max_img_size:
        c, h, w = shape
        # Maintain aspect ratio
        if h == max(shape[-2:]):
            w = int(w * max_img_size / h)
            h = max_img_size
        else:
            h = int(h * max_img_size / w)
            w = max_img_size
    return h, w


def test_max_side_size_is_the_demos_rule():
    rng = np.random.default_rng(0)
    sizes = [(int(h), int(w)) for h, w in rng.integers(1, 5000, size=(3000, 2))]
    sizes += [(n, n) for n in (1, 14, 1023, 1024, 1025, 2048, 4096)]                    # h == w
    sizes += [(1024 * a, 1024 * b) for a in (1, 2, 3, 4) for b in (1, 2, 3, 4)]        # exact multiples of the cap
    sizes += [(1025, w) for w in (1, 13, 14, 500, 1024, 1025)] + [(h, 1025) for h in (1, 14, 768, 1024)]
    sizes += [(4032, 3024), (3024, 4032), (1280, 720), (720, 1280), (3000, 4000), (1, 5000), (5000, 1)]
    for cap in (1024, 518, 224, 14):
        for h, w in sizes:
            assert u.max_side_size(h, w, cap) == demo_size(h, w, cap), (h, w, cap)
    assert u.max_side_size(4032, 3024, 1024) == (1024, 768)
    assert u.max_side_size(720, 1280, 1024) == (576, 1024)
    assert u.max_side_size(1024, 1024, 1024) == (1024, 1024)


def test_list_geometry():
    geo = u._list_geometry([(3024, 4032), (700, 500), (1025, 1025)], 14, None, 1024)
    assert geo[0] == (768, 1024, True) + u.center_crop_box(768, 1024)
    assert geo[1] == (700, 500, False) + u.center_crop_box(700, 500)        # under the cap: crop only
    assert geo[2] == (1024, 1024, True, 1, 1, 1022, 1022)
    assert [g[:3] for g in u._list_geometry([(10, 20), (50, 60)], 14, (98, 126), None)] == [(98, 126, True)] * 2
    assert [g[:3] for g in u._list_geometry([(14, 28)], 14, None, None)] == [(14, 28, False)]


def _img(h, w):
    return np.zeros((h, w, 3), np.uint8)


@pytest.mark.parametrize("items,kw,exc", [
    ([], {}, ValueError),                                                              # empty list
    ([_img(20, 20), np.zeros((20, 20, 3), np.float32)], {}, TypeError),                # wrong dtype
    ([_img(20, 20), torch.zeros(20, 20, 3)], {}, TypeError),
    ([_img(20, 20), "photo.jpg"], {}, TypeError),
    ([_img(20, 20), np.zeros((3, 20, 20), np.uint8)], {}, ValueError),                 # wrong shape
    ([_img(20, 20), np.zeros((20, 20), np.uint8)], {}, ValueError),
    ([_img(20, 20), np.zeros((1, 20, 20, 3), np.uint8)], {}, ValueError),
    ([_img(20, 20), _img(0, 20)], {}, ValueError),                                     # empty image
    ([_img(20, 20), _img(20, 0)], {}, ValueError),
    ([_img(20, 20), _img(13, 40)], {}, ValueError),                                    # smaller than a patch
    ([_img(20, 20)], {"resize": (13, 40)}, ValueError),                                # ... after resizing
    ([_img(20, 20), _img(2000, 20)], {"max_side": 1024}, ValueError),                  # 1024 x 10 after the cap
    ([_img(20, 20)], {"resize": (28, 28), "max_side": 1024}, ValueError),              # both sizing rules
    ([_img(20, 20)], {"max_side": 0}, ValueError),
    ([_img(20, 20)], {"interpolation": "nearest"}, ValueError),
])
def test_list_argument_errors_before_device_work(monkeypatch, items, kw, exc):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(_lib, "require_cuda", no_device)
    with pytest.raises(exc):
        u.preprocess_images(items, **kw)
    with pytest.raises(exc):
        u.preprocess_images(tuple(items), **kw)


def _call(n=1, imgs=None, H=(40,), W=(40,), Hr=(28,), Wr=(28,), interp=0, top=(0,), left=(0,), Hc=(28,), Wc=(28,),
          mean=(0.5, 0.5, 0.5), std=(0.25, 0.25, 0.25), out=FAKE, off=(0,)):
    def arr(t, v):
        return None if v is None else (t * len(v))(*v)
    imgs = [FAKE] * n if imgs is None else imgs
    return _lib.load().anyloc_preprocess_u8_varlen(
        n, arr(C.c_void_p, imgs), arr(C.c_int, H), arr(C.c_int, W), arr(C.c_int, Hr), arr(C.c_int, Wr), interp,
        arr(C.c_int, top), arr(C.c_int, left), arr(C.c_int, Hc), arr(C.c_int, Wc), arr(C.c_float, mean),
        arr(C.c_float, std), C.c_void_p(out), arr(C.c_int64, off), None)


def test_abi_refusals(lib):
    assert _call(n=0) == 0                                             # nothing to do
    cases = {
        "null pointer": dict(imgs=[0]),
        "null pointer (out)": dict(out=0),
        "null pointer (Hr)": dict(Hr=None),
        "unknown interpolation": dict(interp=2),
        "outside the resized": dict(top=(1,)),                         # 1 + 28 > 28
        "outside the 40x40": dict(interp=-1, Hc=(41,)),
        "zero std": dict(std=(0.25, 0.0, 0.25)),
        "negative output offset": dict(off=(-1,)),
        "tap window": dict(W=(28 * 32,)),                                # bilinear: 2 * 32 + 2 > 64
        "n=-1": dict(n=-1),
    }
    for what, kw in cases.items():
        assert _call(**kw) == ARG, what
        assert what.split(" (")[0].split("=")[0] in _lib.last_error(), (what, _lib.last_error())
    # the tap window: bilinear up to 31x, bicubic up to 15.5x horizontally; vertical down-scaling is not limited
    assert _call(W=(28 * 31 + 1,), interp=0) == ARG and _call(W=(434 + 1,), interp=1) == ARG
    # an image beyond the first launch's table is checked before the first launch
    n = _lib.PREPROCESS_VARLEN_BATCH + 3
    assert _call(n=n, H=[40] * n, W=[40] * n, Hr=[28] * n, Wr=[28] * n, top=[0] * (n - 1) + [1], left=[0] * n,
                 Hc=[28] * n, Wc=[28] * n, off=[0] * n) == ARG
    assert f"image {n - 1}" in _lib.last_error()


def test_header_declares_the_list_entry():
    with open(os.path.join(ROOT, "include", "anyloc_b200.h")) as f:
        h = f.read()
    assert re.search(r"int anyloc_preprocess_u8_varlen\(int n, const uint8_t\* const\* imgs,", h)
    assert "demo/anyloc_vlad_generate.py:160-185" in h and "dvgl_benchmark/datasets_ws.py:222-239" in h
    m = re.search(r"#define ANYLOC_PREPROCESS_VARLEN_BATCH (\d+)", h)
    assert m and int(m.group(1)) == _lib.PREPROCESS_VARLEN_BATCH
    assert "anyloc_preprocess_u8_varlen" in _lib.EXPORTS
