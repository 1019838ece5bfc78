"""The fp64 restatement of the antialiased resize that tests/test_preprocess_engine_gpu.py bounds the kernels against,
pinned without a GPU to torch's own float64 antialiased interpolate (align_corners=False, antialias=True, what
torchvision's tensor resize calls): both compute sum_y w_y sum_x w_x v with the same spans and filters in fp64, so they
agree to rounding, within 1e-12 on O(1) values."""
import numpy as np
import pytest
import torch

from tests.test_preprocess_engine_gpu import axis64, pixels64, resize64

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def torch64(img, Hr, Wr, mode):
    v, _ = pixels64(img, MEAN, STD)
    return torch.nn.functional.interpolate(torch.from_numpy(v)[None], size=(Hr, Wr), mode=mode, align_corners=False,
                                           antialias=True)[0].numpy()


@pytest.mark.parametrize("mode,cubic", [("bilinear", 0), ("bicubic", 1)])
@pytest.mark.parametrize("H,W,Hr,Wr", [(37, 53, 37, 53), (70, 90, 70, 33), (126, 154, 63, 22), (1000, 64, 480, 64),
                                       (30, 40, 111, 148), (1, 1, 14, 14), (60, 868, 30, 28), (60, 434, 30, 28),
                                       (5000, 20, 14, 20), (21, 16384, 7, 1400)])
def test_restatement_is_torch_float64(mode, cubic, H, W, Hr, Wr):
    img = np.random.default_rng(H * W + Hr).integers(0, 256, (H, W, 3), dtype=np.uint8)
    ref = torch64(img, Hr, Wr, mode)
    top, left = (1, 2) if Hr > 2 and Wr > 3 else (0, 0)
    Hc, Wc = Hr - top, Wr - left
    o64, _ = resize64(img, Hr, Wr, cubic, top, left, Hc, Wc, MEAN, STD, with_bound=False)
    assert np.abs(o64 - ref[:, top:, left:]).max() <= 1e-12


def test_checkerboard_restatement():
    """the cancelling case: windows of +/- values"""
    yy, xx = np.mgrid[:211, :307]
    img = np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, axis=2)
    for mode, cubic in (("bilinear", 0), ("bicubic", 1)):
        o64, bound = resize64(img, 100, 140, cubic, 0, 0, 100, 140, MEAN, STD)
        assert np.abs(o64 - torch64(img, 100, 140, mode)).max() <= 1e-12
        assert np.isfinite(bound).all() and (bound >= 2.0 ** -24 * np.abs(o64)).all()


@pytest.mark.parametrize("cubic", [0, 1])
def test_axis_weights(cubic):
    """each row of weights sums to 1; a scale of exactly 1 gives the identity (weights exactly 1 and 0)"""
    for n_in, n_out in ((100, 37), (37, 100), (5000, 14), (16384, 16000)):
        W, E, n, r = axis64(n_in, n_out, cubic, np.arange(n_out))
        assert np.abs(np.asarray(W.sum(axis=1)).ravel() - 1).max() < 1e-12
        assert (n >= 1).all() and (r >= 1).all() and (E.data > 0).all()
    W, _, _, _ = axis64(50, 50, cubic, np.arange(50))
    assert np.array_equal(W.toarray(), np.eye(50))
