"""The streamed route of reduce_pca (utilities.py:522-586; scripts/dino_v2_vlad.py:357-369) for databases larger than
the device.  The kernels of csrc/pca.cu element by element against numpy fp64; the route against the in-memory route in
the same process and against the reference's own sklearn calls (oracle restatement).  `_device_budget` and
`_STAGE_BYTES` are monkeypatched so that small inputs take the streamed route in several pieces."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from oracle import anyloc_oracle as ao
from tests.test_pca_gpu import spectrum_data
from tests.util import rel_inf

pytestmark = pytest.mark.gpu

NAN = float("nan")


def vp(t):
    return C.c_void_p(t.data_ptr())


def accumulate(mode, x, mu, out, u_=None):
    """anyloc_pca_accumulate on device tensors; x may be a strided view (unit column stride)"""
    k, ld_u = (u_.shape[1], u_.stride(0)) if u_ is not None else (0, 0)
    rc = _lib.load().anyloc_pca_accumulate(_lib.PCA[mode], vp(x), x.stride(0), x.shape[0], x.shape[1], vp(mu),
                                           vp(u_) if u_ is not None else None, ld_u, k, vp(out), out.stride(0),
                                           _lib.stream_ptr())
    _lib.check(rc, "anyloc_pca_accumulate")


def mirror(a, m):
    _lib.check(_lib.load().anyloc_pca_mirror(vp(a), m, a.stride(0), _lib.stream_ptr()), "anyloc_pca_mirror")


def canvas(rows, cols, dev, pad=3):
    """an fp64 output [rows, cols] of zeros inside a NaN frame: `pad` extra columns per row and extra rows on both
    sides -> (frame, view)"""
    frame = torch.full((rows + 2 * pad, cols + pad), NAN, dtype=torch.float64, device=dev)
    view = frame[pad:pad + rows, :cols]
    view.zero_()
    return frame, view


def check_frame(frame, view_rows, view_cols, pad=3):
    f = frame.cpu().numpy()
    inside = np.zeros(f.shape, bool)
    inside[pad:pad + view_rows, :view_cols] = True
    assert np.isnan(f[~inside]).all(), "a write landed outside the output"
    assert not np.isnan(f[inside]).any()


def rows_data(n, d, seed):
    g = np.random.default_rng(seed)
    x = (g.standard_normal((n, d)) + 2.0 + g.standard_normal(d)).astype(np.float32)     # non-zero mean
    mu = x.astype(np.float64).mean(0)
    return x, mu


SHAPES = [(1, 7), (7, 1), (7, 129), (129, 1000), (1000, 129), (197, 3 * 64 + 5), (64, 64)]


@pytest.mark.parametrize("n,d", SHAPES)
@pytest.mark.parametrize("mode", ["cov", "gram", "vt"])
def test_accumulate_matches_fp64(cuda, mode, n, d):
    x, mu = rows_data(n, d, seed=n * 7 + d)
    xc = x.astype(np.float64) - mu
    # x read through a strided view: rows 5 floats longer than d
    xs = torch.full((n, d + 5), NAN, device=cuda)
    xs[:, :d] = torch.from_numpy(x).to(cuda)
    xv, mud = xs[:, :d], torch.from_numpy(mu).to(cuda)
    if mode == "vt":
        k = min(n, 37)
        uu = np.random.default_rng(1).standard_normal((n, k + 2))
        ud = torch.from_numpy(uu).to(cuda)[:, :k]          # ld_u = k + 2
        ref = uu[:, :k].T @ xc
        frame, out = canvas(k, d, cuda)
        accumulate("vt", xv, mud, out, ud)
        torch.cuda.synchronize()
        check_frame(frame, k, d)
    else:
        ref = xc.T @ xc if mode == "cov" else xc @ xc.T
        m = ref.shape[0]
        frame, out = canvas(m, m, cuda)
        accumulate(mode, xv, mud, out)
        mirror(out, m)
        torch.cuda.synchronize()
        check_frame(frame, m, m)
        o = out.cpu().numpy()
        assert np.array_equal(o, o.T), "not exactly symmetric after the mirror"
    assert rel_inf(out.cpu().numpy(), ref) < 1e-12


@pytest.mark.parametrize("mode,n,d,cuts", [("cov", 1000, 197, [0, 1, 300, 301, 999, 1000]),
                                           ("cov", 129, 64, [0, 64, 129]),
                                           ("gram", 197, 1000, [0, 5, 512, 1000]),
                                           ("gram", 64, 129, [0, 1, 2, 129])])
def test_pieces_equal_one_piece(cuda, mode, n, d, cuts):
    x, mu = rows_data(n, d, seed=3)
    xd, mud = torch.from_numpy(x).to(cuda), torch.from_numpy(mu).to(cuda)
    m = d if mode == "cov" else n
    whole = torch.zeros(m, m, dtype=torch.float64, device=cuda)
    accumulate(mode, xd, mud, whole)
    parts = torch.zeros_like(whole)
    for a, b in zip(cuts[:-1], cuts[1:]):
        if mode == "cov":
            accumulate(mode, xd[a:b], mud, parts)
        else:
            accumulate(mode, xd[:, a:b], mud[a:b], parts)
    mirror(whole, m)
    mirror(parts, m)
    assert rel_inf(parts, whole) < 1e-12
    again = torch.zeros_like(whole)              # a fixed piece size gives the same bits on every run
    for a, b in zip(cuts[:-1], cuts[1:]):
        accumulate(mode, xd[a:b] if mode == "cov" else xd[:, a:b], mud if mode == "cov" else mud[a:b], again)
    mirror(again, m)
    assert torch.equal(again, parts)


@pytest.mark.parametrize("n,d", [(1, 7), (129, 1000), (5000, 33), (100_000, 3)])
def test_colsum(cuda, n, d):
    lib = _lib.load()
    x, _ = rows_data(n, d, seed=5)
    xd = torch.from_numpy(x).to(cuda)
    frame = torch.full((d + 4,), NAN, dtype=torch.float64, device=cuda)
    s = frame[2:2 + d]
    s.fill_(1.5)                                 # the sum is added to what is there
    ws = torch.empty(lib.anyloc_pca_colsum_workspace_bytes(n, d), dtype=torch.uint8, device=cuda)
    _lib.check(lib.anyloc_pca_colsum(vp(xd), d, n, d, vp(s), vp(ws), ws.numel(), _lib.stream_ptr()), "colsum")
    f = frame.cpu().numpy()
    assert np.isnan(f[:2]).all() and np.isnan(f[2 + d:]).all()
    assert rel_inf(s.cpu().numpy(), x.astype(np.float64).sum(0) + 1.5) < 1e-13
    rc = lib.anyloc_pca_colsum(vp(xd), d, n, d, vp(s), vp(ws), ws.numel() - 1, _lib.stream_ptr())
    assert rc == _lib.ERR["workspace"]


def test_abi_refusals(cuda):
    lib = _lib.load()
    x = torch.zeros(8, 8, device=cuda)
    mu = torch.zeros(8, dtype=torch.float64, device=cuda)
    out = torch.full((8, 8), NAN, dtype=torch.float64, device=cuda)
    st = _lib.stream_ptr()
    assert lib.anyloc_pca_accumulate(7, vp(x), 8, 8, 8, vp(mu), None, 0, 0, vp(out), 8, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(0, vp(x), 7, 8, 8, vp(mu), None, 0, 0, vp(out), 8, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(0, vp(x), 8, 8, 8, None, None, 0, 0, vp(out), 8, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(0, vp(x), 8, 8, 8, vp(mu), None, 0, 0, vp(out), 7, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_accumulate(2, vp(x), 8, 8, 8, vp(mu), None, 0, 4, vp(out), 8, st) == _lib.ERR["arg"]
    assert lib.anyloc_pca_mirror(vp(out), 8, 7, st) == _lib.ERR["arg"]
    torch.cuda.synchronize()
    assert torch.isnan(out).all()                # a refusal writes nothing


# ------------------------------------------------------------------ the route
class Forced:
    """reduce_pca forced onto the streamed route: the budget is exactly the m x m matrix and its eigh of the first fit,
    the staging buffers hold `stage_rows` rows of the first fit (column slabs: stage_rows columns); counts the fits"""

    def __init__(self, monkeypatch, n_fit, d, stage_rows):
        m = min(n_fit, d)
        monkeypatch.setattr(u, "_device_budget", lambda dev, release_cache=True: 8 * u._PCA_EIGH_MATRICES * m * m)
        monkeypatch.setattr(u, "_STAGE_BYTES", 4 * stage_rows * (d if n_fit > d else n_fit))
        self.fits = 0
        real = u._PcaDev.fit_streamed

        def counted(pca, *a):
            self.fits += 1
            return real(pca, *a)
        monkeypatch.setattr(u._PcaDev, "fit_streamed", counted)


def compare(o, r, tol=1e-4):
    assert rel_inf(o, r) < tol
    nrm = lambda x: x / np.linalg.norm(x, axis=-1, keepdims=True)
    assert rel_inf(nrm(np.asarray(o)), nrm(np.asarray(r))) < tol


# rank-48 spectra, so k <= 48 keeps every component determined by the data; k = 48 = min(n, d) on the last
@pytest.mark.parametrize("n,d,k,whiten,stage", [(600, 4096, 48, False, 1000), (600, 4096, 32, True, 700),
                                                (5000, 768, 40, True, 1300), (5000, 768, 48, False, 5000),
                                                (500, 48, 48, False, 64)])
def test_streamed_route(cuda, monkeypatch, n, d, k, whiten, stage):
    tr, te = spectrum_data(n, d, min(n, d, 48), 0.88, seed=n + d)
    r_tr, r_te = ao.reduce_pca(tr, te, k, whitening=whiten)
    m_tr, m_te = u.reduce_pca(tr, te, k, whitening=whiten)                  # in memory
    with monkeypatch.context() as mp:
        f = Forced(mp, n, d, stage)
        o_tr, o_te = u.reduce_pca(tr, te, k, whitening=whiten)
        assert f.fits == 1
        a_tr, a_te = u.reduce_pca(tr, te, k, whitening=whiten)
    assert type(o_tr) == np.ndarray and o_tr.dtype == np.float32 and o_tr.shape == (n, k) and o_te.shape == (37, k)
    assert np.array_equal(a_tr, o_tr) and np.array_equal(a_te, o_te)          # bit-identical on a second run
    for o, r, mem in ((o_tr, r_tr, m_tr), (o_te, r_te, m_te)):
        compare(o, r)
        compare(o, mem)


@pytest.mark.parametrize("n,d,lower,low,fallback", [(400, 40, 10, 0.3, 256), (120, 512, 10, 0.3, 32)])
def test_streamed_low_factor(cuda, monkeypatch, n, d, lower, low, fallback):
    tr, te = spectrum_data(n, d, min(n, d, 48), 0.88 if n < d else 0.9, seed=9 + n)
    r_tr, r_te = ao.reduce_pca(tr, te, lower, low_factor=low, fallback=fallback)
    m_tr, m_te = u.reduce_pca(tr, te, lower, low_factor=low, fallback=fallback)
    with monkeypatch.context() as mp:
        f = Forced(mp, n + 37 if n < d else n, d, 50)
        o_tr, o_te = u.reduce_pca(tr, te, lower, low_factor=low, fallback=fallback)
        assert f.fits >= 1
    assert o_tr.shape == r_tr.shape == (n, lower)
    for o, r, mem in ((o_tr, r_tr, m_tr), (o_te, r_te, m_te)):
        assert rel_inf(o, r) < 1e-4 and rel_inf(o, mem) < 1e-4


@pytest.mark.parametrize("kind", ["f64", "noncontig", "torch_cpu", "torch_cuda", "torch_cuda_noncontig"])
@pytest.mark.parametrize("n,d", [(600, 1024), (3000, 256)])
def test_streamed_inputs(cuda, monkeypatch, kind, n, d):
    tr, te = spectrum_data(n, d, 48, 0.88, seed=4)
    r_tr, r_te = ao.reduce_pca(tr, te, 16)
    if kind == "f64":
        a, b = tr.astype(np.float64), te.astype(np.float64)
    elif kind == "noncontig":
        a, b = np.zeros((n, d + 3), np.float32), np.zeros((37, d + 3), np.float32)
        a[:, 1:d + 1], b[:, 1:d + 1] = tr, te
        a, b = a[:, 1:d + 1], b[:, 1:d + 1]
    elif kind == "torch_cpu":
        a, b = torch.from_numpy(tr), torch.from_numpy(te)
    elif kind == "torch_cuda":
        a, b = torch.from_numpy(tr).to(cuda), torch.from_numpy(te).to(cuda)
    else:
        a, b = torch.zeros(n, d + 3, device=cuda), torch.zeros(37, d + 3, device=cuda)
        a[:, :d], b[:, :d] = torch.from_numpy(tr), torch.from_numpy(te)
        a, b = a[:, :d], b[:, :d]
    m_tr, m_te = u.reduce_pca(a, b, 16)
    with monkeypatch.context() as mp:
        f = Forced(mp, n, d, 200)
        o_tr, o_te = u.reduce_pca(a, b, 16)
        assert f.fits == 1
    assert type(o_tr) == type(m_tr) and type(o_te) == type(m_te)
    if isinstance(o_tr, torch.Tensor):
        assert not o_tr.is_cuda and o_tr.dtype == torch.float32
        o_tr, o_te = o_tr.numpy(), o_te.numpy()
        m_tr, m_te = m_tr.numpy(), m_te.numpy()
    for o, r, mem in ((o_tr, r_tr, m_tr), (o_te, r_te, m_te)):
        compare(o, r)
        compare(o, mem)


def test_streamed_k_too_large_and_memory_error(cuda, monkeypatch):
    tr, te = spectrum_data(300, 96, 48, 0.9, seed=2)
    with monkeypatch.context() as mp:
        Forced(mp, 300, 96, 100)
        with pytest.raises(ValueError):
            u.reduce_pca(tr, te, 97)
        mp.setattr(u, "_device_budget", lambda dev, release_cache=True: 48 * 96 * 96 - 1)
        with pytest.raises(MemoryError, match="96 x 96"):
            u.reduce_pca(tr, te, 8)


def test_vlad_dimension(cuda, monkeypatch):
    """3000 x 49 152 (ViT-G/14 VLADs, K = 32), streamed (Gram route) and in memory"""
    n, d = 3000, 49_152
    tr, te = spectrum_data(n, d, 48, 0.88, seed=11)
    m_tr, m_te = u.reduce_pca(tr, te, 32, whitening=True)
    with monkeypatch.context() as mp:
        mp.setattr(u, "_device_budget", lambda dev, release_cache=True: u._pca_in_memory_bytes(n, d, 37) - 1)
        mp.setattr(u, "_STAGE_BYTES", 4 * n * 8192)                        # six column slabs
        o_tr, o_te = u.reduce_pca(tr, te, 32, whitening=True)
    compare(o_tr, m_tr)
    compare(o_te, m_te)
