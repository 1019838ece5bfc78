"""The streamed k-means fit (host descriptors larger than the device) against the in-memory fit.  The device budget
is monkeypatched so that small inputs take the streamed path, with the staging buffer sized for a chosen piece
length P; centres, labels and the number of Lloyd iterations must equal the in-memory fit's bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from oracle import dinov2_restated as dr
from tests import dropin_harness as H
from tests.util import ROOT

pytestmark = pytest.mark.gpu


class Spy:
    """records the labels each fit returns, the in-memory shifts and the streamed finalize calls"""

    def __init__(self, monkeypatch):
        self.labels, self.shifts, self.finalized = [], [], 0
        fp, fs, upd = u._KMeans.fit_predict, u._KMeans._fit_streamed, u._KMeans._update
        lib = _lib.load()
        fin = lib.anyloc_kmeans_finalize

        def fit_predict(km, *a, **k):
            out = fp(km, *a, **k)
            self.labels.append(out.cpu())
            return out

        def fit_streamed(km, *a, **k):
            out = fs(km, *a, **k)
            self.labels.append(out.cpu())
            return out

        def update(km, x, labels, c):
            new_c, err = upd(km, x, labels, c)
            self.shifts.append((float(err), km.tol))
            return new_c, err

        def finalize(*a):
            self.finalized += 1
            return fin(*a)

        monkeypatch.setattr(u._KMeans, "fit_predict", fit_predict)
        monkeypatch.setattr(u._KMeans, "_fit_streamed", fit_streamed)
        monkeypatch.setattr(u._KMeans, "_update", update)
        monkeypatch.setattr(lib, "anyloc_kmeans_finalize", finalize)

    def in_memory_iterations(self):
        """iterations of the synchronous Lloyd loop (the in-memory fit enqueues one speculative update)"""
        for i, (e, tol) in enumerate(self.shifts):
            if e <= tol:
                return i + 1
        return len(self.shifts)


def force_stream(monkeypatch, X, K, copies, P, budget):
    """make the fit of host rows X stream in rounds of P rows per chunk; -> (plan, number of rounds)"""
    dev = torch.device("cuda", 0)
    R, D = X.shape
    with torch.cuda.device(dev):
        chunks, rows_per = u._kmeans_partition(R, D)
    monkeypatch.setattr(u, "_STAGE_BYTES", min(P, rows_per) * chunks * 4 * D)
    monkeypatch.setattr(u, "_device_budget", lambda dev: budget)
    plan = u._host_fit_plan(torch.as_tensor(X), dev, K, copies)
    assert plan is not None and plan[0] == min(P, rows_per)
    return plan, -(-rows_per // plan[0])


def clustered(R, D, K, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn(K, D, generator=g, dtype=torch.float64)
    x = centres[torch.randint(0, K, (R,), generator=g)] + 0.6 * torch.randn(R, D, generator=g, dtype=torch.float64)
    return x.to(dtype)


def run(fit, monkeypatch, stream=None):
    """-> (centres, labels, iterations) of fit(), in memory or streamed per `stream` = (X, K, copies, P, resident)"""
    with monkeypatch.context() as m:
        spy = Spy(m)
        if stream is not None:
            X, K, copies, P, resident = stream
            R, D = X.shape
            row = 4 * D
            budget = {"zero": 0, "all": copies * R * row - 1, "some": (copies * R * row) // 2}[resident]
            (P_, kept), n_rounds = force_stream(m, X, K, copies, P, budget)
            assert {"zero": kept == 0, "some": 0 < kept < n_rounds, "all": kept == n_rounds}[resident], (kept, n_rounds)
        np.random.seed(1234)
        centres = fit()
        iters = spy.finalized if stream is not None else spy.in_memory_iterations()
        return centres, spy.labels[0], iters          # fit_predict streaming records its labels twice


def check_equal(fit, monkeypatch, stream):
    c0, l0, i0 = run(fit, monkeypatch)
    c1, l1, i1 = run(fit, monkeypatch, stream)
    assert not c1.is_cuda and not l1.is_cuda and l1.dtype == torch.int64
    assert i0 == i1 and i0 > 1
    assert torch.equal(c0.cpu(), c1) and torch.equal(l0, l1)
    return c1


def vlad_fit(X, K, mode="cosine"):
    def fit():
        v = u.VLAD(K, dist_mode=mode)
        v.fit(X)
        return v.c_centers
    return fit


# (R, D, K, P, resident): one chunk (R < 256), a short last chunk, the 64-chunk cap; P = 1, prime, >= rows_per
CASES = [(200, 96, 8, 13, "some"), (200, 96, 8, 1, "all"), (3001, 384, 16, 1, "zero"), (3001, 384, 16, 7, "some"),
         (3001, 384, 16, 13, "all"), (3001, 384, 16, 10**6, "zero"), (40_003, 128, 32, 101, "some"),
         (40_003, 128, 32, 10**6, "zero")]


@pytest.mark.parametrize("R,D,K,P,resident", CASES)
def test_vlad_fit_streamed_equals_in_memory(cuda, monkeypatch, R, D, K, P, resident):
    X = clustered(R, D, K, seed=R + D)
    check_equal(vlad_fit(X, K), monkeypatch, (X, K, 2, P, resident))


@pytest.mark.parametrize("mode", ["cosine", "euclidean"])
@pytest.mark.parametrize("P,resident", [(7, "zero"), (11, "some")])
def test_kmeans_fit_predict_streamed(cuda, monkeypatch, mode, P, resident):
    X = clustered(3001, 384, 16, seed=5)

    def fit():
        km = u._KMeans(16, mode=mode)
        km.fit_predict(X)
        return km.centroids
    check_equal(fit, monkeypatch, (X, 16, 1, P, resident))


def test_vlad_fit_euclidean(cuda, monkeypatch):
    X = clustered(2500, 256, 12, seed=6)
    check_equal(vlad_fit(X, 12, "euclidean"), monkeypatch, (X, 12, 2, 5, "some"))


def test_empty_clusters(cuda, monkeypatch):
    """five distinct rows and eight centres: the random draw repeats rows, and a repeated centre gets no members"""
    X = clustered(5, 128, 5, seed=7).repeat(400, 1)
    c = check_equal(vlad_fit(X, 8), monkeypatch, (X, 8, 2, 3, "some"))
    assert (c.abs().sum(1) == 0).any()


def test_float64_numpy_input(cuda, monkeypatch):
    X = clustered(3001, 384, 16, seed=8, dtype=torch.float64).numpy()
    check_equal(vlad_fit(X, 16), monkeypatch, (X, 16, 2, 7, "some"))


def test_non_contiguous_input(cuda, monkeypatch):
    X = clustered(3001, 2 * 384, 16, seed=9)[:, ::2]
    assert not X.is_contiguous()
    check_equal(vlad_fit(X, 16), monkeypatch, (X, 16, 2, 7, "some"))
    Xt = clustered(3001, 384, 16, seed=10).t().contiguous().t()
    assert not Xt.is_contiguous()
    check_equal(vlad_fit(Xt, 16), monkeypatch, (Xt, 16, 2, 13, "zero"))


def test_device_input_never_streams(cuda, monkeypatch):
    monkeypatch.setattr(u, "_device_budget", lambda dev: 0)
    assert u._host_fit_plan(torch.zeros(1000, 64, device=cuda), cuda, 4, 2) is None
    assert u._host_fit_plan(torch.zeros(1000, 64), cuda, 4, 2) is not None


def test_dropin_replay_streamed(cuda, monkeypatch, tmp_path):
    """tests/test_dropin_gpu.py's driver loop: the vocabulary fitted from host descriptors with streaming forced, and
    the descriptors built with it, equal the unforced run's bit for bit"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_anyloc_shim_utilities_stream",
                                                  os.path.join(ROOT, "anyloc_b200", "dropin", "utilities.py"))
    shim = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(shim)
    ds = H.SyntheticVprDataset()
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=3), seed=3).state_dict()
    dino = shim.DinoV2ExtractFeatures("dinov2_vits14", 2, "value", device=cuda, weights=sd)
    descs = []
    for i in range(ds.database_num):
        img = ds[i][0].to(cuda)
        c, h, w = img.shape
        hn, wn = (h // 14) * 14, (w // 14) * 14
        top, left = int(round((h - hn) / 2.0)), int(round((w - wn) / 2.0))
        descs.append(dino(img[None, :, top:top + hn, left:left + wn]).cpu())
    full_db = torch.cat(descs)
    flat = full_db.reshape(-1, full_db.shape[2])

    def build(name):
        np.random.seed(42)
        vlad = shim.VLAD(4, None, cache_dir=str(tmp_path / name))
        vlad.fit(flat)
        return vlad.c_centers, vlad.generate_multi(full_db)

    c0, v0 = build("memory")
    streamed = []
    with monkeypatch.context() as m:
        fs = u._KMeans._fit_streamed
        m.setattr(u._KMeans, "_fit_streamed", lambda km, *a: streamed.append(a[3]) or fs(km, *a))
        force_stream(m, flat, 4, 2, 7, 0)
        c1, v1 = build("streamed")
    assert streamed and streamed[0][1] == 0
    assert torch.equal(c0, c1) and torch.equal(v0, v1)
