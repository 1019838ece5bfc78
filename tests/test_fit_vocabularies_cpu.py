"""fit_vocabularies' host logic without a GPU: its refusals, the workspace and plan arithmetic for V members, and --
over the CPU double, with the shared Lloyd loop replaced by one double fit per member -- the random-choice draws in
member order, cached members and the state every member is left in, against sequential VLAD.fit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u
from tests import dropin_harness as H
from tests.cpu_double import cpu_double


def test_refusals_name_the_members():
    a = u.VLAD(4)
    with pytest.raises(ValueError, match="no VLAD"):
        u.fit_vocabularies([], torch.zeros(10, 8))
    with pytest.raises(ValueError, match=r"members 1 and 3"):
        u.fit_vocabularies([u.VLAD(2), a, u.VLAD(2), a], torch.zeros(10, 8))
    with pytest.raises(ValueError, match=r"members \[1, 2\]"):
        u.fit_vocabularies([a, u.VLAD(4, norm_descs=False), u.VLAD(2, dist_mode="euclidean")], torch.zeros(10, 8))
    assert a.kmeans is None                          # refused before any member is touched


def test_multi_workspace_bytes():
    lib = _lib.load()

    def up(n):
        return -(-n // 256) * 256

    def want(R, D, Ks):
        s = sum(Ks)
        coarse = 0
        if D <= 2048 and R >= 256:
            coarse = up(4 * s * min(R, max(256, (1 << 26) // s // 256 * 256)))
        return 2 * up(4 * s * D) + 2 * up(4 * s) + coarse

    for R, D, Ks in [(10_000, 1536, [32, 64, 128, 256]), (4_000_000, 1536, [32, 64, 128, 256]), (255, 384, [8]),
                     (10_000, 2560, [8, 1]), (1 << 20, 384, [1000, 437]), (256, 1024, [1])]:
        assert lib.anyloc_vlad_assign_multi_workspace_bytes(R, D, len(Ks), (C.c_int * len(Ks))(*Ks)) == want(R, D, Ks)
    # the coarse slice holds at most 2^26 scores (and 256 rows): 4 M rows x sum K = 480 need 7.7 GB unsliced
    big = lib.anyloc_vlad_assign_multi_workspace_bytes(4_000_000, 1536, 4, (C.c_int * 4)(32, 64, 128, 256))
    assert big < (1 << 28) + 8 * 480 * 1536 + 4096


@pytest.mark.parametrize("V", [1, 2, 4])
def test_plan_for_v_members(V):
    R, D, chunks = 10_000, 64, 8
    rows_per, row = -(-R // chunks), 4 * D
    ws = u._fit_ws_bytes(lambda n: 1000 + 8 * n, 5000 * V, V)
    assert ws(100) == 1000 + 800 + 5000 * V + 4 * V * 100            # one label row per member
    need = 2 * R * row + ws(R)
    assert u._kmeans_plan(R, D, chunks, rows_per, need, 2, ws, 1 << 30) is None
    stage = 50 * chunks * row
    rr = 50 * chunks
    fixed = ws(rr) + 4 * R + 3 * rr * row
    plan = u._kmeans_plan(R, D, chunks, rows_per, fixed + 4 * rr * row, 2, ws, stage)
    assert plan == (50, 4)
    assert u._kmeans_plan(R, D, chunks, rows_per, fixed + 4 * rr * row - 1, 2, ws, stage) == (50, 3)


def double_lloyd(kms, x, inits):
    """the shared loop replaced by each member's own (double) fit from its draw"""
    out = []
    for km, i in zip(kms, inits):
        km.fit(x, x[torch.from_numpy(i)])
        out.append(km.centroids)
    return out


def run(tmp_path, arm, specs, X, seed=3, cached=()):
    dirs = [str(tmp_path / arm / f"m{i}") if d else None for i, (K, d) in enumerate(specs)]
    vl = [u.VLAD(K, cache_dir=d) for (K, _), d in zip(specs, dirs)]
    for i in cached:
        torch.save(torch.full((specs[i][0], X.shape[1]), float(i + 1)), os.path.join(dirs[i], "c_centers.pt"))
    np.random.seed(seed)
    if arm == "seq":
        for v in vl:
            v.fit(X)
    else:
        u.fit_vocabularies(vl, X)
    files = [None if d is None else torch.load(os.path.join(d, "c_centers.pt")) for d in dirs]
    return vl, files, np.random.get_state()


@pytest.mark.parametrize("cached", [(), (1,), (0, 2), (0, 1, 2)])
def test_draw_order_and_cached_members(tmp_path, monkeypatch, cached):
    g = torch.Generator().manual_seed(0)
    X = torch.randn(400, 16, generator=g).double().numpy()
    specs = [(3, True), (5, True), (2, True), (4, False)][:3 if len(cached) == 3 else 4]
    monkeypatch.setattr(u, "_lloyd_in_memory", double_lloyd)
    with cpu_double():
        a, fa, ra = run(tmp_path, "seq", specs, X, cached=cached)
        b, fb, rb = run(tmp_path, "multi", specs, X, cached=cached)
    for v, w, x, y in zip(a, b, fa, fb):
        assert torch.equal(v.c_centers, w.c_centers) and torch.equal(v.kmeans.centroids, w.kmeans.centroids)
        assert v.desc_dim == w.desc_dim == 16
        assert (x is None) == (y is None) and (x is None or torch.equal(x, y))
    assert ra[0] == rb[0] and np.array_equal(ra[1], rb[1]) and ra[2:] == rb[2:]
    for i in cached:
        assert (b[i].c_centers == i + 1).all()
    if len(cached) < len(specs):
        assert not np.array_equal(ra[1], np.random.RandomState(3).get_state()[1])        # something was drawn


def test_all_cached_needs_no_rows(tmp_path):
    specs = [(3, True), (2, True)]
    vl = [u.VLAD(K, cache_dir=str(tmp_path / f"m{i}")) for i, (K, _) in enumerate(specs)]
    for i, v in enumerate(vl):
        torch.save(torch.ones(specs[i][0], 8), os.path.join(v.cache_dir, "c_centers.pt"))
    st = np.random.get_state()
    u.fit_vocabularies(vl, None)
    assert all(v.desc_dim == 8 for v in vl) and np.array_equal(np.random.get_state()[1], st[1])


@pytest.mark.skipif(not H.available(), reason="reference tree not present")
def test_unmodified_driver_once_per_k(tmp_path, monkeypatch):
    """the reference's unmodified build_vlads run once per K (RNG running on from one seed, one cache directory per
    K) writes, per K, the c_centers.pt that fit_vocabularies gives from the same seed and database rows"""
    import importlib.util
    from oracle import dinov2_restated as dr
    spec = importlib.util.spec_from_file_location("_anyloc_shim_utilities_fitv_cpu",
                                                  os.path.join(os.path.dirname(u.__file__), "dropin", "utilities.py"))
    shim = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(shim)
    sd = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=3), seed=3).state_dict()
    ds = H.SyntheticVprDataset()
    monkeypatch.setattr(u, "_lloyd_in_memory", double_lloyd)
    Ks = [8, 4, 2]
    seen = []
    fit = u.VLAD.fit
    monkeypatch.setattr(u.VLAD, "fit", lambda self, t: seen.append(t) or fit(self, t))
    with cpu_double(lambda name: sd):
        script = H.load_script(shim)
        np.random.seed(42)
        for K in Ks:
            script.build_vlads(H.make_largs(script, str(tmp_path / f"k{K}"), "dinov2_vits14", 2, "value", K, True),
                               ds, verbose=False)
        np.random.seed(42)
        vl = [u.VLAD(K) for K in Ks]
        u.fit_vocabularies(vl, seen[0])
    for K, v in zip(Ks, vl):
        f = [os.path.join(r, "c_centers.pt") for r, _, fs in os.walk(tmp_path / f"k{K}") if "c_centers.pt" in fs]
        assert len(f) == 1 and torch.equal(torch.load(f[0]), v.c_centers)
