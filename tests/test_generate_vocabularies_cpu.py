"""generate_vocabularies' host logic without a GPU: its refusals (raised before any device work), the chunk plan and
the workspace arithmetic, where a chunk is cut so that each member keeps the assignment route of its own
generate_multi calls, and the refusals of the new C entries (null pointers, dimensions, alignment), in the style of
test_abi_alignment_cpu.py: placeholder device addresses that are never touched."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib, utilities as u

P = 4096                    # placeholder device address, 16-byte aligned
ARG, OK = _lib.ERR["arg"], 0
D_, K_ = 8, 4


def _fitted(K, D, **kw):
    v = u.VLAD(K, **kw)
    v.kmeans = u._KMeans(K, mode=v.mode)
    v.kmeans.centroids = v.c_centers = torch.randn(K, D)
    return v


def test_refusals_before_any_device_work():
    a = _fitted(4, 8)
    x = torch.zeros(2, 3, 8)
    with pytest.raises(ValueError, match="no VLAD"):
        u.generate_vocabularies([], x)
    with pytest.raises(ValueError, match=r"members 1 and 3"):
        u.generate_vocabularies([_fitted(2, 8), a, _fitted(2, 8), a], x)
    with pytest.raises(ValueError, match=r"members \[1, 2\]"):
        u.generate_vocabularies([a, _fitted(4, 8, norm_descs=False), _fitted(2, 8, dist_mode="euclidean")], x)
    with pytest.raises(ValueError, match=r"do not match K=4, D=12"):
        u.generate_vocabularies([_fitted(2, 12), a], torch.zeros(2, 3, 12))
    with pytest.raises(ValueError, match=r"do not match K=4, D=12"):
        u.generate_vocabularies([a], [torch.zeros(3, 12), torch.zeros(1, 12)])
    with pytest.raises(ValueError, match=r"do not match"):
        u.generate_vocabularies([a], np.zeros((2, 3, 12), np.float32))
    # members may mix hard and soft, temperatures and intra_norm; they are only refused for what they share
    with pytest.raises(ValueError, match=r"members \[1\]"):
        u.generate_vocabularies([_fitted(2, 8, vlad_mode="soft", soft_temp=3.0, intra_norm=False),
                                 _fitted(2, 8, dist_mode="euclidean")], x)


def test_unfitted_member_fails_as_generate_multi_does():
    with pytest.raises(AssertionError):
        u.generate_vocabularies([_fitted(2, 8), u.VLAD(3)], torch.zeros(2, 3, 8))
    with pytest.raises(AssertionError):
        u.VLAD(3)._run(torch.zeros(1, 3, 8), None, None)


def test_empty_list_fails_as_generate_multi_does():
    with pytest.raises(RuntimeError):
        u.generate_vocabularies([_fitted(2, 8)], [])
    with pytest.raises(RuntimeError):
        _fitted(2, 8).generate_multi([])


def test_call_images_follow_generate_multi():
    v, w = _fitted(2, 8), _fitted(2, 8)
    w._host_chunk_bytes = 3 * 5 * 8 * 4 + 7           # room for three images of [5, 8]
    X = torch.zeros(10, 5, 8)
    assert u._generate_call_images(v, X, True) == 10  # under the 1 GB chunk: one call
    assert u._generate_call_images(w, X, True) == 3
    assert u._generate_call_images(w, X, False) == 10  # device / numpy input: one call
    assert u._generate_call_images(w, torch.zeros(0, 5, 8), True) == 1


def test_pieces_keep_each_members_call():
    N = 7
    # member 0 calls generate on images 0..9 at once, member 1 in calls of 3: [0,3) [3,6) [6,9) [9,10)
    steps = [(10, 10), (3, 10)]
    assert u._generate_pieces(0, 10, steps, N) == [(0, 3, [70, 21]), (3, 6, [70, 21]), (6, 9, [70, 21]),
                                                    (9, 10, [70, 7])]
    # a chunk that starts inside a call keeps that call's row count
    assert u._generate_pieces(4, 8, steps, N) == [(4, 6, [70, 21]), (6, 8, [70, 21])]
    assert u._generate_pieces(0, 4, [(4, 4)], N) == [(0, 4, [28])]


def test_chunk_bytes_and_plan():
    lib = _lib.load()
    N, D = 529, 1536
    hard, soft = [32, 64, 256], [128]

    def want(b, staged):
        R = b * N
        Kh = (C.c_int * 3)(*hard)
        Ks = (C.c_int * 1)(*soft)
        acc = max([lib.anyloc_vlad_accumulate_workspace_bytes(b, N, D, K, 0) for K in hard] +
                  [lib.anyloc_vlad_accumulate_workspace_bytes(b, N, D, K, 1) for K in soft])
        return (4 * b * D * 480 + (8 * R * D if staged else 0) + lib.anyloc_vlad_label_multi_workspace_bytes(R, D, 3, Kh)
                + 4 * R * 4 + lib.anyloc_vlad_soft_assign_multi_workspace_bytes(D, 1, Ks) + 4 * R * 129 + acc)

    for b in (1, 2, 17, 400):
        for staged in (False, True):
            assert u._generate_chunk_bytes(b, N, D, hard, soft, staged) == want(b, staged)
    # the plan takes the most images that fit, capped
    budget = want(17, True)
    assert u._generate_plan(1000, N, D, hard, soft, True, budget, 65535) == 17
    assert u._generate_plan(1000, N, D, hard, soft, True, budget - 1, 65535) == 16
    assert u._generate_plan(1000, N, D, hard, soft, True, budget, 5) == 5
    assert u._generate_plan(3, N, D, hard, soft, True, budget, 65535) == 3
    with pytest.raises(MemoryError, match=r"one image of 529 x 1536 features needs %d bytes" % want(1, True)):
        u._generate_plan(1000, N, D, hard, soft, True, want(1, True) - 1, 65535)
    # hard or soft members alone
    assert u._generate_chunk_bytes(2, N, D, [], [64], False) < u._generate_chunk_bytes(2, N, D, [64], [64], False)
    assert u._generate_chunk_bytes(2, N, D, [64], [], False) > 0


def test_workspace_bytes():
    lib = _lib.load()

    def up(n):
        return -(-n // 256) * 256

    for R, D, Ks in [(10_000, 1536, [32, 64, 128, 256]), (100, 384, [8]), (255, 1024, [3, 5]), (10_000, 2560, [8, 1])]:
        s = sum(Ks)
        coarse = up(4 * s * min(R, max(256, (1 << 26) // s // 256 * 256))) if D <= 2048 else 0
        arr = (C.c_int * len(Ks))(*Ks)
        # the coarse slice is there for R < 256 too: a member's own call may have 256 rows or more
        assert lib.anyloc_vlad_label_multi_workspace_bytes(R, D, len(Ks), arr) == \
            2 * up(4 * s * D) + 2 * up(4 * s) + coarse
        assert lib.anyloc_vlad_soft_assign_multi_workspace_bytes(D, len(Ks), arr) == up(4 * s * D)
    assert lib.anyloc_vlad_label_multi_workspace_bytes(10, 64, 2, (C.c_int * 2)(4, 0)) == 0
    assert lib.anyloc_vlad_soft_assign_multi_workspace_bytes(64, 0, (C.c_int * 1)(4)) == 0
    # the accumulation: sums of squares [B,K,slices], the tickets on accumulate3, the tables on the sorted route
    for B, N, D, K in [(3, 100, 384, 32), (2, 3942, 1536, 256), (4, 529, 1536, 300), (0, 9, 8, 4)]:
        route = lib.anyloc_vlad_generate_route(B, N, D, K)
        got = lib.anyloc_vlad_accumulate_workspace_bytes(B, N, D, K, 0)
        part = up(4 * B * K * -(-D // 128))
        assert lib.anyloc_vlad_accumulate_workspace_bytes(B, N, D, K, 1) == part      # soft: the sums of squares alone
        if route == 0:
            assert got == part + up(4 * B)
        elif route == 1:
            assert got == part
        else:
            assert got > part + up(8 * B * N)
            # never more than the sorted generate's (which also holds labels, 1/|x| and the assignment buffers)
            assert got < lib.anyloc_vlad_sorted_workspace_bytes(B, N, D, K)
    assert lib.anyloc_vlad_generate_route(2, 3942, 1536, 256) == _lib.VLAD_ROUTE_SORTED


# ------------------------------------------------------------------------------------------------------------------
# The new entries' refusals.  Every call below does no device work even without the checks (nothing to do: R = 0,
# B = 0), so a refused pointer is refused by the check alone.
ALIGN = {
    "anyloc_vlad_label_multi": {"feats": 16, "n_valid": 4, "centers[0]": 4, "centers[1]": 4, "prepared[0]": 16,
                                "prepared[1]": 16, "labels": 4, "inv_norm": 4, "ws": 16},
    "anyloc_vlad_soft_assign_multi": {"feats": 16, "n_valid": 4, "centers[0]": 4, "centers[1]": 4, "assign[0]": 4,
                                      "assign[1]": 4, "inv_norm": 4, "ws": 16},
    "anyloc_vlad_accumulate": {"feats": 16, "n_valid": 4, "labels": 4, "assign": 4, "inv_norm": 4, "centers": 16,
                               "vlad": 16, "ws": 16},
    "anyloc_vlad_accumulate_varlen": {"feats": 16, "row0": 8, "len": 4, "labels": 4, "assign": 4, "inv_norm": 4,
                                      "centers": 16, "vlad": 16, "ws": 16},
}
HOST_ONLY = {"K", "ws_bytes", "stream", "route_rows", "prepared_bytes", "soft_temp"}


def _vp(*xs):
    return (C.c_void_p * len(xs))(*xs)


def _label_multi(lib, p, R=0, N=3, D=D_, Ks=(K_, 3), route=None, null=()):
    V = len(Ks)
    return lib.anyloc_vlad_label_multi(
        None if "feats" in null else p["feats"], p["n_valid"], N, R,
        None if route is None else (C.c_int64 * V)(*route), D, V,
        _vp(p["centers[0]"], p["centers[1]"]), _vp(p["prepared[0]"], p["prepared[1]"]), (C.c_size_t * V)(1 << 20, 1 << 20),
        (C.c_int * V)(*Ks), 0, None if "labels" in null else p["labels"], None if "inv_norm" in null else p["inv_norm"],
        p["ws"], 1 << 20, None)


def _soft_multi(lib, p, R=0, N=3, D=D_, Ks=(K_, 3), null=()):
    V = len(Ks)
    return lib.anyloc_vlad_soft_assign_multi(
        None if "feats" in null else p["feats"], p["n_valid"], N, R, D, V, _vp(p["centers[0]"], p["centers[1]"]),
        (C.c_int * V)(*Ks), (C.c_float * V)(1.0, 0.5), _vp(p["assign[0]"], p["assign[1]"]),
        None if "inv_norm" in null else p["inv_norm"], p["ws"], 1 << 20, None)


def _accumulate(lib, p, B=0, N=9, D=D_, K=K_, soft=False, null=()):
    return lib.anyloc_vlad_accumulate(
        None if "feats" in null else p["feats"], p["n_valid"], None if soft else p["labels"],
        p["assign"] if soft else None, None if "inv_norm" in null else p["inv_norm"], p["centers"], B, N, D, K, 1, 1,
        p["vlad"], p["ws"], 1 << 20, None)


def _accumulate_varlen(lib, p, B=0, R=9, D=D_, K=K_, soft=False, null=()):
    return lib.anyloc_vlad_accumulate_varlen(
        None if "feats" in null else p["feats"], R, p["row0"], p["len"], B, None if soft else p["labels"],
        p["assign"] if soft else None, None if "inv_norm" in null else p["inv_norm"], p["centers"], D, K, 1, 1,
        p["vlad"], p["ws"], 1 << 20, None)


def _calls(lib):
    # hard unless the case is the soft weights' pointer
    return {
        "anyloc_vlad_label_multi": lambda p: _label_multi(lib, p),
        "anyloc_vlad_soft_assign_multi": lambda p: _soft_multi(lib, p),
        "anyloc_vlad_accumulate": lambda p: _accumulate(lib, p, soft=p["assign"] != P),
        "anyloc_vlad_accumulate_varlen": lambda p: _accumulate_varlen(lib, p, soft=p["assign"] != P),
    }


def below(a):
    return {4: (1, 2), 8: (1, 2, 4), 16: (1, 2, 4, 8, 12)}[a]


CASES = [(e, n) for e, ptrs in ALIGN.items() for n in ptrs]


def _msg(entry, name, a):
    m = re.match(r"(\w+)\[(\d)\]", name)
    if m:   # the host arrays' entries are named with their index
        return f"{m.group(1)}[{m.group(2)}] must be {a}-byte aligned"
    return f"{name} must be {a}-byte aligned"


@pytest.mark.parametrize("entry,name", CASES, ids=[f"{e[7:]}-{n}" for e, n in CASES])
def test_entry_refuses_pointer_below_its_alignment(lib, entry, name):
    call = _calls(lib)[entry]
    ptrs = {n: P for n in ALIGN[entry]}
    a = ALIGN[entry][name]
    for off in below(a):
        rc = call(dict(ptrs, **{name: P + off}))
        assert rc == ARG, (entry, name, off, rc, _lib.last_error())
        assert _msg(entry, name, a) in _lib.last_error(), (entry, name, off, _lib.last_error())
    for off in (a, 2 * a, 3 * a):
        assert call(dict(ptrs, **{name: P + off})) == OK, (entry, name, off, _lib.last_error())


def test_table_covers_every_pointer_argument_of_the_new_entries():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "anyloc_b200.h")).read()
    for entry, ptrs in ALIGN.items():
        m = re.search(r"^int " + entry + r"\(([^)]*)\)", src, re.M)
        assert m, entry
        names = {re.sub(r"\W", "", arg.split("*")[-1]) for arg in m.group(1).split(",") if "*" in arg}
        assert names - HOST_ONLY == {re.sub(r"\[\d+\]", "", n) for n in ptrs}, entry


def test_null_and_dimension_refusals(lib):
    p = {n: P for e in ALIGN.values() for n in e}
    for null in ("feats", "labels", "inv_norm"):
        assert _label_multi(lib, p, null=(null,)) == ARG and "null pointer" in _lib.last_error()
    for null in ("feats", "inv_norm"):
        assert _soft_multi(lib, p, null=(null,)) == ARG and "null pointer" in _lib.last_error()
        assert _accumulate(lib, p, null=(null,)) == ARG and "null pointer" in _lib.last_error()
        assert _accumulate_varlen(lib, p, null=(null,)) == ARG and "null pointer" in _lib.last_error()
    assert _label_multi(lib, dict(p, **{"centers[1]": 0})) == ARG and "no centres" in _lib.last_error()
    assert _soft_multi(lib, dict(p, **{"assign[1]": 0})) == ARG and "no assignment" in _lib.last_error()
    # dimensions: D a multiple of 4, R < 2^31, a padded R a multiple of N, K > 0 (soft: <= 2048)
    for kw in (dict(D=6), dict(R=1 << 31), dict(R=7, N=3), dict(N=0, R=3), dict(Ks=(4, 0))):
        assert _label_multi(lib, p, **kw) == ARG, kw
        assert _soft_multi(lib, p, **kw) == ARG, kw
    assert _label_multi(lib, p, route=(256, -1)) == ARG and "route_rows[1]" in _lib.last_error()
    assert _label_multi(lib, p, route=(0, 256)) == OK
    assert _soft_multi(lib, p, Ks=(2049, 3)) == ARG and "1..2048" in _lib.last_error()
    assert _soft_multi(lib, p, Ks=(2048, 3)) == OK
    assert _label_multi(lib, p, Ks=(5000, 3)) == OK                 # hard members take any K
    assert _label_multi(lib, dict(p, n_valid=0), N=0) == OK          # N only counts with n_valid
    # labels XOR assign
    assert lib.anyloc_vlad_accumulate(P, None, P, P, P, P, 0, 9, D_, K_, 1, 1, P, P, 1 << 20, None) == ARG
    assert "labels (hard) OR assign (soft)" in _lib.last_error()
    assert lib.anyloc_vlad_accumulate(P, None, None, None, P, P, 0, 9, D_, K_, 1, 1, P, P, 1 << 20, None) == ARG
    assert lib.anyloc_vlad_accumulate_varlen(P, 9, P, P, 0, P, P, P, P, D_, K_, 1, 1, P, P, 1 << 20, None) == ARG
    for kw in (dict(B=-1), dict(B=65536), dict(D=6), dict(K=0), dict(N=-1)):
        assert _accumulate(lib, p, **kw) == ARG, kw
    for kw in (dict(B=-1), dict(B=65536), dict(D=6), dict(K=0), dict(R=-1), dict(R=1 << 31)):
        assert _accumulate_varlen(lib, p, **kw) == ARG, kw
    # the packed table's pointers: null and alignment before anything else
    assert _accumulate_varlen(lib, dict(p, row0=0)) == ARG and "null pointer" in _lib.last_error()
    assert _accumulate_varlen(lib, dict(p, len=P + 2), B=3) == ARG and "len must be 4-byte" in _lib.last_error()
