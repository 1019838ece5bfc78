"""The error bounds that make VLAD labels and top-k indices exact, checked on what the device's hi-only tensor-core pass
actually returns (tests/test_vlad_bound_cpu.py checks the same bounds on a CPU model of that arithmetic).

Both coarse passes are reached through anyloc_gemm_nt with the arguments their callers use:
  * VLAD (vlad.cu, launch_assign): tf32, the raw fp32 features as a_hi, rna_tf32(c^) as b_hi, no lo operands, the
    centre bias (0 for cosine).  Bounds: the a-priori eps = 2^-9 |x| max|c^| of vlad_rescore_kernel and the
    data-dependent eps' of the CPU test.
  * Retrieval (topk.cu, anyloc_index_search): fp16 hi of kRetrievalScale * y for queries and database, no lo operands,
    alpha = 1 / s^2.  Bound: eps_q = 1.001 (dn_q + DN + dn_q DN) + 3e-5 of topk_candidates_kernel, with dn as
    normalize_rows_split_kernel defines it.  The 3e-5 is the allowance for the fp32 accumulation; the share of it the
    device uses is printed (max |S~ - hi_q.hi_d / s^2| / 3e-5)."""
import numpy as np
import pytest
import torch

from tests.test_vlad_bound_cpu import CASES, coarse_scores, eps_bound, rna_tf32
from tests.util import gemm_nt, split_f16

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


# ---------------------------------------------------------------------------------------------------------- VLAD
@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("D,K", [(384, 5), (1024, 32), (1536, 128), (2048, 200)])
def test_vlad_coarse_bound_on_device(L, name, D, K):
    R = 512                                              # the fast path needs R >= 256 rows
    g = np.random.default_rng(hash((name, D, K, "gpu")) % (2 ** 32))
    x = CASES[name](g, R, D).astype(np.float32)
    c = (g.standard_normal((K, D)) * g.uniform(0.2, 3.0, (K, 1))).astype(np.float32)
    if name == "all_just_below_tf32_ulp":
        c[0] = np.sign(x[0])
    chat = (c / (np.sqrt((c.astype(np.float64) ** 2).sum(1, keepdims=True)) + 1e-8)).astype(np.float32)
    chat_t = rna_tf32(chat)
    xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(chat_t).cuda()
    bias = torch.zeros(K, device="cuda")                 # cbias of the cosine distance
    out = torch.empty(R, K, device="cuda")
    L.check(gemm_nt(L, xd, None, cd, None, R, K, D, pair="tf32", bias=bias, out=out, ldo=K, engine="tc3"), "gemm")
    coarse = out.double().cpu().numpy()
    exact = (xd.double() @ torch.from_numpy(chat).cuda().double().T).cpu().numpy()
    eps, xn, cmax = eps_bound(x, chat, chat_t)
    eps_apriori = 2.0 ** -9 * xn.astype(np.float64) * cmax
    err = np.abs(coarse - exact).max(1)
    r1 = float((err / np.maximum(eps, 1e-300)).max())
    r2 = float((err / np.maximum(eps_apriori, 1e-300)).max())
    # which CPU model of the accumulation the device matches (first 16 rows)
    match = {o: float((coarse_scores(x[:16], chat_t, o) == out[:16].cpu().numpy()).mean())
             for o in ("natural", "trunc")}
    print(f"VLAD coarse {name} D={D} K={K}: max|S~-S64|/eps' {r1:.3f}, /eps_apriori {r2:.3f}; "
          f"bitwise agreement natural {match['natural']:.2f} trunc {match['trunc']:.2f}")
    assert r1 <= 1.0 and r2 <= 1.0, (name, D, K, r1, r2)


# ----------------------------------------------------------------------------------------------------- retrieval
S_RET = 4096.0                                           # kRetrievalScale
ALLOWANCE = 3e-5


def unit_rows(kind, n, D, g, base=None):
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    if kind == "random":
        x = r(n, D)
    elif kind == "positive":                            # every product positive: the largest accumulation bias
        x = torch.rand(n, D, device="cuda", generator=g)
    elif kind == "spiky":                               # 4 large entries, the rest below fp16's normal range once scaled
        x = r(n, D) * 1e-9
        x[:, :4] += 0.5 + torch.rand(n, 4, device="cuda", generator=g)
    elif kind == "near_dup":
        x = base[torch.randint(0, base.shape[0], (n,), device="cuda", generator=g)] + r(n, D) * (1e-4 / D ** 0.5)
    else:
        raise ValueError(kind)
    return (x.double() / x.double().norm(dim=1, keepdim=True)).float()


def dn_rows(y):
    """|s y - hi| / s per row, rounded up as normalize_rows_split_kernel writes it (hi = s y rounded to 11 bits)"""
    a = y * S_RET
    t = a * 8193.0
    e = (a - (t - (t - a))).double()
    return ((e * e).sum(1).sqrt() * 1.001 + y.shape[1] ** 0.5 * 2.98e-8) / S_RET


@pytest.mark.parametrize("kind", ["random", "positive", "spiky", "near_dup"])
@pytest.mark.parametrize("Dv", [256, 3072, 49152])
def test_retrieval_coarse_bound_on_device(L, Dv, kind):
    g = torch.Generator(device="cuda").manual_seed(Dv + len(kind))
    n_q, n_db = 64, 512
    db = unit_rows("random" if kind == "near_dup" else kind, n_db, Dv, g)
    qu = unit_rows(kind, n_q, Dv, g, base=db)
    if kind == "near_dup":
        db = unit_rows("near_dup", n_db, Dv, g, base=db[:32])
    hq, _ = split_f16(L, qu, S_RET)
    hd, _ = split_f16(L, db, S_RET)
    out = torch.empty(n_q, n_db, device="cuda")
    L.check(gemm_nt(L, hq, None, hd, None, n_q, n_db, Dv, pair="f16", alpha=1.0 / (S_RET * S_RET), out=out, ldo=n_db,
                    engine="tc3"), "gemm")
    s = out.double()
    exact = qu.double() @ db.double().T
    dq, DN = dn_rows(qu)[:, None], float(dn_rows(db).max())
    eps = 1.001 * (dq + DN + dq * DN) + ALLOWANCE
    ratio = float(((s - exact).abs() / eps).max())
    acc_err = float((s - (hq.double() @ hd.double().T) / S_RET ** 2).abs().max())
    print(f"retrieval coarse {kind} Dv={Dv}: max|S~-S64|/eps_q {ratio:.3f}; accumulation error {acc_err:.2e} = "
          f"{acc_err / ALLOWANCE:.3f} of the 3e-5 allowance")
    assert ratio <= 1.0, (kind, Dv, ratio)
    assert acc_err <= ALLOWANCE


# -------------------------------------------------------------------------------------------- end-to-end near ties
# Exact score gaps of 2e-6 .. 1e-5: above the 1e-6 under which the other retrieval tests call a query ambiguous, far
# below the coarse passes' error (~1e-4 at these sizes), so only the exact re-scoring can order them.
def _orthonormal_to(q, n, g):
    w = torch.randn(n, q.shape[0], device="cuda", generator=g, dtype=torch.float64)
    w = w - (w @ q)[:, None] * q[None, :]
    return w / w.norm(dim=1, keepdim=True)


def test_topk_near_ties_exact_order(cuda):
    from anyloc_b200 import utilities as u
    g = torch.Generator(device="cuda").manual_seed(17)
    n_q, per_q, n_db, Dv, k = 64, 32, 2048, 3072, 10
    qu = torch.randn(n_q, Dv, device="cuda", generator=g, dtype=torch.float64)
    qu = qu / qu.norm(dim=1, keepdim=True)
    db = torch.randn(n_db, Dv, device="cuda", generator=g, dtype=torch.float64)
    db = db / db.norm(dim=1, keepdim=True)
    for i in range(n_q):                        # rows [32 i, 32 i + 32): scores 0.9 - cumulative gaps of 2e-6 .. 1e-5
        gaps = 2e-6 + 8e-6 * torch.rand(per_q, device="cuda", generator=g, dtype=torch.float64)
        s = 0.9 - torch.cumsum(gaps, 0)
        w = _orthonormal_to(qu[i], per_q, g)
        db[per_q * i:per_q * (i + 1)] = s[:, None] * qu[i][None, :] + (1 - s * s).sqrt()[:, None] * w
    qu32, db32 = qu.float(), db.float()
    q64, d64 = qu32.double(), db32.double()
    exact = (q64 / q64.norm(dim=1, keepdim=True)) @ (d64 / d64.norm(dim=1, keepdim=True)).T
    top = exact.topk(k + 1, dim=1)
    gap = (top.values[:, :-1] - top.values[:, 1:]).min()
    assert 1.5e-6 < float(gap) < 1.2e-5
    _, idx = u.top_k_search(db32, qu32, k, "cosine")
    assert torch.equal(idx.cpu().long(), top.indices[:, :k].cpu()), "top-k order differs from the fp64 order"


def test_vlad_labels_near_ties_exact(cuda):
    from anyloc_b200 import utilities as u
    g = torch.Generator(device="cuda").manual_seed(23)
    R, D, K = 1024, 1024, 32
    c = torch.randn(K, D, device="cuda", generator=g, dtype=torch.float64)
    c = (c / c.norm(dim=1, keepdim=True)).float()
    chat = c.double() / (c.double().norm(dim=1, keepdim=True) + 1e-8)
    a = torch.randint(0, K, (R,), device="cuda", generator=g)
    b = (a + torch.randint(1, K, (R,), device="cuda", generator=g)) % K
    mid = chat[a] + chat[b]
    mid = mid / mid.norm(dim=1, keepdim=True)
    diff = chat[a] - chat[b]
    gap = (2e-6 + 8e-6 * torch.rand(R, device="cuda", generator=g, dtype=torch.float64)) * \
        torch.where(torch.rand(R, device="cuda", generator=g) < 0.5, -1.0, 1.0).double()
    x = (mid + (gap / (diff * diff).sum(1))[:, None] * diff).float()   # x . (c^_a - c^_b) = gap
    scores = x.double() @ chat.T
    best2 = scores.topk(2, dim=1).values
    assert float((best2[:, 0] - best2[:, 1]).min()) > 1.5e-6 and float((best2[:, 0] - best2[:, 1]).max()) < 1.2e-5
    km = u._KMeans(K, mode="cosine")
    km.centroids = c
    labels = km.predict(x)
    assert torch.equal(labels.cpu(), scores.argmax(1).cpu()), "VLAD labels differ from the fp64 argmax"
