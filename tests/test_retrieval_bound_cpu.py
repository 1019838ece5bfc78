"""The retrieval bound of tests/test_retrieval_engine_gpu.py on a CPU model of the kernels' arithmetic: an fp32
evaluation of normalise -> fp16 (or tf32) pairs -> fp32 product -> k best must pass every check, and the wrong
references of the GPU test must violate the bound on that same output."""
import pytest
import torch

from tests.test_retrieval_engine_gpu import IP, L2, S_RET, check, reference, uses_f16


def rows(fam, n, Dv, g):
    x = torch.randn(n, Dv, generator=g, dtype=torch.float64)
    if fam == "near_dup":                              # scores near 1, L2 distances near 0
        base = torch.randn(8, Dv, generator=g, dtype=torch.float64)
        x = base[torch.randint(0, 8, (n,), generator=g)] + x * (1e-4 / Dv ** 0.5)
    return x.float()


def fp32_search(db, qu, k, metric, normalize):
    """the kernels' arithmetic in fp32 on the CPU (reduction orders differ; the bound must not care)"""
    Dv = db.shape[1]

    def prep(x):
        y = x / x.square().sum(1, keepdim=True).sqrt().clamp_min(1e-12) if normalize else x
        if uses_f16(Dv, normalize):
            a = y * S_RET
            hi = a.half().float()
            return (hi + (a - hi).half().float()) / S_RET, y.square().sum(1)
        return y, y.square().sum(1)

    (y, dd), (q, qq) = prep(db), prep(qu)
    s = q @ y.T
    key = s if metric == IP else -((qq[:, None] - 2.0 * s) + dd[None, :])
    key = torch.where(torch.isnan(key), torch.full((), -float("inf")), key)
    order = torch.sort(-key, dim=1, stable=True).indices[:, :k]
    d = key.gather(1, order)
    return (d if metric == IP else -d), order


@pytest.mark.parametrize("fam,Dv,metric,normalize", [("random", 256, IP, 1), ("random", 260, IP, 1),
                                                     ("near_dup", 64, IP, 1), ("near_dup", 256, L2, 1),
                                                     ("random", 256, IP, 0), ("random", 1024, L2, 1)])
def test_fp32_model_within_bound(fam, Dv, metric, normalize):
    g = torch.Generator().manual_seed(Dv + metric)
    db, qu = rows(fam, 1500, Dv, g), rows(fam, 40, Dv, g)
    dist, idx = fp32_search(db, qu, 10, metric, normalize)
    ref, B = reference(db, qu, normalize, metric)
    r, fixed = check(dist, idx, ref, B, metric)
    print(f"{fam} Dv={Dv} metric={metric} normalize={normalize}: worst ratio {r:.3f}, {fixed:.2f} fixed")
    assert r <= 1.0


@pytest.mark.parametrize("mutate,fam,Dv,metric", [("hi_norm", "near_dup", 64, IP), ("drop_tail4", "random", 260, IP),
                                                  ("raw_qq", "random", 256, L2)])
def test_wrong_references_violate_bound(mutate, fam, Dv, metric):
    g = torch.Generator().manual_seed(Dv)
    db, qu = rows(fam, 1500, Dv, g), rows(fam, 40, Dv, g)
    if mutate == "drop_tail4":
        db[:, -4:] += 0.3 * db.norm(dim=1, keepdim=True) / Dv ** 0.5 * 16
        qu[:, -4:] += 0.3 * qu.norm(dim=1, keepdim=True) / Dv ** 0.5 * 16
    if mutate == "raw_qq":
        qu = qu / qu.norm(dim=1, keepdim=True) * 3.0
    dist, idx = fp32_search(db, qu, 10, metric, 1)
    _, B = reference(db, qu, 1, metric)
    wref, _ = reference(db, qu, 1, metric, mutate=mutate)
    r = float(((dist.double() - wref.gather(1, idx)).abs() / B.gather(1, idx)).max())
    print(f"{mutate}: worst ratio {r:.3g}")
    assert r > 1.0
