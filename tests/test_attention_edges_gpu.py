"""Attention (anyloc_attention) at its edges, element by element against fp64 softmax(Q K^T / 8) V on the same inputs:
sequence lengths around the 64-key block (T = 1, 2, 63, 64, 127, 1025), logits up to +-60 (near-one-hot rows, a
dominant key in the last, partial key block, a monotone ramp), all keys equal, and a large (image, head) grid whose
images, permuted, must permute the output bit for bit.  Tensor-core engine in both pair formats, SIMT as the control.

Per element (b, h, t, d), with P the exact probabilities and l_j = sum_i |q_i k_ji| / 8 the magnitude behind logit j:

    |o - o64| <= c u (1 + 2 max_j l_j) (P |V|)_d,   u = 2^-24, c = 32,

the first term for rounding in P.V and the normalisation, the second for logit errors (each logit is good to about
c u l_j, and moves o by at most that times sum_j p_j |v_jd - o_d| <= 2 (P |V|)_d).  For all-equal keys the logits are
bitwise equal, so the logit term is dropped: the output is the mean of V to within fp32 rounding."""
import pytest
import torch

from tests.util import split_tf32

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_ATT = 32


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def attention(L, qkv, heads, pair, engine):
    B, T, D3 = qkv.shape
    D = D3 // 3
    q_hi, q_lo = split_tf32(L, qkv.contiguous())
    dt = torch.float16 if pair == "f16" else torch.float32
    hi, lo = torch.empty(B, T, D, device="cuda", dtype=dt), torch.empty(B, T, D, device="cuda", dtype=dt)
    L.check(L.load().anyloc_attention(L.ptr(q_hi), L.ptr(q_lo), B, T, D, heads, L.ptr(hi), L.ptr(lo), L.PAIR[pair],
                                      L.ENGINE[engine], L.stream_ptr()), "attention")
    torch.cuda.synchronize()
    return hi, lo


def value(L, hi, lo, pair):
    o = hi.double() + lo.double()
    return o / L.ACT_SCALE if pair == "f16" else o


def to_qkv(q, k, v):
    """[B, H, T, 64] x3 -> the row-major [B, T, 3D] buffer (q | k | v thirds)"""
    B, H, T, _ = q.shape
    return torch.cat([t.transpose(1, 2).reshape(B, T, H * 64) for t in (q, k, v)], dim=-1).float().contiguous()


def reference(qkv, heads, logit_term=True):
    B, T, D3 = qkv.shape
    q, k, v = (t.reshape(B, T, heads, 64).transpose(1, 2).double() for t in qkv.chunk(3, dim=-1))
    P = torch.softmax(q @ k.transpose(-1, -2) * 0.125, dim=-1)
    o = P @ v
    scale = P @ v.abs()
    if logit_term:
        lmax = (q.abs() @ k.abs().transpose(-1, -2) * 0.125).amax(-1, keepdim=True)
        scale = scale * (1 + 2 * lmax)
    back = lambda t: t.transpose(1, 2).reshape(B, T, heads * 64)
    return back(o), back(scale)


def check(L, qkv, heads, pair, engine, logit_term=True, what=""):
    out = value(L, *attention(L, qkv, heads, pair, engine), pair)
    ref, scale = reference(qkv, heads, logit_term)
    err = (out - ref).abs()
    worst = float((err / (C_ATT * U * scale)).max())
    B, T, D = ref.shape
    rows = err.view(B, T, heads, 64).amax(-1) / ref.abs().view(B, T, heads, 64).amax(-1).clamp_min(1e-300)
    print(f"attention {what} {pair}/{engine}: max err/bound {worst:.3f}, worst per-row max|do|/max|o| {float(rows.max()):.2e}")
    assert torch.isfinite(out).all() and worst <= 1.0, (what, pair, engine, worst)


def structured(kind, B, heads, T, seed):
    """q, k, v [B, H, T, 64] whose logits reach +-60"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g, dtype=torch.float64)
    v = r(B, heads, T, 64)
    e = torch.zeros(64, device="cuda", dtype=torch.float64)
    e[0] = 1.0
    if kind == "flat":
        return r(B, heads, T, 64) * 1.5, r(B, heads, T, 64) * 1.5, v * 1.5
    if kind == "dominant_last":          # key T-1 (in the last, partial key block) ~60 above all the others
        q = r(B, heads, T, 64) * 0.3 + 22.0 * e
        k = r(B, heads, T, 64) * 0.3
        k[:, :, T - 1] += 22.0 * e
        return q, k, v
    if kind == "ramp":                   # logits rise monotonically over the keys, from about -60 to +60
        q = r(B, heads, T, 64) * 0.1 + 22.0 * e
        ramp = torch.linspace(-21.8, 21.8, T, device="cuda", dtype=torch.float64)
        k = r(B, heads, T, 64) * 0.1 + ramp[:, None] * e
        return q, k, v
    if kind == "equal":                  # every key the same (per image and head): uniform rows whatever the logits
        q = r(B, heads, T, 64) * 8.0
        k = r(B, heads, 1, 64).expand(B, heads, T, 64) * 8.0
        return q, k, v
    raise ValueError(kind)


CONFIGS = [("tf32", "tc3"), ("f16", "tc3"), ("tf32", "simt"), ("f16", "simt")]


@pytest.mark.parametrize("pair,engine", CONFIGS)
@pytest.mark.parametrize("kind", ["flat", "dominant_last", "ramp", "equal"])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 127, 1025])
def test_attention_edges(L, T, kind, pair, engine):
    B, heads = 2, 3
    q, k, v = structured(kind, B, heads, T, seed=T * 10 + len(kind))
    qkv = to_qkv(q, k, v)
    if kind in ("dominant_last", "ramp") and T > 1:     # the construction does what it claims
        ref_lg = (qkv[..., :192].reshape(B, T, heads, 64).transpose(1, 2).double() @
                  qkv[..., 192:384].reshape(B, T, heads, 64).transpose(1, 2).double().transpose(-1, -2)) * 0.125
        assert float(ref_lg.abs().max()) > 50.0
        if kind == "dominant_last":
            assert bool((ref_lg.argmax(-1) == T - 1).all())
    check(L, qkv, heads, pair, engine, logit_term=kind != "equal", what=f"{kind} T={T}")


@pytest.mark.parametrize("pair,engine", CONFIGS[:2])
def test_attention_large_grid_permutation(L, pair, engine):
    """B = 40 images x 24 heads with different data each: correct everywhere, and permuting the images permutes the
    output bit for bit (no state leaks between (image, head) CTAs)"""
    B, heads, T = 40, 24, 130
    g = torch.Generator(device="cuda").manual_seed(40)
    qkv = torch.randn(B, T, 3 * heads * 64, device="cuda", generator=g) * \
        torch.rand(B, 1, 1, device="cuda", generator=g).add(0.5) * 1.5
    check(L, qkv, heads, pair, engine, what="grid 40x24")
    hi, lo = attention(L, qkv, heads, pair, engine)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(3)).cuda()
    hi_p, lo_p = attention(L, qkv[perm].contiguous(), heads, pair, engine)
    assert torch.equal(hi_p, hi[perm]) and torch.equal(lo_p, lo[perm])
