"""GPU parity of the building blocks behind the ViT forward (C ABI: anyloc_gemm_nt with every
epilogue on both engines, anyloc_layernorm_split, anyloc_attention, anyloc_split_tf32) against
plain PyTorch fp64/fp32 references of the same op."""
import ctypes as C

import pytest
import torch

from tests.util import gemm, rel_inf, split_f16
from tests.util import split_tf32 as split

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def test_split_exact(L):
    x = torch.randn(100003, device="cuda") * torch.logspace(-20, 20, 100003, device="cuda")
    hi, lo = split(L, x)
    assert torch.equal(hi + lo, x)
    assert bool(((hi.view(torch.int32) & 0x1FFF) == 0).all())          # tf32: low 13 mantissa bits clear
    assert bool((lo.abs() <= hi.abs() * 2.0 ** -10).all())


def test_split_f16_precision(L):
    x = torch.randn(100003, device="cuda") * 3
    hi, lo = split_f16(L, x, 8.0)
    rec = (hi.double() + lo.double()) / 8.0
    big = x.abs() > 0.05
    assert float(((rec - x.double()).abs() / x.double().abs())[big].max()) < 2.0 ** -21
    assert float((rec - x.double()).abs().max()) < 2.0 ** -21 * 3 * 6


def ref_gemm(a, b, epi, bias, gamma, resid):
    acc = a.double() @ b.double().T
    if bias is not None:
        acc = acc + bias.double()
    if epi in ("bias", "bias_split"):
        return acc
    if epi == "gelu_split":
        return torch.nn.functional.gelu(acc)
    if epi == "swiglu_split":
        return torch.nn.functional.silu(acc[:, 0::2]) * acc[:, 1::2]
    if epi == "ls_resid":
        return resid.double() + gamma.double() * acc
    raise ValueError(epi)


ENGINES = ["simt", "tc3"]


@pytest.mark.parametrize("pair", ["tf32", "f16"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (530, 1152, 384), (1000, 384, 1536), (257, 128, 608),
                                   (2048, 512, 4096), (77, 200, 36)])
@pytest.mark.parametrize("epi", ["bias", "bias_split", "gelu_split", "swiglu_split", "ls_resid"])
def test_gemm_epilogues(L, pair, engine, M, N, K, epi):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=g)
    b = torch.randn(N, K, device="cuda", generator=g) * 0.05
    bias = torch.randn(N, device="cuda", generator=g)
    n_out = N // 2 if epi == "swiglu_split" else N
    gamma = torch.randn(N, device="cuda", generator=g) if epi == "ls_resid" else None
    resid = torch.randn(M, n_out, device="cuda", generator=g) if epi == "ls_resid" else None
    q = 8 if pair == "f16" else 4               # gemm_tc_supported: K a multiple of 16 bytes (operands are aligned)
    if engine == "tc3" and K % q:
        with pytest.raises(L.AnylocError, match=r"rc=-4"):        # ANYLOC_ERR_UNSUPPORTED
            gemm(L, a, b, epi, bias, gamma, resid, engine, pair)
        return
    out = gemm(L, a, b, epi, bias, gamma, resid, engine, pair)
    ref = ref_gemm(a, b, epi, bias, gamma, resid)
    err = rel_inf(out.cpu(), ref.cpu())
    assert err < 2e-6 * max(1.0, (K / 64) ** 0.5), (pair, engine, epi, err)


@pytest.mark.parametrize("pair", ["tf32", "f16"])
@pytest.mark.parametrize("D", [384, 768, 1024, 1536])
def test_layernorm_split(L, pair, D):
    g = torch.Generator(device="cuda").manual_seed(D)
    x = torch.randn(531, D, device="cuda", generator=g) * 3 + 0.5
    w, b = torch.randn(D, device="cuda", generator=g), torch.randn(D, device="cuda", generator=g)
    dt = torch.float16 if pair == "f16" else torch.float32
    hi, lo = torch.empty_like(x, dtype=dt), torch.empty_like(x, dtype=dt)
    L.check(L.load().anyloc_layernorm_split(L.ptr(x), L.ptr(w), L.ptr(b), 531, D, C.c_float(1e-6), L.ptr(hi),
                                            L.ptr(lo), L.PAIR[pair], L.stream_ptr()), "layernorm")
    ref = torch.nn.functional.layer_norm(x.double(), (D,), w.double(), b.double(), 1e-6)
    rec = (hi.double() + lo.double()) / (L.ACT_SCALE if pair == "f16" else 1.0)
    assert rel_inf(rec.cpu(), ref.cpu()) < 2e-6


@pytest.mark.parametrize("pair", ["tf32", "f16"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("B,T,heads", [(2, 257, 6), (1, 530, 24), (3, 64, 2), (1, 1370, 16), (2, 65, 1), (2, 129, 2)])
def test_attention(L, pair, engine, B, T, heads):
    D = heads * 64
    g = torch.Generator(device="cuda").manual_seed(T)
    qkv = torch.randn(B, T, 3 * D, device="cuda", generator=g) * 1.5
    q_hi, q_lo = split(L, qkv)
    dt = torch.float16 if pair == "f16" else torch.float32
    hi, lo = torch.empty(B, T, D, device="cuda", dtype=dt), torch.empty(B, T, D, device="cuda", dtype=dt)
    L.check(L.load().anyloc_attention(L.ptr(q_hi), L.ptr(q_lo), B, T, D, heads, L.ptr(hi), L.ptr(lo),
                                      L.PAIR[pair], L.ENGINE[engine], L.stream_ptr()), "attn")
    torch.cuda.synchronize()
    hi, lo = hi.double() / (L.ACT_SCALE if pair == "f16" else 1.0), lo.double() / (L.ACT_SCALE if pair == "f16" else 1.0)
    q, k, v = (t.reshape(B, T, heads, 64).transpose(1, 2).double() for t in qkv.chunk(3, dim=-1))
    ref = (torch.softmax(q @ k.transpose(-1, -2) * 0.125, dim=-1) @ v).transpose(1, 2).reshape(B, T, D)
    assert rel_inf((hi + lo).cpu(), ref.cpu()) < 5e-6
