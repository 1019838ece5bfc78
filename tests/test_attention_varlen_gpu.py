"""The packed attention of the list calls (anyloc_attention_varlen: attention_wg_varlen_kernel for fp16 and bf16 pairs,
single bf16 and single fp16, attention_tc_varlen_kernel for tf32 pairs), image by image against fp64
softmax(q k^T / 8) v of that image alone, under the bounds of the padded kernels: test_attention_edges_gpu's (c = 32,
u = 2^-24) for the tf32 and fp16 pairs on the fp32 inputs, the attn_bound of test_bf16_kernels_gpu,
test_bf16x3_kernels_gpu and test_f16x1_kernels_gpu for bf16, bf16 pairs and single fp16 on the values of the operands
the kernel reads (the bf16 rounding, the bf16 pair, the fp16 rounding of 8 x over 8).  For fp16 pairs the bound
adds the format's absolute floor (f16_floor): a one-key image with a value of about 1e-5 is off by some 500 times
the relative bound alone, in the packed and the padded kernel alike, because the lo half of its fp16 pair underflows.

In the packed buffer the rows past an image's last key are the next image's (or, with gaps, whatever lies between
images), where the padded kernels read zeros.  So besides accuracy at every tile edge these tests check that nothing
of those rows reaches an image's output: neighbours built to dominate the softmax if a single key leaked, and Inf /
NaN neighbours, under which each image's rows must still equal anyloc_attention on that image alone bit for bit.
Every output buffer is surrounded, and its gaps filled, with NaN bit patterns that must survive the call; the table
is exercised full (128 images), permuted and one past full."""
import ctypes as C
import random

import pytest
import torch

from tests.test_attention_edges_gpu import C_ATT, U, reference, structured, to_qkv
from tests.test_bf16_kernels_gpu import attn_bound, to_bf16
from tests.test_bf16x3_kernels_gpu import attn_bound as pair_attn_bound, pair_of
from tests.test_f16x1_kernels_gpu import attn_bound as f16x1_attn_bound
from tests.util import dptr, split_f16, split_tf32

pytestmark = pytest.mark.gpu

FMTS = ["tf32", "f16", "bf16", "bf16pair", "f16x1"]
SINGLE = ("bf16", "f16x1")      # one array each way, no lo
DTYPE = {"tf32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "bf16pair": torch.bfloat16,
         "f16x1": torch.float16}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
CANARY = {torch.float32: 0x7FC0DEAD, torch.float16: 0x7EAD, torch.bfloat16: 0x7FDA}   # quiet NaNs no kernel writes
LEAD = 16
ARG, UNSUPPORTED = -1, -4
F16_FLOOR = 2.0 ** -28          # absolute error of an fp16 pair of 8x in x once lo is subnormal: 2^-25 / 8
# lengths around the 64-row key blocks and 128-row query tiles, the c2 / c5 lengths, with ties
LENGTHS = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257, 530, 1025, 1370]
TIES = [1, 65, 129, 530, 64]


@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    return _lib


def shuffled(lengths, seed):
    lengths = list(lengths)
    random.Random(seed).shuffle(lengths)
    return lengths


def layout(lens, gap=0):
    """row0 of each image, images in list order with `gap` rows after each one (the last included); total rows"""
    row0, r = [], 0
    for T in lens:
        row0.append(r)
        r += T + gap
    return row0, r


def operands(L, x, fmt):
    """the fp32 rows x [rows, 3D] in the format the qkv epilogue writes: (hi, lo), (bf16, None) or (fp16 of 8 x, None)"""
    if fmt == "tf32":
        return split_tf32(L, x)
    if fmt == "f16":
        return split_f16(L, x, L.ACT_SCALE)
    if fmt == "bf16pair":
        return pair_of(x)
    if fmt == "f16x1":
        return split_f16(L, x, L.ACT_SCALE)[0], None
    return to_bf16(L, x), None


def canary_buf(rows, D, dt):
    n = LEAD + rows * D + 2 * D + LEAD
    return torch.full((n,), CANARY[dt], dtype=BITS[dt], device="cuda").view(dt)


def rows_of(buf, rows, D):
    return buf[LEAD:LEAD + rows * D].view(rows, D)


def canaries_intact(buf, rows, D, row0, lens):
    """every element of buf outside the images' output rows still holds the NaN pattern"""
    bits = buf.view(BITS[buf.dtype]).clone()
    keep = rows_of(bits, rows, D)
    for r, T in zip(row0, lens):
        keep[r:r + T] = CANARY[buf.dtype]
    return bool((bits == CANARY[buf.dtype]).all())


def call(L, ops, row0, lens, heads, fmt, rows):
    """anyloc_attention_varlen into canary-padded outputs -> (rc, o_hi, o_lo)"""
    hi, lo = ops
    D, n = 64 * heads, len(lens)
    o_hi = canary_buf(rows, D, DTYPE[fmt])
    o_lo = canary_buf(rows, D, DTYPE[fmt]) if lo is not None else None
    rc = L.load().anyloc_attention_varlen(dptr(hi), dptr(lo), n, (C.c_int32 * n)(*row0), (C.c_int32 * n)(*lens), D,
                                          heads, dptr(o_hi, LEAD), dptr(o_lo, LEAD), L.PAIR[fmt], L.stream_ptr())
    torch.cuda.synchronize()
    return rc, o_hi, o_lo


def packed(L, ops, row0, lens, heads, fmt, rows):
    """a call that must succeed and leave every canary intact -> (o_hi, o_lo) as [rows, D] views"""
    rc, o_hi, o_lo = call(L, ops, row0, lens, heads, fmt, rows)
    assert rc == 0, L.last_error()
    D = 64 * heads
    for buf in (o_hi, o_lo):
        if buf is not None:
            assert canaries_intact(buf, rows, D, row0, lens), (fmt, "packed output written outside its images")
    return rows_of(o_hi, rows, D), None if o_lo is None else rows_of(o_lo, rows, D)


def padded(L, x, ops, r, T, heads, fmt):
    """anyloc_attention on image (rows [r, r + T)) alone: the tf32 pair of its fp32 rows for the tf32 and fp16 pairs
    (fp16 pairs: converted inside, hi + lo = x), its rows of the packed operands for the formats the qkv epilogue
    writes as such (bf16, bf16 pairs, single fp16) -> (o_hi, o_lo) [T, D]"""
    D = 64 * heads
    dt = DTYPE[fmt]
    if fmt in ("tf32", "f16"):
        q_hi, q_lo = split_tf32(L, x[r:r + T].contiguous())
    else:
        q_hi, q_lo = (None if a is None else a[r:r + T].contiguous() for a in ops)
    o_hi = canary_buf(T, D, dt)
    o_lo = canary_buf(T, D, dt) if fmt not in SINGLE else None
    L.check(L.load().anyloc_attention(dptr(q_hi), dptr(q_lo), 1, T, D, heads, dptr(o_hi, LEAD), dptr(o_lo, LEAD),
                                      L.PAIR[fmt], L.ENGINE["tc3"], L.stream_ptr()), "attention")
    torch.cuda.synchronize()
    for buf in (o_hi, o_lo):
        if buf is not None:
            assert canaries_intact(buf, T, D, [0], [T]), (fmt, T, "padded output written outside its rows")
    return rows_of(o_hi, T, D), None if o_lo is None else rows_of(o_lo, T, D)


def same_bits(a, b):
    return torch.equal(a.view(BITS[a.dtype]), b.view(BITS[b.dtype]))


def equals_padded(L, x, ops, out, row0, lens, heads, fmt, which=None):
    """images `which` (default all) of the packed output bit for bit against their lone anyloc_attention calls"""
    for i in range(len(lens)) if which is None else which:
        r, T = row0[i], lens[i]
        p_hi, p_lo = padded(L, x, ops, r, T, heads, fmt)
        assert same_bits(out[0][r:r + T], p_hi), (fmt, i, T)
        if p_lo is not None:
            assert same_bits(out[1][r:r + T], p_lo), (fmt, i, T)


def value(L, out, fmt):
    hi, lo = out
    if fmt == "bf16":
        return hi.double()
    if fmt == "f16x1":
        return hi.double() / L.ACT_SCALE
    o = hi.double() + lo.double()
    return o / L.ACT_SCALE if fmt == "f16" else o


def f16_floor(x, heads, logit_term):
    """The absolute error of the fp16-pair format, which the relative bound c u (...) leaves out.  A pair (hi, lo) of
    8x is good to 2^-22 |x| only while lo is a normal fp16 number; below, lo's spacing is 2^-24, so the pair is good to
    F16_FLOOR = 2^-25 / 8 absolute.  An image whose v are tiny (T = 1: o = v_0) shows it.  Per element: the V and
    output pairs add F16_FLOOR each, the P pairs (of 1024 p, p <= 1 before the division by l >= 1) 2^-35 per key times
    |v|, and (logit_term) the q and k pairs move each logit by at most F16_FLOOR (|q_i|_1 + max_j |k_j|_1) / 8, which
    moves o by twice that times P|V|.  Doubled for margin; [T, D]."""
    T = x.shape[0]
    q, k, v = (t.reshape(T, heads, 64).transpose(0, 1).double() for t in x.chunk(3, dim=-1))     # [H, T, 64]
    floor = (2 * F16_FLOOR + 2.0 ** -35 * v.abs().sum(-2, keepdim=True)).expand(heads, T, 64)
    if logit_term:
        P = torch.softmax(q @ k.transpose(-1, -2) / 8, dim=-1)
        ds = F16_FLOOR * (q.abs().sum(-1, keepdim=True) + k.abs().sum(-1).amax(-1)[:, None, None]) / 8
        floor = floor + 2 * ds * (P @ v.abs())
    return 2 * floor.transpose(0, 1).reshape(T, heads * 64)


def worst_share(L, x, ops, out, row0, lens, heads, fmt, logit_term=True):
    """max over every image's elements of |o - o64| / bound (asserted finite); o64 from that image's rows alone"""
    got_all = value(L, out, fmt)
    D = 64 * heads
    worst = 0.0
    for r, T in zip(row0, lens):
        got = got_all[r:r + T]
        assert bool(torch.isfinite(got).all()), (fmt, r, T)
        if fmt in ("bf16", "bf16pair", "f16x1"):
            if fmt == "bf16":
                X, bound_of = ops[0][r:r + T].double(), attn_bound
            elif fmt == "bf16pair":
                X, bound_of = ops[0][r:r + T].double() + ops[1][r:r + T].double(), pair_attn_bound
            else:
                X, bound_of = ops[0][r:r + T].double() / L.ACT_SCALE, f16x1_attn_bound
            ref, bound = bound_of(X.reshape(1, T, 3, heads, 64))
            ref, bound = (t[0].transpose(0, 1).reshape(T, D) for t in (ref, bound))
        else:
            ref, scale = reference(x[None, r:r + T], heads, logit_term)
            ref, bound = ref[0], C_ATT * U * scale[0]
            if fmt == "f16":
                bound = bound + f16_floor(x[r:r + T], heads, logit_term)
        worst = max(worst, float(((got - ref).abs() / bound).max()))
    return worst


def images(kind, lens, heads, seed, gap=0):
    """fp32 rows [rows, 3D] of the images (structured(kind) each, its own seed), row0, rows; gap rows are zero"""
    row0, rows = layout(lens, gap)
    x = torch.zeros(rows, 3 * 64 * heads, device="cuda")
    for i, (r, T) in enumerate(zip(row0, lens)):
        x[r:r + T] = to_qkv(*structured(kind, 1, heads, T, seed=seed * 1000 + i))[0]
    return x, row0, rows


# ------------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("kind", ["flat", "dominant_last", "ramp", "equal"])
@pytest.mark.parametrize("heads", [2, 24])
@pytest.mark.parametrize("fmt", FMTS)
def test_packed_against_fp64(L, fmt, heads, kind):
    lens = shuffled(LENGTHS + TIES, seed=heads + len(kind))
    x, row0, rows = images(kind, lens, heads, seed=heads)
    ops = operands(L, x, fmt)
    out = packed(L, ops, row0, lens, heads, fmt, rows)
    worst = worst_share(L, x, ops, out, row0, lens, heads, fmt, logit_term=kind != "equal")
    print(f"packed attention {fmt} heads={heads} {kind}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, (fmt, heads, kind, worst)


@pytest.mark.parametrize("gap", [0, 3])
@pytest.mark.parametrize("heads", [2, 24])
@pytest.mark.parametrize("fmt", FMTS)
def test_packed_equals_padded(L, fmt, heads, gap):
    """each image's rows of the packed call are those of anyloc_attention on that image alone, bit for bit"""
    lens = shuffled(LENGTHS + TIES, seed=7 + heads)
    x, row0, rows = images("flat", lens, heads, seed=11 + gap, gap=gap)
    ops = operands(L, x, fmt)
    equals_padded(L, x, ops, packed(L, ops, row0, lens, heads, fmt, rows), row0, lens, heads, fmt)


# ------------------------------------------------------------------------------------------- the neighbours' rows
@pytest.mark.parametrize("gap", [0, 5])
@pytest.mark.parametrize("fmt", FMTS)
def test_adversarial_neighbours(L, fmt, gap):
    """The rows right after each image (the next image's first three, or the gap) hold a key along that image's
    queries, about 60 logits above its own keys, and values of +-1e3 (8e3 for fp16 pairs, inside their range): one
    leaked key would move the image's output by about 1e3."""
    heads, D = 2, 128
    lens = shuffled(LENGTHS + TIES, seed=3)
    row0, rows = layout(lens, gap)
    g = torch.Generator(device="cuda").manual_seed(5 + gap)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    q, k, v = r(rows, heads, 64) * 0.3, r(rows, heads, 64) * 0.3, r(rows, heads, 64)
    after = []                        # (image, rows right after it)
    for i, (r0, T) in enumerate(zip(row0, lens)):
        d = i % 64                    # image i's queries point along e_d; its neighbours' along other axes
        q[r0:r0 + T, :, d] += 22.0
        end = r0 + T + (gap if gap else min(3, lens[i + 1]) if i + 1 < len(lens) else 0)
        after.append((i, slice(r0 + T, end)))
        k[r0 + T:end] = 0.0
        k[r0 + T:end, :, d] = 22.0
        v[r0 + T:end] = torch.where(r(end - r0 - T, heads, 64) > 0, 1e3, -1e3)
    x = torch.cat([t.reshape(rows, D) for t in (q, k, v)], dim=1).contiguous()
    for i, s in after:                # the construction does what it claims
        if s.stop > s.start:
            r0, T = row0[i], lens[i]
            own = (q[r0:r0 + T].transpose(0, 1) @ k[r0:r0 + T].transpose(0, 1).transpose(1, 2)).amax(-1) / 8
            bad = (q[r0:r0 + T].transpose(0, 1) @ k[s].transpose(0, 1).transpose(1, 2)).amin(-1) / 8
            assert float((bad - own).min()) > 50.0, (i, float((bad - own).min()))
    ops = operands(L, x, fmt)
    out = packed(L, ops, row0, lens, heads, fmt, rows)
    worst = worst_share(L, x, ops, out, row0, lens, heads, fmt)
    print(f"packed attention {fmt} adversarial neighbours gap={gap}: worst err/bound {worst:.3f}")
    assert worst <= 1.0, (fmt, gap, worst)
    equals_padded(L, x, ops, out, row0, lens, heads, fmt)


def poison(t, rows):
    """Inf, -Inf and NaN, column after column, in the given rows of an operand array"""
    bad = torch.tensor([float("inf"), -float("inf"), float("nan")], device="cuda", dtype=t.dtype)
    t[rows] = bad.repeat(t.shape[1] // 3 + 1)[:t.shape[1]]


@pytest.mark.parametrize("gap", [0, 4])
@pytest.mark.parametrize("fmt", FMTS)
def test_nonfinite_neighbour(L, fmt, gap):
    """Inf and NaN in the q, k and v rows right after an image (the next image's first rows, or the gap) leave the
    image's rows bit-identical to its lone call: keys past an image get p = 0, and 0 times Inf or NaN must not reach
    its output."""
    heads = 2
    clean = [1, 2, 63, 65, 129, 193, 530, 1025, 1370, 64, 128]     # images at even positions
    dirty = [5, 64, 70, 1, 200, 3, 129, 2, 90, 66, 1]              # first rows poisoned (gap = 0)
    lens = [T for pair in zip(clean, dirty) for T in pair]
    x, row0, rows = images("flat", lens, heads, seed=21 + gap, gap=gap)
    ops = operands(L, x, fmt)
    for a in ops:
        if a is None:
            continue
        for i, (r0, T) in enumerate(zip(row0, lens)):
            if gap:
                poison(a, slice(r0 + T, r0 + T + gap))
            elif i % 2:
                poison(a, slice(r0, r0 + min(T, 3)))
    out = packed(L, ops, row0, lens, heads, fmt, rows)
    which = range(len(lens)) if gap else range(0, len(lens), 2)
    equals_padded(L, x, ops, out, row0, lens, heads, fmt, which)


# ----------------------------------------------------------------------------------------------------- the table
@pytest.mark.parametrize("fmt", FMTS)
def test_full_table_and_order(L, fmt):
    """128 images of mixed lengths (T = 1 and 2, ties, one active consumer half) in one call: correct, each equal to
    its lone call; the images permuted in the buffer permute the outputs bit for bit; 129 images are refused"""
    heads, n = 2, 128
    rng = random.Random(128)
    lens = [1, 2, 64, 65, 128, 129, 300, 300, 1, 64] + [rng.randint(1, 300) for _ in range(n - 10)]
    lens = shuffled(lens, seed=1)
    x, row0, rows = images("flat", lens, heads, seed=128)
    ops = operands(L, x, fmt)
    out = packed(L, ops, row0, lens, heads, fmt, rows)
    worst = worst_share(L, x, ops, out, row0, lens, heads, fmt)
    print(f"packed attention {fmt} 128 images: worst err/bound {worst:.3f}")
    assert worst <= 1.0, (fmt, worst)
    equals_padded(L, x, ops, out, row0, lens, heads, fmt)

    perm = list(range(n))
    random.Random(2).shuffle(perm)
    lens_p = [lens[i] for i in perm]
    row0_p, _ = layout(lens_p)
    src = torch.cat([torch.arange(row0[i], row0[i] + lens[i]) for i in perm]).cuda()
    ops_p = tuple(None if a is None else a[src].contiguous() for a in ops)
    out_p = packed(L, ops_p, row0_p, lens_p, heads, fmt, rows)
    for k, i in enumerate(perm):
        for a, b in zip(out, out_p):
            if a is not None:
                assert same_bits(b[row0_p[k]:row0_p[k] + lens[i]], a[row0[i]:row0[i] + lens[i]]), (fmt, k, i)

    lens_over = lens + [1]
    row0_over, rows_over = layout(lens_over)
    ops_over = tuple(None if a is None else torch.cat([a, a[:1]]) for a in ops)
    rc, o_hi, o_lo = call(L, ops_over, row0_over, lens_over, heads, fmt, rows_over)
    assert rc == ARG and "out of range" in L.last_error()
    assert all(canaries_intact(b, rows_over, 64 * heads, [], []) for b in (o_hi, o_lo) if b is not None)


@pytest.mark.parametrize("fmt", FMTS)
def test_refusals_write_nothing(L, fmt):
    heads, D = 2, 128
    lens = [65, 130]
    x, row0, rows = images("flat", lens, heads, seed=0)
    hi, lo = operands(L, x, fmt)
    other = "tf32" if fmt in SINGLE else "bf16"
    a, b = dptr(hi), dptr(lo)
    b_bad = dptr(hi) if fmt in SINGLE else dptr(None)         # a lo array for a single format, none for a pair
    cases = [(a, b, [0, 64], lens, heads, fmt, ARG),             # overlapping images
             (a, b, [-1, 65], lens, heads, fmt, ARG),
             (a, b, row0, [0, 130], heads, fmt, ARG),
             (a, b_bad, row0, lens, heads, fmt, ARG),
             (a, b, row0, lens, heads + 1, fmt, ARG),             # D = 128 != 64 heads
             (a, b, row0, lens, heads, other, ARG),               # lo arrays that do not fit the format
             (dptr(hi, 1), b, row0, lens, heads, fmt, UNSUPPORTED)]   # qkv_hi 4 (tf32) or 2 bytes off alignment
    lib = L.load()
    for qh, ql, r0, ln, h, f, want in cases:
        dt = DTYPE[fmt]
        o_hi, o_lo = canary_buf(rows, D, dt), canary_buf(rows, D, dt)
        rc = lib.anyloc_attention_varlen(qh, ql, 2, (C.c_int32 * 2)(*r0), (C.c_int32 * 2)(*ln), D, h,
                                         dptr(o_hi, LEAD), dptr(o_lo if f not in SINGLE else None, LEAD), L.PAIR[f],
                                         L.stream_ptr())
        torch.cuda.synchronize()
        assert rc == want, (fmt, r0, ln, h, f, rc, L.last_error())
        assert canaries_intact(o_hi, rows, D, [], []) and canaries_intact(o_lo, rows, D, [], []), (fmt, r0, ln, h, f)
