"""The four pre-processing kernels (anyloc_preprocess_u8, anyloc_preprocess_resize_u8 and anyloc_preprocess_u8_varlen
with interpolation -1, 0 and 1) checked element by element against fp64 through the C ABI, every output inside a NaN
frame that must come back untouched.

The fp64 reference (`resize64`, numpy only) restates preprocess.cu's formula.  Pixel value v = (p/255 - mean)/std with
mean and std the fp32 values the kernel receives.  Per output index i of an axis of `in` source and `out` resized
elements: scale = in/out, support = taps/2 max(scale, 1), centre = scale (i + 0.5), first = max(floor(centre - support
+ 0.5), 0), n = min(floor(centre + support + 0.5), in) - first, w_j = filter((j - centre + 0.5) / max(scale, 1)) for
j in [first, first + n) (the triangle, or Keys' cubic with a = -0.5), normalised to sum 1.  The output (y, x) is the
resized (top + y, left + x): sum_y w_y sum_x w_x v.  `tests/test_preprocess_engine_cpu.py` pins this restatement to
torch's float64 antialiased interpolate within 1e-12.

The bound, u = 2^-24, per output element:

    |o - o64| <= C u [ (n_x + n_y + r_x + r_y) S + k_v S_v + E ],     C = 2, k_v = 3, u = 2^-24
    S   = sum_y sum_x |w_y| |w_x| |v64|             S_v = sum_y sum_x |w_y| |w_x| (|p/255| + |mean|) / |std|
    E   = sum_y sum_x (e_y |w_x| + |w_y| e_x) |v64|   over each window widened by one tap on both sides
    e   = (L (D_c + D_t) + k_f) / |tot|          r = (n (sum|w~| + L D_t + k_f) + V D_c) / |tot| + 1
    D_c = 2 |centre| / max(scale, 1)             D_t = (2 max_j |j - centre| + 1) / max(scale, 1) + 6

Derivation from the kernels' arithmetic (all four do the same operations per output element):
  * v: three IEEE operations.  fl(p/255) is off by u p/255, and p/255 - mean may cancel, so the error is taken
    relative to (|p/255| + |mean|)/|std|, not |v|: k_v = 3 of S_v.
  * The filter argument t = fl(fl(fl(j - centre) + 0.5) * scale_inv) with centre = fl(fl(in/out) (i + 0.5)) and
    scale_inv = fl(1/scale).  centre carries 2u|centre|, common to every tap of the window: u D_c in argument units.
    The subtraction and the + 0.5 add u|j - centre| and u|j - centre + 0.5|, and scale_inv and the product 3u|t| <= 6u:
    u D_t, different per tap.  D_c grows with the coordinate: a 16 384-wide source at scale ~1 has an absolute filter
    argument error near 2e-3, which moves a weight by as much.  A filter with Lipschitz constant L (1 for the
    triangle, 25/18 = 1.39 for Keys' a = -0.5) moves each weight by L times the argument error; evaluating the filter
    adds k_f = 16 u absolutely (Keys' polynomials reach magnitude 8 before their last subtraction).  After the
    division by the total tot (~ max(scale, 1)) every normalised weight is off by at most e u.  A tap that one side
    includes and the other does not sits at the edge of the support, where the filter is zero, so its weight is within
    e u of zero: the widened windows of E cover it and the window boundary needs no special case.
  * tot is a sum of n weights: n u sum|w~| of rounding and n (L D_t + k_f) u of per-tap weight errors.  The common
    shift moves tot by u D_c sum_j f'(t_j), a Riemann sum of f' whose integral is zero, so by at most V = the total
    variation of f' (4 for the triangle, 6.22 for Keys' cubic) times u D_c, not n times it.  With the division:
    r u |w| on every weight.
  * The horizontal fmaf chain over n_x taps and the vertical one over n_y rows (each with its own weights' r):
    (n_x + n_y) S.
  * C = 2 covers the second-order terms and the computed |w| in place of |w64|.

Cases: identity (bit-identical to anyloc_preprocess_u8) and identity on one axis, integer down-factors 2, 3, 7 and the
tap-window limits (31x bilinear, 15.5x bicubic), 1000 -> 480 and 640 -> 480, up-scaling 1x1 -> 14x14 and 3.7x,
5000 x 56 -> 14 x 56 (hundreds of vertical taps, many row chunks in the list kernel), 16 384-wide sources and the demo's
4032 x 3024 photo at max_side = 1024, the widest list tile (1023 source columns, R = 2 rows per chunk: the 64-tap
window keeps R = 1 out of reach), partial tiles, odd crop offsets,
all-0 / all-255 / 0-255 checkerboard pixels, std = 0.01 and mean = fl(128/255); the crop-only kernel with odd and even
Wc (scalar tail and float2 stores), Wc = 1, and B and Hc at 65 535.  The worst share of the bound per family is
printed at the end."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.util import dptr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C_PRE = 2.0
K_V = 3.0
K_F = 16.0
LIPSCHITZ = {0: 1.0, 1: 25.0 / 18.0}
TV_DF = {0: 4.0, 1: 6.25}                   # total variation of the filter's derivative (Keys a = -0.5: 6.22)
LEAD = 16                                   # NaN frame before and after every output (64 B keeps 16-byte alignment)
NAN32 = 0x7FC0DEAD                          # a quiet-NaN pattern no kernel writes
BILINEAR, BICUBIC = 0, 1
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
WORST = {}


# ------------------------------------------------------------------ the fp64 restatement (numpy, no torch)
def aa_filter64(t, cubic):
    t = np.abs(t)
    if not cubic:
        return np.where(t < 1.0, 1.0 - t, 0.0)
    a = -0.5
    return np.where(t < 1.0, ((a + 2.0) * t - (a + 3.0)) * t * t + 1.0,
                    np.where(t < 2.0, (((t - 5.0) * t + 8.0) * t - 4.0) * a, 0.0))


def axis64(in_size, out_size, cubic, idx):
    """Output indices idx of one axis -> (W [len(idx), in] normalised fp64 weights, Ew [len(idx), in] the absolute
    weight errors e on the widened windows, n [len(idx)] tap counts, r [len(idx)] relative weight errors), both
    matrices scipy CSR."""
    scale = in_size / out_size
    sm = max(scale, 1.0)
    support = (2.0 if cubic else 1.0) * sm
    rows, cols, vals, erows, ecols, evals = [], [], [], [], [], []
    n_taps, rel = np.zeros(len(idx)), np.zeros(len(idx))
    for r, i in enumerate(idx):
        centre = scale * (i + 0.5)
        first = max(math.floor(centre - support + 0.5), 0)
        last = min(math.floor(centre + support + 0.5), in_size)
        j = np.arange(first, last)
        w = aa_filter64((j - centre + 0.5) / sm, cubic)
        tot = w.sum()
        rows += [r] * len(j)
        cols += j.tolist()
        vals += (w / tot).tolist()
        d_c = 2 * abs(centre) / sm
        d_t = (2 * max(abs(first - centre), abs(last - centre)) + 1) / sm + 6
        e = (LIPSCHITZ[cubic] * (d_c + d_t) + K_F) / abs(tot)
        lo, hi = max(first - 1, 0), min(last + 1, in_size)
        erows += [r] * (hi - lo)
        ecols += list(range(lo, hi))
        evals += [e] * (hi - lo)
        n_taps[r] = last - first
        rel[r] = (n_taps[r] * (np.abs(w).sum() + LIPSCHITZ[cubic] * d_t + K_F) + TV_DF[cubic] * d_c) / abs(tot) + 1
    shape = (len(idx), in_size)
    return (sp.csr_matrix((vals, (rows, cols)), shape=shape), sp.csr_matrix((evals, (erows, ecols)), shape=shape),
            n_taps, rel)


def pixels64(img, mean, std):
    """uint8 [H, W, 3] -> (v64 [3, H, W], (|p/255| + |mean|)/|std| [3, H, W]) with mean, std taken as fp32"""
    p = img.astype(np.float64).transpose(2, 0, 1) / 255.0
    m = np.float32(mean).astype(np.float64)[:, None, None]
    s = np.float32(std).astype(np.float64)[:, None, None]
    return (p - m) / s, (np.abs(p) + np.abs(m)) / np.abs(s)


def _sep(Wy, Wx, X):
    """Wy X Wx^T, horizontal first: X [H, W] dense, Wy / Wx sparse"""
    return Wy @ np.asarray((Wx @ X.T).T)


def resize64(img, Hr, Wr, cubic, top, left, Hc, Wc, mean, std, with_bound=True):
    """uint8 [H, W, 3] -> (o64 [3, Hc, Wc], bound [3, Hc, Wc] in absolute units or None)"""
    H, W = img.shape[:2]
    v, vbar = pixels64(img, mean, std)
    Wy, Ey, ny, ry = axis64(H, Hr, cubic, np.arange(top, top + Hc))
    Wx, Ex, nx, rx = axis64(W, Wr, cubic, np.arange(left, left + Wc))
    o = np.stack([_sep(Wy, Wx, v[c]) for c in range(3)])
    if not with_bound:
        return o, None
    aWy, aWx = abs(Wy), abs(Wx)
    bound = []
    for c in range(3):
        av = np.abs(v[c])
        S = _sep(aWy, aWx, av)
        Sv = _sep(aWy, aWx, vbar[c])
        E = _sep(Ey, aWx, av) + _sep(aWy, Ex, av)
        coef = (ny + ry)[:, None] + (nx + rx)[None, :]
        bound.append(C_PRE * U * (coef * S + K_V * Sv + E))
    return o, np.stack(bound)


def crop32(img, top, left, Hc, Wc, mean, std):
    """anyloc_preprocess_u8's operations in IEEE fp32 (numpy rounds each one): [3, Hc, Wc]"""
    p = img[top:top + Hc, left:left + Wc].astype(np.float32).transpose(2, 0, 1)
    m = np.float32(mean)[:, None, None]
    s = np.float32(std)[:, None, None]
    return ((p / np.float32(255.0)) - m) / s


# ------------------------------------------------------------------ device side
@pytest.fixture(scope="module")
def L(cuda):
    from anyloc_b200 import _lib
    _lib.load()
    yield _lib
    if WORST:
        print("\n[worst |o - o64| / bound per kernel and family]")
        for (kern, fam), r in sorted(WORST.items()):
            print(f"  {kern:<14} {fam:<26} {r:.4f}")


def note(kern, fam, r):
    WORST[(kern, fam)] = max(WORST.get((kern, fam), 0.0), r)


def framed(n):
    buf = torch.full((n + 2 * LEAD,), NAN32, dtype=torch.int32, device="cuda")
    return buf


def frame_ok(buf):
    b = buf.cpu()
    return bool((b[:LEAD] == NAN32).all() and (b[-LEAD:] == NAN32).all())


def body(buf, shape):
    b = buf[LEAD:-LEAD]
    assert not bool((b == NAN32).any()), "an output element was not written"
    return b.view(torch.float32).view(shape).cpu().numpy()


def stats(mean, std):
    return (C.c_float * 3)(*mean), (C.c_float * 3)(*std)


def run_crop(L, imgs, top, left, Hc, Wc, mean, std):
    B, H, W = imgs.shape[:3]
    x = imgs.cuda()
    buf = framed(B * 3 * Hc * Wc)
    m3, s3 = stats(mean, std)
    L.check(L.load().anyloc_preprocess_u8(dptr(x), B, H, W, top, left, Hc, Wc, m3, s3, dptr(buf, LEAD),
                                          L.stream_ptr()), "preprocess_u8")
    assert frame_ok(buf)
    return body(buf, (B, 3, Hc, Wc))


def run_resize(L, imgs, Hr, Wr, cubic, top, left, Hc, Wc, mean, std):
    B, H, W = imgs.shape[:3]
    x = imgs.cuda()
    buf = framed(B * 3 * Hc * Wc)
    m3, s3 = stats(mean, std)
    L.check(L.load().anyloc_preprocess_resize_u8(dptr(x), B, H, W, Hr, Wr, cubic, top, left, Hc, Wc, m3, s3,
                                                 dptr(buf, LEAD), L.stream_ptr()), "preprocess_resize_u8")
    assert frame_ok(buf)
    return body(buf, (B, 3, Hc, Wc))


def run_list(L, imgs, geo, interp, mean, std, gap=4):
    """geo[i] = (Hr, Wr, top, left, Hc, Wc); each output starts `gap` floats after the previous one's end, the gaps
    NaN-framed too -> list of [3, Hc, Wc]"""
    n = len(imgs)
    xs = [im.cuda() for im in imgs]
    offs, o = [], LEAD
    for g in geo:
        offs.append(o)
        o += 3 * g[4] * g[5] + gap
    buf = framed(o - LEAD - gap)
    m3, s3 = stats(mean, std)

    def ints(vals):
        return (C.c_int * n)(*vals)
    rc = L.load().anyloc_preprocess_u8_varlen(
        n, (C.c_void_p * n)(*[x.data_ptr() for x in xs]), ints([x.shape[0] for x in xs]), ints([x.shape[1] for x in xs]),
        ints([g[0] for g in geo]), ints([g[1] for g in geo]), interp, ints([g[2] for g in geo]),
        ints([g[3] for g in geo]), ints([g[4] for g in geo]), ints([g[5] for g in geo]), m3, s3, dptr(buf),
        (C.c_int64 * n)(*offs), L.stream_ptr())
    L.check(rc, "preprocess_u8_varlen")
    b = buf.cpu()
    assert frame_ok(buf)
    written = torch.zeros(b.numel(), dtype=torch.bool)
    outs = []
    for off, g in zip(offs, geo):
        k = 3 * g[4] * g[5]
        seg = b[off:off + k]
        assert not bool((seg == NAN32).any()), "an output element was not written"
        written[off:off + k] = True
        outs.append(seg.view(torch.float32).view(3, g[4], g[5]).numpy())
    assert bool((b[~written] == NAN32).all()), "a write outside every image's output"
    return outs


def check_bound(kern, fam, out, o64, bound):
    err = np.abs(out.astype(np.float64) - o64)
    assert np.isfinite(out).all()
    ratio = float((err / bound).max())
    note(kern, fam, ratio)
    assert ratio <= 1.0, (kern, fam, ratio, np.unravel_index(np.argmax(err / bound), err.shape))
    return ratio


# ------------------------------------------------------------------ images
def random_img(H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)


def pattern_img(H, W, kind, seed=0):
    if kind == "zeros":
        return np.zeros((H, W, 3), np.uint8)
    if kind == "ones":
        return np.full((H, W, 3), 255, np.uint8)
    if kind == "checker":
        yy, xx = np.mgrid[:H, :W]
        return np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, axis=2)
    if kind == "smooth":
        yy, xx = np.mgrid[:H, :W]
        f = 127.5 + 120 * np.sin(xx / 37.0 + 0.3) * np.cos(yy / 23.0)
        return np.repeat(f.astype(np.uint8)[..., None], 3, axis=2)
    return random_img(H, W, seed)


def check_resize(L, fam, img, Hr, Wr, cubic, top=None, left=None, Hc=None, Wc=None, stats_=IMAGENET):
    """one image through the single-image resize kernel and the list kernel; both against the fp64 bound, and the
    list kernel's item bit-identical to the single-image kernel"""
    H, W = img.shape[:2]
    if Hc is None:
        top, left, Hc, Wc = (Hr - (Hr // 14) * 14) // 2, (Wr - (Wr // 14) * 14) // 2, (Hr // 14) * 14, (Wr // 14) * 14
        if Hc == 0 or Wc == 0:
            top, left, Hc, Wc = 0, 0, Hr, Wr
    mean, std = stats_
    o64, bound = resize64(img, Hr, Wr, cubic, top, left, Hc, Wc, mean, std)
    out = run_resize(L, torch.from_numpy(img)[None], Hr, Wr, cubic, top, left, Hc, Wc, mean, std)[0]
    check_bound("resize", fam, out, o64, bound)
    (lst,) = run_list(L, [torch.from_numpy(img)], [(Hr, Wr, top, left, Hc, Wc)], cubic, mean, std)
    check_bound("list_resize", fam, lst, o64, bound)
    assert np.array_equal(lst.view(np.uint32), out.view(np.uint32)), fam
    return out


MODES = pytest.mark.parametrize("cubic", [BILINEAR, BICUBIC], ids=["bilinear", "bicubic"])


@MODES
def test_identity_is_the_crop_kernel(L, cubic):
    """scale exactly 1: both filters give weights exactly 1 and 0, so the resize is the crop-only result bit for bit"""
    for H, W, top, left, Hc, Wc in ((37, 53, 0, 0, 37, 53), (64, 96, 3, 5, 57, 77), (14, 14, 0, 0, 14, 14)):
        img = random_img(H, W, H * W)
        crop = run_crop(L, torch.from_numpy(img)[None], top, left, Hc, Wc, *IMAGENET)[0]
        res = run_resize(L, torch.from_numpy(img)[None], H, W, cubic, top, left, Hc, Wc, *IMAGENET)[0]
        (lst,) = run_list(L, [torch.from_numpy(img)], [(H, W, top, left, Hc, Wc)], cubic, *IMAGENET)
        assert np.array_equal(res.view(np.uint32), crop.view(np.uint32))
        assert np.array_equal(lst.view(np.uint32), crop.view(np.uint32))
        assert np.array_equal(crop.view(np.uint32), crop32(img, top, left, Hc, Wc, *IMAGENET).view(np.uint32))


@MODES
def test_identity_on_one_axis(L, cubic):
    img = random_img(70, 90, 11)
    check_resize(L, "one-axis identity", img, 70, 33, cubic, 0, 0, 70, 33)
    check_resize(L, "one-axis identity", img, 29, 90, cubic, 0, 0, 29, 90)
    check_resize(L, "one-axis identity", img, 70, 251, cubic, 1, 3, 69, 247)


@MODES
@pytest.mark.parametrize("f", [2, 3, 7])
def test_integer_down_factors(L, cubic, f):
    img = random_img(14 * 9 * f + f, 14 * 11 * f, f)
    check_resize(L, f"down {f}x", img, img.shape[0] // f, img.shape[1] // f, cubic)


@MODES
def test_tap_window_limit(L, cubic):
    """31x bilinear / 15.5x bicubic horizontally: 2 * 31 + 2 = 4 * 15.5 + 2 = 64 taps"""
    f = 31.0 if cubic == BILINEAR else 15.5
    Wr = 28
    W = int(Wr * f)
    img = random_img(60, W, 31)
    check_resize(L, "tap-window limit", img, 30, Wr, cubic)


@MODES
@pytest.mark.parametrize("src,dst", [((1000, 1000), (480, 480)), ((480, 640), (480, 480)), ((750, 1000), (480, 640))])
def test_non_integer_factors(L, cubic, src, dst):
    img = random_img(*src, seed=src[0] + dst[1])
    check_resize(L, "non-integer", img, *dst, cubic)


@MODES
def test_up_scaling(L, cubic):
    one = random_img(1, 1, 5)
    out = check_resize(L, "up", one, 14, 14, cubic)
    assert np.array_equal(out.view(np.uint32), np.broadcast_to(crop32(one, 0, 0, 1, 1, *IMAGENET), out.shape)
                          .view(np.uint32))                 # one tap of weight 1
    check_resize(L, "up", random_img(30, 40, 6), 111, 148, cubic)      # 3.7x


@MODES
def test_extreme_vertical_down_scaling(L, cubic):
    """5000 x 56 -> 14 x 56: ~714 (bilinear) / ~1430 (bicubic) vertical taps, and about 200 (bilinear) / 250 (bicubic)
    16-row chunks in the list kernel's first tile"""
    img = random_img(5000, 56, 7)
    check_resize(L, "vertical 357x", img, 14, 56, cubic)
    check_resize(L, "vertical 357x", pattern_img(5000, 56, "checker"), 14, 56, cubic)


@MODES
def test_large_coordinates(L, cubic):
    """16 384-wide sources, where the fp32 centre's error grows to ~2u * 16 384, and the demo's 4032 x 3024 photo at
    max_side = 1024 (-> 1024 x 768)"""
    img = random_img(42, 16384, 8)
    check_resize(L, "16384 wide", img, 28, 16000, cubic, 0, 15000, 28, 1000)   # scale ~1, the far end
    check_resize(L, "16384 wide", img, 28, 1400, cubic)                          # 11.7x down
    check_resize(L, "16384 wide", pattern_img(42, 16384, "smooth"), 42, 16380, cubic, 0, 16000, 42, 380)
    photo = pattern_img(4032, 3024, "smooth")
    photo[::3, ::5] = random_img(1344, 605, 9)
    check_resize(L, "4032x3024 max_side", photo, 1024, 768, cubic)


def _span32(i, in_size, out_size, cubic):
    """aa_span_rn in IEEE fp32 -> (first, n)"""
    f = np.float32
    scale = f(in_size) / f(out_size)
    support = f(2.0 if cubic else 1.0) * (scale if scale >= 1 else f(1.0))
    centre = scale * (f(i) + f(0.5))
    first = max(int((centre - support) + f(0.5)), 0)
    return first, min(int((centre + support) + f(0.5)), in_size) - first


def test_list_widest_column_span(L):
    """the widest source-column span a list tile can read.  R = min(16, 6144 // (3 ncols)) source rows per chunk; the
    host's 64-tap window keeps ncols <= 1023 (a 31x bilinear tile: 33 * 31 columns), so the fewest rows per chunk is
    R = 2 -- R = 1 would need ncols > 1024, which no accepted shape reaches.  W = 2014 -> Wr = 65 makes tile 1 read
    1023 columns."""
    W, Wr = 2014, 65
    f0, _ = _span32(32, W, Wr, 0)
    f1, n1 = _span32(63, W, Wr, 0)
    ncols = f1 + n1 - f0
    assert ncols == 1023 and min(16, 6144 // (3 * ncols)) == 2, ncols
    check_resize(L, "list R = 2", random_img(45, W, 12), 40, Wr, BILINEAR, 0, 0, 40, Wr)
    check_resize(L, "list R = 2", pattern_img(45, W, "checker"), 17, Wr, BILINEAR, 0, 0, 17, Wr)


@MODES
def test_partial_tiles_and_odd_offsets(L, cubic):
    img = random_img(301, 403, 13)
    check_resize(L, "partial tiles", img, 157, 211, cubic, 3, 5, 150, 199)         # Hc % 8 = 6, Wc % 32 = 7
    check_resize(L, "partial tiles", img, 77, 97, cubic, 1, 1, 75, 33)             # Wc % 32 = 1, Hc % 8 = 3


@MODES
@pytest.mark.parametrize("kind", ["zeros", "ones", "checker"])
def test_pixel_patterns(L, cubic, kind):
    """the 0/255 checkerboard is the cancelling case: every window sums values of both signs"""
    img = pattern_img(211, 307, kind)
    check_resize(L, kind, img, 100, 140, cubic)
    check_resize(L, kind, img, 72, 99, cubic, 1, 3, 70, 95)


@MODES
def test_statistics(L, cubic):
    half = float(np.float32(128 / 255))
    for name, st in (("std 0.01", ((0.485, 0.456, 0.406), (0.01, 0.01, 0.01))),
                     ("mean fl(128/255)", ((half, half, half), (0.229, 0.224, 0.225))),
                     ("both", ((half, 0.0, 1.0), (0.01, 0.5, 3.0)))):
        for kind in ("random", "checker"):
            img = pattern_img(180, 260, kind, seed=14)
            check_resize(L, name, img, 85, 120, cubic, stats_=st)
            img[...] = 128
            img[::2, ::3] = 127
            check_resize(L, name + " near mean", img, 85, 120, cubic, stats_=st)


def check_crop(L, fam, imgs, top, left, Hc, Wc, st=IMAGENET):
    out = run_crop(L, torch.from_numpy(imgs), top, left, Hc, Wc, *st)
    for b in range(imgs.shape[0]) if imgs.shape[0] <= 4 else (0, imgs.shape[0] // 2, imgs.shape[0] - 1):
        exp = crop32(imgs[b], top, left, Hc, Wc, *st)
        assert np.array_equal(out[b].view(np.uint32), exp.view(np.uint32)), (fam, b)
        v, vbar = pixels64(imgs[b, top:top + Hc, left:left + Wc], *st)
        check_bound("crop", fam, out[b], v, C_PRE * U * K_V * vbar)
    return out


def test_crop_kernel(L):
    for Wc in (1, 2, 27, 28, 511, 512, 513):
        imgs = np.stack([random_img(31, 520, 15 + b) for b in range(2)])
        check_crop(L, "odd/even Wc", imgs, 1, 3, 29, Wc)
    imgs = np.stack([pattern_img(40, 50, k) for k in ("zeros", "ones", "checker")])
    check_crop(L, "patterns", imgs, 0, 1, 40, 49)
    check_crop(L, "std 0.01", imgs, 0, 0, 40, 50, ((0.485, 0.456, 0.406), (0.01, 0.01, 0.01)))
    # the list form: bit-identical to the crop kernel per image
    lst_imgs = [random_img(h, w, h + w) for h, w in ((31, 520), (1, 1), (14, 3), (300, 33))]
    geo = [(0, 0, 1, 3, 29, 27), (0, 0, 0, 0, 1, 1), (0, 0, 0, 1, 14, 2), (0, 0, 7, 0, 290, 33)]
    outs = run_list(L, [torch.from_numpy(i) for i in lst_imgs], geo, -1, *IMAGENET)
    for img, g, o in zip(lst_imgs, geo, outs):
        exp = crop32(img, g[2], g[3], g[4], g[5], *IMAGENET)
        assert np.array_equal(o.view(np.uint32), exp.view(np.uint32)), g
        v, vbar = pixels64(img[g[2]:g[2] + g[4], g[3]:g[3] + g[5]], *IMAGENET)
        check_bound("list_crop", "list", o, v, C_PRE * U * K_V * vbar)


def test_crop_kernel_grid_limits(L):
    """B = 65 535 one-pixel images, and Hc = 65 535 rows (odd and even Wc)"""
    imgs = np.random.default_rng(16).integers(0, 256, (65535, 1, 2, 3), dtype=np.uint8)
    out = run_crop(L, torch.from_numpy(imgs), 0, 1, 1, 1, *IMAGENET)
    exp = ((imgs[:, 0, 1].astype(np.float32) / np.float32(255)) - np.float32(IMAGENET[0])) / np.float32(IMAGENET[1])
    assert np.array_equal(out[:, :, 0, 0].view(np.uint32), exp.view(np.uint32))
    tall = random_img(65535, 3, 17)[None]
    for Wc in (1, 2):
        check_crop(L, "Hc 65535", tall, 0, 1, 65535, Wc)


def test_list_many_images(L):
    """one list call over every interpolation, with images that need a second launch (> 64 images)"""
    rng = np.random.default_rng(18)
    sizes = [(int(h), int(w)) for h, w in rng.integers(14, 90, size=(70, 2))]
    imgs = [random_img(h, w, k) for k, (h, w) in enumerate(sizes)]
    for cubic in (BILINEAR, BICUBIC):
        geo = [(28, 42, 0, 0, 28, 42) if k % 2 else (h // 2 + 1, w // 3 + 1, 1, 0, h // 2, w // 3)
               for k, (h, w) in enumerate(sizes)]
        outs = run_list(L, [torch.from_numpy(i) for i in imgs], geo, cubic, *IMAGENET)
        for img, g, o in zip(imgs, geo, outs):
            o64, bound = resize64(img, g[0], g[1], cubic, g[2], g[3], g[4], g[5], *IMAGENET)
            check_bound("list_resize", "70 images", o, o64, bound)
