"""Drop-in mirror of the hot-path API of AnyLoc's `utilities.py`
(/root/reference/utilities.py): `DinoV2ExtractFeatures` (:219-288), `VLAD` (:624-1008),
`get_top_k_recall` (:390-469) plus the pass-through helpers the callers import from the same
module (`seed_everything` :505-519, `reduce_pca` :522-586, `CustomDataset` :25-74, `to_np`
:79-97).  Same names, argument meaning and error behaviour; the arithmetic runs in hand-written
sm_90a kernels behind the C ABI of include/anyloc_b200.h.  CUDA only -- no CPU fallback.

Put `<repo>/anyloc_b200/dropin` first on PYTHONPATH to make `from utilities import ...` in the
reference's scripts (scripts/dino_v2_vlad.py:37-38,50) resolve here (see INTEGRATION.md).
"""
import ctypes as C
import math
import os
import random
from typing import List, Literal, Tuple, Union

import numpy as np
import torch

from . import _lib
from . import vit as _vit

_DINO_V2_MODELS = Literal["dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14",
                          "dinov2_vits14_reg", "dinov2_vitb14_reg", "dinov2_vitl14_reg", "dinov2_vitg14_reg"]
_DINO_FACETS = Literal["query", "key", "value", "token"]


# ------------------------------------------------------------------ helpers (pass-through)
class CustomDataset:
    """Abstract parent of the reference's custom datasets (utilities.py:25-74)."""

    def __init__(self) -> None:
        self.database_num = None
        self.queries_num = None
        self.soft_positives_per_query = None

    def get_image_paths(self):
        if hasattr(self, "images_paths"):
            return self.images_paths
        raise NotImplementedError("Not handled!")

    def get_positives(self):
        if hasattr(self, "soft_positives_per_query"):
            return self.soft_positives_per_query
        raise NotImplementedError("Not handled!")

    def get_image_relpaths(self, i: Union[int, List[int]]) -> Union[List[str], str]:
        single = type(i) == int
        paths = self.get_image_paths()
        depth = getattr(self, "_imgs_level", 2)
        rel = ["/".join(paths[k].split("/")[-depth:]) for k in ([i] if single else i)]
        return rel[0] if single else rel

    def __getitem__(self, index):
        raise NotImplementedError("Not created!")

    def __len__(self):
        if hasattr(self, "images_paths"):
            return len(self.get_image_paths())
        raise NotImplementedError("Not handled!")


def to_np(x, ret_type=float) -> np.ndarray:
    """utilities.py:79-97."""
    arr = x.detach().cpu().numpy() if type(x) == torch.Tensor else np.array(x)
    return arr.astype(ret_type)


def to_pil_list(x):
    """utilities.py:99-129: an image / batch ([B,C,H,W], [B,H,W,C], [C,H,W] or [H,W,C]) -> list of PIL images, each
    min-max normalised to 0..255.  Host-side helper (visualisation), not on the accelerated path."""
    from PIL import Image
    if type(x) == Image.Image or (type(x) == list and type(x[0]) == Image.Image):
        return x
    x = to_np(x)
    if len(x.shape) == 3:
        x = x[np.newaxis, ...]
    out = []
    for img in x:
        if img.shape[0] in [1, 3]:
            img = img.transpose(1, 2, 0)
        norm = (img - img.min()) / (img.max() - img.min())
        out.append(Image.fromarray((norm * 255).astype(np.uint8)))
    return out


def pad_img(img: np.ndarray, padding: int, color: tuple = (0, 0, 0)) -> np.ndarray:
    """utilities.py:474-500: [H,W,3] -> [H+2P, W+2P, 3] with an RGB border.  Host-side helper."""
    if type(color) == list:
        color = tuple(color)
    assert len(color) == 3, "Color should be (R, G, B) value"
    ret = np.ones((img.shape[0] + 2 * padding, img.shape[1] + 2 * padding, 3), np.uint8) * np.array(color)
    ret[padding:-padding, padding:-padding] = img
    return ret.astype(img.dtype)


def concat_desc_dists_clusters(cluster_centers: torch.Tensor, descs: torch.Tensor) -> torch.Tensor:
    """utilities.py:590-619: per descriptor, the unit residuals to every centre, concatenated and L2-normalised
    ([n, k*d]).  Plain tensor algebra on the caller's device, as in the reference (not on the hot path)."""
    assert type(cluster_centers) == type(descs) == torch.Tensor
    d = descs[:, None, :] - cluster_centers[None, ...]
    d = d / d.norm(dim=-1, keepdim=True)
    cat = d.reshape(d.shape[0], -1)
    return cat / cat.norm(dim=-1, keepdim=True)


def seed_everything(seed=42):
    """utilities.py:505-519."""
    random.seed(seed)
    os.environ["PYTHONHASHSEED"] = str(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    print(f"Seed set to: {seed} (type: {type(seed)})")


def _gemm_nt_dev(a, b, bias=None):
    """C = a @ b.T (+ bias) in fp32-equivalent precision on the tensor-core engine (anyloc_gemm_nt, tf32 (hi,lo) pairs);
    a [M,K], b [N,K] device fp32, K padded to a multiple of 4 with zeros."""
    lib = _lib.load()
    pad = (-a.shape[1]) % 4
    if pad:
        a, b = torch.nn.functional.pad(a, (0, pad)), torch.nn.functional.pad(b, (0, pad))
    a, b = a.contiguous(), b.contiguous()
    M, K = a.shape
    N = b.shape[0]
    out = torch.empty(M, N, device=a.device, dtype=torch.float32)
    with torch.cuda.device(a.device):
        pairs = []
        for t in (a, b):
            hi, lo = torch.empty_like(t), torch.empty_like(t)
            _lib.check(lib.anyloc_split_tf32(_lib.ptr(t), _lib.ptr(hi), _lib.ptr(lo), t.numel(), _lib.stream_ptr()),
                       "anyloc_split_tf32")
            pairs += [hi, lo]
        rc = lib.anyloc_gemm_nt(_lib.ptr(pairs[0]), _lib.ptr(pairs[1]), K, _lib.ptr(pairs[2]), _lib.ptr(pairs[3]), K,
                                M, N, K, _lib.PAIR["tf32"], C.c_float(1.0), _lib.EPI["bias"], _lib.ptr(bias), None, None,
                                _lib.ptr(out), None, N, _lib.PAIR["tf32"], _lib.ENGINE["auto"], _lib.stream_ptr())
    _lib.check(rc, "anyloc_gemm_nt")
    return out


def _flip_signs(vt):
    """The signs of sklearn's `svd_flip(u_based_decision=False)`: each row of vt times the sign of its largest-magnitude
    element (+1 for a zero row) -> [k, 1]"""
    sign = torch.sign(torch.gather(vt, 1, vt.abs().argmax(dim=1, keepdim=True)))
    sign[sign == 0] = 1
    return sign


def _lu_pl(y):
    """P L of the partial-pivoting LU y = P L U, the normaliser `scipy.linalg.lu(y, permute_l=True)[0]` that sklearn's
    randomized range finder applies after each half-step: [m, min(m, w)] for y [m, w].  P is applied as a row
    permutation, never formed."""
    if y.is_cuda:
        # torch's default backend runs MAGMA's batched getrf on one tall matrix: slower than cuSOLVER, and it prints
        # a warning on every call
        prev = torch.backends.cuda.preferred_linalg_library()
        torch.backends.cuda.preferred_linalg_library("cusolver")
        try:
            lu, piv = torch.linalg.lu_factor(y)
        finally:
            torch.backends.cuda.preferred_linalg_library(prev)
    else:
        lu, piv = torch.linalg.lu_factor(y)
    m, r = lu.shape[0], min(lu.shape)
    lo = lu[:, :r].tril(-1)
    lo.diagonal().fill_(1.0)
    perm = np.arange(m)
    for i, p in enumerate(piv.cpu().numpy() - 1):     # LAPACK's row interchanges, in order: y[perm] = L U
        perm[[i, p]] = perm[[p, i]]
    out = torch.empty(m, r, dtype=y.dtype, device=y.device)
    out[torch.from_numpy(perm).to(y.device)] = lo
    return out


class _PcaDev:
    """`sklearn.decomposition.PCA(k, svd_solver="full", whiten=...)` as reduce_pca uses it (utilities.py:560-586), on
    the GPU: the fit is a one-off fp64 eigen-decomposition of the smaller Gram / covariance matrix (torch.linalg.eigh,
    i.e. cuSOLVER: plumbing), the projections -- the part that touches every descriptor -- run as GEMMs on this
    library's tensor-core engine.  Component signs follow sklearn's `svd_flip(u_based_decision=False)`."""

    def __init__(self, n_components, whiten=False):
        self.n_components, self.whiten = int(n_components), bool(whiten)

    def fit(self, x):
        n, d = x.shape
        k = self.n_components
        if not 0 <= k <= min(n, d):
            raise ValueError(f"n_components={k} must be between 0 and min(n_samples, n_features)={min(n, d)} with "
                             "svd_solver='full'")
        return self.fit_shared(_pca_decompose(x))

    def fit_shared(self, eig):
        """fit() from _pca_decompose of the rows, the part of the fit that does not depend on k"""
        mean, xd, s, vec, n = eig
        k = self.n_components
        self.mean_ = mean
        if xd is not None:
            vt = (vec[:, :k].T @ xd) / s[:k, None].clamp_min(1e-300)
        else:
            vt = vec[:, :k].T.contiguous()
        return self._set_components(vt, s, n)

    def _set_components(self, vt, s, n):
        k = self.n_components
        sign = _flip_signs(vt)
        self.components_ = (vt * sign).float().contiguous()
        self.singular_values_ = s[:k].float()
        self.explained_variance_ = (s[:k] ** 2 / (n - 1)).float()
        self.all_singular_values_ = s
        return self

    def fit_streamed(self, rows, plan, dev):
        """fit() on rows (a _PcaRows) fed to the device piece by piece (_pca_plan, _pca_boxes), so that only the m x m
        fp64 matrix, its eigen-decomposition and k x d vectors live there.  Covariance route (n > d): one pass over row
        pieces for the mean, one accumulating C = Xc^T Xc.  Gram route (n <= d): one pass over column slabs of all n
        rows, each giving its columns' mean and its part of G = Xc Xc^T, then a second one for vt = u[:, :k]^T Xc / s.
        The sums are anyloc_pca_colsum / anyloc_pca_accumulate, fp64 on the FP64 tensor cores, centring in registers."""
        n, d = rows.shape
        k = self.n_components
        if not 0 <= k <= min(n, d):
            raise ValueError(f"n_components={k} must be between 0 and min(n_samples, n_features)={min(n, d)} with "
                             "svd_solver='full'")
        return _pca_fit_streamed_dims(rows, plan, [self], dev)[0]

    def fit_randomized(self, rows, w, P, dev):
        """`sklearn.decomposition.PCA(k, svd_solver="randomized")`'s fit with its default parameters (_randomized_svd:
        n_oversamples=10, n_iter="auto", LU-normalised power iterations, transpose="auto"), step for step, on rows (a
        _PcaRows) read in row pieces of P.  w is the test matrix (_pca_test_matrix).  With A = Xc, or Xc^T when
        n < d: n_iter times Q = PL(A Q), Q = PL(A^T Q); then Q = qr(A Q), B = Q^T A = U^ S Vt, U = Q U^.  Every product
        with A is one pass over the rows (anyloc_pca_accumulate "sketch": Xc W, "vt": W^T Xc), fp64 on the FP64 tensor
        cores; LU, QR and SVD are fp64 torch.linalg (cuSOLVER) on the [max(n, d), l] and [min(n, d), l] matrices.
        Also sets fit_rows_: what sklearn's fit_transform returns for the rows, U S (U sqrt(n - 1) when whitening)."""
        n, d = rows.shape
        k = self.n_components
        if not 1 <= k <= min(n, d):
            raise ValueError(f"n_components={k} must be between 1 and min(n_samples, n_features)={min(n, d)} with "
                             "svd_solver='randomized'")
        return _pca_randomized_group(rows, [self], [w], P, dev)[0]

    def transform(self, x):
        y = _gemm_nt_dev(x - self.mean_, self.components_)
        if self.whiten:
            scale = self.explained_variance_.sqrt()
            scale[scale < torch.finfo(scale.dtype).eps] = torch.finfo(scale.dtype).eps
            y = y / scale
        return y


def _pca_decompose(x):
    """The part of _PcaDev.fit on device fp32 rows x [n, d] that does not depend on k: the mean, and the eigenvectors and
    singular values (largest first) of the fp64 Gram (n <= d) or covariance matrix of the centred rows -> (mean, xd,
    s, vec, n).  xd, the centred fp64 rows, is kept for the Gram route's vt only, else None."""
    n, d = x.shape
    mean = x.mean(dim=0)
    xd = (x - mean).double()
    ev, vec = torch.linalg.eigh(xd @ xd.T if n <= d else xd.T @ xd)
    ev, vec = ev.flip(0).clamp_min(0), vec.flip(1)
    return mean, (xd if n <= d else None), ev.sqrt(), vec, n


def _pca_fit_streamed_dims(rows, plan, pcas, dev):
    """_PcaDev.fit_streamed of every _PcaDev in `pcas` on the same rows (a _PcaRows): one mean pass, one accumulation
    of the m x m matrix, one mirror and one eigh for all of them.  On the Gram route the vt pass stages each column slab
    once and accumulates every member's u[:, :k]^T Xc on it, each at its own k -> pcas"""
    n, d = rows.shape
    m = min(n, d)
    boxes = _pca_boxes(n, d, plan)
    with torch.cuda.device(dev):
        mu = torch.zeros(d, dtype=torch.float64, device=dev)
        a = torch.zeros(m, m, dtype=torch.float64, device=dev)
        if n > d:
            for x in _pca_staged(rows, boxes, dev):
                _pca_colsum(x, mu)
            mu /= n
            for x in _pca_staged(rows, boxes, dev):
                _pca_accumulate("cov", x, mu, a)
        else:
            for (_, _, c0, c1), x in zip(boxes, _pca_staged(rows, boxes, dev)):
                _pca_colsum(x, mu[c0:c1])
                mu[c0:c1] /= n
                _pca_accumulate("gram", x, mu[c0:c1], a)
        _lib.check(_lib.load().anyloc_pca_mirror(_lib.ptr(a), m, m, _lib.stream_ptr()), "anyloc_pca_mirror")
        ev, vec = torch.linalg.eigh(a)
        del a
        ev, vec = ev.flip(0).clamp_min(0), vec.flip(1)
        s = ev.sqrt()
        if n <= d:
            us = [vec[:, :p.n_components].contiguous() for p in pcas]
            del vec
            vts = [torch.zeros(u.shape[1], d, dtype=torch.float64, device=dev) for u in us]
            for (_, _, c0, c1), x in zip(boxes, _pca_staged(rows, boxes, dev)):
                for u, vt in zip(us, vts):
                    _pca_accumulate("vt", x, mu[c0:c1], vt[:, c0:c1], u)
            for vt in vts:
                vt /= s[:vt.shape[0], None].clamp_min(1e-300)
        else:
            vts = [vec[:, :p.n_components].T.contiguous() for p in pcas]
        for p, vt in zip(pcas, vts):
            p.mean_ = mu.float()
            p._set_components(vt, s, n)
    return pcas


def _pca_randomized_schedule(n, d, ks):
    """The row passes of randomized fits of n x d rows at every k of ks run together (_pca_randomized_group), in order:
    [(forward, [(member, then)])].  forward: the pass multiplies by A (Xc, or Xc^T when n < d), else by A^T; the
    transpose depends on n < d only, so a pass has one direction for every member.  then: what the member does with
    its product -- "lu" (a power iteration's normaliser), "qr" (the range's basis Q) or "svd" (B = Q^T A and its
    decomposition, the member's last pass).  Members with n_iter = 4 leave after pass 9, those with 7 after pass 15."""
    steps = [2 * _pca_randomized_params(n, d, k)[1] + 2 for k in ks]
    return [(p % 2 == 0, [(i, "lu" if p < s - 2 else "qr" if p == s - 2 else "svd")
                          for i, s in enumerate(steps) if p < s]) for p in range(max(steps))]


def _pca_randomized_group(rows, pcas, ws, P, dev):
    """_PcaDev.fit_randomized of every _PcaDev in `pcas` (test matrix ws[i]) on the same rows (a _PcaRows) read in row
    pieces of P: one mean pass, then the passes of _pca_randomized_schedule.  Each pass stages every row piece once and
    runs the sketch or vt accumulate of every member still running on it -> pcas"""
    n, d = rows.shape
    transpose = n < d
    boxes = _pca_boxes(n, d, ("cov", P))
    with torch.cuda.device(dev):
        mu = torch.zeros(d, dtype=torch.float64, device=dev)
        for x in _pca_staged(rows, boxes, dev):
            _pca_colsum(x, mu)
        mu /= n

        def one_pass(forward, qs):
            """Xc q ([n, width], "sketch") or Xc^T q ([d, width], summed over the row pieces) of every q"""
            sketch = forward != transpose
            qs = [q.contiguous() for q in qs]
            outs = [torch.zeros(*((n, q.shape[1]) if sketch else (q.shape[1], d)), dtype=torch.float64, device=dev)
                    for q in qs]
            for (r0, r1, _, _), x in zip(boxes, _pca_staged(rows, boxes, dev)):
                for q, out in zip(qs, outs):
                    if sketch:
                        _pca_accumulate("sketch", x, mu, out[r0:r1], q)
                    else:
                        _pca_accumulate("vt", x, mu, out, q[r0:r1])
            return outs if sketch else [out.T for out in outs]

        qs = [torch.from_numpy(w).to(device=dev, dtype=torch.float64) for w in ws]
        for forward, live in _pca_randomized_schedule(n, d, [p.n_components for p in pcas]):
            for (i, then), y in zip(live, one_pass(forward, [qs[i] for i, _ in live])):
                if then == "lu":
                    qs[i] = _lu_pl(y)
                elif then == "qr":
                    qs[i] = torch.linalg.qr(y).Q
                else:
                    _pca_randomized_finish(pcas[i], qs[i], y, mu, n, transpose)
                    qs[i] = None
    return pcas


def _pca_randomized_finish(pca, q, y, mu, n, transpose):
    """The end of a randomized fit from Q and y = A^T Q: the SVD of B = Q^T A [l, min(n, d)] through the QR of
    B^T = Q2 R: B = R^T Q2^T, R^T = U^ S W^T"""
    k = pca.n_components
    q2, r = torch.linalg.qr(y)
    uh, s, wt = torch.linalg.svd(r.T)
    vt = wt @ q2.T
    uq = q @ uh
    del q, q2
    u_rows, vt = (vt[:k].T, uq[:, :k].T) if transpose else (uq[:, :k], vt[:k])
    sign = _flip_signs(vt)
    scale = math.sqrt(n - 1) if pca.whiten else s[:k]
    pca.fit_rows_ = (u_rows * (sign.T * scale)).float()
    pca.mean_ = mu.float()
    pca._set_components(vt.contiguous(), s, n)


def reduce_pca(train_descs: np.ndarray, test_descs: np.ndarray, lower_dim: int, low_factor: float = 0.0,
               fallback: int = 256, svd_solver: str = "full", whitening: bool = False) \
        -> Tuple[np.ndarray, np.ndarray]:
    """PCA projection fitted on the training set (utilities.py:522-586; scripts/dino_v2_vlad.py:357-369 reduces the
    database / query VLADs with it).  Same arguments and return types (numpy in -> numpy out, torch tensors accepted);
    the arithmetic runs on the GPU -- see _PcaDev.  svd_solver="randomized" is sklearn's randomized PCA with its
    defaults, step for step and from the same draw of numpy's global generator (_reduce_pca_randomized); it has no
    limit on min(n_samples, n_features).  Every other `svd_solver` gives the exact ("full") decomposition.

    When the in-memory fit would not fit the device (_pca_plan), the rows stream through it instead
    (_reduce_pca_streamed); when not even the m x m matrix (m = min(n_samples, n_features)) and its eigen-decomposition
    fit, MemoryError."""
    assert 0 <= low_factor <= 1
    as_np = type(train_descs) == np.ndarray
    dev = _lib.require_cuda(None)
    (n, d), n_te = train_descs.shape, test_descs.shape[0]
    if svd_solver == "randomized" and (low_factor == 0.0 or n < d):
        tr, te = _reduce_pca_randomized(train_descs, test_descs, lower_dim, low_factor, fallback, whitening, dev)
        return (tr.numpy(), te.numpy()) if as_np else (tr, te)
    if svd_solver == "randomized":
        # a randomized fit of all min(n, d) components spans the whole space, i.e. is the exact fit; sklearn's still
        # draws its test matrix from numpy's global generator, so draw it too and leave that generator where it does
        out = reduce_pca(train_descs, test_descs, lower_dim, low_factor, fallback, "full", whitening)
        _pca_skip_test_matrix(n, d, d)
        return out
    n_fit, n_held = (n + n_te, n + n_te) if low_factor != 0.0 and n < d else (n, n_te)     # fallback: cat(tr, te)
    plan = _pca_plan(n_fit, d, n_held, _device_budget(dev), _STAGE_BYTES)       # the first fit's
    if plan is not None:
        tr, te = _reduce_pca_streamed(train_descs, test_descs, lower_dim, low_factor, fallback, whitening, plan, dev)
        return (tr.numpy(), te.numpy()) if as_np else (tr, te)
    tr, te = _as_device_f32(train_descs, dev), _as_device_f32(test_descs, dev)

    def ret(a, b):
        return (a.cpu().numpy(), b.cpu().numpy()) if as_np else (a.cpu(), b.cpu())

    if low_factor == 0.0:
        pca = _PcaDev(lower_dim, whiten=whitening).fit(tr)
        return ret(pca.transform(tr), pca.transform(te))
    n_samples, n_components = tr.shape
    if n_samples < n_components:
        print(f"Too few samples, fallback to {fallback}d first")
        both = torch.cat((tr, te))
        both = _PcaDev(fallback).fit(both).transform(both)
        tr, te = both[:n_samples].contiguous(), both[n_samples:].contiguous()
    n_low = int(low_factor * lower_dim)
    n_top = lower_dim - n_low
    print(f"Up: {n_top}, Down: {n_low}")
    pca = _PcaDev(tr.shape[1]).fit(tr)
    basis = torch.cat((pca.components_[:n_top], pca.components_[-n_low:])).contiguous()
    return ret(_gemm_nt_dev(tr - pca.mean_, basis), _gemm_nt_dev(te - pca.mean_, basis))


class _PcaRows:
    """The rows of one or more [n_i, d] matrices stacked -- reduce_pca's training rows, or its training and test rows
    for the `fallback` pre-reduction -- as numpy arrays or tensors of any dtype and strides, on the host or a device.
    Read box by box; no input is ever copied whole, converted whole or pinned."""

    def __init__(self, parts):
        self.parts = [torch.from_numpy(p) if type(p) == np.ndarray else p.detach() for p in parts]
        self.shape = (sum(p.shape[0] for p in self.parts), self.parts[0].shape[1])
        self.is_cuda = all(p.is_cuda for p in self.parts)

    def _slices(self, r0, r1, c0, c1):
        o = 0
        for p in self.parts:
            a, b = max(r0 - o, 0), min(r1 - o, p.shape[0])
            if a < b:
                yield p[a:b, c0:c1]
            o += p.shape[0]

    def gather(self, dst, box):
        """rows[r0:r1, c0:c1] -> the host fp32 matrix dst"""
        o = 0
        for s in self._slices(*box):
            dst[o:o + s.shape[0]].copy_(s)
            o += s.shape[0]

    def on_device(self, box, dev):
        """rows[r0:r1, c0:c1] as a device fp32 matrix with unit column stride: a view of the input where it is one
        already, else a converted copy of the box"""
        s = list(self._slices(*box))
        if (len(s) == 1 and s[0].device == dev and s[0].dtype == torch.float32 and s[0].stride(1) == 1 and
                s[0].stride(0) >= s[0].shape[1]):
            return s[0]
        return torch.cat([t.to(device=dev, dtype=torch.float32) for t in s]).contiguous()


def _pca_staged(rows, boxes, dev):
    """Yield rows[r0:r1, c0:c1] for each box in order, as a device fp32 matrix with unit column stride.  Device rows are
    read in place.  Host rows are gathered into one of two pinned stages and copied to the device on a side stream;
    box j+1 is gathered and its copy queued when the caller resumes the generator, i.e. once it has queued its work on
    box j, so the gather and the copy overlap that work."""
    if rows.is_cuda:
        for b in boxes:
            yield rows.on_device(b, dev)
        return
    if not boxes:
        return
    cap = max((r1 - r0) * (c1 - c0) for r0, r1, c0, c1 in boxes)
    host = [torch.empty(cap, pin_memory=True) for _ in range(min(2, len(boxes)))]
    raw = [torch.empty(cap, device=dev) for _ in host]
    cs, xs = torch.cuda.current_stream(), torch.cuda.Stream()
    # the stages come from torch's allocator on cs and may reuse memory that work already queued on cs still reads
    # (the previous pass's last pieces): the side stream's copies into them start after that work
    xs.wait_stream(cs)
    copied, freed = [None, None], [None, None]

    def stage(j):
        r0, r1, c0, c1 = boxes[j]
        s, size = j & 1, (r1 - r0) * (c1 - c0)
        if copied[s] is not None:
            copied[s].synchronize()                    # the stage's previous copy is done
        rows.gather(host[s][:size].view(r1 - r0, c1 - c0), boxes[j])
        with torch.cuda.stream(xs):
            if freed[s] is not None:
                xs.wait_event(freed[s])                # the caller's work on the box before is done with raw[s]
            raw[s][:size].copy_(host[s][:size], non_blocking=True)
            copied[s] = torch.cuda.Event()
            copied[s].record(xs)

    stage(0)
    for j, (r0, r1, c0, c1) in enumerate(boxes):
        s = j & 1
        cs.wait_event(copied[s])
        yield raw[s][:(r1 - r0) * (c1 - c0)].view(r1 - r0, c1 - c0)
        freed[s] = torch.cuda.Event()
        freed[s].record(cs)
        if j + 1 < len(boxes):
            stage(j + 1)


def _pca_colsum(x, out):
    """out[c] += sum_r x[r, c] (fp64) for a device fp32 matrix x with unit column stride"""
    lib = _lib.load()
    rows, cols = x.shape
    ws = _lib.workspaces.get(x.device, lib.anyloc_pca_colsum_workspace_bytes(rows, cols), "pca")
    _lib.check(lib.anyloc_pca_colsum(C.c_void_p(x.data_ptr()), x.stride(0), rows, cols, C.c_void_p(out.data_ptr()),
                                     _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "anyloc_pca_colsum")


def _pca_accumulate(mode, x, mu, out, u=None):
    """anyloc_pca_accumulate(ANYLOC_PCA_<mode>) of the device fp32 matrix x (unit column stride) centred by mu into the
    fp64 view out (unit column stride)"""
    rows, cols = x.shape
    k, ld_u = (u.shape[1], u.stride(0)) if u is not None else (0, 0)
    _lib.check(_lib.load().anyloc_pca_accumulate(
        _lib.PCA[mode], C.c_void_p(x.data_ptr()), x.stride(0), rows, cols, C.c_void_p(mu.data_ptr()), _lib.ptr(u),
        ld_u, k, C.c_void_p(out.data_ptr()), out.stride(0), _lib.stream_ptr()), "anyloc_pca_accumulate")


def _pca_project_streamed(rows, project, k, dev):
    """project(x) (device rows -> [rows, k] fp32) of every row of `rows`, fed in row pieces of at most one staging
    buffer -> host fp32 [n, k]"""
    return _pca_project_dims(rows, [project], [k], dev)[0]


def _pca_project_dims(rows, projects, ks, dev):
    """_pca_project_streamed of several projections (projects[i] -> [rows, ks[i]]): each row piece is staged once and
    every projection runs on it -> [host fp32 [n, ks[i]]]"""
    n, d = rows.shape
    outs = [torch.empty(n, k) for k in ks]
    boxes = _pca_boxes(n, d, ("cov", max(1, min(n, _STAGE_BYTES // (4 * d)))))
    with torch.cuda.device(dev):
        for (r0, r1, _, _), x in zip(boxes, _pca_staged(rows, boxes, dev)):
            for out, project in zip(outs, projects):
                out[r0:r1].copy_(project(x))
    return outs


def _pca_fit_any(rows, k, dev):
    """_PcaDev(k) fitted on `rows` (a _PcaRows): in memory when that fits the device, else streamed"""
    n, d = rows.shape
    plan = _pca_plan(n, d, 0, _device_budget(dev), _STAGE_BYTES)
    if plan is None:
        return _PcaDev(k).fit(torch.cat([_as_device_f32(p, dev) for p in rows.parts]))
    return _PcaDev(k).fit_streamed(rows, plan, dev)


def _reduce_pca_streamed(train_descs, test_descs, lower_dim, low_factor, fallback, whitening, plan, dev):
    """reduce_pca for rows the in-memory route cannot hold: the same steps (fallback pre-reduction, fit, whitening,
    top / bottom basis).  The first fit is streamed by `plan` (_PcaDev.fit_streamed); the fit after the fallback
    pre-reduction, on its far smaller rows, is streamed only when it has to be.  Every projection streams in row pieces
    straight into host fp32 outputs -> (tr, te) host tensors"""
    tr, te = _PcaRows([train_descs]), _PcaRows([test_descs])
    if low_factor == 0.0:
        pca = _PcaDev(lower_dim, whiten=whitening).fit_streamed(tr, plan, dev)
        return (_pca_project_streamed(tr, pca.transform, lower_dim, dev),
                _pca_project_streamed(te, pca.transform, lower_dim, dev))
    n_samples, n_components = tr.shape
    if n_samples < n_components:
        print(f"Too few samples, fallback to {fallback}d first")
        pca = _PcaDev(fallback).fit_streamed(_PcaRows(tr.parts + te.parts), plan, dev)
        tr = _PcaRows([_pca_project_streamed(tr, pca.transform, fallback, dev)])
        te = _PcaRows([_pca_project_streamed(te, pca.transform, fallback, dev)])
    n_low = int(low_factor * lower_dim)
    n_top = lower_dim - n_low
    print(f"Up: {n_top}, Down: {n_low}")
    if n_samples < n_components:
        pca = _pca_fit_any(tr, tr.shape[1], dev)
    else:
        pca = _PcaDev(n_components).fit_streamed(tr, plan, dev)
    basis = torch.cat((pca.components_[:n_top], pca.components_[-n_low:])).contiguous()

    def project(x):
        return _gemm_nt_dev(x - pca.mean_, basis)
    return (_pca_project_streamed(tr, project, basis.shape[0], dev),
            _pca_project_streamed(te, project, basis.shape[0], dev))


def _pca_randomized_params(n, d, k):
    """(l, n_iter, transpose) of sklearn's PCA(k, svd_solver="randomized") on n x d rows with its defaults: l = k + 10
    test vectors (n_oversamples), n_iter = 7 power iterations when k < 0.1 min(n, d), else 4 (iterated_power="auto"),
    and the transpose A = Xc^T when n < d (_randomized_svd's transpose="auto")"""
    return k + 10, 7 if k < 0.1 * min(n, d) else 4, n < d


def _pca_test_matrix(n, d, k, f32):
    """The Gaussian test matrix of sklearn's _randomized_range_finder, [min(n, d), l] (A.shape[1] of the possibly
    transposed A), drawn as it draws it: np.random.normal from numpy's global generator, rounded to fp32 for fp32 rows"""
    w = np.random.normal(size=(min(n, d), _pca_randomized_params(n, d, k)[0]))
    return w.astype(np.float32) if f32 else w


def _pca_skip_test_matrix(n, d, k, chunk=1 << 22):
    """Advance numpy's global generator past _pca_test_matrix(n, d, k) without holding it: the legacy Gaussian sampler
    yields the same sequence, and ends in the same state, whether the values are drawn at once or in pieces"""
    total = min(n, d) * _pca_randomized_params(n, d, k)[0]
    for i in range(0, total, chunk):
        np.random.normal(size=min(chunk, total - i))


def _pca_fit_randomized(rows, k, dev, whiten=False):
    """_PcaDev(k, whiten).fit_randomized on `rows` (a _PcaRows).  Device fp32 rows with unit column stride are read in
    place.  Other rows are uploaded once as fp32 when they fit the device beside the fit's matrices
    (_pca_randomized_plan), else every pass streams them in row pieces through the pinned stages."""
    n, d = rows.shape
    if not 1 <= k <= min(n, d):
        raise ValueError(f"n_components={k} must be between 1 and min(n_samples, n_features)={min(n, d)} with "
                         "svd_solver='randomized'")
    f32 = all(q.dtype == torch.float32 for q in rows.parts)
    P = min(n, _PCA_PIECE_MAX_ROWS)
    if not _pca_in_place(rows, dev):
        plan = _pca_randomized_plan(n, d, _pca_randomized_params(n, d, k)[0], _device_budget(dev), _STAGE_BYTES)
        if plan is None:
            rows = _pca_upload(rows, dev)
        else:
            P = plan
    w = _pca_test_matrix(n, d, k, f32)
    return _PcaDev(k, whiten=whiten).fit_randomized(rows, w, P, dev)


def _pca_in_place(rows, dev):
    """whether a randomized fit reads `rows` (a _PcaRows) in place: one device fp32 matrix with unit column stride"""
    p = rows.parts[0]
    d = rows.shape[1]
    return (len(rows.parts) == 1 and p.device == dev and p.dtype == torch.float32 and p.stride(1) == 1 and
            p.stride(0) >= d)


def _pca_upload(rows, dev):
    """`rows` (a _PcaRows) uploaded once as one device fp32 matrix, through the pinned stages -> _PcaRows"""
    n, d = rows.shape
    x = torch.empty(n, d, device=dev)
    boxes = _pca_boxes(n, d, ("cov", max(1, min(n, _STAGE_BYTES // (4 * d)))))
    with torch.cuda.device(dev):
        for (r0, r1, _, _), piece in zip(boxes, _pca_staged(rows, boxes, dev)):
            x[r0:r1].copy_(piece)
    return _PcaRows([x])


def _reduce_pca_randomized(train_descs, test_descs, lower_dim, low_factor, fallback, whitening, dev):
    """reduce_pca(svd_solver="randomized") for low_factor == 0 and for the low_factor branch's `fallback`
    pre-reduction (n_samples < n_features), whose fits are sklearn's randomized ones (_pca_fit_randomized).  As sklearn's
    fit_transform, a fit's own rows come back as U S from the fit; other rows are projected in row pieces straight into
    host fp32 outputs.  The low_factor branch's fit of the full basis on the pre-reduced rows is the exact one
    (_pca_fit_any), as in reduce_pca -> (tr, te) host tensors"""
    tr, te = _PcaRows([train_descs]), _PcaRows([test_descs])
    if low_factor == 0.0:
        pca = _pca_fit_randomized(tr, lower_dim, dev, whiten=whitening)
        return pca.fit_rows_.cpu(), _pca_project_streamed(te, pca.transform, lower_dim, dev)
    n = tr.shape[0]
    print(f"Too few samples, fallback to {fallback}d first")
    both = _pca_fit_randomized(_PcaRows(tr.parts + te.parts), fallback, dev).fit_rows_
    tr, te = both[:n].contiguous(), both[n:].contiguous()
    n_low = int(low_factor * lower_dim)
    n_top = lower_dim - n_low
    print(f"Up: {n_top}, Down: {n_low}")
    pca = _pca_fit_any(_PcaRows([tr]), fallback, dev)
    _pca_skip_test_matrix(n, fallback, fallback)            # as in reduce_pca: the full basis is the exact fit
    basis = torch.cat((pca.components_[:n_top], pca.components_[-n_low:])).contiguous()
    with torch.cuda.device(dev):
        return _gemm_nt_dev(tr - pca.mean_, basis).cpu(), _gemm_nt_dev(te - pca.mean_, basis).cpu()


# ------------------------------------------------------------------ several PCA dimensions from one fit (extension)
def reduce_pca_dims(train_descs: Union[np.ndarray, torch.Tensor], test_descs: Union[np.ndarray, torch.Tensor],
                    lower_dims: List[int], low_factor: float = 0.0, fallback: int = 256, svd_solver: str = "full",
                    whitening: bool = False) -> List[Tuple[np.ndarray, np.ndarray]]:
    """reduce_pca at every dimension of `lower_dims`, sharing the work that does not depend on the dimension -> a list
    of (train_i, test_i).  Element i equals, bit for bit and in type and dtype, reduce_pca(train_descs, test_descs,
    lower_dims[i], low_factor, fallback, svd_solver, whitening) run in list order from the same numpy global generator
    state, and numpy's generator ends where those calls leave it.  Dimensions may repeat and come in any order.

    Shared: the exact fit's mean, Gram / covariance matrix and eigh (each member then takes its own vt at its own k);
    the low_factor branch's exact `fallback` pre-reduction and full-basis fit; the randomized fits' mean pass and every
    row pass of their power iterations (_pca_randomized_group).  Streamed passes stage each row piece once for all
    members.  The randomized members draw their test matrices in list order, each its own draw.

    Unlike the sequential calls, which stop at the first bad member, every refusal comes before any work and leaves
    the generator untouched: ValueError for an empty list, a dimension out of range for the solver, or an exact fit
    whose m = min(n_samples, n_features) is beyond what the eigensolver takes (_PCA_EIGH_MAX_M).  MemoryError only where
    a member's own call would raise it; members that do not fit on the device together run in consecutive groups."""
    assert 0 <= low_factor <= 1
    dims = [int(k) for k in lower_dims]
    as_np = type(train_descs) == np.ndarray
    (n, d), n_te = train_descs.shape, test_descs.shape[0]
    _pca_dims_check(n, d, n_te, dims, low_factor, fallback, svd_solver)
    dev = _lib.require_cuda(None)
    draws = [_pca_member_draws(n, d, n_te, k, low_factor, fallback, svd_solver) for k in dims]
    if svd_solver == "randomized" and (low_factor == 0.0 or n < d):
        outs = _reduce_pca_dims_randomized(train_descs, test_descs, dims, low_factor, fallback, whitening, draws, dev)
    else:
        outs = _reduce_pca_dims_exact(train_descs, test_descs, dims, low_factor, fallback, whitening, dev)
        _pca_draw(sum(draws, []), False)        # randomized with low_factor, n >= d: the skips of the exact fits
    return [(a.numpy(), b.numpy()) if as_np else (a, b) for a, b in outs]


def _pca_dims_check(n, d, n_te, dims, low_factor, fallback, svd_solver):
    """reduce_pca_dims' refusals, before any work: the messages of _PcaDev.fit and _pca_fit_randomized for the fits each
    member's call would make, and the exact fits' m beyond _PCA_EIGH_MAX_M"""
    if not dims:
        raise ValueError("reduce_pca_dims: lower_dims is empty")

    def full(k, rows, cols):
        if not 0 <= k <= min(rows, cols):
            raise ValueError(f"n_components={k} must be between 0 and min(n_samples, n_features)={min(rows, cols)} "
                             "with svd_solver='full'")
        if min(rows, cols) > _PCA_EIGH_MAX_M:
            raise ValueError(f"reduce_pca_dims: m = min(n_samples, n_features) = {min(rows, cols)} is beyond the "
                             f"{_PCA_EIGH_MAX_M} x {_PCA_EIGH_MAX_M} fp64 matrices the eigensolver (torch.linalg.eigh, "
                             "cuSOLVER syevd) takes; svd_solver='randomized' has no such limit")

    def randomized(k, rows, cols):
        if not 1 <= k <= min(rows, cols):
            raise ValueError(f"n_components={k} must be between 1 and min(n_samples, n_features)={min(rows, cols)} "
                             "with svd_solver='randomized'")
    if svd_solver == "randomized" and low_factor == 0.0:
        for k in dims:
            randomized(k, n, d)
    elif low_factor == 0.0:
        for k in dims:
            full(k, n, d)
    elif n < d:                     # the fallback pre-reduction, then the full basis of the [n, fallback] rows
        (randomized if svd_solver == "randomized" else full)(fallback, n + n_te, d)
        full(fallback, n, fallback)
    else:                           # the full basis of the rows
        full(d, n, d)


def _pca_member_draws(n, d, n_te, k, low_factor, fallback, svd_solver):
    """What reduce_pca(n x d training rows, n_te test rows, k, ...) takes from numpy's global generator, in order:
    [(n', d', k', draw)], draw=True for _pca_test_matrix(n', d', k'), False for _pca_skip_test_matrix(n', d', k')"""
    if svd_solver != "randomized":
        return []
    if low_factor == 0.0:
        return [(n, d, k, True)]
    if n < d:                       # the randomized fallback pre-reduction, then the exact full-basis fit's skip
        return [(n + n_te, d, fallback, True), (n, fallback, fallback, False)]
    return [(n, d, d, False)]


def _pca_draw(draws, f32):
    """Take `draws` (_pca_member_draws) from numpy's global generator in order -> the test matrices drawn"""
    ws = []
    for a, b, k, draw in draws:
        if draw:
            ws.append(_pca_test_matrix(a, b, k, f32))
        else:
            _pca_skip_test_matrix(a, b, k)
    return ws


def _pca_member_bytes(m, d, k):
    """Device bytes one member of an exact sweep adds to the shared fit: its fp64 u [m, k] and vt [k, d], and its fp32
    components [k, d]"""
    return 8 * k * (m + d) + 4 * k * d


def _pca_exact_groups(m, d, ks, fixed, budget):
    """Consecutive groups of an exact sweep's members (dimensions ks) that share one fit: members join the group
    before while its _pca_member_bytes, summed, fit the `budget` beside the `fixed` bytes of the fit itself
    (_pca_in_memory_bytes in memory, the m x m matrix and its eigh streamed).  A member that does not fit with the
    group starts the next -> [[member index]]"""
    groups, used = [], 0
    for i, k in enumerate(ks):
        b = _pca_member_bytes(m, d, k)
        if groups and fixed + used + b <= budget:
            groups[-1].append(i)
            used += b
        else:
            groups.append([i])
            used = b
    return groups


def _pca_randomized_groups(n, d, ls, plans, in_place, budget, stage_bytes):
    """Consecutive groups of a randomized sweep's members (ls[i] = k + 10 test vectors, plans[i] its own call's
    _pca_randomized_plan, None for rows read in place) that run their fits together -> [(members, P, upload)].  The
    mean pass's fp64 column sums depend on the row pieces, so a group's members are those whose own calls read the rows
    in the same pieces: in place or uploaded in pieces of min(n, 2^20) rows, or streamed in pieces of plans[i] rows.
    Members join the group before while the fits' matrices (_pca_randomized_bytes, summed) fit the `budget` beside the
    rows: nothing for rows read in place, the uploaded rows (4 n d) beside the larger of the matrices and the upload's
    two staging copies, or two device copies of a streamed piece.  A member that does not fit with the group starts
    the next; alone, it runs as its own call does."""
    piece = 4 * d * max(1, min(n, stage_bytes // (4 * d)))

    def fits(mats, plan):
        if in_place:
            return mats <= budget
        if plan is None:
            return 4 * n * d + max(mats, 2 * piece) <= budget
        return mats + 8 * d * plan <= budget
    groups, mats = [], 0
    for i, (l, plan) in enumerate(zip(ls, plans)):
        b = _pca_randomized_bytes(n, d, l)
        if groups and plans[groups[-1][0][-1]] == plan and fits(mats + b, plan):
            groups[-1][0].append(i)
            mats += b
        else:
            groups.append(([i], min(n, _PCA_PIECE_MAX_ROWS) if plan is None else plan, not in_place and plan is None))
            mats = b
    return groups


def _pca_randomized_dims(rows, ks, whiten, draws, dev):
    """_pca_fit_randomized(rows, ks[i], dev, whiten) for every i, group by group (_pca_randomized_groups): a group
    takes its members' draws (_pca_member_draws) in list order, uploads the rows once if its members' own calls would,
    and runs its fits together (_pca_randomized_group).  Yields (members, fitted _PcaDevs) per group."""
    n, d = rows.shape
    f32 = all(q.dtype == torch.float32 for q in rows.parts)
    in_place = _pca_in_place(rows, dev)
    ls = [_pca_randomized_params(n, d, k)[0] for k in ks]
    budget = _device_budget(dev)
    plans = [None if in_place else _pca_randomized_plan(n, d, l, budget, _STAGE_BYTES) for l in ls]
    for group, P, upload in _pca_randomized_groups(n, d, ls, plans, in_place, budget, _STAGE_BYTES):
        ws = _pca_draw(sum((draws[i] for i in group), []), f32)
        pcas = [_PcaDev(ks[i], whiten=whiten) for i in group]
        yield group, _pca_randomized_group(_pca_upload(rows, dev) if upload else rows, pcas, ws, P, dev)


def _reduce_pca_dims_randomized(train_descs, test_descs, dims, low_factor, fallback, whitening, draws, dev):
    """reduce_pca_dims for the routes of _reduce_pca_randomized -> [(tr, te) host tensors]"""
    tr, te = _PcaRows([train_descs]), _PcaRows([test_descs])
    outs = []
    if low_factor == 0.0:
        for group, pcas in _pca_randomized_dims(tr, dims, whitening, draws, dev):
            tes = _pca_project_dims(te, [p.transform for p in pcas], [dims[i] for i in group], dev)
            outs += [(p.fit_rows_.cpu(), t) for p, t in zip(pcas, tes)]
        return outs
    n = tr.shape[0]
    # every member's own call draws its own fallback test matrix, so the pre-reductions are a randomized sweep too
    for group, pcas in _pca_randomized_dims(_PcaRows(tr.parts + te.parts), [fallback] * len(dims), False, draws, dev):
        for i, j in enumerate(group):
            both, pcas[i] = pcas[i].fit_rows_, None
            low_tr, low_te = both[:n].contiguous(), both[n:].contiguous()
            print(f"Too few samples, fallback to {fallback}d first")
            basis, mean = _pca_low_factor_basis(_pca_fit_any(_PcaRows([low_tr]), fallback, dev), dims[j], low_factor)
            with torch.cuda.device(dev):
                outs.append((_gemm_nt_dev(low_tr - mean, basis).cpu(), _gemm_nt_dev(low_te - mean, basis).cpu()))
    return outs


def _pca_low_factor_basis(pca, lower_dim, low_factor):
    """reduce_pca's low_factor basis: the top n_top and bottom n_low components of a full-basis fit, printing the split
    as reduce_pca does -> (basis, mean)"""
    n_low = int(low_factor * lower_dim)
    n_top = lower_dim - n_low
    print(f"Up: {n_top}, Down: {n_low}")
    return torch.cat((pca.components_[:n_top], pca.components_[-n_low:])).contiguous(), pca.mean_


def _reduce_pca_dims_exact(train_descs, test_descs, dims, low_factor, fallback, whitening, dev):
    """reduce_pca_dims for the exact routes of reduce_pca and _reduce_pca_streamed; the route is the one every member's
    own call takes, as it does not depend on the dimension -> [(tr, te) host tensors]"""
    (n, d), n_te = train_descs.shape, test_descs.shape[0]
    n_fit, n_held = (n + n_te, n + n_te) if low_factor != 0.0 and n < d else (n, n_te)
    budget = _device_budget(dev)
    plan = _pca_plan(n_fit, d, n_held, budget, _STAGE_BYTES)
    if low_factor != 0.0:
        return _reduce_pca_dims_low_factor(train_descs, test_descs, dims, low_factor, fallback, plan, dev)
    m, outs = min(n, d), []
    if plan is None:
        tr, te = _as_device_f32(train_descs, dev), _as_device_f32(test_descs, dev)
        for group in _pca_exact_groups(m, d, dims, _pca_in_memory_bytes(n, d, n_te), budget):
            eig = _pca_decompose(tr)
            pcas = [_PcaDev(dims[i], whiten=whitening).fit_shared(eig) for i in group]
            del eig
            outs += [(p.transform(tr).cpu(), p.transform(te).cpu()) for p in pcas]
        return outs
    tr, te = _PcaRows([train_descs]), _PcaRows([test_descs])
    for group in _pca_exact_groups(m, d, dims, 8 * _PCA_EIGH_MATRICES * m * m, budget):
        pcas = _pca_fit_streamed_dims(tr, plan, [_PcaDev(dims[i], whiten=whitening) for i in group], dev)
        projects, ks = [p.transform for p in pcas], [dims[i] for i in group]
        outs += zip(_pca_project_dims(tr, projects, ks, dev), _pca_project_dims(te, projects, ks, dev))
    return outs


def _reduce_pca_dims_low_factor(train_descs, test_descs, dims, low_factor, fallback, plan, dev):
    """reduce_pca_dims' exact low_factor branch: the fallback pre-reduction and the full-basis fit, which do not depend
    on the dimension, once; then each member's own top / bottom basis.  In memory (plan None) as reduce_pca, else
    streamed as _reduce_pca_streamed, whose final projections stage each row piece once for all members."""
    n_samples, n_components = train_descs.shape
    few = n_samples < n_components
    if plan is None:
        tr, te = _as_device_f32(train_descs, dev), _as_device_f32(test_descs, dev)
        if few:
            both = torch.cat((tr, te))
            both = _PcaDev(fallback).fit(both).transform(both)
            tr, te = both[:n_samples].contiguous(), both[n_samples:].contiguous()
        pca = _PcaDev(tr.shape[1]).fit(tr)
        outs = []
        for k in dims:
            if few:
                print(f"Too few samples, fallback to {fallback}d first")
            basis, mean = _pca_low_factor_basis(pca, k, low_factor)
            outs.append((_gemm_nt_dev(tr - mean, basis).cpu(), _gemm_nt_dev(te - mean, basis).cpu()))
        return outs
    tr, te = _PcaRows([train_descs]), _PcaRows([test_descs])
    if few:
        pre = _PcaDev(fallback).fit_streamed(_PcaRows(tr.parts + te.parts), plan, dev)
        tr = _PcaRows([_pca_project_streamed(tr, pre.transform, fallback, dev)])
        te = _PcaRows([_pca_project_streamed(te, pre.transform, fallback, dev)])
        pca = _pca_fit_any(tr, tr.shape[1], dev)
    else:
        pca = _PcaDev(n_components).fit_streamed(tr, plan, dev)
    bases = []
    for k in dims:
        if few:
            print(f"Too few samples, fallback to {fallback}d first")
        bases.append(_pca_low_factor_basis(pca, k, low_factor))

    def project(basis, mean):
        return lambda x: _gemm_nt_dev(x - mean, basis)
    projects, ks = [project(*b) for b in bases], [b[0].shape[0] for b in bases]
    return list(zip(_pca_project_dims(tr, projects, ks, dev), _pca_project_dims(te, projects, ks, dev)))


# ------------------------------------------------------------------ image pre-processing (extension)
IMAGENET_MEAN = (0.485, 0.456, 0.406)       # dvgl_benchmark/datasets_ws.py:22
IMAGENET_STD = (0.229, 0.224, 0.225)


def center_crop_box(h: int, w: int, patch: int = 14) -> Tuple[int, int, int, int]:
    """(top, left, h_new, w_new) of `T.CenterCrop(((h // 14) * 14, (w // 14) * 14))`
    (scripts/dino_v2_vlad.py:174-176); torchvision places the window at int(round((h - h_new) / 2.0))."""
    h_new, w_new = (h // patch) * patch, (w // patch) * patch
    return int(round((h - h_new) / 2.0)), int(round((w - w_new) / 2.0)), h_new, w_new


_INTERP = {"bilinear": 0, "bicubic": 1}


def max_side_size(h: int, w: int, max_side: int) -> Tuple[int, int]:
    """The size the reference demo resizes an h x w photo to (demo/anyloc_vlad_generate.py:165-173): when the longer
    side is over `max_side` it becomes `max_side` and the other side keeps the aspect ratio, rounded down; otherwise
    (h, w) unchanged."""
    if max(h, w) > max_side:
        if h == max(h, w):
            w = int(w * max_side / h)
            h = max_side
        else:
            h = int(h * max_side / w)
            w = max_side
    return h, w


def _resized_size(H, W, resize, max_side):
    """-> (hr, wr, resized): the size an H x W image is resized to before the centre crop, and whether it is resized"""
    if max_side is not None:
        hr, wr = max_side_size(H, W, int(max_side))
        return hr, wr, (hr, wr) != (H, W)
    if resize is not None:
        return int(resize[0]), int(resize[1]), True
    return H, W, False


def _list_geometry(shapes, patch, resize, max_side):
    """Per (H, W) of a list: (hr, wr, resized, top, left, hc, wc); ValueError for an image smaller than one patch after
    the resize.  Pure: no device work."""
    geo = []
    for k, (H, W) in enumerate(shapes):
        hr, wr, resized = _resized_size(H, W, resize, max_side)
        top, left, hc, wc = center_crop_box(hr, wr, patch) if hr > 0 and wr > 0 else (0, 0, 0, 0)
        if hc == 0 or wc == 0:
            raise ValueError(f"image {k} ({H}x{W}, resized to {hr}x{wr}) is smaller than one {patch}x{patch} patch")
        geo.append((hr, wr, resized, top, left, hc, wc))
    return geo


def _check_resize_args(resize, max_side, interpolation):
    if interpolation not in _INTERP:
        raise ValueError(f"interpolation must be one of {sorted(_INTERP)}, got {interpolation!r}")
    if resize is not None and max_side is not None:
        raise ValueError("give resize=(h, w) or max_side, not both")
    if max_side is not None and int(max_side) < 1:
        raise ValueError(f"max_side must be positive, got {max_side!r}")


def _preprocess_list(items, mean, std, patch, device, resize, interpolation, max_side):
    """preprocess_images on a list / tuple of [H_i,W_i,3] uint8 images (see there)"""
    _check_resize_args(resize, max_side, interpolation)
    if len(items) == 0:
        raise ValueError("preprocess_images got an empty list")
    imgs = []
    for k, x in enumerate(items):
        if type(x) == np.ndarray:
            x = torch.from_numpy(x)
        if not isinstance(x, torch.Tensor):
            raise TypeError(f"preprocess_images: item {k} is a {type(x).__name__}, expected a uint8 array or tensor")
        if x.dtype != torch.uint8:
            raise TypeError(f"preprocess_images expects uint8 pixels, got {x.dtype} (item {k})")
        if x.dim() != 3 or x.shape[-1] != 3:
            raise ValueError(f"preprocess_images expects list items [H,W,3], got {tuple(x.shape)} (item {k})")
        if x.shape[0] == 0 or x.shape[1] == 0:
            raise ValueError(f"preprocess_images: item {k} is empty ({tuple(x.shape)})")
        imgs.append(x)
    geo = _list_geometry([(x.shape[0], x.shape[1]) for x in imgs], patch, resize, max_side)
    on_dev = {x.device for x in imgs if x.is_cuda}
    if len(on_dev) > 1:
        raise ValueError(f"preprocess_images: the list's device images are on several devices {sorted(map(str, on_dev))}")
    dev = _lib.require_cuda(on_dev.pop() if on_dev else (torch.device(device) if device is not None else None))
    with torch.cuda.device(dev):
        # host images: gathered into one pinned buffer, one copy; device images: read in place
        src = [x.contiguous() if x.is_cuda else None for x in imgs]
        host = [k for k, x in enumerate(imgs) if not x.is_cuda]
        if host:
            staging = torch.empty(sum(imgs[k].numel() for k in host), dtype=torch.uint8, pin_memory=True)
            views, o = {}, 0
            for k in host:
                n = imgs[k].numel()
                staging[o:o + n].view(imgs[k].shape).copy_(imgs[k])
                views[k], o = (o, n), o + n
            dbuf = staging.to(dev, non_blocking=True)
            for k, (o, n) in views.items():
                src[k] = dbuf[o:o + n]
        sizes = [3 * g[5] * g[6] for g in geo]
        offs = np.concatenate(([0], np.cumsum(sizes)[:-1])).astype(np.int64)
        flat = torch.empty(int(sum(sizes)), device=dev, dtype=torch.float32)
        m3 = (C.c_float * 3)(*[float(v) for v in mean])
        s3 = (C.c_float * 3)(*[float(v) for v in std])
        for resized in (False, True):
            idx = [k for k, g in enumerate(geo) if g[2] == resized]
            if not idx:
                continue
            n = len(idx)

            def ints(col):
                return (C.c_int * n)(*[int(col(k)) for k in idx])
            rc = _lib.load().anyloc_preprocess_u8_varlen(
                n, (C.c_void_p * n)(*[src[k].data_ptr() for k in idx]), ints(lambda k: imgs[k].shape[0]),
                ints(lambda k: imgs[k].shape[1]), ints(lambda k: geo[k][0]), ints(lambda k: geo[k][1]),
                _INTERP[interpolation] if resized else -1, ints(lambda k: geo[k][3]), ints(lambda k: geo[k][4]),
                ints(lambda k: geo[k][5]), ints(lambda k: geo[k][6]), m3, s3, _lib.ptr(flat),
                (C.c_int64 * n)(*[int(offs[k]) for k in idx]), _lib.stream_ptr())
            _lib.check(rc, "anyloc_preprocess_u8_varlen")
    if resize is not None:
        return flat.view(len(geo), 3, geo[0][5], geo[0][6])
    return [flat[o:o + s].view(3, g[5], g[6]) for o, s, g in zip(offs.tolist(), sizes, geo)]


def preprocess_images(imgs: Union[np.ndarray, torch.Tensor, list, tuple], mean=IMAGENET_MEAN, std=IMAGENET_STD,
                      patch: int = 14, device: Union[str, torch.device, None] = None,
                      resize: Union[Tuple[int, int], None] = None, interpolation: str = "bilinear",
                      max_side: Union[int, None] = None):
    """uint8 RGB images [B,H,W,3] (or one [H,W,3]) -> the extractor's input [B,3,H',W'] on the GPU: the reference's
    `base_transform` (ToTensor + Normalize, dvgl_benchmark/datasets_ws.py:20-23), optionally the dataset loader's
    `T.functional.resize(img, resize)` (:233-235, `resize=(480, 640)` is the reference default, configs.py:141; or the
    demo's bicubic down-scaling, demo/anyloc_vlad_generate.py:165-177) and the centre crop to a multiple of the patch
    size (scripts/dino_v2_vlad.py:174-176) in ONE kernel.  Without `resize` the result is bit-identical to the
    torchvision pipeline; with it, antialiased bilinear / bicubic resampling as torchvision applies to tensors (fp32
    rounding differences only).  A quarter of the host->device bytes of sending normalised fp32 images.

    `max_side` applies the demo's rule instead of a fixed `resize`: an image whose longer side is over `max_side` is
    resized to the size `max_side_size` gives (demo/anyloc_vlad_generate.py:165-177, `max_side=1024`,
    `interpolation="bicubic"` there), any other is only normalised and cropped.

    `imgs` may also be a list or tuple of differently sized [H_i,W_i,3] uint8 arrays or tensors, on the host or the
    device (host images are gathered into one pinned buffer and copied once; device images are read in place), all
    pre-processed in one launch per 64 images (two groups when `max_side` resizes some images and not others).  With
    `resize` every item has the same size and the result is one [B,3,h,w] tensor; otherwise it is a list of [3,h_i,w_i]
    views of one allocation, which DinoV2ExtractFeatures and DinoV2MultiExtractFeatures take as a list input.  Each
    item is bit-identical to this function on that image alone."""
    if isinstance(imgs, (list, tuple)):
        return _preprocess_list(imgs, mean, std, patch, device, resize, interpolation, max_side)
    if type(imgs) == np.ndarray:
        imgs = torch.from_numpy(imgs)
    if imgs.dtype != torch.uint8:
        raise TypeError(f"preprocess_images expects uint8 pixels, got {imgs.dtype}")
    if imgs.dim() == 3:
        imgs = imgs[None]
    if imgs.dim() != 4 or imgs.shape[-1] != 3:
        raise ValueError(f"preprocess_images expects [B,H,W,3], got {tuple(imgs.shape)}")
    _check_resize_args(resize, max_side, interpolation)
    dev = _lib.require_cuda(imgs.device if imgs.is_cuda else (torch.device(device) if device is not None else None))
    x = imgs.to(dev, non_blocking=True).contiguous()
    B, H, W, _ = x.shape
    hr, wr, resized = _resized_size(H, W, resize, max_side)
    top, left, hc, wc = center_crop_box(hr, wr, patch)
    if hc == 0 or wc == 0:
        raise ValueError(f"image {hr}x{wr} is smaller than one {patch}x{patch} patch")
    out = torch.empty(B, 3, hc, wc, device=dev, dtype=torch.float32)
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(dev):
        if not resized:
            _lib.check(_lib.load().anyloc_preprocess_u8(_lib.ptr(x), B, H, W, top, left, hc, wc, m3, s3, _lib.ptr(out),
                                                        _lib.stream_ptr()), "anyloc_preprocess_u8")
        else:
            _lib.check(_lib.load().anyloc_preprocess_resize_u8(_lib.ptr(x), B, H, W, hr, wr, _INTERP[interpolation], top,
                                                               left, hc, wc, m3, s3, _lib.ptr(out), _lib.stream_ptr()),
                       "anyloc_preprocess_resize_u8")
    return out


# ------------------------------------------------------------------ extractor
class _HookHandle:
    def remove(self):
        pass


PRECISIONS = ("auto", "tf32x3", "f16x3", "bf16", "fp8", "f16x1", "bf16pair")
# precisions whose GEMM operands are fp16 (scaled by 8): an operand beyond fp16's range overflows, which the guard catches
_FP16_RANGE = ("f16x3", "f16x1")


def resolve_precision(precision, gemm_engine="auto"):
    """The extractor's precision: the argument, else $ANYLOC_B200_PRECISION, else "auto".  ValueError on an unknown
    name, and on "bf16", "fp8", "f16x1" or "bf16pair" with gemm_engine="simt" (single bf16, e4m3 and fp16 and the bf16
    pairs run on the tensor cores only)."""
    precision = precision or os.environ.get("ANYLOC_B200_PRECISION", "auto")
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be 'auto', 'tf32x3', 'f16x3', 'bf16', 'fp8', 'f16x1' or 'bf16pair', got "
                         f"{precision!r}")
    if precision in ("bf16", "fp8", "f16x1", "bf16pair") and gemm_engine == "simt":
        raise ValueError(f"precision={precision!r} runs on the tensor cores only; use gemm_engine='auto' or 'tc3'")
    return precision


class _GuardedExtractor:
    """What DinoV2ExtractFeatures and DinoV2MultiExtractFeatures share: the uploaded backbone (blocks 0.._depth()-1),
    the precision choice and the fp16-range guard around each call.  A subclass sets the call options and defines
    `_depth()` and `_extract(img)` -> (every output row in one tensor, what __call__ returns)."""

    def _load(self, dino_model, dev, weights, gemm_engine, precision):
        sd = weights if weights is not None else _vit.resolve_state_dict(dino_model, dev)
        # only the blocks the forward runs (early exit at the deepest hooked module) are uploaded
        precision = resolve_precision(precision, gemm_engine)
        self._auto = precision == "auto"
        self._state_dict = sd if self._auto else None     # kept for the tf32x3 re-upload on an fp16-range overflow
        self.precision = "f16x3" if self._auto else precision
        self.dino_model = _vit.VitWeights(dino_model, sd, dev, depth=self._depth(),
                                          pair={"f16x3": "f16", "tf32x3": "tf32", "bf16": "bf16",
                                                "fp8": "fp8", "f16x1": "f16x1", "bf16pair": "bf16pair"}[self.precision])
        self.gemm_engine = gemm_engine
        self.fh_handle = _HookHandle()
        self._hook_out = None
        # fp16-range guard of the f16x3 and f16x1 formats: "sync" = checked before __call__ returns (one host sync per call),
        # "deferred" = the flag of call i is read at call i+1 / raise_if_overflowed() (no sync on the hot loop),
        # "off".  precision="auto" always checks synchronously (it has to decide before returning).
        self.check_finite = os.environ.get("ANYLOC_B200_CHECK_FINITE", "sync")
        if self.check_finite in ("1", "0"):
            self.check_finite = "sync" if self.check_finite == "1" else "off"
        self._pending_flag = None

    _OVERFLOW_MSG = ("f16x3 precision overflowed the fp16 operand range (|8*x| > 65504 somewhere in the network); "
                     "construct the extractor with precision='tf32x3' (or 'auto')")
    _OVERFLOW_MSG_F16X1 = ("f16x1 precision overflowed the fp16 operand range (|8*x| > 65504 somewhere in the network); "
                           "construct the extractor with precision='bf16' (the same speed, with fp32's exponent range)")

    def _overflow_msg(self):
        return self._OVERFLOW_MSG_F16X1 if self.precision == "f16x1" else self._OVERFLOW_MSG

    def raise_if_overflowed(self):
        """Deferred mode: reads the finite-flag of the last call (one host sync)."""
        flag, self._pending_flag = self._pending_flag, None
        if flag is not None and not bool(flag):
            raise _lib.AnylocError(self._overflow_msg())

    def _switch_to_tf32(self):
        print("anyloc_b200: f16x3 operands overflowed the fp16 range -- switching this extractor to tf32x3 "
              "(full fp32 exponent range, ~2x slower)")
        dev, name = self.dino_model.device, self.dino_model.name
        self.dino_model = None
        torch.cuda.empty_cache()
        self.dino_model = _vit.VitWeights(name, self._state_dict, dev, depth=self._depth(), pair="tf32")
        self.precision, self._auto, self._state_dict = "tf32x3", False, None

    def _guarded(self, img):
        """self._extract(img)[1] under the fp16-range guard: every output row is checked in one reduction"""
        with torch.no_grad():
            if self.check_finite == "deferred" and not self._auto:
                self.raise_if_overflowed()
            packed, out = self._extract(img)
            if self.precision not in _FP16_RANGE or (self.check_finite == "off" and not self._auto):
                return out
            flag = torch.isfinite(packed).all()
            if self.check_finite == "deferred" and not self._auto:
                self._pending_flag = flag
                return out
            if bool(flag):
                return out
            if not self._auto:
                raise _lib.AnylocError(self._overflow_msg())
            self._switch_to_tf32()
            return self._extract(img)[1]


class DinoV2ExtractFeatures(_GuardedExtractor):
    """Extract features from an intermediate layer of DINOv2 (utilities.py:219-288).

    Same constructor and call signature.  The forward stops at the hooked module (blocks
    0..layer-1, then either the whole block `layer` ("token") or norm1 + the requested third of
    its qkv projection), which is output-identical to the reference's full forward + hook.
    Extra keyword-only arguments: `weights` (an upstream state_dict, else see
    vit.resolve_state_dict), `gemm_engine` ("auto" | "tc3" | "simt") and `precision`: how fp32
    operands are fed to the tensor cores -- "tf32x3" (tf32 (hi,lo) pairs, full fp32 exponent range),
    "f16x3" (fp16 (hi,lo) pairs with power-of-two scaling: same ~22-bit products on the 2x faster
    kind::f16 path; operands beyond the fp16 range overflow to inf/NaN instead of losing accuracy
    silently, and the call raises) or "auto" (the default: f16x3 until a call overflows, then that
    call is redone and the extractor stays in tf32x3 -- trained DINOv2 checkpoints have outlier
    activations that random-init weights do not).  All accumulate in fp32 with round-to-nearest
    chunk accumulation.  "bf16" is the fast mode, never chosen by "auto": every GEMM and attention
    operand is one round-to-nearest bf16 value (fp32's exponent range, so no overflow guard), one
    bf16 MMA per product instead of three; the residual stream, LayerNorm statistics, softmax,
    accumulators and outputs stay fp32.  Its outputs are those of the model run on bf16-rounded
    activations (about 1e-2 relative), not fp32 parity; it needs gemm_engine "auto" or "tc3".
    "fp8" is faster still and also never chosen by "auto": the block GEMMs run one e4m3 MMA per
    product on e4m3 weights (one power-of-two scale per matrix) and e4m3 activations (one
    power-of-two scale per token row, so an image's rows never depend on the other images of a
    call); the patch embedding and the attention run as in "bf16", and what stays fp32 in "bf16"
    stays fp32.  Its error is that of the model run on e4m3-rounded GEMM inputs (about 2^-4
    relative per operand); it needs gemm_engine "auto" or "tc3".
    "f16x1" runs at bf16's rate with fp16's 11 significant bits, and is also never chosen by
    "auto": every GEMM and attention operand is one fp16 value, the hi half of the f16x3 pair
    (about 2^-11 relative per operand, 8x finer than bf16), one fp16 MMA per product; what stays
    fp32 in "bf16" stays fp32.  It keeps fp16's range, so the f16x3 overflow guard applies, and an
    overflow raises naming "bf16" (same speed, fp32's exponent range) as the way out.  Not a
    parity mode; it needs gemm_engine "auto" or "tc3".
    "bf16pair" sits between the parity formats and the single-MMA ones, and is also never chosen by
    "auto": every GEMM and attention operand is a bf16 pair, hi = bf16_rn(x), lo = bf16_rn(x - hi)
    (about 16 significant bits), with three bf16 MMAs per product like f16x3, the same operand
    bytes and fp32's exponent range -- no scale and no overflow guard, so activations that overflow
    f16x3 stay finite.  What stays fp32 in "bf16" stays fp32.  Its error is that of products
    rounded to about 16 significant bits (2^-16 relative, where f16x3 and tf32x3 keep about 22),
    so it is not a parity mode, and its effect on recall with trained checkpoints has not been
    measured.  It needs gemm_engine "auto" or "tc3".

    `dino_model` may also name a backbone with register tokens, `dinov2_vit{s,b,l,g}14_reg`.  As
    in the reference, only row 0 (cls) is dropped, so its 4 register rows come first: an output
    holds [cls (with use_cls), r0..r3, the N patch rows], and `out[:, 4:]` (without use_cls) or
    `out[:, 5:]` (with it) are the patch features alone."""

    def __init__(self, dino_model: _DINO_V2_MODELS, layer: int, facet: _DINO_FACETS = "token",
                 use_cls=False, norm_descs=True, device: str = "cpu", *, weights=None,
                 gemm_engine: str = "auto", precision: str = None) -> None:
        self.vit_type: str = dino_model
        self.device = torch.device(device)
        dev = _lib.require_cuda(self.device)
        if facet not in _lib.FACET:
            raise ValueError(f"facet must be one of {sorted(_lib.FACET)}, got {facet!r}")
        self.layer: int = layer
        self.facet = facet
        self.use_cls = use_cls
        self.norm_descs = norm_descs
        self._load(dino_model, dev, weights, gemm_engine, precision)

    def _depth(self):
        return self.layer + 1

    def _extract(self, img):
        """-> (every output row in one tensor, what __call__ returns)"""
        if isinstance(img, (list, tuple)):
            packed, n = self.dino_model.extract_varlen(img, self.layer, self.facet, self.use_cls, self.norm_descs,
                                                       self.gemm_engine)
            return packed, list(packed.split(n))
        out = self.dino_model.extract(img, self.layer, self.facet, self.use_cls, self.norm_descs, self.gemm_engine)
        return out, out

    def __call__(self, img):
        """img [B,3,H,W] -> [B, (1 +) R + N, D] (R = 4 register rows for the *_reg models, else 0); or a list/tuple of
        differently sized images [3,H_i,W_i] / [1,3,H_i,W_i], all on the extractor's device -> a list of [n_i, D] (views of one packed output), computed in one forward
        pass; item i is bit-identical to self(img[i][None])[0] when both run the tensor-core GEMMs (under "auto" a lone
        image of fewer than 32 tokens takes the SIMT GEMMs, except with precision "bf16", "fp8", "f16x1" or "bf16pair",
        which always run them)."""
        return self._guarded(img)

    def __del__(self):
        pass


class DinoV2MultiExtractFeatures(_GuardedExtractor):
    """Extension (not in the reference): the features of several (layer, facet) taps of DINOv2 from ONE forward pass.

    AnyLoc's layer and facet ablations read many taps of the same images (scripts/dino_v2_vlad_ablations.sh,
    dino_v2_vlad_viz.py, dino_v2_sim_facets.py); with one DinoV2ExtractFeatures per tap each of them reruns blocks
    0..layer and uploads its own weights.  Here blocks 0..max(layer) are uploaded once and run once per call, and every
    tap keeps what that pass computes.  `taps` is a list of distinct (layer, facet) pairs; `use_cls`, `norm_descs`,
    `device`, `weights`, `gemm_engine` and `precision` mean what they mean for DinoV2ExtractFeatures and apply to
    every tap.  Each output is bit-identical to DinoV2ExtractFeatures(dino_model, layer, facet, use_cls, norm_descs)
    on the same images with the same weights, precision and engine, and has its row layout: [cls (with use_cls),
    the 4 register rows of a *_reg model, the patch rows]."""

    def __init__(self, dino_model: _DINO_V2_MODELS, taps, use_cls=False, norm_descs=True, device: str = "cpu", *,
                 weights=None, gemm_engine: str = "auto", precision: str = None) -> None:
        self.vit_type: str = dino_model
        self.device = torch.device(device)
        dev = _lib.require_cuda(self.device)
        if dino_model not in _vit.ARCHS:
            raise ValueError(f"unknown DINOv2 model {dino_model!r}; expected one of {sorted(_vit.ARCHS)}")
        self.taps = _vit.check_taps(taps, _vit.ARCHS[dino_model][1])
        self.use_cls = use_cls
        self.norm_descs = norm_descs
        self._load(dino_model, dev, weights, gemm_engine, precision)

    def _depth(self):
        return 1 + max(layer for layer, _ in self.taps)

    def _extract(self, img):
        if isinstance(img, (list, tuple)):
            packed, n = self.dino_model.extract_taps_varlen(img, self.taps, self.use_cls, self.norm_descs,
                                                            self.gemm_engine)
            return packed, {t: list(packed[k].split(n)) for k, t in enumerate(self.taps)}
        packed = self.dino_model.extract_taps(img, self.taps, self.use_cls, self.norm_descs, self.gemm_engine)
        return packed, {t: packed[k] for k, t in enumerate(self.taps)}

    def __call__(self, img):
        """img [B,3,H,W] -> {(layer, facet): [B, (1 +) R + N, D]}; a list/tuple of differently sized images (as for
        DinoV2ExtractFeatures) -> {(layer, facet): [list of [n_i, D]]}.  All outputs are views of one allocation."""
        return self._guarded(img)


# ------------------------------------------------------------------ VLAD
def _as_device_f32(x, device):
    """x as a contiguous fp32 tensor on `device` whose data_ptr() is 16-byte aligned.  The kernels read rows with float4
    loads, and a contiguous view at an odd storage offset (`buf[1:].view(B, N, D)`) passes `.contiguous()` unchanged, so
    such a view is copied; every other tensor is returned as before."""
    if type(x) == np.ndarray:
        x = torch.from_numpy(x)
    x = x.detach().to(device=device, dtype=torch.float32).contiguous()
    return x if x.data_ptr() % 16 == 0 else x.clone()


def _packed_rows(items):
    """The [R, D] view of one buffer whose consecutive row ranges the items are, or None.  `ext(list)` and
    `DinoV2MultiExtractFeatures(list)` return such views of their packed output, and the packed aggregations read them
    in place.  Every item must be a 2-D fp32 tensor with unit column stride and rows D apart, on the storage of the
    first one, starting where the previous item ends; the first row must be 16-byte aligned (float4 loads)."""
    if not items or not all(isinstance(q, torch.Tensor) for q in items):
        return None
    first = items[0]
    if first.dim() != 2 or first.dtype != torch.float32:
        return None
    D = first.shape[1]
    storage, off = first.untyped_storage().data_ptr(), first.storage_offset()
    for q in items:
        if (q.dim() != 2 or q.dtype != torch.float32 or q.device != first.device or q.shape[1] != D
                or q.untyped_storage().data_ptr() != storage or q.storage_offset() != off):
            return None
        if q.shape[0] > 0 and (q.stride(1) != 1 and D > 1 or q.stride(0) != D and q.shape[0] > 1):
            return None
        off += q.shape[0] * D
    if first.data_ptr() % 16:
        return None
    R = sum(q.shape[0] for q in items)
    return first.detach().as_strided((R, D), (D, 1), first.storage_offset())


def _pack_list(items, device):
    """A list of [n_i, D] feature sets -> (feats [R, D] contiguous fp32 on `device`, row0, lens): image i is rows
    row0[i] .. row0[i] + lens[i] of feats.  Consecutive views of one buffer on `device` (_packed_rows) are passed as
    that buffer, without a copy; anything else is packed once with one torch.cat (host items through
    _as_device_f32)."""
    lens = [int(q.shape[0]) for q in items]
    row0 = [0] * len(items)
    for i in range(1, len(items)):
        row0[i] = row0[i - 1] + lens[i - 1]
    feats = _packed_rows(items)
    if feats is None or feats.device != torch.device(device):
        feats = torch.cat([_as_device_f32(q, device) for q in items])
        feats = feats if feats.data_ptr() % 16 == 0 else feats.clone()
    return feats, row0, lens


def _table_dev(row0, lens, dev):
    """row0 [B] int64 and len [B] int32 on `dev` (the packed entries' table)"""
    return (torch.tensor(row0, dtype=torch.int64).to(dev, non_blocking=True),
            torch.tensor(lens, dtype=torch.int32).to(dev, non_blocking=True))


def _normalize_rows_dev(x):
    """F.normalize(x) of a device matrix [R,D] (utilities.py:782-783)."""
    y = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _lib.check(_lib.load().anyloc_l2_normalize_rows(_lib.ptr(x), x.shape[0], x.shape[1], x.shape[1],
                                                        _lib.ptr(y), _lib.stream_ptr()), "l2_normalize_rows")
    return y


# ------------------------------------------------------------------ k-means on host rows larger than the device
_STAGE_BYTES = 1 << 30      # each of the two pinned staging buffers of a streamed fit: at most 2 GiB of host memory pinned


def _device_budget(dev, release_cache=True):
    """Device bytes a k-means fit or an index may allocate: free memory once torch has returned its unused cached
    segments, less a 1 GiB margin for the allocator and other work on the device.  Cached bytes inside partly used
    segments are not counted: a multi-GB allocation cannot be served from them.  release_cache=False leaves torch's
    cache alone and counts none of it, a lower bound for callers that only need to know that something fits."""
    if release_cache:
        torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(dev)
    return free - (1 << 30)


def _stream_rounds(R, chunks, rows_per, P):
    """The rounds of a streamed k-means pass over R rows split into `chunks` chunks of `rows_per` rows (the last may be
    shorter; anyloc_kmeans_partition): round j holds rows [c*rows_per + j*P, c*rows_per + (j+1)*P) of every chunk c,
    clipped to the chunk -> list of rounds, each a list of (first row, rows) per chunk.  Fed in order, the rounds give
    every chunk its rows in row order, the order in which anyloc_kmeans_update sums them."""
    rounds = []
    for j in range(-(-rows_per // P)):
        pieces = []
        for c in range(chunks):
            lo = c * rows_per + j * P
            pieces.append((lo, max(0, min(R, (c + 1) * rows_per, lo + P) - lo)))
        rounds.append(pieces)
    return rounds


def _kmeans_plan(R, D, chunks, rows_per, budget, copies, ws_bytes, stage_bytes):
    """Where a fit on R host rows of dimension D runs, given `budget` free device bytes.  -> None: in memory, when
    `copies` device copies of the rows plus `ws_bytes(R)` (workspaces and labels of an R-row pass) fit.  Else (P,
    resident): streamed in rounds of P rows per chunk (a round fills a `stage_bytes` staging buffer), the first
    `resident` rounds kept on the device after iteration 0 beside the labels of all rows and the round buffers."""
    row = 4 * D
    if copies * R * row + ws_bytes(R) <= budget:
        return None
    P = max(1, min(rows_per, stage_bytes // (chunks * row)))
    n_rounds = -(-rows_per // P)
    rr = chunks * P
    fixed = _kmeans_stream_bytes(R, D, chunks, P, copies, ws_bytes)
    return P, int(max(0, min(n_rounds, (budget - fixed) // (rr * row))))


def _kmeans_stream_bytes(R, D, chunks, P, copies, ws_bytes):
    """Device bytes of a streamed fit with no round resident: the workspaces and labels of one round of chunks * P
    rows, the labels of all R rows, two transfer buffers and the normalised round"""
    rr = chunks * P
    return ws_bytes(rr) + 4 * R + (1 + copies) * rr * 4 * D


def _kmeans_fit_plan(R, D, chunks, rows_per, budget, free, copies, ws_bytes, stage_bytes):
    """_kmeans_plan, with MemoryError naming the bytes when the streamed fit does not fit the `free` device bytes
    even with no round resident (the partial sums alone are chunks * K * D * 4 bytes: 403 MB at K = 1024, D = 1536)"""
    plan = _kmeans_plan(R, D, chunks, rows_per, budget, copies, ws_bytes, stage_bytes)
    if plan is not None:
        need = _kmeans_stream_bytes(R, D, chunks, plan[0], copies, ws_bytes)
        if need > free:
            raise MemoryError(f"VLAD.fit: the streamed k-means fit of {R} x {D} rows needs {need} bytes of device "
                              f"memory (workspaces, labels and round buffers), {free} are free")
    return plan


def _kmeans_tiled(K):
    """whether the k-means update takes the cluster-tiled kernels: anyloc_kmeans_update keeps (K * 128 + K) * 4 bytes
    of partial sums in shared memory and refuses K beyond them"""
    return (K * 128 + K) * 4 > _lib.KMEANS_SMEM_BYTES


# device bytes of torch.linalg.eigh (cuSOLVER syevd) on an m x m fp64 matrix, in 8 m^2 units: the matrix, the
# eigenvectors and the workspace, which cusolverDnXsyevd_bufferSize puts at 4.0 matrices (CUDA 12.8's cuSOLVER on an
# H100, m = 10 000 to 26 733)
_PCA_EIGH_MATRICES = 6
# the largest m that workspace query accepts there; from m = 26 734 on it returns CUSOLVER_STATUS_INVALID_VALUE
_PCA_EIGH_MAX_M = 26_733


def _pca_in_memory_bytes(n, d, n_held):
    """Peak device bytes of reduce_pca's in-memory route (_PcaDev) on n rows of dimension d, beside n_held more rows
    it holds: the fp32 rows and their centred fp32 and fp64 copies (16 n d), the other rows (4 n_held d), and the m x m
    fp64 matrix, m = min(n, d), with what eigh needs for it."""
    m = min(n, d)
    return 16 * n * d + 4 * n_held * d + 8 * _PCA_EIGH_MATRICES * m * m


def _pca_plan(n, d, n_held, budget, stage_bytes):
    """Where reduce_pca fits n rows of dimension d, beside n_held more rows, given `budget` free device bytes.
    -> None: in memory, when _pca_in_memory_bytes fits.  Else streamed (_PcaDev.fit_streamed): ("cov", P) for n > d,
    the rows fed in pieces of P rows; ("gram", W) for n <= d, the columns fed in slabs of W columns of all n rows.  A
    piece fills at most one `stage_bytes` staging buffer, and two device copies of it fit beside the m x m matrix.
    MemoryError when not even the m x m matrix and its eigh fit, or m is beyond _PCA_EIGH_MAX_M: reduce_pca has no
    top-k eigensolver."""
    if _pca_in_memory_bytes(n, d, n_held) <= budget:
        return None
    m = min(n, d)
    eig = 8 * _PCA_EIGH_MATRICES * m * m
    if m > _PCA_EIGH_MAX_M:
        raise MemoryError(f"reduce_pca: m = min(n_samples, n_features) = {m} is beyond the {_PCA_EIGH_MAX_M} x "
                          f"{_PCA_EIGH_MAX_M} fp64 matrices the eigensolver (torch.linalg.eigh, cuSOLVER syevd) takes; "
                          "svd_solver='randomized' has no such limit")
    if eig > budget:
        raise MemoryError(f"reduce_pca: the {m} x {m} fp64 Gram / covariance matrix (m = min(n_samples, n_features)) "
                          f"and its eigen-decomposition need {eig} bytes of device memory, {budget} are free; "
                          "svd_solver='randomized' needs far less")
    spare = (budget - 8 * m * m) // 2               # per device copy of a piece, beside the accumulating matrix
    if n > d:
        return "cov", int(max(1, min(n, stage_bytes // (4 * d), spare // (4 * d))))
    return "gram", int(max(1, min(d, stage_bytes // (4 * n), spare // (4 * n))))


_PCA_PIECE_MAX_ROWS = 1 << 20      # anyloc_pca_accumulate's "sketch" output has at most 2^20 rows


def _pca_randomized_bytes(n, d, l):
    """Peak device bytes of the randomized fit's matrices (_PcaDev.fit_randomized) beside its rows, l = k + 10: three
    fp64 [max(n, d), l] and three fp64 [min(n, d), l] (a pass's product, its LU factor and P L beside the basis the
    product came from; at the end Q, U = Q U^, B^T, its QR and vt), and the fp32 fit rows and components"""
    return 8 * l * (3 * max(n, d) + 3 * min(n, d)) + 4 * l * (n + d)


def _pca_randomized_plan(n, d, l, budget, stage_bytes):
    """Where reduce_pca's randomized fit (l = k + 10 test vectors) reads n rows of dimension d that are not device fp32
    already, given `budget` free device bytes.  -> None: uploaded once as fp32 [n, d], when that fits beside the fit's
    matrices (_pca_randomized_bytes) and, during the upload, beside two staging copies.  Else P: every pass streams the
    rows in pieces of P rows, a piece filling at most one `stage_bytes` staging buffer with two device copies beside the
    matrices.  MemoryError when not even the matrices and two one-row pieces fit."""
    mats = _pca_randomized_bytes(n, d, l)
    piece = 4 * d * max(1, min(n, stage_bytes // (4 * d)))
    if 4 * n * d + max(mats, 2 * piece) <= budget:
        return None
    if mats + 8 * d > budget:
        raise MemoryError(f"reduce_pca(svd_solver='randomized'): the fp64 [{max(n, d)}, {l}] and [{min(n, d)}, {l}] "
                          f"matrices of the randomized fit and their factorisations need {mats} bytes of device memory "
                          f"and a piece of one row {8 * d} more, {budget} are free")
    return int(max(1, min(n, _PCA_PIECE_MAX_ROWS, stage_bytes // (4 * d), (budget - mats) // (8 * d))))


def _pca_boxes(n, d, plan):
    """The pieces (r0, r1, c0, c1) of rows [n, d] a streamed PCA pass reads, in order: pieces of P rows over all
    columns ("cov", P), or slabs of P columns over all rows ("gram", P)"""
    route, P = plan
    if route == "cov":
        return [(r0, min(n, r0 + P), 0, d) for r0 in range(0, n, P)]
    return [(0, n, c0, min(d, c0 + P)) for c0 in range(0, d, P)]


def _host_fit_plan(X, dev, K, copies):
    """_kmeans_plan for host rows X on `dev`; None (the in-memory fit) for device rows."""
    return _host_plan(X, dev, [K], copies, lambda lib, n, D: lib.anyloc_vlad_workspace_bytes(1, n, D, K))


def _host_fit_plan_multi(X, dev, Ks, copies):
    """_host_fit_plan for vocabularies of Ks[v] clusters fitted together (fit_vocabularies): the shared assignment's
    workspace, every member's round workspace and one row of labels per member."""
    arr = (C.c_int * len(Ks))(*Ks)
    return _host_plan(X, dev, Ks, copies,
                      lambda lib, n, D: lib.anyloc_vlad_assign_multi_workspace_bytes(n, D, len(Ks), arr))


def _fit_ws_bytes(assign_bytes, upd_bytes, V):
    """ws_bytes(n) of _kmeans_plan for V vocabularies fitted together: the assignment workspace of an n-row pass, the
    members' round workspaces (upd_bytes in all; chunks * K * D partial sums each, whatever the round) and V rows of
    n labels"""
    return lambda n: assign_bytes(n) + upd_bytes + 4 * V * n


def _host_plan(X, dev, Ks, copies, assign_bytes):
    if dev.type != "cuda" or X.is_cuda:
        return None
    lib = _lib.load()
    R, D = X.shape
    with torch.cuda.device(dev):
        chunks, rows_per = _kmeans_partition(R, D)
        upd = sum(lib.anyloc_kmeans_round_workspace_bytes(R, D, K) for K in Ks)
        ws_bytes = _fit_ws_bytes(lambda n: assign_bytes(lib, n, D), upd, len(Ks))
        budget = _device_budget(dev)
        return _kmeans_fit_plan(R, D, chunks, rows_per, budget, torch.cuda.mem_get_info(dev)[0], copies, ws_bytes,
                                _STAGE_BYTES)


def _kmeans_partition(R, D):
    """(chunks, rows_per) of anyloc_kmeans_update on the current device"""
    chunks, rows_per = C.c_int(), C.c_int64()
    _lib.check(_lib.load().anyloc_kmeans_partition(R, D, C.byref(chunks), C.byref(rows_per)), "anyloc_kmeans_partition")
    return chunks.value, rows_per.value


class _KMeans:
    """GPU stand-in for `fast_pytorch_kmeans.KMeans` as the reference uses it (utilities.py:766,
    :772, :786-787, :849): `.centroids`, `.fit(X)`, `.predict(X)`; cosine / euclidean similarity,
    numpy-seeded random-choice init, <=100 Lloyd iterations, tol 1e-4."""

    def __init__(self, n_clusters, max_iter=100, tol=1e-4, verbose=0, mode="euclidean", minibatch=None):
        if mode not in _lib.DIST:
            raise NotImplementedError(mode)
        self.n_clusters, self.max_iter, self.tol, self.mode = n_clusters, max_iter, tol, mode
        self.verbose, self.minibatch = verbose, minibatch
        self.centroids = None

    def _assign(self, x, centers):
        lib = _lib.load()
        R, D = x.shape
        K = centers.shape[0]
        labels = torch.empty(R, dtype=torch.int32, device=x.device)
        with torch.cuda.device(x.device):
            ws = _lib.workspaces.get(x.device, lib.anyloc_vlad_workspace_bytes(1, R, D, K), "kmeans")
            _lib.check(lib.anyloc_vlad_assign(_lib.ptr(x), _lib.ptr(centers), R, D, K, _lib.DIST[self.mode],
                                              _lib.ptr(labels), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                       "anyloc_vlad_assign")
        return labels

    def _update(self, x, labels, c):
        """one Lloyd centroid update (anyloc_kmeans_update) -> (new centres, sum of squared centre shifts as a device
        tensor -- or a float, from a synchronous implementation)"""
        lib = _lib.load()
        n, D = x.shape
        K = c.shape[0]
        new_c = torch.empty_like(c)
        err = torch.zeros(1, device=x.device)
        with torch.cuda.device(x.device):
            ws = _lib.workspaces.get(x.device, lib.anyloc_kmeans_workspace_bytes(n, D, K), "kmeans_upd")
            if _kmeans_tiled(K):
                _lib.check(lib.anyloc_kmeans_update_tiled(_lib.ptr(x), _lib.ptr(labels), _lib.ptr(c), n, D, K, 0,
                                                          _lib.ptr(new_c), _lib.ptr(err), _lib.ptr(ws), ws.numel(),
                                                          _lib.stream_ptr()), "anyloc_kmeans_update_tiled")
            else:
                _lib.check(lib.anyloc_kmeans_update(_lib.ptr(x), _lib.ptr(labels), _lib.ptr(c), n, D, K,
                                                    _lib.ptr(new_c), _lib.ptr(err), _lib.ptr(ws), ws.numel(),
                                                    _lib.stream_ptr()), "anyloc_kmeans_update")
        return new_c, err              # err stays on the device: fit_predict reads it one iteration late

    def predict(self, X):
        dev = _lib.require_cuda(X.device if isinstance(X, torch.Tensor) and X.is_cuda else None)
        was_cpu = not (isinstance(X, torch.Tensor) and X.is_cuda)
        labels = self._assign(_as_device_f32(X, dev), _as_device_f32(self.centroids, dev)).to(torch.int64)
        return labels.cpu() if was_cpu else labels

    def fit_predict(self, X, centroids=None):
        dev = _lib.require_cuda(X.device if X.is_cuda else None)
        was_cpu = not X.is_cuda
        plan = _host_fit_plan(X, dev, self.n_clusters, copies=1)
        if plan is not None:
            return self._fit_streamed(X, centroids, False, plan, dev)
        x = _as_device_f32(X, dev)
        n, D = x.shape
        K = self.n_clusters
        if centroids is None:
            init = np.random.choice(n, size=[K], replace=False)      # numpy RNG, as upstream
            c = x[torch.from_numpy(init).to(dev)].contiguous()
        else:
            c = _as_device_f32(centroids, dev)
        # Lloyd iterations without a host sync on the critical path: iteration i+1 is enqueued BEFORE the convergence
        # test of iteration i is read (its error travels to pinned host memory behind an event), so the device never
        # idles on the host; when iteration i turns out to have converged, the speculative iteration is simply dropped
        # -- centres and labels are exactly those of the synchronous loop (fpk: break after the update whose shift <= tol)
        labels, pending = None, None            # pending = (labels_i, c_{i+1}, host error, event) of the previous iteration
        hosts = None
        for it in range(self.max_iter):
            labels_i = self._assign(x, c)
            c_next, err = self._update(x, labels_i, c)
            if not isinstance(err, torch.Tensor):                 # synchronous implementation (tests' CPU double)
                labels, c = labels_i, c_next
                if err <= self.tol:
                    break
                continue
            if hosts is None:
                hosts = [torch.empty(1, dtype=torch.float32).pin_memory() for _ in range(2)]
            host = hosts[it & 1]
            host.copy_(err, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            if pending is not None:
                pending[3].synchronize()
                if float(pending[2][0]) <= self.tol:               # the PREVIOUS iteration had converged
                    labels, c = pending[0], pending[1]
                    pending = None
                    break
            pending = (labels_i, c_next, host, ev)
            labels, c = labels_i, c_next
        if pending is not None:
            pending[3].synchronize()                               # results of the last enqueued iteration are final
        self.centroids = c.cpu() if was_cpu else c
        labels = labels.to(torch.int64)
        return labels.cpu() if was_cpu else labels

    def fit(self, X, centroids=None):
        self.fit_predict(X, centroids)

    def _fit_streamed(self, X, centroids, normalize, plan, dev):
        """fit_predict on host rows X [R,D] (any float dtype and strides) too large for the device, rows L2-normalised
        first when `normalize` (VLAD.fit).  Each Lloyd pass feeds the rows in rounds of P rows per chunk of the
        in-memory update (_RoundFeed), so centres and labels are bit-identical to the in-memory fit's.  The shift is
        read after every iteration: a speculative extra pass would cost a full transfer."""
        X = X.detach()
        R, D = X.shape
        K = self.n_clusters
        with torch.cuda.device(dev):
            if centroids is None:
                c = _streamed_init(X, K, normalize, dev)
            else:
                c = _as_device_f32(centroids, dev)
            feed = _RoundFeed(X, normalize, plan, dev, self.max_iter)
            ws = _lib.workspaces.get(dev, _lib.load().anyloc_kmeans_round_workspace_bytes(R, D, K), "kmeans_upd")
            for it in range(self.max_iter):
                labels_r = []
                for j, x in feed.iteration(it):
                    labels_r.append(self._assign(x, c))
                    _accumulate_round(x, labels_r[-1], R, feed.sizes[j], feed.piece[j], K, int(j > 0), ws)
                c_next, err = torch.empty_like(c), torch.zeros(1, device=dev)
                _finalize(c, R, c_next, err, ws)
                labels, c = labels_r, c_next
                if float(err) <= self.tol:
                    break
            feed.close()
            out = torch.empty(R, dtype=torch.int64)
            out[feed.order()] = torch.cat(labels).to(torch.int64).cpu()
        self.centroids = c.cpu()
        return out


def _streamed_init(X, K, normalize, dev):
    """the in-memory fit's random-choice init (numpy RNG), gathered from host rows X and normalised like the rows"""
    init = np.random.choice(X.shape[0], size=[K], replace=False)
    c = _as_device_f32(X[torch.from_numpy(init)], dev)
    return _normalize_rows_dev(c) if normalize else c


def _accumulate_round(x, labels, R, round_rows, piece, K, resume, ws):
    """one round of a K-cluster k-means sum (anyloc_kmeans_accumulate_round, or its tiled form for K >= 437)"""
    lib = _lib.load()
    D = x.shape[1]
    if _kmeans_tiled(K):
        _lib.check(lib.anyloc_kmeans_accumulate_round_tiled(_lib.ptr(x), _lib.ptr(labels), R, round_rows, piece, D, K,
                                                            0, resume, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                   "anyloc_kmeans_accumulate_round_tiled")
    else:
        _lib.check(lib.anyloc_kmeans_accumulate_round(_lib.ptr(x), _lib.ptr(labels), R, round_rows, piece, D, K,
                                                      resume, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                   "anyloc_kmeans_accumulate_round")


def _finalize(c, R, c_next, err, ws):
    """anyloc_kmeans_finalize: the centres c_next and the shift err [1] from the sums in ws"""
    K, D = c.shape
    _lib.check(_lib.load().anyloc_kmeans_finalize(_lib.ptr(c), R, D, K, _lib.ptr(c_next), _lib.ptr(err), _lib.ptr(ws),
                                                  ws.numel(), _lib.stream_ptr()), "anyloc_kmeans_finalize")


class _StagePair:
    """The double buffering of a streamed pass (_RoundFeed, _ImageFeed): per slot a pinned host buffer and a device
    buffer of `shape` fp32, and one copy stream.  fill(s, n, gather) waits until slot s's previous copy is done, lets
    gather(host) write the first n rows of its host buffer and queues their copy to the device behind the slot's last
    release; take(s, n) makes the current stream wait for that copy and returns the n device rows; release(s) records
    the work queued so far on the current stream as the rows' last use.  So the gather and copy of one slot overlap
    the device work on the other.  Built and used under torch.cuda.device(dev)."""

    def __init__(self, shape, dev, slots=2):
        self.host = [torch.empty(shape, pin_memory=True) for _ in range(slots)]
        self.raw = [torch.empty(shape, device=dev) for _ in range(slots)]
        self.cs, self.xs = torch.cuda.current_stream(), torch.cuda.Stream()
        self.copied, self.freed = [None] * slots, [None] * slots

    def fill(self, s, n, gather):
        if self.copied[s] is not None:
            self.copied[s].synchronize()                               # the staging buffer's previous copy is done
        gather(self.host[s])
        with torch.cuda.stream(self.xs):
            if self.freed[s] is not None:
                self.xs.wait_event(self.freed[s])
            self.raw[s][:n].copy_(self.host[s][:n], non_blocking=True)
            self.copied[s] = torch.cuda.Event()
            self.copied[s].record(self.xs)

    def take(self, s, n):
        self.cs.wait_event(self.copied[s])
        return self.raw[s][:n]

    def release(self, s):
        self.freed[s] = torch.cuda.Event()
        self.freed[s].record(self.cs)

    def close(self):
        self.xs.synchronize()


class _RoundFeed:
    """The rounds of a streamed k-means pass over host rows X [R,D] (any float dtype and strides), on the device, for
    plan (P, resident) of _kmeans_plan: round j holds P rows of every chunk of the in-memory update (_stream_rounds),
    chunk after chunk, so a pass that sums the rounds in order sums each chunk in row order.  Rows are L2-normalised
    on the device when `normalize`.  The first `resident` rounds are copied and normalised once, in iteration 0; the
    others cross the host link every iteration through two pinned staging buffers, the gather and copy of one round
    overlapping the device work on the one before.  A round crosses the link once per iteration however much work is
    enqueued on it.  Built and iterated under torch.cuda.device(dev)."""

    def __init__(self, X, normalize, plan, dev, max_iter):
        P, self.resident = plan
        self.X, self.normalize = X, normalize
        R, D = X.shape
        chunks, rows_per = _kmeans_partition(R, D)
        self.rounds = _stream_rounds(R, chunks, rows_per, P)
        self.piece = [pcs[0][1] for pcs in self.rounds]                # every chunk's piece but the last one's
        self.sizes = [(chunks - 1) * pcs[0][1] + pcs[-1][1] for pcs in self.rounds]
        self.offs = np.concatenate([[0], np.cumsum(self.sizes)]).tolist()
        self.kept = torch.empty(self.offs[self.resident], D, device=dev)
        self.pair = _StagePair((self.sizes[0], D), dev)
        self.transfers = ((it, j) for it in range(max_iter)
                          for j in range(0 if it == 0 else self.resident, len(self.rounds)))
        self.staged, self.taken = [], 0
        self._stage()

    def _stage(self):
        """gather the next transferred round into a staging buffer and queue its copy to the device"""
        t = next(self.transfers, None)
        if t is None:
            return
        j, s = t[1], len(self.staged) & 1
        piece = self.piece[j]

        def gather(host):
            for ci, (lo, m) in enumerate(self.rounds[j]):
                host[ci * piece:ci * piece + m].copy_(self.X[lo:lo + m])
        self.pair.fill(s, self.sizes[j], gather)
        self.staged.append((t, s))

    def iteration(self, it):
        """yields (j, x) for every round j of Lloyd iteration `it`, x [sizes[j], D] the round's rows on the device; the
        caller enqueues its work on x on the current stream before it asks for the next round"""
        for j in range(len(self.rounds)):
            x = self.kept[self.offs[j]:self.offs[j + 1]]
            moved = it == 0 or j >= self.resident
            if moved:
                t, s = self.staged[self.taken]
                self.taken += 1
                x = self.pair.take(s, self.sizes[j])
                if self.normalize:
                    x = _normalize_rows_dev(x)
                if j < self.resident:
                    self.kept[self.offs[j]:self.offs[j + 1]].copy_(x)
            yield j, x
            if moved:
                self.pair.release(s)
                self._stage()

    def close(self):
        self.pair.close()                                              # a round staged for an iteration not run

    def order(self):
        """the host row of every row of the rounds, in round order"""
        return torch.from_numpy(np.concatenate([np.arange(lo, lo + m) for pcs in self.rounds for lo, m in pcs]))


def _assign_multi(x, centres, mode):
    """labels [V, R] int32 of the rows x [R, D] against each of V centre sets (anyloc_vlad_assign_multi): row v is
    _KMeans._assign(x, centres[v]) bit for bit"""
    lib = _lib.load()
    R, D = x.shape
    V = len(centres)
    Ks = (C.c_int * V)(*[c.shape[0] for c in centres])
    ptrs = (C.c_void_p * V)(*[c.data_ptr() for c in centres])
    labels = torch.empty(V, R, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        ws = _lib.workspaces.get(x.device, lib.anyloc_vlad_assign_multi_workspace_bytes(R, D, V, Ks), "kmeans")
        _lib.check(lib.anyloc_vlad_assign_multi(_lib.ptr(x), R, D, V, ptrs, Ks, _lib.DIST[mode], _lib.ptr(labels),
                                                _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "anyloc_vlad_assign_multi")
    return labels


def _accumulate_round_multi(x, labels, Ks, ws, R, round_rows, piece, resume):
    """one round of the k-means sums of V vocabularies of Ks[v] clusters on the same rows x: the members below K = 437
    in one fused accumulate (anyloc_kmeans_accumulate_round_multi), the others in their own tiled round"""
    lib = _lib.load()
    D = x.shape[1]
    fused = [v for v, K in enumerate(Ks) if not _kmeans_tiled(K)]
    for v in range(len(Ks)):
        if v not in fused:
            _accumulate_round(x, labels[v], R, round_rows, piece, Ks[v], resume, ws[v])
    if fused:
        n = len(fused)
        _lib.check(lib.anyloc_kmeans_accumulate_round_multi(
            _lib.ptr(x), n, (C.c_void_p * n)(*[labels[v].data_ptr() for v in fused]),
            (C.c_int * n)(*[Ks[v] for v in fused]), R, round_rows, piece, D, resume,
            (C.c_void_p * n)(*[ws[v].data_ptr() for v in fused]), (C.c_size_t * n)(*[ws[v].numel() for v in fused]),
            _lib.stream_ptr()), "anyloc_kmeans_accumulate_round_multi")


def _finalize_multi(c, R, ws):
    """anyloc_kmeans_finalize of every member -> (new centres, shifts [V] on the device)"""
    nxt = [torch.empty_like(ci) for ci in c]
    err = torch.zeros(len(c), device=c[0].device)
    for v in range(len(c)):
        _finalize(c[v], R, nxt[v], err[v:v + 1], ws[v])
    return nxt, err


def _lloyd_in_memory(kms, x, inits):
    """the Lloyd loops of several k-means (kms, one _KMeans each, inits their random-choice draws) on the same device
    rows x, each centre set bit for bit what kms[v].fit(x) gives.  Each iteration assigns the rows to every active
    vocabulary at once and sums them in one fused pass.  As in fit_predict, iteration i + 1 is enqueued before the
    shifts of iteration i are read; a member whose shift was within its tol keeps the centres of iteration i and takes
    no part in later passes."""
    R, D = x.shape
    dev = x.device
    n = len(kms)
    with torch.cuda.device(dev):
        c = [x[torch.from_numpy(i).to(dev)].contiguous() for i in inits]
        ws = [torch.empty(_lib.load().anyloc_kmeans_round_workspace_bytes(R, D, km.n_clusters), dtype=torch.uint8,
                          device=dev) for km in kms]
        _, rows_per = _kmeans_partition(R, D)
        final = [None] * n
        hosts = [torch.empty(n, dtype=torch.float32).pin_memory() for _ in range(2)]
        pending = None                              # (members, their next centres, host shifts, event) of iteration i
        for it in range(max(km.max_iter for km in kms)):
            act = [m for m in range(n) if final[m] is None and it < kms[m].max_iter]
            if not act:
                break
            labels = _assign_multi(x, [c[m] for m in act], kms[0].mode)
            _accumulate_round_multi(x, labels, [kms[m].n_clusters for m in act], [ws[m] for m in act], R, R,
                                    rows_per, 0)
            nxt, err = _finalize_multi([c[m] for m in act], R, [ws[m] for m in act])
            host = hosts[it & 1]
            host[:len(act)].copy_(err, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            if pending is not None:
                pending[3].synchronize()
                for i, m in enumerate(pending[0]):
                    if final[m] is None and float(pending[2][i]) <= kms[m].tol:     # converged in the previous one
                        final[m] = pending[1][i]
            pending = (act, nxt, host, ev)
            for i, m in enumerate(act):
                c[m] = nxt[i]
        if pending is not None:
            pending[3].synchronize()
        return [c[m] if final[m] is None else final[m] for m in range(n)]


def _lloyd_streamed(kms, X, normalize, plan, dev):
    """_lloyd_in_memory on host rows X too large for the device (plan of _host_fit_plan_multi), rows normalised on
    the device when `normalize`: every round of _RoundFeed crosses the link once per iteration and is assigned and
    summed for all active members before the next.  The shifts are read after every iteration, as in _fit_streamed.
    The members' random-choice draws are taken here, in member order."""
    R, D = X.shape
    n = len(kms)
    with torch.cuda.device(dev):
        c = [_streamed_init(X, km.n_clusters, normalize, dev) for km in kms]
        feed = _RoundFeed(X, normalize, plan, dev, max(km.max_iter for km in kms))
        ws = [torch.empty(_lib.load().anyloc_kmeans_round_workspace_bytes(R, D, km.n_clusters), dtype=torch.uint8,
                          device=dev) for km in kms]
        final = [None] * n
        for it in range(max(km.max_iter for km in kms)):
            act = [m for m in range(n) if final[m] is None and it < kms[m].max_iter]
            if not act:
                break
            for j, x in feed.iteration(it):
                labels = _assign_multi(x, [c[m] for m in act], kms[0].mode)
                _accumulate_round_multi(x, labels, [kms[m].n_clusters for m in act], [ws[m] for m in act], R,
                                        feed.sizes[j], feed.piece[j], int(j > 0))
            nxt, err = _finalize_multi([c[m] for m in act], R, [ws[m] for m in act])
            err = err.cpu()
            for i, m in enumerate(act):
                c[m] = nxt[i]
                if float(err[i]) <= kms[m].tol:
                    final[m] = c[m]
        feed.close()
        return c


VLAD_KERNEL_DESCRIPTION = ("VLAD: gemm_tc3_kernel<false, 0> (wgmma tf32 coarse scores straight from the fp32 features) -> "
                           "vlad_rescore_kernel (exact fp32 re-scoring of the candidates within the tf32 bound + row norms) "
                           "-> vlad_accumulate3_kernel (label-sorted residual sums + fused normalisation); prepared "
                           "vocabulary, 3 launches")


class VLAD:
    """Hard- and soft-assignment VLAD with the reference's constructor and methods (utilities.py:624-1008).

    `generate` / `generate_multi` take what the reference takes (CPU tensors / numpy arrays /
    ragged lists) and return what it returns (CPU tensors); CUDA tensors are also accepted and
    then stay on the device (the batched fast path).  The on-disk caches are honoured in the
    reference's own file formats: the vocabulary (`c_centers.pt`), and per image the labels
    (`<id>_l.pt`) / soft assignment (`<id>_s.pt`) and residual tensor (`<id>_r.pt`) are READ when
    present; labels / soft assignments are written like the reference does, the residual tensor
    (>=100 MB per image at ViT-G, K=32) only when `self.cache_residuals = True` or through
    `generate_res_vec(..., cache_id)`.  `vlad_mode="soft"` follows the reference's soft branch
    (:862-887), including its summation over the residuals to all centres."""

    def __init__(self, num_clusters: int, desc_dim: Union[int, None] = None, intra_norm: bool = True,
                 norm_descs: bool = True, dist_mode: str = "cosine", vlad_mode: str = "hard",
                 soft_temp: float = 1.0, cache_dir: Union[str, None] = None) -> None:
        self.num_clusters = num_clusters
        self.desc_dim = desc_dim
        self.intra_norm = intra_norm
        self.norm_descs = norm_descs
        self.mode = dist_mode
        self.vlad_mode = str(vlad_mode).lower()
        assert self.vlad_mode in ["soft", "hard"]
        self.soft_temp = soft_temp
        self.c_centers = None
        self.kmeans = None
        self._centers_dev = {}
        self._prepared_dev = None
        self.cache_residuals = False     # extension: write `<id>_r.pt` like the reference (104 MB per image at c2)
        self.cache_dir = cache_dir
        if self.cache_dir is not None:
            self.cache_dir = os.path.abspath(os.path.expanduser(self.cache_dir))
            if not os.path.exists(self.cache_dir):
                os.makedirs(self.cache_dir)
                print(f"Created cache directory: {self.cache_dir}")
            else:
                print(f"Warning: Cache directory already exists: {self.cache_dir}")
        else:
            print("VLAD caching is disabled.")

    # -- cache predicates (utilities.py:688-746)
    def can_use_cache_vlad(self):
        if self.cache_dir is None or not os.path.exists(self.cache_dir):
            return False
        return os.path.exists(f"{self.cache_dir}/c_centers.pt")

    def can_use_cache_ids(self, cache_ids: Union[List[str], str, None], only_residuals: bool = False) -> bool:
        if not self.can_use_cache_vlad() or cache_ids is None:
            return False
        if isinstance(cache_ids, str):
            cache_ids = [cache_ids]
        suffix = "l" if self.vlad_mode == "hard" else "s"
        for cid in cache_ids:
            if not os.path.exists(f"{self.cache_dir}/{cid}_r.pt"):
                return False
            if not only_residuals and not os.path.exists(f"{self.cache_dir}/{cid}_{suffix}.pt"):
                return False
        return True

    # -- vocabulary (utilities.py:749-791)
    def fit(self, train_descs: Union[np.ndarray, torch.Tensor, None]):
        if self._fit_from_cache():
            return
        if train_descs is None:
            raise ValueError("No training descriptors given")
        if type(train_descs) == np.ndarray:
            train_descs = torch.from_numpy(train_descs).to(torch.float32)
        if self.desc_dim is None:
            self.desc_dim = train_descs.shape[1]
        dev = _lib.require_cuda(train_descs.device if train_descs.is_cuda else None)
        was_cpu = not train_descs.is_cuda
        plan = _host_fit_plan(train_descs, dev, self.num_clusters, copies=1 + bool(self.norm_descs))
        if plan is not None:        # too large for the device: normalised round by round inside the streamed fit
            self.kmeans._fit_streamed(train_descs, None, self.norm_descs, plan, dev)
        else:
            x = _as_device_f32(train_descs, dev)
            if self.norm_descs:
                x = _normalize_rows_dev(x)
            self.kmeans.fit(x)
        self._set_vocabulary(self.kmeans.centroids.cpu() if was_cpu else self.kmeans.centroids)

    def _fit_from_cache(self):
        """the start of fit: a fresh k-means, and the cached vocabulary when there is one -> whether it was loaded"""
        self.kmeans = _KMeans(self.num_clusters, mode=self.mode)
        self._centers_dev = {}
        self._prepared_dev = None
        if not self.can_use_cache_vlad():
            return False
        print("Using cached cluster centers")
        self.c_centers = torch.load(f"{self.cache_dir}/c_centers.pt")
        self.kmeans.centroids = self.c_centers
        if self.desc_dim is None:
            self.desc_dim = self.c_centers.shape[1]
            print(f"Desc dim set to {self.desc_dim}")
        return True

    def _set_vocabulary(self, c):
        """the end of fit: the fitted centres c, written to the cache directory when there is one"""
        self.c_centers = c
        self.kmeans.centroids = self.c_centers
        if self.cache_dir is not None:
            print("Caching cluster centers")
            torch.save(self.c_centers.cpu(), f"{self.cache_dir}/c_centers.pt")

    def fit_and_generate(self, train_descs: Union[np.ndarray, torch.Tensor]) -> torch.Tensor:
        if type(train_descs) == np.ndarray:
            train_descs = torch.from_numpy(train_descs).to(torch.float32)
        self.fit(train_descs.reshape(-1, train_descs.shape[-1]))
        return self.generate_multi(train_descs)

    # -- device plumbing
    def _centers_on(self, dev):
        cc = self.c_centers
        key = (dev.index, id(cc), getattr(cc, "_version", None), cc.data_ptr() if isinstance(cc, torch.Tensor) else None)
        if key not in self._centers_dev:
            self._centers_dev = {key: _as_device_f32(self.c_centers, dev)}
        return self._centers_dev[key]

    def _prepared_on(self, dev, centers):
        """Device blob of anyloc_vlad_prepare for the current vocabulary (recomputed when c_centers is replaced or
        modified in place, or the distance mode changes)."""
        cc = self.c_centers
        key = (dev.index, id(cc), getattr(cc, "_version", None), self.mode, centers.data_ptr())
        cache = getattr(self, "_prepared_dev", None)
        if cache is None or cache[0] != key:
            lib = _lib.load()
            K, D = centers.shape
            blob = torch.empty(lib.anyloc_vlad_prepared_bytes(D, K), dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.anyloc_vlad_prepare(_lib.ptr(centers), D, K, _lib.DIST[self.mode], _lib.ptr(blob),
                                                   blob.numel(), _lib.stream_ptr()), "anyloc_vlad_prepare")
            self._prepared_dev = cache = (key, blob)
        return cache[1]

    def _run(self, feats, n_valid, dev, want_labels=False):
        """feats [B,N,D] device fp32; n_valid [B] int32 device or None -> ([B,K*D], labels|None)
        (soft mode: the [B,N,K] assignment probabilities take the place of the labels)."""
        assert self.kmeans is not None
        assert self.c_centers is not None
        lib = _lib.load()
        B, N, D = feats.shape
        K = self.num_clusters
        centers = self._centers_on(dev)
        if centers.shape != (K, D):
            raise ValueError(f"cluster centres {tuple(centers.shape)} do not match K={K}, D={D}")
        out = torch.empty(B, K * D, device=dev, dtype=torch.float32)
        labels = torch.empty(B, N, device=dev, dtype=torch.int32) if want_labels else None
        if self.vlad_mode == "soft":        # utilities.py:862-887
            assign = torch.empty(B, N, K, device=dev, dtype=torch.float32) if want_labels else None
            with torch.cuda.device(dev):
                ws = _lib.workspaces.get(dev, lib.anyloc_vlad_workspace_bytes(B, N, D, K), "vlad")
                rc = lib.anyloc_vlad_generate_soft(_lib.ptr(feats), _lib.ptr(n_valid), _lib.ptr(centers), B, N, D, K,
                                                   float(self.soft_temp), int(bool(self.norm_descs)),
                                                   int(bool(self.intra_norm)), _lib.ptr(out), _lib.ptr(assign),
                                                   _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
            _lib.check(rc, "anyloc_vlad_generate_soft")
            return out, assign
        # the sorted route only for shapes the shared-memory accumulations refuse: every other shape keeps its bits
        sorted_route = lib.anyloc_vlad_generate_route(B, N, D, K) == _lib.VLAD_ROUTE_SORTED
        generate, name, ws_bytes = ((lib.anyloc_vlad_generate_sorted, "anyloc_vlad_generate_sorted",
                                     lib.anyloc_vlad_sorted_workspace_bytes) if sorted_route else
                                    (lib.anyloc_vlad_generate_prepared, "anyloc_vlad_generate_prepared",
                                     lib.anyloc_vlad_workspace_bytes))
        with torch.cuda.device(dev):
            ws = _lib.workspaces.get(dev, ws_bytes(B, N, D, K), "vlad")
            prep = self._prepared_on(dev, centers)
            rc = generate(_lib.ptr(feats), _lib.ptr(n_valid), _lib.ptr(centers), _lib.ptr(prep), prep.numel(), B, N, D,
                          K, _lib.DIST[self.mode], int(bool(self.norm_descs)), int(bool(self.intra_norm)),
                          _lib.ptr(out), _lib.ptr(labels), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, name)
        return out, labels

    def _run_varlen(self, feats, row0, lens, dev, want_labels=False):
        """feats [R,D] device fp32 holding image i at rows row0[i] .. + lens[i] -> ([B,K*D], labels [R] | None); each
        descriptor is bitwise _run's on the padded batch [B, max(lens), D] with n_valid = lens (soft mode: the [R,K]
        assignment in place of the labels).  One launch sequence whatever B is, and no padded copy."""
        assert self.kmeans is not None
        assert self.c_centers is not None
        lib = _lib.load()
        R, D = feats.shape
        B, K = len(lens), self.num_clusters
        centers = self._centers_on(dev)
        if centers.shape != (K, D):
            raise ValueError(f"cluster centres {tuple(centers.shape)} do not match K={K}, D={D}")
        out = torch.empty(B, K * D, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            r0, ln = _table_dev(row0, lens, dev)
            if self.vlad_mode == "soft":
                assign = torch.empty(R, K, device=dev, dtype=torch.float32) if want_labels else None
                ws = _lib.workspaces.get(dev, lib.anyloc_vlad_soft_varlen_workspace_bytes(R, B, D, K), "vlad")
                rc = lib.anyloc_vlad_generate_soft_varlen(
                    _lib.ptr(feats), R, _lib.ptr(r0), _lib.ptr(ln), B, _lib.ptr(centers), D, K, float(self.soft_temp),
                    int(bool(self.norm_descs)), int(bool(self.intra_norm)), _lib.ptr(out), _lib.ptr(assign),
                    _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
                _lib.check(rc, "anyloc_vlad_generate_soft_varlen")
                return out, assign
            labels = torch.empty(R, device=dev, dtype=torch.int32) if want_labels else None
            ws = _lib.workspaces.get(dev, lib.anyloc_vlad_varlen_workspace_bytes(R, B, max(lens), D, K), "vlad")
            prep = self._prepared_on(dev, centers)
            rc = lib.anyloc_vlad_generate_varlen(
                _lib.ptr(feats), R, _lib.ptr(r0), _lib.ptr(ln), B, _lib.ptr(centers), _lib.ptr(prep), prep.numel(), D, K,
                _lib.DIST[self.mode], int(bool(self.norm_descs)), int(bool(self.intra_norm)), _lib.ptr(out),
                _lib.ptr(labels), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "anyloc_vlad_generate_varlen")
        return out, labels

    # -- per-image cache (utilities.py:843-852 labels, :864-878 soft assignment, :951-970 residuals)
    def _cache_path(self, cache_id, suffix):
        return f"{self.cache_dir}/{cache_id}_{suffix}.pt"

    def _cache_active(self, cache_id):
        return cache_id is not None and self.can_use_cache_vlad()

    def _residuals_dev(self, x, dev):
        """x [N,D] device fp32 -> residual tensor [N,K,D] on the device (anyloc_vlad_residuals)."""
        centers = self._centers_on(dev)
        N, D = x.shape
        K = centers.shape[0]
        if centers.shape[1] != D:
            raise ValueError(f"cluster centres {tuple(centers.shape)} do not match descriptor dim {D}")
        out = torch.empty(N, K, D, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(_lib.load().anyloc_vlad_residuals(_lib.ptr(x), _lib.ptr(centers), N, D, K,
                                                         int(bool(self.norm_descs)), _lib.ptr(out), _lib.stream_ptr()),
                       "anyloc_vlad_residuals")
        return out

    def _from_residuals_dev(self, resid, labels, assign, dev):
        """descriptor [K*D] (device) of one image from its residual tensor + hard labels | soft assignment"""
        lib = _lib.load()
        N, K, D = resid.shape
        out = torch.empty(K * D, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            ws = _lib.workspaces.get(dev, lib.anyloc_vlad_from_residuals_workspace_bytes(D, K), "vlad_cache")
            _lib.check(lib.anyloc_vlad_from_residuals(_lib.ptr(resid), _lib.ptr(labels), _lib.ptr(assign), N, D, K,
                                                      int(bool(self.intra_norm)), _lib.ptr(out), _lib.ptr(ws),
                                                      ws.numel(), _lib.stream_ptr()), "anyloc_vlad_from_residuals")
        return out

    def _generate_cached(self, query_descs, cache_id, dev):
        """The reference's cache-aware path, file for file: residuals from `<id>_r.pt` when present (else computed
        from the features; written back only when `self.cache_residuals`), labels from `<id>_l.pt` / soft assignment
        from `<id>_s.pt` when present (else computed AND saved, like the reference).  Files are CPU tensors in the
        reference's own format, so a directory populated by either implementation serves both.  -> [K*D] device."""
        suffix = "l" if self.vlad_mode == "hard" else "s"
        have_r = os.path.isfile(self._cache_path(cache_id, "r"))
        have_a = os.path.isfile(self._cache_path(cache_id, suffix))
        x = None
        if query_descs is not None:
            x = _as_device_f32(query_descs, dev)
        elif not (have_r and have_a):
            raise ValueError(f"no descriptors given and the cache of {cache_id!r} is incomplete")
        if not have_r and not have_a and not getattr(self, "cache_residuals", False):
            # nothing cached yet: the fused fast path, keeping the assignment for the next run
            out, assign = self._run(x.unsqueeze(0), None, dev, want_labels=True)
            self._save_assignment(cache_id, suffix, assign[0])
            return out[0]
        if have_r:
            resid = torch.load(self._cache_path(cache_id, "r")).to(device=dev, dtype=torch.float32).contiguous()
        else:
            resid = self._residuals_dev(x, dev)
            if getattr(self, "cache_residuals", False):
                cid_dir = f"{self.cache_dir}/{os.path.split(cache_id)[0]}"
                if not os.path.isdir(cid_dir):
                    os.makedirs(cid_dir)
                    print(f"Created directory: {cid_dir}")
                torch.save(resid.cpu(), self._cache_path(cache_id, "r"))
        if have_a:
            assign = torch.load(self._cache_path(cache_id, suffix)).to(dev)
        else:
            _, assign = self._run(x.unsqueeze(0), None, dev, want_labels=True)
            assign = assign[0]
            self._save_assignment(cache_id, suffix, assign)
        if self.vlad_mode == "hard":
            return self._from_residuals_dev(resid, assign.to(torch.int32).contiguous(), None, dev)
        return self._from_residuals_dev(resid, None, assign.to(torch.float32).contiguous(), dev)

    def _save_assignment(self, cache_id, suffix, assign):
        cid_dir = f"{self.cache_dir}/{os.path.split(cache_id)[0]}"
        if not os.path.isdir(cid_dir):
            os.makedirs(cid_dir)
            print(f"Created directory: {cid_dir}")
        # the reference stores kmeans.predict's int64 labels / the fp32 [q, c] soft assignment, on the CPU
        a = assign.to(torch.int64) if suffix == "l" else assign
        torch.save(a.cpu(), self._cache_path(cache_id, suffix))

    # -- descriptors (utilities.py:819-926)
    def generate(self, query_descs: Union[np.ndarray, torch.Tensor, None], cache_id: Union[str, None] = None) \
            -> torch.Tensor:
        on_dev = isinstance(query_descs, torch.Tensor) and query_descs.is_cuda
        dev = _lib.require_cuda(query_descs.device if on_dev else None)
        if self._cache_active(cache_id):
            out = self._generate_cached(query_descs, cache_id, dev)
            return out if on_dev else out.cpu()
        x = _as_device_f32(query_descs, dev)
        out, _ = self._run(x.unsqueeze(0), None, dev)
        return out[0] if on_dev else out[0].cpu()

    def generate_multi(self, multi_query: Union[np.ndarray, torch.Tensor, list],
                       cache_ids: Union[List[str], None] = None) -> Union[torch.Tensor, list]:
        if cache_ids is not None and self.can_use_cache_vlad() and any(c is not None for c in cache_ids):
            # cache-aware: image by image like the reference (:917-918); `multi_query` may be [None] * n when
            # can_use_cache_ids() said the cache is complete (scripts/dino_v2_vlad.py:224-228)
            res = [self.generate(q, c) for (q, c) in zip(multi_query, cache_ids)]
            return torch.stack(res)
        if isinstance(multi_query, (list, tuple)):
            if len(multi_query) == 0:
                return torch.stack([])      # same failure as the reference on an empty list
            on_dev = all(isinstance(q, torch.Tensor) and q.is_cuda for q in multi_query)
            dev = _lib.require_cuda(multi_query[0].device if on_dev else None)
            # packed: the items' rows in one [R, D] buffer (ext(list)'s own, when the items are its views)
            feats, row0, lens = _pack_list(multi_query, dev)
            out, _ = self._run_varlen(feats, row0, lens, dev)
            return out if on_dev else out.cpu()
        was_np = type(multi_query) == np.ndarray
        on_dev = isinstance(multi_query, torch.Tensor) and multi_query.is_cuda
        dev = _lib.require_cuda(multi_query.device if on_dev else None)
        if not on_dev and not was_np and multi_query.numel() * 4 > self._host_chunk_bytes:
            # large host batches (the driver hands over [n_imgs, n_patches, D] on the CPU): stream chunks
            step = max(1, self._host_chunk_bytes // (multi_query[0].numel() * 4))
            return torch.cat([self._run(_as_device_f32(multi_query[i:i + step], dev), None, dev)[0].cpu()
                              for i in range(0, multi_query.shape[0], step)])
        out, _ = self._run(_as_device_f32(multi_query, dev), None, dev)
        return out if on_dev else out.cpu()

    _host_chunk_bytes = 1 << 30

    # -- residual tensors (utilities.py:928-1008)
    def generate_res_vec(self, query_descs: Union[np.ndarray, torch.Tensor],
                         cache_id: Union[str, None] = None) -> torch.Tensor:
        assert self.kmeans is not None
        assert self.c_centers is not None
        if self._cache_active(cache_id) and os.path.isfile(self._cache_path(cache_id, "r")):
            return torch.load(self._cache_path(cache_id, "r"))
        on_dev = isinstance(query_descs, torch.Tensor) and query_descs.is_cuda
        dev = _lib.require_cuda(query_descs.device if on_dev else None)
        resid = self._residuals_dev(_as_device_f32(query_descs, dev), dev)
        resid = resid if on_dev else resid.cpu()
        if self._cache_active(cache_id):           # explicit request for the residual tensor: cache it as the reference does
            cid_dir = f"{self.cache_dir}/{os.path.split(cache_id)[0]}"
            if not os.path.isdir(cid_dir):
                os.makedirs(cid_dir)
                print(f"Created directory: {cid_dir}")
            torch.save(resid.cpu(), self._cache_path(cache_id, "r"))
        return resid

    def generate_multi_res_vec(self, multi_query: Union[np.ndarray, torch.Tensor, list],
                               cache_ids: Union[List[str], None] = None) -> Union[torch.Tensor, list]:
        if cache_ids is None:
            cache_ids = [None] * len(multi_query)
        res = [self.generate_res_vec(q, c) for (q, c) in zip(multi_query, cache_ids)]
        try:
            return torch.stack(res)
        except (TypeError, RuntimeError):
            return res              # ragged inputs stay a list


# ------------------------------------------------------------------ sibling aggregators (extension)
def fit_vocabularies(vlads: List[VLAD], train_descs: Union[np.ndarray, torch.Tensor]) -> None:
    """Fit every VLAD in `vlads` from one pass over `train_descs` per Lloyd iteration (extension: a sweep over the
    vocabulary size, such as the reference's ablations over num_clusters, otherwise reads the rows once per K).

    `train_descs` is what VLAD.fit takes: numpy, CPU or CUDA tensor, any float dtype or strides, host rows larger than
    the device.  Afterwards every member is in exactly the state `for v in vlads: v.fit(train_descs)` leaves it in,
    from the same numpy RNG state: c_centers (on the input's device), kmeans.centroids, desc_dim, the c_centers.pt of
    a member with a cache_dir, and the numpy RNG state itself (the random-choice inits are drawn in member order).  A
    member with cached centres loads them, draws nothing and takes no part in the pass; so does a member whose
    cache_dir an earlier member writes, once that member's centres are saved.  Each member keeps its own
    iteration count and convergence test and drops out of the passes once converged.

    The members must agree in norm_descs and dist_mode (they share the normalised rows and the score GEMM); vlad_mode
    and soft_temp do not enter the fit.  ValueError for an empty list, a VLAD listed twice or members that differ."""
    vlads = _check_members(vlads, "fit_vocabularies", "the rows and the scores")
    todo, later, written = [], [], set()
    for v in vlads:
        if v.cache_dir is not None and v.cache_dir in written:
            later.append(v)         # its own fit would load the centres an earlier member writes there
        elif not v._fit_from_cache():
            todo.append(v)
            if v.cache_dir is not None:
                written.add(v.cache_dir)
    if not todo:
        return
    if train_descs is None:
        raise ValueError("No training descriptors given")
    if type(train_descs) == np.ndarray:
        train_descs = torch.from_numpy(train_descs).to(torch.float32)
    for v in todo:
        if v.desc_dim is None:
            v.desc_dim = train_descs.shape[1]
    dev = _lib.require_cuda(train_descs.device if train_descs.is_cuda else None)
    was_cpu = not train_descs.is_cuda
    kms, norm = [v.kmeans for v in todo], bool(todo[0].norm_descs)
    plan = _host_fit_plan_multi(train_descs, dev, [km.n_clusters for km in kms], copies=1 + norm)
    if plan is not None:        # too large for the device: streamed, each round shared by all members
        centres = _lloyd_streamed(kms, train_descs.detach(), norm, plan, dev)
    else:
        x = _as_device_f32(train_descs, dev)
        if norm:
            x = _normalize_rows_dev(x)
        inits = [np.random.choice(x.shape[0], size=[km.n_clusters], replace=False) for km in kms]
        centres = _lloyd_in_memory(kms, x, inits)
    for v, c in zip(todo, centres):
        v._set_vocabulary(c.cpu() if was_cpu else c)
    for v in later:
        v._fit_from_cache()


def _check_members(vlads, who, what):
    """the rules fit_vocabularies and generate_vocabularies share: a non-empty list of distinct VLADs that agree in
    norm_descs and dist_mode -> the list"""
    vlads = list(vlads)
    if not vlads:
        raise ValueError(f"{who}: no VLAD given")
    first, twice = {}, []
    for i, v in enumerate(vlads):
        if id(v) in first:
            twice.append(f"{first[id(v)]} and {i}")
        first.setdefault(id(v), i)
    if twice:
        raise ValueError(f"{who}: the same VLAD is listed more than once (members {', '.join(twice)})")
    key = (bool(vlads[0].norm_descs), vlads[0].mode)
    odd = [i for i, v in enumerate(vlads) if (bool(v.norm_descs), v.mode) != key]
    if odd:
        raise ValueError(f"{who}: members {odd} differ from member 0 (norm_descs={key[0]}, dist_mode={key[1]!r}) in "
                         f"norm_descs or dist_mode; the members share {what}")
    return vlads


def _generate_call_images(v, X, host_tensor):
    """the images per call that v.generate_multi(X) makes on a [n, N, D] input: a host tensor larger than
    v._host_chunk_bytes in chunks of that size, anything else in one call"""
    n, N, D = X.shape
    if host_tensor and n * N * D * 4 > v._host_chunk_bytes:
        return max(1, v._host_chunk_bytes // (N * D * 4))
    return max(1, n)


def _generate_pieces(i0, i1, steps, N):
    """images [i0, i1) cut wherever one of member v's generate_multi calls ends (steps[v] = (images per call, n)) ->
    [(p0, p1, route_rows)], route_rows[v] = the rows of member v's call that holds images p0 .. p1: their count picks
    the member's assignment route"""
    cuts = sorted({i0, i1} | {c for s, _ in steps for c in range((i0 // s + 1) * s, i1, s)})
    return [(p0, p1, [N * (min(n, (p0 // s + 1) * s) - p0 // s * s) for s, n in steps])
            for p0, p1 in zip(cuts[:-1], cuts[1:])]


def _generate_chunk_bytes(b, N, D, hard_Ks, soft_Ks, staged):
    """device bytes of a chunk of b images [b, N, D] in generate_vocabularies: its features (two staging copies when
    they come from the host), every member's descriptors, the hard members' labels, 1/|x| and shared assignment
    workspace, the soft members' assignments, 1/|x| and centres, and the largest accumulation workspace"""
    lib = _lib.load()
    R = b * N
    need = 4 * b * D * (sum(hard_Ks) + sum(soft_Ks)) + (2 * 4 * R * D if staged else 0)
    if hard_Ks:
        need += (lib.anyloc_vlad_label_multi_workspace_bytes(R, D, len(hard_Ks), (C.c_int * len(hard_Ks))(*hard_Ks))
                 + 4 * R * (len(hard_Ks) + 1))
    if soft_Ks:
        need += (lib.anyloc_vlad_soft_assign_multi_workspace_bytes(D, len(soft_Ks), (C.c_int * len(soft_Ks))(*soft_Ks))
                 + 4 * R * (sum(soft_Ks) + 1))
    return need + max([lib.anyloc_vlad_accumulate_workspace_bytes(b, N, D, K, 0) for K in hard_Ks] +
                      [lib.anyloc_vlad_accumulate_workspace_bytes(b, N, D, K, 1) for K in soft_Ks])


def _generate_plan(n, N, D, hard_Ks, soft_Ks, staged, budget, cap):
    """images per chunk of generate_vocabularies on [n, N, D] features: the most, up to `cap`, whose
    _generate_chunk_bytes fit `budget`.  MemoryError naming the bytes when not even one image fits."""
    need1 = _generate_chunk_bytes(1, N, D, hard_Ks, soft_Ks, staged)
    if need1 > budget:
        raise MemoryError(f"generate_vocabularies: one image of {N} x {D} features needs {need1} bytes of device "
                          f"memory (its features, every member's descriptor and the workspaces), {budget} are free")
    lo, hi = 1, max(1, min(n, cap))
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if _generate_chunk_bytes(mid, N, D, hard_Ks, soft_Ks, staged) <= budget:
            lo = mid
        else:
            hi = mid - 1
    return lo


def _generate_shared(vlads, x, outs, dev, route_rows=None, table=None):
    """every member's descriptors of the device features x into outs[v] [B, K_v * D]: padded x [B, N, D] with
    route_rows[v] (the rows of member v's own call), or packed x [R, D] with table = (row0, lens).  The hard members'
    labels and 1/|x| come from one anyloc_vlad_label_multi, the soft members' assignments from one
    anyloc_vlad_soft_assign_multi, then each member accumulates alone."""
    lib = _lib.load()
    D = x.shape[-1]
    if table is None:
        B, N = x.shape[0], x.shape[1]
        R = B * N
    else:
        row0, lens = table
        B, N, R = len(lens), max(lens), x.shape[0]
        route_rows = [B * N] * len(vlads)
        r0, ln = _table_dev(row0, lens, dev)
    centres = [v._centers_on(dev) for v in vlads]
    nd = int(bool(vlads[0].norm_descs))

    def accumulate(i, labels, assign, inv):
        v = vlads[i]
        K = v.num_clusters
        ws = _lib.workspaces.get(dev, lib.anyloc_vlad_accumulate_workspace_bytes(B, N, D, K, int(assign is not None)),
                                 "vlad")
        if table is None:
            _lib.check(lib.anyloc_vlad_accumulate(
                _lib.ptr(x), None, _lib.ptr(labels), _lib.ptr(assign), _lib.ptr(inv), _lib.ptr(centres[i]), B, N, D,
                K, nd, int(bool(v.intra_norm)), _lib.ptr(outs[i]), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                "anyloc_vlad_accumulate")
        else:
            _lib.check(lib.anyloc_vlad_accumulate_varlen(
                _lib.ptr(x), R, _lib.ptr(r0), _lib.ptr(ln), B, _lib.ptr(labels), _lib.ptr(assign), _lib.ptr(inv),
                _lib.ptr(centres[i]), D, K, nd, int(bool(v.intra_norm)), _lib.ptr(outs[i]), _lib.ptr(ws), ws.numel(),
                _lib.stream_ptr()), "anyloc_vlad_accumulate_varlen")

    hard = [i for i, v in enumerate(vlads) if v.vlad_mode != "soft"]
    soft = [i for i, v in enumerate(vlads) if v.vlad_mode == "soft"]
    with torch.cuda.device(dev):
        if hard:
            V = len(hard)
            Ks = (C.c_int * V)(*[vlads[i].num_clusters for i in hard])
            preps = [vlads[i]._prepared_on(dev, centres[i]) for i in hard]
            labels = torch.empty(V, R, dtype=torch.int32, device=dev)
            inv = torch.empty(R, dtype=torch.float32, device=dev)
            ws = _lib.workspaces.get(dev, lib.anyloc_vlad_label_multi_workspace_bytes(R, D, V, Ks), "vlad_multi")
            _lib.check(lib.anyloc_vlad_label_multi(
                _lib.ptr(x), None, 1, R, (C.c_int64 * V)(*[route_rows[i] for i in hard]), D, V,
                (C.c_void_p * V)(*[centres[i].data_ptr() for i in hard]), (C.c_void_p * V)(*[p.data_ptr() for p in preps]),
                (C.c_size_t * V)(*[p.numel() for p in preps]), Ks, _lib.DIST[vlads[0].mode], _lib.ptr(labels),
                _lib.ptr(inv), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "anyloc_vlad_label_multi")
            for j, i in enumerate(hard):
                accumulate(i, labels[j], None, inv)
        if soft:
            V = len(soft)
            Ks = (C.c_int * V)(*[vlads[i].num_clusters for i in soft])
            assign = [torch.empty(R, vlads[i].num_clusters, dtype=torch.float32, device=dev) for i in soft]
            inv = torch.empty(R, dtype=torch.float32, device=dev)
            ws = _lib.workspaces.get(dev, lib.anyloc_vlad_soft_assign_multi_workspace_bytes(D, V, Ks), "vlad_soft_multi")
            _lib.check(lib.anyloc_vlad_soft_assign_multi(
                _lib.ptr(x), None, 1, R, D, V, (C.c_void_p * V)(*[centres[i].data_ptr() for i in soft]), Ks,
                (C.c_float * V)(*[float(vlads[i].soft_temp) for i in soft]),
                (C.c_void_p * V)(*[a.data_ptr() for a in assign]), _lib.ptr(inv), _lib.ptr(ws), ws.numel(),
                _lib.stream_ptr()), "anyloc_vlad_soft_assign_multi")
            for j, i in enumerate(soft):
                accumulate(i, None, assign[j], inv)


class _ImageFeed:
    """Chunks of images [i0, i1) of host features X [n, N, D] (torch CPU tensor of any float dtype and strides) on
    the device as fp32, chunk c in slot c % 2 of a _StagePair: the gather and copy of one chunk overlap the device work
    on the one before.  Built and used under torch.cuda.device(dev)."""

    def __init__(self, X, step, dev):
        n, N, D = X.shape
        self.X = X
        self.spans = [(i, min(n, i + step)) for i in range(0, n, step)]
        self.pair = _StagePair((step, N, D), dev, slots=min(2, len(self.spans)))
        self.stage(0)

    def stage(self, c):
        """gather chunk c into its staging buffer and queue its copy to the device"""
        if c < len(self.spans):
            i0, i1 = self.spans[c]
            self.pair.fill(c & 1, i1 - i0, lambda host: host[:i1 - i0].copy_(self.X[i0:i1]))

    def take(self, c):
        """chunk c's features [i1 - i0, N, D] on the device, once the current stream has waited for their copy"""
        i0, i1 = self.spans[c]
        return self.pair.take(c & 1, i1 - i0)

    def release(self, c):
        """the work on chunk c is queued: its buffer may be refilled after it"""
        self.pair.release(c & 1)

    def close(self):
        self.pair.close()


def generate_vocabularies(vlads: List[VLAD], multi_query: Union[np.ndarray, torch.Tensor, list]) -> List[torch.Tensor]:
    """Every VLAD's descriptors of `multi_query` from one read of the features (extension: a sweep over the
    vocabulary size, such as the reference's ablations over num_clusters, otherwise reads the features, and for host
    features moves them over the host link, once per vocabulary).

    `multi_query` is what VLAD.generate_multi takes without cache_ids: a numpy array or a CPU or CUDA tensor
    [n, N, D], or a list of [N_i, D] items (consecutive views of one CUDA buffer, as ext(list) returns, are read in
    place).  Element i of the result is bit for bit vlads[i].generate_multi(multi_query), on the same device.  Members
    may differ in num_clusters, vlad_mode, soft_temp and intra_norm; they must agree in norm_descs and dist_mode, as in
    fit_vocabularies.  ValueError for an empty list, a VLAD listed twice, members that differ, or centres that do not
    match D.  The per-image caches are not read or written.

    The hard members' labels come from one shared assignment pass, the soft members' probabilities from one shared
    pass, and each member then accumulates its descriptors alone.  Host [n, N, D] features are staged to the device in
    chunks of images, once for all members, the copy of the next chunk overlapping the work on this one; a chunk is as
    large as its features, every member's descriptors and the workspaces allow, and MemoryError names the bytes when
    one image does not fit.  Device features are aggregated in chunks of the same size, lists in one pass."""
    vlads = _check_members(vlads, "generate_vocabularies", "the features' norms and the assignment scores")
    is_list = isinstance(multi_query, (list, tuple))
    if is_list and len(multi_query) == 0:
        return torch.stack([])      # generate_multi's failure on an empty list
    for v in vlads:
        assert v.kmeans is not None
        assert v.c_centers is not None
    D = int(multi_query[0].shape[-1]) if is_list else int(multi_query.shape[-1])
    for v in vlads:
        if tuple(v.c_centers.shape) != (v.num_clusters, D):
            raise ValueError(f"cluster centres {tuple(v.c_centers.shape)} do not match K={v.num_clusters}, D={D}")
    if is_list:
        on_dev = all(isinstance(q, torch.Tensor) and q.is_cuda for q in multi_query)
        dev = _lib.require_cuda(multi_query[0].device if on_dev else None)
        feats, row0, lens = _pack_list(multi_query, dev)
        outs = [torch.empty(len(lens), v.num_clusters * D, device=dev) for v in vlads]
        _generate_shared(vlads, feats, outs, dev, table=(row0, lens))
        return outs if on_dev else [o.cpu() for o in outs]
    was_np = type(multi_query) == np.ndarray
    on_dev = isinstance(multi_query, torch.Tensor) and multi_query.is_cuda
    dev = _lib.require_cuda(multi_query.device if on_dev else None)
    X = torch.from_numpy(multi_query) if was_np else multi_query.detach()
    n, N, _ = X.shape
    steps = [(_generate_call_images(v, X, not on_dev and not was_np), n) for v in vlads]
    hard_Ks = [v.num_clusters for v in vlads if v.vlad_mode != "soft"]
    soft_Ks = [v.num_clusters for v in vlads if v.vlad_mode == "soft"]
    with torch.cuda.device(dev):
        if on_dev:
            x = _as_device_f32(X, dev)
            res = [torch.empty(n, v.num_clusters * D, device=dev) for v in vlads]
        else:
            res = [torch.empty(n, v.num_clusters * D) for v in vlads]
        if n == 0 or N == 0:                                           # zero descriptors, as the generate calls give
            for o in res:
                o.zero_()
            return res
        cap = 65535 if on_dev else max(1, min(65535, _STAGE_BYTES // (N * D * 4)))
        # torch's cache is only released (a device synchronisation) when the free bytes alone would cut the batch
        step = _generate_plan(n, N, D, hard_Ks, soft_Ks, not on_dev, _device_budget(dev, release_cache=False), cap)
        if step < min(n, cap):
            step = _generate_plan(n, N, D, hard_Ks, soft_Ks, not on_dev, _device_budget(dev), cap)
        if on_dev:
            for i0 in range(0, n, step):
                i1 = min(n, i0 + step)
                for p0, p1, rr in _generate_pieces(i0, i1, steps, N):
                    _generate_shared(vlads, x[p0:p1], [o[p0:p1] for o in res], dev, route_rows=rr)
            return res
        feed = _ImageFeed(X, step, dev)
        outs = [torch.empty(step, v.num_clusters * D, device=dev) for v in vlads]
        try:
            for c, (i0, i1) in enumerate(feed.spans):
                xc = feed.take(c)
                for p0, p1, rr in _generate_pieces(i0, i1, steps, N):
                    _generate_shared(vlads, xc[p0 - i0:p1 - i0], [o[p0 - i0:p1 - i0] for o in outs], dev,
                                     route_rows=rr)
                feed.release(c)
                feed.stage(c + 1)                                      # while the device works on chunk c
                for r, o in zip(res, outs):
                    r[i0:i1].copy_(o[:i1 - i0])
        finally:
            feed.close()
        return res


_POOL = {"average": 0, "avg": 0, "mean": 0, "max": 1, "gem": 2}


def pool_descriptors(patch_descs: Union[torch.Tensor, list], method: str = "gem", gem_p: float = 3.0,
                     gem_use_abs: bool = False) -> torch.Tensor:
    """Global descriptors [N, d_dim] from patch features [N, n_p, d_dim] the way the reference's other DINOv2
    scripts pool them: `get_gem_descriptors` (scripts/dino_v2_gem.py:170-189; `gem_p`, `gem_use_abs`) and the
    "average" / "max" pooling of scripts/dino_v2_gp.py:130-135.  CPU in -> CPU out, CUDA in -> CUDA out.

    A list (or tuple) of [n_i, d_dim] feature sets of differently sized images, such as ext(list) returns, gives
    [len(list), d_dim] from one launch: the items are read where they lie when they are consecutive views of one
    buffer (ext(list)'s), else packed once.  Row i is bitwise what the [N, n_p, d_dim] call gives for item i zero-padded
    to the longest item; an empty item gives NaN.  CUDA out when every item is a CUDA tensor, else CPU out."""
    if method not in _POOL:
        raise NotImplementedError(f"ID: {method}")          # scripts/dino_v2_gp.py:134-135
    if isinstance(patch_descs, (list, tuple)):
        return _pool_list(list(patch_descs), method, gem_p, gem_use_abs)
    assert len(patch_descs.shape) == len(("N", "n_p", "d_dim"))
    on_dev = patch_descs.is_cuda
    dev = _lib.require_cuda(patch_descs.device if on_dev else None)
    x = _as_device_f32(patch_descs, dev)
    B, N, D = x.shape
    out = torch.empty(B, D, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().anyloc_pool(_lib.ptr(x), None, B, N, D, _POOL[method], float(gem_p),
                                           int(bool(gem_use_abs)), _lib.ptr(out), _lib.stream_ptr()), "anyloc_pool")
    return out if on_dev else out.cpu()


def _pool_list(items, method, gem_p, gem_use_abs):
    if not items:
        raise ValueError("pool_descriptors: an empty list has no feature dimension")
    on_dev = all(isinstance(q, torch.Tensor) and q.is_cuda for q in items)
    dev = _lib.require_cuda(items[0].device if on_dev else None)
    feats, row0, lens = _pack_list(items, dev)
    R, D = feats.shape
    out = torch.empty(len(items), D, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        r0, ln = _table_dev(row0, lens, dev)
        _lib.check(_lib.load().anyloc_pool_varlen(_lib.ptr(feats), R, _lib.ptr(r0), _lib.ptr(ln), len(items), D,
                                                  _POOL[method], float(gem_p), int(bool(gem_use_abs)), _lib.ptr(out),
                                                  _lib.stream_ptr()), "anyloc_pool_varlen")
    return out if on_dev else out.cpu()


# ------------------------------------------------------------------ retrieval
_SEARCH_Q_CHUNK = 4096      # queries per anyloc_index_search call: bounds the [n_q, n_db] score matrix
_STREAM_K_MAX = 4096        # anyloc_index_search_continue merges the running k best in shared memory
_COARSE_K_MAX = 64          # the coarse route's largest k (COARSE_K_MAX in csrc/topk.cu)
PLACEMENTS = ("device", "split")


def resolve_placement(placement=None):
    """The index placement of top_k_search / get_top_k_recall: the argument, else $ANYLOC_B200_INDEX_PLACEMENT, else
    "device".  ValueError on an unknown name."""
    placement = placement or os.environ.get("ANYLOC_B200_INDEX_PLACEMENT", "device")
    if placement not in PLACEMENTS:
        raise ValueError(f"placement must be 'device' or 'split', got {placement!r}")
    return placement


def _stream_fixed_bytes(P, row, index_bytes, ws_bytes):
    """device bytes of a streamed search besides its resident pieces: two transfer buffers of P fp32 rows (the copy of
    one piece overlaps the work on the one before), the blob a piece is prepared into and a P-row search workspace"""
    return 2 * P * row + index_bytes(P) + ws_bytes(P)


def _search_plan(n_db, Dv, n_q_chunk, budget, stage_bytes, index_bytes, ws_bytes):
    """Where a search over n_db rows of dimension Dv runs, given `budget` free device bytes.  -> None (resident): the
    index, index_bytes(n_db), and the workspace of an n_q_chunk-query search, ws_bytes(n_db, n_q_chunk), fit.  Else
    (P, resident): the database is searched in pieces of P rows -- as many as fill a `stage_bytes` staging buffer, fewer
    when one piece's device buffers would not fit the budget -- and the first `resident` pieces are prepared once and
    kept on the device; the others are prepared again for every search from the index's host copy."""
    if index_bytes(n_db) + ws_bytes(n_db, n_q_chunk) <= budget:
        return None
    fixed = _piece_fixed(Dv, n_q_chunk, index_bytes, ws_bytes)
    P = _piece_rows(n_db, Dv, budget, stage_bytes, fixed)
    n_pieces = -(-n_db // P)
    return P, int(max(0, min(n_pieces, (budget - fixed(P)) // index_bytes(P))))


def _piece_fixed(Dv, n_q_chunk, index_bytes, ws_bytes):
    """P -> _stream_fixed_bytes of P-row pieces"""
    return lambda p: _stream_fixed_bytes(p, 4 * Dv, index_bytes, lambda n: ws_bytes(n, n_q_chunk))


def _piece_rows(n_db, Dv, budget, stage_bytes, fixed):
    """rows per piece: as many as fill the staging buffer, fewer when one piece's buffers, fixed(P), would not fit the
    budget (at least one row)"""
    P = max(1, min(n_db, stage_bytes // (4 * Dv)))
    if fixed(P) > budget:
        lo, hi = 1, P
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if fixed(mid) <= budget else (lo, mid - 1)
        P = lo
    return P


def _add_plan(ntotal, n, capacity, held, grow, Dv, n_q_chunk, budget, stage_bytes, index_bytes, ws_bytes):
    """Where n host rows go when they join an index of `ntotal` rows.  Its blob has room for `capacity` rows and takes
    `held` device bytes (0: no blob).  Those bytes are already allocated, so `budget` does not include them.  `grow` is
    the capacity a resident add would reserve (FlatIndex doubles).
    -> ("resident", capacity to reserve): the rows stay on the device.  Growing the blob holds the old and the new blob
       at once while the rows are copied, and a search then holds the new blob and its workspace; both peaks must fit.
       When the doubled blob does not fit, a blob of exactly the rows is tried.
    -> ("stream", P, resident pieces): a fresh index is planned by _search_plan.  An index that already holds a blob
       keeps it, since its rows have no host copy.  The blob stays counted as used, and only one piece's buffers must
       fit beside it; no further pieces are kept."""
    total = ntotal + n
    if not held:
        plan = _search_plan(total, Dv, n_q_chunk, budget, stage_bytes, index_bytes, ws_bytes)
        return ("resident", total) if plan is None else ("stream",) + plan
    ws = ws_bytes(total, n_q_chunk)
    if total <= capacity:
        if ws <= budget:
            return "resident", capacity
    else:
        for cap in dict.fromkeys((grow, total)):
            new = index_bytes(cap)
            if new <= budget and new + ws <= budget + held:
                return "resident", cap
    fixed = _piece_fixed(Dv, n_q_chunk, index_bytes, ws_bytes)
    return "stream", _piece_rows(total, Dv, budget, stage_bytes, fixed), 0


def _search_pieces(n_db, n_resident, P):
    """The pieces of a streamed search, in row order: (first row, rows, resident) -- the n_resident rows kept on the
    device, then the host rows, each in pieces of at most P rows."""
    return ([(r, min(P, n_resident - r), True) for r in range(0, n_resident, P)] +
            [(r, min(P, n_db - r), False) for r in range(n_resident, n_db, P)])


TOPK_KERNEL_DESCRIPTION = ("retrieval: gemm_tc3_kernel<true, 0> (wgmma, hi-only: ONE fp16 pass = coarse "
                           "scores with a rigorous per-query error bound) over a prepared database index -> "
                           "topk_candidates_kernel -> topk_rescore_kernel (exact fp32 re-scoring of the candidates from the "
                           "(hi,lo) pairs + k-best); 3-term GEMM + topk_select2_kernel as the device-gated fallback")


class _PinnedRows:
    """[n, d] fp16 rows in host memory page-locked to the byte: a plain host allocation registered with
    cudaHostRegister (torch's pinned allocator rounds each request up to a power of two and keeps freed blocks locked
    in its cache).  `done` is an event after the last device work that uses the rows; release() waits for it, then
    unlocks them."""

    def __init__(self, n, d):
        self.t = torch.empty(n, d, dtype=torch.float16)
        self.nbytes, self.done = self.t.numel() * 2, None
        if self.nbytes:
            torch.cuda.check_error(torch.cuda.cudart().cudaHostRegister(self.t.data_ptr(), self.nbytes, 0))

    def ptr(self):
        return C.c_void_p(self.t.data_ptr())

    def used(self):
        """record the device work queued so far on the current stream as the last use"""
        self.done = torch.cuda.Event()
        self.done.record()

    def release(self):
        if self.nbytes:
            if self.done is not None:
                self.done.synchronize()
            torch.cuda.check_error(torch.cuda.cudart().cudaHostUnregister(self.t.data_ptr()))
            self.nbytes = 0

    def __del__(self):
        try:
            self.release()
        except Exception:       # at interpreter exit the CUDA runtime may already be gone, and the lock with it
            pass


class FlatIndex:
    """GPU stand-in for `faiss.IndexFlatIP` / `IndexFlatL2` as get_top_k_recall drives them (utilities.py:439-450):
    `add(db)` normalises the rows (when `norm_descs`) and stores them once as the operand pairs of the score GEMM
    (anyloc_index_add); `search(qu, k)` is exact -- k best per query, best first, lowest database index first among
    equal scores.  Rows may be added in chunks (e.g. descriptor batches as they leave the all-gather).

    Host rows whose index (plus the score workspace of a 4096-query search) does not fit the free device memory make
    the index stream: it keeps its own host copy of the rows that do not fit, as faiss keeps its own, and every search
    moves them over the link once, piece by piece, merging each piece's k best on the device
    (anyloc_index_search_continue).  The rows added before streaming began, and as many leading pieces as the device
    holds, stay prepared on the device.  The answer is the resident search's, bit for bit, except in a query batch where
    the coarse route's 3-term fallback fires (DESIGN §4.5).  A streamed index answers k <= 4096.  Device rows never make
    an index stream; device rows added to an index that already streams join its host copy once its device blob is
    full, as host rows do.

    placement="split" keeps the low fp16 halves of the rows (half the index) in page-locked host memory and the rest on
    the device, so an index up to about twice the device memory is searched without streaming.  It needs an fp16-pair
    inner-product index: method="cosine", norm_descs=True and d % 8 == 0.  The answer is the resident index's, bit for
    bit.  The coarse route reads the lo rows of each query's candidates only; every other search (k > 64, fewer than
    32 queries, fewer than 1024 rows, a batch whose candidate lists overflow) copies every lo row to the device once.
    A split index answers k <= 4096 and never streams.  Growing it holds the old and the new device part at once, so
    rows added in chunks without a reserved `capacity` fill at most about half the device; reserve the capacity to fill
    it.  When the doubled device part does not fit, the largest one that does is taken; when not even the rows fit,
    add raises MemoryError."""

    def __init__(self, d: int, method: str = "cosine", norm_descs: bool = True, capacity: int = 0, device=None, *,
                 placement: str = "device"):
        if method not in _lib.METRIC:
            raise NotImplementedError(f"Method: {method}")
        if placement not in PLACEMENTS:
            raise ValueError(f"placement must be 'device' or 'split', got {placement!r}")
        if placement == "split" and not (method == "cosine" and norm_descs and int(d) % 8 == 0):
            raise ValueError("placement='split' holds an fp16-pair inner-product index: it needs method='cosine', "
                             f"norm_descs=True and d % 8 == 0 (got method={method!r}, norm_descs={norm_descs}, d={d})")
        self.d, self.method, self.norm_descs = int(d), method, bool(norm_descs)
        self.dp = self.d + (-self.d) % 4            # zero columns change neither norms nor scores
        self.ntotal, self.capacity = 0, 0
        self._blob, self._dev = None, (torch.device(device) if device is not None else None)
        self._split = placement == "split"
        self._lo = None                             # split: the lo halves, _PinnedRows [capacity, d]
        self._xs = None                             # split: the side stream of the exact route
        self._split_counts = []                     # split: (unique, all) candidate rows of each coarse query chunk
        # streamed index: {"P": rows per piece, "host": [(first row, fp32 rows [m, d] on the host), ...]}; the device
        # blob then holds rows [0, capacity) and the host copy rows [capacity, ntotal)
        self._stream = None
        if capacity:
            self._reserve(int(capacity), _lib.require_cuda(self._dev))

    def _reserve(self, capacity, dev):
        if self._split:
            return self._reserve_split(capacity, dev)
        lib = _lib.load()
        norm = int(self.norm_descs)
        blob = torch.empty(lib.anyloc_index_bytes(capacity, self.dp, norm), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.anyloc_index_init(_lib.ptr(blob), blob.numel(), capacity, self.dp, norm, _lib.stream_ptr()),
                       "anyloc_index_init")
            if self.ntotal:         # growth: the used rows of every section move into the larger blob
                _lib.check(lib.anyloc_index_copy(_lib.ptr(blob), blob.numel(), capacity, _lib.ptr(self._blob),
                                                 self._blob.numel(), self.capacity, self.ntotal, self.dp, norm,
                                                 _lib.stream_ptr()), "anyloc_index_copy")
        self._blob, self.capacity, self._dev = blob, capacity, dev

    def _reserve_split(self, capacity, dev, need=0):
        """a device part of `capacity` rows, or, when that does not fit, of the most rows that fit if those are at
        least `need`"""
        lib = _lib.load()
        nbytes = lib.anyloc_index_split_bytes(capacity, self.dp)
        with torch.cuda.device(dev):
            budget = _device_budget(dev)
        if nbytes > budget and need:
            fit = max(0, budget - 2048) // (2 * self.dp + 8)     # 2048: the header and the sections' alignment
            if need <= fit < capacity:
                capacity, nbytes = fit, lib.anyloc_index_split_bytes(fit, self.dp)
        if nbytes > budget:
            raise MemoryError(f"placement='split': the device part of a {capacity}-row index of dimension {self.d} "
                              f"({nbytes / 2**30:.2f} GiB: the fp16 hi halves, |y|^2 and dn) does not fit the "
                              f"{budget / 2**30:.2f} GiB free on {dev}; a split index does not stream")
        blob = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        lo = _PinnedRows(capacity, self.dp)
        with torch.cuda.device(dev):
            _lib.check(lib.anyloc_index_split_init(_lib.ptr(blob), blob.numel(), capacity, self.dp, _lib.stream_ptr()),
                       "anyloc_index_split_init")
            if self.ntotal:
                _lib.check(lib.anyloc_index_split_copy(_lib.ptr(blob), blob.numel(), capacity, _lib.ptr(self._blob),
                                                       self._blob.numel(), self.capacity, self.ntotal, self.dp,
                                                       _lib.stream_ptr()), "anyloc_index_split_copy")
                if self._lo.done is not None:
                    self._lo.done.synchronize()                 # the old lo rows are final once the adds are done
                lo.t[:self.ntotal].copy_(self._lo.t[:self.ntotal])
        if self._lo is not None:
            self._lo.release()
        self._blob, self._lo, self.capacity, self._dev = blob, lo, capacity, dev

    def reset(self):
        """faiss `index.reset()`: forget the rows, keep the allocation (a streamed index drops its host copy and
        chooses again at the next add)."""
        self._stream = None
        if self._blob is not None and self.ntotal:
            self.ntotal = 0
            self._reserve_header_only()
        self.ntotal = 0

    def _reserve_header_only(self):
        with torch.cuda.device(self._dev):
            if self._split:
                _lib.check(_lib.load().anyloc_index_split_init(_lib.ptr(self._blob), self._blob.numel(), self.capacity,
                                                               self.dp, _lib.stream_ptr()), "anyloc_index_split_init")
                return
            _lib.check(_lib.load().anyloc_index_init(_lib.ptr(self._blob), self._blob.numel(), self.capacity, self.dp,
                                                     int(self.norm_descs), _lib.stream_ptr()), "anyloc_index_init")

    def add(self, x: Union[np.ndarray, torch.Tensor]):
        on_dev = isinstance(x, torch.Tensor) and x.is_cuda
        dev = _lib.require_cuda(x.device if on_dev else self._dev)
        n = x.shape[0]
        if x.shape[1] != self.d:
            raise ValueError(f"index dimension {self.d}, got rows of {x.shape[1]}")
        grow = max(self.ntotal + n, 2 * self.capacity if self.ntotal else 0)
        if self._stream is None and not on_dev and n and not self._split:
            # first against the free memory as it is; torch's cache is emptied only when that is not enough
            plan = self._plan(n, grow, dev, release_cache=False)
            if plan[0] != "resident":
                plan = self._plan(n, grow, dev)
            if plan[0] == "resident":
                grow = plan[1]
            else:
                self._stream = {"P": plan[1], "host": []}
                if self._blob is None and plan[2]:          # the leading pieces that stay prepared on the device
                    self._reserve(min(plan[1] * plan[2], n), dev)
                self._dev = dev
        if self._stream is not None:
            m = max(0, min(n, self.capacity - self.ntotal))     # the device blob fills first, the host copy after it
            if m:
                self._prepare(x[:m], dev)
            if n > m:
                rows = torch.from_numpy(x[m:]) if type(x) == np.ndarray else x[m:].detach()
                host = torch.empty(tuple(rows.shape), dtype=torch.float32)
                host.copy_(rows)
                self._stream["host"].append((self.ntotal + m, host))
            self.ntotal += n
            return
        if self.ntotal + n > self.capacity:
            if self._split:
                self._reserve_split(grow, dev, need=self.ntotal + n)
            else:
                self._reserve(grow, dev)
        self._prepare(x, dev)
        self.ntotal += n

    def _prepare(self, x, dev):
        """rows x into the device blob at row ntotal"""
        on_dev = isinstance(x, torch.Tensor) and x.is_cuda
        n = x.shape[0]
        lib = _lib.load()
        # host rows are streamed in chunks of <= 1 GiB so that no second full copy of the database sits in HBM
        step = n if on_dev else max(1, (1 << 30) // (self.dp * 4))
        with torch.cuda.device(dev):
            for i in range(0, n, step):
                rows = _as_device_f32(x[i:i + step], dev)
                if self.dp != self.d:
                    rows = torch.nn.functional.pad(rows, (0, self.dp - self.d))
                if self._split:
                    _lib.check(lib.anyloc_index_split_add(_lib.ptr(self._blob), self._blob.numel(), self.capacity,
                                                          self._lo.ptr(), self.ntotal + i, _lib.ptr(rows),
                                                          rows.shape[0], self.dp, _lib.stream_ptr()),
                               "anyloc_index_split_add")
                    self._lo.used()
                    continue
                _lib.check(lib.anyloc_index_add(_lib.ptr(self._blob), self._blob.numel(), self.capacity,
                                                self.ntotal + i, _lib.ptr(rows), rows.shape[0], self.dp,
                                                int(self.norm_descs), _lib.stream_ptr()), "anyloc_index_add")

    def _plan(self, n, grow, dev, release_cache=True):
        """_add_plan for n more host rows on `dev`"""
        lib = _lib.load()
        norm = int(self.norm_descs)
        with torch.cuda.device(dev):
            budget = _device_budget(dev, release_cache=release_cache)
        held = self._blob.numel() if self._blob is not None else 0
        return _add_plan(self.ntotal, n, self.capacity, held, grow, self.dp, _SEARCH_Q_CHUNK, budget, _STAGE_BYTES,
                         lambda m: lib.anyloc_index_bytes(m, self.dp, norm),
                         lambda m, q: lib.anyloc_index_search_workspace_bytes(m, q, self.dp, norm))

    def add_at(self, x: torch.Tensor, row_offset: int):
        """Prepare device rows `x` into rows [row_offset, row_offset + len(x)) of the (already reserved) index -- for
        callers that receive the database out of order, e.g. chunk by chunk from an all-gather (dist.py).  `ntotal`
        becomes the highest row written; the caller must fill every row below it before searching."""
        if self._stream is not None:
            raise ValueError("add_at on an index that streams host rows: reserve the capacity and add device rows, or "
                             "use add()")
        if self._split:
            raise ValueError("add_at on an index with placement='split': use add()")
        n = x.shape[0]
        if self._blob is None or row_offset < 0 or row_offset + n > self.capacity:
            raise ValueError(f"rows [{row_offset}, {row_offset + n}) outside the reserved capacity {self.capacity}")
        rows = _as_device_f32(x, self._dev)
        if self.dp != self.d:
            rows = torch.nn.functional.pad(rows, (0, self.dp - self.d))
        with torch.cuda.device(self._dev):
            _lib.check(_lib.load().anyloc_index_add(_lib.ptr(self._blob), self._blob.numel(), self.capacity, row_offset,
                                                    _lib.ptr(rows), n, self.dp, int(self.norm_descs), _lib.stream_ptr()),
                       "anyloc_index_add")
        self.ntotal = max(self.ntotal, row_offset + n)

    def search(self, qu: Union[np.ndarray, torch.Tensor], k: int, n_q_chunk: int = _SEARCH_Q_CHUNK):
        """-> (dist, idx) [n_q, k], on the device for device queries, else on the host.  The queries are searched
        n_q_chunk at a time.  The decision to stream (add) budgets the workspace of the default chunk.  A larger
        n_q_chunk, and the device copy of the queries (n_q x d x 4 bytes) with the outputs, come out of the 1 GiB margin
        of that decision; a streamed search of many queries may need a smaller n_q_chunk or fewer queries per call.
        A streamed index answers k <= 4096 (the running k best are merged in shared memory)."""
        if self.ntotal == 0:
            raise ValueError("search on an empty index")
        if self._stream is not None and k > _STREAM_K_MAX:
            raise ValueError(f"k={k}: an index that streams host rows answers k <= {_STREAM_K_MAX}")
        if self._split and k > _STREAM_K_MAX:
            raise ValueError(f"k={k}: an index with placement='split' answers k <= {_STREAM_K_MAX}")
        on_dev = isinstance(qu, torch.Tensor) and qu.is_cuda
        dev = self._dev
        q = _as_device_f32(qu, dev)
        if self.dp != self.d:
            q = torch.nn.functional.pad(q, (0, self.dp - self.d))
        if self._stream is not None or self._split:
            dist, idx = (self._search_split if self._split else self._search_streamed)(q, k, n_q_chunk)
            return (dist, idx) if on_dev else (dist.cpu(), idx.cpu())
        lib = _lib.load()
        n_q = q.shape[0]
        dist = torch.empty(n_q, k, device=dev, dtype=torch.float32)
        idx = torch.empty(n_q, k, device=dev, dtype=torch.int64)
        with torch.cuda.device(dev):
            for i in range(0, n_q, n_q_chunk):          # bounds the [n_q, n_db] score matrix
                m = min(n_q_chunk, n_q - i)
                ws = _lib.workspaces.get(dev, lib.anyloc_index_search_workspace_bytes(self.ntotal, m, self.dp,
                                                                                     int(self.norm_descs)), "topk")
                rc = lib.anyloc_index_search(_lib.ptr(self._blob), self._blob.numel(), self.capacity, self.ntotal,
                                             _lib.ptr(q[i:i + m]), m, self.dp, k, _lib.METRIC[self.method],
                                             int(self.norm_descs), _lib.ptr(dist[i:i + m]), _lib.ptr(idx[i:i + m]),
                                             _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
                _lib.check(rc, "anyloc_index_search")
        return (dist, idx) if on_dev else (dist.cpu(), idx.cpu())

    def _gather(self, dst, r0, m):
        """rows [r0, r0 + m) of the host copy -> dst[:m, :d]"""
        for first, rows in self._stream["host"]:
            lo, hi = max(r0, first), min(r0 + m, first + rows.shape[0])
            if lo < hi:
                dst[lo - r0:hi - r0, :self.d].copy_(rows[lo - first:hi - first])

    def _search_streamed(self, q, k, n_q_chunk):
        """The k best of every query over the pieces of _search_pieces, in row order.  Database pieces are the outer
        loop and query chunks the inner one, so each host row crosses the link once per search.  A host piece is
        gathered into one of two pinned staging buffers and copied to the device on a side stream while the device
        prepares and searches the piece before it."""
        lib = _lib.load()
        dev, dp, norm, metric = self._dev, self.dp, int(self.norm_descs), _lib.METRIC[self.method]
        P, n_q = self._stream["P"], q.shape[0]
        pieces = _search_pieces(self.ntotal, min(self.ntotal, self.capacity), P)
        host_pieces = [p for p in pieces if not p[2]]
        pad = float("inf") if self.method == "l2" else -float("inf")
        with torch.cuda.device(dev):
            dist = torch.full((n_q, k), pad, device=dev, dtype=torch.float32)     # the empty running list
            idx = torch.full((n_q, k), -1, device=dev, dtype=torch.int64)
            ws = _lib.workspaces.get(dev, lib.anyloc_index_search_workspace_bytes(
                min(P, self.ntotal), min(n_q_chunk, n_q), dp, norm), "topk")
            cs = torch.cuda.current_stream()
            if host_pieces:
                cap = max(m for _, m, _ in host_pieces)
                blob = torch.empty(lib.anyloc_index_bytes(cap, dp, norm), dtype=torch.uint8, device=dev)
                raw = [torch.empty(cap, dp, device=dev) for _ in range(2)]
                host = [torch.empty(cap, dp, pin_memory=True) for _ in range(2)]
                if dp != self.d:
                    for h in host:
                        h[:, self.d:] = 0
                xs = torch.cuda.Stream()
                copied, freed = [None, None], [None, None]
                todo, staged = iter(host_pieces), []

                def stage():
                    """gather the next host piece into a staging buffer and queue its copy to the device"""
                    p = next(todo, None)
                    if p is None:
                        return
                    s = len(staged) & 1
                    if copied[s] is not None:
                        copied[s].synchronize()                     # the staging buffer's previous copy is done
                    self._gather(host[s], p[0], p[1])
                    with torch.cuda.stream(xs):
                        if freed[s] is not None:
                            xs.wait_event(freed[s])
                        raw[s][:p[1]].copy_(host[s][:p[1]], non_blocking=True)
                        copied[s] = torch.cuda.Event()
                        copied[s].record(xs)
                    staged.append((s, copied[s]))

                if not pieces[0][2]:
                    stage()
            for j, (r0, m, resident) in enumerate(pieces):
                if resident:
                    src, src_cap, first = self._blob, self.capacity, r0
                else:
                    s, ev = staged[j - (len(pieces) - len(host_pieces))]
                    cs.wait_event(ev)
                    _lib.check(lib.anyloc_index_init(_lib.ptr(blob), blob.numel(), cap, dp, norm, _lib.stream_ptr()),
                               "anyloc_index_init")
                    _lib.check(lib.anyloc_index_add(_lib.ptr(blob), blob.numel(), cap, 0, _lib.ptr(raw[s]), m, dp,
                                                    norm, _lib.stream_ptr()), "anyloc_index_add")
                    freed[s] = torch.cuda.Event()
                    freed[s].record(cs)
                    src, src_cap, first = blob, cap, 0
                for i in range(0, n_q, n_q_chunk):
                    c = min(n_q_chunk, n_q - i)
                    _lib.check(lib.anyloc_index_search_continue(
                        _lib.ptr(src), src.numel(), src_cap, first, m, r0, self.ntotal, _lib.ptr(q[i:i + c]), c, dp, k,
                        metric, norm, _lib.ptr(dist[i:i + c]), _lib.ptr(idx[i:i + c]), _lib.ptr(ws), ws.numel(),
                        _lib.stream_ptr()), "anyloc_index_search_continue")
                if host_pieces and (not resident or j + 1 == len(pieces) - len(host_pieces)):
                    stage()                 # the gather of the next host piece overlaps the work just queued
        return dist, idx

    def _search_split(self, q, k, n_q_chunk):
        """Each query chunk tries the coarse route (anyloc_index_split_search).  Its unique candidate rows are gathered
        into a device stage of exactly their size and re-scored there (anyloc_index_split_rescore); when the stage does
        not fit the free device memory, the re-scoring reads lo from host memory instead.  The chunks the coarse route
        leaves go through the exact route over pieces, together, so every lo row crosses the link once per search.
        Returns after the device work is done: that work reads the index's host memory."""
        lib = _lib.load()
        dev, dp, n_q = self._dev, self.dp, q.shape[0]
        dist = torch.empty(n_q, k, device=dev, dtype=torch.float32)
        idx = torch.empty(n_q, k, device=dev, dtype=torch.int64)
        counts, exact = (C.c_int64 * 2)(), []
        self._split_counts = []
        blob = (_lib.ptr(self._blob), self._blob.numel(), self.capacity)
        with torch.cuda.device(dev):
            for i in range(0, n_q, n_q_chunk):
                m = min(n_q_chunk, n_q - i)
                ws = _lib.workspaces.get(dev, lib.anyloc_index_split_search_workspace_bytes(self.ntotal, m, dp), "topk")
                _lib.check(lib.anyloc_index_split_search(*blob, self.ntotal, _lib.ptr(q[i:i + m]), m, dp, k,
                                                         _lib.ptr(ws), ws.numel(), counts, _lib.stream_ptr()),
                           "anyloc_index_split_search")
                if counts[0] < 0:
                    exact.append((i, m))
                    continue
                self._split_counts.append((counts[0], counts[1]))
                nbytes = lib.anyloc_index_split_stage_bytes(counts[0], dp)
                stage = self._split_stage(nbytes, dev)
                _lib.check(lib.anyloc_index_split_rescore(
                    *blob, self._lo.ptr(), self.ntotal, m, dp, k, _lib.ptr(ws), ws.numel(), counts[0],
                    _lib.ptr(stage), nbytes if stage is not None else 0, _lib.ptr(dist[i:i + m]),
                    _lib.ptr(idx[i:i + m]), _lib.stream_ptr()), "anyloc_index_split_rescore")
            if exact:
                self._search_split_exact(q, k, exact, dist, idx)
            torch.cuda.current_stream().synchronize()
        return dist, idx

    @staticmethod
    def _split_stage(nbytes, dev):
        """a device stage of nbytes, or None when it does not fit the free memory (torch's cache emptied only if needed)"""
        for release in (False, True):
            if nbytes <= _device_budget(dev, release_cache=release):
                return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        return None

    def _search_split_exact(self, q, k, chunks, dist, idx):
        """The query chunks `chunks` [(first query, queries)] by the exact route: the index is rebuilt piece by piece as
        ordinary index blobs (anyloc_index_split_piece, on a side stream, two blobs so that the copy of piece j+1
        overlaps the search of piece j) and searched by anyloc_index_search_continue.  It asks for at least 65 best,
        which takes the exact route on every batch: the 3-term product the resident index's overflow fallback uses,
        in the same (score, index) order, so the first k columns are the resident answer."""
        lib = _lib.load()
        dev, dp, n = self._dev, self.dp, self.ntotal
        ke = max(k, _COARSE_K_MAX + 1)
        ib = lambda p: lib.anyloc_index_bytes(p, dp, 1)
        wb = lambda p: lib.anyloc_index_search_workspace_bytes(p, max(m for _, m in chunks), dp, 1)
        fixed = lambda p: 2 * ib(p) + wb(p)
        P = _piece_rows(n, dp, _device_budget(dev, release_cache=False), _STAGE_BYTES, fixed)
        if P < min(n, _STAGE_BYTES // (4 * dp)):      # fewer rows than a full piece: empty torch's cache and plan again
            P = _piece_rows(n, dp, _device_budget(dev), _STAGE_BYTES, fixed)
        run = [(torch.full((m, ke), -float("inf"), device=dev), torch.full((m, ke), -1, device=dev, dtype=torch.int64))
               for _, m in chunks]
        blobs = [torch.empty(ib(P), dtype=torch.uint8, device=dev) for _ in range(2)]
        ws = _lib.workspaces.get(dev, wb(P), "topk")
        if self._xs is None or self._xs.device != dev:
            self._xs = torch.cuda.Stream(dev)
        cs, xs = torch.cuda.current_stream(), self._xs
        xs.wait_stream(cs)
        freed = [None, None]
        for j, r0 in enumerate(range(0, n, P)):
            m, s = min(P, n - r0), j & 1
            with torch.cuda.stream(xs):
                if freed[s] is not None:
                    xs.wait_event(freed[s])             # the search of piece j-2 is done with this blob
                _lib.check(lib.anyloc_index_split_piece(
                    _lib.ptr(blobs[s]), blobs[s].numel(), P, _lib.ptr(self._blob), self._blob.numel(), self.capacity,
                    self._lo.ptr(), r0, m, dp, _lib.stream_ptr()), "anyloc_index_split_piece")
                ready = torch.cuda.Event()
                ready.record(xs)
            cs.wait_event(ready)
            for (i, c), (d, x) in zip(chunks, run):
                _lib.check(lib.anyloc_index_search_continue(
                    _lib.ptr(blobs[s]), blobs[s].numel(), P, 0, m, r0, n, _lib.ptr(q[i:i + c]), c, dp, ke, 0, 1,
                    _lib.ptr(d), _lib.ptr(x), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "anyloc_index_search_continue")
            freed[s] = torch.cuda.Event()
            freed[s].record(cs)
        for (i, c), (d, x) in zip(chunks, run):
            dist[i:i + c], idx[i:i + c] = d[:, :k], x[:, :k]


def top_k_search(db: torch.Tensor, qu: torch.Tensor, k: int, method: str = "cosine",
                 norm_descs: bool = True, *, placement: str = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exact k-nearest search on the GPU (the `faiss.IndexFlatIP/L2` `add` + `search` of get_top_k_recall,
    utilities.py:435-450).  Device tensors out; a host database larger than the device streams (FlatIndex).
    `placement` (else $ANYLOC_B200_INDEX_PLACEMENT, else "device") is FlatIndex's."""
    if method not in _lib.METRIC:
        raise NotImplementedError(f"Method: {method}")
    placement = resolve_placement(placement)
    dev = _lib.require_cuda(db.device if db.is_cuda else None)
    index = FlatIndex(db.shape[1], method, norm_descs, capacity=db.shape[0] if db.is_cuda else 0, device=dev,
                      placement=placement)
    index.add(db)
    return index.search(qu.to(dev), k)


def get_top_k_recall(top_k: List[int], db: torch.Tensor, qu: torch.Tensor, gt_pos: np.ndarray,
                     method: str = "cosine", norm_descs: bool = True, use_gpu: bool = False,
                     use_percentage: bool = True, sub_sample_db: int = 1, sub_sample_qu: int = 1) \
        -> Tuple[np.ndarray, np.ndarray, dict]:
    """utilities.py:390-469.  `use_gpu` is accepted for signature compatibility; the search always
    runs on the GPU.  Host tensors in -> host tensors out (like faiss with torch_utils).  The signature is the
    reference's, so the index placement comes from $ANYLOC_B200_INDEX_PLACEMENT ("device" when unset; "split":
    FlatIndex's placement="split")."""
    if method not in _lib.METRIC:
        raise NotImplementedError(f"Method: {method}")
    placement = resolve_placement()
    as_numpy = type(db) == np.ndarray
    if as_numpy:
        db, qu = torch.from_numpy(db), torch.from_numpy(np.asarray(qu))
    if len(qu.shape) == 1:
        qu = qu.unsqueeze(0)
    on_dev = db.is_cuda
    dev = _lib.require_cuda(db.device if on_dev else None)
    # host rows: add() reserves the index once it knows it fits, and streams the search when it does not
    index = FlatIndex(db.shape[1], method, norm_descs, capacity=db.shape[0] if on_dev else 0, device=dev,
                      placement=placement)
    index.add(db)                                   # host rows are streamed in <= 1 GiB chunks
    distances, indices = index.search(_as_device_f32(qu, dev), max(top_k))
    idx_host = indices.cpu().numpy()
    recalls = dict(zip(top_k, [0] * len(top_k)))
    for i_qu, qu_retr in enumerate(idx_host):
        correct_retr = gt_pos[i_qu * sub_sample_qu]
        for i_rec in top_k:
            if np.any(np.isin(qu_retr[:i_rec] * sub_sample_db, correct_retr)):
                recalls[i_rec] += 1
    if use_percentage:
        for k in recalls:
            recalls[k] /= len(idx_host)
    if not on_dev:
        distances, indices = distances.cpu(), indices.cpu()
    if as_numpy:
        distances, indices = distances.numpy(), indices.numpy()
    return distances, indices, recalls


seed_everything()       # import side effect of the reference module (utilities.py:1011)
