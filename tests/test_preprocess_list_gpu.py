"""List pre-processing on the GPU (anyloc_preprocess_u8_varlen through utilities.preprocess_images): every item of a
list call is bit-identical to preprocess_images on that image alone (anyloc_preprocess_u8 / anyloc_preprocess_resize_u8),
the crop-only path is bit-identical to torchvision, the resize paths stay within the existing 2e-5 of torchvision's
antialiased resize, the C ABI writes each image's region in full and nothing else, host / device / mixed lists agree,
and a list feeds the extractor's packed forward unchanged."""
import ctypes as C

import numpy as np
import pytest
import torch

from anyloc_b200 import _lib

pytestmark = pytest.mark.gpu

BATCH = _lib.PREPROCESS_VARLEN_BATCH


@pytest.fixture(scope="module")
def u(cuda):
    from anyloc_b200 import utilities
    return utilities


def photos(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in sizes]


def assert_items_equal_single(u, imgs, out, **kw):
    """item i of a list call == preprocess_images(imgs[i][None], **kw)[0], bit for bit"""
    assert len(out) == len(imgs)
    for i, x in enumerate(imgs):
        ref = u.preprocess_images(x[None], **kw)[0]
        assert out[i].shape == ref.shape, (i, tuple(x.shape), out[i].shape, ref.shape)
        assert torch.equal(out[i], ref), (i, tuple(x.shape), float((out[i] - ref).abs().max()))


# sources around a fixed output size: up- and down-scaling on either axis, odd sizes, 14x14
RESIZE_LISTS = {
    "mixed": ((98, 126), [(14, 14), (37, 53), (480, 640), (99, 127), (1000, 21), (61, 1900), (98, 126)]),
    "strip": ((14, 700), [(300, 700), (7, 350), (50, 2000), (14, 701)]),            # a 1 x 50-patch output strip
    "square14": ((14, 14), [(14, 14), (15, 29), (333, 210), (1, 1)]),
}


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
@pytest.mark.parametrize("case", sorted(RESIZE_LISTS))
def test_resize_list_bit_identical(u, mode, case):
    size, sizes = RESIZE_LISTS[case]
    imgs = photos(sizes, seed=len(case))
    out = u.preprocess_images(imgs, resize=size, interpolation=mode)
    assert torch.is_tensor(out) and out.shape == (len(imgs), 3) + tuple(u.center_crop_box(*size)[2:])
    assert_items_equal_single(u, imgs, out, resize=size, interpolation=mode)


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
def test_tap_window_limit(u, mode):
    """horizontal down-scaling at the 64-tap window: 31x (bilinear) / 15.5x (bicubic); vertical down-scaling is not
    limited"""
    W = 28 * 31 if mode == "bilinear" else 434
    imgs = photos([(56, W), (28 * 40, W), (30, W)], seed=5)
    out = u.preprocess_images(imgs, resize=(28, 28), interpolation=mode)
    assert_items_equal_single(u, imgs, out, resize=(28, 28), interpolation=mode)
    with pytest.raises(_lib.AnylocError, match="tap window"):
        u.preprocess_images(imgs + photos([(56, W + 1)], seed=6), resize=(28, 28), interpolation=mode)


@pytest.mark.parametrize("mode", ["bicubic", "bilinear"])
def test_max_side_list_bit_identical(u, mode):
    """the demo's flow: phone photos capped at a 1024 long side (resized), smaller ones only cropped"""
    sizes = [(3024, 4032), (4032, 3024), (720, 1280), (1000, 1000), (1025, 1025), (1024, 1030), (500, 301), (14, 14)]
    imgs = photos(sizes, seed=7)
    out = u.preprocess_images(imgs, max_side=1024, interpolation=mode)
    assert isinstance(out, list)
    assert out[0].shape == (3, 756, 1022) and out[1].shape == (3, 1022, 756) and out[6].shape == (3, 490, 294)
    assert_items_equal_single(u, imgs, out, max_side=1024, interpolation=mode)
    # views of one allocation
    assert all(o.untyped_storage().data_ptr() == out[0].untyped_storage().data_ptr() for o in out)


def test_crop_only_list_matches_torchvision(u):
    from torchvision import transforms as T
    sizes = [(14, 14), (15, 29), (37, 53), (14, 700), (322, 322), (480, 640), (701, 333)]
    imgs = photos(sizes, seed=8)
    out = u.preprocess_images(imgs)
    assert_items_equal_single(u, imgs, out)
    tf = T.Compose([T.ToTensor(), T.Normalize(mean=u.IMAGENET_MEAN, std=u.IMAGENET_STD)])
    for x, o in zip(imgs, out):
        h, w = x.shape[:2]
        ref = T.CenterCrop(((h // 14) * 14, (w // 14) * 14))(tf(x.numpy()))
        assert torch.equal(o.cpu(), ref)
    # custom statistics and patch size
    kw = dict(mean=(0.5, 0.4, 0.3), std=(0.2, 0.25, 0.5), patch=8)
    assert_items_equal_single(u, imgs, u.preprocess_images(imgs, **kw), **kw)


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
def test_resize_lists_match_torchvision(u, mode):
    import torchvision.transforms.functional as TF
    from torchvision import transforms as T
    imgs = photos([(720, 1280), (333, 517), (1200, 900), (40, 60)], seed=9)
    interp = T.InterpolationMode.BILINEAR if mode == "bilinear" else T.InterpolationMode.BICUBIC
    tf = T.Compose([T.ToTensor(), T.Normalize(mean=u.IMAGENET_MEAN, std=u.IMAGENET_STD)])
    for kw in (dict(resize=(480, 640)), dict(max_side=500)):
        out = u.preprocess_images(imgs, interpolation=mode, **kw)
        for x, o in zip(imgs, out):
            h, w = kw.get("resize") or u.max_side_size(x.shape[0], x.shape[1], kw["max_side"])
            ref = tf(x.numpy())
            if (h, w) != tuple(x.shape[:2]):
                ref = TF.resize(ref, [h, w], interpolation=interp, antialias=True)
            ref = T.CenterCrop(((h // 14) * 14, (w // 14) * 14))(ref)
            assert o.shape == ref.shape
            assert float((o.cpu() - ref).abs().max()) < 2e-5


@pytest.mark.parametrize("n", [1, BATCH - 1, BATCH, BATCH + 1, 2 * BATCH])
@pytest.mark.parametrize("mode", [None, "bilinear", "bicubic"])
def test_list_lengths(u, n, mode):
    """lists of one image, and on both sides of the per-launch table limit and of twice it"""
    rng = np.random.default_rng(n)
    imgs = photos([tuple(int(v) for v in rng.integers(30, 90, 2)) for _ in range(n)], seed=n)
    kw = {} if mode is None else dict(max_side=48, interpolation=mode)
    out = u.preprocess_images(imgs, **kw)
    assert_items_equal_single(u, imgs, out, **kw)


def test_uniform_batch_with_max_side(u):
    """max_side on a uniform batch yields a uniform batch, equal to the list call on its images"""
    img = torch.randint(0, 256, (3, 600, 900, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(10))
    out = u.preprocess_images(img, max_side=448, interpolation="bicubic")
    assert out.shape == (3, 3, 294, 448)
    lst = u.preprocess_images(list(img), max_side=448, interpolation="bicubic")
    assert all(torch.equal(a, b) for a, b in zip(out, lst))
    small = u.preprocess_images(img, max_side=900)                           # not over the cap: crop only
    assert torch.equal(small, u.preprocess_images(img))


def test_host_device_and_mixed_inputs(u):
    imgs = photos([(300, 400), (57, 91), (1280, 720), (14, 28)], seed=11)
    for kw in ({}, dict(max_side=640, interpolation="bicubic"), dict(resize=(224, 224))):
        ref = u.preprocess_images(imgs, **kw)
        variants = ([x.numpy() for x in imgs], [x.cuda() for x in imgs],
                    [x.cuda() if i % 2 else x.numpy() for i, x in enumerate(imgs)],
                    tuple(x.cuda() if i % 2 == 0 else x for i, x in enumerate(imgs)),
                    [x.cuda().permute(1, 0, 2).contiguous().permute(1, 0, 2) for x in imgs])   # non-contiguous
        for v in variants:
            out = u.preprocess_images(v, **kw)
            assert all(torch.equal(a, b) for a, b in zip(out, ref))


def test_abi_regions_and_refusals(u):
    """each image's region of a NaN-filled output is written in full, nothing outside (gaps between the regions and
    after the last one) is; a refusal writes nothing"""
    lib = _lib.load()
    imgs = [x.cuda() for x in photos([(40, 60), (100, 30), (14, 14), (77, 91)], seed=12)]
    n = len(imgs)
    mean, std = (C.c_float * 3)(*u.IMAGENET_MEAN), (C.c_float * 3)(*u.IMAGENET_STD)

    def ints(v):
        return (C.c_int * n)(*v)
    for interp, hw in ((-1, None), (0, (28, 42)), (1, (56, 14))):
        H, W = [x.shape[0] for x in imgs], [x.shape[1] for x in imgs]
        Hr, Wr = (H, W) if hw is None else ([hw[0]] * n, [hw[1]] * n)
        boxes = [u.center_crop_box(h, w) for h, w in zip(Hr, Wr)]
        sizes = [3 * b[2] * b[3] for b in boxes]
        offs, o = [], 5
        for s in sizes:
            offs.append(o)
            o += s + 7                                  # gaps between the regions
        out = torch.full((o + 11,), float("nan"), device="cuda")
        args = [n, (C.c_void_p * n)(*[x.data_ptr() for x in imgs]), ints(H), ints(W), ints(Hr), ints(Wr), interp,
                ints([b[0] for b in boxes]), ints([b[1] for b in boxes]), ints([b[2] for b in boxes]),
                ints([b[3] for b in boxes]), mean, std, _lib.ptr(out), (C.c_int64 * n)(*offs), _lib.stream_ptr()]
        _lib.check(lib.anyloc_preprocess_u8_varlen(*args), "anyloc_preprocess_u8_varlen")
        written = torch.zeros_like(out, dtype=torch.bool)
        for i, x in enumerate(imgs):
            kw = {} if hw is None else dict(resize=hw, interpolation=("bilinear", "bicubic")[interp])
            ref = u.preprocess_images(x[None], **kw)[0]
            assert torch.equal(out[offs[i]:offs[i] + sizes[i]].view(ref.shape), ref), (interp, i)
            written[offs[i]:offs[i] + sizes[i]] = True
        assert bool(out[~written].isnan().all()) and not bool(out[written].isnan().any())
        # refusals: a crop outside the last image, a zero std -- nothing written
        fresh = torch.full_like(out, float("nan"))
        bad = list(args)
        bad[13] = _lib.ptr(fresh)
        bad[8] = ints([b[1] for b in boxes][:-1] + [Wr[-1]])          # left
        assert lib.anyloc_preprocess_u8_varlen(*bad) == _lib.ERR["arg"]
        bad[8] = args[8]
        bad[12] = (C.c_float * 3)(0.2, 0.0, 0.2)                      # std
        assert lib.anyloc_preprocess_u8_varlen(*bad) == _lib.ERR["arg"]
        assert bool(fresh.isnan().all())


def test_list_feeds_the_extractor(u):
    """DinoV2ExtractFeatures(list) on the list output == per-image pre-processing + a single-image extract, bit for bit
    (tensor-core engine, ViT-S/14 random init)"""
    from oracle import dinov2_restated as dr
    model = dr.perturb(dr.build("dinov2_vits14", seed=0, depth_override=2), seed=1)
    ext = u.DinoV2ExtractFeatures("dinov2_vits14", 1, "value", device="cuda", weights=model.state_dict(),
                                  gemm_engine="tc3")
    imgs = photos([(300, 400), (200, 150), (140, 98), (60, 75)], seed=13)
    pre = u.preprocess_images(imgs, max_side=224, interpolation="bicubic")
    feats = ext(pre)
    for x, f in zip(imgs, feats):
        ref = ext(u.preprocess_images(x[None], max_side=224, interpolation="bicubic"))[0]
        assert torch.equal(f, ref)
