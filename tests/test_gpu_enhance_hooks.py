"""ContrastImage, ModulateImage, GrayscaleImage and FunctionImage on the GPU, through the device and the host-buffer entry
points, against the oracle (itself pinned to the reference by test_oracle_enhance_vs_ref.py):

- bit exact: Function Polynomial / Undefined, Grayscale without a gamma step, Modulate in HCL, HCLp, HSB, HSL, HSV, HWB;
- <= 1 ULP of the float Quantum where the CUDA math library stands in for glibc: Contrast (sin), Function Sinusoid /
  Arcsin / Arctan, Grayscale with a gamma step, Modulate in HSI, LCHab, LCHuv.  In LCHab / LCHuv with the chroma scaled,
  an achromatic pixel's hue is atan2 of rounding residues (in the reference as well) and the scaled +0.5 chroma gives it
  a real magnitude: exactly the pixels with r == g == b are left out of the bar there, and they are the only ones over it.

Plus 8192^2 RGBA images, an RGBA buffer 4 bytes off a 16-byte boundary, the declines (MB200_EUNSUPPORTED / MB200_EINVAL
leave the buffer untouched) and the Python layer's re-layout (Grayscale) and re-tag (Modulate)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

import enhance_cases as ec
import imagemagick_b200 as im
from imagemagick_b200 import _lib
from util import make_image, ulp_distance

pytestmark = pytest.mark.gpu

CHANNELS = [1, 2, 3, 4]
SIZES = [(37, 23), (1, 17), (19, 1)]


def both(fn, src, *args):
    """The operator through the device entry point and through the host-buffer one: (pixels, colorspace) of each."""
    out = []
    for img in (im.Image(torch.from_numpy(src.copy()).cuda()), im.Image(src.copy())):
        assert fn(img, *args) is True
        pixels = img.pixels.cpu().numpy() if img.on_device else img.pixels
        out.append((pixels, img.colorspace))
    return out


def ulps(got, want):
    """Per-sample ULP distance; NaN must sit exactly where the oracle has NaN."""
    assert got.shape == want.shape
    nan_got, nan_want = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_got, nan_want), int(np.sum(nan_got != nan_want))
    return ulp_distance(np.where(nan_got, np.float32(0), got), np.where(nan_want, np.float32(0), want))


def assert_within(got, want, bar, what, exempt=None):
    d = ulps(got, want)
    if exempt is not None:
        over = d.max(axis=2) > bar
        assert not np.any(over & ~exempt), (what, int(np.sum(over & ~exempt)))
        d = np.where(exempt[..., None], 0, d)
    assert int(d.max()) <= bar, (what, int(d.max()))


def achromatic(src):
    return (src[..., 0] == src[..., 1]) & (src[..., 1] == src[..., 2]) if src.shape[2] >= 3 else np.ones(src.shape[:2], bool)


# ------------------------------------------------------------------------------------------------------------ Contrast
@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("sharpen", [True, False])
def test_contrast(ch, sharpen):
    for src in [ec.mosaic(37, ch)] + [make_image(w, h, ch, seed=w + h) for w, h in SIZES]:
        want = ec.orc_contrast(src, sharpen)
        for got, cs in both(im.ContrastImage, src, sharpen):
            assert cs == im.sRGBColorspace
            assert_within(got, want, 1, src.shape)


def test_contrast_three_times():
    src = ec.mosaic(29, 4, seed=5)
    want = src
    for _ in range(3):
        want = ec.orc_contrast(want, True)
    img = im.Image(torch.from_numpy(src).cuda())
    for _ in range(3):
        im.ContrastImage(img, True)
    assert_within(img.pixels.cpu().numpy(), want, 1, "x3")


# ------------------------------------------------------------------------------------------------------------ Modulate
MODULATE_BAR = {"HSI": 1, "LCH": 1, "LCHab": 1, "LCHuv": 1}


def check_modulate(src, geometry, space=None, illuminant=None):
    want = ec.orc_modulate(src, geometry, space, illuminant)
    cs, _ = ec.modulate_settings(space, illuminant)
    lch = cs in (ec.LCH, ec.LCHAB, ec.LCHUV)
    saturation = ec.modulate_percentages(geometry)[1]
    exempt = achromatic(src) if lch and saturation != 100.0 else None
    artifacts = {}
    if space is not None:
        artifacts["modulate:colorspace"] = space
    if illuminant is not None:
        artifacts["color:illuminant"] = illuminant
    for got, _ in both(im.ModulateImage, src, geometry, artifacts):
        assert_within(got, want, 1 if lch or cs == ec.HSI else 0, (space, geometry, src.shape), exempt)


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("space", list(ec.MODULATE_SPACES), ids=str)
def test_modulate(space, ch):
    src = ec.mosaic(31, ch, seed=21)
    for geometry in ec.GEOMETRIES:
        check_modulate(src, geometry, space)


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("illuminant", ["D50", "A", "bogus"])
@pytest.mark.parametrize("space", ["LCHab", "LCHuv", "HSB"])
def test_modulate_illuminant(space, illuminant, ch):
    check_modulate(ec.mosaic(23, ch, seed=31), "90,140,130", space, illuminant)


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("space", ["HCL", "HSI", "LCHab"])
def test_modulate_sizes(space, ch):
    for w, h in SIZES:
        check_modulate(make_image(w, h, ch, seed=3 * w + h, kind="hdr"), "120,70,40", space)
    for geometry in ["130", "70,160", "90x110", "90x110,170"]:
        check_modulate(ec.mosaic(17, ch, seed=41), geometry, space)


def test_modulate_retag_and_parse():
    src = ec.mosaic(17, 4, seed=41)
    want = ec.orc_modulate(src, "90,110,170", "HWB")
    for colorspace, after in [(im.LabColorspace, im.sRGBColorspace), (im.RGBColorspace, im.RGBColorspace),
                              (im.HSLColorspace, im.sRGBColorspace)]:
        img = im.Image(torch.from_numpy(src).cuda(), colorspace)
        im.ModulateImage(img, "90,110,170", {"modulate:colorspace": "HWB"})
        assert img.colorspace == after
        assert_within(img.pixels.cpu().numpy(), want, 0, colorspace)
    img = im.Image(src.copy())
    for bad in ["", "a,b", "1,2,3,4", "90,110x170"]:
        with pytest.raises(im.MagickB200Error) as e:
            im.ModulateImage(img, bad)
        assert e.value.code == _lib.EINVAL
    np.testing.assert_array_equal(img.pixels, src)


# ----------------------------------------------------------------------------------------------------------- Grayscale
GAMMA_STEP = {(5, ec.RGB), (7, ec.RGB), (0, ec.RGB), (6, ec.SRGB), (8, ec.SRGB)}


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("method", range(10))
def test_grayscale(method, ch):
    src = ec.mosaic(33, ch, seed=51)
    keep = [0, ch - 1] if ch in (2, 4) else [0]
    for colorspace in ([ec.SRGB, ec.RGB] if ch >= 3 else [ec.GRAY]):
        want = ec.orc_grayscale(src, method, colorspace)
        bar = 1 if (method, colorspace) in GAMMA_STEP else 0
        # the C ABI writes channel 0 and leaves the others
        lib = _lib.load()
        host = src.copy()
        _lib.check(lib.mb200_grayscale_image(host.ctypes.data, src.shape[1], src.shape[0], ch, method, colorspace))
        np.testing.assert_array_equal(host[..., 1:], src[..., 1:])
        assert_within(host[..., keep], want, bar, (method, colorspace, "C ABI"))
        # the Python layer re-lays the cache out to gray (+ alpha) and re-tags the image
        for img in (im.Image(torch.from_numpy(src).cuda(), colorspace), im.Image(src.copy(), colorspace)):
            assert im.GrayscaleImage(img, method) is True
            pixels = img.pixels.cpu().numpy() if img.on_device else img.pixels
            assert pixels.shape == want.shape and pixels.flags["C_CONTIGUOUS"]
            assert img.colorspace == (im.LinearGRAYColorspace if method in (6, 8) else im.GRAYColorspace)
            assert_within(pixels, want, bar, (method, colorspace))


# ------------------------------------------------------------------------------------------------------------ Function
def _function_id(case):
    return f"{['undefined', 'arcsin', 'arctan', 'polynomial', 'sinusoid'][case[0]]}{len(case[1])}-" + \
        "_".join(f"{p:g}" for p in case[1][:4])


def function_bar(function):
    return 0 if function in (ec.POLYNOMIAL, ec.UNDEFINED) else 1


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("case", ec.FUNCTION_CASES, ids=_function_id)
def test_function(case, ch):
    function, params = case
    src = ec.mosaic(27, ch, seed=61)
    want = ec.orc_function(src, function, params, -1)
    for got, _ in both(im.FunctionImage, src, function, params):
        assert_within(got, want, function_bar(function), case)


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("mask", ["R", "RGB", "alpha"])
def test_function_channels(mask, ch):
    src = ec.mosaic(21, ch, seed=71)
    bits = ec.update_mask(ec.CHANNEL_MASKS[mask], ch)
    for function, params in [(ec.POLYNOMIAL, [1.5, -0.25, 0.125]), (ec.SINUSOID, [2.0, 30.0]), (ec.ARCTAN, [])]:
        want = ec.orc_function(src, function, params, ec.CHANNEL_MASKS[mask])
        for got, _ in both(im.FunctionImage, src, function, params, bits):
            assert_within(got, want, function_bar(function), (mask, function))


def test_function_sizes():
    for ch in CHANNELS:
        for w, h in SIZES:
            src = make_image(w, h, ch, seed=w * h, kind="hdr")
            want = ec.orc_function(src, ec.ARCSIN, [0.6, 0.4], -1)
            for got, _ in both(im.FunctionImage, src, ec.ARCSIN, [0.6, 0.4]):
                assert_within(got, want, 1, (w, h, ch))


# ------------------------------------------------------------------------------------- declines, alignment, full size
def test_declines_leave_the_buffer():
    lib = _lib.load()
    src = ec.mosaic(19, 4, seed=81)
    h, w, ch = src.shape
    dev = torch.from_numpy(src).cuda()
    p33 = (C.c_double * 33)(*ec.POLYNOMIAL_33[1])
    s = None
    calls = [
        (_lib.EUNSUPPORTED, lambda b, d: lib.mb200_function_image_dev(b, w, h, ch, ec.POLYNOMIAL, 33, p33, 15, s) if d
         else lib.mb200_function_image(b, w, h, ch, ec.POLYNOMIAL, 33, p33, 15)),
        (_lib.EINVAL, lambda b, d: lib.mb200_function_image_dev(b, w, h, ch, 5, 0, None, 15, s) if d
         else lib.mb200_function_image(b, w, h, ch, -1, 0, None, 15)),
        (_lib.EINVAL, lambda b, d: lib.mb200_grayscale_image_dev(b, w, h, ch, 10, ec.SRGB, s) if d
         else lib.mb200_grayscale_image(b, w, h, ch, -1, ec.SRGB)),
        (_lib.EINVAL, lambda b, d: lib.mb200_modulate_image_dev(b, w, h, ch, 90.0, 110.0, 120.0, ec.LCHAB, 11, s) if d
         else lib.mb200_modulate_image(b, w, h, ch, 90.0, 110.0, 120.0, ec.LCHAB, -1)),
        (_lib.EINVAL, lambda b, d: lib.mb200_contrast_image_dev(b, w, h, 5, 1, s) if d
         else lib.mb200_contrast_image(b, w, h, 0, 1)),
    ]
    launches = im.launch_count()
    for code, call in calls:
        host = src.copy()
        assert call(host.ctypes.data, False) == code
        np.testing.assert_array_equal(host, src)
        assert call(dev.data_ptr(), True) == code
    torch.cuda.synchronize()
    assert im.launch_count() == launches
    np.testing.assert_array_equal(dev.cpu().numpy(), src)
    with pytest.raises(im.MagickB200Error) as e:
        im.FunctionImage(im.Image(src.copy()), ec.POLYNOMIAL, ec.POLYNOMIAL_33[1])
    assert e.value.code == _lib.EUNSUPPORTED


def test_unaligned_rgba():
    """An RGBA buffer 4 bytes off a 16-byte boundary takes the per-channel path and gives the aligned bits."""
    src = ec.mosaic(45, 4, seed=91)
    n = src.size
    for op, args in [(im.ContrastImage, (True,)), (im.ModulateImage, ("80,130,150", {"modulate:colorspace": "HSV"})),
                     (im.FunctionImage, (ec.SINUSOID, [2.0, 10.0]))]:
        aligned = im.Image(torch.from_numpy(src).cuda())
        store = torch.empty(n + 4, dtype=torch.float32, device="cuda")
        view = store[1:n + 1].view(src.shape)
        view.copy_(torch.from_numpy(src))
        unaligned = im.Image(view)
        assert unaligned.pixels.data_ptr() % 16 == 4
        op(aligned, *args)
        op(unaligned, *args)
        assert_within(unaligned.pixels.cpu().numpy(), aligned.pixels.cpu().numpy(), 0, op.__name__)
    gray = torch.empty(n + 4, dtype=torch.float32, device="cuda")
    view = gray[1:n + 1].view(src.shape)
    view.copy_(torch.from_numpy(src))
    _lib.check(_lib.load().mb200_grayscale_image_dev(view.data_ptr(), src.shape[1], src.shape[0], 4, 7, ec.SRGB, None))
    _lib.check(_lib.load().mb200_synchronize(None))
    want = ec.orc_grayscale(src, 7, ec.SRGB)
    assert_within(view.cpu().numpy()[..., [0, 3]], want, 0, "grayscale")


@pytest.mark.parametrize("op", ["contrast", "modulate", "grayscale", "function"])
def test_full_size_rgba(op):
    size = 8192
    src = make_image(size, size, 4, seed=101)
    img = im.Image(torch.from_numpy(src).cuda())
    if op == "contrast":
        want, bar = ec.orc_contrast(src, False), 1
        im.ContrastImage(img, False)
    elif op == "modulate":
        want, bar = ec.orc_modulate(src, "90,120,130", "HSB"), 0
        im.ModulateImage(img, "90,120,130", {"modulate:colorspace": "HSB"})
    elif op == "grayscale":
        want, bar = ec.orc_grayscale(src, 8, ec.SRGB), 1
        im.GrayscaleImage(img, 8)
    else:
        want, bar = ec.orc_function(src, ec.POLYNOMIAL, [0.5, -0.5, 0.75, 0.1], -1), 0
        im.FunctionImage(img, ec.POLYNOMIAL, [0.5, -0.5, 0.75, 0.1])
    assert_within(img.pixels.cpu().numpy(), want, bar, op)
