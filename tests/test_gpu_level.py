"""The level and stretch operators on the GPU -- LevelImage, LevelizeImage, MinMaxStretchImage / AutoLevelImage,
ContrastStretchImage / NormalizeImage, LinearStretchImage, GammaImage -- through the device and the host-buffer entry
points, against the oracle (itself pinned to the reference by test_oracle_level_vs_ref.py):

- bit exact, with the same "histogram:*" property: ContrastStretch, Normalize, LinearStretch, AutoLevel, Gamma, and Level
  / Levelize / MinMaxStretch at gamma 1;
- <= 1 ULP of the float Quantum at other gammas (CUDA pow stands in for glibc's).

Plus the per-channel AutoLevel launch order, a flat 8192^2 RGBA image whose 67 M pixels all land in one histogram bin,
8192^2 RGBA ContrastStretch and AutoLevel, an RGBA buffer 4 bytes off a 16-byte boundary, the device gray scan, the
Python layer's GRAY re-layout, and the declines (MB200_EINVAL / MB200_EUNSUPPORTED leave the buffer untouched)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

import imagemagick_b200 as im
import level_cases as lc
from imagemagick_b200 import _lib
from util import make_image, ulp_distance

pytestmark = pytest.mark.gpu

CHANNELS = [1, 2, 3, 4]


def py_call(img, op, a, b, g, mask):
    """The Python operator of ref_level_op's `op` on `img` (ChannelType mask -> `channels` selection); the property or ''."""
    channels = None if mask < 0 else lc.update_mask(mask, img.channels)
    if op == lc.LEVEL:
        return im.LevelImage(img, a, b, g, channels) and ""
    if op == lc.LEVELIZE:
        return im.LevelizeImage(img, a, b, g, channels) and ""
    if op == lc.MINMAX:
        return im.MinMaxStretchImage(img, a, b, g, channels) and ""
    if op == lc.AUTO_LEVEL:
        return im.AutoLevelImage(img, channels) and ""
    if op == lc.CONTRAST_STRETCH:
        return im.ContrastStretchImage(img, a, b, channels)
    if op == lc.NORMALIZE:
        return im.NormalizeImage(img, channels)
    if op == lc.LINEAR_STRETCH:
        return im.LinearStretchImage(img, a, b, channels)
    return im.GammaImage(img, g, channels) and ""


def ulps(got, want):
    assert got.shape == want.shape
    nan_got, nan_want = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_got, nan_want), int(np.sum(nan_got != nan_want))
    return ulp_distance(np.where(nan_got, np.float32(0), got), np.where(nan_want, np.float32(0), want))


def check(src, op, a=0.0, b=0.0, g=1.0, mask=-1, bar=0, what=""):
    want, want_prop = lc.orc_run(src, op, a, b, g, mask)
    for img in (im.Image(torch.from_numpy(src.copy()).cuda()), im.Image(src.copy())):
        prop = py_call(img, op, a, b, g, mask)
        got = img.pixels.cpu().numpy() if img.on_device else img.pixels
        assert int(ulps(got, want).max(initial=0)) <= bar, (what, img.on_device)
        assert prop == want_prop, (what, prop, want_prop)


@pytest.mark.parametrize("ch", CHANNELS)
def test_level_levelize(ch):
    src = lc.sources(ch)["mosaic"]
    for black, white, gamma in lc.LEVEL_ARGS:
        bar = 0 if gamma == 1.0 else 1
        check(src, lc.LEVEL, black, white, gamma, bar=bar, what=("level", black, white, gamma))
        check(src, lc.LEVELIZE, black, white, gamma, bar=bar, what=("levelize", black, white, gamma))
    for name, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.LEVEL, 1000.0, 60000.0, 1.0, mask, what=("level", name))
        check(src, lc.LEVELIZE, 1000.0, 60000.0, 0.45, mask, bar=1, what=("levelize", name))


@pytest.mark.parametrize("ch", CHANNELS)
def test_gamma(ch):
    src = lc.sources(ch)["mosaic"]
    for gamma in lc.GAMMAS:
        check(src, lc.GAMMA, g=gamma, what=("gamma", gamma))
    for name, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.GAMMA, g=2.2, mask=mask, what=("gamma", name))


@pytest.mark.parametrize("ch", CHANNELS)
def test_auto_level(ch):
    for name, src in lc.sources(ch).items():
        check(src, lc.AUTO_LEVEL, what=("auto level", name))
        for mname, mask in lc.CHANNEL_MASKS.items():
            if mask >= 0:
                check(src, lc.AUTO_LEVEL, mask=mask, what=("auto level", name, mname))
    src = lc.sources(ch)["mosaic"]
    for black, white, gamma in lc.MINMAX_ARGS:
        bar = 0 if gamma == 1.0 else 1
        check(src, lc.MINMAX, black, white, gamma, bar=bar, what=("minmax", black, white, gamma))
        check(src, lc.MINMAX, black, white, gamma, 0x17, bar=bar, what=("minmax RGBA", black, white, gamma))


@pytest.mark.parametrize("ch", CHANNELS)
def test_contrast_stretch(ch):
    for name, src in lc.sources(ch).items():
        n = src.shape[0] * src.shape[1]
        check(src, lc.NORMALIZE, what=("normalize", name))
        for black, white in lc.stretch_points(n):
            check(src, lc.CONTRAST_STRETCH, black, white, what=("stretch", name, black, white))
    src = lc.sources(ch)["mosaic"]
    n = src.shape[0] * src.shape[1]
    for mname, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.NORMALIZE, mask=mask, what=("normalize", mname))
        check(src, lc.CONTRAST_STRETCH, 0.1 * n, 0.95 * n, mask=mask, what=("stretch", mname))


@pytest.mark.parametrize("ch", [3, 4])
def test_contrast_stretch_gray_relayout(ch):
    for name, src in lc.gray_sources(ch).items():
        n = src.shape[0] * src.shape[1]
        check(src, lc.NORMALIZE, what=("normalize", name))
        check(src, lc.CONTRAST_STRETCH, 0.05 * n, 0.9 * n, what=("stretch", name))
        for mname, mask in lc.CHANNEL_MASKS.items():
            if mask >= 0:
                check(src, lc.NORMALIZE, mask=mask, what=("normalize", name, mname))
        img = im.Image(torch.from_numpy(src.copy()).cuda())
        im.NormalizeImage(img)
        gray = name != "near gray"
        assert img.channels == (ch - 2 if gray else ch)
        assert img.colorspace == (im.GRAYColorspace if gray else im.sRGBColorspace)


@pytest.mark.parametrize("ch", CHANNELS)
def test_linear_stretch(ch):
    for name, src in lc.sources(ch).items():
        n = src.shape[0] * src.shape[1]
        for black, white in lc.stretch_points(n):
            check(src, lc.LINEAR_STRETCH, black, white, what=("linear", name, black, white))
    src = lc.sources(ch)["mosaic"]
    n = src.shape[0] * src.shape[1]
    for mname, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.LINEAR_STRETCH, 0.02 * n, 0.01 * n, mask=mask, what=("linear", mname))


@pytest.mark.parametrize("ch", CHANNELS)
def test_identify_gray(ch):
    srcs = {**(lc.gray_sources(ch) if ch >= 3 else {}), **lc.sources(ch)}
    for name, src in srcs.items():
        h, w, _ = src.shape
        want = lc.oracle().orc_identify_gray(lc.util.P(src.copy()), w, h, ch)
        assert im.IdentifyImageGray(im.Image(torch.from_numpy(src.copy()).cuda())) == want, name
        assert im.IdentifyImageGray(im.Image(src.copy())) == want, name


def test_per_channel_auto_level_launches():
    """Per channel, AutoLevel runs range (rows + merge) then level for each selected colour channel in channel order:
    three launches per channel, none for alpha.  The default mask takes one range and one level."""
    src = lc.sources(4)["mosaic"]
    img = im.Image(torch.from_numpy(src.copy()).cuda())
    before = im.launch_count()
    im.AutoLevelImage(img, 0b1111)
    torch.cuda.synchronize()
    assert im.launch_count() - before == 3 * 3
    before = im.launch_count()
    im.AutoLevelImage(img, 0b1010)
    assert im.launch_count() - before == 3
    before = im.launch_count()
    im.AutoLevelImage(img)
    assert im.launch_count() - before == 3


def test_flat_8192_one_bin():
    """All 67 108 864 pixels of a flat 8192^2 RGBA image land in one bin: LinearStretch's black search stops at that bin
    for a black point of exactly N and runs off the end for N + 1."""
    size = 8192
    n = size * size
    value = 20000.0
    dev = torch.full((size, size, 4), value, dtype=torch.float32, device="cuda")
    img = im.Image(dev)
    prop = im.LinearStretchImage(img, float(n), float(n))
    assert prop == "%gx%g%%" % (100.0 * value / 65535, 100.0 * value / 65535)
    img = im.Image(torch.full((size, size, 4), value, dtype=torch.float32, device="cuda"))
    prop = im.LinearStretchImage(img, float(n + 1), 0.0)
    assert prop.startswith("100x")


@pytest.mark.parametrize("op", ["contrast stretch", "auto level"])
def test_8192_rgba(op):
    size = 8192
    src = make_image(size, size, 4, seed=111, kind="alpha_blocks")
    src[::97, ::89, 0] = np.nan
    img = im.Image(torch.from_numpy(src).cuda())
    n = size * size
    if op == "contrast stretch":
        want, want_prop = lc.orc_run(src, lc.CONTRAST_STRETCH, 0.01 * n, 0.97 * n)
        assert im.ContrastStretchImage(img, 0.01 * n, 0.97 * n) == want_prop
    else:
        want, _ = lc.orc_run(src, lc.AUTO_LEVEL)
        im.AutoLevelImage(img)
    got = img.pixels.cpu().numpy()
    assert int(ulps(got, want).max()) == 0


def test_unaligned_rgba():
    """An RGBA buffer 4 bytes off a 16-byte boundary takes the per-channel path and gives the aligned bits."""
    src = lc.sources(4)["mosaic"]
    n = src.size
    for op, a, b, g in [(lc.LEVEL, 1000.0, 60000.0, 1.0), (lc.LEVELIZE, 1000.0, 60000.0, 1.0), (lc.AUTO_LEVEL, 0, 0, 1),
                        (lc.GAMMA, 0, 0, 2.2), (lc.NORMALIZE, 0, 0, 1)]:
        want, want_prop = lc.orc_run(src, op, a, b, g)
        flat = torch.empty(n + 1, dtype=torch.float32, device="cuda")
        view = flat[1:].view(src.shape)
        view.copy_(torch.from_numpy(src))
        assert view.data_ptr() % 16 == 4
        img = im.Image(view)
        assert py_call(img, op, a, b, g, -1) == want_prop
        assert int(ulps(img.pixels.cpu().numpy(), want).max()) == 0, op


def test_declines_leave_the_buffer():
    lib = _lib.load()
    src = lc.sources(4)["mosaic"]
    h, w, ch = src.shape
    dev = torch.from_numpy(src).cuda()
    black, white = (C.c_float * 4)(), (C.c_float * 4)()
    lo, hi = C.c_double(), C.c_double()
    big = 1 << 16                       # 2^32 pixels: refused before the buffer is touched
    s = None
    calls = [
        (_lib.EINVAL, lambda b, d: lib.mb200_contrast_stretch_image_dev(b, w, h, ch, 0.0, 0.0, 0, 15, None, white, s) if d
         else lib.mb200_contrast_stretch_image(b, w, h, ch, 0.0, 0.0, 0, 15, black, None)),
        (_lib.EINVAL, lambda b, d: lib.mb200_linear_stretch_image_dev(b, w, h, ch, 0.0, 0.0, 15, None, C.byref(hi), s) if d
         else lib.mb200_linear_stretch_image(b, w, h, ch, 0.0, 0.0, 15, C.byref(lo), None)),
        (_lib.EINVAL, lambda b, d: lib.mb200_level_image_dev(b, w, h, 5, 0.0, 1.0, 1.0, 15, s) if d
         else lib.mb200_level_image(b, 0, h, ch, 0.0, 1.0, 1.0, 15)),
        (_lib.EINVAL, lambda b, d: lib.mb200_levelize_image_dev(b, w, 0, ch, 0.0, 1.0, 1.0, 15, s) if d
         else lib.mb200_levelize_image(b, w, h, 0, 0.0, 1.0, 1.0, 15)),
        (_lib.EINVAL, lambda b, d: lib.mb200_minmax_stretch_image_dev(b, w, h, 0, 0.0, 0.0, 1.0, 0, 15, s) if d
         else lib.mb200_minmax_stretch_image(b, w, h, 5, 0.0, 0.0, 1.0, 0, 15)),
        (_lib.EINVAL, lambda b, d: lib.mb200_gamma_image_dev(b, 0, h, ch, 2.2, 15, s) if d
         else lib.mb200_gamma_image(b, w, h, 7, 2.2, 15)),
        (_lib.EINVAL, lambda b, d: lib.mb200_identify_gray_dev(b, w, h, ch, None, s) if d
         else lib.mb200_identify_gray(b, w, h, ch, None)),
        (_lib.EUNSUPPORTED, lambda b, d: lib.mb200_contrast_stretch_image_dev(b, big, big, ch, 0.0, 0.0, 0, 15, black,
                                                                               white, s) if d
         else lib.mb200_contrast_stretch_image(b, big, big, ch, 0.0, 0.0, 0, 15, black, white)),
        (_lib.EUNSUPPORTED, lambda b, d: lib.mb200_linear_stretch_image_dev(b, big, big, ch, 0.0, 0.0, 15, C.byref(lo),
                                                                             C.byref(hi), s) if d
         else lib.mb200_linear_stretch_image(b, big, big, ch, 0.0, 0.0, 15, C.byref(lo), C.byref(hi))),
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
    # a linear image's intensity histogram is declined by the Python layer before any call
    with pytest.raises(im.MagickB200Error) as e:
        im.NormalizeImage(im.Image(src.copy(), im.RGBColorspace))
    assert e.value.code == _lib.EUNSUPPORTED
    # per channel, the reference levels a CMYK image's K too: declined, the buffer untouched
    cmyk = im.Image(torch.from_numpy(src.copy()).cuda(), im.CMYKColorspace)
    with pytest.raises(im.MagickB200Error) as e:
        im.AutoLevelImage(cmyk, 0b1111)
    assert e.value.code == _lib.EUNSUPPORTED
    np.testing.assert_array_equal(cmyk.pixels.cpu().numpy(), src)
