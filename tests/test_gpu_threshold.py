"""AdaptiveThresholdImage, AutoThresholdImage, RangeThresholdImage and PerceptibleImage on the GPU, through the device
and the host-buffer entry points of the Python layer, against the oracle (itself pinned to the reference by
test_oracle_threshold_vs_ref.py): 0 ULP with identical NaN positions, and the same "auto-threshold:threshold" value.

Plus both AdaptiveThreshold kernel families (launch counters, identical bits across the tile / direct switch), widths
around the tile's 32 columns and heights around its 32-row band, an 8192^2 RGBA `-lat 15x15+5%` checked whole and
repeated, an RGBA buffer 4 bytes off a 16-byte boundary, gray RangeThreshold through the sRGB transform, and the
declines, which leave `dst` untouched."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

import imagemagick_b200 as im
import threshold_cases as tc
import util
from imagemagick_b200 import _lib
from util import make_image

pytestmark = pytest.mark.gpu

CHANNELS = [1, 2, 3, 4]


def same(got, want, what):
    assert got.shape == want.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    assert util.max_ulp(np.where(np.isnan(got), 0, got).astype(np.float32),
                        np.where(np.isnan(want), 0, want).astype(np.float32)) == 0, what


def py_call(img, op, args, mask):
    channels = None if mask < 0 else tc.update_mask(mask, img.channels)
    if op == tc.ADAPTIVE:
        return im.AdaptiveThresholdImage(img, int(args[0]), int(args[1]), args[2], channels), ""
    if op == tc.AUTO:
        return img, "%g%%" % im.AutoThresholdImage(img, int(args[0]))
    if op == tc.RANGE:
        im.RangeThresholdImage(img, *args, channels=channels)
        return img, ""
    im.PerceptibleImage(img, args[0], channels)
    return img, ""


def check(src, op, args, mask=-1, what=""):
    want, want_prop = tc.orc_run(src, op, args, mask)
    for img in (im.Image(torch.from_numpy(src.copy()).cuda()), im.Image(src.copy())):
        out, prop = py_call(img, op, args, mask)
        got = out.pixels.cpu().numpy() if out.on_device else out.pixels
        same(got, want, (what, img.on_device))
        assert prop == want_prop, (what, prop, want_prop)


def counter(name):
    return util.get_option(name)


@pytest.mark.parametrize("ch", CHANNELS)
def test_adaptive_threshold(ch):
    for name, src in tc.sources(ch).items():
        for ww, wh, bias in tc.WINDOWS:
            check(src, tc.ADAPTIVE, (ww, wh, bias), what=(name, ww, wh, bias))
    for mname, mask in tc.CHANNEL_MASKS.items():
        check(tc.sources(ch)["mosaic"], tc.ADAPTIVE, (5, 3, 300.0), mask, what=mname)


@pytest.mark.parametrize("ch", CHANNELS)
def test_adaptive_threshold_families(ch):
    """The tile and the direct family give the same bits; the launch counters prove which served each call."""
    for (w, h) in [(31, 31), (32, 32), (33, 33), (65, 63), (97, 7), (5, 70)]:
        src = make_image(w, h, ch, seed=w * h + ch, kind="hdr")
        for ww, wh in [(3, 3), (15, 15), (40, 9), (200, 200)]:
            want, _ = tc.orc_run(src, tc.ADAPTIVE, (ww, wh, 250.0))
            results = {}
            for direct in (0, 1):
                util.set_option("no_adaptive_tile", direct)
                t0, d0 = counter("adaptive_threshold_tile_launches"), counter("adaptive_threshold_direct_launches")
                got = im.AdaptiveThresholdImage(im.Image(torch.from_numpy(src).cuda()), ww, wh, 250.0).pixels.cpu().numpy()
                t1, d1 = counter("adaptive_threshold_tile_launches"), counter("adaptive_threshold_direct_launches")
                tile = ww < 200 and not direct          # a 200x200 tile does not fit in shared memory
                assert (t1 - t0, d1 - d0) == ((1, 0) if tile else (0, 1)), (w, h, ww, wh, direct)
                same(got, want, (w, h, ww, wh, direct))
                results[direct] = got
            util.set_option("no_adaptive_tile", 0)
            assert results[0].tobytes() == results[1].tobytes()


def test_adaptive_threshold_8192_rgba():
    """-lat 15x15+5% on 8192^2 RGBA, checked whole against the oracle, twice with identical bits."""
    src = make_image(8192, 8192, 4, seed=77)
    want, _ = tc.orc_run(src, tc.ADAPTIVE, (15, 15, 65535.0 * 0.05))
    x = im.Image(torch.from_numpy(src).cuda())
    a = im.AdaptiveThresholdImage(x, 15, 15, 65535.0 * 0.05).pixels.cpu().numpy()
    b = im.AdaptiveThresholdImage(x, 15, 15, 65535.0 * 0.05).pixels.cpu().numpy()
    assert np.array_equal(a, want)
    assert a.tobytes() == b.tobytes()


def test_adaptive_threshold_unaligned_rgba():
    src = make_image(37, 29, 4, seed=3, kind="hdr")
    want, _ = tc.orc_run(src, tc.ADAPTIVE, (7, 5, -100.0))
    n = src.size
    big = torch.zeros(2 * n + 8, device="cuda")
    s, d = big[1:1 + n], big[n + 2:2 * n + 2]                   # 4 bytes off a 16-byte boundary
    s.copy_(torch.from_numpy(src.ravel()).cuda())
    lib = _lib.load()
    _lib.check(lib.mb200_adaptive_threshold_image_dev(s.data_ptr(), d.data_ptr(), 37, 29, 4, 7, 5, -100.0, 0xF, None))
    torch.cuda.synchronize()
    same(d.cpu().numpy().reshape(29, 37, 4), want, "unaligned")


@pytest.mark.parametrize("ch", CHANNELS)
def test_auto_threshold(ch):
    for name, src in tc.auto_sources(ch).items():
        for method in tc.AUTO_METHODS:
            check(src, tc.AUTO, (method,), what=(name, method))


@pytest.mark.parametrize("ch", CHANNELS)
def test_auto_threshold_bin_edges_one_by_one(ch):
    """Each sample near a 256-bin edge decides the threshold of its own image: the bins match the oracle's one by one."""
    want = tc.edge_thresholds(lambda img: float(tc.orc_run(img, tc.AUTO, (tc.OTSU,))[1].rstrip("%")), ch)
    for device in (True, False):
        def run(img):
            x = im.Image(torch.from_numpy(img.copy()).cuda() if device else img.copy())
            return float("%g" % im.AutoThresholdImage(x, im.OTSUThresholdMethod))      # as the property prints it
        got = tc.edge_thresholds(run, ch)
        assert np.array_equal(got, want), (device, np.flatnonzero(got != want)[:8])


@pytest.mark.parametrize("ch", [3, 4])
def test_range_threshold(ch):
    for k, limits in enumerate(tc.RANGES):
        for name, src in (("limits", tc.range_source(ch)), ("mosaic", tc.sources(ch)["mosaic"])):
            for mname, mask in tc.CHANNEL_MASKS.items():
                check(src, tc.RANGE, limits, mask, what=(name, k, mname))


@pytest.mark.parametrize("ch", [1, 2])
def test_range_threshold_gray(ch):
    """A gray image is transformed to sRGB first; the result equals the oracle on the transformed image."""
    src = make_image(19, 11, ch, seed=8)
    rgb = im.Image(torch.from_numpy(src.copy()).cuda(), im.GRAYColorspace)
    im.TransformImageColorspace(rgb, im.sRGBColorspace)
    want, _ = tc.orc_run(rgb.pixels.cpu().numpy(), tc.RANGE, tc.RANGES[0])
    img = im.Image(torch.from_numpy(src.copy()).cuda(), im.GRAYColorspace)
    im.RangeThresholdImage(img, *tc.RANGES[0])
    assert img.channels == ch + 2 and img.colorspace == im.sRGBColorspace
    same(img.pixels.cpu().numpy(), want, "gray")


@pytest.mark.parametrize("ch", CHANNELS)
def test_perceptible(ch):
    src = tc.perceptible_source(ch)
    for eps in tc.EPSILONS:
        for mname, mask in tc.CHANNEL_MASKS.items():
            check(src, tc.PERCEPTIBLE, (eps,), mask, what=(eps, mname))


def test_declines_leave_dst_untouched():
    lib = _lib.load()
    src = torch.from_numpy(make_image(16, 8, 4, seed=1)).cuda()
    dst = torch.full_like(src, 7.0)
    big = 4097                                                  # MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW + 1
    assert lib.mb200_adaptive_threshold_image_dev(src.data_ptr(), dst.data_ptr(), 16, 8, 4, big, 3, 0.0, 0xF, None) == _lib.EUNSUPPORTED
    assert lib.mb200_adaptive_threshold_image_dev(src.data_ptr(), dst.data_ptr(), 16, 8, 5, 3, 3, 0.0, 0xF, None) == _lib.EINVAL
    t = C.c_double(-1.0)
    assert lib.mb200_auto_threshold_image_dev(dst.data_ptr(), 16, 8, 4, 9, C.byref(t), None) == _lib.EINVAL
    gray = torch.full((8, 16, 1), 7.0, device="cuda")
    assert lib.mb200_range_threshold_image_dev(gray.data_ptr(), 16, 8, 1, 0.0, 1.0, 2.0, 3.0, 0, 1, None) == _lib.EUNSUPPORTED
    torch.cuda.synchronize()
    assert bool((dst == 7.0).all()) and bool((gray == 7.0).all()) and t.value == -1.0
