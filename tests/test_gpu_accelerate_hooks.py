"""DespeckleImage, LocalContrastImage and WaveletDenoiseImage on the GPU: the device and host-buffer entry points are
bit exact against the oracle (itself pinned to the reference by test_oracle_hooks_vs_ref.py), and the declines return
MB200_EUNSUPPORTED without writing the destination."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

import imagemagick_b200 as im
from imagemagick_b200 import _lib
from test_oracle_hooks_vs_ref import (KINDS, hook_image, oracle_despeckle, oracle_local_contrast, oracle_wavelet)
from util import digest

pytestmark = pytest.mark.gpu


def both(fn, src, *args):
    """The operator through the device entry point and through the host-buffer one."""
    dev = fn(im.Image(torch.from_numpy(src).cuda()), *args).pixels.cpu().numpy()
    host = fn(im.Image(src.copy()), *args).pixels
    return dev, host


def assert_same(got, want, what):
    assert got.shape == want.shape, what
    assert digest(got) == digest(want), (what, int(np.sum(~((got == want) | (np.isnan(got) & np.isnan(want))))))


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_despeckle_bit_exact(ch, kind):
    for w, h in [(37, 23), (19, 41), (1, 17), (23, 1), (2, 2), (97, 70)]:
        src = hook_image(w, h, ch, kind)
        want = oracle_despeckle(src)
        for got in both(im.DespeckleImage, src):
            assert_same(got, want, (w, h))


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["noise", "alpha_blocks", "hdr", "posterised", "black"])
def test_local_contrast_bit_exact(ch, kind):
    cases = [(61, 47, 0.0, 12.5), (61, 47, 10.0, 12.5), (61, 47, 40.0, -40.0), (61, 47, 100.0, 100.0),
             (61, 47, 250.0, 0.0), (61, 47, 491.0, 12.5), (23, 67, 164.0, 60.0), (23, 67, -20.0, -12.5),
             (1100, 9, 60.0, 12.5)]
    for w, h, radius, strength in cases:
        src = hook_image(w, h, ch, kind)
        want = oracle_local_contrast(src, radius, strength)
        for got in both(im.LocalContrastImage, src, radius, strength):
            assert_same(got, want, (w, h, radius, strength))


def test_local_contrast_black_pixels_nan_on_the_gpu():
    src = hook_image(61, 47, 3, "black")
    got = im.LocalContrastImage(im.Image(torch.from_numpy(src).cuda()), 10.0, 12.5).pixels.cpu().numpy()
    black = (src == 0).all(axis=2)
    assert np.isnan(got[black]).all() and not np.isnan(got[~black]).any()


def test_local_contrast_wide_kernel():
    """width in the hundreds: (ssize_t) (1500 * 0.002 * 120) = 360, 719 taps per pass, several shared-memory chunks."""
    src = hook_image(1500, 400, 4, "alpha_blocks")
    want = oracle_local_contrast(src, 120.0, 12.5)
    for got in both(im.LocalContrastImage, src, 120.0, 12.5):
        assert_same(got, want, "width 360")


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_wavelet_denoise_bit_exact(ch, kind):
    cases = [(32, 32, 0.0, 0.0), (33, 45, 500.0, 0.0), (45, 32, 500.0, 0.3), (64, 37, 6553.5, 1.0),
             (37, 64, 6553.5, 0.3), (40, 33, 20000.0, 0.0), (300, 200, 3000.0, 0.3)]
    for w, h, threshold, softness in cases:
        src = hook_image(w, h, ch, kind)
        want = oracle_wavelet(src, threshold, softness)
        for got in both(im.WaveletDenoiseImage, src, threshold, softness):
            assert_same(got, want, (w, h, threshold, softness))


def _declines(dev_fn, host_fn, src, *args):
    lib = _lib.load()
    h, w, ch = src.shape
    d_src = torch.from_numpy(src).cuda()
    d_dst = torch.full_like(d_src, -3.0)
    rc = getattr(lib, dev_fn)(d_src.data_ptr(), d_dst.data_ptr(), w, h, ch, *args, None)
    torch.cuda.synchronize()
    assert rc == _lib.EUNSUPPORTED and bool((d_dst == -3.0).all())
    dst = np.full_like(src, -3.0)
    rc = getattr(lib, host_fn)(src.ctypes.data_as(C.c_void_p), dst.ctypes.data_as(C.c_void_p), w, h, ch, *args)
    assert rc == _lib.EUNSUPPORTED and bool((dst == -3.0).all())


def test_declines_leave_dst_untouched():
    # LocalContrast: width 61 > columns - 1 = 60; a tall image whose width exceeds its columns; a non-finite radius
    _declines("mb200_local_contrast_image_dev", "mb200_local_contrast_image", hook_image(61, 47, 3, "noise"), 500.0, 12.5)
    _declines("mb200_local_contrast_image_dev", "mb200_local_contrast_image", hook_image(3, 600, 4, "noise"), 2.5, 12.5)
    _declines("mb200_local_contrast_image_dev", "mb200_local_contrast_image", hook_image(30, 30, 1, "noise"),
              float("inf"), 12.5)
    # WaveletDenoise: below 32 samples per line
    for w, h in [(31, 40), (40, 31)]:
        _declines("mb200_wavelet_denoise_image_dev", "mb200_wavelet_denoise_image", hook_image(w, h, 3, "noise"), 500.0, 0.0)
    # ... while the bounds themselves are served
    src = hook_image(61, 47, 3, "noise")
    assert_same(im.LocalContrastImage(im.Image(src), 492.0, 12.5).pixels, oracle_local_contrast(src, 492.0, 12.5), "492")
    src = hook_image(32, 32, 4, "noise")
    assert_same(im.WaveletDenoiseImage(im.Image(src), 500.0, 0.3).pixels, oracle_wavelet(src, 500.0, 0.3), "32x32")


def test_unaligned_device_pointers():
    """The kernels load and store scalars: an RGBA buffer 4 bytes off a 16-byte boundary is served, bit exact."""
    lib = _lib.load()
    src = hook_image(45, 38, 4, "alpha_blocks")
    n = src.size
    d = torch.empty(2 * n + 2, dtype=torch.float32, device="cuda")
    d_src, d_dst = d[1:n + 1], d[n + 1:2 * n + 1]
    d_src.copy_(torch.from_numpy(src.ravel()))
    runs = [("mb200_despeckle_image_dev", (), oracle_despeckle(src)),
            ("mb200_local_contrast_image_dev", (20.0, 30.0), oracle_local_contrast(src, 20.0, 30.0)),
            ("mb200_wavelet_denoise_image_dev", (2000.0, 0.3), oracle_wavelet(src, 2000.0, 0.3))]
    for fn, args, want in runs:
        _lib.check(getattr(lib, fn)(d_src.data_ptr(), d_dst.data_ptr(), 45, 38, 4, *args, None))
        torch.cuda.synchronize()
        assert_same(d_dst.cpu().numpy().reshape(src.shape), want, fn)


@pytest.mark.parametrize("op", ["despeckle", "local_contrast", "wavelet"])
def test_full_size_rgba(op):
    """One 8192^2 RGBA image per operator (LocalContrast at the CLI's 10x12.5: width 163)."""
    src = hook_image(8192, 8192, 4, "alpha_blocks", seed=11)
    fn, args, want = {
        "despeckle": (im.DespeckleImage, (), oracle_despeckle),
        "local_contrast": (im.LocalContrastImage, (10.0, 12.5), oracle_local_contrast),
        "wavelet": (im.WaveletDenoiseImage, (6553.5, 0.0), oracle_wavelet),
    }[op]
    got = fn(im.Image(torch.from_numpy(src).cuda()), *args).pixels.cpu().numpy()
    assert_same(got, want(src, *args), op)
