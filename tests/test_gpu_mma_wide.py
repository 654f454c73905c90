"""The wide-tile pass of conv_mma.cu (mma.sync.m16n8k16.f64, 16 outputs per tile) for RGBA windows of 18-33 taps,
against the oracle and against the 8x8x4 kernel it replaces there (`mma_wide` 0).

Bar: <= 1 ULP of the float Quantum against the reference arithmetic and >= 99.99 % bit-identical; the two tilings
accumulate in FP64 in a different association, so they may differ by 1 ULP in a few samples."""
import numpy as np
import pytest

import util
from util import P, make_image, max_ulp, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")

FAMILIES = ("conv_mma_launches", "conv_mma_wide_launches", "conv_pair_launches", "conv_pair_async_launches",
            "conv_generic_launches")


def _dev(a):
    import torch
    return im.Image(torch.from_numpy(a).cuda())


def _host(img):
    return img.pixels.cpu().numpy() if img.on_device else img.pixels


def orc(fn, src, *args):
    h, w, ch = src.shape
    dst = np.empty_like(src)
    assert getattr(oracle(), fn)(P(src), P(dst), w, h, ch, *args) == 0
    return dst


def counted(fn, **options):
    for k, v in options.items():
        util.set_option(k, v)
    n0 = {f: util.get_option(f) for f in FAMILIES}
    out = fn()
    return out, {f: util.get_option(f) - n0[f] for f in FAMILIES}


def positive_taps(n):
    """Exact binary fractions, a peak off the centre: every window sum is exact in FP64 up to its last additions."""
    i = np.arange(n)
    return (1.0 + (5 * i) % 11 + (i == n // 3) * 8) / 16.0


def kernel_string(values, axis):
    body = ",".join(repr(float(v)) for v in values)
    n, o = len(values), len(values) // 3
    return f"{n}x1+{o}+0: {body}" if axis == 0 else f"1x{n}+0+{o}: {body}"


def oracle_kernel(values, axis):
    v = np.asarray(values, np.float64)
    o = len(values) // 3
    return util.orc_kernel_from_array(v.reshape(1, -1) if axis == 0 else v.reshape(-1, 1),
                                      o if axis == 0 else 0, 0 if axis == 0 else o)


# 1-, 15- and 17-pixel lines along the filter axis, and sizes that are not multiples of 16
SIZES = [(1, 37), (15, 40), (17, 33), (37, 1), (40, 15), (33, 17), (259, 131), (131, 259)]


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("n", [18, 25, 33])
def test_wide_1d_kernels_against_the_oracle_and_the_8x8x4_kernel(n, axis):
    values = positive_taps(n)
    ks = kernel_string(values, axis)
    k = oracle_kernel(values, axis)
    exact = total = differing = 0
    for i, (w, h) in enumerate(SIZES):
        src = make_image(w, h, 4, seed=100 * n + i, kind=("noise", "alpha_blocks", "hdr")[i % 3])
        want = util.orc_morphology(src, im.ConvolveMorphology, 1, [k])
        run = lambda: _host(im.MorphologyImage(_dev(src), im.ConvolveMorphology, 1, ks))
        got, c = counted(run, conv_mma=1, mma_wide=1)
        assert c["conv_mma_wide_launches"] == 1 and c["conv_mma_launches"] == 1, c
        narrow, c = counted(run, mma_wide=0)
        assert c["conv_mma_wide_launches"] == 0 and c["conv_mma_launches"] == 1, c
        d = util.ulp_distance(got, want)
        assert d.max() <= 1, (n, axis, (w, h), int(d.max()))
        assert max_ulp(got, narrow) <= 1, (n, axis, (w, h))
        exact += int((d == 0).sum())
        total += d.size
        differing += int((got != narrow).sum())
    print(f"\n{n} taps, axis {axis}: {differing} of {total} samples differ by 1 ULP from the 8x8x4 kernel")
    assert exact / total >= 0.9999, (n, axis, exact / total)


@pytest.mark.parametrize("radius,sigma", [(9.0, 3.0), (12.0, 3.0), (0.0, 4.0), (16.0, 5.0)])
def test_wide_blur_against_the_oracle_and_the_8x8x4_kernel(radius, sigma):
    src = make_image(1031, 517, 4, seed=42, kind="alpha_blocks")
    want = orc("orc_blur", src, radius, sigma)
    got, c = counted(lambda: _host(im.BlurImage(_dev(src), radius, sigma)), conv_mma=1, mma_wide=-1)
    assert c["conv_mma_wide_launches"] == 2 and c["conv_mma_launches"] == 2, c
    d = util.ulp_distance(got, want)
    assert d.max() <= 1 and (d == 0).mean() >= 0.9999, (int(d.max()), float((d == 0).mean()))
    narrow, c = counted(lambda: _host(im.BlurImage(_dev(src), radius, sigma)), mma_wide=0)
    assert c["conv_mma_wide_launches"] == 0 and c["conv_mma_launches"] == 2, c
    assert max_ulp(got, narrow) <= 1
    print(f"\nblur({radius}, {sigma}): {int((got != narrow).sum())} of {got.size} samples differ by 1 ULP "
          "from the 8x8x4 kernel")


def test_wide_strip_seams_give_identical_bits():
    """mma_strip 8 and 24 are rounded up to 16 and 32: every output keeps its k-grouping, so its bits."""
    for (w, h) in ((40, 1500), (1500, 40)):
        src = make_image(w, h, 4, seed=9, kind="alpha_blocks")
        want = orc("orc_blur", src, 0.0, 4.0)
        first = None
        for strip in (8, 24, 512):
            got, c = counted(lambda: _host(im.BlurImage(_dev(src), 0.0, 4.0)), conv_mma=1, mma_strip=strip)
            assert c["conv_mma_wide_launches"] == 2, c
            assert max_ulp(got, want) <= 1
            if first is None:
                first = got
            else:
                assert np.array_equal(got, first), ((w, h), strip, max_ulp(got, first))


@pytest.mark.parametrize("radius,sigma", [(9.0, 3.0), (12.0, 3.6), (0.0, 4.0)])
def test_wide_non_finite_samples_stay_local(radius, sigma):
    """inf / NaN inside, next to and outside the windows of a 16-output block: the flagged blocks take the scalar
    path and poison exactly the outputs the reference poisons."""
    src = make_image(150, 110, 4, seed=21)
    src[30, 40, 0] = np.inf
    src[31, 90, 3] = -np.inf
    src[80, 20, 1] = np.nan
    src[100, 140, 0] = np.inf
    src[0, 0, 2] = np.inf
    src[109, 149, 3] = np.nan
    src[64, 47, 2] = np.nan           # on a 16-position block boundary of both axes
    src[48, 96, 1] = -np.inf
    want = orc("orc_blur", src, radius, sigma)
    got, c = counted(lambda: _host(im.BlurImage(_dev(src), radius, sigma)), conv_mma=1)
    assert c["conv_mma_wide_launches"] == 2, c
    assert np.isfinite(want).mean() > 0.3
    assert np.array_equal(np.isnan(got), np.isnan(want))
    inf = np.isinf(want)
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], want[inf])
    ok = np.isfinite(want)
    d = util.ulp_distance(np.where(ok, got, np.float32(0)), np.where(ok, want, np.float32(0)))
    assert d.max() <= 1


@pytest.mark.parametrize("args", [(0.0, 4.0, 1.5, 0.02), (12.0, 3.0, 0.8, 0.0)])
def test_wide_unsharp_epilogue_equals_the_separate_point_pass(args):
    src = make_image(333, 217, 4, seed=5, kind="alpha_blocks")
    want = orc("orc_unsharp", src, *args)
    fused, c = counted(lambda: _host(im.UnsharpMaskImage(_dev(src), *args)), conv_mma=1)
    assert c["conv_mma_wide_launches"] == 2, c
    assert max_ulp(fused, want) <= 1
    unfused, c = counted(lambda: _host(im.UnsharpMaskImage(_dev(src), *args)), no_fused_unsharp=1)
    assert c["conv_mma_wide_launches"] == 2, c
    assert np.array_equal(fused, unfused)


def test_wide_unaligned_source_declines_to_the_generic_kernel():
    """The row pass reads the unaligned source and declines to the DFMA generic kernel; the column pass reads the
    aligned intermediate and runs on the wide tiles."""
    import torch
    src = make_image(131, 97, 4, seed=8, kind="alpha_blocks")
    flat = torch.empty(src.size + 1, dtype=torch.float32, device="cuda")
    t = flat[1:].view(src.shape)
    t.copy_(torch.from_numpy(src))
    img = im.Image(t)
    assert img.pixels.data_ptr() % 16 == 4
    got, c = counted(lambda: _host(im.BlurImage(img, 0.0, 4.0)), conv_mma=1)
    assert c["conv_generic_launches"] == 1 and c["conv_mma_wide_launches"] == 1, c
    assert max_ulp(got, orc("orc_blur", src, 0.0, 4.0)) <= 1


def test_wide_launch_counter_under_each_mma_wide_value():
    src = make_image(67, 45, 4, seed=2)
    for wide, n_wide in ((-1, 2), (0, 0), (1, 2)):
        _, c = counted(lambda: _host(im.BlurImage(_dev(src), 0.0, 4.0)), conv_mma=-1, mma_wide=wide)
        assert c["conv_mma_launches"] == 2 and c["conv_mma_wide_launches"] == n_wide, (wide, c)
        # 17 taps keep the 8x8x4 tiles; the rank-1 passes with a double intermediate keep them too
        _, c = counted(lambda: _host(im.BlurImage(_dev(src), 0.0, 2.0)))
        assert c["conv_mma_launches"] == 2 and c["conv_mma_wide_launches"] == 0, (wide, c)
        _, c = counted(lambda: _host(im.GaussianBlurImage(_dev(src), 0.0, 4.0)), conv_mma=1)
        assert c["conv_mma_launches"] == 2 and c["conv_mma_wide_launches"] == 0, (wide, c)
        util.set_option("conv_mma", -1)
    for bad in (-2, 2):
        with pytest.raises(Exception):
            util.set_option("mma_wide", bad)
    assert util.get_option("mma_wide") == 1
