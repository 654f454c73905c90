"""TransformImageColorspace to and from GRAY, LinearGRAY and CMYK (the colourspaces that change the channel layout),
through mb200_transform_colorspace_layout[_dev] and the Python layer, against the oracle (itself pinned to the reference
by test_oracle_layout_vs_ref.py):

- bit exact: sRGB <-> GRAY and sRGB <-> CMYK, with and without alpha, NaN / +-inf and near-black samples included;
- <= 1 ULP: sRGB <-> LinearGRAY (a gamma step);
- hops through the in-place legs: the result is exactly the direct leg composed with the in-place leg the library
  runs on its own, and against the oracle it is bounded by what a 1-ULP error of the sRGB intermediate can become: for
  a hop into a layout space the oracle's direct leg is evaluated on every intermediate within 1 ULP per channel, and
  the GPU's sample must be one of those values (a red error scaled into a smaller gray, or divided by 1 - K near black,
  is covered exactly).  Where the in-place leg's own contract lets the intermediate differ by a sub-1e-6 residue
  instead, the composition check is what pins the pixel.

Plus 8192^2 RGBA -> GA and -> CMYKA, buffers off their vector alignment, a guard region after dst, every decline code
with dst untouched, and the Python layer's re-layout and re-tag.  The declines of the host entry point and the layout
rule need no device."""
from __future__ import annotations

import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import imagemagick_b200 as im
import layout_cases as lc
from imagemagick_b200 import _lib
from util import P, make_image, ulp_distance, ulp_or_noise

gpu = pytest.mark.gpu
DIRECT = [(lc.SRGB, lc.GRAY), (lc.SRGB, lc.LINEAR_GRAY), (lc.GRAY, lc.SRGB), (lc.LINEAR_GRAY, lc.SRGB),
          (lc.SRGB, lc.CMYK), (lc.CMYK, lc.SRGB)]
SCRGB, TRANSPARENT = 22, 24


def _id(pair):
    return f"{lc.NAMES[pair[0]]}-{lc.NAMES[pair[1]]}"


def ulps(got, want):
    """Per-sample ULP distance; NaN must sit exactly where the oracle has NaN."""
    assert got.shape == want.shape, (got.shape, want.shape)
    nan_got, nan_want = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_got, nan_want), int(np.sum(nan_got != nan_want))
    return ulp_distance(np.where(nan_got, np.float32(0), got), np.where(nan_want, np.float32(0), want))


def stream():
    """torch's current stream (its legacy default stream is named explicitly: NULL means the library's own stream)."""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream or 1)


def run_dev(src, from_cs, to_cs, settings=None, offset=0, guard=0):
    """The device entry point on src (`offset` floats into its allocation) into a dst `offset` floats into a buffer with
    `guard` sentinel floats after it.  Returns (rc, dst, guard samples)."""
    h, w, ch = src.shape
    out_ch = lc.channels(to_cs, ch != lc.channels(from_cs, False))
    d_src = torch.empty(src.size + offset, dtype=torch.float32, device="cuda")
    d_src[offset:] = torch.from_numpy(src.ravel())
    d_dst = torch.full((h * w * out_ch + offset + guard,), -7.0, dtype=torch.float32, device="cuda")
    rc = _lib.load().mb200_transform_colorspace_layout_dev(d_src.data_ptr() + 4 * offset, ch, d_dst.data_ptr() + 4 * offset,
                                                           out_ch, w, h, from_cs, to_cs, lc.options(settings), stream())
    torch.cuda.synchronize()
    host = d_dst.cpu().numpy()
    return rc, host[offset:offset + h * w * out_ch].reshape(h, w, out_ch), host[offset + h * w * out_ch:]


def run_host(src, from_cs, to_cs, settings=None):
    h, w, ch = src.shape
    out = np.full((h, w, lc.channels(to_cs, ch != lc.channels(from_cs, False))), -7.0, np.float32)
    rc = _lib.load().mb200_transform_colorspace_layout(P(src), ch, P(out), out.shape[2], w, h, from_cs, to_cs,
                                                       lc.options(settings))
    return rc, out


def gpu_both(src, from_cs, to_cs, settings=None):
    rc, dev, _ = run_dev(src, from_cs, to_cs, settings)
    assert rc == 0, _lib.load().mb200_last_error()
    rc, host = run_host(src, from_cs, to_cs, settings)
    assert rc == 0, _lib.load().mb200_last_error()
    return [dev, host]


def in_place(src, from_cs, to_cs, settings=None):
    """The library's own in-place leg (3 / 4 channels) on the device."""
    h, w, ch = src.shape
    d = torch.from_numpy(src.copy()).cuda()
    assert _lib.load().mb200_transform_colorspace_ex_dev(d.data_ptr(), w, h, ch, from_cs, to_cs, lc.options(settings),
                                                         stream()) == 0
    return d.cpu().numpy()


# ------------------------------------------------------------------------------------------------------ direct legs
@gpu
@pytest.mark.parametrize("alpha", [False, True])
@pytest.mark.parametrize("pair", DIRECT, ids=_id)
def test_direct_legs(pair, alpha):
    from_cs, to_cs = pair
    bar = 1 if lc.LINEAR_GRAY in pair else 0
    for src in [lc.source(from_cs, alpha)] + [make_image(w, h, lc.channels(from_cs, alpha), seed=w + h, kind="hdr")
                                              for w, h in [(1, 29), (31, 1)]]:
        want = lc.orc_layout(src, from_cs, to_cs)
        for got in gpu_both(src, from_cs, to_cs):
            assert int(ulps(got, want).max()) <= bar, src.shape


@gpu
@pytest.mark.parametrize("pair", [(lc.SRGB, lc.GRAY), (lc.SRGB, lc.CMYK), (lc.CMYK, lc.SRGB), (lc.GRAY, lc.SRGB)], ids=_id)
def test_direct_legs_unaligned_with_guard(pair):
    """Both buffers 4 bytes off their float4 / float2 alignment, and 64 sentinel floats after dst stay untouched."""
    from_cs, to_cs = pair
    for alpha in (False, True):
        src = lc.source(from_cs, alpha, w=41, seed=3)
        want = lc.orc_layout(src, from_cs, to_cs)
        for offset in (0, 1):
            rc, got, guard = run_dev(src, from_cs, to_cs, offset=offset, guard=64)
            assert rc == 0
            assert int(ulps(got, want).max()) == 0, (alpha, offset)
            assert np.all(guard == -7.0)


@gpu
@pytest.mark.parametrize("to_cs", [lc.GRAY, lc.CMYK], ids=lambda c: lc.NAMES[c])
def test_full_size_rgba(to_cs):
    """8192^2 RGBA -> GA / CMYKA on the device, bit exact."""
    src = make_image(8192, 8192, 4, seed=1)
    want = lc.orc_layout(src, lc.SRGB, to_cs)
    rc, got, guard = run_dev(src, lc.SRGB, to_cs, guard=16)
    assert rc == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.all(guard == -7.0)


# ------------------------------------------------------------------------------------------------------ hops
def _perturbed(x):
    """x with every colour channel moved by -1, 0 or +1 ULP: all 27 combinations (alpha unchanged)."""
    steps = [np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf))]
    for combo in itertools.product(range(3), repeat=3):
        y = x.copy()
        for c, k in enumerate(combo):
            y[..., c] = steps[k][..., c]
        yield y


@gpu
@pytest.mark.parametrize("layout", lc.LAYOUT, ids=lambda c: lc.NAMES[c])
@pytest.mark.parametrize("space", lc.HOP_SPACES, ids=lambda c: lc.NAMES[c])
def test_hop_into_layout(space, layout):
    """space -> sRGB (in-place leg on a temporary) -> layout."""
    for alpha in (False, True):
        src = make_image(33, 19, 3 + alpha, seed=space + layout)
        gpu_rgb = in_place(src, space, lc.SRGB)
        for got in gpu_both(src, space, layout):
            # exactly the direct leg on the library's own intermediate (<= 1 ULP for LinearGRAY's gamma step)
            bar = 1 if layout == lc.LINEAR_GRAY else 0
            assert int(ulps(got, lc.orc_layout(gpu_rgb, lc.SRGB, layout)).max()) <= bar
            # against the oracle: the value of the direct leg at some intermediate within 1 ULP of the oracle's
            rgb = src.copy()
            assert lc.oracle().orc_colorspace_layout(P(src), src.shape[2], P(rgb), rgb.shape[2], 33, 19, space, lc.SRGB,
                                                     None) == 0
            # the in-place leg's own contract (test_gpu_parity): <= 1 ULP, or a difference below 1e-6 absolute
            assert int(ulp_or_noise(gpu_rgb, rgb).max()) <= 1, "in-place leg"
            within = (ulp_distance(gpu_rgb, rgb)[..., :3] <= 1).all(axis=2)
            best = None
            for y in _perturbed(rgb):
                d = ulps(got, lc.orc_layout(y, lc.SRGB, layout)).max(axis=2)
                best = d if best is None else np.minimum(best, d)
            assert int(np.where(within, best, 0).max()) <= bar, (lc.NAMES[space], lc.NAMES[layout], alpha)
            # an intermediate off by more than 1 ULP is a sub-1e-6 residue of the in-place leg; the direct leg on the
            # library's intermediate (checked above) is what those pixels hold


@gpu
@pytest.mark.parametrize("layout", lc.LAYOUT, ids=lambda c: lc.NAMES[c])
@pytest.mark.parametrize("space", lc.HOP_SPACES, ids=lambda c: lc.NAMES[c])
def test_hop_out_of_layout(space, layout):
    """layout -> sRGB (direct leg into dst) -> space (in-place leg on dst): exactly the composition of the library's own
    legs, and within 1 ULP of the oracle where the direct leg is exact (GRAY, CMYK) and the in-place leg is a smooth
    function of its input (the polar hue of LCHab and the tabled Log / YCC legs take the composition check only)."""
    for alpha in (False, True):
        src = lc.source(layout, alpha, w=23, seed=space)
        for got in gpu_both(src, layout, space):
            rc, rgb, _ = run_dev(src, layout, lc.SRGB)
            assert rc == 0
            assert int(ulps(got, in_place(rgb, lc.SRGB, space)).max()) == 0
            if layout != lc.LINEAR_GRAY and space not in (lc.LCHAB, lc.LOG, lc.YCC):
                assert int(ulps(got, lc.orc_layout(src, layout, space)).max()) <= 1, (lc.NAMES[space], alpha)


@gpu
@pytest.mark.parametrize("pair", [(lc.GRAY, lc.CMYK), (lc.CMYK, lc.GRAY), (lc.LINEAR_GRAY, lc.GRAY),
                                  (lc.GRAY, lc.LINEAR_GRAY), (lc.CMYK, lc.LINEAR_GRAY)], ids=_id)
def test_between_layout_spaces(pair):
    from_cs, to_cs = pair
    bar = 1 if lc.LINEAR_GRAY in pair else 0
    for alpha in (False, True):
        src = lc.source(from_cs, alpha, seed=13)
        want = lc.orc_layout(src, from_cs, to_cs)
        for got in gpu_both(src, from_cs, to_cs):
            d = ulps(got, want)
            if from_cs == lc.LINEAR_GRAY:
                # the 1-ULP gamma step of the first leg passes through the second: compose the two direct legs instead
                rc, rgb, _ = run_dev(src, from_cs, lc.SRGB)
                assert rc == 0
                d = ulps(got, lc.orc_layout(rgb, lc.SRGB, to_cs))
            assert int(d.max()) <= bar, alpha


@gpu
def test_hop_settings_reach_the_in_place_legs():
    src = make_image(29, 17, 4, seed=5)
    for space, settings in [(lc.LAB, {"color:illuminant": "D50"}), (lc.LOG, {"reference-white": "700"})]:
        for got in gpu_both(src, space, lc.GRAY, settings):
            assert int(ulps(got, lc.orc_layout(in_place(src, space, lc.SRGB, settings), lc.SRGB, lc.GRAY)).max()) == 0
        assert not np.array_equal(gpu_both(src, space, lc.GRAY, settings)[0], gpu_both(src, space, lc.GRAY)[0])


# ------------------------------------------------------------------------------------------------------ declines
DECLINES = [
    (lc.GRAY, 3, lc.SRGB, 3, _lib.EINVAL),           # a gray source has 1 or 2 channels
    (lc.SRGB, 4, lc.CMYK, 4, _lib.EINVAL),           # RGBA -> CMYKA has 5
    (lc.SRGB, 4, lc.GRAY, 1, _lib.EINVAL),           # alpha is carried over
    (lc.CMYK, 6, lc.SRGB, 5, _lib.EINVAL),
    (SCRGB, 3, lc.GRAY, 1, _lib.EUNSUPPORTED),
    (lc.GRAY, 1, TRANSPARENT, 3, _lib.EUNSUPPORTED),
]


def test_host_declines_leave_dst_untouched():
    """Checked before anything is staged: no device is needed."""
    lib = _lib.load()
    for from_cs, ch, to_cs, out_ch, code in DECLINES:
        src = make_image(7, 5, ch, seed=1)
        dst = np.full((5, 7, out_ch), -7.0, np.float32)
        assert lib.mb200_transform_colorspace_layout(P(src), ch, P(dst), out_ch, 7, 5, from_cs, to_cs, None) == code
        assert np.all(dst == -7.0)
    bad = im.ColorspaceOptions()
    bad.set, bad.illuminant = 1, 11
    src, dst = make_image(7, 5, 3, seed=1), np.full((5, 7, 1), -7.0, np.float32)
    assert lib.mb200_transform_colorspace_layout(P(src), 3, P(dst), 1, 7, 5, lc.LAB, lc.GRAY, C.byref(bad)) == _lib.EINVAL
    assert lib.mb200_transform_colorspace_layout(P(src), 3, P(src), 3, 7, 5, lc.SRGB, lc.LAB, None) == _lib.EINVAL
    assert np.all(dst == -7.0)


def test_layout_rule_and_python_image():
    lib = _lib.load()
    assert [lib.mb200_colorspace_channels(cs, a) for cs in (lc.GRAY, lc.LINEAR_GRAY, lc.CMYK, lc.SRGB, lc.LAB, SCRGB)
            for a in (0, 1)] == [1, 2, 1, 2, 4, 5, 3, 4, 3, 4, 3, 4]
    assert im.Image(np.zeros((2, 3, 5), np.float32), im.CMYKColorspace).channels == 5
    with pytest.raises(ValueError):
        im.Image(np.zeros((2, 3, 5), np.float32))


@gpu
def test_device_declines_leave_dst_untouched():
    for from_cs, ch, to_cs, out_ch, code in DECLINES:
        src = make_image(7, 5, ch, seed=1)
        h, w = 5, 7
        d_src = torch.from_numpy(src).cuda()
        d_dst = torch.full((h, w, out_ch), -7.0, device="cuda")
        assert _lib.load().mb200_transform_colorspace_layout_dev(d_src.data_ptr(), ch, d_dst.data_ptr(), out_ch, w, h,
                                                                 from_cs, to_cs, None, stream()) == code
        assert bool((d_dst == -7.0).all())


@gpu
def test_in_place_entry_points_still_decline_layout_spaces():
    lib = _lib.load()
    for from_cs, to_cs in [(lc.SRGB, lc.GRAY), (lc.GRAY, lc.SRGB), (lc.SRGB, lc.CMYK), (lc.LINEAR_GRAY, lc.LAB)]:
        src = make_image(7, 5, 4, seed=2)
        d = torch.from_numpy(src).cuda()
        assert lib.mb200_transform_colorspace_dev(d.data_ptr(), 7, 5, 4, from_cs, to_cs, stream()) == _lib.EUNSUPPORTED
        assert np.array_equal(d.cpu().numpy(), src)
        host = src.copy()
        assert lib.mb200_transform_colorspace(P(host), 7, 5, 4, from_cs, to_cs) == _lib.EUNSUPPORTED
        assert np.array_equal(host, src)


# ------------------------------------------------------------------------------------------------------ Python layer
@gpu
@pytest.mark.parametrize("device", [True, False])
def test_python_relayout_and_retag(device):
    src = make_image(17, 11, 4, seed=9)

    def image(pixels, cs):
        return im.Image(torch.from_numpy(pixels.copy()).cuda() if device else pixels.copy(), cs)

    def pixels(img):
        assert img.on_device == device
        return img.pixels.cpu().numpy() if device else img.pixels

    img = image(src, im.sRGBColorspace)
    assert im.TransformImageColorspace(img, im.GRAYColorspace) is True
    assert img.colorspace == im.GRAYColorspace and img.channels == 2
    assert np.array_equal(pixels(img), lc.orc_layout(src, lc.SRGB, lc.GRAY))
    gray = pixels(img).copy()
    im.TransformImageColorspace(img, im.CMYKColorspace)
    assert img.colorspace == im.CMYKColorspace and img.channels == 5
    assert np.array_equal(pixels(img), lc.orc_layout(gray, lc.GRAY, lc.CMYK))
    cmyk = pixels(img).copy()
    im.TransformImageColorspace(img, im.LabColorspace)
    assert img.colorspace == im.LabColorspace and img.channels == 4
    assert np.array_equal(pixels(img), in_place(lc.orc_layout(cmyk, lc.CMYK, lc.SRGB), lc.SRGB, lc.LAB))
    img = image(src[..., :3], im.RGBColorspace)
    im.TransformImageColorspace(img, im.LinearGRAYColorspace)
    assert img.colorspace == im.LinearGRAYColorspace and img.channels == 1
    with pytest.raises(im.MagickB200Error):
        im.TransformImageColorspace(image(src[..., :3], 22), im.GRAYColorspace)
