"""The oracle against the real reference, bit for bit, for the in-place enhance operators: ContrastImage,
ModulateImage (every "modulate:colorspace" plus a space it does not know, and none; reference whites), GrayscaleImage
(all ten PixelIntensityMethods on sRGB, linear RGB and GRAY images, with the re-laid-out GRAY cache) and FunctionImage
(every function with 0-5 parameters, under `-channel` selections).  Inputs mix noise, alpha blocks, HDR values, gray
pixels (black and white among them) and NaN / +-inf samples (enhance_cases.mosaic).

The reference's results are stored as digests in tests/golden/enhance_digests.json (enhance_cases.reference); re-record
them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_enhance_vs_ref.py

where oracle/_ref is built."""
import ctypes as C

import pytest

import enhance_cases as ec
from enhance_cases import reference
from util import P, digest, make_image

CHANNELS = [1, 2, 3, 4]
SIZES = [(37, 23), (1, 17), (19, 1)]


def ref_contrast(src, sharpen, times=1):
    h, w, ch = src.shape
    out = src.copy()
    for _ in range(times):
        assert ec.ref().ref_contrast(P(out), w, h, ch, -1, int(sharpen)) == 0
    return out


def ref_modulate(src, geometry, space=None, illuminant=None, colorspace=-1):
    h, w, ch = src.shape
    out = src.copy()
    assert ec.ref().ref_modulate(P(out), w, h, ch, colorspace, geometry.encode(), ec.artifacts(space, illuminant)) == 0
    return out


def ref_grayscale(src, method, colorspace):
    h, w, ch = src.shape
    buf = src.copy()
    out_ch = ec.ref().ref_grayscale(P(buf), w, h, ch, colorspace if ch >= 3 else -1, method)
    assert out_ch == (2 if ch in (2, 4) else 1)
    return buf.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy()


def ref_function(src, function, params, mask):
    h, w, ch = src.shape
    out = src.copy()
    arr = (C.c_double * max(1, len(params)))(*params)
    assert ec.ref().ref_function(P(out), w, h, ch, function, len(params), arr, mask) == 0
    return out


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("sharpen", [True, False])
def test_contrast(ch, sharpen):
    src = ec.mosaic(37, ch)
    assert digest(ec.orc_contrast(src, sharpen)) == reference("mosaic", lambda: ref_contrast(src, sharpen))
    for w, h in SIZES:
        img = make_image(w, h, ch, seed=w + h)
        assert digest(ec.orc_contrast(img, sharpen)) == reference(f"{w}x{h}", lambda: ref_contrast(img, sharpen))


@pytest.mark.parametrize("ch", [3, 4])
def test_contrast_three_times(ch):
    src = ec.mosaic(29, ch, seed=5)
    out = src
    for _ in range(3):
        out = ec.orc_contrast(out, True)
    assert digest(out) == reference("sharpen x3", lambda: ref_contrast(src, True, times=3))


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("space", list(ec.MODULATE_SPACES), ids=str)
def test_modulate(space, ch):
    src = ec.mosaic(31, ch, seed=21)
    for geometry in ec.GEOMETRIES:
        got = ec.orc_modulate(src, geometry, space)
        assert digest(got) == reference(geometry, lambda: ref_modulate(src, geometry, space)), geometry


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("illuminant", ["D50", "A", "bogus"])
@pytest.mark.parametrize("space", ["LCHab", "LCHuv", "HSB"])
def test_modulate_illuminant(space, illuminant, ch):
    src = ec.mosaic(23, ch, seed=31)
    got = ec.orc_modulate(src, "90,140,130", space, illuminant)
    assert digest(got) == reference("90,140,130", lambda: ref_modulate(src, "90,140,130", space, illuminant))


@pytest.mark.parametrize("space", ["HCL", "HWB", "LCHuv"])
def test_modulate_geometry_forms(space):
    """A single number (brightness only), 'x' as the first separator (ParseGeometry's rho x sigma), and an image tagged
    with a colourspace that is not sRGB-compatible (re-tagged sRGB, pixels untouched)."""
    src = ec.mosaic(17, 4, seed=41)
    for geometry in ["130", "70,160", "90x110", "90x110,170"]:
        got = ec.orc_modulate(src, geometry, space)
        assert digest(got) == reference(geometry, lambda: ref_modulate(src, geometry, space)), geometry
    got = ec.orc_modulate(src, "90,110,170", space)
    assert digest(got) == reference("from Lab", lambda: ref_modulate(src, "90,110,170", space, colorspace=ec.LAB))


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("space", ["HCL", "HSI", "LCHab"])
def test_modulate_sizes(space, ch):
    for w, h in SIZES:
        img = make_image(w, h, ch, seed=3 * w + h, kind="hdr")
        got = ec.orc_modulate(img, "120,70,40", space)
        assert digest(got) == reference(f"{w}x{h}", lambda: ref_modulate(img, "120,70,40", space))


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("method", range(10))
def test_grayscale(method, ch):
    src = ec.mosaic(33, ch, seed=51)
    for colorspace in ([ec.SRGB, ec.RGB] if ch >= 3 else [ec.GRAY]):
        got = ec.orc_grayscale(src, method, colorspace)
        assert got.shape[2] == (2 if ch in (2, 4) else 1)
        assert digest(got) == reference(f"cs{colorspace}", lambda: ref_grayscale(src, method, colorspace)), colorspace
    img, cs = make_image(1, 13, ch, seed=method), (ec.SRGB if ch >= 3 else ec.GRAY)
    assert digest(ec.orc_grayscale(img, method, cs)) == reference("1x13", lambda: ref_grayscale(img, method, cs))


def _function_id(case):
    return f"{['undefined', 'arcsin', 'arctan', 'polynomial', 'sinusoid'][case[0]]}{len(case[1])}-" + \
        "_".join(f"{p:g}" for p in case[1][:4])


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("case", ec.FUNCTION_CASES + [ec.POLYNOMIAL_33], ids=_function_id)
def test_function(case, ch):
    function, params = case
    src = ec.mosaic(27, ch, seed=61)
    got = ec.orc_function(src, function, params, -1)
    assert digest(got) == reference("all", lambda: ref_function(src, function, params, -1))


@pytest.mark.parametrize("ch", CHANNELS)
@pytest.mark.parametrize("mask", ["R", "RGB", "alpha"])
def test_function_channels(mask, ch):
    src = ec.mosaic(21, ch, seed=71)
    for function, params in [(ec.POLYNOMIAL, [1.5, -0.25, 0.125]), (ec.SINUSOID, [2.0, 30.0]), (ec.ARCTAN, [])]:
        m = ec.CHANNEL_MASKS[mask]
        got = ec.orc_function(src, function, params, m)
        assert digest(got) == reference(f"f{function}", lambda: ref_function(src, function, params, m)), function


@pytest.mark.parametrize("ch", CHANNELS)
def test_function_sizes(ch):
    for w, h in SIZES:
        img = make_image(w, h, ch, seed=w * h, kind="hdr")
        got = ec.orc_function(img, ec.ARCSIN, [0.6, 0.4], -1)
        assert digest(got) == reference(f"{w}x{h}", lambda: ref_function(img, ec.ARCSIN, [0.6, 0.4], -1))
