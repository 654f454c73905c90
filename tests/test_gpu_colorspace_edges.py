"""The in-place TransformImageColorspace kernels (colorspace.cu, hexcone.cu) against the oracle on the edge images of
colorspace_edge_cases -- signed zeros, denormals, HDRI samples up to FLT_MAX, +-inf, NaN and float sweeps across every
boundary the kernels decide on -- through the device entry point (torch) and the host entry point (NumPy); the oracle is
pinned to the reference on the same images by test_oracle_colorspace_edges_vs_ref.py.

Asserted for every leg: NaN exactly where the oracle has NaN, the same infinity with the same sign where it has one, alpha
bit-identical to the input, and every finite sample within the leg's documented bar (DESIGN.md section 4): 0 ULP for the
matrix / LUT, YCC, forward Log and hexcone legs (HSI 1 ULP), 1 ULP for Lab / XYZ / linear RGB, the inverse Log leg and
the XYZ family.  The Lab / XYZ and XYZ-family legs treat as rounding noise a component whose reference value is the
difference of two equal numbers: below 1e-6 Quantum units (util.ulp_or_noise), or -- for the components that are such
differences (cancelling()), at HDRI magnitudes where that noise grows with the operands -- within 2^-36 of the pixel's
largest component; the hue of LCH / LCHab / LCHuv is not compared where the chroma is such noise.  The inverse legs of
RESIDUE_INVERSE fed components far outside their forward range have only their non-finite samples compared.  Then the
shapes: pixel counts around colorspace_kernel's 1024-pixel CTA footprint and the one-pixel-per-thread kernels' 256-pixel
blocks, a ragged 2-D image, RGB buffers one float into their allocation and unaligned RGBA."""
import ctypes as C

import numpy as np
import pytest

import colorspace_edge_cases as ec
import util
from util import P, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")


def exact_bar(cs, forward):
    if cs in ec.MATRIX or cs == ec.YCC or (cs == ec.LOG and forward):
        return 0
    if cs in ec.HEXCONE:
        return 1 if cs == 7 else 0
    return None                       # <= 1 ULP with the rounding-noise rule


def orc(src, frm, to, values=None):
    h, w, ch = src.shape
    out = src.copy()
    opts = C.byref(util.ColorspaceOptions.of(**values)) if values else None
    assert oracle().orc_colorspace_ex(P(out), w, h, ch, frm, to, opts) == 0
    return out


def on_device(src, frm, to, settings=None):
    import torch
    img = im.Image(torch.from_numpy(src.copy()).cuda(), colorspace=frm)
    assert im.TransformImageColorspace(img, to, settings=settings) is True and img.colorspace == to
    return img.pixels.cpu().numpy()


def on_host(src, frm, to, settings=None):
    img = im.Image(src.copy(), colorspace=frm)
    assert im.TransformImageColorspace(img, to, settings=settings) is True and img.colorspace == to
    return img.pixels


def mismatches(got, want, src, frm, to):
    """Boolean mask of the samples (colour channels) where `got` misses the bar of the leg frm -> to."""
    g, w = got[..., :3].astype(np.float64), want[..., :3].astype(np.float64)
    bad = (np.isnan(g) != np.isnan(w)) | (np.isinf(g) != np.isinf(w))
    bad |= np.isinf(g) & np.isinf(w) & (np.signbit(g) != np.signbit(w))
    fin = np.isfinite(g) & np.isfinite(w)
    gf, wf = np.where(fin, got[..., :3], np.float32(0)), np.where(fin, want[..., :3], np.float32(0))
    forward = frm == ec.SRGB
    cs = to if forward else frm
    if not forward and cs in RESIDUE_INVERSE:
        lo, hi = RESIDUE_INVERSE[cs]
        fin &= np.all((src[..., :3] >= lo) & (src[..., :3] <= hi), axis=-1, keepdims=True)
    bar = exact_bar(cs, forward)
    if bar is not None and cs != 7:
        return bad | (fin & (util.ulp_distance(gf, wf) > bar))
    plain = cs in (ec.RGB, ec.LOG, 7)               # independent channels / no cancellation: ULPs only
    d = util.ulp_distance(gf, wf) if plain else util.ulp_or_noise(gf, wf)
    # a component that is the difference of huge operands carries their rounding residue, which scales with them:
    # 2^-36 of the pixel's largest component (~70 000 double ULPs of it, DESIGN.md section 4)
    scale = np.max(np.abs(np.where(fin, w, 0.0)), axis=-1, keepdims=True)
    with np.errstate(invalid="ignore"):          # inf - inf where both are inf: compared above
        noise = (np.abs(g - w) <= scale * 2.0 ** -36) & cancelling(cs, forward, src)
    d = np.where(noise, 0, d)
    if forward and cs in ec.POLAR:                 # hue of an achromatic pixel: atan2 of two residues
        chroma_noise = np.abs(w[..., 1] - 32767.5) <= np.maximum(1e-4, scale[..., 0] * 2.0 ** -36)
        d[..., 2] = np.where(chroma_noise, 0, d[..., 2])
    return bad | (fin & (d > (bar or 1)))


# Inverse legs (space -> sRGB) whose result on components far outside what their forward leg produces (hue 1e16, chroma
# 1e13, samples that decode to 1e12 ...) is the residue of cancelling huge intermediates that went through the CUDA math
# library or a contracted matrix product: LCH / LCHab / LCHuv and Oklch take cos / sin of the hue, Jzazbz raises to the
# powers 1/0.159 and 1/134, DisplayP3 / Adobe98 and Oklab multiply decoded samples / cubes by a matrix whose FMAs the
# compiler contracts ahead of xyz_to_rgb's.  Only their non-finite samples are compared outside the range given here
# (Jzazbz: the range its forward leg gives in-range sRGB).  Every other inverse leg keeps its bar on every finite sample.
RESIDUE_INVERSE = {12: (-2 * ec.QR, 2 * ec.QR), 13: (-2 * ec.QR, 2 * ec.QR), 14: (-2 * ec.QR, 2 * ec.QR),
                   39: (-2 * ec.QR, 2 * ec.QR), 34: (0.0, ec.QR), 35: (-2 * ec.QR, 2 * ec.QR),
                   36: (-2 * ec.QR, 2 * ec.QR), 38: (-2 * ec.QR, 2 * ec.QR)}
# forward output channels that are differences of like terms: Lab / Luv / Jzazbz / Oklab a, b, the LCH / Oklch chroma,
# the RGB primaries and LMS rows of mixed sign
_CANCELLING_FORWARD = {ec.LAB: (1, 2), 12: (1,), 13: (1,), 14: (1,), 17: (1, 2), 34: (1, 2), 38: (1, 2), 39: (1,),
                       35: (0, 1, 2), 36: (0, 1, 2), 37: (0, 1, 2), 16: (0, 1, 2), 40: (0, 1, 2)}


def cancelling(cs, forward, src):
    """Mask (broadcast to the colour channels) of the output components that are a difference of like terms."""
    mask = np.zeros(src.shape[:2] + (3,), bool)
    if forward:
        mask[..., list(_CANCELLING_FORWARD.get(cs, ()))] = True
    elif cs == 7:
        # HSI: the channel the sector leaves to 3 I - lead - low (hexcone.cuh from_hsi)
        h = 360.0 * (src[..., 0].astype(np.float64) / ec.QR)
        with np.errstate(invalid="ignore"):
            h = h - 360.0 * np.floor(h / 360.0)
            third = np.where(h < 120.0, 0, np.where(h < 240.0, 1, 2))
        rest = np.choose(third, [1, 2, 0])
        for c in range(3):
            mask[..., c] = rest == c
    elif cs not in (ec.RGB, ec.LOG):
        mask[:] = True                            # the outputs of xyz_to_rgb / Oklab's matrix: rows of mixed sign
    return mask


def check(got, want, src, frm, to, what):
    assert got.shape == want.shape
    if src.shape[2] == 4:
        assert np.array_equal(got[..., 3].view(np.int32), src[..., 3].view(np.int32)), (what, "alpha changed")
    bad = mismatches(got, want, src, frm, to)
    if bad.any():
        at = np.argwhere(bad.any(axis=-1))[:6]
        rows = [(tuple(int(i) for i in a), src[tuple(a)][:3].tolist(), got[tuple(a)][:3].tolist(), want[tuple(a)][:3].tolist())
                for a in at]
        g, w = got[..., :3].astype(np.float64), want[..., :3].astype(np.float64)
        fin = np.isfinite(g) & np.isfinite(w)
        scale = np.max(np.abs(np.where(fin, w, 0.0)), axis=-1, keepdims=True)
        rel = np.where(bad & fin, np.abs(g - w) / np.maximum(scale, 1e-300), 0.0)
        pytest.fail(f"{what} {frm}->{to}: {int(bad.sum())} samples off ({int((bad & ~fin).sum())} non-finite, worst "
                    f"|got - oracle| / pixel scale {rel.max():.3g}); (pixel, input, got, oracle): {rows}")


def run_leg(src, frm, to, what, settings=None, values=None):
    want = orc(src, frm, to, values)
    check(on_device(src, frm, to, settings), want, src, frm, to, f"{what} device")
    check(on_host(src, frm, to, settings), want, src, frm, to, f"{what} host")
    return want


@pytest.mark.parametrize("cs", ec.SPACES)
def test_edge_legs(cs):
    for ch in (3, 4):
        fwd = run_leg(ec.edge_image(ch), ec.SRGB, cs, f"{ch}ch forward")
        run_leg(ec.inverse_source(fwd, ch), cs, ec.SRGB, f"{ch}ch inverse")


SETTINGS = [(ec.LAB, {"color:illuminant": "D50"}, dict(illuminant="D50")),
            (34, {"white-luminance": "203"}, dict(white_luminance=203.0))]


@pytest.mark.parametrize("case", range(len(SETTINGS)), ids=["Lab-D50", "Jzazbz-203"])
def test_edge_legs_with_settings(case):
    cs, settings, values = SETTINGS[case]
    for ch in (3, 4):
        fwd = run_leg(ec.edge_image(ch), ec.SRGB, cs, f"{ch}ch forward", settings, values)
        run_leg(ec.inverse_source(fwd, ch), cs, ec.SRGB, f"{ch}ch inverse", settings, values)


# ---- named minimal cases: one pixel set per defect the edge images can expose
INF, NAN = np.float32(np.inf), np.float32(np.nan)


def _pixels(rows, ch):
    a = np.array(rows, np.float32)
    if ch == 4:
        a = np.concatenate([a, np.full((len(a), 1), 30000.0, np.float32)], axis=1)
    return np.ascontiguousarray(a[None])


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("cs", [ec.LAB, ec.XYZ, ec.RGB, 17, 36, 34, 38, ec.LOG])
def test_plus_inf_sample_decodes_to_nan(cs, ch):
    """A +inf sRGB sample takes the decode curve's out-of-line path (beyond the tabled exponents); the reference's frexp /
    Chebyshev chain makes it NaN, and so must every kernel that decodes it (Lab, XYZ, linear RGB, the XYZ family via
    rgb_to_xyz and Oklab, Log)."""
    run_leg(_pixels([[INF, 1000, 1000], [1000, INF, 1000], [1000, 1000, INF], [INF, INF, INF], [NAN, 1000, 1000]], ch),
            ec.SRGB, cs, "+inf decode")


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("cs", [ec.RGB, ec.XYZ, ec.LAB, 17, 25, 36, 38, 16])
def test_plus_inf_and_nan_encode_to_nan(cs, ch):
    """Infinite and NaN arguments of EncodePixelGamma on the way back to sRGB (linear RGB, XYZ, Lab, Luv, xyY, Adobe98,
    Oklab, LMS): the reference's chain gives NaN, not a huge finite value that rounds to +inf."""
    run_leg(_pixels([[INF, 1000, 1000], [1000, INF, 1000], [1000, 1000, INF], [INF, INF, INF], [NAN, 1000, 1000],
                     [1000, NAN, 1000]], ch), cs, ec.SRGB, "+inf encode")


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("cs", [ec.LAB, 13, 17])
def test_lab_cube_root_above_float_range(cs, ch):
    """Tristimulus ratios at and above FLT_MAX (sRGB samples from ~7e20 up): the cube root's single-precision seed would
    overflow; the reference's pow(t, 1/3) is finite there."""
    v = [7.1e20, 1e21, 1e25, 6.4e23, 1e30, 3.0e38]
    run_leg(_pixels([[x, x, x] for x in v] + [[x, 0, 0] for x in v] + [[0, x, 1000] for x in v], ch), ec.SRGB, cs,
            "cube root")


# ---- shapes
SIZES = [1, 3, 255, 256, 257, 1023, 1024, 1025, 4095, 4097]
SHAPE_LEGS = [(ec.SRGB, ec.LAB), (ec.SRGB, ec.XYZ), (ec.SRGB, ec.RGB), (ec.LAB, ec.SRGB), (ec.XYZ, ec.SRGB),
              (ec.RGB, ec.SRGB), (ec.SRGB, 17), (ec.SRGB, 30), (ec.SRGB, ec.LOG), (ec.SRGB, ec.YCC), (ec.SRGB, 8)]


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("leg", SHAPE_LEGS, ids=lambda p: f"{p[0]}-{p[1]}")
def test_pixel_counts(leg, ch):
    """colorspace_kernel's four-pixels-per-thread loop tail and prefetch guard (1024 pixels per CTA) and the last block
    of the one-pixel-per-thread kernels, on the edge pixels."""
    frm, to = leg
    edge = ec.edge_image(ch)
    for n in SIZES:
        run_leg(ec.pixels_of(edge, n), frm, to, f"{n} px")
    run_leg(np.ascontiguousarray(np.resize(edge, (29, 37, ch))), frm, to, "29x37")


@pytest.mark.parametrize("leg", SHAPE_LEGS, ids=lambda p: f"{p[0]}-{p[1]}")
def test_rgb_one_float_into_the_allocation(leg):
    """RGB buffers need no alignment: a buffer that starts 4 bytes into its allocation, with sentinels after it."""
    import torch
    frm, to = leg
    sentinel = np.float32(-12345.5)
    for n in (257, 1025):
        src = ec.pixels_of(ec.edge_image(3), n)
        want = orc(src, frm, to)
        store = torch.full((3 * n + 9,), float(sentinel), dtype=torch.float32, device="cuda")
        store[1:1 + 3 * n] = torch.from_numpy(src.ravel()).cuda()
        view = store[1:1 + 3 * n].view(1, n, 3)
        img = im.Image(view, colorspace=frm)
        assert img.pixels.data_ptr() % 16 == 4
        im.TransformImageColorspace(img, to)
        host = store.cpu().numpy()
        check(host[1:1 + 3 * n].reshape(1, n, 3), want, src, frm, to, f"offset {n} px")
        assert host[0] == sentinel and np.all(host[1 + 3 * n:] == sentinel)


@pytest.mark.parametrize("leg", [(ec.SRGB, ec.LAB), (ec.LAB, ec.SRGB), (ec.SRGB, 17), (ec.SRGB, 30)],
                         ids=lambda p: f"{p[0]}-{p[1]}")
def test_unaligned_rgba_is_refused_untouched(leg):
    import torch
    from imagemagick_b200 import _lib
    frm, to = leg
    n = 300
    src = ec.pixels_of(ec.edge_image(4), n)
    store = torch.zeros(4 * n + 4, dtype=torch.float32, device="cuda")
    store[1:1 + 4 * n] = torch.from_numpy(src.ravel()).cuda()
    before = store.cpu().numpy()
    rc = _lib.load().mb200_transform_colorspace_ex_dev(C.c_void_p(store.data_ptr() + 4), n, 1, 4, frm, to, None, None)
    torch.cuda.synchronize()
    assert rc == _lib.EINVAL
    assert np.array_equal(store.cpu().numpy().view(np.int32), before.view(np.int32))
