"""The stencil kernels (stencils.cu: Statistic, Rotational, Bilateral, Selective, Adaptive blur / sharpen; pointwise.cu:
MotionBlur) against the oracle, bit for bit with NaN where the oracle has NaN, through the device entry point (torch) and
the host entry point (NumPy).  The oracle is pinned to the reference on the same edge images by
test_oracle_stencil_edges_vs_ref.py.

Beyond the edge images: widths around the kernels' 128-thread x-blocks, 1 x 1 / 1 x N / N x 1 images and a 65535-row
image (the grid's y limit; 65536 rows are declined), windows larger than the image and at the 255 / 256 limit (motion
blur: 129 taps), one 2048 x 2048 RGBA image per operator, unaligned RGBA (refused), and a sentinel-filled destination
that every decline leaves untouched."""
import ctypes as C

import numpy as np
import pytest

import stencil_edge_cases as ec
from util import P, make_image, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")
torch = pytest.importorskip("torch")
EINVAL, EUNSUPPORTED = -1, -5                   # MB200_EINVAL, MB200_EUNSUPPORTED

FUNCTIONS = {"statistic": "StatisticImage", "rotational_blur": "RotationalBlurImage", "bilateral_blur": "BilateralBlurImage",
             "selective_blur": "SelectiveBlurImage", "adaptive_blur": "AdaptiveBlurImage",
             "adaptive_sharpen": "AdaptiveSharpenImage", "motion_blur": "MotionBlurImage"}
SENTINEL = np.float32(-12345.5)


def orc(op, src, args):
    h, w, ch = src.shape
    dst = np.full_like(src, SENTINEL)
    assert getattr(oracle(), "orc_" + op)(P(src), P(dst), w, h, ch, *args) == 0, (op, src.shape, args)
    return dst


def on_device(op, src, args):
    return getattr(im, FUNCTIONS[op])(im.Image(torch.from_numpy(src).cuda()), *args).pixels.cpu().numpy()


def on_host(op, src, args):
    return getattr(im, FUNCTIONS[op])(im.Image(src.copy()), *args).pixels


def same(got, want, what):
    """Bit-identical, except that any NaN matches any NaN."""
    assert got.shape == want.shape, what
    nan = np.isnan(want)
    g, w = np.where(nan, np.float32(0), got), np.where(nan, np.float32(0), want)
    bad = (np.isnan(got) != nan) | (g.view(np.int32) != w.view(np.int32))
    if bad.any():
        at = [tuple(int(i) for i in a) for a in np.argwhere(bad)[:6]]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} samples differ; (index, got, oracle): "
                    f"{[(a, float(got[a]), float(want[a])) for a in at]}")


def run(op, src, args, what, host=True):
    want = orc(op, src, args)
    same(on_device(op, src, args), want, f"{op} {args} {what} device")
    if host:
        same(on_host(op, src, args), want, f"{op} {args} {what} host")


# ---- the edge images of the reference suite
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("stat", range(1, 11))
def test_statistic_edges(stat, ch):
    for name, src, args in ec.cases("statistic", ch, stat):
        run("statistic", src, args, name)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("op", ec.OPERATORS[1:])
def test_operator_edges(op, ch):
    for name, src, args in ec.cases(op, ch):
        run(op, src, args, name)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("case", list(ec.NAMED))
def test_named_reproductions(case, ch):
    """The kernels restate the oracle's arithmetic, so they shared its defects: the adaptive edge map's range over rows
    that start with NaN, and the alpha channel's contrast in SelectiveBlur of gray + alpha and RGBA images."""
    op, build, args = ec.NAMED[case]
    run(op, build(ch), args, case)


# ---- geometry
ARGS = {"statistic": [(4, 3, 3), (3, 5, 2), (1, 1, 7)], "rotational_blur": [(10.0,), (-30.0,)],
        "bilateral_blur": [(5, 3, 20.0, 1.5)], "selective_blur": [(0.0, 1.0, 6553.5)], "adaptive_blur": [(0.0, 1.0)],
        "adaptive_sharpen": [(2.0, 1.5)], "motion_blur": [(5.0, 2.0, 30.0), (3.0, 1.0, 200.0)]}


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("op", ec.OPERATORS)
def test_x_block_edges(op, ch):
    """Widths 127, 128, 129 and 257 against the 128-thread x-blocks, and thin images."""
    for w, h in [(127, 3), (128, 2), (129, 3), (257, 2), (1, 1), (1, 40), (40, 1), (300, 1)]:
        src = ec.special_image(ch, w=w, h=h, every=5)
        for args in ARGS[op]:
            run(op, src, args, f"{w}x{h}")


@pytest.mark.parametrize("op", ec.OPERATORS)
def test_65535_rows_run_and_65536_are_declined(op):
    args = ARGS[op][0]
    src = ec.special_image(2, w=1, h=65535, every=11)
    run(op, src, args, "1x65535", host=False)
    declined(op, make_image(1, 65536, 2), args, EUNSUPPORTED)


def declined(op, src, args, code, src_offset=0, dst_offset=0):
    """The device and host entry points return `code` and leave a sentinel-filled destination untouched."""
    from imagemagick_b200 import _lib
    lib = _lib.load()
    h, w, ch = src.shape
    n = src.size
    d_src = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
    d_src[src_offset:src_offset + n] = torch.from_numpy(src.ravel()).cuda()
    d_dst = torch.full((n + 4,), float(SENTINEL), dtype=torch.float32, device="cuda")
    fn = getattr(lib, f"mb200_{op}_image_dev")
    rc = fn(C.c_void_p(d_src.data_ptr() + 4 * src_offset), C.c_void_p(d_dst.data_ptr() + 4 * dst_offset), w, h, ch, *args,
            None)
    torch.cuda.synchronize()
    assert rc == code, (op, args, rc)
    assert bool((d_dst == float(SENTINEL)).all()), (op, args, "device destination written")
    if src_offset or dst_offset:
        return
    dst = np.full_like(src, SENTINEL)
    rc = getattr(lib, f"mb200_{op}_image")(C.c_void_p(src.ctypes.data), C.c_void_p(dst.ctypes.data), w, h, ch, *args)
    assert rc == code, (op, args, rc, "host")
    assert np.all(dst == SENTINEL), (op, args, "host destination written")


# ---- windows
@pytest.mark.parametrize("ch", [1, 4])
def test_statistic_windows(ch):
    """Windows larger than the image, 1 x 1, even windows, and 255 (accepted) against 256 (declined).  Mode and Nonpeak
    walk the window once per distinct value, so their large windows run on a few-level image."""
    src = ec.special_image(ch, w=19, h=7, every=5)
    poster = ec.gray_posterised(ch)
    for stat in range(1, 11):
        for win in [(1, 1), (2, 2), (6, 4), (2, 8), (25, 9), (9, 25)]:
            run("statistic", src, (stat, *win), f"19x7 {win}")
        big = poster if stat in (6, 7) else src
        run("statistic", big, (stat, 255, 255), "255x255", host=False)
        run("statistic", big, (stat, 255, 1), "255x1", host=False)
        for win in [(256, 1), (1, 256), (256, 256)]:
            declined("statistic", big, (stat, *win), EUNSUPPORTED)
    declined("statistic", src, (11, 3, 3), EINVAL)
    declined("statistic", src, (0, 3, 3), EINVAL)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_bilateral_windows(ch):
    src = ec.special_image(ch, w=19, h=7, every=5)
    for args in [(1, 1, 10.0, 1.0), (1, 9, 20.0, 2.0), (25, 9, 20.0, 3.0), (255, 255, 20.0, 40.0), (255, 1, 5.0, 9.0)]:
        run("bilateral_blur", src, args, "19x7", host=args[0] < 255)
    for args in [(4, 4, 20.0, 1.5), (3, 2, 20.0, 1.5), (256, 1, 20.0, 1.5), (1, 257, 20.0, 1.5), (257, 257, 20.0, 1.5)]:
        declined("bilateral_blur", src, args, EUNSUPPORTED)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_selective_and_adaptive_windows(ch):
    """radius 127 gives a 255-wide window (accepted), 128 a 257-wide one (declined)."""
    src = ec.special_image(ch, w=19, h=7, every=5)
    for args in [(12.0, 3.0, 20000.0), (127.0, 30.0, 20000.0)]:
        run("selective_blur", src, args, "19x7", host=False)
    declined("selective_blur", src, (128.0, 30.0, 20000.0), EUNSUPPORTED)
    for op in ("adaptive_blur", "adaptive_sharpen"):
        for args in [(12.0, 3.0), (127.0, 30.0)]:
            run(op, src, args, "19x7", host=False)
        declined(op, src, (128.0, 30.0), EUNSUPPORTED)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_motion_blur_tap_limit(ch):
    src = ec.special_image(ch, w=40, h=30, every=5)
    for angle in (0.0, 37.0, -90.0):
        run("motion_blur", src, (64.0, 20.0, angle), "129 taps")
        declined("motion_blur", src, (65.0, 20.0, angle), EUNSUPPORTED)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_rotational_blur_angles(ch):
    """Angle 0 (n = 2 samples), negative angles, whole turns, and an odd square image whose diagonal pixels have
    blur_radius / radius = 1, 2, 3."""
    src = ec.special_image(ch, w=41, h=41, every=5)
    for angle in (0.0, -0.0, -15.0, 360.0, -360.0, 720.0, 1.0):
        run("rotational_blur", src, (angle,), "41x41")
    declined("rotational_blur", ec.special_image(ch), (-0.5,), EUNSUPPORTED)      # |4 rad sqrt(r) + 2| < 2: n = 1


# ---- large images
@pytest.mark.parametrize("op", ec.OPERATORS)
def test_2048_rgba(op):
    src = ec.special_image(4, w=2048, h=2048, seed=8, every=997)
    args = {"statistic": (4, 5, 5), "rotational_blur": (5.0,), "bilateral_blur": (5, 5, 20.0, 1.5),
            "selective_blur": (0.0, 1.0, 6553.5), "adaptive_blur": (0.0, 1.0), "adaptive_sharpen": (0.0, 1.0),
            "motion_blur": (10.0, 3.0, 30.0)}[op]
    run(op, src, args, "2048x2048")


# ---- errors
@pytest.mark.parametrize("op", ec.OPERATORS)
def test_unaligned_rgba_is_refused_untouched(op):
    src = ec.special_image(4, w=33, h=9)
    args = ARGS[op][0]
    declined(op, src, args, EINVAL, src_offset=1)
    declined(op, src, args, EINVAL, dst_offset=1)
