"""The separable passes beyond the blur defaults: 1-D user kernels (asymmetric, off-centre, mixed-sign and zero-sum taps,
Convolve and Correlate), every kernel family the dispatcher can choose for a 1-D convolution or a resize axis, and
every developer knob of DESIGN §10 (set at run time with mb200_set_option).

Every case reads the per-family launch counters, so a case cannot pass on a fallback kernel.  Bars: <= 1 ULP against
the oracle (non-finite results identical); kernels of one family that only restage data give identical bits."""
import numpy as np
import pytest

import util
from util import P, make_image, max_ulp, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")

CONV_FAMILIES = ("conv_mma_launches", "conv_pair_launches", "conv_pair_async_launches", "conv_generic_launches")
RESIZE_FAMILIES = ("resize_v_stream_launches", "resize_h_tma_launches", "resize_h_stream_launches",
                   "resize_regular_launches", "resize_gather_launches")


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


def orc_resize(src, ow, oh, filt):
    h, w, ch = src.shape
    dst = np.empty((oh, ow, ch), np.float32)
    assert oracle().orc_resize(P(src), w, h, ch, P(dst), ow, oh, filt) == 0
    return dst


def counted(fn, families):
    """Runs fn(); returns its result and how many launches of each family it made."""
    c0 = {f: util.get_option(f) for f in families}
    out = fn()
    return out, {f: util.get_option(f) - c0[f] for f in families}


def set_options(**options):
    for name, value in options.items():
        util.set_option(name, value)


def assert_matches(got, want, what, taps_abs_sum=None):
    """<= 1 ULP where the oracle is finite; NaN and inf exactly where the oracle has them.

    taps_abs_sum (1-D kernels on images with alpha): colour values whose alpha-weighted tap sum -- the oracle's alpha
    result -- cancels to below 1e-6 of its scale are excluded from the ULP bar.  There the colour sum cancels as well
    (all taps of a zero-sum kernel read one clamped pixel), PerceptibleReciprocal multiplies its rounding residue by up
    to 1e12, and the value depends on the order of summation and on FMA contraction: it carries no significant bits."""
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    inf = np.isinf(want)
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], want[inf]), what
    ok = np.isfinite(want)
    ch = want.shape[2]
    if taps_abs_sum is not None and ch in (2, 4):
        cancelled = np.abs(want[..., ch - 1].astype(np.float64)) <= 1e-6 * 65535.0 * taps_abs_sum
        ok = ok & ~(cancelled[..., None] & (np.arange(ch) < ch - 1))
    d = util.ulp_distance(np.where(ok, got, np.float32(0)), np.where(ok, want, np.float32(0)))
    assert d.max() <= 1, (what, int(d.max()))


# ---- 1. 1-D user kernels against the oracle ---------------------------------------------------------------------------
LENGTHS = [1, 2, 8, 9, 10, 16, 17, 18, 25, 26, 32, 33, 34, 49, 50, 65, 66]
TAPS = ["asymmetric", "mixed", "zero_sum", "negative"]
KINDS = ["noise", "alpha_blocks", "hdr"]
# narrow, short, 1-wide and 1-tall images (shorter than most windows); no size is a multiple of 8 or 32
SIZES = [(37, 29), (5, 43), (43, 3), (1, 19), (19, 1), (61, 35), (13, 13)]
# RGBA passes: the matrix kernels, the DFMA pair kernels, the generic kernels
RGBA_MODES = {"mma": dict(conv_mma=1), "pair": dict(conv_mma=0, pair=1), "generic": dict(conv_mma=0, pair=0)}


def taps(n, kind):
    """Taps that are exact binary fractions (the window sums do not depend on the order of summation beyond the
    rounding every kernel shares)."""
    i = np.arange(n)
    if kind == "asymmetric":
        return (1.0 + (3 * i) % 7) / 8.0
    if kind == "mixed":
        v = ((5 * i) % 9 - 4) / 4.0
        v[0] = 1.25                      # never all zero, never symmetric
        return v
    if kind == "zero_sum":
        v = ((7 * i) % 11 - 5) / 4.0
        if n > 1:
            v[-1] = -v[:-1].sum()
        else:
            v[0] = 0.0
        return v
    return -(1.0 + i % 3) / 4.0          # negative


def origins(n):
    c = n // 2
    out = {0, n - 1, c}
    if n % 2 == 0:
        out |= {c - 1, c + 1} - {n}
    return sorted(o for o in out if 0 <= o < n)


def kernel_string(values, axis, origin):
    """axis 0: a row kernel (Nx1, the row pass); axis 1: a column kernel (1xN, the column pass)."""
    n = len(values)
    body = ",".join("nan" if np.isnan(v) else repr(float(v)) for v in values)
    return f"{n}x1+{origin}+0: {body}" if axis == 0 else f"1x{n}+0+{origin}: {body}"


def oracle_kernel(values, axis, origin):
    v = np.asarray(values, np.float64)
    return util.orc_kernel_from_array(v.reshape(1, -1) if axis == 0 else v.reshape(-1, 1),
                                      origin if axis == 0 else 0, 0 if axis == 0 else origin)


def expected_conv_family(n, ch, mode, nan=False, bias=0.0):
    """The family that must serve a 1-D convolution pass (None: the dense 2-D kernel, which has no counter)."""
    if nan or n > 65:
        return None
    if ch == 4 and bias == 0.0 and n <= 33 and mode in ("mma", "pair"):
        return "conv_mma_launches" if mode == "mma" else "pair"
    return "conv_generic_launches"


def assert_conv_counts(counts, expected, passes=1):
    if expected == "pair":
        assert counts["conv_pair_launches"] + counts["conv_pair_async_launches"] == passes, counts
        assert counts["conv_mma_launches"] == 0 and counts["conv_generic_launches"] == 0, counts
    else:
        for f in CONV_FAMILIES:
            assert counts[f] == (passes if f == expected else 0), (expected, counts)


def run_1d(src, method, ks, mode, bias=0.0):
    if src.shape[2] == 4:
        set_options(**RGBA_MODES[mode])
    return counted(lambda: _host(im.MorphologyImage(_dev(src), method, 1, ks, bias=bias)), CONV_FAMILIES)


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("n", LENGTHS)
def test_1d_user_kernels_against_the_oracle(n, axis):
    """Asymmetric windows with the origin at both ends and around the centre: Convolve reflects the taps and the origin
    (morphology.c:2612-2626), Correlate rotates the kernel first (:3779-3793).  A wrong origin, a missing reflection or a
    shifted source block changes every output."""
    case = 0
    for oi, origin in enumerate(origins(n)):
        for ti, tk in enumerate(TAPS):
            values = taps(n, tk)
            ks = kernel_string(values, axis, origin)
            k = oracle_kernel(values, axis, origin)
            for method in (im.ConvolveMorphology, im.CorrelateMorphology):
                ch = 1 + (oi + ti + method) % 4
                w, h = SIZES[case % len(SIZES)]
                kind = KINDS[case % len(KINDS)]
                case += 1
                src = make_image(w, h, ch, seed=1000 * n + case, kind=kind)
                want = util.orc_morphology(src, method, 1, [k])
                for mode in (RGBA_MODES if ch == 4 else ("default",)):
                    got, counts = run_1d(src, method, ks, mode)
                    assert_conv_counts(counts, expected_conv_family(n, ch, mode))
                    assert_matches(got, want, (ks, method, ch, kind, (w, h), mode), np.abs(values).sum())


@pytest.mark.parametrize("name", ["comet:0x2", "comet:0x3+90", "comet:0x1.5", "comet:0x2.5+90"])
def test_comet_kernels(name):
    """The built-in comet kernel: one-sided, origin at the head."""
    (values, x, y), = im.AcquireKernelInfo(name).arrays()
    assert 1 in values.shape and len(set(values.ravel())) > 1
    k = util.orc_kernel_from_array(values, x, y)
    n = values.size
    for ch in (1, 2, 3, 4):
        for kind in KINDS:
            src = make_image(47, 31, ch, seed=ch * 7 + len(kind), kind=kind)
            for method in (im.ConvolveMorphology, im.CorrelateMorphology):
                want = util.orc_morphology(src, method, 1, [k])
                for mode in (RGBA_MODES if ch == 4 else ("default",)):
                    got, counts = run_1d(src, method, name, mode)
                    assert_conv_counts(counts, expected_conv_family(n, ch, mode))
                    assert_matches(got, want, (name, ch, kind, method, mode))


@pytest.mark.parametrize("n", [5, 9, 17, 26, 33, 50])
def test_1d_kernels_with_bias_take_the_generic_kernels(n):
    for axis in (0, 1):
        values = taps(n, "mixed")
        origin = n - 1
        ks, k = kernel_string(values, axis, origin), oracle_kernel(values, axis, origin)
        for ch in (1, 2, 3, 4):
            src = make_image(41, 27, ch, seed=n + ch, kind="alpha_blocks")
            want = util.orc_morphology(src, im.ConvolveMorphology, 1, [k], bias=100.0)
            for mode in (("mma", "pair") if ch == 4 else ("default",)):
                got, counts = run_1d(src, im.ConvolveMorphology, ks, mode, bias=100.0)
                assert_conv_counts(counts, expected_conv_family(n, ch, mode, bias=100.0))
                assert_matches(got, want, (ks, ch, mode))


@pytest.mark.parametrize("n", [2, 5, 10, 33])
def test_1d_kernels_with_nan_cells(n):
    """A NaN cell drops out of the sum; the reference's column path (width-1 kernels) then scales gamma by
    height / count (morphology.c:2654-2807): the product sends both shapes to the dense kernel with that scale."""
    for axis in (0, 1):
        values = taps(n, "asymmetric")
        values[(2 * n) // 3] = np.nan
        origin = n // 3
        ks, k = kernel_string(values, axis, origin), oracle_kernel(values, axis, origin)
        for ch in (1, 2, 3, 4):
            for kind in KINDS:
                src = make_image(39, 23, ch, seed=n * 3 + ch, kind=kind)
                for method in (im.ConvolveMorphology, im.CorrelateMorphology):
                    want = util.orc_morphology(src, method, 1, [k])
                    got, counts = run_1d(src, method, ks, "mma" if ch == 4 else "default")
                    assert_conv_counts(counts, expected_conv_family(n, ch, "mma", nan=True))
                    assert_matches(got, want, (ks, ch, kind, method))


@pytest.mark.parametrize("n", [9, 10, 17, 26, 33])
def test_1d_non_finite_samples_near_off_centre_windows(n):
    """inf / NaN pixels poison exactly the outputs whose (off-centre) window holds them, on every RGBA kernel family."""
    src = make_image(150, 110, 4, seed=21 + n)
    src[30, 40, 0] = np.inf
    src[31, 90, 3] = -np.inf
    src[80, 20, 1] = np.nan
    src[100, 140, 0] = np.inf
    src[0, 0, 2] = np.inf
    src[109, 149, 3] = np.nan
    for axis in (0, 1):
        for origin in (0, n - 1, n // 3):
            values = taps(n, "asymmetric")
            ks, k = kernel_string(values, axis, origin), oracle_kernel(values, axis, origin)
            want = util.orc_morphology(src, im.ConvolveMorphology, 1, [k])
            assert np.isfinite(want).mean() > 0.5
            for mode in RGBA_MODES:
                got, counts = run_1d(src, im.ConvolveMorphology, ks, mode)
                assert_conv_counts(counts, expected_conv_family(n, 4, mode))
                assert_matches(got, want, (ks, mode))


# ---- 2. convolution variants: matrix knobs, DFMA pair kernels, generic kernels ---------------------------------------
# (radius, sigma) -> 13 (padded), 17 (exact), 27 (padded), 33 (exact) taps
WINDOWS = [(6.0, 2.0), (8.0, 2.5), (13.0, 3.5), (16.0, 4.0)]
UNSHARP = (1.5, 0.02)
OPS = ["blur", "unsharp", "gaussian"]


def nt_of(ntaps):
    return min(t for t in (9, 17, 25, 33) if t >= ntaps)


def run_op(op, src, radius, sigma):
    d = _dev(src)
    if op == "blur":
        return _host(im.BlurImage(d, radius, sigma))
    if op == "unsharp":
        return _host(im.UnsharpMaskImage(d, radius, sigma, *UNSHARP))
    return _host(im.GaussianBlurImage(d, radius, sigma))


def oracle_op(op, src, radius, sigma):
    if op == "blur":
        return orc("orc_blur", src, radius, sigma)
    if op == "unsharp":
        return orc("orc_unsharp", src, radius, sigma, *UNSHARP)
    return orc("orc_gaussian_blur", src, radius, sigma)


def assert_exact_enough(got, want, what):
    d = util.ulp_distance(got, want)
    assert d.max() <= 1 and (d == 0).mean() >= 0.9999, (what, int(d.max()), float((d == 0).mean()))


def assert_passthrough(op, src, got, radius, sigma):
    """UnsharpMask keeps the source value where |2 (src - blur)| < threshold (effect.c:4358-4364): 0 ULP there."""
    if op != "unsharp":
        return
    blur = orc("orc_blur", src, radius, sigma)
    passthrough = np.abs(2.0 * (src.astype(np.float64) - blur.astype(np.float64))) < 65535.0 * UNSHARP[1]
    assert passthrough.any() and np.array_equal(got[passthrough], src[passthrough])


@pytest.fixture(scope="module")
def big_rgba():
    return make_image(259, 257, 4, seed=77, kind="alpha_blocks")


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("op", OPS)
def test_mma_tuning_variants_give_identical_bits(op, window, big_rgba):
    radius, sigma = window
    want = oracle_op(op, big_rgba, radius, sigma)
    first = None
    util.set_option("conv_mma", 1)
    for minb in (3, 4):
        for strip in (8, 64, 512):
            for l2pf in (0, 1):
                set_options(mma_minb=minb, mma_strip=strip, mma_l2pf=l2pf)
                got, counts = counted(lambda: run_op(op, big_rgba, radius, sigma), CONV_FAMILIES)
                assert_conv_counts(counts, "conv_mma_launches", passes=2)
                if first is None:
                    first = got
                    assert_exact_enough(got, want, (op, window))
                    assert_passthrough(op, big_rgba, got, radius, sigma)
                else:
                    assert np.array_equal(got, first), (op, window, minb, strip, l2pf, max_ulp(got, first))


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("op", OPS)
def test_dfma_pair_variants_give_identical_bits(op, window, big_rgba):
    """The pair kernels' register ring against their cp.async ring, and the rotations per strip, at padded and exact
    windows; the fused UnsharpMask epilogue against the separate point pass; the DFMA result against the matrix one."""
    radius, sigma = window
    ntaps = 2 * int(radius) + 1
    want = oracle_op(op, big_rgba, radius, sigma)
    util.set_option("conv_mma", 1)
    mma = run_op(op, big_rgba, radius, sigma)
    util.set_option("conv_mma", 0)
    first = None
    for pa in (0, 1):
        for pac in (0, 1):
            for rot in (1, 3, 16):
                set_options(pair_async=pa, pair_async_col=pac, col_rot=rot, row_pair_rot=rot)
                got, counts = counted(lambda: run_op(op, big_rgba, radius, sigma), CONV_FAMILIES)
                # row pass: the cp.async ring when pair_async; column pass: also needs pair_async_col, and the
                # rank-1 column pass (double sums in) always uses the register ring
                n_async = pa + (pa * pac if op != "gaussian" else 0)
                assert counts["conv_pair_async_launches"] == n_async, (op, pa, pac, counts)
                assert counts["conv_pair_launches"] == 2 - n_async, (op, pa, pac, counts)
                assert counts["conv_mma_launches"] == 0 and counts["conv_generic_launches"] == 0
                if first is None:
                    first = got
                    assert_exact_enough(got, want, (op, window))
                    assert max_ulp(got, mma) <= 1, (op, window)
                    assert_passthrough(op, big_rgba, got, radius, sigma)
                else:
                    assert np.array_equal(got, first), (op, window, pa, pac, rot, max_ulp(got, first))
    assert nt_of(ntaps) in (17, 25, 33)
    if op == "unsharp":
        util.set_option("no_fused_unsharp", 1)
        for pa in (0, 1):
            util.set_option("pair_async", pa)
            unfused, counts = counted(lambda: run_op(op, big_rgba, radius, sigma), CONV_FAMILIES)
            assert counts["conv_pair_launches"] + counts["conv_pair_async_launches"] == 2
            assert np.array_equal(unfused, first), (window, pa)


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("op", ["blur", "unsharp"])
def test_generic_kernel_rotations_give_identical_bits(op, window, big_rgba):
    radius, sigma = window
    want = oracle_op(op, big_rgba, radius, sigma)
    set_options(conv_mma=0, pair=0)
    first = None
    for row_rot, col_rot in ((0, 16), (1, 1), (5, 3)):
        set_options(row_rot=row_rot, col_rot=col_rot)
        got, counts = counted(lambda: run_op(op, big_rgba, radius, sigma), CONV_FAMILIES)
        assert_conv_counts(counts, "conv_generic_launches", passes=2)
        if first is None:
            first = got
            assert_exact_enough(got, want, (op, window))
            assert_passthrough(op, big_rgba, got, radius, sigma)
        else:
            assert np.array_equal(got, first), (op, window, row_rot, col_rot, max_ulp(got, first))


# ---- 3. resize variants ---------------------------------------------------------------------------------------------
# every streaming (S, N): Lanczos (2, 12), Lanczos2 / Mitchell (2, 8), Triangle (2, 4), Lanczos (3, 19), (4, 24), (4, 16)
RESIZES = [(im.LanczosFilter, 2), (im.Lanczos2Filter, 2), (im.MitchellFilter, 2), (im.TriangleFilter, 2),
           (im.LanczosFilter, 3), (im.LanczosFilter, 4), (im.Lanczos2Filter, 4)]
# (S, N) of the regular kernels of resize.cu; 3x Lanczos has 19 interior taps and takes the gather kernels
REGULAR = {(im.LanczosFilter, 2), (im.Lanczos2Filter, 2), (im.MitchellFilter, 2), (im.TriangleFilter, 2),
           (im.LanczosFilter, 4), (im.Lanczos2Filter, 4)}
STAGING = [dict(resize_tma=1), dict(resize_tma=2), dict(resize_tma=0, resize_chunk=16, resize_slots=0),
           dict(resize_tma=0, resize_chunk=16, resize_slots=2), dict(resize_tma=0, resize_chunk=8, resize_slots=3),
           dict(resize_tma=0, resize_chunk=8, resize_slots=0)]
OUT_W, OUT_H = 127, 99          # columns not a multiple of 8, rows not a multiple of 32 (the sources neither)


@pytest.mark.parametrize("filt,ratio", RESIZES)
def test_resize_staging_variants_give_identical_bits(filt, ratio):
    src = make_image(OUT_W * ratio, OUT_H * ratio, 4, seed=5 * filt + ratio, kind="alpha_blocks")
    want = orc_resize(src, OUT_W, OUT_H, filt)
    first = None
    for staging in STAGING:
        for strip in (0, 24, 7):
            set_options(resize_strip=strip, **staging)
            got, counts = counted(lambda: _host(im.ResizeImage(_dev(src), OUT_W, OUT_H, filt)), RESIZE_FAMILIES)
            h_family = "resize_h_tma_launches" if staging["resize_tma"] else "resize_h_stream_launches"
            for f in RESIZE_FAMILIES:
                assert counts[f] == (1 if f in ("resize_v_stream_launches", h_family) else 0), (staging, strip, counts)
            if first is None:
                first = got
                assert max_ulp(got, want) <= 1, (filt, ratio)
            else:
                assert np.array_equal(got, first), (filt, ratio, staging, strip, max_ulp(got, first))


@pytest.mark.parametrize("filt,ratio", RESIZES)
def test_resize_regular_kernels_all_channel_counts(filt, ratio):
    set_options(resize_regular_h=1, no_resize_stream=1)
    for ch in (1, 2, 3, 4):
        src = make_image(OUT_W * ratio, OUT_H * ratio, ch, seed=ch + filt, kind="hdr" if ch == 3 else "alpha_blocks")
        want = orc_resize(src, OUT_W, OUT_H, filt)
        got, counts = counted(lambda: _host(im.ResizeImage(_dev(src), OUT_W, OUT_H, filt)), RESIZE_FAMILIES)
        regular = 0
        if (filt, ratio) in REGULAR:
            # the vertical regular kernel always; the horizontal one while its tile of 32 outputs (the widest source
            # span, S * 31 + N pixels, odd pitch) fits 48 KB of shared memory
            s_n = {(im.LanczosFilter, 2): (2, 12), (im.Lanczos2Filter, 2): (2, 8), (im.MitchellFilter, 2): (2, 8),
                   (im.TriangleFilter, 2): (2, 4), (im.LanczosFilter, 4): (4, 24), (im.Lanczos2Filter, 4): (4, 16)}
            stride, ntaps = s_n[filt, ratio]
            regular = 1 + (32 * ((stride * 31 + ntaps) | 1) * ch * 4 <= 48 * 1024)
        assert counts["resize_regular_launches"] == regular and counts["resize_gather_launches"] == 2 - regular, \
            (filt, ratio, ch, counts)
        assert counts["resize_v_stream_launches"] + counts["resize_h_tma_launches"] + counts["resize_h_stream_launches"] == 0
        assert max_ulp(got, want) <= 1, (filt, ratio, ch)


def test_resize_strip_count_past_the_grid_limit_falls_back():
    """resize_strip = 1 on a 140000-row axis needs more than 65535 strips: the streaming launch declines and the regular
    kernel serves the axis, with the same result."""
    src = make_image(8, 140000, 4, seed=3)
    want = orc_resize(src, 8, 70000, im.TriangleFilter)
    streamed, counts = counted(lambda: _host(im.ResizeImage(_dev(src), 8, 70000, im.TriangleFilter)), RESIZE_FAMILIES)
    assert counts["resize_v_stream_launches"] == 1 and counts["resize_regular_launches"] == 0, counts
    assert max_ulp(streamed, want) <= 1
    util.set_option("resize_strip", 1)
    got, counts = counted(lambda: _host(im.ResizeImage(_dev(src), 8, 70000, im.TriangleFilter)), RESIZE_FAMILIES)
    assert counts["resize_v_stream_launches"] == 0 and counts["resize_regular_launches"] == 1, counts
    assert max_ulp(got, want) <= 1


def test_resize_table_cache_eviction():
    """The axis tables are cached per (device, filter, options, in_n, out_n), at most 64 of them.  Resizes through 70
    more keys evict the first one; coming back to it rebuilds its tables, and the streaming kernels serve it again
    with the same bits."""
    src = make_image(254, 198, 4, seed=21, kind="alpha_blocks")
    want = orc_resize(src, 127, 99, im.LanczosFilter)
    first, counts = counted(lambda: _host(im.ResizeImage(_dev(src), 127, 99, im.LanczosFilter)), RESIZE_FAMILIES)
    assert counts["resize_v_stream_launches"] == 1, counts
    assert max_ulp(first, want) <= 1
    for k in range(70):                  # 70 distinct x keys (2 (64 + k) -> 64 + k), one shared y key
        other = make_image(2 * (64 + k), 16, 4, seed=k, kind="alpha_blocks")
        got = _host(im.ResizeImage(_dev(other), 64 + k, 8, im.LanczosFilter))
        assert max_ulp(got, orc_resize(other, 64 + k, 8, im.LanczosFilter)) <= 1, k
    again, counts = counted(lambda: _host(im.ResizeImage(_dev(src), 127, 99, im.LanczosFilter)), RESIZE_FAMILIES)
    assert counts["resize_v_stream_launches"] == 1, counts
    assert np.array_equal(again, first)


# ---- 4. device buffers that are not 16-byte aligned -----------------------------------------------------------------
def _unaligned(a):
    """A pixel cache whose data pointer is one float past a 16-byte boundary."""
    import torch
    flat = torch.empty(a.size + 1, dtype=torch.float32, device="cuda")
    t = flat[1:].view(a.shape)
    t.copy_(torch.from_numpy(a))
    img = im.Image(t)
    assert img.pixels.data_ptr() % 16 == 4
    return img


@pytest.mark.parametrize("op", ["blur", "unsharp"])
def test_unaligned_source_convolution(op):
    """The matrix and pair kernels need 16-byte aligned pixels: they decline the row pass, which reads the unaligned
    source, and the generic kernel serves it; the column pass reads the aligned intermediate."""
    src = make_image(131, 97, 4, seed=8, kind="alpha_blocks")
    radius, sigma = 8.0, 2.5
    fn = {"blur": lambda img: im.BlurImage(img, radius, sigma),
          "unsharp": lambda img: im.UnsharpMaskImage(img, radius, sigma, *UNSHARP)}[op]
    want = oracle_op(op, src, radius, sigma)
    aligned = _host(fn(_dev(src)))
    for mode, column_family in (("mma", "conv_mma_launches"), ("pair", "pair")):
        set_options(**RGBA_MODES[mode])
        got, counts = counted(lambda: _host(fn(_unaligned(src))), CONV_FAMILIES)
        assert counts["conv_generic_launches"] == 1, (mode, counts)
        if column_family == "pair":
            assert counts["conv_pair_launches"] + counts["conv_pair_async_launches"] == 1, counts
        else:
            assert counts[column_family] == 1, counts
        assert max_ulp(got, aligned) <= 1 and max_ulp(got, want) <= 1, mode
    # both passes on the generic kernels: the unaligned source gives the aligned source's bits
    set_options(**RGBA_MODES["generic"])
    got, counts = counted(lambda: _host(fn(_unaligned(src))), CONV_FAMILIES)
    assert_conv_counts(counts, "conv_generic_launches", passes=2)
    assert np.array_equal(got, _host(fn(_dev(src))))
    assert max_ulp(got, want) <= 1


def test_unaligned_source_resize():
    """The resize kernels move whole 16-byte pixels (float4 loads, 16-byte cp.async and TMA copies), so an unaligned
    pixel cache is resized through aligned copies: the same kernels serve it and give the aligned run's bits.  x is
    reduced less than y, so the horizontal pass is the one that reads the source."""
    src = make_image(254, 396, 4, seed=12, kind="alpha_blocks")
    ow, oh = 127, 99
    for staging in STAGING[:1] + STAGING[2:3]:
        set_options(**staging)
        h_family = "resize_h_tma_launches" if staging["resize_tma"] else "resize_h_stream_launches"
        aligned, counts = counted(lambda: _host(im.ResizeImage(_dev(src), ow, oh, im.LanczosFilter)), RESIZE_FAMILIES)
        assert counts[h_family] == 1 and counts["resize_v_stream_launches"] == 1, counts
        got, counts = counted(lambda: _host(im.ResizeImage(_unaligned(src), ow, oh, im.LanczosFilter)), RESIZE_FAMILIES)
        assert counts[h_family] == 1 and counts["resize_v_stream_launches"] == 1, counts
        assert np.array_equal(got, aligned)
        assert max_ulp(got, orc_resize(src, ow, oh, im.LanczosFilter)) <= 1


# ---- every family is reachable through the knobs ---------------------------------------------------------------------
def test_every_launch_family_is_reachable():
    """One small run per family; prints the process totals of every counter (with -s)."""
    rgba = make_image(67, 45, 4, seed=2)
    gray = make_image(67, 45, 1, seed=2)
    big = make_image(254, 198, 4, seed=2)
    runs = [
        ("conv_mma_launches", dict(conv_mma=1), lambda: im.BlurImage(_dev(rgba), 0.0, 2.0)),
        ("conv_pair_launches", dict(conv_mma=0, pair_async=0), lambda: im.BlurImage(_dev(rgba), 0.0, 2.0)),
        ("conv_pair_async_launches", dict(conv_mma=0, pair_async=1), lambda: im.BlurImage(_dev(rgba), 0.0, 2.0)),
        ("conv_generic_launches", {}, lambda: im.BlurImage(_dev(gray), 0.0, 2.0)),
        ("resize_v_stream_launches", {}, lambda: im.ResizeImage(_dev(big), 127, 99, im.LanczosFilter)),
        ("resize_h_tma_launches", dict(resize_tma=1), lambda: im.ResizeImage(_dev(big), 127, 99, im.LanczosFilter)),
        ("resize_h_stream_launches", dict(resize_tma=0), lambda: im.ResizeImage(_dev(big), 127, 99, im.LanczosFilter)),
        ("resize_regular_launches", {}, lambda: im.ResizeImage(_dev(big[..., :1].copy()), 127, 99, im.LanczosFilter)),
        ("resize_gather_launches", {}, lambda: im.ResizeImage(_dev(big), 100, 77, im.LanczosFilter)),
    ]
    for family, options, fn in runs:
        set_options(**options)
        _, counts = counted(lambda: _host(fn()), (family,))
        assert counts[family] > 0, family
        util.reset_options()
    totals = {f: util.get_option(f) for f in CONV_FAMILIES + RESIZE_FAMILIES}
    print("\nlaunches per kernel family since process start:")
    for f, v in totals.items():
        print(f"  {f:28s} {v}")
    assert all(v > 0 for v in totals.values()), totals
