"""The 2-D neighbourhood kernels family by family: the dense register-tiled convolution (every channel count and rows-per-
thread R), the compacted-cell kernel, the min/max kernel and the register-streaming erode / dilate, the rank-1 split of
RGBA convolutions, the boundaries between them, non-finite samples, unaligned device buffers and the declines.

Every case reads the per-family launch counters, so a case cannot pass on a fallback kernel.  Bars: convolution <= 1
ULP against the oracle where it is finite, NaN and inf exactly where it has them; erode / dilate and the methods built
on them bit exact (NaN exactly where the oracle has it, -0 == +0); kernels that only re-tile the same sums give
identical bits to one another."""
import ctypes as C

import numpy as np
import pytest

import util
from util import P, digest, make_image

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")

DENSE = ("conv2d_dense_r8_launches", "conv2d_dense_r4_launches", "conv2d_dense_r2_launches")
MORPH = ("morph2d_launches", "minmax2d_launches", "morph_stream_launches")
CONV1D = ("conv_mma_launches", "conv_pair_launches", "conv_pair_async_launches", "conv_generic_launches")
FAMILIES = DENSE + MORPH + CONV1D
ERODE, DILATE = im.ErodeMorphology, im.DilateMorphology


def _dev(a):
    import torch
    return im.Image(torch.from_numpy(a).cuda())


def _host(img):
    return img.pixels.cpu().numpy() if img.on_device else img.pixels


def _unaligned(a):
    """A pixel cache whose data pointer is one float past a 16-byte boundary."""
    import torch
    flat = torch.empty(a.size + 1, dtype=torch.float32, device="cuda")
    t = flat[1:].view(a.shape)
    t.copy_(torch.from_numpy(a))
    img = im.Image(t)
    assert img.pixels.data_ptr() % 16 == 4
    return img


def counted(fn):
    """Runs fn(); returns its result and how many launches of each family it made."""
    c0 = {f: util.get_option(f) for f in FAMILIES}
    out = fn()
    return out, {f: util.get_option(f) - c0[f] for f in FAMILIES}


def assert_only(counts, expected, n=None):
    """Every launch of the families above is one of `expected` (n of them when given, else at least one)."""
    got = sum(counts[f] for f in expected)
    assert (got == n if n is not None else got > 0), (expected, counts)
    assert all(counts[f] == 0 for f in FAMILIES if f not in expected), (expected, counts)


def assert_matches(got, want, what, taps_abs_sum=None):
    """<= 1 ULP where the oracle is finite; NaN and inf exactly where the oracle has them.  taps_abs_sum (images with
    alpha): colour values whose alpha sum cancels to below 1e-6 of its scale carry no significant bits and are excluded
    from the ULP bar (as in the separable tests)."""
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


def assert_bits(got, want, what):
    """Bit exact, NaN exactly where `want` has it (util.digest: one NaN, -0 == +0)."""
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    assert digest(got) == digest(want), (what, util.max_ulp(np.nan_to_num(got), np.nan_to_num(want)))


def awkward(w, h, ch, seed, kind="noise"):
    """NaN, +inf and -inf in colour and in alpha: interior window centres, first / last rows and columns and corners
    (replicated by the edge clamp), and an all-NaN 3x3 block (the CPU oracle-vs-reference tests use the same layout)."""
    a = make_image(w, h, ch, seed=seed, kind=kind)
    last = ch - 1
    for value, y, x, c in [(np.nan, h // 2, w // 3, 0), (np.inf, h // 3, w // 2, min(1, last)),
                           (-np.inf, 2 * h // 3, 2 * w // 3, 0), (np.nan, h // 4, 3 * w // 4, last),
                           (np.inf, 3 * h // 4, w // 4, last), (-np.inf, h // 5, w // 5, last),
                           (np.nan, 0, w // 2, 0), (np.inf, h - 1, w // 3, last), (-np.inf, h // 2, 0, min(2, last)),
                           (np.nan, h // 3, w - 1, last), (np.nan, 0, 0, last), (np.inf, h - 1, w - 1, 0),
                           (-np.inf, 0, w - 1, 0), (np.nan, h - 1, 0, 0)]:
        a[y, x, c] = value
    a[h - 6:h - 3, w // 2 + 2:w // 2 + 5, :] = np.nan
    return a


def taps_2d(kw, kh, kind):
    """Exact binary fractions in row-major order.  "row" / "column": mixed-sign taps on the middle row / column only,
    zero elsewhere (still 2-D kernels, and not rank-1 splittable: negative taps)."""
    i = np.arange(kw * kh)
    if kind == "asymmetric":
        v = (1.0 + (3 * i) % 7) / 8.0
    else:
        v = ((5 * i + i // kw) % 9 - 4) / 4.0
        v[0] = 1.25
        if kind == "zero_sum":
            v[-1] = -v[:-1].sum()
    v = v.reshape(kh, kw)
    if kind == "row":
        v[np.arange(kh) != kh // 2, :] = 0.0
    elif kind == "column":
        v[:, np.arange(kw) != kw // 2] = 0.0
    return v


def kernel_string(values, x, y):
    kh, kw = values.shape
    body = " ".join(",".join("nan" if np.isnan(t) else repr(float(t)) for t in row) for row in values)
    return f"{kw}x{kh}+{x}+{y}: {body}"


def oracle_kernels(string):
    return [util.orc_kernel_from_array(v, x, y) for v, x, y in im.AcquireKernelInfo(string).arrays()]


def run_morph(src_img, method, its, string, bias=0.0):
    return counted(lambda: _host(im.MorphologyImage(src_img, method, its, string, bias=bias)))


# ---- the launcher's choice, restated ----------------------------------------------------------------------------------
def tile_bytes(kw, kh, ch, rows):
    """Dynamic shared memory of conv2d_dense_kernel: the taps (padded to an even count) and the staged tile of doubles."""
    return (((kw * kh + 1) & ~1) + (32 + kw - 1) * (8 * rows + kh - 1) * ch) * 8


def conv2d_family(kw, kh, ch, forced=0, aligned=True):
    """The family that serves a 2-D Convolve with all-finite taps (None: declined)."""
    if aligned:
        rows = 8 if tile_bytes(kw, kh, ch, 8) <= 110 * 1024 else 4 if tile_bytes(kw, kh, ch, 4) <= 110 * 1024 else \
            2 if tile_bytes(kw, kh, ch, 2) <= 200 * 1024 else 0
        if forced and tile_bytes(kw, kh, ch, forced) <= 200 * 1024:
            rows = forced
        if rows:
            return f"conv2d_dense_r{rows}_launches"
    return "morph2d_launches" if (32 + kw - 1) * (8 + kh - 1) * ch * 4 <= 200 * 1024 else None


def minmax_family(kw, kh, cells, ch, aligned=True):
    """Erode / dilate outside the streaming table (or with a `changed` count)."""
    if cells <= 1024 and kw <= 33 and 64 * (32 + kh - 1) * ch * 4 <= 160 * 1024 and (ch != 4 or aligned):
        return "minmax2d_launches"
    return "morph2d_launches" if (32 + kw - 1) * (8 + kh - 1) * ch * 4 <= 200 * 1024 else None


# square kernels: the last size of each family (R = 8, 4, 2, compacted); past the last one the call is declined
SWITCHES = {1: (57, 66, 101, None), 2: (34, 46, 76, 141), 3: (22, 34, 62, 112), 4: (14, 26, 52, 94)}


def test_family_prediction_matches_the_documented_switches():
    order = list(DENSE) + ["morph2d_launches", None]
    for ch, last in SWITCHES.items():
        fams = [conv2d_family(n, n, ch) for n in range(3, 160)]
        changes = [(n, f) for n, f, prev in zip(range(3, 160), fams, [fams[0]] + fams[:-1]) if f != prev]
        assert [f for _, f in changes] == order[1:len(changes) + 1], (ch, changes)
        assert [n - 1 for n, _ in changes] == [v for v in last if v is not None], (ch, changes)


# ---- 1. dense convolution, every (CH, R) instantiation ----------------------------------------------------------------
# (kw, kh, x, y, taps, method, bias); Correlate rotates the kernel (and its origin) before the dense kernel sees it
DENSE_KERNELS = [(5, 5, 0, 0, "asymmetric", 1, 0.0), (5, 5, 4, 4, "mixed", 2, 0.0), (3, 31, 0, 30, "zero_sum", 1, 0.0),
                 (31, 3, 30, 0, "mixed", 2, 100.0), (7, 4, 3, 2, "zero_sum", 1, -50.0), (9, 9, 8, 0, "asymmetric", 2, 0.0),
                 (7, 5, 0, 4, "row", 1, 0.0), (5, 7, 2, 3, "column", 2, 25.0), (4, 6, 1, 5, "mixed", 1, 0.0)]


def dense_sizes(rows):
    """Widths that are not a multiple of 32, heights around 8R, one row, one column, smaller than the kernel."""
    return [(37, 8 * rows - 1), (45, 8 * rows), (33, 8 * rows + 1), (1, 19), (19, 1), (3, 2), (70, 13)]


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_dense_convolution_every_instantiation(ch):
    util.set_option("no_rank1", 1)
    case = 0
    for kw, kh, x, y, kind, method, bias in DENSE_KERNELS:
        values = taps_2d(kw, kh, kind)
        string = kernel_string(values, x, y)
        k = oracle_kernels(string)
        for rows in (8, 4, 2):
            for w, h in dense_sizes(rows):
                img_kind = ("noise", "alpha_blocks", "hdr")[case % 3]
                case += 1
                src = make_image(w, h, ch, seed=case + 100 * ch, kind=img_kind)
                want = util.orc_morphology(src, method, 1, k, bias=bias)
                first = None
                for forced in (rows,) + tuple(r for r in (8, 4, 2) if r != rows):
                    util.set_option("conv2d_rows", forced)
                    got, counts = run_morph(_dev(src), method, 1, string, bias)
                    assert_only(counts, (f"conv2d_dense_r{forced}_launches",), 1)
                    if first is None:
                        first = got
                        assert_matches(got, want, (string, method, bias, ch, (w, h), img_kind), np.abs(values).sum())
                    else:
                        assert digest(got) == digest(first), (string, ch, (w, h), rows, forced)


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_dense_automatic_rows_at_every_switch(ch):
    """Square kernels on both sides of every switch of the automatic choice (and the decline past the compacted
    kernel's shared memory), on small images so that the oracle stays fast."""
    util.set_option("no_rank1", 1)
    sizes = sorted({n + d for n in SWITCHES[ch] if n is not None for d in (0, 1)})
    for n in sizes:
        family = conv2d_family(n, n, ch)
        values = taps_2d(n, n, "mixed")
        string = kernel_string(values, n // 3, n - 1)
        src = make_image(21, 11, ch, seed=n, kind="alpha_blocks")
        if family is None:
            continue                                     # the declines: section 6
        want = util.orc_morphology(src, im.ConvolveMorphology, 1, oracle_kernels(string))
        got, counts = run_morph(_dev(src), im.ConvolveMorphology, 1, string)
        assert_only(counts, (family,), 1)
        assert_matches(got, want, (n, ch, family), np.abs(values).sum())


def test_forced_rows_that_do_not_fit_keep_the_automatic_choice():
    """conv2d_rows = 8 on a one-channel 101x101 kernel: the R = 8 tile (>= 200 KB) does not fit, R = 2 serves it."""
    n = 101
    assert tile_bytes(n, n, 1, 8) > 200 * 1024 and conv2d_family(n, n, 1) == "conv2d_dense_r2_launches"
    util.set_option("conv2d_rows", 8)
    values = taps_2d(n, n, "mixed")
    string = kernel_string(values, 50, 50)
    src = make_image(9, 7, 1, seed=3)
    got, counts = run_morph(_dev(src), im.ConvolveMorphology, 1, string)
    assert_only(counts, ("conv2d_dense_r2_launches",), 1)
    assert_matches(got, util.orc_morphology(src, im.ConvolveMorphology, 1, oracle_kernels(string)), n)


# ---- 2. the rank-1 split of RGBA convolutions -------------------------------------------------------------------------
def outer(n, x, y, bump=None):
    a = (1.0 + np.minimum(np.arange(n), n - 1 - np.arange(n)) % 4) / 8.0
    b = (2.0 + np.arange(n) % 3) / 4.0
    v = np.outer(a, b)
    if bump is not None:
        v[bump] += 0.5
    return v, kernel_string(v, x, y)


@pytest.mark.parametrize("n,x,y", [(33, 16, 16), (33, 0, 32), (33, 32, 3), (5, 4, 0), (35, 17, 17), (35, 0, 34)])
def test_rank1_split_boundary(n, x, y):
    """Up to 33x33 a non-negative rank-1 kernel is two 1-D passes; past it, with no_rank1, with one cell off the
    product, or with iterations (the `changed` count), the dense kernel serves it."""
    src = make_image(71, 43, 4, seed=n + x, kind="alpha_blocks")
    values, string = outer(n, x, y)
    want = util.orc_morphology(src, im.ConvolveMorphology, 1, oracle_kernels(string))
    got, counts = run_morph(_dev(src), im.ConvolveMorphology, 1, string)
    if n <= 33:
        assert_only(counts, CONV1D, 2)
    else:
        assert_only(counts, (conv2d_family(n, n, 4),), 1)
    assert_matches(got, want, (n, x, y), np.abs(values).sum())
    dense = conv2d_family(n, n, 4)
    util.set_option("no_rank1", 1)
    got2, counts = run_morph(_dev(src), im.ConvolveMorphology, 1, string)
    assert_only(counts, (dense,), 1)
    assert_matches(got2, want, (n, x, y, "no_rank1"), np.abs(values).sum())
    util.set_option("no_rank1", 0)
    values, string = outer(n, x, y, bump=(n // 3, n // 2))
    got, counts = run_morph(_dev(src), im.ConvolveMorphology, 1, string)
    assert_only(counts, (dense,), 1)
    assert_matches(got, util.orc_morphology(src, im.ConvolveMorphology, 1, oracle_kernels(string)), (n, "bump"),
                   np.abs(values).sum())
    values, string = outer(n, x, y)
    got, counts = run_morph(_dev(src), im.ConvolveMorphology, 3, string)
    assert_only(counts, (dense,), 3)
    assert_matches(got, util.orc_morphology(src, im.ConvolveMorphology, 3, oracle_kernels(string)), (n, "its"),
                   np.abs(values).sum() ** 3)


# ---- 3. non-finite samples on the dense and the compacted kernels -----------------------------------------------------
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_convolution_non_finite_samples(ch):
    """inf / NaN samples poison exactly the outputs whose window holds them: on the dense kernel the rows outside an
    output's window must not add 0 * inf; a NaN cell sends the kernel to the compacted-cell kernel."""
    util.set_option("no_rank1", 1)
    for kw, kh, x, y, kind in [(5, 5, 0, 4, "asymmetric"), (4, 7, 3, 0, "mixed"), (11, 3, 5, 1, "zero_sum")]:
        for forced in (8, 4, 2):
            util.set_option("conv2d_rows", forced)
            for nan_cell in (False, True):
                values = taps_2d(kw, kh, kind)
                if nan_cell:
                    values[kh // 2, kw - 1] = np.nan
                    if forced != 8:
                        continue
                string = kernel_string(values, x, y)
                family = "morph2d_launches" if nan_cell else f"conv2d_dense_r{forced}_launches"
                for w, h in ((45, 8 * forced + 1), (37, 29)):
                    src = awkward(w, h, ch, seed=7 * ch + kw)
                    for method in (im.ConvolveMorphology, im.CorrelateMorphology):
                        want = util.orc_morphology(src, method, 1, oracle_kernels(string))
                        got, counts = run_morph(_dev(src), method, 1, string)
                        assert_only(counts, (family,), 1)
                        assert_matches(got, want, (string, ch, forced, method, (w, h)), np.nansum(np.abs(values)))


# ---- 4. erode / dilate across the three kernels -----------------------------------------------------------------------
TABLE_SHAPES = ["Disk:1", "Square:2", "Disk:3", "Octagon:3", "Plus:4", "Diamond:5", "Disk:5", "Rectangle:3x3+1+0"]
OTHER_SHAPES = ["Disk:6", "Ring:2,3.5", "Rectangle:4x3+0+2", "3x3+2+0: 1,nan,1 0,1,0 1,0.5,nan", "Diamond:7"]


def nan_centred(w, h, ch, seed):
    """awkward() plus NaN centres in every channel next to finite neighbours, and a NaN pixel in the corner."""
    a = awkward(w, h, ch, seed)
    a[h // 2 + 3, w // 2 - 5, :] = np.nan
    a[5, 9, ch - 1] = np.nan
    a[h - 1, w - 1, :] = np.nan
    return a


@pytest.mark.parametrize("ch", [1, 4])
@pytest.mark.parametrize("shape", TABLE_SHAPES)
def test_streaming_erode_dilate(shape, ch):
    src = nan_centred(67, 45, ch, seed=len(shape) + ch)
    k = oracle_kernels(shape)
    for method in (ERODE, DILATE):
        want = util.orc_morphology(src, method, 1, k)
        got, counts = run_morph(_dev(src), method, 1, shape)
        assert_only(counts, ("morph_stream_launches",), 1)
        assert_bits(got, want, (shape, ch, method))


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("shape", OTHER_SHAPES + ["Disk:3"])
def test_minmax2d_erode_dilate(shape, ch):
    """Shapes outside the streaming table, and every shape on 2 or 3 channels."""
    src = nan_centred(53, 71, ch, seed=len(shape) * ch)
    k = oracle_kernels(shape)
    streamed = shape == "Disk:3" and ch in (1, 4)
    for method in (ERODE, DILATE):
        want = util.orc_morphology(src, method, 1, k)
        got, counts = run_morph(_dev(src), method, 1, shape)
        assert_only(counts, ("morph_stream_launches" if streamed else "minmax2d_launches",), 1)
        assert_bits(got, want, (shape, ch, method))


BOUNDARIES = [("Rectangle:33x3+16+1", 33, 3, 99), ("Rectangle:34x3+16+1", 34, 3, 102),
              ("Rectangle:32x32+15+15", 32, 32, 1024), ("Rectangle:32x33+15+15", 32, 33, 1056),
              ("1x101+0+50: " + ",".join(["1"] * 101), 1, 101, 101), ("101x1+50+0: " + ",".join(["1"] * 101), 101, 1, 101)]


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("case", range(len(BOUNDARIES)))
def test_minmax2d_boundaries(case, ch):
    """Kernel width 33 vs 34, 1024 vs 1056 active cells, a 1x101 and a 101x1 line."""
    string, kw, kh, cells = BOUNDARIES[case]
    family = minmax_family(kw, kh, cells, ch)
    assert family == ("minmax2d_launches" if cells <= 1024 and kw <= 33 else "morph2d_launches"), (string, ch)
    src = nan_centred(47, 39, ch, seed=case + 10 * ch)
    k = oracle_kernels(string)
    for method in (ERODE, DILATE):
        want = util.orc_morphology(src, method, 1, k)
        got, counts = run_morph(_dev(src), method, 1, string)
        assert_only(counts, (family,), 1)
        assert_bits(got, want, (string, ch, method))


COMPOUND = [im.OpenMorphology, im.CloseMorphology, im.SmoothMorphology, im.EdgeInMorphology, im.EdgeOutMorphology,
            im.EdgeMorphology, im.TopHatMorphology, im.BottomHatMorphology]


@pytest.mark.parametrize("its", [1, 3, -1])
@pytest.mark.parametrize("shape,ch", [("Disk:2", 4), ("Disk:2", 1), ("Ring:2,3.5", 2), ("Rectangle:34x2+33+1", 3)])
def test_methods_built_on_erode_dilate(shape, ch, its):
    """Erode, Dilate and the compound methods with iterations 1, 3 and -1.  With more than one iteration the `changed`
    count decides, which the streaming kernel does not produce: the min/max kernel serves the table shapes."""
    src = nan_centred(39, 27, ch, seed=ch + its)
    k = oracle_kernels(shape)
    cells = sum(int(np.nansum(v >= 0.5)) for v, _, _ in im.AcquireKernelInfo(shape).arrays())
    kw = im.AcquireKernelInfo(shape).arrays()[0][0].shape[1]
    kh = im.AcquireKernelInfo(shape).arrays()[0][0].shape[0]
    fam = minmax_family(kw, kh, cells, ch)
    if its == 1 and shape == "Disk:2" and ch in (1, 4):
        fam = "morph_stream_launches"
    for method in [ERODE, DILATE] + COMPOUND:
        want = util.orc_morphology(src, method, its, k)
        got, counts = run_morph(_dev(src), method, its, shape)
        assert_only(counts, (fam,))
        assert_bits(got, want, (shape, ch, its, method))


def padded(shape, pad):
    """The kernel of `shape` with `pad` NaN columns on the right: the same neighbourhood, too wide for the min/max
    kernel (width > 33), so the generic kernel serves it."""
    (v, x, y), = im.AcquireKernelInfo(shape).arrays()
    return kernel_string(np.concatenate([v, np.full((v.shape[0], pad), np.nan)], axis=1), x, y)


@pytest.mark.parametrize("ch", [1, 4])
def test_the_three_erode_dilate_kernels_give_identical_bits(ch):
    src = nan_centred(131, 77, ch, seed=5 + ch)
    wide = padded("Disk:3", 30)
    for method in (ERODE, DILATE):
        want = util.orc_morphology(src, method, 1, oracle_kernels("Disk:3"))
        streamed, counts = run_morph(_dev(src), method, 1, "Disk:3")
        assert_only(counts, ("morph_stream_launches",), 1)
        util.set_option("no_morph_stream", 1)
        minmax, counts = run_morph(_dev(src), method, 1, "Disk:3")
        assert_only(counts, ("minmax2d_launches",), 1)
        util.set_option("no_morph_stream", 0)
        generic, counts = run_morph(_dev(src), method, 1, wide)
        assert_only(counts, ("morph2d_launches",), 1)
        assert_bits(streamed, want, (ch, method))
        assert_bits(minmax, streamed, (ch, method))
        assert_bits(generic, streamed, (ch, method))


def orc_primitive(src, method, kernel, bias=0.0):
    h, w, ch = src.shape
    dst = np.empty_like(src)
    changed = util.oracle().orc_morphology_primitive(P(src), P(dst), w, h, ch, method, C.byref(kernel), bias)
    return dst, changed


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_changed_count_on_each_family(ch):
    """MorphologyPrimitive's `changed` (channel values that moved by >= 1e-12, over the channel count) equals the
    oracle's on the min/max, the generic, the dense and the compacted kernels."""
    util.set_option("no_rank1", 1)
    src = nan_centred(45, 37, ch, seed=30 + ch)
    conv = kernel_string(taps_2d(5, 4, "mixed") / 8.0, 1, 3)
    conv_nan = kernel_string(np.where(np.arange(20).reshape(4, 5) == 7, np.nan, taps_2d(5, 4, "mixed") / 8.0), 1, 3)
    cases = [(ERODE, "Disk:3", "minmax2d_launches"), (DILATE, "Ring:2,3.5", "minmax2d_launches"),
             (ERODE, padded("Disk:3", 30), "morph2d_launches"), (DILATE, padded("Square:1", 33), "morph2d_launches"),
             (im.ConvolveMorphology, conv, "conv2d_dense_r8_launches"), (im.ConvolveMorphology, conv_nan, "morph2d_launches")]
    for method, string, family in cases:
        (k,) = oracle_kernels(string)
        want, want_changed = orc_primitive(src, method, k)
        (out, changed), counts = counted(lambda: im.MorphologyPrimitive(_dev(src), method, string))
        assert_only(counts, (family,), 1)
        got = _host(out)
        if method == im.ConvolveMorphology:
            assert_matches(got, want, (string, ch))
        else:
            assert_bits(got, want, (string, ch))
        assert changed == want_changed and changed > 0, (string[:20], ch, changed, want_changed)


# ---- 5. unaligned RGBA device buffers ---------------------------------------------------------------------------------
def unaligned_dst_morphology(src, method, its, string):
    """mb200_morphology_image_dev into a destination that starts 4 bytes past a 16-byte boundary."""
    import torch
    from imagemagick_b200 import _lib
    s = torch.from_numpy(src).cuda()
    flat = torch.full((src.size + 1,), -7.0, dtype=torch.float32, device="cuda")
    d = flat[1:].view(src.shape)
    assert d.data_ptr() % 16 == 4
    k = im.AcquireKernelInfo(string)
    h, w, ch = src.shape
    rc = _lib.load().mb200_morphology_image_dev(s.data_ptr(), d.data_ptr(), w, h, ch, int(method), int(its), k._ptr,
                                                0.0, C.c_void_p(torch.cuda.current_stream().cuda_stream or 1))
    torch.cuda.synchronize()
    return rc, d.cpu().numpy()


@pytest.mark.parametrize("shape", ["Disk:3", "Disk:6"])
def test_unaligned_rgba_erode_dilate(shape):
    """The min/max and streaming kernels move float4 pixels and decline unaligned RGBA: the generic kernel serves it
    with the aligned run's bits, for an unaligned source and for an unaligned destination."""
    src = nan_centred(75, 41, 4, seed=len(shape))
    family = "morph_stream_launches" if shape == "Disk:3" else "minmax2d_launches"
    for method in (ERODE, DILATE, im.OpenMorphology):
        aligned, _ = run_morph(_dev(src), method, 1, shape)
        assert_bits(aligned, util.orc_morphology(src, method, 1, oracle_kernels(shape)), (shape, method))
        got, counts = run_morph(_unaligned(src), method, 1, shape)
        # the primitive that reads the unaligned source; Open's second one reads an aligned temporary
        assert counts["morph2d_launches"] == 1 and counts[family] == (method == im.OpenMorphology), counts
        assert_bits(got, aligned, (shape, method, "src"))
        (rc, got), counts = counted(lambda: unaligned_dst_morphology(src, method, 1, shape))
        assert rc == 0
        assert counts["morph2d_launches"] == 1, counts      # the primitive that writes dst; Open's first one does not
        assert_bits(got, aligned, (shape, method, "dst"))


def test_unaligned_rgba_convolution():
    """The dense kernel needs aligned buffers; the compacted-cell kernel serves unaligned ones within 1 ULP."""
    util.set_option("no_rank1", 1)
    src = awkward(69, 37, 4, seed=4)
    values = taps_2d(7, 5, "mixed")
    string = kernel_string(values, 6, 1)
    want = util.orc_morphology(src, im.ConvolveMorphology, 1, oracle_kernels(string))
    aligned, counts = run_morph(_dev(src), im.ConvolveMorphology, 1, string)
    assert_only(counts, ("conv2d_dense_r8_launches",), 1)
    got, counts = run_morph(_unaligned(src), im.ConvolveMorphology, 1, string)
    assert_only(counts, ("morph2d_launches",), 1)
    assert_matches(got, want, "src", np.abs(values).sum())
    assert_matches(got, aligned, "src vs aligned", np.abs(values).sum())
    (rc, got), counts = counted(lambda: unaligned_dst_morphology(src, im.ConvolveMorphology, 1, string))
    assert rc == 0
    assert_only(counts, ("morph2d_launches",), 1)
    assert_matches(got, want, "dst", np.abs(values).sum())


def test_unaligned_rgba_difference_methods():
    """The erode / dilate stages run on the generic kernel; the Difference composite then needs aligned RGBA buffers.
    Edge composites two aligned temporaries and gives the aligned run's bits; EdgeIn / EdgeOut / TopHat / BottomHat
    composite onto the unaligned source and fail cleanly."""
    src = nan_centred(53, 35, 4, seed=9)
    for method in (im.EdgeMorphology, im.EdgeInMorphology, im.EdgeOutMorphology, im.TopHatMorphology,
                   im.BottomHatMorphology):
        aligned, _ = run_morph(_dev(src), method, 1, "Disk:3")
        if method == im.EdgeMorphology:
            got, counts = run_morph(_unaligned(src), method, 1, "Disk:3")
            assert_only(counts, ("morph2d_launches",), 2)
            assert_bits(got, aligned, method)
        else:
            with pytest.raises(im.MagickB200Error, match="16-byte aligned"):
                im.MorphologyImage(_unaligned(src), method, 1, "Disk:3")


# ---- 6. declines ------------------------------------------------------------------------------------------------------
def test_declines_leave_dst_untouched_and_launch_nothing():
    """RGBA GaussianBlurImage(0, 20) (a 103x103 kernel) and a two-channel 142x142 user kernel need more shared memory
    than any 2-D kernel has: MB200_EUNSUPPORTED, nothing written, nothing launched."""
    from imagemagick_b200 import _lib
    lib = _lib.load()
    rgba = make_image(40, 30, 4, seed=1)
    ga = make_image(40, 30, 2, seed=2)
    assert conv2d_family(103, 103, 4) is None and conv2d_family(142, 142, 2) is None
    big = kernel_string(taps_2d(142, 142, "mixed"), 70, 70)
    big_kernel = im.AcquireKernelInfo(big)             # owns the kernel list the host call below points to
    runs = [(lambda img: im.GaussianBlurImage(img, 0.0, 20.0), rgba,
             lambda s, d: lib.mb200_gaussian_blur_image(P(s), P(d), 40, 30, 4, 0.0, 20.0)),
            (lambda img: im.MorphologyImage(img, im.ConvolveMorphology, 1, big), ga,
             lambda s, d: lib.mb200_morphology_image(P(s), P(d), 40, 30, 2, im.ConvolveMorphology, 1,
                                                     big_kernel._ptr, 0.0))]
    for op, src, host_call in runs:
        _, counts = counted(lambda: pytest.raises(im.MagickB200Error, op, _dev(src)))
        assert all(v == 0 for v in counts.values()), counts
        dst = np.full_like(src, 12345.0)
        rc, counts = counted(lambda: host_call(src, dst))
        assert rc == _lib.EUNSUPPORTED
        assert all(v == 0 for v in counts.values()), counts
        assert np.all(dst == 12345.0)


# ---- 7. every new family is reachable ---------------------------------------------------------------------------------
def test_every_neighbourhood_family_is_reachable():
    rgba = make_image(67, 45, 4, seed=2)
    gray = make_image(67, 45, 1, seed=2)
    runs = [("conv2d_dense_r8_launches", 0, lambda: im.SharpenImage(_dev(rgba), 2.0, 1.0)),
            ("conv2d_dense_r4_launches", 4, lambda: im.SharpenImage(_dev(gray), 2.0, 1.0)),
            ("conv2d_dense_r2_launches", 2, lambda: im.EdgeImage(_dev(rgba), 1.0)),
            ("morph2d_launches", 0, lambda: im.MorphologyImage(_dev(rgba), ERODE, 1, padded("Disk:2", 30))),
            ("minmax2d_launches", 0, lambda: im.MorphologyImage(_dev(gray), DILATE, 1, "Disk:6")),
            ("morph_stream_launches", 0, lambda: im.MorphologyImage(_dev(rgba), DILATE, 1, "Disk:3"))]
    for family, rows, fn in runs:
        util.set_option("conv2d_rows", rows)
        _, counts = counted(lambda: _host(fn()))
        assert counts[family] > 0, (family, counts)
    totals = {f: util.get_option(f) for f in DENSE + MORPH}
    print("\nlaunches per 2-D kernel family since process start:")
    for f, v in totals.items():
        print(f"  {f:28s} {v}")
    assert all(v > 0 for v in totals.values()), totals
