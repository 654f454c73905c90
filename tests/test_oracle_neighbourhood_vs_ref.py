"""The oracle against the real reference, bit for bit, where the GPU tests of the 2-D neighbourhood kernels lean on it:
erode / dilate and the methods built on them on images with NaN and +-inf samples (at window centres, next to the
image edge where the clamp replicates them, in an all-NaN block), 2-D Convolve / Correlate with asymmetric, mixed-sign
and zero-sum user kernels at every corner origin and the centre, and iterated runs (the `changed` loop).

The reference's results are stored as digests in tests/golden/ref_digests.json (util.reference); re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_neighbourhood_vs_ref.py

where oracle/_ref is built."""
import numpy as np
import pytest

import util
from util import P, digest, make_image, reference

ERODE, DILATE, OPEN, CLOSE, SMOOTH, EDGE_IN, TOP_HAT = 3, 4, 8, 9, 12, 13, 16
CONVOLVE, CORRELATE = 1, 2


def ref_morphology(src, method, its, name):
    h, w, ch = src.shape
    a = np.empty_like(src)
    assert util.ref().ref_morphology(P(src), P(a), w, h, ch, method, its, name.encode()) == 0
    return a


def kernel_values(vals, x, y):
    return np.concatenate([[vals.shape[0], vals.shape[1], x, y], np.asarray(vals, np.float64).ravel()])


def kernel_list(string):
    """The product's host-side expansion of a kernel string as oracle kernels; it must equal the reference's own."""
    im = pytest.importorskip("imagemagick_b200")
    mine = im.AcquireKernelInfo(string).arrays()

    def ref_list():
        out, idx = [], 0
        while (k := util.ref_kernel(string, idx)) is not None:
            out.append(kernel_values(*k))
            idx += 1
        return np.concatenate(out)
    assert digest(np.concatenate([kernel_values(*k) for k in mine])) == reference("kernels", ref_list), string
    return [util.orc_kernel_from_array(v, x, y) for v, x, y in mine]


def awkward(w, h, ch, seed, kind="noise"):
    """make_image with NaN, +inf and -inf in colour and in alpha: at interior window centres, on the first / last row
    and column and in the corners (the edge clamp replicates them), and one all-NaN 3x3 block."""
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
    """Exact binary fractions in row-major order: asymmetric, mixed-sign, or mixed-sign summing to exactly zero."""
    i = np.arange(kw * kh)
    if kind == "asymmetric":
        v = (1.0 + (3 * i) % 7) / 8.0
    else:
        v = ((5 * i + i // kw) % 9 - 4) / 4.0
        v[0] = 1.25
        if kind == "zero_sum":
            v[-1] = -v[:-1].sum()
    return v.reshape(kh, kw)


def user_kernel(values, x, y):
    kh, kw = values.shape
    body = " ".join(",".join("nan" if np.isnan(t) else repr(float(t)) for t in row) for row in values)
    return f"{kw}x{kh}+{x}+{y}: {body}"


# ---- erode / dilate and the methods built on them, non-finite samples --------------------------------------------------
# table shapes of the streaming kernel, shapes outside it (Disk:6, a ring, off-centre rectangles, a user kernel with
# holes), a 34-wide rectangle (past the min/max kernel's width limit) and a 1x11 line
MORPH_KERNELS = [("disk2", "Disk:2"), ("square1", "Square:1"), ("disk6", "Disk:6"), ("ring", "Ring:2,3.5"),
                 ("rect_off", "Rectangle:4x3+0+2"), ("rect34", "Rectangle:34x2+33+1"), ("line", "1x11+0+3: " + ",".join(["1"] * 11)),
                 ("holes", "3x3+2+0: 1,nan,1 0,1,0 1,0.5,nan")]
MORPH_METHODS = [ERODE, DILATE, OPEN, CLOSE, SMOOTH, EDGE_IN, TOP_HAT]


@pytest.mark.parametrize("name,string", MORPH_KERNELS, ids=[k for k, _ in MORPH_KERNELS])
def test_morphology_non_finite_samples_bit_exact(name, string):
    """Erode starts from the centre value and keeps it unless a sample is smaller (morphology.c:2980-3006): a NaN centre
    stays NaN, NaN neighbours are skipped.  Dilate starts from 0 and skips NaN samples (:3007-3036)."""
    kernels = kernel_list(string)
    for ch in (1, 2, 3, 4):
        src = awkward(41, 29, ch, seed=60 + ch, kind="hdr" if ch == 3 else "noise")
        for method in MORPH_METHODS:
            b = util.orc_morphology(src, method, 1, kernels)
            assert method != ERODE or np.isnan(b).any()        # the NaN centres survive
            assert digest(b) == reference(f"{ch},{method}", lambda: ref_morphology(src, method, 1, string)), \
                (string, ch, method)


# ---- 2-D Convolve / Correlate with user kernels ------------------------------------------------------------------------
def conv_kernels():
    out = []
    for kw, kh in ((3, 3), (4, 4), (5, 3), (2, 6), (7, 7), (55, 55)):
        for oi, (x, y) in enumerate(((0, 0), (kw - 1, 0), (0, kh - 1), (kw - 1, kh - 1), (kw // 2, kh // 2))):
            kind = ("asymmetric", "mixed", "zero_sum")[(oi + kw) % 3]
            out.append(pytest.param(user_kernel(taps_2d(kw, kh, kind), x, y), id=f"{kw}x{kh}+{x}+{y}-{kind}"))
    return out


@pytest.mark.parametrize("string", conv_kernels())
def test_convolve_user_kernels_bit_exact(string):
    """Convolve reflects the kernel and its origin (morphology.c:2612-2626), Correlate rotates it first (:3779-3793);
    zero-sum taps give PerceptibleReciprocal a weight sum near zero of either sign.  The awkward image spreads NaN and
    inf over every window that holds one; the clean alpha-block image keeps most outputs finite for the big kernel."""
    kernels = kernel_list(string)
    for ch in (1, 2, 3, 4):
        for label, src in (("awkward", awkward(37, 27, ch, seed=80 + ch)),
                           ("alpha_blocks", make_image(37, 27, ch, seed=90 + ch, kind="alpha_blocks"))):
            for method in (CONVOLVE, CORRELATE):
                b = util.orc_morphology(src, method, 1, kernels)
                assert digest(b) == reference(f"{ch},{label},{method}", lambda: ref_morphology(src, method, 1, string)), \
                    (string, ch, label, method)


# ---- iterated runs: the `changed` loop --------------------------------------------------------------------------------
ITERATED = [(CONVOLVE, "3x3: 0.0625,0.125,0.0625 0.125,0.25,0.125 0.0625,0.125,0.0625"),
            (CONVOLVE, "3x2+0+1: 0.125,0.25,0.125 0.25,0.125,0.125"),
            (ERODE, "Disk:1"), (ERODE, "Rectangle:3x2+0+1"), (DILATE, "Diamond:1")]


@pytest.mark.parametrize("its", [3, -1])
@pytest.mark.parametrize("case", range(len(ITERATED)))
def test_iterated_convolve_and_erode_bit_exact(case, its):
    """`iterations` repeats the primitive while it changes anything (morphology.c:3919-3962); -1 means up to
    max(columns, rows) times."""
    method, string = ITERATED[case]
    kernels = kernel_list(string)
    for ch in (1, 2, 3, 4):
        src = awkward(31, 23, ch, seed=100 + ch)
        b = util.orc_morphology(src, method, its, kernels)
        assert digest(b) == reference(f"{ch}", lambda: ref_morphology(src, method, its, string)), (string, ch, its)
