"""The oracle against the real reference, bit for bit, for the directly applied morphology methods: MorphologyImage with
Distance (21) and Voronoi (22), MorphologyPrimitiveDirect's two sequential sweeps.  The kernels (direct_cases.KERNELS) are
the four distance kernels at radii 1-4, with and without a scale, and user kernels with off-centre origins, asymmetric
values, NaN cells, 1xN / Nx1 shapes and kernel lists (only the head kernel is used).  The inputs (direct_cases.sources)
are binary shapes, noise, HDR values below 0 and above QuantumRange (where "before the pass" and "live" differ), +-inf
and NaN samples, and 1x1 / 1xN / Nx1 images, on 1-4 channels.  Each stored result pins the head kernel the reference
parsed, the pixels, the channel count of the result and its alpha trait (Voronoi adds an alpha channel to an image
without one and leaves the alpha trait at Copy).

The reference's results are stored in tests/golden/direct_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_direct_vs_ref.py

where oracle/_ref is built."""
import numpy as np
import pytest

import direct_cases as dc
from util import make_image

CHANNELS = [1, 2, 3, 4]


def check(src, method, kernel, case):
    got = dc.orc_key(src, method, kernel)
    want = dc.reference(case, lambda: dc.ref_key(src, method, kernel))
    assert got == want, case


@pytest.mark.parametrize("ch", CHANNELS)
def test_distance(ch):
    for name, src in dc.sources(ch).items():
        for kernel in dc.KERNELS:
            check(src, dc.DISTANCE, kernel, f"{kernel} {name}")


@pytest.mark.parametrize("ch", CHANNELS)
def test_voronoi(ch):
    """Voronoi's three differences from Distance, and its alpha epilogue: the source's alpha (or, without alpha, its
    intensity in a new channel) and ClampPixel on the swept channels."""
    for name, src in dc.sources(ch).items():
        for kernel in dc.KERNELS:
            check(src, dc.VORONOI, kernel, f"{kernel} {name}")


@pytest.mark.parametrize("method", [dc.DISTANCE, dc.VORONOI])
def test_iterations_ignored(method):
    """MorphologyApply runs the direct primitive once, whatever the iteration count (only 0 is a null operation)."""
    src = dc.sources(4)["shapes"]
    want = dc.orc_key(src, method, "Euclidean:2")
    for its in (2, 5, -1):
        h, w, ch = src.shape
        got = dc.reference(f"iterations {its}", lambda: dc.result_key(
            dc.digest(dc.kernel_values(*dc.util.ref_kernel("Euclidean:2"))),
            *dc.ref_run(src, method, "Euclidean:2", its)))
        assert got == want, its


def test_larger_image():
    """A 150x130 binary RGBA image: rows and columns well beyond every kernel."""
    src = dc.shapes(150, 130, 4, seed=21)
    for kernel in ("Euclidean:4", "Chebyshev:1", "3x3+2+2:5,-,1 2,0,3 -,4,-"):
        for method in (dc.DISTANCE, dc.VORONOI):
            check(src, method, kernel, f"{kernel} {method}")


def test_hdr_before_and_live_differ():
    """Negative kernel values over HDR noise: a value updated earlier in the same row is below the value the row had
    before the pass, so reading one for the other changes the result."""
    src = make_image(31, 17, 3, seed=9, kind="hdr")
    for kernel in ("3x3:-3000,-2000,-1000 -500,0,-500 -1000,-2000,-3000", "5x1+2+0:-100,-50,0,-50,-100"):
        got = dc.orc_run(src, dc.DISTANCE, kernel)[0]
        assert np.isfinite(got).all() and (got < src.min()).any()        # Voronoi's composite clamps these to 0
        for method in (dc.DISTANCE, dc.VORONOI):
            check(src, method, kernel, f"{kernel} {method}")
