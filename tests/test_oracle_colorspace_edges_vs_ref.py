"""The oracle against the real reference, bit for bit, for every in-place TransformImageColorspace leg on the edge images of
colorspace_edge_cases: sRGB <-> Lab / XYZ / linear RGB, the XYZ family, the hue / saturation spaces, the matrix and LUT
spaces, Log and YCC, each forward from sRGB and back to sRGB (from the forward output and from the special values written
directly as that space's components), RGB and RGBA, plus a D50 Lab and a Jzazbz with a white luminance set.  The GPU
suite (test_gpu_colorspace_edges.py) compares the kernels with this oracle.

util.digest hashes every NaN as one value and -0 as +0, so each result also stores a digest of where its zeros are
negative: the sign of a zero is pinned separately (the sign of an infinity is part of the main digest).

The reference's results are stored in tests/golden/colorspace_edge_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_colorspace_edges_vs_ref.py

where oracle/_ref is built."""
import ctypes as C

import numpy as np
import pytest

import colorspace_edge_cases as ec
import util
from util import P, ROOT, digest

DIGESTS = ROOT / "tests" / "golden" / "colorspace_edge_digests.json"
# "<digest>/<zero-sign digest>" of what the reference computed for each case of the running test
reference = util.ReferenceStore(DIGESTS, util.REF_SO)


def key(a):
    return f"{digest(a)}/{util.zero_signs(a)}"


def orc(src, frm, to, values=None):
    h, w, ch = src.shape
    out = src.copy()
    opts = C.byref(util.ColorspaceOptions.of(**values)) if values else None
    assert util.oracle().orc_colorspace_ex(P(out), w, h, ch, frm, to, opts) == 0
    return out


def ref(src, frm, to, defines=None):
    h, w, ch = src.shape
    out = src.copy()
    if defines:
        assert util.ref().ref_colorspace_defines(P(out), w, h, ch, frm, to, defines.encode()) == 0
    else:
        assert util.ref().ref_colorspace(P(out), w, h, ch, frm, to) == 0
    return out


def check(src, frm, to, case, settings=None):
    defines, values = settings or (None, None)
    got = orc(src, frm, to, values)
    if src.shape[2] == 4:
        assert np.array_equal(got[..., 3].view(np.int32), src[..., 3].view(np.int32)), case     # alpha untouched
    assert key(got) == reference(case, lambda: key(ref(src, frm, to, defines))), case
    return got


@pytest.mark.parametrize("cs", ec.SPACES)
def test_edge_legs(cs):
    """sRGB -> cs on the edge image, then cs -> sRGB on that output stacked on the edge image read as cs samples."""
    for ch in (3, 4):
        fwd = check(ec.edge_image(ch), ec.SRGB, cs, f"{ch} forward")
        check(ec.inverse_source(fwd, ch), cs, ec.SRGB, f"{ch} inverse")


SETTINGS = [(ec.LAB, "color:illuminant=D50", dict(illuminant="D50")),
            (34, "white-luminance=203", dict(white_luminance=203.0))]


@pytest.mark.parametrize("case", range(len(SETTINGS)), ids=["Lab-D50", "Jzazbz-203"])
def test_edge_legs_with_settings(case):
    cs, defines, values = SETTINGS[case]
    for ch in (3, 4):
        fwd = check(ec.edge_image(ch), ec.SRGB, cs, f"{ch} forward", (defines, values))
        check(ec.inverse_source(fwd, ch), cs, ec.SRGB, f"{ch} inverse", (defines, values))
