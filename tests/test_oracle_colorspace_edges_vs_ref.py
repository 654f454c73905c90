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
import atexit
import ctypes as C
import json
import os

import numpy as np
import pytest

import colorspace_edge_cases as ec
import util
from util import P, ROOT, digest

DIGESTS = ROOT / "tests" / "golden" / "colorspace_edge_digests.json"
_stored = None
_recorded = {}


def _save_recorded():
    data = json.loads(DIGESTS.read_text()) if DIGESTS.exists() else {}
    for (test, case), value in _recorded.items():
        data.setdefault(test, {})[case] = value
    DIGESTS.write_text("{\n" + ",\n".join(json.dumps(t) + ": " + json.dumps(c, separators=(",", ":"))
                                           for t, c in sorted(data.items())) + "\n}\n")


def _signs(a):
    return digest((a == 0) & np.signbit(a))


def reference(case, run):
    """"<digest>/<zero-sign digest>" of what the reference computed for `case` of the running test.  With
    MB200_RECORD_REFERENCE=1 and oracle/_ref built, run() computes it with the reference and it is recorded when the
    process exits."""
    global _stored
    test = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0].split("::", 1)
    test = test[0].rsplit("/", 1)[-1] + "::" + test[-1]
    if os.environ.get("MB200_RECORD_REFERENCE") == "1" and util.have_ref():
        if not _recorded:
            atexit.register(_save_recorded)
        out = run()
        _recorded[test, case] = f"{digest(out)}/{_signs(out)}"
        return _recorded[test, case]
    if _stored is None:
        _stored = json.loads(DIGESTS.read_text())
    stored = _stored.get(test, {})
    assert case in stored, f"no stored reference result for {test} / {case}"
    return stored[case]


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
    assert f"{digest(got)}/{_signs(got)}" == reference(case, lambda: ref(src, frm, to, defines)), case
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
