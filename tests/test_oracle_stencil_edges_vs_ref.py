"""The oracle against the real reference, bit for bit, for the stencil operators -- StatisticImage (all ten types),
RotationalBlurImage, BilateralBlurImage, SelectiveBlurImage, AdaptiveBlurImage, AdaptiveSharpenImage and MotionBlurImage
-- on the edge images of stencil_edge_cases, 1-4 channels: special values in every channel and in alpha, rows that start
with NaN, posterised images with thresholds at (and one ULP either side of) contrasts that occur in them, 1x1 / 1xN / Nx1
/ 2x2 images and windows larger than the image.  The GPU suite (test_gpu_stencil_edges.py) compares the kernels with this
oracle.

util.digest hashes every NaN as one value and -0 as +0, so each result also stores a digest of where its zeros are
negative.  BilateralBlurImage's pixels next to a full-range 8-bit intensity jump are left out (set to 0 on both sides):
there the reference reads an element of its intensity table that it never initialises (stencil_edge_cases.full_jump).

The reference's results are stored in tests/golden/stencil_edge_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_stencil_edges_vs_ref.py

where oracle/_ref is built."""
import numpy as np
import pytest

import stencil_edge_cases as ec
import util
from util import P, ROOT, digest

DIGESTS = ROOT / "tests" / "golden" / "stencil_edge_digests.json"
# "<digest>/<zero-sign digest>" of what the reference computed for each case of the running test
reference = util.ReferenceStore(DIGESTS, util.REF_SO)


def key(a):
    return f"{digest(a)}/{util.zero_signs(a)}"


def _call(lib, name, src, args):
    h, w, ch = src.shape
    out = np.full_like(src, -12345.5)
    assert getattr(lib, name)(P(src), P(out), w, h, ch, *args) == 0, (name, src.shape, args)
    return out


def _masked(out, src, op, args):
    if op == "bilateral_blur":
        out = out.copy()
        out[ec.full_jump(src, args[0], args[1])] = 0.0
    return out


def check(op, src, args, case):
    got = _masked(_call(util.oracle(), "orc_" + op, src, args), src, op, args)
    want = reference(case, lambda: key(_masked(_call(util.ref(), "ref_" + op, src, args), src, op, args)))
    assert key(got) == want, case


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("stat", range(1, 11))
def test_statistic_edges(stat, ch):
    for name, src, args in ec.cases("statistic", ch, stat):
        check("statistic", src, args, f"{ch} {name}")


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("op", ec.OPERATORS[1:])
def test_operator_edges(op, ch):
    for name, src, args in ec.cases(op, ch):
        check(op, src, args, f"{ch} {name}")


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("case", list(ec.NAMED))
def test_named_reproductions(case, ch):
    op, build, args = ec.NAMED[case]
    check(op, build(ch), args, f"{ch}")
