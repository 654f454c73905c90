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
import atexit
import json
import os

import numpy as np
import pytest

import stencil_edge_cases as ec
import util
from util import P, ROOT, digest

DIGESTS = ROOT / "tests" / "golden" / "stencil_edge_digests.json"
_stored = {}                    # digest file -> its contents
_recorded = {}                  # digest file -> {(test, case): result}


def _save_recorded():
    for path, recorded in _recorded.items():
        data = json.loads(path.read_text()) if path.exists() else {}
        for (test, case), value in recorded.items():
            data.setdefault(test, {})[case] = value
        path.write_text("{\n" + ",\n".join(json.dumps(t) + ": " + json.dumps(c, separators=(",", ":"))
                                            for t, c in sorted(data.items())) + "\n}\n")


def _signs(a):
    return digest((a == 0) & np.signbit(a))


def reference(case, run, digests=DIGESTS):
    """"<digest>/<zero-sign digest>" of what the reference computed for `case` of the running test, stored in the file
    `digests`.  With MB200_RECORD_REFERENCE=1 and oracle/_ref built, run() computes it with the reference and it is
    recorded when the process exits."""
    test = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0].split("::", 1)
    test = test[0].rsplit("/", 1)[-1] + "::" + test[-1]
    if os.environ.get("MB200_RECORD_REFERENCE") == "1" and util.have_ref():
        if not _recorded:
            atexit.register(_save_recorded)
        out = run()
        recorded = _recorded.setdefault(digests, {})
        recorded[test, case] = f"{digest(out)}/{_signs(out)}"
        return recorded[test, case]
    if digests not in _stored:
        _stored[digests] = json.loads(digests.read_text())
    stored = _stored[digests].get(test, {})
    assert case in stored, f"no stored reference result for {test} / {case}"
    return stored[case]


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
    want = reference(case, lambda: _masked(_call(util.ref(), "ref_" + op, src, args), src, op, args))
    assert f"{digest(got)}/{_signs(got)}" == want, case


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
