"""The oracle against the real reference, bit for bit, for ResizeImage, SampleImage, ScaleImage and ThumbnailImage on
the edge images and geometries of resample_edge_cases, 1-4 channels: special values in every channel and in alpha,
whole NaN rows and columns, infinite alpha lines, blocks whose products are all -0, 1 x 1 / 1 x N / N x 1 / 2 x 2
sources, reductions to one row or column, same-size resizes with a filter, the regular table's threshold, factors one
double ULP apart, and every filter.  The GPU suite (test_gpu_resample_edges.py) compares the kernels with this oracle.

Each result is stored as "<digest>/<zero-sign digest>" (test_oracle_stencil_edges_vs_ref.reference) in
tests/golden/resample_edge_digests.json, since util.digest hashes -0 as +0; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_resample_edges_vs_ref.py

where oracle/_ref is built."""
import numpy as np
import pytest

import resample_edge_cases as rc
import test_oracle_stencil_edges_vs_ref as stencil
import util
from util import P, digest

DIGESTS = util.ROOT / "tests" / "golden" / "resample_edge_digests.json"


def _run(lib, name, src, ow, oh, *args):
    h, w, ch = src.shape
    out = np.full((oh, ow, ch), -12345.5, np.float32)
    assert getattr(lib, name)(P(src), w, h, ch, P(out), ow, oh, *args) == 0, (name, src.shape, ow, oh, args)
    return out


def check(op, src, ow, oh, args, case):
    got = _run(util.oracle(), "orc_" + op, src, ow, oh, *args)
    want = stencil.reference(case, lambda: _run(util.ref(), "ref_" + op, src, ow, oh, *args), DIGESTS)
    assert f"{digest(got)}/{stencil._signs(got)}" == want, case


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_resize_edges(ch):
    for name, src, ow, oh, f in rc.resize_cases(ch):
        check("resize", src, ow, oh, (f,), f"{ch} {name}")


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("op", ["sample", "scale"])
def test_sample_and_scale_edges(op, ch):
    for name, src, ow, oh in rc.sample_cases(ch):
        check(op, src, ow, oh, (), f"{ch} {name}")


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
def test_thumbnail_edges(ch):
    for name, src, ow, oh in rc.thumbnail_cases(ch):
        check("thumbnail", src, ow, oh, (), f"{ch} {name}")


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("case", list(rc.NAMED))
def test_named_reproductions(case, ch):
    build, ow, oh, f = rc.NAMED[case]
    check("resize", build(ch), ow, oh, (f,), f"{ch}")
