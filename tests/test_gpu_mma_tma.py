"""The TMA-fed wide-tile pass of conv_mma.cu against the digests of the register-fed kernel it replaced
(tests/golden/mma_wide_digests.json: the same bits on every sample), and its edge clamping against the oracle on images
shorter than one 16-position box along the filter axis."""
import json
from pathlib import Path

import numpy as np
import pytest

import mma_wide_cases
import util

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")

DIGESTS = json.loads((Path(__file__).parent / "golden" / "mma_wide_digests.json").read_text())
CASES = {c[0]: c for c in mma_wide_cases.cases()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_wide_pass_keeps_the_register_fed_bits(name):
    _, kind, w, h, make = CASES[name]
    got, wide = mma_wide_cases.run(im, kind, make())
    assert wide == (2 if kind == "unsharp" else 1), (name, wide)
    assert mma_wide_cases.sha256(got) == DIGESTS[name], name


@pytest.mark.parametrize("kind", ["row", "column"])
@pytest.mark.parametrize("n", mma_wide_cases.RAGGED)
def test_wide_pass_clamps_to_the_edge_like_the_oracle(n, kind):
    w, h = (n, 23) if kind == "row" else (23, n)
    src = mma_wide_cases.non_finite(w, h, 7 + n) if n >= 31 else mma_wide_cases.rgba(w, h, 7 + n)
    k = im.AcquireKernelInfo("blur:0x4" if kind == "row" else "blur:0x4+90")
    (values, ox, oy), = k.arrays()
    want = util.orc_morphology(src, im.ConvolveMorphology, 1, [util.orc_kernel_from_array(values, ox, oy)])
    got, wide = mma_wide_cases.run(im, kind, src)
    assert wide == 1
    assert np.array_equal(np.isnan(got), np.isnan(want))
    inf = np.isinf(want)
    assert np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], want[inf])
    ok = np.isfinite(want)
    d = util.ulp_distance(np.where(ok, got, np.float32(0)), np.where(ok, want, np.float32(0)))
    assert d.max() <= 1, (n, kind, int(d.max()))
