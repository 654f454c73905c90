"""The oracle against the real reference, bit for bit, for AdaptiveThresholdImage, AutoThresholdImage,
RangeThresholdImage and PerceptibleImage on 1-4 channels (threshold_cases): windows 1x1, 1xN, Nx1, odd, even and larger
than the image with positive, zero and negative bias; NaN early in a row, +-inf, HDR values, posterised levels with
ties at the mean; `-channel` masks; every AutoThreshold method on bimodal, flat, single-level and all-NaN images and on
intensities a few float steps either side of every bin edge, with the "auto-threshold:threshold" property; samples at
and beside each RangeThreshold limit, equal limits; Perceptible's +-0, denormals and +-epsilon.

The reference's results are stored in tests/golden/threshold_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_threshold_vs_ref.py

where oracle/_ref is built."""
import numpy as np
import pytest

import threshold_cases as tc
from threshold_cases import reference, result_key

CHANNELS = [1, 2, 3, 4]


def check(src, op, args, case, mask=-1):
    got = result_key(*tc.orc_run(src, op, args, mask))
    want = reference(case, lambda: tc.ref_run(src, op, args, mask))
    assert got == want, case


@pytest.mark.parametrize("ch", CHANNELS)
def test_adaptive_threshold(ch):
    for name, src in tc.sources(ch).items():
        for ww, wh, bias in tc.WINDOWS:
            check(src, tc.ADAPTIVE, (ww, wh, bias), f"{name} {ww}x{wh}{bias:+g}")
    src = tc.sources(ch)["mosaic"]
    for mname, mask in tc.CHANNEL_MASKS.items():
        check(src, tc.ADAPTIVE, (5, 3, 300.0), f"mask {mname}", mask)


@pytest.mark.parametrize("ch", CHANNELS)
def test_auto_threshold(ch):
    for name, src in tc.auto_sources(ch).items():
        for method in tc.AUTO_METHODS:
            check(src, tc.AUTO, (method,), f"{name} method {method}")


def ref_threshold(img):
    return float(tc.ref_run(img, tc.AUTO, (tc.OTSU,))[1].rstrip("%"))


def orc_threshold(img):
    return float(tc.orc_run(img, tc.AUTO, (tc.OTSU,))[1].rstrip("%"))


@pytest.mark.parametrize("ch", CHANNELS)
def test_auto_threshold_bin_edges_one_by_one(ch):
    """Each sample near a bin edge decides the threshold of its own image (threshold_cases.edge_pairs)."""
    got = tc.edge_thresholds(orc_threshold, ch)
    want = reference("edge thresholds", lambda: (tc.edge_thresholds(ref_threshold, ch), ""))
    assert result_key(got, "") == want
    assert len(np.unique(got)) > 200                         # the images really do land in different bins


@pytest.mark.parametrize("ch", [3, 4])
def test_range_threshold(ch):
    for k, limits in enumerate(tc.RANGES):
        for name, src in (("limits", tc.range_source(ch)), ("mosaic", tc.sources(ch)["mosaic"])):
            for mname, mask in tc.CHANNEL_MASKS.items():
                check(src, tc.RANGE, limits, f"{name} {k} mask {mname}", mask)


@pytest.mark.parametrize("ch", CHANNELS)
def test_perceptible(ch):
    src = tc.perceptible_source(ch)
    for eps in tc.EPSILONS:
        for mname, mask in tc.CHANNEL_MASKS.items():
            check(src, tc.PERCEPTIBLE, (eps,), f"eps {eps:g} mask {mname}", mask)
