"""The oracle against the real reference, bit for bit, for the level and stretch operators: LevelImage, LevelizeImage,
MinMaxStretchImage, AutoLevelImage, ContrastStretchImage, NormalizeImage, LinearStretchImage and GammaImage on 1-4
channels, under the default channel mask and `-channel` selections (one that leaves channel 0 out, and RGBA, which keeps
every trait at its default but is not AllChannels).  Inputs (level_cases.sources / gray_sources) mix noise, alpha
blocks, HDR values, gray pixels, NaN / +-inf, black, white and flat images, rows that start with NaN, an all-NaN image,
1xN / Nx1 lines and gray-valued / bilevel sRGB images (ContrastStretch's GRAY re-layout).  Each stored result pins the
pixels, the channel count the cache is left with and the "histogram:*" property.

The reference's results are stored in tests/golden/level_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_level_vs_ref.py

where oracle/_ref is built."""
import pytest

import level_cases as lc
from level_cases import reference, result_key

CHANNELS = [1, 2, 3, 4]


def check(src, op, case, a=0.0, b=0.0, g=1.0, mask=-1):
    got = result_key(*lc.orc_run(src, op, a, b, g, mask))
    want = reference(case, lambda: lc.ref_run(src, op, a, b, g, mask))
    assert got == want, case


@pytest.mark.parametrize("ch", CHANNELS)
def test_level(ch):
    src = lc.sources(ch)["mosaic"]
    for k, (black, white, gamma) in enumerate(lc.LEVEL_ARGS):
        check(src, lc.LEVEL, f"level {k}", black, white, gamma)
        check(src, lc.LEVELIZE, f"levelize {k}", black, white, gamma)
    for name, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.LEVEL, f"level mask {name}", 1000.0, 60000.0, 2.2, mask)
        check(src, lc.LEVELIZE, f"levelize mask {name}", 1000.0, 60000.0, 0.45, mask)


@pytest.mark.parametrize("ch", CHANNELS)
def test_gamma(ch):
    src = lc.sources(ch)["mosaic"]
    for gamma in lc.GAMMAS:
        check(src, lc.GAMMA, f"gamma {gamma}", g=gamma)
    for name, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.GAMMA, f"gamma mask {name}", g=2.2, mask=mask)


@pytest.mark.parametrize("ch", CHANNELS)
def test_minmax_stretch(ch):
    for name, src in lc.sources(ch).items():
        check(src, lc.AUTO_LEVEL, f"auto level {name}")
        for mname, mask in lc.CHANNEL_MASKS.items():
            if mask >= 0:
                check(src, lc.AUTO_LEVEL, f"auto level {name} mask {mname}", mask=mask)
    src = lc.sources(ch)["mosaic"]
    for k, (black, white, gamma) in enumerate(lc.MINMAX_ARGS):
        check(src, lc.MINMAX, f"minmax {k}", black, white, gamma)
        check(src, lc.MINMAX, f"minmax {k} mask RGBA", black, white, gamma, 0x17)


@pytest.mark.parametrize("ch", CHANNELS)
def test_contrast_stretch(ch):
    for name, src in lc.sources(ch).items():
        n = src.shape[0] * src.shape[1]
        check(src, lc.NORMALIZE, f"normalize {name}")
        for k, (black, white) in enumerate(lc.stretch_points(n)):
            check(src, lc.CONTRAST_STRETCH, f"stretch {name} {k}", black, white)
    src = lc.sources(ch)["mosaic"]
    n = src.shape[0] * src.shape[1]
    for mname, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.NORMALIZE, f"normalize mask {mname}", mask=mask)
        check(src, lc.CONTRAST_STRETCH, f"stretch mask {mname}", 0.1 * n, 0.95 * n, mask=mask)


@pytest.mark.parametrize("ch", [3, 4])
def test_contrast_stretch_gray_relayout(ch):
    """Gray-valued and bilevel sRGB images are re-laid out to GRAY (plus alpha) before the histogram; a pixel one float
    step off gray is not."""
    for name, src in lc.gray_sources(ch).items():
        n = src.shape[0] * src.shape[1]
        check(src, lc.NORMALIZE, f"normalize {name}")
        check(src, lc.CONTRAST_STRETCH, f"stretch {name}", 0.05 * n, 0.9 * n)
        for mname, mask in lc.CHANNEL_MASKS.items():
            if mask >= 0:
                check(src, lc.NORMALIZE, f"normalize {name} mask {mname}", mask=mask)


@pytest.mark.parametrize("ch", CHANNELS)
def test_linear_stretch(ch):
    for name, src in lc.sources(ch).items():
        n = src.shape[0] * src.shape[1]
        for k, (black, white) in enumerate(lc.stretch_points(n)):
            check(src, lc.LINEAR_STRETCH, f"linear {name} {k}", black, white)
    src = lc.sources(ch)["mosaic"]
    n = src.shape[0] * src.shape[1]
    for mname, mask in lc.CHANNEL_MASKS.items():
        check(src, lc.LINEAR_STRETCH, f"linear mask {mname}", 0.02 * n, 0.01 * n, mask=mask)


@pytest.mark.parametrize("ch", [3, 4])
def test_identify_gray(ch):
    """The oracle's IdentifyImageGray scan agrees with the re-layout the reference takes (channel count after Normalize)."""
    for name, src in {**lc.gray_sources(ch), "mosaic": lc.sources(ch)["mosaic"]}.items():
        h, w, _ = src.shape
        kind = lc.oracle().orc_identify_gray(lc.util.P(src.copy()), w, h, ch)
        want = reference(f"normalize {name}", lambda: lc.ref_run(src, lc.NORMALIZE)) if name != "mosaic" else None
        if want is not None:
            assert int(want.split("/")[1]) == (ch - 2 if kind else ch), name
        assert kind == {"gray": 1, "bilevel": 2, "near gray": 0, "mosaic": 0}[name], name
