"""The oracle against the real reference, bit for bit, for TransformImageColorspace to and from the colourspaces that
change the channel layout: every direct leg (sRGB <-> GRAY, LinearGRAY, CMYK) with and without alpha, hops from one
space of each route family of the in-place legs in both directions, GRAY <-> CMYK and LinearGRAY <-> GRAY, reference
settings on the hops, and 1xN / Nx1 images.  Inputs mix noise, alpha blocks, HDR values, gray pixels, NaN / +-inf,
exact black and near-black samples (layout_cases.source).  Each stored result also pins the image type the reference
leaves (layout_cases.expected_type, which the MagickCore shim restates).

The reference's results are stored as digests in tests/golden/layout_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_layout_vs_ref.py

where oracle/_ref is built."""
import pytest

import layout_cases as lc
from layout_cases import reference
from util import digest, make_image

DIRECT = [(lc.SRGB, lc.GRAY), (lc.SRGB, lc.LINEAR_GRAY), (lc.GRAY, lc.SRGB), (lc.LINEAR_GRAY, lc.SRGB),
          (lc.SRGB, lc.CMYK), (lc.CMYK, lc.SRGB)]
BETWEEN = [(lc.GRAY, lc.CMYK), (lc.CMYK, lc.GRAY), (lc.LINEAR_GRAY, lc.GRAY), (lc.GRAY, lc.LINEAR_GRAY),
           (lc.CMYK, lc.LINEAR_GRAY), (lc.LINEAR_GRAY, lc.CMYK)]


def _id(pair):
    return f"{lc.NAMES[pair[0]]}-{lc.NAMES[pair[1]]}"


def check(src, from_cs, to_cs, case, settings=None):
    alpha = src.shape[2] != lc.channels(from_cs, False)
    got = lc.orc_layout(src, from_cs, to_cs, settings)
    assert got.shape[2] == lc.channels(to_cs, alpha)
    want, kind = reference(case, lambda: lc.ref_layout(src, from_cs, to_cs, settings)).split("/")
    assert digest(got) == want, case
    if to_cs in lc.LAYOUT:
        assert int(kind) == lc.expected_type(to_cs, alpha), case


@pytest.mark.parametrize("alpha", [False, True])
@pytest.mark.parametrize("pair", DIRECT + BETWEEN, ids=_id)
def test_layout_legs(pair, alpha):
    from_cs, to_cs = pair
    check(lc.source(from_cs, alpha), from_cs, to_cs, "mosaic")


@pytest.mark.parametrize("alpha", [False, True])
@pytest.mark.parametrize("pair", DIRECT, ids=_id)
def test_layout_legs_lines(pair, alpha):
    from_cs, to_cs = pair
    for w, h in [(1, 29), (31, 1)]:
        img = make_image(w, h, lc.channels(from_cs, alpha), seed=w + 2 * h, kind="hdr")
        check(img, from_cs, to_cs, f"{w}x{h}")


@pytest.mark.parametrize("layout", lc.LAYOUT, ids=lambda c: lc.NAMES[c])
@pytest.mark.parametrize("space", lc.HOP_SPACES, ids=lambda c: lc.NAMES[c])
def test_hops(space, layout):
    """space -> sRGB -> layout and back, through the in-place legs; the source is the raw mosaic tagged `space`."""
    for alpha in (False, True):
        check(lc.source(space, alpha, seed=21), space, layout, f"to a{int(alpha)}")
        check(lc.source(layout, alpha, seed=23), layout, space, f"from a{int(alpha)}")


@pytest.mark.parametrize("layout", lc.LAYOUT, ids=lambda c: lc.NAMES[c])
def test_hop_settings(layout):
    """The image settings of the in-place legs reach the hops: a D50 reference white (Lab, LCHab) and Log's film
    settings."""
    for space, settings in [(lc.LAB, {"color:illuminant": "D50"}), (lc.LCHAB, {"color:illuminant": "A"}),
                            (lc.LOG, {"reference-white": "700", "film-gamma": "0.5"})]:
        check(lc.source(space, True, w=19, seed=31), space, layout, f"to {space}", settings)
        check(lc.source(layout, True, w=19, seed=33), layout, space, f"from {space}", settings)
