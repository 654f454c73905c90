"""DistortImage / RotateImage on the host: the planner (mb200_distort_plan / mb200_rotate_plan) gives the reference's
output columns, rows and page for every case of distort_cases, with no device; integral rotations and a
"distort:scale" below 0.1 are refused as the reference refuses them.  The reference's results are stored in
tests/golden/distort_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_distort_vs_ref.py

where oracle/_ref is built.  tests/test_gpu_distort.py checks the pixels against the same digests."""
import ctypes as C

import pytest

import distort_cases as dc

CASES = dc.cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_matches_reference_geometry(name):
    src, kw = CASES[name]
    want = dc.reference(name, lambda: dc.run_ref(src, **kw))
    assert want != "none", name
    got = dc.plan_geometry(src, **kw)
    assert "/".join(map(str, got)) == "/".join(want.split("/")[:4]), name


@pytest.mark.parametrize("degrees", [0.0, 90.0, -90.0, 180.0, 270.0, 360.0, 450.0, -1e-15])
def test_integral_rotations_refused(degrees):
    import imagemagick_b200 as im
    plan = im.DistortParams()
    assert im._lib.load().mb200_rotate_plan(degrees, 10, 10, 0, 0, C.byref(plan)) == im._lib.EUNSUPPORTED


def test_scale_below_tenth_rejected():
    import imagemagick_b200 as im
    src = dc.sources(3)["noise"]
    assert dc.reference("scale 0.09 rejected", lambda: dc.run_ref(src, dc.SRT, [20.0], scale=0.09)) == "none"
    with pytest.raises(im.MagickB200Error):
        im.DistortPlan(im.Image(src), dc.SRT, [20.0], scale=0.09)


@pytest.mark.parametrize("method,args", [(dc.SRT, []), (dc.SRT, [1, 2, 3, 4, 5, 6, 7, 8]), (dc.SRT, [0.0, 10.0]),
                                         (dc.AFFINE, [1, 2, 3]), (dc.AFFINE_PROJECTION, [1, 2, 3, 4, 5]),
                                         (dc.PERSPECTIVE_PROJECTION, [1, 2, 3]),
                                         (dc.RIGID_AFFINE, [3.0, 2.0, 5.5, 7.25])])
def test_argument_errors(method, args):
    """The reference's argument errors (RigidAffine's 4x4 solve is singular with one pair): no image there,
    MB200_EINVAL here."""
    import imagemagick_b200 as im
    src = dc.sources(3)["noise"]
    assert dc.reference(f"error {method} {args}", lambda: dc.run_ref(src, method, args)) == "none"
    with pytest.raises(im.MagickB200Error) as e:
        im.DistortPlan(im.Image(src), method, args)
    assert e.value.code == im._lib.EINVAL


def test_scale_zero_rejected():
    """distort:scale=0 is below 0.1, as the reference rejects it; an unset scale is a separate case."""
    import imagemagick_b200 as im
    src = dc.sources(3)["noise"]
    assert dc.reference("scale 0 rejected", lambda: dc.run_ref(src, dc.SRT, [20.0], scale=0.0)) == "none"
    with pytest.raises(im.MagickB200Error) as e:
        im.DistortPlan(im.Image(src), dc.SRT, [20.0], scale=0.0)
    assert e.value.code == im._lib.EINVAL


@pytest.mark.parametrize("method", [9, 10, 11, 14, 16, 18])
def test_other_methods_declined(method):
    """Polynomial, Arc, Polar, Barrel, Shepards and Resize are left to the reference: MB200_EUNSUPPORTED, no device."""
    import imagemagick_b200 as im
    with pytest.raises(im.MagickB200Error) as e:
        im.DistortPlan(im.Image(dc.sources(3)["noise"]), method, [1.0, 2.0, 3.0, 4.0])
    assert e.value.code == im._lib.EUNSUPPORTED


def test_cmyk_declined():
    """A CMYK image's fourth channel is black, not alpha: declined before anything is resampled."""
    import imagemagick_b200 as im
    image = im.Image(dc.sources(4)["noise"], im.CMYKColorspace)
    with pytest.raises(im.MagickB200Error) as e:
        im.DistortImage(image, dc.SRT, [30.0])
    assert e.value.code == im._lib.EUNSUPPORTED
    with pytest.raises(im.MagickB200Error):
        im.RotateImage(image, 30.0)


def test_alpha_gained_inside_distort_declined():
    """A background or matte colour with an alpha trait on an image without alpha, outside the virtual-pixel methods
    that add the alpha first: the reference adds it inside DistortImage, which is left to the reference."""
    import imagemagick_b200 as im
    image = im.Image(dc.sources(3)["noise"])
    for kw in (dict(background=(0.0, 0.0, 0.0, 0.0)), dict(matte_color=(1.0, 2.0, 3.0, 4.0))):
        with pytest.raises(im.MagickB200Error) as e:
            im.DistortImage(image, dc.SRT, [30.0], **kw)
        assert e.value.code == im._lib.EUNSUPPORTED
