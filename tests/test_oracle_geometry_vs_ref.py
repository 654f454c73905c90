"""The orientation and crop operators on the host: for every case of geometry_cases, the planner (mb200_geometry_plan)
gives the reference's output columns, rows and page, and its map, applied with NumPy indexing, gives the reference's
pixels bit for bit -- with no device.  The declines are the reference's GeometryDoesNotContainImage outcomes and its
clones.  The reference's results are stored in tests/golden/geometry_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_geometry_vs_ref.py

where oracle/_ref is built.  tests/test_gpu_geometry.py checks the kernel against the same digests."""
import ctypes as C
import subprocess

import pytest

import geometry_cases as gc
from util import ROOT

CASES = gc.cases()
DECLINES = gc.declines()


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_matches_reference(name):
    case = CASES[name]
    want = gc.reference_of(name, case)
    assert want != "none", name
    p = gc.plan(case)
    assert gc.plan_key_prefix(p) == "/".join(want.split("/")[:6]), name
    got = gc.apply_plan(case["src"], p)
    assert f"{got.shape[2]}/{gc.bits_digest(got)}" == "/".join(want.split("/")[6:]), name


@pytest.mark.parametrize("name", sorted(DECLINES))
def test_declines(name):
    """MB200_EUNSUPPORTED from the planner and from the operator, with no device touched; the reference answers these
    with its own 1x1 transparent image, no image, or a clone."""
    import imagemagick_b200 as im
    case = DECLINES[name]
    want = gc.reference_of(name, case)
    if case["op"] == gc.CROP and "zero area" not in name:
        assert want.startswith("1/1/"), want           # the reference's transparent pixel
    elif case["op"] == gc.AUTO_ORIENT or case["op"] == gc.ROTATE:
        assert want.split("/")[:2] == ["33", "17"], want  # a clone
    else:
        assert want == "none", want
    with pytest.raises(im.MagickB200Error) as e:
        gc.plan(case)
    assert e.value.code == im._lib.EUNSUPPORTED
    with pytest.raises(im.MagickB200Error) as e:
        gc.run_lib(case)
    assert e.value.code == im._lib.EUNSUPPORTED


def test_plan_argument_errors():
    import imagemagick_b200 as im
    lib = im._lib.load()
    plan = im.GeometryParams()
    page = im.Page()
    args = (C.c_long * 4)(1, 1, 0, 0)
    assert lib.mb200_geometry_plan(8, 10, 10, C.byref(page), args, C.byref(plan)) == im._lib.EINVAL
    assert lib.mb200_geometry_plan(gc.FLIP, 0, 10, C.byref(page), args, C.byref(plan)) == im._lib.EINVAL
    assert lib.mb200_geometry_plan(gc.CROP, 10, 10, C.byref(page), None, C.byref(plan)) == im._lib.EINVAL


def test_plans_that_do_not_fit_the_source_are_rejected():
    """mb200_geometry_image checks a caller's plan against the source before anything is staged."""
    import numpy as np

    import imagemagick_b200 as im
    lib = im._lib.load()
    src = np.zeros((4, 5, 4), np.float32)
    dst = np.zeros(64, np.float32)
    for fields in (dict(map=0, columns=6, rows=4), dict(map=4, columns=5, rows=4), dict(map=8, columns=1, rows=1),
                   dict(map=0, columns=3, rows=2, src_x=3), dict(map=0, columns=5, rows=4, roll_x=5),
                   dict(map=6, columns=4, rows=5, roll_y=1), dict(map=0, columns=2, rows=2, src_y=-1)):
        p = im.GeometryParams(**fields)
        assert lib.mb200_geometry_image(src.ctypes.data, 5, 4, 4, dst.ctypes.data, C.byref(p)) == im._lib.EINVAL, fields
    p = im.GeometryParams(map=0, columns=1, rows=1)
    assert lib.mb200_geometry_image(src.ctypes.data, 5, 4, 6, dst.ctypes.data, C.byref(p)) == im._lib.EINVAL


def test_rotate_image_still_refuses_integral_angles():
    """Integral rotations have their own entry point; RotateImage's planner keeps declining them."""
    import imagemagick_b200 as im
    plan = im.DistortParams()
    for degrees in (90.0, 180.0, 270.0, -90.0):
        assert im._lib.load().mb200_rotate_plan(degrees, 10, 10, 0, 0, C.byref(plan)) == im._lib.EUNSUPPORTED


def test_geometry_harness_declines_without_a_device():
    """geometry_harness (ld --wrap build of the unmodified reference) without a device: every new wrapped entry point
    declines before touching the device and returns exactly what the stock function returns."""
    import imagemagick_b200 as im
    exe = ROOT / "imagemagick_b200" / "lib" / "geometry_harness"
    if not exe.exists():
        pytest.skip("geometry_harness not built (needs the reference tree: python __graft_entry__.py)")
    if im._lib.load().mb200_device_count() != 0:
        pytest.skip("device present: the GPU variant is tests/test_gpu_geometry.py::test_geometry_harness_on_the_gpu")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-500:]
    assert "FAIL" not in p.stdout and "gpu hits 0" in p.stdout
