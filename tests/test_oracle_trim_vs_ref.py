"""GetImageBoundingBox and TrimImage on the host: for every case of trim_cases, row summaries built by a NumPy statement
of IsFuzzyEquivalencePixelInfo (float64, no contraction, so the same bits as the reference's double arithmetic), run
through mb200_bounding_box_from_rows, give the reference's box; mb200_trim_plan, with the plan's map applied by NumPy
indexing, gives TrimImage's size, page and pixels bit for bit -- with no device.  The reference's results are stored in
tests/golden/trim_digests.json; re-record them with

    MB200_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_trim_vs_ref.py

where oracle/_ref is built.  tests/test_gpu_trim.py checks the kernel against the same digests."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import geometry_cases as gc
import trim_cases as tc
from util import ROOT

CASES = tc.cases()
TRIMS = sorted(n for n, c in CASES.items() if c["trim"])


def host_box(case):
    import imagemagick_b200 as im
    src = case["src"]
    h, w, _ = src.shape
    rows = np.ascontiguousarray(tc.row_summaries(src, case["fuzz"], case["colorspace"]))
    box = im.Page()
    warning = C.c_int(-1)
    im._lib.check(im._lib.load().mb200_bounding_box_from_rows(rows.ctypes.data, w, h, im.trim_edges(case["edges"]),
                                                               C.byref(box), C.byref(warning)))
    return box, warning.value


def host_plan(case, box):
    import imagemagick_b200 as im
    h, w, _ = case["src"].shape
    page = im.Page(*case["page"])
    size = None if case["min_size"] is None else (C.c_size_t * 2)(*case["min_size"])
    plan = im.GeometryParams()
    rc = im._lib.load().mb200_trim_plan(w, h, C.byref(page), C.byref(box), case["gravity"], size, C.byref(plan))
    return rc, plan


@pytest.mark.parametrize("name", sorted(CASES))
def test_bounding_box_matches_reference(name):
    case = CASES[name]
    want = tc.box_reference(name, case)
    box, warning = host_box(case)
    assert tc.box_key((box.width, box.height, box.x, box.y), warning) == want, name


@pytest.mark.parametrize("name", TRIMS)
def test_trim_plan_matches_reference(name):
    import imagemagick_b200 as im
    case = CASES[name]
    want = tc.trim_reference(name, case)
    box, _ = host_box(case)
    rc, plan = host_plan(case, box)
    if tc.zero_box(tc.box_reference(name, case)) or rc == im._lib.EUNSUPPORTED:
        # a zero box (the reference's transparent 1x1 clone) or a box the crop declines (a 1x1 image without a mismatch
        # gives x = y = 1; the reference's CropImage warns)
        assert tc.declined_by_reference(tc.box_reference(name, case), want), want
        assert rc == im._lib.EUNSUPPORTED
        return
    assert rc == 0, (name, im._lib.load().mb200_last_error())
    got = gc.apply_plan(case["src"], plan)
    assert f"{gc.plan_key_prefix(plan)}/{got.shape[2]}/{gc.bits_digest(got)}/0" == want, name


def test_single_column_width_two():
    """The final `width -= x - 1` in size_t (attribute.c:558): a one-column image whose column differs gives width 2."""
    import imagemagick_b200 as im
    rows = np.zeros((5, 4), np.uint32)
    rows[2] = (1, 0, 1, 0)                            # row 2 mismatches the top-left and bottom-left pixels
    box = im.Page()
    assert im._lib.load().mb200_bounding_box_from_rows(rows.ctypes.data, 1, 5, -1, C.byref(box), None) == 0
    assert (box.width, box.height, box.x, box.y) == (2, 1, 0, 2)


def test_target3_rule_reads_the_width_the_row_started_with():
    """A row whose only mismatch is against the bottom-right pixel sets the height only when that x is below the width
    the rows above left (attribute.c:529-535)."""
    import imagemagick_b200 as im
    lib = im._lib.load()
    w = 10
    rows = np.zeros((6, 4), np.uint32)
    rows[1] = (w - 2, 5, 0, 0)                        # x 2..4 on row 1: width 4
    rows[4] = (0, 0, 0, w - 3)                        # target 3 first mismatches at x = 3 < 4: height 4
    box = im.Page()
    assert lib.mb200_bounding_box_from_rows(rows.ctypes.data, w, 6, -1, C.byref(box), None) == 0
    assert (box.width, box.height, box.x, box.y) == (3, 4, 2, 1)
    rows[4] = (0, 0, 0, w - 4)                        # x = 4 is not below the width: no height, a zero box
    assert lib.mb200_bounding_box_from_rows(rows.ctypes.data, w, 6, -1, C.byref(box), None) == 0
    assert (box.width, box.height, box.x, box.y) == (4, 0, 2, 1)


def test_argument_errors():
    import imagemagick_b200 as im
    lib = im._lib.load()
    rows = np.zeros((4, 4), np.uint32)
    box, plan, page = im.Page(), im.GeometryParams(), im.Page()
    EINVAL = im._lib.EINVAL
    assert lib.mb200_bounding_box_from_rows(None, 4, 4, -1, C.byref(box), None) == EINVAL
    assert lib.mb200_bounding_box_from_rows(rows.ctypes.data, 0, 4, -1, C.byref(box), None) == EINVAL
    assert lib.mb200_bounding_box_from_rows(rows.ctypes.data, 4, 0, -1, C.byref(box), None) == EINVAL
    for edges in (-2, 16):
        assert lib.mb200_bounding_box_from_rows(rows.ctypes.data, 4, 4, edges, C.byref(box), None) == EINVAL
    good = im.Page(2, 2, 1, 1)
    assert lib.mb200_trim_plan(4, 4, C.byref(page), C.byref(good), 10, None, C.byref(plan)) == EINVAL
    assert lib.mb200_trim_plan(4, 4, C.byref(page), C.byref(good), -1, None, C.byref(plan)) == EINVAL
    assert lib.mb200_trim_plan(4, 4, None, C.byref(good), 0, None, C.byref(plan)) == EINVAL
    assert lib.mb200_trim_plan(4, 4, C.byref(page), C.byref(im.Page(0, 2, 4, 0)), 0, None,
                               C.byref(plan)) == im._lib.EUNSUPPORTED
    assert lib.mb200_trim_plan(4, 4, C.byref(page), C.byref(good), 0, None, C.byref(plan)) == 0
    assert (plan.columns, plan.rows, plan.src_x, plan.src_y) == (2, 2, 1, 1)


def test_trim_plan_declines_where_the_crop_does():
    """The box of a 1x1 image without a mismatch is 1x1+1+1, a crop of zero area."""
    import imagemagick_b200 as im
    lib = im._lib.load()
    plan = im.GeometryParams()
    page, box = im.Page(), im.Page(1, 1, 1, 1)
    assert lib.mb200_trim_plan(1, 1, C.byref(page), C.byref(box), 0, None, C.byref(plan)) == im._lib.EUNSUPPORTED


def test_bad_options_are_rejected_before_the_device():
    """Checked on the host: no device is needed to get MB200_EINVAL."""
    import imagemagick_b200 as im
    lib = im._lib.load()
    src = np.zeros((3, 4, 5), np.float32)
    box = im.Page()
    for ch, cs, edges in ((5, tc.SRGB, -1), (3, tc.CMYK, -1), (4, tc.SRGB, 16), (4, tc.SRGB, -2), (6, tc.CMYK, -1)):
        options = im.TrimOptions(0.0, edges, cs)
        assert lib.mb200_bounding_box(src.ctypes.data, 4, 3, ch, C.byref(options), C.byref(box),
                                      None) == im._lib.EINVAL
    assert lib.mb200_bounding_box(src.ctypes.data, 4, 3, 4, None, C.byref(box), None) == im._lib.EINVAL


def test_trim_edges_parsing():
    import imagemagick_b200 as im
    assert im.trim_edges(None) == im.TRIM_EDGES_UNSET
    assert im.trim_edges("") == 0
    assert im.trim_edges("North,SOUTH") == im.TrimEdgeNorth | im.TrimEdgeSouth
    assert im.trim_edges(" north,west ") == 0          # tokens are not stripped (StringToken)
    assert im.trim_edges("West,nowhere,EAST") == im.TrimEdgeWest | im.TrimEdgeEast



def test_trim_harness_declines_without_a_device():
    """trim_harness (ld --wrap build of the unmodified reference) without a device: both wraps decline before touching
    the device and return exactly what the stock functions return."""
    import imagemagick_b200 as im
    exe = ROOT / "imagemagick_b200" / "lib" / "trim_harness"
    if not exe.exists():
        pytest.skip("trim_harness not built (needs the reference tree: python __graft_entry__.py)")
    if im._lib.load().mb200_device_count() != 0:
        pytest.skip("device present: the GPU variant is tests/test_gpu_trim.py::test_trim_harness_on_the_gpu")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-500:]
    assert "FAIL" not in p.stdout and "gpu hits 0" in p.stdout
