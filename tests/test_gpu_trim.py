"""GetImageBoundingBox and TrimImage on the GPU against the reference's stored results (tests/golden/trim_digests.json,
the cases of trim_cases).  On every case the device and the host entry points give the reference's box and warning, and
TrimImage gives its pixels (every bit), size and page, or declines where the reference answers with its 1x1 image.
Also: the trim's crop written inside a sentinel-filled guard band, a misaligned RGBA source (the word path of the scan),
one bounding_box_launches per box and one more geometry_launches per trim, and a 16384 x 16384 RGBA image (4 GiB: byte
offsets beyond 32 bits) with a known box, an image of 70 000 rows (the grid-stride loop over rows beyond the grid's
65 535), and the MagickCore shim's trim_harness."""
from __future__ import annotations

import ctypes as C
import subprocess

import numpy as np
import pytest

import geometry_cases as gc
import imagemagick_b200 as im
import trim_cases as tc
from imagemagick_b200 import _lib
from util import ROOT, get_option

pytestmark = pytest.mark.gpu
CASES = tc.cases()
TRIMS = sorted(n for n, c in CASES.items() if c["trim"])
SENTINEL = 0x7FBADBAD                # a NaN payload no case produces
GUARD = 1024                         # words on each side


def lib_box_key(case, device):
    box, warning = im.BoundingBoxWarning(tc.image(case, device), case["fuzz"], case["edges"])
    return tc.box_key(box, warning)


def lib_trim(case, device):
    return im.TrimImage(tc.image(case, device), case["fuzz"], case["edges"], case["min_size"], case["gravity"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_bounding_box_device_and_host_match_reference(name):
    case = CASES[name]
    want = tc.box_reference(name, case)
    assert lib_box_key(case, True) == want, name
    assert lib_box_key(case, False) == want, name


@pytest.mark.parametrize("name", TRIMS)
def test_trim_device_and_host_match_reference(name):
    case = CASES[name]
    want = tc.trim_reference(name, case)
    for device in (True, False):
        try:
            out = lib_trim(case, device)
        except im.MagickB200Error as e:
            # the reference's transparent 1x1 clone of a zero box, or its warned answer to a crop it rejects
            assert e.code == _lib.EUNSUPPORTED, name
            assert tc.declined_by_reference(tc.box_reference(name, case), want), want
            continue
        assert tc.lib_trim_key(out, device) == want, (name, device)


@pytest.mark.parametrize("name", ["rgba page canvas corners", "cmyka edges 'east,west' corners",
                                  "gray min size grow gravity 5 corners", "rgba 70x45 equal fuzz 0"])
def test_trim_into_a_guarded_buffer(name):
    """The trim's crop through mb200_geometry_image_dev into the middle of a sentinel-filled buffer: the guard words
    stay, and the output is the reference's."""
    import torch
    case = CASES[name]
    img = tc.image(case, True)
    box, _ = im.BoundingBoxWarning(img, case["fuzz"], case["edges"])
    page = im.Page(*case["page"])
    size = None if case["min_size"] is None else (C.c_size_t * 2)(*case["min_size"])
    plan = im.GeometryParams()
    h, w, ch = case["src"].shape
    assert _lib.load().mb200_trim_plan(w, h, C.byref(page), C.byref(im.Page(*box)), case["gravity"], size,
                                       C.byref(plan)) == 0
    n = plan.columns * plan.rows * ch
    buf = torch.full((2 * GUARD + n,), SENTINEL, dtype=torch.int32, device="cuda")
    dst = buf[GUARD: GUARD + n]
    assert _lib.load().mb200_geometry_image_dev(img.pixels.data_ptr(), w, h, ch, dst.data_ptr(), C.byref(plan),
                                                None) == 0
    words = buf.cpu().numpy().view(np.uint32)
    assert (words[:GUARD] == SENTINEL).all() and (words[GUARD + n:] == SENTINEL).all(), name
    got = words[GUARD: GUARD + n].view(np.float32).reshape(plan.rows, plan.columns, ch)
    assert f"{gc.plan_key_prefix(plan)}/{ch}/{gc.bits_digest(got)}/0" == tc.trim_reference(name, case), name


@pytest.mark.parametrize("name", ["rgba 70x45 corners fuzz 0", "rgba 257x129 special frame fuzz moderate",
                                  "rgba 40x600 special corners fuzz 0", "rgba transparent fuzz 0"])
def test_misaligned_rgba_source_takes_the_word_path(name):
    import torch
    case = CASES[name]
    src = np.ascontiguousarray(case["src"])
    h, w, ch = src.shape
    buf = torch.zeros(src.size + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(src.reshape(-1)).cuda()
    view = buf[1:]
    assert view.data_ptr() % 16 != 0
    options = im.TrimOptions(case["fuzz"], im.trim_edges(case["edges"]), case["colorspace"])
    box, warning = im.Page(), C.c_int(0)
    assert _lib.load().mb200_bounding_box_dev(view.data_ptr(), w, h, ch, C.byref(options), C.byref(box),
                                              C.byref(warning), None) == 0
    assert tc.box_key((box.width, box.height, box.x, box.y), warning.value) == tc.box_reference(name, case)


def test_launch_counts():
    case = CASES["rgba 70x45 corners fuzz 0"]
    img = tc.image(case, True)
    boxes, crops = get_option("bounding_box_launches"), get_option("geometry_launches")
    im.GetImageBoundingBox(img)
    assert (get_option("bounding_box_launches") - boxes, get_option("geometry_launches") - crops) == (1, 0)
    im.TrimImage(img)
    assert (get_option("bounding_box_launches") - boxes, get_option("geometry_launches") - crops) == (2, 1)


def test_16384_rgba_known_box():
    """4 GiB: byte offsets beyond 32 bits.  A background with equal corners, a block near the right edge and one pixel
    near the bottom-left: the box is known, and the trim is the slice of the source."""
    import torch
    n = 16384
    src = torch.full((n, n, 4), 1000.0, dtype=torch.float32, device="cuda")
    src[..., 3] = 65535.0
    src[9000:9101, 15000:16000, 0] = 40000.0
    src[16000, 3, 1] = 11000.0                  # within a fuzz of 20000, not of 0
    image = im.Image(src)
    before = get_option("bounding_box_launches")
    assert im.GetImageBoundingBox(image) == (16000 - 3, 16000 - 9000 + 1, 3, 9000)
    assert im.GetImageBoundingBox(image, fuzz=20000.0) == (15999 - 14999, 9100 - 8999, 15000, 9000)
    out = im.TrimImage(image)
    assert (out.columns, out.rows, out.page) == (15997, 7001, (3, 9000))
    assert torch.equal(out.pixels, src[9000:16001, 3:16000])
    assert get_option("bounding_box_launches") - before == 3
    del out, image, src
    torch.cuda.empty_cache()


def test_rows_beyond_the_grid():
    """70 000 rows of one gray column: more rows than the grid's y dimension (65 535), so CTAs take a second row through
    the grid-stride loop.  The box is known, and the host rule on NumPy summaries gives the same."""
    import torch
    h = 70000
    src = np.full((h, 1, 1), 30000.0, np.float32)
    src[66000, 0, 0] = 1000.0
    src[69000, 0, 0] = np.nan                   # equal to everything: no mismatch
    src[69500, 0, 0] = 50000.0
    box, warning = im.BoundingBoxWarning(im.Image(torch.from_numpy(src).cuda(), tc.SRGB))
    assert (box, warning) == ((2, 69500 - 65999, 0, 66000), False)
    rows = np.ascontiguousarray(tc.row_summaries(src, 0.0, tc.SRGB))
    host = im.Page()
    assert _lib.load().mb200_bounding_box_from_rows(rows.ctypes.data, 1, h, -1, C.byref(host), None) == 0
    assert (host.width, host.height, host.x, host.y) == box


def test_trim_harness_on_the_gpu():
    """Both wraps through the shim against __real_ (box, severity, pixels, size, page, type, channels), the zero box
    served with the reference's own 1x1 clone, and the declines falling back."""
    exe = ROOT / "imagemagick_b200" / "lib" / "trim_harness"
    if not exe.exists():
        pytest.skip("trim_harness not built (needs the reference headers)")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(p.stdout)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "FAIL" not in p.stdout and "gpu hits" in p.stdout and "gpu hits 0" not in p.stdout
