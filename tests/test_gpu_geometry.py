"""The orientation and crop operators on the GPU against the reference's stored results (tests/golden/
geometry_digests.json, the cases of geometry_cases).  On every case the device entry point gives the reference's pixels
(every bit: NaN payloads, -0, denormals), size and page; on the size grid of the 3-, 4- and 5-channel layouts the host
entry point does too.  The size grid's outputs are also written inside a sentinel-filled guard band that must stay
untouched: 16-byte aligned for every layout, and misaligned by one word for 2 and 4 channels, which moves those to the
word-by-word path.  Also: one geometry_launches per call, a 16384 x 16384 RGBA transpose and 90-degree rotation (4 GiB
each way: byte offsets beyond 32 bits), and the MagickCore shim's geometry_harness."""
from __future__ import annotations

import ctypes as C
import subprocess

import numpy as np
import pytest

import geometry_cases as gc
import imagemagick_b200 as im
from imagemagick_b200 import _lib
from util import ROOT, get_option

pytestmark = pytest.mark.gpu
CASES = gc.cases()
GRID = [n for n in sorted(CASES) if "page" not in n and not n.startswith(("roll ", "auto-orient"))
        or n.startswith("roll 5,-3")]
SENTINEL = 0x7FBADBAD                # a NaN payload no case produces
GUARD = 1024                         # words on each side


def guarded_run(name, misalign):
    """mb200_geometry_image_dev into the middle of a sentinel-filled buffer: the guard words stay, and the output is the
    reference's."""
    import torch
    case = CASES[name]
    p = gc.plan(case)
    src = torch.from_numpy(np.ascontiguousarray(case["src"])).cuda()
    h, w, ch = case["src"].shape
    n = p.columns * p.rows * ch
    buf = torch.full((2 * GUARD + n + misalign,), SENTINEL, dtype=torch.int32, device="cuda")
    dst = buf[GUARD + misalign: GUARD + misalign + n]
    assert _lib.load().mb200_geometry_image_dev(src.data_ptr(), w, h, ch, dst.data_ptr(), C.byref(p), None) == 0
    words = buf.cpu().numpy().view(np.uint32)
    assert (words[:GUARD + misalign] == SENTINEL).all() and (words[GUARD + misalign + n:] == SENTINEL).all(), name
    got = words[GUARD + misalign: GUARD + misalign + n].view(np.float32).reshape(p.rows, p.columns, ch)
    assert f"{ch}/{gc.bits_digest(got)}" == "/".join(gc.reference_of(name, case).split("/")[6:]), name


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_reference(name):
    case = CASES[name]
    assert gc.key(gc.run_lib(case, device=True)) == gc.reference_of(name, case), name
    if name in GRID:
        guarded_run(name, 0)


@pytest.mark.parametrize("name", [n for n in GRID if CASES[n]["layout"] in ("rgb", "rgba", "cmyka")])
def test_host_matches_reference(name):
    case = CASES[name]
    assert gc.key(gc.run_lib(case, device=False)) == gc.reference_of(name, case), name


@pytest.mark.parametrize("name", [n for n in GRID if CASES[n]["layout"] in ("ga", "rgba", "cmyk")])
def test_misaligned_output_takes_the_word_path(name):
    guarded_run(name, 1)


def test_one_launch_per_call():
    before = get_option("geometry_launches")
    for name in ("transpose rgba 257x129", "flip rgba 257x129", "roll 5,-3 rgba 257x129"):
        gc.run_lib(CASES[name], device=True)
    assert get_option("geometry_launches") - before == 3


def test_16384_rgba_transpose_and_rotate():
    """4 GiB each way: byte offsets beyond 32 bits.  Every source word is its own element index, so the expected result
    of a pure permutation is known everywhere: the whole output is compared on the device with torch's permute / flip,
    and sampled rows (the first, the last and rows in between) with NumPy's transpose / rot90 of the same pattern."""
    import torch
    n = 16384
    src = torch.arange(n * n * 4, dtype=torch.int32, device="cuda").view(n, n, 4)
    image = im.Image(src.view(torch.float32))
    rows = [0, 1, 5000, 8191, 8192, 12345, n - 2, n - 1]
    for op in ("transpose", "rotate 90"):
        out = im.TransposeImage(image) if op == "transpose" else im.IntegralRotateImage(image, 1)
        assert (out.columns, out.rows) == (n, n)
        got = out.pixels.view(torch.int32)
        want = src.permute(1, 0, 2) if op == "transpose" else src.flip(0).permute(1, 0, 2)
        assert torch.equal(got, want), op
        for y in rows:                                   # output row y is source column y
            col = (np.arange(n, dtype=np.int64)[:, None] * n + y) * 4 + np.arange(4)     # src[:, y] as indices
            expect = col if op == "transpose" else col[::-1]                          # clockwise: rows reversed
            assert np.array_equal(got[y].cpu().numpy(), expect.astype(np.int32)), (op, y)
        del out, got, want
    del image, src
    torch.cuda.empty_cache()


def test_geometry_harness_on_the_gpu():
    """Each new wrapped entry point, AutoOrientImage and CropImageToTiles through the shim against __real_ (pixels,
    size, page, type, orientation, channels), and a Resize -> CropImageToTiles -> Flop -> Blur chain both ways."""
    exe = ROOT / "imagemagick_b200" / "lib" / "geometry_harness"
    if not exe.exists():
        pytest.skip("geometry_harness not built (needs the reference headers)")
    p = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(p.stdout)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "FAIL" not in p.stdout and "gpu hits" in p.stdout and "gpu hits 0" not in p.stdout
