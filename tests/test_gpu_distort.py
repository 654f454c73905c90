"""DistortImage / RotateImage on the GPU against the reference's stored results (tests/golden/distort_digests.json, the
cases of distort_cases): the device and the host entry points give the reference's pixels, geometry and page bit for
bit.  Also: identical bits over three runs and one distort_launches per call, an unaligned device buffer, a many-CTA
rotation and perspective, and the declines (MB200_EUNSUPPORTED with dst untouched)."""
from __future__ import annotations

import numpy as np
import pytest

import distort_cases as dc
import imagemagick_b200 as im
from imagemagick_b200 import _lib
from util import get_option, make_image

pytestmark = pytest.mark.gpu
CASES = dc.cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_reference(name):
    src, kw = CASES[name]
    assert dc.key(dc.run_lib(src, device=True, **kw)) == dc.reference(name, lambda: dc.run_ref(src, **kw)), name


@pytest.mark.parametrize("name", [n for n in sorted(CASES) if n.endswith("ch4") or n.startswith("rotate")])
def test_host_matches_reference(name):
    src, kw = CASES[name]
    assert dc.key(dc.run_lib(src, device=False, **kw)) == dc.reference(name, lambda: dc.run_ref(src, **kw)), name


def test_repeatable_and_one_launch():
    src = make_image(1000, 700, 4, seed=11, kind="alpha_blocks")
    runs = []
    before = get_option("distort_launches")
    for _ in range(3):
        runs.append(dc.run_lib(src, dc.ROTATE, [30.0], bg=dc.GRAY_BG, device=True)[0])
    assert get_option("distort_launches") - before == 3
    assert all(np.array_equal(r.view(np.uint32), runs[0].view(np.uint32)) for r in runs)


def test_unaligned_device_buffer():
    import torch
    src = make_image(61, 47, 3, seed=4)
    flat = torch.empty(src.size + 1, dtype=torch.float32, device="cuda")
    flat[1:] = torch.from_numpy(src.ravel()).cuda()
    image = im.Image.__new__(im.Image)
    image.pixels, image.colorspace, image.page = flat[1:].view(47, 61, 3), im.sRGBColorspace, (0, 0)
    got = im.DistortImage(image, dc.SRT, [0.8, 33.0], True).pixels.cpu().numpy()
    want = dc.run_lib(src, dc.SRT, [0.8, 33.0], bestfit=True, device=True)[0]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("kw", [dict(filter=1), dict(virtual_pixel=6), dict(virtual_pixel=4), dict(interpolate=8)])
def test_declines_leave_dst_untouched(kw):
    import ctypes as C
    import torch
    src = torch.from_numpy(make_image(20, 16, 4, seed=2)).cuda()
    image = im.Image(src)
    plan = im.DistortPlan(image, dc.SRT, [25.0])
    dst = torch.full((plan.rows, plan.columns, 4), 7.0, device="cuda")
    opts = im.ResampleOptions(filter=kw.get("filter", 0), virtual_pixel=kw.get("virtual_pixel", 0),
                              interpolate=kw.get("interpolate", 0))
    rc = _lib.load().mb200_distort_image_dev(src.data_ptr(), 20, 16, 4, dst.data_ptr(), C.byref(plan), C.byref(opts),
                                             None)
    assert rc == _lib.EUNSUPPORTED
    assert bool((dst == 7.0).all())


def test_horizon_without_alpha_declined():
    src = make_image(37, 29, 3, seed=5)
    with pytest.raises(im.MagickB200Error) as e:
        dc.run_lib(src, *dc.MAPS["horizon"], bestfit=True, device=True)
    assert e.value.code == _lib.EUNSUPPORTED
