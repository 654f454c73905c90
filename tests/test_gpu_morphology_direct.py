"""MorphologyImage's directly applied methods, Distance and Voronoi, on the GPU (csrc/morph_direct.cu: the two sweeps
of MorphologyPrimitiveDirect as skewed wavefronts), through the device and the host-buffer entry points:

- bit for bit against the reference's stored results (tests/golden/direct_digests.json, the digests
  test_oracle_direct_vs_ref.py pins the oracle to) over the same kernels and inputs;
- bit for bit against the oracle on images of many bands and several CTAs per channel, up to 4096^2 RGBA;
- three runs of one call give the same bits (a race between the bands would show here);
- exactly two launches per call (forward, reverse), an unaligned device buffer, and the declines.

The argument checks at the end run without a device."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import direct_cases as dc
import imagemagick_b200 as im
from imagemagick_b200 import _lib
from util import digest, get_option, make_image

CHANNELS = [1, 2, 3, 4]


def gpu_key(img, method, kernel):
    out = im.MorphologyDirectImage(img, method, kernel)
    pixels = out.pixels.cpu().numpy() if out.on_device else out.pixels
    return dc.result_key(digest(dc.kernel_values(*dc.head_kernel(kernel))), pixels, dc.alpha_trait(method, img.channels))


def run_both(src, method, kernel):
    """The device and the host result of MorphologyDirectImage, as numpy arrays."""
    import torch
    dev = im.MorphologyDirectImage(im.Image(torch.from_numpy(src.copy()).cuda()), method, kernel).pixels.cpu().numpy()
    host = im.MorphologyDirectImage(im.Image(src.copy()), method, kernel).pixels
    return dev, host


@pytest.mark.gpu
@pytest.mark.parametrize("method", [dc.DISTANCE, dc.VORONOI])
@pytest.mark.parametrize("ch", CHANNELS)
def test_against_reference(ch, method):
    """Every case of test_oracle_direct_vs_ref.py's test_distance / test_voronoi, on the device and from host buffers."""
    import torch
    test = f"test_oracle_direct_vs_ref.py::test_{'distance' if method == dc.DISTANCE else 'voronoi'}[{ch}]"
    for name, src in dc.sources(ch).items():
        for kernel in dc.KERNELS:
            case = f"{kernel} {name}"
            if method == dc.VORONOI and ch in (1, 3):
                with pytest.raises(im.MagickB200Error) as e:
                    im.MorphologyDirectImage(im.Image(torch.from_numpy(src).cuda()), method, kernel)
                assert e.value.code == _lib.EUNSUPPORTED
                continue
            want = dc.reference(case, lambda: dc.ref_key(src, method, kernel), test=test)
            assert gpu_key(im.Image(torch.from_numpy(src.copy()).cuda()), method, kernel) == want, (case, "device")
            assert gpu_key(im.Image(src.copy()), method, kernel) == want, (case, "host")


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,ch", [(300, 257, 4), (77, 130, 2), (1000, 40, 3), (33, 1000, 1), (5, 200, 4)])
def test_many_bands(w, h, ch):
    """Images of several 32-row bands per channel, against the oracle: kernels with 1-4 rows above the origin, wide
    reaches to the right and left, and a single-row kernel (rows independent)."""
    for kind, src in (("shapes", dc.shapes(w, h, ch, seed=w + h)), ("specials", dc.specials(w, h, ch, seed=w)),
                      ("nan inf", dc.nan_inf(w, h, ch, seed=h))):
        for kernel in ("Euclidean", "Euclidean:4", "Chebyshev:2", "4x3+1+2:10,20,-,5 0,-,7,30 8,9,3,2",
                       "5x2+4+0:9,8,7,6,5 1,-,2,-,3", "5x1+3+0:300,200,0,100,400"):
            for method in (dc.DISTANCE, dc.VORONOI) if ch in (2, 4) else (dc.DISTANCE,):
                want = dc.orc_run(src, method, kernel)[0]
                for got in run_both(src, method, kernel):
                    assert digest(got) == digest(want), (kind, kernel, method)


@pytest.mark.gpu
def test_4096_rgba_against_oracle():
    import torch
    src = dc.shapes(4096, 4096, 4, seed=77)
    src[::61, ::53, 1] = np.nan
    img = im.Image(torch.from_numpy(src).cuda())
    for method, kernel in ((dc.DISTANCE, "Euclidean"), (dc.VORONOI, "Chebyshev:1")):
        want = dc.orc_run(src, method, kernel)[0]
        got = im.MorphologyDirectImage(img, method, kernel).pixels.cpu().numpy()
        assert digest(got) == digest(want), method


@pytest.mark.gpu
def test_repeatable_and_two_launches():
    """Three runs of the same call give identical bits, and each call is exactly two launches of the sweep kernel."""
    import torch
    src = dc.shapes(2048, 1536, 4, seed=5)
    img = im.Image(torch.from_numpy(src).cuda())
    for method, kernel in ((dc.DISTANCE, "Euclidean:4"), (dc.VORONOI, "Euclidean"), (dc.DISTANCE, "Manhattan:1")):
        before = get_option("morph_direct_launches")
        runs = [im.MorphologyDirectImage(img, method, kernel).pixels.cpu().numpy() for _ in range(3)]
        assert get_option("morph_direct_launches") - before == 6
        assert digest(runs[0]) == digest(runs[1]) == digest(runs[2]), (method, kernel)


@pytest.mark.gpu
def test_unaligned_device_buffer():
    import torch
    src = dc.sources(4)["specials"]
    flat = torch.empty(src.size + 1, dtype=torch.float32, device="cuda")
    view = flat[1:].view(src.shape)
    view.copy_(torch.from_numpy(src))
    assert view.data_ptr() % 16 == 4
    for method in (dc.DISTANCE, dc.VORONOI):
        got = im.MorphologyDirectImage(im.Image(view), method, "Euclidean:3").pixels.cpu().numpy()
        assert digest(got) == digest(dc.orc_run(src, method, "Euclidean:3")[0]), method


@pytest.mark.gpu
def test_declines_leave_dst():
    """Declines on the device: dst untouched and nothing launched.  MorphologyImage keeps declining Distance / Voronoi."""
    import torch
    lib = _lib.load()
    src = dc.sources(3)["noise"]
    h, w, ch = src.shape
    dev = torch.from_numpy(src).cuda()
    dst = torch.full_like(dev, 7.0)
    k = im.AcquireKernelInfo("Euclidean:2")
    launches = im.launch_count()
    assert lib.mb200_morphology_direct_image_dev(dev.data_ptr(), dst.data_ptr(), w, h, ch, dc.VORONOI, k._ptr,
                                                 None) == _lib.EUNSUPPORTED
    assert lib.mb200_morphology_direct_image_dev(dev.data_ptr(), dst.data_ptr(), w, h, ch, im.DilateMorphology, k._ptr,
                                                 None) == _lib.EINVAL
    for method in (dc.DISTANCE, dc.VORONOI):
        assert lib.mb200_morphology_image_dev(dev.data_ptr(), dst.data_ptr(), w, h, 4 if method == dc.VORONOI else ch,
                                              method, 1, k._ptr, 0.0, None) == _lib.EUNSUPPORTED
    torch.cuda.synchronize()
    assert im.launch_count() == launches
    assert bool((dst == 7.0).all())


def test_argument_checks_without_a_device():
    """The C-ABI checks its arguments before it touches the device, so these hold on any machine."""
    lib = _lib.load()
    src = make_image(9, 7, 4, seed=1)
    dst = np.full_like(src, 7.0)
    rgb = make_image(9, 7, 3, seed=1)
    k = im.AcquireKernelInfo("Euclidean:2")
    outside = im.AcquireKernelInfo("3x3:1,2,3 4,5,6 7,8,9")
    outside._ptr.contents.x = 3
    negative = im.AcquireKernelInfo("3x3:1,2,3 4,5,6 7,8,9")
    negative._ptr.contents.y = -1
    disk = im.AcquireKernelInfo("Disk:70")                  # 141x141: more than the wavefront's shared memory holds
    S, D = src.ctypes.data, dst.ctypes.data
    cases = [
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 4, im.ErodeMorphology, k._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 4, 23, k._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 4, dc.DISTANCE, None)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 4, dc.DISTANCE, outside._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 4, dc.VORONOI, negative._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 0, 7, 4, dc.DISTANCE, k._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 5, dc.DISTANCE, k._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image(S, S, 9, 7, 4, dc.DISTANCE, k._ptr)),
        (_lib.EUNSUPPORTED, lambda: lib.mb200_morphology_direct_image(rgb.ctypes.data, D, 9, 7, 3, dc.VORONOI,
                                                                      k._ptr)),
        (_lib.EUNSUPPORTED, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 1, dc.VORONOI, k._ptr)),
        (_lib.EUNSUPPORTED, lambda: lib.mb200_morphology_direct_image(S, D, 9, 7, 4, dc.DISTANCE,
                                                                      disk._ptr)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image_dev(S, D, 9, 7, 4, 20, k._ptr, None)),
        (_lib.EINVAL, lambda: lib.mb200_morphology_direct_image_dev(S, D, 9, 7, 4, dc.DISTANCE, outside._ptr, None)),
        (_lib.EUNSUPPORTED, lambda: lib.mb200_morphology_direct_image_dev(S, D, 9, 7, 2 + 1, dc.VORONOI, k._ptr,
                                                                          None)),
    ]
    for n, (code, call) in enumerate(cases):
        assert call() == code, (n, lib.mb200_last_error())
        assert (dst == 7.0).all(), n
    with pytest.raises(im.MagickB200Error) as e:
        im.MorphologyDirectImage(im.Image(rgb), im.VoronoiMorphology, "Euclidean")
    assert e.value.code == _lib.EUNSUPPORTED
