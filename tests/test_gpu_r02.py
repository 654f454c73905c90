"""Round-2 parity cases (VERDICT r01 "What's weak" 1-3): the PerceptibleReciprocal clamp around its threshold,
non-finite HDRI samples next to zero-padded taps, config 3's position-dependent weights along the WHOLE axis, the
pixel-cache residency API and a sharded batch."""
import ctypes as C

import numpy as np
import pytest

import util
from util import P, make_image, max_ulp, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")
torch = pytest.importorskip("torch")


def _dev(a):
    return im.Image(torch.from_numpy(a).cuda())


def _host(img):
    return img.pixels.cpu().numpy() if img.on_device else img.pixels


def orc(fn, src, *args):
    h, w, ch = src.shape
    dst = np.empty_like(src)
    assert getattr(oracle(), fn)(P(src), P(dst), w, h, ch, *args) == 0
    return dst


def assert_same_specials_and_ulp(got, want, bar=1):
    """NaN where the reference has NaN, the same infinity where it has one, <= bar ULP elsewhere."""
    assert np.array_equal(np.isnan(got), np.isnan(want))
    inf = np.isinf(want)
    assert np.array_equal(np.isinf(got), inf)
    assert np.array_equal(got[inf], want[inf])
    ok = np.isfinite(want)
    d = util.ulp_distance(np.where(ok, got, np.float32(0)), np.where(ok, want, np.float32(0)))
    assert d.max() <= bar, int(d.max())


# ---- PerceptibleReciprocal: QS * sum(k * alpha) on both sides of MagickEpsilon (pixel-accessor.h:242-254, morphology.c:3197)
@pytest.mark.parametrize("sigma", [1.0, 2.0, 4.0, 2.6])
def test_reciprocal_clamp_around_the_threshold(sigma):
    rng = np.random.default_rng(11)
    h, w = 96, 160
    src = (rng.random((h, w, 4), dtype=np.float32) * np.float32(65535)).astype(np.float32)
    # alpha: mostly exactly 0; isolated pixels whose alpha puts QS*k*alpha a little below / above 1e-12 for the centre
    # tap (k ~ 0.1-0.4) and far below it for the outer taps -- every neighbourhood weight sum is "one tap" sized
    alpha = np.zeros((h, w), np.float32)
    ys, xs = np.mgrid[4:h:9, 4:w:11]
    vals = (6.5535e-8 / 0.2) * np.float32(2.0) ** rng.integers(-6, 7, size=ys.shape)
    alpha[ys, xs] = vals.astype(np.float32)
    alpha[:8, :8] = 65535.0                                   # an opaque corner keeps ordinary arithmetic in the picture
    alpha[40:44, 100:104] = np.float32(1e-30)                # denormal-range weight sums
    src[..., 3] = alpha
    for fn, args, op in (("orc_blur", (0.0, sigma), lambda d: im.BlurImage(d, 0.0, sigma)),
                         ("orc_gaussian_blur", (0.0, min(sigma, 2.0)), lambda d: im.GaussianBlurImage(d, 0.0, min(sigma, 2.0)))):
        want = orc(fn, src, *args)
        got = _host(op(_dev(src)))
        assert np.isfinite(want).all()
        assert max_ulp(got, want) <= 1, (fn, sigma, max_ulp(got, want))
    # the resize kernels carry the same clamp (resize.c:3472-3484)
    want = np.empty((h // 2, w // 2, 4), np.float32)
    assert oracle().orc_resize(P(src), w, h, 4, P(want), w // 2, h // 2, 22) == 0
    assert max_ulp(_host(im.ResizeImage(_dev(src), w // 2, h // 2, im.LanczosFilter)), want) <= 1


# ---- zero-padded taps must not touch non-finite samples (conv1d.cu: 17 < ntaps < 25, 25 < ntaps < 33, ...)
@pytest.mark.parametrize("ch", [1, 3, 4])
@pytest.mark.parametrize("radius,sigma", [(0.0, 2.4), (0.0, 3.6), (13.0, 3.0), (2.0, 1.0), (0.0, 4.0)])
def test_non_finite_samples_next_to_padded_taps(ch, radius, sigma):
    src = make_image(150, 110, ch, seed=21)
    src[30, 40, 0] = np.inf
    src[31, 90, ch - 1] = -np.inf
    src[80, 20, min(1, ch - 1)] = np.nan
    src[100, 140, 0] = np.inf
    want = orc("orc_blur", src, radius, sigma)
    got = _host(im.BlurImage(_dev(src), radius, sigma))
    assert np.isfinite(want).mean() > 0.3          # the poison stays local in the reference ...
    assert_same_specials_and_ulp(got, want)          # ... and is the same set of outputs here


def test_non_finite_samples_rank1_gaussian():
    src = make_image(120, 90, 4, seed=22)
    src[40, 50, 1] = np.inf
    src[60, 70, 3] = np.nan
    want = orc("orc_gaussian_blur", src, 0.0, 1.3)
    got = _host(im.GaussianBlurImage(_dev(src), 0.0, 1.3))
    assert_same_specials_and_ulp(got, want)


# ---- config 3: every weight-run boundary and the far end of the axis against the oracle -----------------------------
@pytest.mark.parametrize("axis", [0, 1])
def test_config3_strips_cover_the_whole_axis(axis):
    """bisect = (o+0.5)/factor + eps changes binade along the axis and the streaming kernels switch weight runs there
    (resize.c:3398-3443, :3614-3657).  A 16384-long strip (64 pixels wide) resized 2x is small enough for the oracle and
    contains every run boundary, the clipped windows at both ends and the last outputs."""
    long, short = 16384, 64
    rng = np.random.default_rng(33)
    shape = (short, long, 4) if axis == 0 else (long, short, 4)
    src = (rng.random(shape, dtype=np.float32) * np.float32(65535)).astype(np.float32)
    src[: shape[0] // 3, : shape[1] // 3, 3] = 0.0
    h, w = shape[0], shape[1]
    want = np.empty((h // 2, w // 2, 4), np.float32)
    assert oracle().orc_resize(P(src), w, h, 4, P(want), w // 2, h // 2, 22) == 0
    families = ("resize_v_stream_launches", "resize_h_tma_launches", "resize_h_stream_launches", "resize_regular_launches",
                "resize_gather_launches")
    n0 = im.launch_count()
    c0 = [util.get_option(f) for f in families]
    got = _host(im.ResizeImage(_dev(src), w // 2, h // 2, im.LanczosFilter))
    assert im.launch_count() - n0 == 2
    # the long axis on the streaming kernels (borders ride along), the 64 -> 32 axis (too short for the run detection)
    # on the gather kernel
    v, tma, cp, regular, gather = (util.get_option(f) - c for f, c in zip(families, c0))
    assert (v, tma + cp) == ((0, 1) if axis == 0 else (1, 0)) and regular == 0 and gather == 1
    d = util.ulp_distance(got, want)
    assert d.max() <= 1
    assert (d == 0).mean() > 0.9999
    # the long axis on its own (the other axis 1:1), so that a first-pass difference cannot hide behind the second
    ow, oh = (w // 2, h) if axis == 0 else (w, h // 2)
    want = np.empty((oh, ow, 4), np.float32)
    assert oracle().orc_resize(P(src), w, h, 4, P(want), ow, oh, 22) == 0
    got = _host(im.ResizeImage(_dev(src), ow, oh, im.LanczosFilter))
    assert max_ulp(got, want) <= 1


# ---- pixel cache staged into HBM: bounce ring, residency, lazy synchronisation ---------------------------------------
def _stats():
    out = (C.c_ulonglong * 6)()
    from imagemagick_b200 import _lib
    _lib.load().mb200_cache_stats(out)
    return list(out)


def test_pageable_buffers_take_the_bounce_ring_and_keep_their_bits():
    # > 4 MiB and not a multiple of the 16 MiB chunk: exercises the ring wrap-around and the ragged tail
    src = make_image(2311, 1013, 4, seed=5)             # 37.5 MB
    s0 = _stats()
    got = im.BlurImage(im.Image(src), 0.0, 1.0).pixels          # host-buffer entry point
    s1 = _stats()
    assert s1[5] - s0[5] == 2 * src.nbytes                     # both directions went through the ring
    dev = _host(im.BlurImage(_dev(src), 0.0, 1.0))
    assert np.array_equal(got, dev)
    crop = np.ascontiguousarray(src[:64, :96])
    assert max_ulp(got[:48, :80], orc("orc_blur", crop, 0.0, 1.0)[:48, :80]) <= 1


def test_cache_residency_lazy_chain_moves_source_and_result_only():
    from imagemagick_b200 import _lib
    lib = _lib.load()
    w = h = 1024
    src = make_image(w, h, 4, seed=9)
    mid = np.empty_like(src)
    out = np.empty((h // 2, w // 2, 4), np.float32)
    want_mid = _host(im.BlurImage(_dev(src), 0.0, 2.0))
    want_out = _host(im.ResizeImage(_dev(want_mid), w // 2, h // 2, im.LanczosFilter))
    vp = lambda a: C.c_void_p(a.ctypes.data)
    for a in (src, mid, out):
        _lib.check(lib.mb200_cache_attach(vp(a), a.nbytes, 1))
    try:
        assert lib.mb200_cache_resident(vp(src)) == 2
        # eager (default): results land in the host buffers, the source is uploaded for every operator
        s0 = _stats()
        _lib.check(lib.mb200_blur_image(vp(src), vp(mid), w, h, 4, 0.0, 2.0))
        _lib.check(lib.mb200_resize_image(vp(mid), w, h, 4, vp(out), w // 2, h // 2, im.LanczosFilter))
        s1 = _stats()
        assert np.array_equal(mid, want_mid) and np.array_equal(out, want_out)
        assert s1[1] - s0[1] == src.nbytes + mid.nbytes and s1[3] - s0[3] == mid.nbytes + out.nbytes
        # lazy: one upload, nothing comes back until mb200_cache_sync
        assert lib.mb200_cache_set_lazy(1) == 0
        mid[:] = 0
        out[:] = 0
        _lib.check(lib.mb200_cache_host_written(vp(src)))
        _lib.check(lib.mb200_cache_host_written(vp(mid)))
        _lib.check(lib.mb200_cache_host_written(vp(out)))
        s0 = _stats()
        _lib.check(lib.mb200_blur_image(vp(src), vp(mid), w, h, 4, 0.0, 2.0))
        _lib.check(lib.mb200_resize_image(vp(mid), w, h, 4, vp(out), w // 2, h // 2, im.LanczosFilter))
        s1 = _stats()
        assert s1[1] - s0[1] == src.nbytes and s1[3] - s0[3] == 0 and s1[4] - s0[4] == 1
        assert not out.any() and lib.mb200_cache_resident(vp(out)) == 1
        _lib.check(lib.mb200_cache_sync(vp(out)))
        assert np.array_equal(out, want_out) and lib.mb200_cache_resident(vp(out)) == 3
        assert not mid.any()                                   # the intermediate never left HBM
        s2 = _stats()
        assert s2[3] - s1[3] == out.nbytes
        # a second chain on the unchanged source: no upload at all
        _lib.check(lib.mb200_blur_image(vp(src), vp(mid), w, h, 4, 0.0, 2.0))
        assert _stats()[1] == s2[1]
        # the host rewrites the source: the stale HBM copy must not be used
        src[:] = src[::-1].copy()
        _lib.check(lib.mb200_cache_host_written(vp(src)))
        _lib.check(lib.mb200_blur_image(vp(src), vp(mid), w, h, 4, 0.0, 2.0))
        _lib.check(lib.mb200_cache_sync(vp(mid)))
        assert np.array_equal(mid, want_mid[::-1])
    finally:
        lib.mb200_cache_set_lazy(0)
        for a in (src, mid, out):
            lib.mb200_cache_detach(vp(a))
    assert lib.mb200_cache_resident(vp(src)) == -1


def test_in_place_operators_on_attached_buffers():
    from imagemagick_b200 import _lib
    lib = _lib.load()
    src = make_image(300, 200, 4, seed=3)
    want = src.copy()
    assert oracle().orc_colorspace(P(want), 300, 200, 4, 23, 11) == 0
    buf = src.copy()
    vp = C.c_void_p(buf.ctypes.data)
    _lib.check(lib.mb200_cache_attach(vp, buf.nbytes, 0))
    try:
        _lib.check(lib.mb200_transform_colorspace(vp, 300, 200, 4, im.sRGBColorspace, im.LabColorspace))
        assert max_ulp(buf, want) <= 1
    finally:
        lib.mb200_cache_detach(vp)


# ---- configs[4]: a sharded batch (image i -> rank i mod N); two images of a shard against the oracle -------------------
def test_sharded_batch_two_images_against_the_oracle():
    from imagemagick_b200 import dist as mdist
    world, n_images, size = 8, 20, 512
    taps = im.AcquireKernelInfo("blur:0x4").arrays()[0][0].ravel()
    job = mdist.FilterJob.unpack(mdist.FilterJob(0.0, 4.0, size // 2, size // 2, im.LanczosFilter, taps).pack())
    kernel = mdist.blur_kernel_from_taps(job.taps)
    for rank in (0, 5):
        mine = mdist.shard_indices(n_images, rank, world)
        assert mine == list(range(rank, n_images, world))
        batch = {i: make_image(size, size, 4, seed=1000 + i, kind="alpha_blocks" if i % 2 else "noise") for i in mine}
        results = mdist.run_pipeline({i: _dev(a) for i, a in batch.items()}, kernel, job)
        assert sorted(results) == mine
        for i in mine[:2]:
            blurred = orc("orc_blur", batch[i], 0.0, 4.0)
            want = np.empty((size // 2, size // 2, 4), np.float32)
            assert oracle().orc_resize(P(blurred), size, size, 4, P(want), size // 2, size // 2, 22) == 0
            got = _host(results[i])
            # two <= 1 ULP operators in sequence: the second one sees inputs that may differ by 1 ULP
            assert util.ulp_distance(got, want).max() <= 2
            assert util.frac_exact(got, want) > 0.999


def test_fp64_probe_reports_a_sane_rate():
    from imagemagick_b200 import _lib
    rate = C.c_double(0)
    _lib.check(_lib.load().mb200_probe_fp64_fma_rate(C.byref(rate)))
    assert 5e12 < rate.value < 4e13


def test_host_buffer_calls_from_two_application_threads():
    """Every application thread gets its own library stream (runtime.cu default_stream): concurrent callers overlap and
    still produce the single-threaded bits; an attached buffer written by one thread and read by another is ordered by
    the entry's event."""
    import threading
    from imagemagick_b200 import _lib
    lib = _lib.load()
    imgs = [make_image(700, 500, 4, seed=40 + k) for k in range(4)]
    want = [_host(im.ResizeImage(im.BlurImage(_dev(a), 0.0, 2.0), 350, 250, im.LanczosFilter)) for a in imgs]
    got = [None] * 4
    errors = []
    dev = torch.cuda.current_device()

    def worker(k):
        try:
            _lib.check(lib.mb200_set_device(dev))
            for _ in range(3):
                b = im.BlurImage(im.Image(imgs[k]), 0.0, 2.0)
                got[k] = im.ResizeImage(b, 350, 250, im.LanczosFilter).pixels
        except Exception as exc:
            errors.append(exc)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errors, errors
    for k in range(4):
        assert np.array_equal(got[k], want[k])
    # producer / consumer across threads on an attached, lazily synchronised buffer
    src, mid = imgs[0], np.empty_like(imgs[0])
    out = np.empty((250, 350, 4), np.float32)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    for a in (src, mid, out):
        _lib.check(lib.mb200_cache_attach(vp(a), a.nbytes, 0))
    lib.mb200_cache_set_lazy(1)
    try:
        def producer():
            lib.mb200_set_device(dev)
            _lib.check(lib.mb200_blur_image(vp(src), vp(mid), 700, 500, 4, 0.0, 2.0))

        def consumer():
            lib.mb200_set_device(dev)
            _lib.check(lib.mb200_resize_image(vp(mid), 700, 500, 4, vp(out), 350, 250, im.LanczosFilter))
            _lib.check(lib.mb200_cache_sync(vp(out)))
        for fn in (producer, consumer):
            t = threading.Thread(target=fn)
            t.start()
            t.join()
        assert np.array_equal(out, want[0])
    finally:
        lib.mb200_cache_set_lazy(0)
        for a in (src, mid, out):
            lib.mb200_cache_detach(vp(a))


# ---- EqualizeImage / EmbossImage (enhance.c:2040, effect.c:1600) --------------------------------------------------------
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["noise", "gradient", "hdr"])
@pytest.mark.parametrize("sync", [True, False])
def test_equalize_bit_exact(ch, kind, sync):
    src = make_image(301, 157, ch, seed=51, kind=kind)
    want = src.copy()
    assert oracle().orc_equalize(P(want), 301, 157, ch, int(sync)) == 0
    d = _dev(src)
    assert im.EqualizeImage(d, sync)
    assert np.array_equal(_host(d), want)
    h = im.Image(src.copy())
    assert im.EqualizeImage(h, sync)
    assert np.array_equal(h.pixels, want)


@pytest.mark.parametrize("ch", [1, 3, 4])
@pytest.mark.parametrize("radius,sigma", [(0.0, 1.0), (0.0, 2.0), (2.0, 0.7)])
def test_emboss(ch, radius, sigma):
    """Kernel taps bit-identical to the oracle's (pinned to the reference); the convolution within 1 ULP; the
    equalisation -- a discontinuous function of the convolved values: one sample crossing a histogram bin moves the whole
    map -- bit exact ON THE SAME convolved image, and the end-to-end result identical to the reference's wherever the
    convolution was (which is nearly everywhere)."""
    k = util.OrcKernel()
    assert oracle().orc_emboss_kernel(radius, sigma, C.byref(k)) == 0
    from imagemagick_b200 import _lib
    mine = im.KernelInfo(_lib.load().mb200_emboss_kernel(radius, sigma)).arrays()[0][0]
    assert np.array_equal(mine, k.array())
    src = make_image(211, 133, ch, seed=52, kind="alpha_blocks" if ch == 4 else "noise")
    conv_want = util.orc_morphology(src, im.ConvolveMorphology, 1, [k])
    conv_got = _host(im.ConvolveImage(_dev(src), im.KernelInfo(_lib.load().mb200_emboss_kernel(radius, sigma))))
    assert max_ulp(conv_got, conv_want) <= 1
    got = _host(im.EmbossImage(_dev(src), radius, sigma))
    eq = conv_got.copy()
    assert oracle().orc_equalize(P(eq), 211, 133, ch, 1) == 0
    assert np.array_equal(got, eq)
    want = orc("orc_emboss", src, radius, sigma)
    if np.array_equal(conv_got, conv_want):
        assert np.array_equal(got, want)
    assert util.frac_exact(got, want) > 0.99


# ---- rank-4 stencils: StatisticImage, RotationalBlurImage, BilateralBlurImage (oracles pinned to the reference) ----------
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("stat", [1, 2, 3, 4, 5, 6, 7, 8, 9, 10])
@pytest.mark.parametrize("win", [(3, 3), (5, 3), (1, 7), (4, 4)])
def test_statistic_image_bit_exact(ch, stat, win):
    src = make_image(97, 61, ch, seed=61, kind="hdr" if stat in (1, 10) else "noise")
    want = orc("orc_statistic", src, stat, win[0], win[1])
    got = _host(im.StatisticImage(_dev(src), stat, win[0], win[1]))
    assert_same_specials_and_ulp(got, want, bar=0)


@pytest.mark.parametrize("ch", [1, 3, 4])
@pytest.mark.parametrize("stat", [4, 6, 7])
@pytest.mark.parametrize("win", [(3, 3), (5, 5), (4, 2), (1, 7), (1, 1), (9, 9)])
def test_rank_statistics_on_few_levels(ch, stat, win):
    """Median, Mode and Nonpeak read the reference's 16-bit skip list (statistic.c:2784, :2809, :2843).  A posterised image
    has few distinct levels: counts tie (the mode is the smallest of the most frequent values), the median sits on the
    window's smallest / largest level (Nonpeak steps off it), flat regions have one level only."""
    src = make_image(97, 61, ch, seed=63, kind="noise")
    poster = (np.round(src / 16384.0) * 16384.0).astype(np.float32)
    poster[10:30, 10:50] = 32768.0
    poster[40:50, 60:90] += np.float32(0.4)            # rounds to the same 16-bit value
    for image in (src, poster):
        want = orc("orc_statistic", image, stat, win[0], win[1])
        got = _host(im.StatisticImage(_dev(image), stat, win[0], win[1]))
        assert np.array_equal(got, want), (ch, stat, win)
    h = im.StatisticImage(im.Image(poster), stat, win[0], win[1]).pixels          # host-buffer entry point
    assert np.array_equal(h, orc("orc_statistic", poster, stat, win[0], win[1]))


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("size,angle", [((120, 80), 10.0), ((64, 64), 45.0), ((201, 33), 3.0), ((50, 90), -20.0)])
def test_rotational_blur_bit_exact(ch, size, angle):
    w, h = size
    src = make_image(w, h, ch, seed=62, kind="alpha_blocks" if ch in (2, 4) else "noise")
    want = orc("orc_rotational_blur", src, angle)
    got = _host(im.RotationalBlurImage(_dev(src), angle))
    assert max_ulp(got, want) == 0


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("win,isig,ssig", [((5, 5), 0.75, 2.0), ((7, 3), 12.0, 1.5), ((3, 9), 40.0, 4.0)])
def test_bilateral_blur_bit_exact(ch, win, isig, ssig):
    src = make_image(90, 70, ch, seed=63, kind="alpha_blocks" if ch in (2, 4) else "gradient")
    want = orc("orc_bilateral_blur", src, win[0], win[1], isig, ssig)
    got = _host(im.BilateralBlurImage(_dev(src), win[0], win[1], isig, ssig))
    assert max_ulp(got, want) == 0
    with pytest.raises(im.MagickB200Error) as e:
        im.BilateralBlurImage(_dev(src), 4, 4, isig, ssig)
    assert e.value.code == -5


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("args", [(0.0, 1.0, 6553.5), (0.0, 2.0, 20000.0), (2.0, 1.0, 1000.0), (0.0, 1.5, 131070.0), (0.0, 1.0, 0.0)])
@pytest.mark.parametrize("kind", ["gradient", "noise"])
def test_selective_blur_bit_exact(ch, args, kind):
    """SelectiveBlurImage (effect.c:3406); threshold 0 selects no tap (every pixel keeps its centre value)."""
    src = make_image(90, 70, ch, seed=64, kind="alpha_blocks" if ch in (2, 4) and kind == "gradient" else kind)
    want = orc("orc_selective_blur", src, *args)
    got = _host(im.SelectiveBlurImage(_dev(src), *args))
    assert max_ulp(got, want) == 0


@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("fn", ["adaptive_blur", "adaptive_sharpen"])
@pytest.mark.parametrize("args", [(0.0, 1.0), (0.0, 2.0), (3.0, 1.5), (0.0, 0.0)])
@pytest.mark.parametrize("kind", ["gradient", "noise"])
def test_adaptive_blur_and_sharpen_bit_exact(ch, fn, args, kind):
    """AdaptiveBlurImage / AdaptiveSharpenImage (effect.c:128 / :447): the edge map (edge -> auto-level -> blur ->
    auto-level) selects a kernel size per pixel, so every stage has to be bit exact; sigma 0 is a plain copy."""
    src = make_image(97, 64, ch, seed=66, kind="alpha_blocks" if ch in (2, 4) and kind == "gradient" else kind)
    want = orc("orc_" + fn, src, *args)
    op = im.AdaptiveBlurImage if fn == "adaptive_blur" else im.AdaptiveSharpenImage
    got = _host(op(_dev(src), *args))
    assert max_ulp(got, want) == 0


def test_selective_blur_host_buffers_through_the_c_abi():
    src = make_image(64, 48, 4, seed=65, kind="alpha_blocks")
    want = orc("orc_selective_blur", src, 0.0, 1.5, 9000.0)
    got = np.empty_like(src)
    from imagemagick_b200 import _lib
    rc = _lib.load().mb200_selective_blur_image(C.c_void_p(src.ctypes.data), C.c_void_p(got.ctypes.data), 64, 48, 4, 0.0, 1.5, 9000.0)
    assert rc == 0 and max_ulp(got, want) == 0


# ---- fused vertical + horizontal ResizeImage (equal integer reduction on both axes) ------------------------------------
@pytest.mark.parametrize("filt", [22, 12, 11])            # Lanczos (12 taps at 2x), Mitchell, Catrom (8 taps)
@pytest.mark.parametrize("size", [(2048, 1536), (2222, 1554), (4096, 130), (140, 4100)])
@pytest.mark.parametrize("kind", ["noise", "alpha_blocks"])
def test_fused_resize_matches_the_oracle_and_the_two_pass_kernels(filt, size, kind):
    w, h = size
    src = make_image(w, h, 4, seed=71, kind=kind)
    d = _dev(src)
    two_pass = _host(im.ResizeImage(d, w // 2, h // 2, filt))
    util.set_option("resize_fused", 1)                    # opt-in kernel (measured slower than the two passes)
    n0 = im.launch_count()
    got = _host(im.ResizeImage(d, w // 2, h // 2, filt))
    launches = im.launch_count() - n0
    util.set_option("resize_fused", 0)
    assert launches == 2                                  # the fused kernel + the border outputs
    # same arithmetic in the same order, same float rounding between the passes: identical bits
    assert np.array_equal(got, two_pass)
    want = np.empty((h // 2, w // 2, 4), np.float32)
    assert oracle().orc_resize(P(src), w, h, 4, P(want), w // 2, h // 2, filt) == 0
    d_ = util.ulp_distance(got, want)
    assert d_.max() <= 1
    assert (d_ == 0).mean() > 0.9999


# ---- ScaleImage (resize.c:4106): the reference's sequential state machine as host-built term lists + a gather kernel ------
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("sizes", [((640, 480), (320, 240)), ((673, 451), (291, 313)), ((400, 300), (1000, 750)),
                                   ((530, 370), (530, 200)), ((530, 370), (170, 370)), ((333, 211), (334, 212)),
                                   ((1000, 30), (70, 90)), ((1024, 1024), (341, 341))])
def test_scale_image_bit_exact(ch, sizes):
    (w, h), (ow, oh) = sizes
    src = make_image(w, h, ch, seed=91, kind="alpha_blocks" if ch in (2, 4) else "noise")
    want = np.empty((oh, ow, ch), np.float32)
    assert oracle().orc_scale(P(src), w, h, ch, P(want), ow, oh) == 0
    got = _host(im.ScaleImage(_dev(src), ow, oh))
    assert np.array_equal(got, want)
    assert np.array_equal(im.ScaleImage(im.Image(src), ow, oh).pixels, want)       # host-buffer entry point
