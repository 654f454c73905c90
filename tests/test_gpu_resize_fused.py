"""The fused vertical + horizontal ResizeImage kernel (resize_stream.cu) for equal integer reductions of RGBA images.

It keeps the vertically filtered, float-rounded intermediate in shared memory and does the two passes' arithmetic in
their order, so every case asks for the bits of the two streaming passes (no_resize_fused=1), and for <= 1 ULP and
>= 99.99 % exact against the oracle.  The launch counters say which path ran, so no case can pass on the other one."""
import numpy as np
import pytest

import util
from resample_edge_cases import SERVED          # (filter, ratio) -> (stride, taps) of the streamed runs
from util import P, make_image, oracle

pytestmark = pytest.mark.gpu

im = pytest.importorskip("imagemagick_b200")

FAMILIES = ("resize_fused_launches", "resize_v_stream_launches", "resize_h_tma_launches", "resize_h_stream_launches")


def _dev(a):
    import torch
    return im.Image(torch.from_numpy(a).cuda())


def _host(img):
    return img.pixels.cpu().numpy() if img.on_device else img.pixels


def counted(fn):
    c0 = {f: util.get_option(f) for f in FAMILIES}
    out = fn()
    return out, {f: util.get_option(f) - c0[f] for f in FAMILIES}


def two_pass(fn):
    util.set_option("no_resize_fused", 1)
    out, counts = counted(fn)
    util.set_option("no_resize_fused", 0)
    assert counts["resize_fused_launches"] == 0 and counts["resize_v_stream_launches"] == 1, counts
    return out


def fused(fn):
    util.set_option("resize_fused", 1)
    out, counts = counted(fn)
    util.set_option("resize_fused", 0)
    assert counts["resize_fused_launches"] == 1 and counts["resize_v_stream_launches"] == 0, counts
    return out


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check_oracle(got, src, ow, oh, filt):
    h, w, _ = src.shape
    want = np.empty((oh, ow, 4), np.float32)
    assert oracle().orc_resize(P(src), w, h, 4, P(want), ow, oh, filt) == 0
    finite = np.isfinite(want)
    assert np.array_equal(finite, np.isfinite(got))
    d = util.ulp_distance(np.where(finite, got, 0).astype(np.float32), np.where(finite, want, 0).astype(np.float32))
    assert d.max() <= 1
    assert (d == 0).mean() >= 0.9999


# ---- every served (S, N), ragged sizes, several tiles per axis with seams inside and across the weight runs ----------
@pytest.mark.parametrize("kind", ["noise", "alpha_blocks", "hdr"])
@pytest.mark.parametrize("filt,ratio", sorted(SERVED))
def test_every_served_pair_gives_the_two_pass_bits(filt, ratio, kind):
    ow, oh = 373, 259                  # not multiples of the tile's 4*NW columns or 31 rows
    src = make_image(ow * ratio, oh * ratio, 4, seed=11 * filt + ratio, kind=kind)
    d = _dev(src)
    run = lambda: _host(im.ResizeImage(d, ow, oh, filt))   # noqa: E731
    got = fused(run)
    assert same_bits(got, two_pass(run))
    check_oracle(got, src, ow, oh, filt)


def test_headline_size_whole_image():
    """8192^2 -> 4096^2 Lanczos, the benchmark's resize: the automatic path is the fused kernel, with the two passes'
    bits on the whole image; three runs give the same bits."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(3)
    src = torch.rand(8192, 8192, 4, device="cuda", generator=g) * 65535
    src[:2048, :2048, 3] = 0.0
    img = im.Image(src)
    run = lambda: im.ResizeImage(img, 4096, 4096, im.LanczosFilter).pixels   # noqa: E731
    first, counts = counted(run)
    assert counts["resize_fused_launches"] == 1 and counts["resize_v_stream_launches"] == 0, counts
    for _ in range(2):
        assert torch.equal(run().view(torch.int32), first.view(torch.int32))
    assert torch.equal(two_pass(run).view(torch.int32), first.view(torch.int32))


def test_unaligned_source_goes_through_aligned_copies():
    import torch
    src = make_image(2 * 173, 2 * 131, 4, seed=12, kind="alpha_blocks")
    flat = torch.empty(src.size + 1, dtype=torch.float32, device="cuda")
    t = flat[1:].view(src.shape)
    t.copy_(torch.from_numpy(src))
    assert t.data_ptr() % 16 == 4
    got = fused(lambda: _host(im.ResizeImage(im.Image(t), 173, 131, 22)))
    assert same_bits(got, fused(lambda: _host(im.ResizeImage(_dev(src), 173, 131, 22))))
    check_oracle(got, src, 173, 131, 22)


def test_repeated_runs_give_identical_bits():
    src = make_image(2 * 373, 2 * 259, 4, seed=4, kind="noise")
    d = _dev(src)
    runs = [fused(lambda: _host(im.ResizeImage(d, 373, 259, 22))) for _ in range(3)]
    assert same_bits(runs[0], runs[1]) and same_bits(runs[0], runs[2])


def test_tile_rows_past_the_grid_limit_fall_back_to_the_two_passes():
    """More than 65535 tile rows (31 output rows each) do not fit the grid: the fused launch declines even when forced
    and the two streaming passes serve the image."""
    import torch
    oh = 31 * 65536 + 1000
    src = torch.rand(2 * oh, 128, 4, device="cuda") * 65535
    img = im.Image(src)
    run = lambda: im.ResizeImage(img, 64, oh, im.TriangleFilter).pixels   # noqa: E731
    util.set_option("resize_fused", 1)
    got, counts = counted(run)
    util.set_option("resize_fused", 0)
    assert counts["resize_fused_launches"] == 0 and counts["resize_v_stream_launches"] == 1, counts
    assert torch.equal(got.view(torch.int32), two_pass(run).view(torch.int32))
