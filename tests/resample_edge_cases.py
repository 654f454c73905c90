"""Edge-case inputs shared by the tests of the resampling operators (ResizeImage, SampleImage, ScaleImage and
ThumbnailImage): the oracle-against-reference suite (test_oracle_resample_edges_vs_ref.py) and the GPU suite
(test_gpu_resample_edges.py) run the same images and geometries, for 1-4 channels.

* dense / sparse: stencil_edge_cases.special_image with a special value in every 7th sample, or in about 1 sample in
  100 (most outputs stay finite, so a window that is one tap too wide or too narrow shows up as a stray NaN or inf).
* nan_lines: whole rows and columns of NaN, at the image borders and in the interior.
* inf_alpha_lines: whole rows and columns of +inf and -inf in the last channel only (alpha, where there is one).
* opposite_infinities: alpha +inf and -inf in one column window, each under colour of its own sign.  There gamma is
  inf + -inf = NaN and PerceptibleReciprocal(NaN) is 1e12 (resize.c:3522), so the vertical pass gives +inf colour under
  NaN alpha, which the horizontal pass turns into NaN.
* transparent_negative / negative_zero: blocks whose every product w * QS * alpha * colour is -0 under positive weights
  (alpha +0 over negative HDR colour; opaque -0 colour).  The reference starts each sum from pixel = 0.0
  (resize.c:3493), so 0.0 + -0 gives +0 there; a kernel that seeds its accumulator with the first product keeps -0.

The geometries cover 1 x N, N x 1, 2 x 2 and 1 x 1 sources, reductions to one row or column (each window is the whole
axis), same-size resizes with an explicit filter (factor 1: scale = 1 + 1e-12, so every window has tiny off-centre
weights), the 64-output threshold of the regular table (126 -> 63 against 128 -> 64), sizes whose two factors differ by
one double ULP at a nominal 2x (748 x 518 -> 374 x 259 has x_factor 0.49999999999999994 < y_factor 0.5, 746 x 748 ->
373 x 374 the opposite: they decide the pass order, resize.c:3846), an anisotropic resize and a 16x reduction (96
Lanczos taps, which no streaming kernel serves)."""
import numpy as np

from stencil_edge_cases import special_image
from util import make_image

F32 = np.float32

# resample.h: 1 Point, 2 Box, 3 Triangle, 8 Gaussian, 11 Catrom, 12 Mitchell, 13 Jinc, 22 Lanczos, 23 LanczosSharp,
# 24 Lanczos2; 0 is ResizeImage's default (Mitchell with alpha, Lanczos without, Point at factor 1)
FILTERS = [0, 1, 2, 3, 8, 11, 12, 13, 22, 23, 24]
ALL_FILTERS = list(range(1, 34))
# (filter, ratio) -> (stride, taps) of the streamed runs: every pair the streaming and fused kernels serve (shared with
# test_gpu_resize_fused.py)
SERVED = {(22, 2): (2, 12), (24, 2): (2, 8), (12, 2): (2, 8), (3, 2): (2, 4), (22, 3): (3, 19), (22, 4): (4, 24),
          (24, 4): (4, 16)}


def dense(ch, w=37, h=23, seed=3):
    return special_image(ch, w=w, h=h, seed=seed, every=7)


def sparse(ch, w, h, seed=5, every=100):
    return special_image(ch, w=w, h=h, seed=seed, every=every)


def nan_lines(ch, w=146, h=138, seed=6):
    img = make_image(w, h, ch, seed=seed, kind="hdr")
    img[[0, h // 2, h - 1], :, :] = np.nan
    img[:, [0, w // 3, w - 1], :] = np.nan
    return np.ascontiguousarray(img)


def inf_alpha_lines(ch, w=146, h=138, seed=7):
    img = make_image(w, h, ch, seed=seed)
    img[0, :, ch - 1] = np.inf
    img[h // 2 + 1, :, ch - 1] = -np.inf
    img[:, 0, ch - 1] = -np.inf
    img[:, w // 2, ch - 1] = np.inf
    return np.ascontiguousarray(img)


def opposite_infinities(ch, w=16, h=16):
    img = make_image(w, h, ch, seed=8)
    img[6, 7, :] = 1000.0
    img[7, 7, :] = -1000.0
    img[6, 7, ch - 1] = np.inf
    img[7, 7, ch - 1] = -np.inf
    return np.ascontiguousarray(img)


def _blocks(img, colour, alpha):
    """Sets an interior block and a block in the top-left corner (clipped windows, the border outputs)."""
    h, w, ch = img.shape
    colours = ch - 1 if ch in (2, 4) else ch
    for rows, cols in ((slice(h // 6, h - h // 6), slice(w // 7, w - w // 7)), (slice(0, h // 4), slice(0, w // 4))):
        img[rows, cols, :colours] = colour
        if ch in (2, 4):
            img[rows, cols, ch - 1] = alpha
    return np.ascontiguousarray(img)


def transparent_negative(ch, w=144, h=136):
    """Alpha +0 over negative HDR colour (without alpha: only the negative colour)."""
    return _blocks(make_image(w, h, ch, seed=9, kind="hdr"), F32(-5000.0), F32(0.0))


def negative_zero(ch, w=144, h=136):
    """Opaque blocks of -0.0 colour."""
    return _blocks(make_image(w, h, ch, seed=10), F32(-0.0), F32(65535.0))


SHAPES = [(1, 1), (1, 17), (17, 1), (2, 2)]                      # (rows, columns)


def shapes(ch):
    """{name: small image cut from a dense special image}."""
    img = special_image(ch, every=3)
    return {f"{h}x{w}": np.ascontiguousarray(img[:h, 5:5 + w]) for h, w in SHAPES}


# (columns, rows) of the small images' outputs: enlargements, reductions to one row / column / pixel, same size
SHAPE_OUTPUTS = {"1x1": [(4, 3), (1, 1)], "1x17": [(3, 8), (1, 40), (5, 1)], "17x1": [(8, 3), (40, 1), (1, 5)],
                 "2x2": [(1, 1), (5, 5), (2, 1), (2, 2)]}
DENSE_OUTPUTS = [(18, 11), (74, 46), (37, 23), (37, 1), (1, 23), (1, 1), (13, 40)]


def resize_cases(ch):
    """[(name, image, columns, rows, filter)]: the oracle is pinned to the reference on these, the kernels to the
    oracle.  The minimal reproductions of NAMED run separately."""
    out = []
    d = dense(ch)
    out += [(f"dense {ow}x{oh} f{f}", d, ow, oh, f) for f in FILTERS for ow, oh in DENSE_OUTPUTS]
    out += [(f"{n} {ow}x{oh} f{f}", img, ow, oh, f) for n, img in shapes(ch).items() for ow, oh in SHAPE_OUTPUTS[n]
            for f in (0, 1, 3, 22)]
    small = dense(ch, w=24, h=20, seed=4)
    out += [(f"dense 24x20 {ow}x{oh} f{f}", small, ow, oh, f) for f in ALL_FILTERS for ow, oh in [(12, 10), (40, 33)]]
    # the streamed runs: every served (filter, ratio), 96 x 80 outputs (enough for Lanczos' clipped border windows)
    for (f, r) in sorted(SERVED):
        out.append((f"sparse served f{f} {r}x", sparse(ch, 96 * r, 80 * r, seed=f + r, every=25 * r * r), 96, 80, f))
    lines = {"NaN lines": nan_lines(ch), "inf alpha lines": inf_alpha_lines(ch)}
    out += [(f"{n} 73x69 f{f}", img, 73, 69, f) for n, img in lines.items() for f in (0, 3, 22, 12, 24)]
    out += [(f"{n} 200x150 f{f}", img, 200, 150, f) for n, img in lines.items() for f in (0, 22)]
    out += [(f"{n} 49x46 f22", img, 49, 46, 22) for n, img in lines.items()]       # ratio ~2.98
    # the regular table's 64-output threshold, one axis on each side
    for w, h in [(128, 126), (126, 128)]:
        img = sparse(ch, w, h, seed=12)
        out += [(f"sparse {w}x{h} f{f}", img, w // 2, h // 2, f) for f in (0, 3, 22)]
    # factors one double ULP apart at a nominal 2x: the pass order and the fused kernel's equal-factor test
    for (w, h), (ow, oh) in [((748, 518), (374, 259)), ((746, 748), (373, 374))]:
        img = sparse(ch, w, h, seed=13)
        out += [(f"sparse {w}x{h} {ow}x{oh} f{f}", img, ow, oh, f) for f in (3, 22)]
    aniso = sparse(ch, 40, 130, seed=14)
    out += [(f"sparse 40x130 100x65 f{f}", aniso, 100, 65, f) for f in (0, 3, 22, 13)]
    wide = sparse(ch, 1024, 48, seed=15, every=20000)
    out += [(f"sparse 1024x48 64x3 f{f}", wide, 64, 3, f) for f in (0, 22)]                        # 16x: 96 taps
    # -0 blocks with x_factor > y_factor: the horizontal pass runs first and the streamed vertical pass second
    out += [(f"{n} 746x748 373x374 f3", build(ch, 746, 748), 373, 374, 3)
            for n, build in [("transparent negative", transparent_negative), ("negative zero", negative_zero)]]
    return out


def sample_cases(ch):
    """[(name, image, columns, rows)] for SampleImage and ScaleImage."""
    out = []
    d = dense(ch)
    out += [(f"dense {ow}x{oh}", d, ow, oh) for ow, oh in DENSE_OUTPUTS + [(36, 22), (38, 24), (5, 3)]]
    out += [(f"{n} {ow}x{oh}", img, ow, oh) for n, img in shapes(ch).items() for ow, oh in SHAPE_OUTPUTS[n]]
    for name, img in {"NaN lines": nan_lines(ch), "inf alpha lines": inf_alpha_lines(ch),
                      "transparent negative": transparent_negative(ch), "negative zero": negative_zero(ch),
                      "opposite infinities": opposite_infinities(ch)}.items():
        h, w = img.shape[:2]
        out += [(f"{name} {ow}x{oh}", img, ow, oh) for ow, oh in [(w // 2, h // 2), (w // 3, h // 5), (2 * w + 1, h + 3)]]
    out += [(f"sparse 748x518 {ow}x{oh}", sparse(ch, 748, 518, seed=13), ow, oh) for ow, oh in [(374, 259), (101, 7)]]
    return out


def thumbnail_cases(ch):
    """[(name, image, columns, rows)] for ThumbnailImage: the sample (factors > 4), box (> 2) and resize stages."""
    out = []
    d = dense(ch)
    out += [(f"dense {ow}x{oh}", d, ow, oh) for ow, oh in [(18, 11), (9, 5), (5, 4), (74, 46), (1, 1), (37, 1)]]
    out += [(f"{n} {ow}x{oh}", img, ow, oh) for n, img in shapes(ch).items() for ow, oh in SHAPE_OUTPUTS[n]]
    for name, img in {"sparse": sparse(ch, 146, 138, seed=16), "NaN lines": nan_lines(ch),
                      "inf alpha lines": inf_alpha_lines(ch), "transparent negative": transparent_negative(ch),
                      "negative zero": negative_zero(ch)}.items():
        out += [(f"{name} {ow}x{oh}", img, ow, oh) for ow, oh in [(12, 11), (30, 29), (70, 66), (100, 90)]]
    return out


# The minimal reproductions: (image builder, columns, rows, filter) of the output.  The signed-zero ones are
# the streamed and fused kernels' seed (the reference gives +0 under Triangle's positive weights); 128 -> 64 is the
# smallest size whose runs are streamed, Lanczos 2x needs about 80 outputs per axis.
NAMED = {
    "transparent negative Triangle 2x": (lambda ch: transparent_negative(ch, 128, 128), 64, 64, 3),
    "negative zero Triangle 2x": (lambda ch: negative_zero(ch, 128, 128), 64, 64, 3),
    "transparent negative Lanczos 2x": (lambda ch: transparent_negative(ch, 192, 160), 96, 80, 22),
    "negative zero Lanczos 2x": (lambda ch: negative_zero(ch, 192, 160), 96, 80, 22),
    "transparent negative 144x136 Triangle 2x": (transparent_negative, 72, 68, 3),
    "negative zero 144x136 Mitchell 2x": (negative_zero, 72, 68, 12),
    "opposite infinite alphas Triangle 2x": (opposite_infinities, 8, 8, 3),
}
