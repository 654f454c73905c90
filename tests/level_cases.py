"""Inputs, parameter sets and runners shared by the tests of the level and stretch operators (LevelImage, LevelizeImage,
MinMaxStretchImage / AutoLevelImage, ContrastStretchImage / NormalizeImage, LinearStretchImage, GammaImage): the
oracle-against-reference suite and the GPU suite run the same cases.

The oracle is oracle/level_oracle.c (oracle/liblevel_oracle.so) and the reference driver oracle/ref_level.c
(oracle/_ref/libmagickref_level.so), both built by oracle/Makefile.  What the reference computed for every case is stored
in tests/golden/level_digests.json as "digest/channels/property" (the digest of the resulting cache, its channel count
and the operator's "histogram:*" property), keyed like enhance_cases keys its own file; re-record it with
MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C

import numpy as np

import enhance_cases
import util
from util import ROOT, digest, make_image

ORACLE_SO = ROOT / "oracle" / "liblevel_oracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_level.so"
DIGESTS = ROOT / "tests" / "golden" / "level_digests.json"
_libs = {}

_fp = C.POINTER(C.c_float)
_sz, _i, _d, _u = C.c_size_t, C.c_int, C.c_double, C.c_uint

# ref_level_op's operator numbers
LEVEL, LEVELIZE, MINMAX, AUTO_LEVEL, CONTRAST_STRETCH, NORMALIZE, LINEAR_STRETCH, GAMMA = range(8)

# ChannelType masks (pixel.h: Red / Gray 0x1, Green 0x2, Blue 0x4, Alpha 0x10); -1 = the default mask (AllChannels).
# "GB" leaves channel 0 out; "RGBA" selects every channel and so keeps every trait at its default, but it is not
# AllChannels, so the histogram operators switch to per-channel histograms and MinMaxStretch to its per-channel loop.
CHANNEL_MASKS = {"all": -1, "R": 0x1, "GB": 0x6, "alpha": 0x10, "RGBA": 0x17}

# (black, white, gamma) of LevelImage / LevelizeImage: identity, plain, gamma 2.2 / 0.45 / 0 / negative, inverted, equal
LEVEL_ARGS = [(0.0, 65535.0, 1.0), (1000.0, 60000.0, 1.0), (5000.0, 50000.0, 2.2), (5000.0, 50000.0, 0.45),
              (-2000.0, 70000.0, 0.0), (100.0, 65535.0, -1.5), (60000.0, 1000.0, 1.0), (30000.0, 30000.0, 1.0)]
GAMMAS = [1.0, 0.0, 0.45, 2.2, -0.8]
# (black, white, gamma) of MinMaxStretchImage; the first is AutoLevelImage's
MINMAX_ARGS = [(0.0, 0.0, 1.0), (500.0, 1000.0, 1.0), (-300.0, 0.0, 2.2)]


def stretch_points(n: int):
    """(black, white) points of ContrastStretch / LinearStretch for an image of n pixels: 0, the CLI's 2% x 1%, equal,
    inverted and beyond n."""
    return [(0.0, 0.0), (0.02 * n, 0.99 * n), (0.3 * n, 0.3 * n), (0.9 * n, 0.1 * n), (1.5 * n, 2.0 * n)]


def sources(ch: int, w: int = 23, seed: int = 5):
    """name -> image: enhance_cases.mosaic (noise, alpha blocks, HDR, gray pixels, NaN / +-inf), black, white, flat, rows
    that start with NaN, an all-NaN image, and 1xN / Nx1 lines."""
    out = {"mosaic": enhance_cases.mosaic(w, ch, seed=seed)}
    out["black"] = np.zeros((4, w, ch), np.float32)
    out["white"] = np.full((4, w, ch), 65535.0, np.float32)
    out["flat"] = np.full((4, w, ch), 1234.5, np.float32)
    nan_rows = make_image(w, 6, ch, seed=seed + 7, kind="hdr")
    nan_rows[::2, 0, 0] = np.nan
    out["nan rows"] = nan_rows
    out["all nan"] = np.full((3, w, ch), np.nan, np.float32)
    out["1xN"] = make_image(1, 29, ch, seed=seed + 8, kind="hdr")
    out["Nx1"] = make_image(31, 1, ch, seed=seed + 9)
    return out


def gray_sources(ch: int, w: int = 21, seed: int = 9):
    """3-4 channel sRGB images whose pixels are all gray (r = g = b) or all black / white (bilevel); alpha is noise."""
    base = make_image(w, 7, ch, seed=seed, kind="alpha_blocks")
    gray = base.copy()
    gray[..., 1:3] = gray[..., :1]
    bilevel = base.copy()
    bilevel[..., :3] = np.where(bilevel[..., :1] > 32768.0, np.float32(65535.0), np.float32(0.0))
    near = gray.copy()                       # one pixel off gray by one float step: not gray
    near[3, 4, 1] = np.nextafter(near[3, 4, 1], np.float32(np.inf))
    return {"gray": gray, "bilevel": bilevel, "near gray": near}


def update_mask(channel_mask: int, ch: int) -> int:
    return enhance_cases.update_mask(channel_mask, ch)


def oracle():
    """The plain-C oracle; (re)built when stale."""
    if "oracle" not in _libs:
        o = util.load_oracle(ORACLE_SO)
        o.orc_level.argtypes = [_fp, _sz, _sz, _i, _d, _d, _d, _u]
        o.orc_levelize.argtypes = [_fp, _sz, _sz, _i, _d, _d, _d, _u]
        o.orc_minmax_stretch.argtypes = [_fp, _sz, _sz, _i, _d, _d, _d, _i, _u]
        o.orc_identify_gray.argtypes = [_fp, _sz, _sz, _i]
        o.orc_contrast_stretch.argtypes = [_fp, _sz, _sz, _i, _d, _d, _i, _u, C.c_char_p]
        o.orc_linear_stretch.argtypes = [_fp, _sz, _sz, _i, _d, _d, _u, C.c_char_p]
        o.orc_gamma.argtypes = [_fp, _sz, _sz, _i, _d, _u]
        _libs["oracle"] = o
    return _libs["oracle"]


def ref():
    """The real reference's operators; only where oracle/_ref has been built from a reference source tree."""
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        r.ref_level_op.argtypes = [_fp, _sz, _sz, _i, _i, _d, _d, _d, C.c_long, C.c_char_p, C.POINTER(_d)]
        _libs["ref"] = r
    return _libs["ref"]


def ref_run(src, op, a=0.0, b=0.0, g=1.0, mask=-1):
    """(pixels, property) the reference leaves."""
    h, w, ch = src.shape
    buf = src.copy()
    prop = C.create_string_buffer(64)
    out_ch = ref().ref_level_op(util.P(buf), w, h, ch, op, a, b, g, mask, prop, None)
    assert out_ch > 0, out_ch
    return buf.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy(), prop.value.decode()


def orc_run(src, op, a=0.0, b=0.0, g=1.0, mask=-1):
    """(pixels, property) of the oracle, with the reference driver's operator numbering and ChannelType mask."""
    h, w, ch = src.shape
    buf = src.copy()
    prop = C.create_string_buffer(64)
    um, per = update_mask(mask, ch), int(mask >= 0)
    n = float(w * h)
    o, out_ch = oracle(), ch
    if op == LEVEL:
        assert o.orc_level(util.P(buf), w, h, ch, a, b, g, um) == 0
    elif op == LEVELIZE:
        assert o.orc_levelize(util.P(buf), w, h, ch, a, b, g, um) == 0
    elif op in (MINMAX, AUTO_LEVEL):
        if op == AUTO_LEVEL:
            a, b, g = 0.0, 0.0, 1.0
        assert o.orc_minmax_stretch(util.P(buf), w, h, ch, a, b, g, per, um) == 0
    elif op in (CONTRAST_STRETCH, NORMALIZE):
        if op == NORMALIZE:
            a, b = 0.02 * n, 0.99 * n
        out_ch = o.orc_contrast_stretch(util.P(buf), w, h, ch, a, b, per, um, prop)
        assert out_ch in (1, 2, 3, 4)
    elif op == LINEAR_STRETCH:
        assert o.orc_linear_stretch(util.P(buf), w, h, ch, a, b, um, prop) == 0
    elif op == GAMMA:
        assert o.orc_gamma(util.P(buf), w, h, ch, g, um) == 0
    return buf.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy(), prop.value.decode()


def result_key(pixels, prop) -> str:
    return f"{digest(pixels)}/{pixels.shape[2]}/{prop}"


_store = util.ReferenceStore(DIGESTS, REF_SO)


def reference(case: str, run):
    """What the reference computed for `case` of the running test, as result_key() of the (pixels, property) run()
    returns with the reference itself when recording."""
    return _store(case, lambda: result_key(*run()))
