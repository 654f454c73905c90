"""Inputs, parameter sets and runners shared by the tests of AdaptiveThresholdImage, AutoThresholdImage,
RangeThresholdImage and PerceptibleImage: the oracle-against-reference suite and the GPU suite run the same cases.

The oracle is oracle/threshold_oracle.c (oracle/libthreshold_oracle.so) and the reference driver oracle/ref_threshold.c
(oracle/_ref/libmagickref_threshold.so), both built by oracle/Makefile.  What the reference computed for every case
is stored in tests/golden/threshold_digests.json as "digest/channels/property"; re-record it with
MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C

import numpy as np

import enhance_cases
import util
from util import ROOT, digest, make_image

ORACLE_SO = ROOT / "oracle" / "libthreshold_oracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_threshold.so"
DIGESTS = ROOT / "tests" / "golden" / "threshold_digests.json"
_libs = {}

_fp, _dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
_sz, _i, _d, _u = C.c_size_t, C.c_int, C.c_double, C.c_uint

# ref_threshold_op's operator numbers
ADAPTIVE, AUTO, RANGE, PERCEPTIBLE = range(4)
QR = 65535.0

# ChannelType masks (Red / Gray 0x1, Green 0x2, Blue 0x4, Alpha 0x10); -1 = the default mask (AllChannels)
CHANNEL_MASKS = {"all": -1, "RGB": 0x7, "R": 0x1, "GB": 0x6, "alpha": 0x10, "RGBA": 0x17}

# (width, height, bias) of AdaptiveThresholdImage: 1x1, 1xN, Nx1, odd and even, larger than the images, +-0 bias
WINDOWS = [(1, 1, 0.0), (1, 5, 0.0), (6, 1, 100.0), (3, 3, 0.0), (4, 4, -500.0), (5, 3, QR * 0.05), (8, 6, 0.0),
           (15, 15, QR * 0.05), (40, 33, -1000.0), (0, 3, 0.0), (3, 0, 0.0)]

AUTO_METHODS = [0, 1, 2, 3]          # Undefined (OTSU), Kapur, OTSU, Triangle
OTSU = 2

# (low_black, low_white, high_white, high_black) of RangeThresholdImage
RANGES = [(10000.0, 20000.0, 40000.0, 50000.0), (0.0, 0.0, 65535.0, 65535.0), (30000.0, 30000.0, 30000.0, 30000.0),
          (-100.0, 50.5, 60000.0, 70000.0)]
EPSILONS = [0.0, 1.0, 1.0e-3, 1000.0, -5.0, 1.0e-40]


def sources(ch: int, w: int = 23, seed: int = 5):
    """name -> image: enhance_cases.mosaic (noise, alpha blocks, HDR, gray pixels, NaN / +-inf), NaN early in a row,
    +-inf (inf - inf in the running sum), posterised 8-bit levels with ties at the mean, and 1x1 / 1xN / Nx1 images."""
    out = {"mosaic": enhance_cases.mosaic(w, ch, seed=seed)}
    nan = make_image(w, 9, ch, seed=seed + 1)
    nan[2, 1, :] = np.nan
    nan[5, 0, 0] = np.nan
    out["nan"] = nan
    inf = make_image(w, 7, ch, seed=seed + 2, kind="hdr")
    inf[1, 3, :] = np.inf
    inf[1, 9, :] = -np.inf
    inf[4, 0, 0] = np.inf
    out["inf"] = inf
    out["hdr"] = make_image(w, 8, ch, seed=seed + 3, kind="hdr")
    post = make_image(w, 8, ch, seed=seed + 4)
    out["posterised"] = (np.floor(post / 257.0 / 64.0) * 64.0 * 257.0).astype(np.float32)
    out["flat"] = np.full((5, w, ch), 257.0 * 100, np.float32)
    out["1x1"] = make_image(1, 1, ch, seed=seed + 5)
    out["1xN"] = make_image(1, 17, ch, seed=seed + 6, kind="hdr")
    out["Nx1"] = make_image(19, 1, ch, seed=seed + 7)
    return out


def auto_sources(ch: int, seed: int = 3):
    """AutoThreshold's images: bimodal, flat, single level, all NaN, and intensities a few float steps either side of
    every bin edge 257k + 128.5."""
    rng = np.random.default_rng(seed)
    out = {}
    bi = np.where(rng.random((12, 20, 1)) < 0.4, rng.normal(12000, 3000, (12, 20, 1)), rng.normal(50000, 4000, (12, 20, 1)))
    out["bimodal"] = np.repeat(bi, ch, axis=2).astype(np.float32)
    out["flat"] = make_image(20, 12, ch, seed=seed, kind="gradient")
    out["single"] = np.full((6, 7, ch), 30000.0, np.float32)
    out["all nan"] = np.full((4, 5, ch), np.nan, np.float32)
    edges = np.float32(257.0 * np.arange(256) + 128.5)
    vals = [np.nextafter(edges, np.float32(d * np.inf)) if d else edges for d in (-1, 0, 1)]
    vals += [np.nextafter(vals[0], np.float32(-np.inf)), np.nextafter(vals[2], np.float32(np.inf))]
    gray = np.stack(vals).astype(np.float32).reshape(5 * 256, 1, 1)
    img = np.repeat(gray, ch, axis=2).reshape(40, 32, ch).copy()
    if ch in (2, 4):
        img[..., -1] = 65535.0
    out["bin edges"] = img
    return out


def edge_pairs(ch: int):
    """One 2x1 image per intensity 2 float steps below, 1 below, at, 1 above and 2 above every bin edge 257k + 128.5,
    beside a QuantumRange pixel.  OTSU's threshold of two histogram spikes is the lower spike's bin, so each image's
    threshold is the bin its edge pixel lands in: every edge sample is pinned individually."""
    edges = np.float32(257.0 * np.arange(256) + 128.5)
    below1, above1 = np.nextafter(edges, np.float32(-np.inf)), np.nextafter(edges, np.float32(np.inf))
    vals = [np.nextafter(below1, np.float32(-np.inf)), below1, edges, above1, np.nextafter(above1, np.float32(np.inf))]
    for v in np.stack(vals, axis=1).reshape(-1):
        img = np.full((1, 2, ch), 65535.0, np.float32)
        img[0, 0, : (1 if ch < 3 else 3)] = v
        yield img


def edge_thresholds(run, ch: int):
    """The thresholds `run(image)` returns on every edge_pairs image, as a (1, n, 1) float64 array."""
    return np.array([run(img) for img in edge_pairs(ch)], np.float64).reshape(1, -1, 1)


def range_source(ch: int):
    """Samples exactly at and one float step beside each limit of RANGES[0], plus noise and NaN."""
    base = make_image(16, 6, ch, seed=21, kind="hdr")
    lims = np.array(RANGES[0], np.float32)
    vals = np.concatenate([lims, np.nextafter(lims, np.float32(-np.inf)), np.nextafter(lims, np.float32(np.inf))])
    base.reshape(-1)[: vals.size] = vals
    base[5, 5, :] = np.nan
    return base


def perceptible_source(ch: int):
    """+-0, denormals, +-epsilon and their neighbours, NaN and +-inf among noise."""
    base = make_image(16, 5, ch, seed=31, kind="hdr")
    specials = np.array([0.0, -0.0, 1e-40, -1e-40, 1.0, -1.0, np.nextafter(np.float32(1), np.float32(0)), 1e-3, -1e-3,
                         1000.0, -1000.0, 999.99994, np.nan, np.inf, -np.inf, 5.0, -5.0], np.float32)
    base.reshape(-1)[: specials.size] = specials
    return base


def update_mask(channel_mask: int, ch: int) -> int:
    return enhance_cases.update_mask(channel_mask, ch)


def oracle():
    """The plain-C oracle; (re)built when stale."""
    if "oracle" not in _libs:
        o = util.load_oracle(ORACLE_SO)
        o.orc_adaptive_threshold.argtypes = [_fp, _fp, _sz, _sz, _i, _sz, _sz, _d, _u]
        o.orc_auto_threshold.argtypes = [_fp, _sz, _sz, _i, _i, _dp]
        o.orc_range_threshold.argtypes = [_fp, _sz, _sz, _i, _d, _d, _d, _d, _i, _u]
        o.orc_perceptible.argtypes = [_fp, _sz, _sz, _i, _d, _u]
        _libs["oracle"] = o
    return _libs["oracle"]


def ref():
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        r.ref_threshold_op.argtypes = [_fp, _sz, _sz, _i, _i, _dp, C.c_long, C.c_char_p]
        _libs["ref"] = r
    return _libs["ref"]


def ref_run(src, op, args, mask=-1):
    """(pixels, property) the reference leaves."""
    h, w, ch = src.shape
    buf = np.zeros(w * h * 4, np.float32)
    buf[: src.size] = src.ravel()
    prop = C.create_string_buffer(64)
    a = (C.c_double * 4)(*(list(args) + [0.0] * (4 - len(args))))
    out_ch = ref().ref_threshold_op(util.P(buf), w, h, ch, op, a, mask, prop)
    assert out_ch > 0, out_ch
    return buf[: w * h * out_ch].reshape(h, w, out_ch).copy(), prop.value.decode()


def orc_run(src, op, args, mask=-1):
    """(pixels, property) of the oracle, with the reference driver's operator numbering and ChannelType mask."""
    h, w, ch = src.shape
    buf = src.copy()
    um = update_mask(mask, ch)
    o, prop = oracle(), ""
    if op == ADAPTIVE:
        out = np.empty_like(src)
        assert o.orc_adaptive_threshold(util.P(buf), util.P(out), w, h, ch, int(args[0]), int(args[1]), args[2], um) == 0
        buf = out
    elif op == AUTO:
        t = C.c_double()
        assert o.orc_auto_threshold(util.P(buf), w, h, ch, int(args[0]), C.byref(t)) == 0
        prop = "%g%%" % t.value
    elif op == RANGE:
        assert o.orc_range_threshold(util.P(buf), w, h, ch, *args, int(mask >= 0), um) == 0
    else:
        assert o.orc_perceptible(util.P(buf), w, h, ch, args[0], um) == 0
    return buf, prop


def result_key(pixels, prop) -> str:
    return f"{digest(pixels)}/{pixels.shape[2]}/{prop}"


_store = util.ReferenceStore(DIGESTS, REF_SO)


def reference(case: str, run):
    """What the reference computed for `case` of the running test, as result_key() of the (pixels, property) run()
    returns with the reference itself when recording."""
    return _store(case, lambda: result_key(*run()))
