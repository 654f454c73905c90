"""Inputs, parameter sets and checkers shared by the enhance operator tests (ContrastImage, ModulateImage,
GrayscaleImage, FunctionImage): the oracle-against-reference suite and the GPU suite run the same cases.

The oracle is oracle/enhance_oracle.c (oracle/libenhance_oracle.so) and the reference driver oracle/ref_enhance.c
(oracle/_ref/libmagickref_enhance.so), both built by oracle/Makefile.  What the reference computed for every case is
stored as a digest (util.digest) in tests/golden/enhance_digests.json, keyed like util.reference keys
tests/golden/ref_digests.json; re-record it with MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C

import numpy as np

import util
from util import ROOT, digest, make_image

ORACLE_SO = ROOT / "oracle" / "libenhance_oracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_enhance.so"
DIGESTS = ROOT / "tests" / "golden" / "enhance_digests.json"
_libs = {}

_fp, _dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
_sz, _i, _d = C.c_size_t, C.c_int, C.c_double

SRGB, RGB, GRAY, LINEAR_GRAY = 23, 21, 3, 33
HCL, HCLP, HSB, HSI, HSL, HSV, HWB, LAB, LCH, LCHAB, LCHUV = 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14
ILLUMINANTS = {"A": 0, "D50": 3, "D65": 5}
# "modulate:colorspace" artifact -> the ColorspaceType the operator uses (anything but the nine spaces is HSL)
MODULATE_SPACES = {"HCL": HCL, "HCLp": HCLP, "HSB": HSB, "HSI": HSI, "HSL": HSL, "HSV": HSV, "HWB": HWB, "LCH": LCH,
                   "LCHab": LCHAB, "LCHuv": LCHUV, "Lab": HSL, None: HSL}
# every brightness / saturation of 0, 50, 150, 200 and every hue of 0, 50, 100, 150, 199, 300 appears
GEOMETRIES = ["0,50,0", "50,0,50", "150,200,100", "200,150,150", "100,100,199", "80,120,300"]

UNDEFINED, ARCSIN, ARCTAN, POLYNOMIAL, SINUSOID = range(5)
# (function, parameters): 0-5 parameters of each, Arcsin at width 0 and pegged at +-1, a sinusoid at frequency 1000,
# polynomials of 1-8 terms
FUNCTION_CASES = (
    [(UNDEFINED, []), (UNDEFINED, [0.3, 0.7])]
    + [(POLYNOMIAL, [0.5, -1.25, 0.75, 2.0, -0.375, 0.125, 1.5, -0.0625][:k]) for k in range(1, 9)]
    + [(SINUSOID, [3.0, 45.0, 0.4, 0.55, 7.0][:k]) for k in range(6)] + [(SINUSOID, [1000.0, 10.0])]
    + [(ARCSIN, [0.8, 0.45, 0.9, 0.4, 3.0][:k]) for k in range(6)]
    + [(ARCSIN, [0.0, 0.5]), (ARCSIN, [0.25, 0.5, 1.0, 0.5]), (ARCSIN, [1.0, 0.0, 1.0, 0.5])]
    + [(ARCTAN, [4.0, 0.6, 0.8, 0.45, -2.0][:k]) for k in range(6)]
)
POLYNOMIAL_33 = (POLYNOMIAL, [((k * 7) % 11 - 5) / 8.0 for k in range(33)])
# ChannelType masks of the reference (pixel.h: Red / Gray 0x1, Green 0x2, Blue 0x4, Alpha 0x10): -1 = the default
CHANNEL_MASKS = {"all": -1, "R": 0x1, "RGB": 0x7, "alpha": 0x10}


def update_mask(channel_type: int, ch: int) -> int:
    """The Update channels (bit c = channel c) a ChannelType mask leaves on a `ch`-channel image (alpha is last)."""
    if channel_type < 0:
        return (1 << ch) - 1
    colour = [0x1, 0x2, 0x4][: (1 if ch < 3 else 3)]
    bits = [bool(channel_type & m) for m in colour]
    if ch in (2, 4):
        bits.append(bool(channel_type & 0x10))
    return sum(1 << c for c, on in enumerate(bits) if on)


def mosaic(w: int, ch: int, seed: int = 11) -> np.ndarray:
    """Rows of noise, alpha_blocks, hdr (negative and > 65535), gray pixels (r = g = b, black and white among them) and
    NaN / +-inf samples, stacked into one image `w` columns wide."""
    parts = [make_image(w, 5, ch, seed=seed), make_image(w, 6, ch, seed=seed + 1, kind="alpha_blocks"),
             make_image(w, 5, ch, seed=seed + 2, kind="hdr")]
    gray = make_image(w, 4, ch, seed=seed + 3)
    gray[..., 1:min(ch, 3)] = gray[..., :1]
    gray[0, ::2, :min(ch, 3)] = 0.0
    gray[0, 1::2, :min(ch, 3)] = 65535.0
    gray[1, ::3, :min(ch, 3)] = 32768.0
    parts.append(gray)
    odd = make_image(w, 3, ch, seed=seed + 4)
    for k, value in enumerate([np.nan, np.inf, -np.inf]):
        odd[k, k::3, k % ch] = value
        odd[(k + 1) % 3, (k + 1)::4, ch - 1] = value
    parts.append(odd)
    return np.ascontiguousarray(np.concatenate(parts, axis=0))


def oracle():
    """The plain-C oracle; (re)built when stale, like conftest.py does for oracle/liboracle.so."""
    if "oracle" not in _libs:
        o = util.load_oracle(ORACLE_SO)
        o.orc_contrast.argtypes = [_fp, _sz, _sz, _i, _i]
        o.orc_modulate.argtypes = [_fp, _sz, _sz, _i, _d, _d, _d, _i, _i]
        o.orc_grayscale.argtypes = [_fp, _sz, _sz, _i, _i, _i]
        o.orc_function.argtypes = [_fp, _sz, _sz, _i, _i, _sz, _dp, C.c_uint]
        _libs["oracle"] = o
    return _libs["oracle"]


def ref():
    """The real reference's operators; only where oracle/_ref has been built from a reference source tree."""
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        r.ref_contrast.argtypes = [_fp, _sz, _sz, _i, _i, _i]
        r.ref_modulate.argtypes = [_fp, _sz, _sz, _i, _i, C.c_char_p, C.c_char_p]
        r.ref_grayscale.argtypes = [_fp, _sz, _sz, _i, _i, _i]
        r.ref_function.argtypes = [_fp, _sz, _sz, _i, _i, _sz, _dp, C.c_long]
        _libs["ref"] = r
    return _libs["ref"]


_store = util.ReferenceStore(DIGESTS, REF_SO)


def reference(case: str, run):
    """Digest of what the reference computed for `case` of the running test: of the output array run() returns with
    the reference itself when recording."""
    return _store(case, lambda: digest(run()))


def modulate_percentages(geometry: str):
    parts = geometry.split(",")
    vals = [float(v) for v in parts[0].split("x", 1) + parts[1:]]
    return (vals + [100.0, 100.0])[:3]


def modulate_settings(space, illuminant=None):
    """(colorspace, illuminant) the operator uses for the artifacts: an unparsable illuminant resets the space to HSL."""
    cs = MODULATE_SPACES.get(space, HSL)
    if illuminant is None:
        return cs, 5
    if illuminant not in ILLUMINANTS:
        return HSL, 5
    return cs, ILLUMINANTS[illuminant]


def artifacts(space, illuminant=None) -> bytes:
    parts = []
    if space is not None:
        parts.append(f"modulate:colorspace={space}")
    if illuminant is not None:
        parts.append(f"color:illuminant={illuminant}")
    return ";".join(parts).encode()


def orc_contrast(src, sharpen):
    h, w, ch = src.shape
    out = src.copy()
    assert oracle().orc_contrast(util.P(out), w, h, ch, int(sharpen)) == 0
    return out


def orc_modulate(src, geometry, space=None, illuminant=None):
    h, w, ch = src.shape
    out = src.copy()
    cs, ill = modulate_settings(space, illuminant)
    assert oracle().orc_modulate(util.P(out), w, h, ch, *modulate_percentages(geometry), cs, ill) == 0
    return out


def orc_grayscale(src, method, colorspace):
    h, w, ch = src.shape
    buf = src.copy()
    out_ch = oracle().orc_grayscale(util.P(buf), w, h, ch, method, colorspace)
    assert out_ch in (1, 2)
    return buf.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy()


def orc_function(src, function, params, mask):
    h, w, ch = src.shape
    out = src.copy()
    arr = (C.c_double * max(1, len(params)))(*params)
    assert oracle().orc_function(util.P(out), w, h, ch, function, len(params), arr, update_mask(mask, ch)) == 0
    return out
