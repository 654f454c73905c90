"""Inputs and runners shared by the tests of TransformImageColorspace to and from the colourspaces that change the channel
layout (GRAY, LinearGRAY, CMYK): the oracle-against-reference suite and the GPU suite run the same cases.

The oracle is oracle/layout_oracle.c (oracle/liblayout_oracle.so) and the reference driver oracle/ref_layout.c
(oracle/_ref/libmagickref_layout.so), both built by oracle/layout.mk.  What the reference computed for every case is
stored as a digest (util.digest) in tests/golden/layout_digests.json, keyed like enhance_cases keys its own file;
re-record it with MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import atexit
import ctypes as C
import json
import os
import subprocess

import numpy as np

import enhance_cases
import util
from util import ROOT, digest, make_image

ORACLE_SO = ROOT / "oracle" / "liblayout_oracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_layout.so"
DIGESTS = ROOT / "tests" / "golden" / "layout_digests.json"
_libs = {}

_fp = C.POINTER(C.c_float)
_sz, _i = C.c_size_t, C.c_int

CMYK, GRAY, LINEAR_GRAY, SRGB, RGB, LAB, XYZ = 2, 3, 33, 23, 21, 11, 26
HSL, LCHAB, LUV, YIQ, LOG, YCC = 8, 13, 17, 30, 15, 28
LAYOUT = [GRAY, LINEAR_GRAY, CMYK]
NAMES = {CMYK: "CMYK", GRAY: "GRAY", LINEAR_GRAY: "LinearGRAY", SRGB: "sRGB", RGB: "RGB", LAB: "Lab", XYZ: "XYZ",
         HSL: "HSL", LCHAB: "LCHab", LUV: "Luv", YIQ: "YIQ", LOG: "Log", YCC: "YCC"}
# one space of each route family of the in-place legs: core (Lab, XYZ, RGB), hexcone, XYZ family, matrix, Log, YCC
HOP_SPACES = [LAB, XYZ, RGB, HSL, LCHAB, LUV, YIQ, LOG, YCC]


def channels(colorspace: int, alpha: bool) -> int:
    return (4 if colorspace == CMYK else 1 if colorspace in (GRAY, LINEAR_GRAY) else 3) + int(alpha)


def source(colorspace: int, alpha: bool, w: int = 37, seed: int = 11) -> np.ndarray:
    """enhance_cases.mosaic in the layout of `colorspace` (noise, alpha blocks, HDR, gray pixels, NaN / +-inf), plus rows
    of exact black, near-black (every colour sample below QuantumRange * MagickEpsilon: only K changes in sRGB -> CMYK)
    and samples just above that threshold."""
    ch = channels(colorspace, alpha)
    parts = []
    for c0 in range(0, ch, 4):             # the mosaic has at most four channels: CMYKA takes two, side by side
        parts.append(enhance_cases.mosaic(w, min(4, ch - c0), seed=seed + c0))
    img = np.concatenate(parts, axis=2)
    dark = make_image(w, 3, ch, seed=seed + 9)
    colour = ch - int(alpha)
    dark[0, :, :colour] = 0.0
    dark[1, :, :colour] = np.float32(3e-8) * np.arange(w, dtype=np.float32)[:, None] % np.float32(6.5e-8)
    dark[2, :, :colour] = np.float32(6.6e-8)
    dark[2, ::2, :colour] = -np.float32(6.0e-8)
    return np.ascontiguousarray(np.concatenate([img, dark], axis=0).astype(np.float32))


def oracle():
    """The plain-C oracle; (re)built when stale."""
    if "oracle" not in _libs:
        srcs = [ROOT / "oracle" / n for n in ("layout_oracle.c", "oracle.c", "oracle.h")]
        if not ORACLE_SO.exists() or any(ORACLE_SO.stat().st_mtime < s.stat().st_mtime for s in srcs):
            env = dict(os.environ)
            env.pop("CC", None)
            subprocess.run(["make", "-C", str(ROOT / "oracle"), "-f", "layout.mk", "port"], check=True, env=env,
                           stdout=subprocess.DEVNULL)
        o = C.CDLL(str(ORACLE_SO))
        o.orc_colorspace_channels.argtypes = [_i, _i]
        o.orc_colorspace_layout.argtypes = [_fp, _i, _fp, _i, _sz, _sz, _i, _i, C.c_void_p]
        _libs["oracle"] = o
    return _libs["oracle"]


def ref():
    """The real reference's TransformImageColorspace; only where oracle/_ref has been built from a reference source tree."""
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        r.ref_colorspace_layout.argtypes = [_fp, _fp, _sz, _sz, _i, _i, _i, C.c_char_p, C.POINTER(_i)]
        _libs["ref"] = r
    return _libs["ref"]


def options(settings):
    """orc_colorspace_options (== mb200_colorspace_options) of a settings dict, by the Python API's own parse."""
    from imagemagick_b200.api import colorspace_options_from_settings
    o = colorspace_options_from_settings(settings)
    return None if o is None else C.byref(o)


def orc_layout(src, from_cs, to_cs, settings=None):
    h, w, ch = src.shape
    out = np.empty((h, w, channels(to_cs, ch != channels(from_cs, False))), np.float32)
    assert oracle().orc_colorspace_layout(util.P(src), ch, util.P(out), out.shape[2], w, h, from_cs, to_cs,
                                          options(settings)) == 0
    return out


def ref_layout(src, from_cs, to_cs, settings=None):
    """(pixels, image type) the reference leaves."""
    h, w, ch = src.shape
    out = np.empty((h, w, 5), np.float32)
    kind = C.c_int(-1)
    defines = ";".join(f"{k}={v}" for k, v in (settings or {}).items()).encode()
    out_ch = ref().ref_colorspace_layout(util.P(src), util.P(out), w, h, ch, from_cs, to_cs, defines, C.byref(kind))
    assert out_ch > 0, out_ch
    return out.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy(), kind.value


_stored = None
_recorded = {}


def _save_recorded():
    data = json.loads(DIGESTS.read_text()) if DIGESTS.exists() else {}
    for (test, case), value in _recorded.items():
        data.setdefault(test, {})[case] = value
    DIGESTS.write_text("{\n" + ",\n".join(json.dumps(t) + ": " + json.dumps(c, separators=(",", ":"))
                                           for t, c in sorted(data.items())) + "\n}\n")


def reference(case: str, run):
    """What the reference computed for `case` of the running test: the digest of its pixels and the image type, as
    "digest/type".  With MB200_RECORD_REFERENCE=1 and the reference driver built, run() computes it with the reference
    itself and the result is recorded when the process exits."""
    global _stored
    test = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0].split("::", 1)
    test = test[0].rsplit("/", 1)[-1] + "::" + test[-1]
    if os.environ.get("MB200_RECORD_REFERENCE") == "1" and REF_SO.exists():
        if not _recorded:
            atexit.register(_save_recorded)
        pixels, kind = run()
        _recorded[test, case] = f"{digest(pixels)}/{kind}"
        return _recorded[test, case]
    if _stored is None:
        _stored = json.loads(DIGESTS.read_text())
    stored = _stored.get(test, {})
    assert case in stored, f"no stored reference result for {test} / {case}"
    return stored[case]


# ImageType (MagickCore/image.h:38-51) the reference leaves for a layout target: GrayscaleType for GRAY / LinearGRAY,
# ColorSeparation[Alpha]Type for CMYK (every other target keeps the image's type; the shim harness checks that case)
GRAYSCALE, COLOR_SEPARATION, COLOR_SEPARATION_ALPHA = 2, 8, 9


def expected_type(to_cs, alpha):
    if to_cs == CMYK:
        return COLOR_SEPARATION_ALPHA if alpha else COLOR_SEPARATION
    return GRAYSCALE
