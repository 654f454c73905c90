"""Cases and runners shared by the tests of DistortImage / RotateImage: the planner-against-reference suite on the CPU and
the GPU suite run the same cases.

The reference driver is oracle/ref_distort.c (oracle/_ref/libmagickref_distort.so, built by oracle/distort.mk).  What the
reference computed for every case is stored in tests/golden/distort_digests.json as "columns/rows/page_x/page_y/
channels/digest", keyed by case name; re-record it with MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C
import json
import os

import numpy as np

import util
from util import ROOT, digest, make_image

REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_distort.so"
DIGESTS = ROOT / "tests" / "golden" / "distort_digests.json"
_libs = {}

AFFINE, AFFINE_PROJECTION, SRT, PERSPECTIVE, PERSPECTIVE_PROJECTION, RIGID_AFFINE = 1, 2, 3, 4, 5, 19
ROTATE = 0
BACKGROUND, EDGE, TRANSPARENT, BLACK, GRAY, WHITE_VP = 1, 3, 7, 9, 10, 11
QR = 65535.0
OPAQUE_BG = (QR, QR, QR, QR)
GRAY_BG = (20000.0, 20000.0, 20000.0, QR)
NONE_BG = (0.0, 0.0, 0.0, 0.0)                 # -background none
MATTE = (48573.0, 48573.0, 48573.0, QR)

# method -> argument lists: every argument-count branch of GenerateCoefficients
MAPS = {
    "affine1": (AFFINE, [3.0, 2.0, 5.5, 7.25]),
    "affine2": (AFFINE, [0, 0, 2, 1, 20, 0, 21, 5]),
    "affine3": (AFFINE, [0, 0, 1, 2, 20, 0, 22, 3, 0, 20, -1, 23]),
    "affine5": (AFFINE, [0, 0, 1, 2, 20, 0, 22, 3, 0, 20, -1, 23, 20, 20, 21.5, 26, 10, 10, 11, 12.5]),
    "affine_projection": (AFFINE_PROJECTION, [0.9, 0.3, -0.2, 1.1, 3.5, -2.0]),
    "rigid2": (RIGID_AFFINE, [0, 0, 2, 1, 20, 0, 21, 5]),
    "rigid3": (RIGID_AFFINE, [0, 0, 2, 1, 20, 0, 21, 5, 0, 20, -3, 19]),
    "srt1": (SRT, [30.0]),
    "srt2": (SRT, [0.5, 30.0]),
    "srt3": (SRT, [10.0, 8.0, -20.0]),
    "srt4": (SRT, [10.0, 8.0, 2.0, 15.0]),
    "srt5": (SRT, [10.0, 8.0, 1.5, 0.75, 60.0]),
    "srt6": (SRT, [10.0, 8.0, 0.8, 45.0, 12.0, 9.0]),
    "srt7": (SRT, [10.0, 8.0, 1.2, 0.6, -33.0, 2.0, 3.0]),
    "perspective": (PERSPECTIVE, [0, 0, 3, 2, 36, 0, 30, 4, 0, 28, 1, 25, 36, 28, 33, 27]),
    "perspective3": (PERSPECTIVE, [0, 0, 3, 2, 36, 0, 30, 4, 0, 28, 1, 25]),
    "perspective_projection": (PERSPECTIVE_PROJECTION, [1.2, 0.1, 2.0, 0.05, 0.9, -1.0, 0.004, 0.002]),
    "horizon": (PERSPECTIVE_PROJECTION, [1.0, 0.2, 0.0, 0.0, 1.0, 0.0, 0.0, -0.045]),
    "minify": (SRT, [0.04, 10.0]),
    "magnify": (SRT, [3.0, 20.0]),
}
ANGLES = [30.0, -45.5, 89.9, 135.0, 200.0]
FILTERS = [f for f in range(0, 34) if f != 1]           # every FilterType but Point
VPS = [0, BACKGROUND, EDGE, TRANSPARENT, BLACK, GRAY, WHITE_VP]


def sources(ch: int, w: int = 37, h: int = 29, seed: int = 5):
    """name -> image: noise, alpha blocks, HDR, +-inf / NaN samples, and 1x1, 1xN, Nx1 images."""
    spec = make_image(w, h, ch, seed=seed + 3, kind="hdr")
    rng = np.random.default_rng(seed)
    for value in (np.inf, -np.inf, np.nan):
        spec.ravel()[rng.integers(0, spec.size, size=spec.size // 60)] = value
    return {"noise": make_image(w, h, ch, seed=seed), "alpha": make_image(w, h, ch, seed=seed + 1, kind="alpha_blocks"),
            "hdr": make_image(w, h, ch, seed=seed + 2, kind="hdr"), "specials": spec,
            "1x1": make_image(1, 1, ch, seed=seed + 4), "1xN": make_image(1, 13, ch, seed=seed + 5),
            "Nx1": make_image(15, 1, ch, seed=seed + 6)}


def ref():
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        _fp, _dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
        r.ref_distort.argtypes = [_fp, C.c_size_t, C.c_size_t, C.c_int, C.c_long, C.c_long, C.c_int, _dp, C.c_size_t,
                                  C.c_int, C.c_int, C.c_int, C.c_int, _dp, C.c_int, _dp, C.c_int, C.c_char_p, _fp,
                                  C.c_size_t, C.POINTER(C.c_long)]
        _libs["ref"] = r
    return _libs["ref"]


def _d(values):
    return (C.c_double * max(1, len(values)))(*[float(v) for v in values])


def run_ref(src, method, args, bestfit=False, filter=0, vp=0, bg=OPAQUE_BG, bg_alpha=False, matte=MATTE,
            page=(0, 0), viewport=None, scale=None, artifacts=None, interpolate=0, matte_alpha=False):
    """(pixels, (columns, rows, page_x, page_y)) the reference returns, or None where it returns no image."""
    h, w, ch = src.shape
    lines = dict(artifacts or {})
    if viewport is not None:
        lines["distort:viewport"] = "%dx%d%+d%+d" % tuple(viewport)
    if scale is not None:
        lines["distort:scale"] = repr(float(scale))
    text = "\n".join(f"{k}={v}" for k, v in lines.items()).encode() or None
    cap = (1 << 22) + 16 * src.size
    out = np.empty(cap, np.float32)
    geom = (C.c_long * 4)()
    src = np.ascontiguousarray(src, np.float32)
    n = ref().ref_distort(util.P(src), w, h, ch, page[0], page[1], method, _d(args), len(args), int(bestfit), filter,
                          interpolate, vp, _d(bg), int(bg_alpha), _d(matte), int(matte_alpha), text, util.P(out), cap, geom)
    if n <= 0:
        return None
    cols, rows = geom[0], geom[1]
    return out[: cols * rows * n].reshape(rows, cols, n).copy(), tuple(geom)


def key(result) -> str:
    if result is None:
        return "none"
    pixels, g = result
    return f"{g[0]}/{g[1]}/{g[2]}/{g[3]}/{pixels.shape[2]}/{digest(pixels)}"


_stored = None
_recorded = {}


def _save_recorded():
    data = json.loads(DIGESTS.read_text()) if DIGESTS.exists() else {}
    data.update(_recorded)
    DIGESTS.write_text("{\n" + ",\n".join(json.dumps(k) + ": " + json.dumps(v) for k, v in sorted(data.items())) + "\n}\n")


def reference(case: str, run) -> str:
    """What the reference computed for `case`, as key().  With MB200_RECORD_REFERENCE=1 and the reference driver built,
    run() computes it with the reference itself and the result is recorded when the process exits."""
    global _stored
    if os.environ.get("MB200_RECORD_REFERENCE") == "1" and REF_SO.exists():
        if not _recorded:
            import atexit
            atexit.register(_save_recorded)
        _recorded[case] = key(run())
        return _recorded[case]
    if _stored is None:
        _stored = json.loads(DIGESTS.read_text())
    assert case in _stored, f"no stored reference result for {case}"
    return _stored[case]


def cases():
    """name -> (src, kwargs of run_ref).  Each case is one the library serves: the image already has the channels of
    the reference's result (an opaque alpha is added where a Transparent virtual pixel or a background with alpha
    gives the result one)."""
    out = {}
    for ch in (1, 2, 3, 4):
        srcs = sources(ch)
        for name, (method, args) in MAPS.items():
            for sname, src in srcs.items():
                kw = dict(method=method, args=args, bestfit=name.startswith(("srt", "affine_p", "perspective_p")))
                if name == "horizon" and ch in (1, 3):
                    continue                  # the reference blends the horizon with an alpha carried along the row
                out[f"{name} {sname} ch{ch}"] = (src, kw)
        src = srcs["noise"]
        for deg in ANGLES:
            out[f"rotate {deg} ch{ch}"] = (src, dict(method=ROTATE, args=[deg], bg=GRAY_BG))
        for f in FILTERS:
            out[f"filter {f} ch{ch}"] = (src, dict(method=SRT, args=[0.7, 25.0], filter=f))
        for vp in VPS:
            for bname, bg in (("opaque", GRAY_BG), ("none", NONE_BG)):
                if (vp == TRANSPARENT or bname == "none") and ch in (1, 3):
                    continue
                out[f"vp {vp} {bname} ch{ch}"] = (srcs["alpha"], dict(method=SRT, args=[1.3, 40.0], vp=vp, bg=bg,
                                                                      bg_alpha=bname == "none", bestfit=True))
        out[f"viewport ch{ch}"] = (src, dict(method=SRT, args=[20.0], viewport=(30, 20, -5, 3)))
        for sc in (0.5, 2.0):
            out[f"scale {sc} ch{ch}"] = (src, dict(method=SRT, args=[20.0], scale=sc, bestfit=True))
        out[f"page ch{ch}"] = (src, dict(method=SRT, args=[15.0], bestfit=True, page=(4, -3)))
        out[f"page nobestfit ch{ch}"] = (src, dict(method=SRT, args=[15.0], page=(4, -3)))
        # Bilinear interpolate where EWA finds no weight, a matte colour with an alpha trait on the horizon, the
        # filter:* expert settings through the cylindrical filter, and the alpha channel the reference adds
        out[f"bilinear ch{ch}"] = (srcs["specials"], dict(method=SRT, args=[0.04, 10.0], interpolate=5, vp=EDGE))
        if ch in (2, 4):
            out[f"matte alpha ch{ch}"] = (srcs["noise"], dict(method=PERSPECTIVE_PROJECTION, args=MAPS["horizon"][1],
                                                               bestfit=True, matte=(9000.0, 9000.0, 9000.0, 30000.0),
                                                               matte_alpha=True))
        for i, art in enumerate(({"filter:blur": "0.8"}, {"filter:window": "Hann", "filter:lobes": "2"},
                                 {"filter:support": "1.5"}, {"filter:b": "0.2", "filter:c": "0.4"},
                                 {"filter:sigma": "0.8"})):
            out[f"artifacts {i} ch{ch}"] = (src, dict(method=SRT, args=[0.8, 20.0], artifacts=art,
                                                      filter=8 if "filter:sigma" in art else 0))
        if ch in (1, 3):
            out[f"gains alpha bg none ch{ch}"] = (src, dict(method=ROTATE, args=[30.0], bg=NONE_BG, bg_alpha=True))
            out[f"gains alpha transparent ch{ch}"] = (src, dict(method=SRT, args=[1.3, 40.0], vp=TRANSPARENT,
                                                               bestfit=True))
    # images of many CTAs (128 threads along x) and rows
    out["large rotate 1000x700 ch4"] = (make_image(1000, 700, 4, seed=11, kind="alpha_blocks"),
                                        dict(method=ROTATE, args=[30.0], bg=GRAY_BG))
    out["large perspective 2048 ch4"] = (make_image(2048, 2048, 4, seed=12),
                                         dict(method=PERSPECTIVE, bestfit=True, vp=EDGE,
                                              args=[0, 0, 100, 150, 2047, 0, 1800, 60, 0, 2047, -200, 1900,
                                                    2047, 2047, 2200, 2000]))
    out["large horizon 1536x1024 ch4"] = (make_image(1536, 1024, 4, seed=13, kind="alpha_blocks"),
                                          dict(method=PERSPECTIVE_PROJECTION, bestfit=False,
                                               args=[1.0, 0.3, 0.0, 0.0, 1.0, 0.0, 0.0, -0.0012]))
    return out


def run_lib(src, method, args, bestfit=False, filter=0, vp=0, bg=OPAQUE_BG, bg_alpha=False, matte=MATTE,
            page=(0, 0), viewport=None, scale=None, artifacts=None, interpolate=0, matte_alpha=False, device=False):
    """The library's result for the same case, as (pixels, (columns, rows, page_x, page_y))."""
    import imagemagick_b200 as im
    if device:
        import torch
        image = im.Image(torch.from_numpy(np.ascontiguousarray(src)).cuda())
    else:
        image = im.Image(src)
    image.page = page
    bgc = tuple(bg) if bg_alpha else tuple(bg[:3])
    matte = tuple(matte) if matte_alpha else tuple(matte[:3])
    if method == ROTATE:
        out = im.RotateImage(image, args[0], background=bgc, filter=filter, matte_color=matte)
    else:
        out = im.DistortImage(image, method, args, bestfit, filter=filter, virtual_pixel=vp, background=bgc,
                              matte_color=matte, viewport=viewport, scale=scale, artifacts=artifacts,
                              interpolate=interpolate)
    pixels = out.pixels.cpu().numpy() if device else out.pixels
    return pixels, (out.columns, out.rows, out.page[0], out.page[1])


def plan_geometry(src, method, args, bestfit=False, page=(0, 0), viewport=None, scale=None, **_):
    """(columns, rows, page_x, page_y) of the host planner."""
    import imagemagick_b200 as im
    image = im.Image(src)
    image.page = page
    if method == ROTATE:
        plan = im.DistortParams()
        util_check = im._lib.load().mb200_rotate_plan(float(args[0]), image.columns, image.rows, page[0], page[1],
                                                       C.byref(plan))
        im._lib.check(util_check)
    else:
        plan = im.DistortPlan(image, method, args, bestfit, viewport, scale)
    return (plan.columns, plan.rows, plan.page_x, plan.page_y)
