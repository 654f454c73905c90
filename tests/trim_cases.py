"""Cases and runners shared by the tests of GetImageBoundingBox and TrimImage: the host suite (NumPy row summaries,
mb200_bounding_box_from_rows and mb200_trim_plan) and the GPU suite run the same cases.

The reference driver is oracle/ref_trim.c (oracle/_ref/libmagickref_trim.so, built by oracle/Makefile), run with one
thread (the reference's threaded result depends on the OpenMP schedule; see there).  What the reference computed for
every case is stored in tests/golden/trim_digests.json, keyed by case name: the bounding box and the exception severity afterwards as "width/height/x/y/severity"; for a case that also trims,
under "trim <name>", TrimImage's result in the geometry_cases.key format followed by "/severity".  Re-record it with
MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C

import numpy as np

import geometry_cases as gc
import util
from util import ROOT

REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_trim.so"
DIGESTS = ROOT / "tests" / "golden" / "trim_digests.json"
OPTION_WARNING = 310                     # MagickCore/exception.h: GeometryDoesNotContainImage's severity
_libs = {}

CMYK, HSL, SRGB = 2, 8, 23
# name -> (channels, colourspace)
LAYOUTS = {"gray": (1, SRGB), "ga": (2, SRGB), "rgb": (3, SRGB), "rgba": (4, SRGB), "cmyk": (4, CMYK),
           "cmyka": (5, CMYK), "hsl": (3, HSL)}
ALPHA = {"ga", "rgba", "cmyka"}
# 1x1, 1xN, Nx1, ragged sizes, and one of 512 rows or more (where the reference's threaded result would depend on the
# OpenMP schedule)
SIZES = [(1, 1), (1, 13), (15, 1), (70, 45), (257, 129), (40, 600)]
KINDS = ["equal", "corners", "special frame", "special corners"]
FUZZ = {"0": 0.0, "moderate": 5000.0, "huge": 1.0e12}
EDGES = ["north", "east,west", "North,SOUTH", "north,east,south,west", "bogus", "", " north", "West,nowhere,EAST"]
MIN_SIZES = {"grow": (60, 40), "past the edge": (200, 150), "one side": (80, 5)}
GRAVITIES = range(10)

_SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0, 3.0e6, -2.0e5], np.float32)


def background(layout: str) -> np.ndarray:
    ch, cs = LAYOUTS[layout]
    base = {1: [30000.0], 2: [30000.0, 65535.0], 3: [1000.0, 20000.0, 50000.0], 4: [1000.0, 20000.0, 50000.0, 65535.0],
            5: [1000.0, 2000.0, 3000.0, 40000.0, 65535.0]}[ch]
    if cs == CMYK and ch == 4:
        base = [1000.0, 2000.0, 3000.0, 40000.0]
    if cs == HSL:
        base = [100.0, 30000.0, 40000.0]        # hue just above 0: the object's hues wrap around QuantumRange
    return np.array(base, np.float32)


def source(layout: str, size, kind: str, seed: int = 5) -> np.ndarray:
    """A framed object on a background: the object is noise inside [w/5, w - w/4) x [h/6, h - h/3) (at least one pixel
    where the image has room), the frame the background, with the corners and the frame varied by `kind`."""
    ch, cs = LAYOUTS[layout]
    w, h = size
    rng = np.random.default_rng(seed + 101 * w + 13 * h + 7 * ch + 3 * len(kind))
    bg = background(layout)
    img = np.empty((h, w, ch), np.float32)
    img[:] = bg
    x0, y0 = w // 5, h // 6
    x1, y1 = max(x0 + 1, w - w // 4), max(y0 + 1, h - h // 3)
    if kind != "uniform":
        obj = (rng.random((y1 - y0, x1 - x0, ch)) * 65535.0).astype(np.float32)
        if cs == HSL:
            obj[..., 0] = 65535.0 - (rng.random(obj.shape[:2]) * 200.0).astype(np.float32)   # across the hue wrap
            obj[..., 1:] = bg[1:]
        if kind == "transparent":
            obj[..., -1] = (rng.random(obj.shape[:2]) * 0.03).astype(np.float32)          # QuantumScale^2 a b <= 1e-12
            img[..., -1] = 0.01
            obj[::3, ::4, -1] = 65535.0                                                    # the alpha term decides
        img[y0:y1, x0:x1] = obj
    corners = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)]
    if kind == "corners":
        for k, (y, x) in enumerate(corners):
            img[y, x] = bg + np.float32(3000.0 * k)
    elif kind == "bottom-right":                   # rows below the object end the box through the target[3] rule
        img[h - 1, w - 1] = bg + np.float32(9000.0)
    elif kind == "special frame":
        flat = img.reshape(-1, ch)
        pos = rng.integers(0, flat.shape[0], size=max(1, flat.shape[0] // 25))
        flat[pos, rng.integers(0, ch, size=pos.size)] = _SPECIAL[rng.integers(0, _SPECIAL.size, size=pos.size)]
        for y, x in corners:
            img[y, x] = bg
    elif kind == "special corners":
        for k, (y, x) in enumerate(corners):
            img[y, x, k % ch] = _SPECIAL[k]
    return img


def ref():
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        _lp = C.POINTER(C.c_long)
        r.ref_trim.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, _lp, C.c_double,
                               C.c_char_p, C.c_char_p, C.c_int, C.c_int, _lp, C.POINTER(C.c_int), C.POINTER(C.c_float),
                               C.c_size_t, _lp, C.c_int]
        _libs["ref"] = r
    return _libs["ref"]


def _ref_call(case, op):
    src = np.ascontiguousarray(case["src"], np.float32)
    h, w, ch = src.shape
    cs = case["colorspace"]
    cap = 4 * src.size + 64
    out = np.empty(cap, np.float32)
    box = (C.c_long * 4)()
    geom = (C.c_long * 7)()
    sev = C.c_int(0)
    edges = None if case["edges"] is None else case["edges"].encode()
    min_size = None if case["min_size"] is None else ("%dx%d" % case["min_size"]).encode()
    n = ref().ref_trim(util.P(src), w, h, ch, int(cs == CMYK), cs if cs != CMYK else -1,
                       (C.c_long * 4)(*case["page"]), case["fuzz"], edges, min_size, case["gravity"], op, box,
                       C.byref(sev), util.P(out), cap, geom, 1)
    return n, tuple(box), sev.value, out, tuple(geom[:6])


def ref_box_key(case) -> str:
    n, box, sev, _, _ = _ref_call(case, 0)
    assert n == 0
    return "/".join(str(v) for v in box) + f"/{sev}"


def ref_trim_key(case) -> str:
    n, _, sev, out, geom = _ref_call(case, 1)
    if n <= 0:
        return f"none/{sev}"
    cols, rows = geom[0], geom[1]
    return gc.key((out[: cols * rows * n].reshape(rows, cols, n), geom)) + f"/{sev}"


# What the reference computed for a case name, as ref_box_key() or, under "trim <name>", ref_trim_key()
reference = util.ReferenceStore(DIGESTS, REF_SO, by_test=False)


def box_reference(name, case) -> str:
    return reference(name, lambda: ref_box_key(case))


def trim_reference(name, case) -> str:
    return reference("trim " + name, lambda: ref_trim_key(case))


def _case(out, name, layout, size, kind, fuzz=0.0, edges=None, min_size=None, gravity=0, page=(0, 0, 0, 0), trim=False):
    out[name] = dict(layout=layout, size=size, kind=kind, src=source(layout, size, kind), colorspace=LAYOUTS[layout][1],
                     fuzz=fuzz, edges=edges, min_size=min_size, gravity=gravity, page=page, trim=trim)


def cases():
    """name -> case.  Every case has a bounding box; those with trim=True are trimmed too."""
    out = {}
    for layout in LAYOUTS:
        for size in SIZES:
            for kind in KINDS:
                for fname in ("0", "moderate"):
                    _case(out, f"{layout} {size[0]}x{size[1]} {kind} fuzz {fname}", layout, size, kind, FUZZ[fname],
                          trim=True)
            _case(out, f"{layout} {size[0]}x{size[1]} bottom-right", layout, size, "bottom-right")
            _case(out, f"{layout} {size[0]}x{size[1]} uniform", layout, size, "uniform", trim=True)
            _case(out, f"{layout} {size[0]}x{size[1]} equal fuzz huge", layout, size, "equal", FUZZ["huge"], trim=True)
        if layout in ALPHA:
            for fname in FUZZ:
                _case(out, f"{layout} transparent fuzz {fname}", layout, (70, 45), "transparent", FUZZ[fname], trim=True)
    for fname in FUZZ:
        _case(out, f"hsl hue wrap fuzz {fname}", "hsl", (70, 45), "equal", FUZZ[fname], trim=True)
    for layout in ("rgba", "gray", "cmyka"):
        for edges in EDGES:
            for kind in ("equal", "corners"):
                _case(out, f"{layout} edges '{edges}' {kind}", layout, (70, 45), kind, edges=edges, trim=True)
        for edges in ("north", "east,west"):
            _case(out, f"{layout} 1x13 edges '{edges}'", layout, (1, 13), "equal", edges=edges)
            _case(out, f"{layout} 15x1 edges '{edges}'", layout, (15, 1), "corners", edges=edges)
        for pname, page in gc.PAGES.items():
            for kind in ("equal", "corners"):
                _case(out, f"{layout} page {pname} {kind}", layout, (70, 45), kind, page=page, trim=True)
    for mname, min_size in MIN_SIZES.items():
        for gravity in GRAVITIES:
            for pname in ("zero", "canvas"):
                _case(out, f"rgba min size {mname} gravity {gravity} page {pname}", "rgba", (70, 45), "equal",
                      min_size=min_size, gravity=gravity, page=gc.PAGES[pname], trim=True)
        _case(out, f"gray min size {mname} gravity 5 corners", "gray", (70, 45), "corners", min_size=min_size,
              gravity=5, trim=True)
    return out


def declined_by_reference(box_key: str, trim_key: str) -> bool:
    """Where the library's TrimImage declines, the reference answers without a crop of its own: a zero box (its
    transparent 1x1 clone at -1-1), or a box its CropImage rejects with a warning (its 1x1 image, or none)."""
    if zero_box(box_key):
        return trim_key.startswith("1/1/") and trim_key.split("/")[4:6] == ["-1", "-1"]
    return trim_key == f"none/{OPTION_WARNING}" or (trim_key.startswith("1/1/") and
                                                   trim_key.endswith(f"/{OPTION_WARNING}"))


def zero_box(key: str) -> bool:
    w, h = key.split("/")[:2]
    return w == "0" or h == "0"


def image(case, device=False):
    import imagemagick_b200 as im
    src = case["src"]
    if device:
        import torch
        src = torch.from_numpy(np.ascontiguousarray(src)).cuda()
    img = im.Image(src, case["colorspace"])
    img.page = tuple(case["page"][2:])
    img.page_size = tuple(case["page"][:2])
    return img


def box_key(box, warning) -> str:
    """A library box (width, height, x, y) and its warning flag as the reference's key."""
    w, h, x, y = box
    return f"{gc.signed(w)}/{gc.signed(h)}/{x}/{y}/{OPTION_WARNING if warning else 0}"


def lib_trim_key(out, device=False) -> str:
    pixels = out.pixels.cpu().numpy() if device else out.pixels
    g = (out.columns, out.rows, gc.signed(out.page_size[0]), gc.signed(out.page_size[1]), out.page[0], out.page[1])
    return gc.key((pixels, g)) + "/0"


# ---- a NumPy statement of IsFuzzyEquivalencePixelInfo (pixel.c:6028-6106): float64 without contraction ----
_QS = 1.0 / 65535.0
_SQ1_2 = 0.70710678118654752440084436210484903928483593768847


def _fields(a: np.ndarray, cs: int):
    """GetPixelInfoPixel's red, green, blue, black, alpha (float64) of pixels a[..., ch]."""
    a = a.astype(np.float64)
    ch = a.shape[-1]
    gray = ch < 3
    red = a[..., 0]
    green = red if gray else a[..., 1]
    blue = red if gray else a[..., 2]
    black = a[..., 3] if cs == CMYK else np.zeros_like(red)
    alpha = a[..., ch - 1] if (ch == 2 or (ch == 4 and cs != CMYK) or ch == 5) else np.full_like(red, 65535.0)
    return red, green, blue, black, alpha


def mismatch(pixels: np.ndarray, target: np.ndarray, fuzz: float, cs: int) -> np.ndarray:
    """True where IsFuzzyEquivalencePixelInfo(pixel, target) is false."""
    ch = pixels.shape[-1]
    has_alpha = ch == 2 or (ch == 4 and cs != CMYK) or ch == 5
    p = _fields(pixels, cs)
    q = _fields(target.reshape(1, ch), cs)
    q = [v[0] for v in q]
    fz = fuzz if fuzz > _SQ1_2 else _SQ1_2
    fz = fz * fz
    shape = pixels.shape[:-1]
    res = np.zeros(shape, bool)
    done = np.zeros(shape, bool)
    dist = np.zeros(shape)
    scale = np.ones(shape)

    def test(limit):
        nonlocal res, done
        m = (dist > limit) & ~done
        res |= m
        done |= m

    with np.errstate(all="ignore"):
        if has_alpha:
            pix = p[4] - q[4]
            dist = pix * pix
            test(fz)
            scale = _QS * p[4]
            scale = scale * (_QS * q[4])
            done |= scale <= 1.0e-12
        if cs == CMYK:
            pix = p[3] - q[3]
            dist = dist + pix * pix * scale
            test(fz)
            scale = scale * (_QS * (65535.0 - p[3]))
            scale = scale * (_QS * (65535.0 - q[3]))
        dist = dist * 3.0
        fz3 = fz * 3.0
        pix = p[0] - q[0]
        if cs in (4, 5, 6, 7, 8, 9):             # HCL, HCLp, HSB, HSI, HSL, HSV
            pix = np.where(np.abs(pix) > 65535.0 / 2.0, pix - 65535.0, pix)
            pix = pix * 2.0
        dist = dist + pix * pix * scale
        test(fz3)
        for k in (1, 2):
            pix = p[k] - q[k]
            dist = dist + pix * pix * scale
            test(fz3)
    return res


def row_summaries(src: np.ndarray, fuzz: float, cs: int) -> np.ndarray:
    """The rows x 4 words of mb200_bounding_box_from_rows, from the NumPy comparison."""
    h, w, _ = src.shape
    targets = [src[0, 0], src[0, w - 1], src[h - 1, 0], src[h - 1, w - 1]]
    m = [mismatch(src, t, fuzz, cs) for t in targets]
    out = np.zeros((h, 4), np.uint32)
    any0, any1, any3 = m[0].any(1), m[1].any(1), m[3].any(1)
    out[:, 0] = np.where(any0, w - m[0].argmax(1), 0)
    out[:, 1] = np.where(any1, w - m[1][:, ::-1].argmax(1), 0)
    out[:, 2] = m[2].any(1)
    out[:, 3] = np.where(any3, w - m[3].argmax(1), 0)
    return out
