"""Cases and runners shared by the tests of the orientation and crop operators (CropImage, ShaveImage, FlipImage,
FlopImage, TransposeImage, TransverseImage, IntegralRotateImage, RollImage, AutoOrientImage): the planner-against-
reference suite on the CPU and the GPU suite run the same cases.

The reference driver is oracle/ref_geometry.c (oracle/_ref/libmagickref_geometry.so, built by oracle/Makefile).  What
the reference computed for every case is stored in tests/golden/geometry_digests.json as "columns/rows/page_width/
page_height/page_x/page_y/channels/digest", keyed by case name; the digest is over the raw 32-bit words, so NaN payloads
and -0 count.  Re-record it with MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C
import hashlib

import numpy as np

import util
from util import ROOT

REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_geometry.so"
DIGESTS = ROOT / "tests" / "golden" / "geometry_digests.json"
_libs = {}

CROP, SHAVE, FLIP, FLOP, TRANSPOSE, TRANSVERSE, ROTATE, ROLL = range(8)
AUTO_ORIENT = 8                   # the reference driver's AutoOrientImage; the library dispatches it in Python
UNARY = {"flip": FLIP, "flop": FLOP, "transpose": TRANSPOSE, "transverse": TRANSVERSE}

# name -> (channels, CMYK)
LAYOUTS = {"gray": (1, False), "ga": (2, False), "rgb": (3, False), "rgba": (4, False), "cmyk": (4, True),
           "cmyka": (5, True)}
# 1x1, 1xN, Nx1, and sizes that are not multiples of the 32-pixel tile
SIZES = [(1, 1), (1, 13), (15, 1), (33, 17), (257, 129), (70, 45)]
# page width, height, x, y: none, a positive and a negative offset, a virtual canvas larger than the image
PAGES = {"zero": (0, 0, 0, 0), "pos": (0, 0, 5, 3), "neg": (0, 0, -7, -2), "canvas": (100, 80, 10, 20)}
# crop geometries (width, height, x, y) on the 33x17 image: inside, touching and crossing each edge, negative offsets,
# zero width / height (the page's), larger than the image
CROPS = {"inside": (10, 8, 5, 4), "left": (10, 8, 0, 4), "top": (10, 8, 5, 0), "right": (10, 8, 23, 4),
         "bottom": (10, 8, 5, 9), "out left": (10, 8, -4, 4), "out top": (10, 8, 5, -3), "out right": (10, 8, 28, 4),
         "out bottom": (10, 8, 5, 13), "negative": (10, 8, -3, -2), "zero width": (0, 8, 5, 4),
         "zero height": (10, 0, 5, 4), "zero both": (0, 0, 3, 2), "larger": (100, 100, -5, -5), "whole": (33, 17, 0, 0)}
# the two GeometryDoesNotContainImage outcomes: no overlap with the virtual canvas (the reference's 1x1 image), and
# zero area after clamping (no image); relative to the page offset
CROP_DECLINES = {"beyond right": (10, 8, 40, 4), "before left": (10, 8, -20, 4), "below": (10, 8, 5, 30),
                 "zero area": (10, 8, 33, 4)}
SHAVES = {"0x0": (0, 0), "3x2": (3, 2), "16x8": (16, 8), "0x5": (0, 5)}
SHAVE_DECLINES = {"half width": (17, 2), "half height": (3, 9)}
ROLLS = {"zero": (0, 0), "positive": (5, 3), "negative": (-5, -3), "beyond": (40, 20), "multiple": (33, 17),
         "negative multiple": (-66, 34), "negative beyond": (-70, -40)}
ROTATIONS = [1, 2, 3, 5, -1]
ROTATION_DECLINES = [0, 4]

_SPECIAL_WORDS = np.array([0x7FC00001, 0xFFC12345, 0x7FA00000, 0xFF800001,   # quiet / signalling NaNs with payloads
                           0x7F800000, 0xFF800000, 0x80000000,               # +inf, -inf, -0
                           0x00000001, 0x807FFFFF, 0x00400000], np.uint32)   # denormals


def source(w: int, h: int, ch: int, seed: int = 3) -> np.ndarray:
    """Noise with HDR values and every special bit pattern scattered through it."""
    rng = np.random.default_rng(seed + 31 * w + 7 * h + ch)
    a = (rng.random((h, w, ch)) * 65535.0).astype(np.float32)
    flat = a.reshape(-1)
    n = flat.size
    hdr = rng.integers(0, n, size=max(1, n // 20))
    flat[hdr] = (rng.standard_normal(hdr.size) * 1e6).astype(np.float32)
    words = flat.view(np.uint32)
    pos = rng.integers(0, n, size=max(1, n // 10))
    words[pos] = _SPECIAL_WORDS[rng.integers(0, _SPECIAL_WORDS.size, size=pos.size)]
    return a


def ref():
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        _lp = C.POINTER(C.c_long)
        r.ref_geometry.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_size_t, C.c_int, C.c_int, _lp, C.c_int, _lp,
                                   C.POINTER(C.c_float), C.c_size_t, _lp]
        _libs["ref"] = r
    return _libs["ref"]


def _longs(values, n=4):
    v = list(values) + [0] * (n - len(values))
    return (C.c_long * n)(*[int(x) for x in v])


def run_ref(src, cmyk, op, args=(), page=(0, 0, 0, 0)):
    """(pixels, (columns, rows, page_width, page_height, page_x, page_y)) the reference returns, or None."""
    h, w, ch = src.shape
    cap = 4 * src.size + 64
    out = np.empty(cap, np.float32)
    geom = (C.c_long * 7)()
    src = np.ascontiguousarray(src, np.float32)
    n = ref().ref_geometry(util.P(src), w, h, ch, int(cmyk), _longs(page), op, _longs(args), util.P(out), cap, geom)
    if n <= 0:
        return None
    cols, rows = geom[0], geom[1]
    return out[: cols * rows * n].reshape(rows, cols, n).copy(), tuple(geom[:6])


def bits_digest(pixels: np.ndarray) -> str:
    """SHA-256 prefix of the raw words: every bit counts."""
    a = np.ascontiguousarray(pixels, np.float32)
    h = hashlib.sha256(f"{a.shape}".encode())
    h.update(a.view(np.uint32).tobytes())
    return h.hexdigest()[:12]


def key(result) -> str:
    if result is None:
        return "none"
    pixels, g = result
    return "/".join(str(v) for v in g) + f"/{pixels.shape[2]}/{bits_digest(pixels)}"


_store = util.ReferenceStore(DIGESTS, REF_SO, by_test=False)


def reference(case: str, run) -> str:
    """What the reference computed for `case`, as key() of what run() returns with the reference itself when
    recording."""
    return _store(case, lambda: key(run()))


def _case(out, name, layout, size, op, args=(), page=(0, 0, 0, 0)):
    ch, cmyk = LAYOUTS[layout]
    out[name] = dict(layout=layout, size=size, src=source(*size, ch), cmyk=cmyk, op=op, args=tuple(args), page=page)


def cases():
    """name -> case: every one the library serves (bit exact)."""
    out = {}
    for layout in LAYOUTS:
        for size in SIZES:
            tag = f"{layout} {size[0]}x{size[1]}"
            for name, op in UNARY.items():
                _case(out, f"{name} {tag}", layout, size, op)
            for r in ROTATIONS:
                _case(out, f"rotate {r} {tag}", layout, size, ROTATE, (r,))
            _case(out, f"roll 5,-3 {tag}", layout, size, ROLL, (5, -3))
            _case(out, f"crop half {tag}", layout, size, CROP, (max(1, size[0] // 2), max(1, size[1] // 2),
                                                                size[0] // 4, size[1] // 4))
    for layout in ("rgba", "cmyka", "gray"):
        for pname, page in PAGES.items():
            tag = f"{layout} page {pname}"
            for name, op in UNARY.items():
                _case(out, f"{name} {tag}", layout, (33, 17), op, page=page)
            for r in (1, 2, 3):
                _case(out, f"rotate {r} {tag}", layout, (33, 17), ROTATE, (r,), page)
            for cname, g in CROPS.items():        # relative to the page offset, which the crop geometry includes
                _case(out, f"crop {cname} {tag}", layout, (33, 17), CROP, (g[0], g[1], g[2] + page[2], g[3] + page[3]),
                      page)
            for sname, s in SHAVES.items():
                _case(out, f"shave {sname} {tag}", layout, (33, 17), SHAVE, s, page)
            for o in range(2, 9):
                _case(out, f"auto-orient {o} {tag}", layout, (33, 17), AUTO_ORIENT, (o,), page)
        for rname, r in ROLLS.items():
            _case(out, f"roll {rname} {layout}", layout, (33, 17), ROLL, r, PAGES["pos"])
    return out


def declines():
    """name -> case the library declines (MB200_EUNSUPPORTED) and the reference answers in its own way."""
    out = {}
    for layout in ("rgba", "gray"):
        for pname in ("zero", "canvas"):
            page = PAGES[pname]
            for cname, g in CROP_DECLINES.items():
                _case(out, f"crop {cname} {layout} page {pname}", layout, (33, 17), CROP,
                      (g[0], g[1], g[2] + page[2], g[3] + page[3]), page)
            for sname, s in SHAVE_DECLINES.items():
                _case(out, f"shave {sname} {layout} page {pname}", layout, (33, 17), SHAVE, s, page)
        for r in ROTATION_DECLINES:
            _case(out, f"rotate {r} {layout}", layout, (33, 17), ROTATE, (r,))
        for o in (0, 1):
            _case(out, f"auto-orient {o} {layout}", layout, (33, 17), AUTO_ORIENT, (o,))
    return out


def reference_of(name, case):
    return reference(name, lambda: run_ref(case["src"], case["cmyk"], case["op"], case["args"], case["page"]))


def image(case, device=False):
    import imagemagick_b200 as im
    src = case["src"]
    if device:
        import torch
        src = torch.from_numpy(np.ascontiguousarray(src)).cuda()
    img = im.Image(src, im.CMYKColorspace if case["cmyk"] else im.sRGBColorspace)
    img.page = tuple(case["page"][2:])
    img.page_size = tuple(case["page"][:2])
    return img


def run_lib(case, device=False):
    """The library's result for the case, as (pixels, (columns, rows, page_width, page_height, page_x, page_y))."""
    import imagemagick_b200 as im
    img = image(case, device)
    op, args = case["op"], case["args"]
    if op == AUTO_ORIENT:
        out = im.AutoOrientImage(img, args[0])
    else:
        fn = {CROP: im.CropImage, SHAVE: im.ShaveImage, FLIP: im.FlipImage, FLOP: im.FlopImage,
              TRANSPOSE: im.TransposeImage, TRANSVERSE: im.TransverseImage, ROTATE: im.IntegralRotateImage,
              ROLL: im.RollImage}[op]
        out = fn(img, *args)
    pixels = out.pixels.cpu().numpy() if device else out.pixels
    return pixels, (out.columns, out.rows, signed(out.page_size[0]), signed(out.page_size[1]), out.page[0], out.page[1])


def signed(v: int) -> int:
    """A size_t page width as the reference driver reports it (a long)."""
    return C.c_long(v).value


def plan(case):
    """The host plan of the case (AutoOrient dispatched as the library dispatches it)."""
    import imagemagick_b200 as im
    op, args = case["op"], case["args"]
    if op == AUTO_ORIENT:
        op, args = {2: (FLOP, ()), 3: (ROTATE, (2,)), 4: (FLIP, ()), 5: (TRANSPOSE, ()), 6: (ROTATE, (1,)),
                    7: (TRANSVERSE, ()), 8: (ROTATE, (3,))}.get(args[0], (ROTATE, (0,)))
    return im.GeometryPlan(image(case), op, args)


def plan_key_prefix(p) -> str:
    return "/".join(str(v) for v in (p.columns, p.rows, signed(p.page.width), signed(p.page.height), p.page.x, p.page.y))


def apply_plan(src: np.ndarray, p) -> np.ndarray:
    """The plan's map applied with NumPy indexing: an independent statement of out(x, y) = in(map(x, y))."""
    ow, oh = p.columns, p.rows
    swap = bool(p.map & 4)
    rw, rh = (oh, ow) if swap else (ow, oh)
    y = np.arange(oh)[:, None]
    x = np.arange(ow)[None, :]
    if swap:
        uc, vc = y + 0 * x, x + 0 * y
    else:
        uc, vc = (x - p.roll_x) % rw + 0 * y, (y - p.roll_y) % rh + 0 * x
    u = rw - 1 - uc if p.map & 1 else uc
    v = rh - 1 - vc if p.map & 2 else vc
    return src.view(np.uint32)[p.src_y + v, p.src_x + u].view(np.float32)
