"""Inputs, kernels and runners shared by the tests of the directly applied morphology methods, Distance and Voronoi
(MorphologyPrimitiveDirect): the oracle-against-reference suite and the GPU suite run the same cases.

The oracle is oracle/direct_oracle.c (oracle/libdirect_oracle.so) and the reference driver oracle/ref_direct.c
(oracle/_ref/libmagickref_direct.so), both built by oracle/Makefile.  What the reference computed for every case is stored
in tests/golden/direct_digests.json as "kernel/digest/channels/alpha_trait" (the digest of the head kernel the reference
parsed, the digest of the resulting cache, its channel count and alpha trait), keyed like level_cases keys its own file;
re-record it with MB200_RECORD_REFERENCE=1 where oracle/_ref is built."""
import ctypes as C

import numpy as np

import util
from util import ROOT, digest, make_image

ORACLE_SO = ROOT / "oracle" / "libdirect_oracle.so"
REF_SO = ROOT / "oracle" / "_ref" / "libmagickref_direct.so"
DIGESTS = ROOT / "tests" / "golden" / "direct_digests.json"
_libs = {}

_fp = C.POINTER(C.c_float)
_sz, _i, _l = C.c_size_t, C.c_int, C.c_long

DISTANCE, VORONOI = 21, 22
COPY_TRAIT, BLEND_TRAIT = 1, 4            # PixelTrait (pixel.h)

# The four distance kernels at radii 1-4 (the default radius is 1), and with a scale
DISTANCE_KERNELS = ([f"{n}:{r}" for n in ("Chebyshev", "Manhattan", "Octagonal", "Euclidean") for r in (1, 2, 3, 4)]
                    + ["Euclidean", "Euclidean:4,20!", "Chebyshev:1,50%", "Manhattan:2,300"])
# User kernels: off-centre origins, asymmetric values, NaN ("-") cells, 1xN / Nx1, a kernel list (only its head is used)
USER_KERNELS = ["3x3+0+0:0,1,2 3,4,5 6,7,8", "3x3+2+2:5,-,1 2,0,3 -,4,-", "4x3+1+2:10,20,-,5 0,-,7,30 8,9,3,2",
                "5x2+4+0:9,8,7,6,5 1,-,2,-,3", "1x5:300,200,0,100,400", "5x1+3+0:300,200,0,100,400",
                "2x2+1+1:-,7 5,0", "3x3:-,-,- -,0,- -,-,-", "Euclidean:2;Chebyshev:1", "Manhattan:1;Euclidean:3"]
KERNELS = DISTANCE_KERNELS + USER_KERNELS


def shapes(w: int, h: int, ch: int, seed: int) -> np.ndarray:
    """A binary image (0 or QuantumRange) of discs and bars: what a distance transform is usually run on."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = np.full((h, w, ch), 65535.0, np.float32)
    for c in range(ch):
        for _ in range(3):
            cx, cy, r = rng.integers(0, w), rng.integers(0, h), rng.integers(1, max(2, min(w, h) // 3))
            out[(xx - cx) ** 2 + (yy - cy) ** 2 <= r * r, c] = 0.0
        out[int(rng.integers(0, h)), :, c] = 0.0
    return out


def specials(w: int, h: int, ch: int, seed: int) -> np.ndarray:
    """HDR noise with +-inf and NaN samples scattered in it."""
    out = make_image(w, h, ch, seed=seed, kind="hdr")
    rng = np.random.default_rng(seed + 1)
    for value in (np.inf, -np.inf, np.nan):
        idx = rng.integers(0, out.size, size=max(1, out.size // 40))
        out.ravel()[idx] = value
    return out


def nan_inf(w: int, h: int, ch: int, seed: int) -> np.ndarray:
    """HDR noise with NaN and +inf samples but no -inf, which would flood every pixel a kernel reaches: NaN samples
    are then skipped against finite neighbours, and the order of the recurrence shows in the result."""
    out = make_image(w, h, ch, seed=seed, kind="hdr")
    rng = np.random.default_rng(seed + 1)
    for value in (np.inf, np.nan):
        idx = rng.integers(0, out.size, size=max(1, out.size // 12))
        out.ravel()[idx] = value
    return out


def sources(ch: int, w: int = 29, h: int = 23, seed: int = 3):
    """name -> image: binary shapes, noise, HDR (values below 0 and above QuantumRange), +-inf / NaN samples, NaN / +inf
    samples, and 1x1, 1xN and Nx1 images."""
    return {"shapes": shapes(w, h, ch, seed), "noise": make_image(w, h, ch, seed=seed + 1),
            "hdr": make_image(w, h, ch, seed=seed + 2, kind="hdr"), "specials": specials(w, h, ch, seed + 3),
            "nan inf": nan_inf(w, h, ch, seed + 7),
            "1x1": make_image(1, 1, ch, seed=seed + 4), "1xN": shapes(1, 17, ch, seed + 5),
            "Nx1": shapes(19, 1, ch, seed + 6)}


def oracle():
    """The plain-C oracle; (re)built when stale."""
    if "oracle" not in _libs:
        o = util.load_oracle(ORACLE_SO)
        o.orc_morphology_direct.argtypes = [_fp, _fp, _sz, _sz, _i, _i, C.POINTER(util.OrcKernel)]
        _libs["oracle"] = o
    return _libs["oracle"]


def ref():
    """The real reference's MorphologyImage; only where oracle/_ref has been built from a reference source tree."""
    if "ref" not in _libs:
        r = C.CDLL(str(REF_SO))
        r.ref_morphology_direct.argtypes = [_fp, _fp, _sz, _sz, _i, _i, _l, C.c_char_p, C.POINTER(_i)]
        _libs["ref"] = r
    return _libs["ref"]


def kernel_values(vals, x, y) -> np.ndarray:
    """A kernel's shape, origin and values as one array (the digest of a kernel)."""
    return np.concatenate([[vals.shape[0], vals.shape[1], x, y], np.asarray(vals, np.float64).ravel()])


def head_kernel(string: str):
    """(values, x, y) of the first kernel of the list the product's host-side parser makes of `string`."""
    import imagemagick_b200 as im
    return im.AcquireKernelInfo(string).arrays()[0]


def ref_run(src, method, kernel: str, iterations: int = 1):
    """(pixels, alpha_trait) the reference's MorphologyImage leaves."""
    h, w, ch = src.shape
    out = np.empty((h, w, ch + 1), np.float32)
    trait = _i(-1)
    out_ch = ref().ref_morphology_direct(util.P(src), util.P(out), w, h, ch, method, iterations, kernel.encode(),
                                         C.byref(trait))
    assert out_ch > 0, out_ch
    return out.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy(), trait.value


def alpha_trait(method: int, ch: int) -> int:
    """The alpha trait of the result: Voronoi leaves CopyPixelTrait (morphology.c:3766-3774), Distance the source's."""
    if method == VORONOI:
        return COPY_TRAIT
    return BLEND_TRAIT if ch in (2, 4) else 0


def orc_run(src, method, kernel: str):
    """(pixels, alpha_trait) of the oracle on the head kernel of `kernel`."""
    h, w, ch = src.shape
    vals, x, y = head_kernel(kernel)
    k = util.orc_kernel_from_array(vals, x, y)
    out = np.empty((h, w, ch + 1), np.float32)
    try:
        out_ch = oracle().orc_morphology_direct(util.P(src), util.P(out), w, h, ch, method, C.byref(k))
    finally:
        util.oracle().orc_kernel_free(C.byref(k))
    assert out_ch in (ch, ch + 1), out_ch
    return out.ravel()[: w * h * out_ch].reshape(h, w, out_ch).copy(), alpha_trait(method, ch)


def result_key(kernel_digest: str, pixels, trait) -> str:
    return f"{kernel_digest}/{digest(pixels)}/{pixels.shape[2]}/{trait}"


def orc_key(src, method, kernel: str) -> str:
    return result_key(digest(kernel_values(*head_kernel(kernel))), *orc_run(src, method, kernel))


def ref_key(src, method, kernel: str) -> str:
    return result_key(digest(kernel_values(*util.ref_kernel(kernel))), *ref_run(src, method, kernel))


# What the reference computed for `case` of the running test (or of `test`, "<file>::<test>[<params>]"), as result_key()
reference = util.ReferenceStore(DIGESTS, REF_SO)
