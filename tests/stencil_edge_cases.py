"""Edge-case inputs shared by the tests of the stencil operators (stencils.cu, and MotionBlurImage in pointwise.cu): the
oracle-against-reference suite (test_oracle_stencil_edges_vs_ref.py) and the GPU suite (test_gpu_stencil_edges.py) run
the same images.

* special_image: seeded noise with the special values of SPECIAL (signed zeros, float denormals, the samples around
  QuantumRange, HDR values above it and below 0, +-3.4e38, +-FLT_MAX, +-inf, NaN) scattered through every channel,
  alpha included (so alpha is also 0 and negative somewhere).
* nan_row_image: rows that start with NaN.  GetImageRange (statistic.c:1895) seeds each row's extremes with the row's
  first sample, so such a row is dropped from AdaptiveBlur / AdaptiveSharpen's auto-level, together with whatever
  extreme value it holds.
* posterised_image and thresholds: few levels, and SelectiveBlur thresholds equal to contrasts that occur in the image
  and one double ULP either side of them.
* NAMED: the minimal reproductions of the defects these images exposed, one per operator family.

BilateralBlurImage reads intensity_gaussian[510] (an 8-bit intensity difference of exactly +255), which the reference
never initialises (effect.c:951-952); full_jump() marks the output pixels whose window holds such a tap, where the
reference's result is undefined."""
import numpy as np

from util import make_image

F32 = np.float32
QR = 65535.0
FLT_MAX = float(np.finfo(np.float32).max)

SPECIAL = [0.0, -0.0, 1e-45, 1e-40, 1e-38, 0.4, 65534.6, 65535.0, float(np.nextafter(F32(65535), F32(np.inf))), 70000.0,
           1e6, 1e20, 3.4e38, FLT_MAX, -1.0, -70000.0, -3.4e38, -FLT_MAX, np.inf, -np.inf, np.nan]


def special_image(ch, w=37, h=23, seed=3, kind="noise", every=7):
    """make_image(kind) with SPECIAL cycled through every `every`-th sample (offset per channel), alpha included."""
    img = make_image(w, h, ch, seed=seed, kind=kind)
    rng = np.random.default_rng(seed + 100)
    for c in range(ch):
        flat = img[..., c].reshape(-1)
        at = rng.permutation(flat.size)[: flat.size // every]
        flat[at] = np.resize(np.array(SPECIAL, F32), at.size)
        img[..., c] = flat.reshape(h, w)
    return np.ascontiguousarray(img)


def nan_row_image(ch, w=64, h=48, column0=False):
    """A gradient whose row 20 starts with NaN and holds a 1e6 spike at column 40 (the edge map's maximum), or
    (column0) whose every row starts with NaN, which leaves GetImageRange no row at all."""
    img = make_image(w, h, ch, kind="gradient")
    if column0:
        img[:, 0, 0] = np.nan
    else:
        img[20, 0, 0] = np.nan
    img[20, 40, : min(3, ch)] = 1e6
    return np.ascontiguousarray(img)


LEVELS = np.array([0.0, 1000.0, 4097.0, 30001.0, 65535.0], F32)


def posterised_image(ch, w=40, h=30, seed=5):
    """Colour channels posterised to LEVELS, alpha left as noise."""
    img = make_image(w, h, ch, seed=seed)
    colour = ch - 1 if ch in (2, 4) else ch
    rng = np.random.default_rng(seed)
    img[..., :colour] = LEVELS[rng.integers(0, len(LEVELS), (h, w, colour))]
    return np.ascontiguousarray(img)


def intensity(img):
    """GetPixelIntensity (Rec709Luma, pixel.c:2428) of every pixel, in double; gray images give the gray sample itself
    (one channel) or weigh it as (g, g, g) (gray + alpha)."""
    x = img.astype(np.float64)
    if img.shape[2] == 1:
        return x[..., 0]
    r, g, b = (x[..., 0], x[..., 0], x[..., 0]) if img.shape[2] == 2 else (x[..., 0], x[..., 1], x[..., 2])
    with np.errstate(invalid="ignore", over="ignore"):
        return 0.212656 * r + 0.715158 * g + 0.072186 * b


def gray_clone_intensity(img):
    """The intensity SelectiveBlurImage compares for channels without the Blend trait (effect.c:3629): that of the
    pixel in a GRAY clone, which holds the float intensity (colorspace.c:943; a gray image is left as it is) and keeps
    alpha as a second channel."""
    ch = img.shape[2]
    if ch == 2:
        return intensity(img)
    with np.errstate(over="ignore"):
        g = intensity(img).astype(F32)[..., None]
    return intensity(np.concatenate([g, g], axis=2)) if ch == 4 else g[..., 0].astype(np.float64)


def thresholds(img, n=2):
    """The n most frequent non-zero contrasts |intensity(neighbour) - intensity(centre)| between 4-neighbours, for the
    gray-clone comparison and (with alpha) the blended one, each with its double neighbours either side."""
    centre = intensity(img)
    out = set()
    for lum in ([gray_clone_intensity(img), centre] if img.shape[2] in (2, 4) else [gray_clone_intensity(img)]):
        with np.errstate(invalid="ignore"):
            d = np.concatenate([np.abs(lum[1:, :] - centre[:-1, :]).ravel(), np.abs(lum[:, 1:] - centre[:, :-1]).ravel(),
                                np.abs(lum[:-1, :] - centre[1:, :]).ravel(), np.abs(lum[:, :-1] - centre[:, 1:]).ravel()])
        d = d[np.isfinite(d) & (d > 0)]
        values, counts = np.unique(d, return_counts=True)
        for t in values[np.argsort(-counts, kind="stable")][:n]:
            out.update([float(t), float(np.nextafter(t, 0.0)), float(np.nextafter(t, np.inf))])
    return sorted(out)


def _chars(img):
    """ScaleQuantumToChar (quantum.h:113-124) of the float intensity of every pixel (BilateralBlurImage's tonal index)."""
    with np.errstate(over="ignore", invalid="ignore"):
        q = intensity(img).astype(F32)
        t = q / F32(257.0)
        return np.where(np.isnan(q) | (q <= 0), 0, np.where(t >= 255, 255, np.floor(t + F32(0.5)))).astype(np.int32)


def full_jump(img, width, height):
    """(rows, columns) mask of the pixels of 8-bit intensity 0 whose width x height window (edge replicated) holds a pixel
    of intensity 255: the taps where the reference reads its uninitialised intensity_gaussian[510]."""
    c = _chars(img)
    h, w = c.shape
    hit = np.zeros((h, w), bool)
    for dy in range(-(height // 2), height // 2 + 1):
        for dx in range(-(width // 2), width // 2 + 1):
            hit |= c[np.clip(np.arange(h) + dy, 0, h - 1)][:, np.clip(np.arange(w) + dx, 0, w - 1)] == 255
    return hit & (c == 0)


def gray_posterised(ch, w=20, h=10, seed=9):
    """Every channel on LEVELS (alpha too): few distinct 16-bit values, so Mode / Nonpeak stay cheap at 255 x 255."""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(LEVELS[rng.integers(0, len(LEVELS), (h, w, ch))])


OPERATORS = ["statistic", "rotational_blur", "bilateral_blur", "selective_blur", "adaptive_blur", "adaptive_sharpen",
             "motion_blur"]
SHAPES = [(1, 1), (1, 17), (17, 1), (2, 2)]                      # (rows, columns)


def shapes(ch):
    """{name: small image cut from a dense special image}."""
    img = special_image(ch, every=3)
    return {f"{h}x{w}": np.ascontiguousarray(img[:h, 5:5 + w]) for h, w in SHAPES}


def cases(op, ch, stat=None):
    """[(name, image, arguments after (src, dst, columns, rows, channels))] of the edge images for one operator (for
    StatisticImage, of one statistic type): the oracle is pinned to the reference on these, and the kernels to the
    oracle."""
    src = special_image(ch)
    out = []
    if op == "statistic":                          # even windows, 1x1, and a window larger than the 37 x 23 image
        out += [(f"special {win}", src, (stat, *win)) for win in [(3, 3), (4, 2), (1, 1), (1, 7), (41, 31)]]
        out += [(f"{n} {win}", img, (stat, *win)) for n, img in shapes(ch).items() for win in [(3, 3), (1, 5)]]
    elif op == "rotational_blur":                  # angle 0 gives n = 2 samples; 9 x 9 has blur_radius / radius = 1, 2
        out += [(f"special {a}", src, (a,)) for a in [0.0, 10.0, -20.0, 360.0, -400.0]]
        out += [(f"9x9 {a}", special_image(ch, w=9, h=9), (a,)) for a in [30.0, -90.0]]
        out += [(n, img, (45.0,)) for n, img in shapes(ch).items()]
    elif op == "bilateral_blur":
        for kind in ["noise", "hdr"]:
            img = special_image(ch, kind=kind)
            out += [(f"special {kind} {a}", img, a)
                    for a in [(5, 3, 20.0, 1.5), (3, 3, 0.75, 2.0), (1, 1, 10.0, 1.0), (3, 9, 40.0, 4.0)]]
        out += [(n, img, (5, 5, 20.0, 1.5)) for n, img in shapes(ch).items()]
    elif op == "selective_blur":                   # threshold 0 selects nothing, +inf every finite contrast
        out += [(f"special {t}", src, (0.0, 1.0, t)) for t in [0.0, 1000.0, 6553.5, np.inf]]
        poster = posterised_image(ch)
        out += [(f"posterised {t!r}", poster, (0.0, 1.0, t)) for t in thresholds(poster) + [29001.0, 30001.0, 3097.0, 4097.0]]
        out += [(n, img, (2.0, 1.0, 20000.0)) for n, img in shapes(ch).items()]
    elif op in ("adaptive_blur", "adaptive_sharpen"):        # sigma 0 is a copy
        images = {"special": src, "hdr special": special_image(ch, kind="hdr", every=31), "NaN-led row": nan_row_image(ch),
                  "NaN column": nan_row_image(ch, column0=True), "hdr": make_image(37, 23, ch, seed=4, kind="hdr")}
        out += [(f"{n} {a}", img, a) for n, img in images.items() for a in [(0.0, 1.0), (2.0, 1.5), (0.0, 0.0)]]
        out += [(n, img, (0.0, 1.0)) for n, img in shapes(ch).items()]
    elif op == "motion_blur":
        out += [(f"special {a}", src, a) for a in [(0.0, 1.0, 0.0), (5.0, 2.0, 30.0), (3.0, 1.0, -135.0), (0.0, 0.5, 90.0)]]
        out += [(n, img, (4.0, 2.0, 45.0)) for n, img in shapes(ch).items()]
    return out


# The minimal reproductions of what these images showed: (operator, image builder, arguments).  The adaptive and
# selective ones were defects of the oracle and the kernels; the bilateral one is the reference's undefined read, which
# full_jump masks.
def _bilateral_spike(ch):
    img = make_image(37, 23, ch, seed=11)
    img[7, 9, :] = 3.4e38
    return img


def _adaptive_nan_row(ch):
    return nan_row_image(ch)


def _selective_posterised(ch):
    return posterised_image(ch)


NAMED = {
    "adaptive NaN-led row": ("adaptive_blur", _adaptive_nan_row, (0.0, 1.0)),
    "adaptive sharpen NaN-led row": ("adaptive_sharpen", _adaptive_nan_row, (0.0, 1.0)),
    "adaptive NaN column": ("adaptive_blur", lambda ch: nan_row_image(ch, column0=True), (0.0, 1.0)),
    "selective alpha at a contrast 29001": ("selective_blur", _selective_posterised, (0.0, 1.0, 29001.0)),
    "selective alpha at a contrast 30001": ("selective_blur", _selective_posterised, (0.0, 1.0, 30001.0)),
    "bilateral 3.4e38 beside a black pixel": ("bilateral_blur", _bilateral_spike, (5, 3, 20.0, 1.5)),
}
