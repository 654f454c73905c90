"""Edge-case inputs shared by the tests of the in-place TransformImageColorspace legs (colorspace.cu, hexcone.cu): the
oracle-against-reference suite (test_oracle_colorspace_edges_vs_ref.py) and the GPU suite (test_gpu_colorspace_edges.py)
run the same images.

Every value of VALUES appears in red, green and blue on its own next to ordinary samples, and in all three at once (a
gray).  The values are the special ones (signed zeros, denormals, the samples around QuantumRange, powers of ten up to
FLT_MAX, negatives, +-inf, NaN) and float sweeps of +-4 ULPs around the boundaries the kernels decide on:

* the decode toe of the sRGB curve, 0.0404482362771076 * QuantumRange (colorspace.cu's kToeLimitF is the float below it);
* the encode toe, 0.0031306684425005883 * QuantumRange, which a linear-RGB sample meets on the way back to sRGB;
* the sample whose gamma argument (QuantumScale * p + 0.055) / 1.055 reaches 2^63, where kDecodeScale's tabled exponents end;
* gray samples whose tristimulus ratio lies in every binade from 2^-7 to past FLT_MAX (the cube root's whole argument range).

Then explicit pixels (boundary_pixels):

* the CIE epsilon 216 / 24389 (the Lab toe) for each of the three ratios tx = X / Xn, ty = Y / Yn, tz = Z / Zn, found by
  bisection on the ratio as the Lab kernel and the oracle compute it (cie_ratio): once as a gray -- the other two ratios
  then lie on either side of the epsilon (the white-normalised row sums of the RGB -> XYZ matrix differ from 1 by up to
  1.4e-4, some 1100 float steps of the sample), so the pixel takes the out-of-line branch and its exact comparison -- and
  once with one channel at 0 so that the other two ratios lie well above the epsilon, where the fast path's high-word
  test (colorspace.cu kCieEpsHi) decides alone.  Every sweep reaches a ratio below the epsilon's high word, one in that
  word at or below the epsilon, one in it above the epsilon and one in the next word (cie_sweeps asserts it);
* the Lab L sample at kCieK * kCieEps = 8 (the inverse toe of L) with a neutral a / b.

The RGBA images carry the special values in alpha as well; every leg must leave alpha bit-identical."""
from fractions import Fraction
import numpy as np

from util import make_image

QR = 65535.0
F32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)

SRGB, RGB, LAB, XYZ, LOG, YCC = 23, 21, 11, 26, 15, 28
CORE = [LAB, XYZ, RGB]
HEXCONE = [4, 5, 6, 7, 8, 9, 10]                                # HCL, HCLp, HSB, HSI, HSL, HSV, HWB
XYZ_FAMILY = [12, 13, 14, 16, 17, 25, 34, 35, 36, 37, 38, 39, 40]
POLAR = (12, 13, 14)                                            # LCH, LCHab, LCHuv: hue = atan2 of two differences
MATRIX = [1, 18, 19, 20, 27, 29, 30, 31, 32]                    # CMY, OHTA, Rec601YCbCr, Rec709YCbCr, YCbCr, YDbDr, YIQ, YPbPr, YUV
SPACES = CORE + XYZ_FAMILY + HEXCONE + MATRIX + [LOG, YCC]


def ulps(x, n=4):
    """x rounded to float and its n float neighbours on either side."""
    x = F32(x)
    out = [x]
    lo = hi = x
    for _ in range(n):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo, hi]
    return sorted(out)


def first_float_above(pred, lo, hi):
    """The smallest positive float p in (lo, hi] with pred(p), by bisection on the float bit patterns (pred monotone)."""
    a, b = int(F32(lo).view(np.int32)), int(F32(hi).view(np.int32))
    assert not pred(float(np.int32(a).view(F32))) and pred(float(np.int32(b).view(F32)))
    while b - a > 1:
        m = (a + b) // 2
        if pred(float(np.int32(m).view(F32))):
            b = m
        else:
            a = m
    return F32(np.int32(b).view(F32))


def gamma_arg(p):
    """The argument DecodePixelGamma hands to DecodeGamma (pixel.c:322), in double."""
    return (p / QR + 0.055) / 1.055


def linear_unit(p):
    """The decoded sample in [0, 1] units, x^2.4 in double: the Chebyshev series agrees with it to ~1e-16 relative, and a
    float step of the sample moves it by ~1e-7, so a crossing found on this model is the oracle's and the kernel's unless
    it falls within 1e-9 of a float step -- the sweeps below reach 12 steps either side."""
    return gamma_arg(p) ** 2.4


def sample_of_linear(t):
    """The sRGB sample whose decoded value is t (in [0, 1] units), in double."""
    return QR * (1.055 * t ** (1.0 / 2.4) - 0.055)


CIE_EPS = 216.0 / 24389.0
CIE_EPS_HI = 0x3f822354                        # its high word (colorspace.cu kCieEpsHi)
# ConvertRGBToXYZ's rows (colorspace-private.h:759) and the D65 white (:32-46)
M = ((0.4123955889674142161, 0.3575834307637148171, 0.1804926473817015735),
     (0.2125862307855955516, 0.7151703037034108499, 0.07220049864333622685),
     (0.01929721549174694484, 0.1191838645808485318, 0.9504971251315797660))
WHITE = (0.95047, 1.0, 1.08883)


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def cie_ratio(k, rgb):
    """Ratio k (0 tx, 1 ty, 2 tz) of a pixel whose channels decode to rgb (unit range), as the oracle computes it
    ((M r) / white, colorspace-private.h:1075) and as the Lab kernel does (rgb_to_lab_unit: the row divided by the white
    folded into the constants, two FMAs); both are returned."""
    r, g, b = rgb
    oracle = (M[k][0] * r + M[k][1] * g + M[k][2] * b) / WHITE[k]
    w = [M[k][j] / WHITE[k] for j in range(3)]
    kernel = _fma(w[2], b, _fma(w[1], g, w[0] * r))
    return oracle, kernel


def _high_word(t):
    return int(np.array(t, np.float64).view(np.int64)) >> 32


# the channels that carry the swept sample, per ratio and kind: all three (a gray), or two with the third at 0 so that
# the other two ratios are well above the epsilon (tx: G = B, ty: R = B, tz: R = G)
CIE_CHANNELS = {"gray": ((0, 1, 2),) * 3, "fast": ((1, 2), (0, 2), (0, 1))}


def cie_sweeps(n=12):
    """{(kind, k): float32 samples}: n float steps either side of the sample at which ratio k crosses the epsilon."""
    out = {}
    for kind, chans in CIE_CHANNELS.items():
        for k in range(3):
            def ratios(p):
                u = linear_unit(p)
                return [cie_ratio(j, [u if c in chans[k] else 0.0 for c in range(3)]) for j in range(3)]

            p0 = first_float_above(lambda p: ratios(p)[k][0] > CIE_EPS, 1000.0, 20000.0)
            assert first_float_above(lambda p: ratios(p)[k][1] > CIE_EPS, 1000.0, 20000.0) == p0   # oracle == kernel
            sweep = np.array(ulps(p0, n), F32)
            t = [ratios(float(p))[k][1] for p in sweep]
            hi = [_high_word(v) for v in t]
            assert any(h < CIE_EPS_HI for h in hi) and any(h == CIE_EPS_HI + 1 for h in hi), (kind, k)
            assert any(h == CIE_EPS_HI and v <= CIE_EPS for h, v in zip(hi, t)), (kind, k)
            assert any(h == CIE_EPS_HI and v > CIE_EPS for h, v in zip(hi, t)), (kind, k)
            if kind == "fast":       # the two other ratios stay above the epsilon's high word across the sweep
                assert all(_high_word(ratios(float(p))[j][1]) > CIE_EPS_HI for p in sweep for j in range(3) if j != k)
            out[kind, k] = sweep
    return out
TOE = 0.0404482362771076 * QR                 # DecodePixelGamma's toe limit (pixel.c:320)
ENCODE_TOE = 0.0031306684425005883 * QR       # EncodePixelGamma's (pixel.c:447)

SPECIAL = ([0.0, -0.0, 1e-45, 1e-40, 1e-30, 1e-10, 0.4, 1.0, 255.0, 65534.6, 65535.0]
           + [float(np.nextafter(F32(65535), F32(0))), float(np.nextafter(F32(65535), F32(np.inf))), 70000.0, 1e6]
           + [10.0 ** k for k in range(10, 39)] + [FLT_MAX]
           + [-1.0, -70000.0, -FLT_MAX, np.inf, -np.inf, np.nan])


def sweeps():
    """{name: float32 array} of the boundary sweeps listed in the module docstring."""
    table_edge = first_float_above(lambda p: gamma_arg(p) >= 2.0 ** 63, 1e23, 1e24)
    binades = []
    for k in range(-7, 270):                     # tx = 2^k ... 2^269 (p = FLT_MAX gives ~2^269)
        for m in (1.0, 1.5):
            p = sample_of_linear(m * 2.0 ** k)
            if p < FLT_MAX:
                binades.append(F32(p))
    return {
        "decode toe": np.array(ulps(TOE), F32),
        "encode toe": np.array(ulps(ENCODE_TOE), F32),
        "table edge": np.array(ulps(table_edge), F32),
        "cube root binades": np.array(binades, F32),
        "lab L toe": np.array(ulps(8.0 / 100.0 * QR), F32),
    }


def values():
    return np.concatenate([np.array(SPECIAL, F32)] + list(sweeps().values())).astype(F32)


def boundary_pixels():
    """(n, 3) float32 pixels of the CIE epsilon sweeps and the Lab inverse toe (module docstring)."""
    out = []
    for (kind, k), sweep in cie_sweeps().items():
        px = np.zeros((len(sweep), 3), F32)
        for c in CIE_CHANNELS[kind][k]:
            px[:, c] = sweep
        out.append(px)
    lab_toe = sweeps()["lab L toe"]                 # Lab L around 8 with a neutral a / b
    out.append(np.stack([lab_toe, np.full_like(lab_toe, 32767.5), np.full_like(lab_toe, 32767.5)], axis=1))
    return np.concatenate(out).astype(F32)


def edge_pixels(seed=5):
    """(n, 3) float32 colour triplets: every value alone in R, G and B beside ordinary samples, then as a gray, then the
    boundary pixels."""
    v = values()
    ordinary = make_image(len(v), 3, 3, seed=seed)[..., 0].T.astype(F32)       # (n, 3) samples in 0..65535
    out = []
    for c in range(3):
        p = ordinary.copy()
        p[:, c] = v
        out.append(p)
    out.append(np.repeat(v[:, None], 3, axis=1))
    out.append(boundary_pixels())
    return np.concatenate(out).astype(F32)


def edge_image(ch, width=37, seed=5):
    """The edge pixels as a (rows, width, ch) image (the last row padded with ordinary samples); RGBA carries the special
    values, cycled, in alpha."""
    px = edge_pixels(seed)
    rows = -(-len(px) // width)
    img = make_image(width, rows, ch, seed=seed + 1)
    flat = img.reshape(-1, ch)
    flat[: len(px), :3] = px
    if ch == 4:
        special = np.array(SPECIAL, F32)
        flat[:, 3] = np.resize(special, len(flat))
        flat[1::3, 3] = F32(65535.0)
    return np.ascontiguousarray(img)


def pixels_of(img, n):
    """The first n pixels of img, cycled, as a (1, n, ch) image."""
    flat = img.reshape(-1, img.shape[2])
    return np.ascontiguousarray(np.resize(flat, (n, img.shape[2]))[None])


def inverse_source(forward_output, ch, seed=5):
    """Input of an inverse leg: the forward leg's output of the edge image stacked on the edge image itself, whose
    samples are then read as that space's own components (special values written directly as L, a, b / X, Y, Z / ...)."""
    return np.ascontiguousarray(np.concatenate([forward_output, edge_image(ch, seed=seed)], axis=0))
