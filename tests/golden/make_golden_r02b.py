"""Generates the second golden set from the REAL reference (oracle/_ref/libmagickref.so): ResizeImage with the Jinc and
Kaiser filters, the hue / saturation colourspaces (HCL, HCLp, HSB, HSI, HSL, HSV, HWB) and the XYZ-derived ones (LMS,
CAT02LMS, Luv, xyY, DisplayP3, Adobe98, ProPhoto) in both directions, TransformImageColorspace under image settings
(illuminant, white luminance, the Log film settings) and the Log / YCC spaces:   python tests/golden/make_golden_r02b.py
The outputs are stored as digests in tests/golden/ref_digests.json ("r02b_golden/..."), the kernel expansions and the
case lists as arrays in tests/golden/r02b_golden.npz.  tests/test_golden.py pins the oracle (CPU) and, through it, the
CUDA path (-m gpu) to them."""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import util  # noqa: E402
from test_golden import r02b_source as source  # noqa: E402

OUT = Path(__file__).resolve().parent / "r02b_golden.npz"
W, H = 41, 31
HEXCONE = {"hcl": 4, "hclp": 5, "hsb": 6, "hsi": 7, "hsl": 8, "hsv": 9, "hwb": 10,
           "lch": 12, "lchab": 13, "lchuv": 14, "oklab": 38, "oklch": 39, "jzazbz": 34, "lms": 16, "luv": 17, "xyy": 25, "displayp3": 35, "adobe98": 36, "prophoto": 37, "cat02lms": 40}


KERNEL_STRINGS = [
    "Comet:0x2", "Comet:0x1.5+90", "Comet:5x2+180", "Laplacian", "Laplacian:1", "Laplacian:2", "Laplacian:3", "Laplacian:5",
    "Laplacian:7", "Laplacian:15", "Laplacian:19", "Sobel", "Sobel:90", "Sobel:45", "Sobel:180", "Sobel:270", "Sobel:135",
    "Roberts", "Roberts:90", "Prewitt:45", "Compass:270", "Kirsch:315", "Sobel:@", "Sobel:0>", "Kirsch:<",
    "FreiChen", "FreiChen:1", "FreiChen:2", "FreiChen:10", "FreiChen:13", "FreiChen:17,45", "FreiChen:19", "FreiChen:0,90",
    "FreiChen:90", "Ring:2,3.5", "Ring:1,2.5,3", "Ring", "Ring:0,0", "Peaks:1.9", "Peaks:2,4", "Peaks", "Edges", "Corners",
    "Diagonals", "Diagonals:1", "Diagonals:2,90", "LineEnds", "LineEnds:1", "LineEnds:2,90", "LineEnds:3>", "LineEnds:4@",
    "LineJunctions", "LineJunctions:1", "LineJunctions:3,180", "LineJunctions:4", "LineJunctions:5@", "Ridges", "Ridges:2",
    "ConvexHull", "Skeleton", "Skeleton:1", "Skeleton:2", "Skeleton:3", "ThinSE:482", "ThinSE:41", "ThinSE:87x90",
    "ThinSE:481,45", "ThinSE:823>", "ThinSE:49<", "ThinSE:44@", "Chebyshev", "Chebyshev:2", "Chebyshev:1,50%",
    "Manhattan:2,100", "Manhattan:3,4!", "Octagonal", "Octagonal:3", "Euclidean", "Euclidean:2", "Euclidean:4,10!",
    "3>: 0,0,nan 0,1,1 nan,1,nan", "3@: 1,0,0 0,1,0 0,0,-", "3<: 1,2,3 4,5,6 7,8,9", "3x1>: 1,2,3", "2x2>: 1,2,3,4",
    "4x3+1+1<: 1,2,3,4,5,6,7,8,9,10,11,12", "Unity", "Binomial:2", "Disk:2.5", "Square:2>", "Plus:2@", "Blur:0x2>",
    "Gaussian:0x1@", "Rectangle:3x2+1+0>", "Octagon:2>", "Sobel@", "Kirsch@"]


def kernel_goldens(out):
    """The reference's own expansion of kernel strings (AcquireKernelInfo, morphology.c:485): every list element's values
    and origin; a string the reference rejects is recorded with count 0."""
    for n, name in enumerate(KERNEL_STRINGS):
        idx = 0
        while True:
            k = util.ref_kernel(name, idx)
            if k is None:
                break
            out[f"kernel/{n}/{idx}/values"] = k[0]
            out[f"kernel/{n}/{idx}/origin"] = np.array([k[1], k[2]], np.int64)
            idx += 1
        out[f"kernel/{n}/count"] = np.array([idx], np.int64)
    out["kernel/strings"] = np.array(KERNEL_STRINGS)


# ResizeImage with "-define filter:*" artifacts (AcquireResizeFilter, resize.c:999-1226): (filter, defines)
RESIZE_DEFINES = [(22, "filter:blur=0.8"), (22, "filter:lobes=2"), (8, "filter:sigma=0.75"), (16, "filter:kaiser-beta=4.5"),
                  (12, "filter:b=0.2;filter:c=0.6"), (3, "filter:window=Hann"), (13, "filter:lobes=5;filter:blur=0.9")]


# TransformImageColorspace under image settings (colorspace.c:761, :996, :1085-1095) and the Log / YCC spaces:
# (from, to, "key=value;..." -- "color:" keys are artifacts, the others properties)
COLORSPACE_DEFINES = [(23, 11, "color:illuminant=D50"), (11, 23, "color:illuminant=D50"), (23, 13, "color:illuminant=F11"),
                      (14, 23, "color:illuminant=E"), (23, 17, "color:illuminant=D75"), (17, 23, "color:illuminant=A"),
                      (23, 34, "white-luminance=203"), (34, 23, "white-luminance=203"),
                      (23, 15, ""), (15, 23, ""), (23, 15, "film-gamma=0.5;reference-black=64;reference-white=940"),
                      (15, 23, "film-gamma=0.65;reference-white=700"), (23, 28, ""), (28, 23, ""), (21, 28, ""), (28, 11, "")]


def main():
    r, P = util.ref(), util.P
    out = {}
    kernel_goldens(out)
    src4 = source(4)
    for n, (frm, to, defines) in enumerate(COLORSPACE_DEFINES):
        buf = src4.copy()
        assert r.ref_colorspace_defines(P(buf), W, H, 4, frm, to, defines.encode()) == 0
        util.record("r02b_golden/colordef", str(n), buf)
    out["colordef/cases"] = np.array([f"{f}|{t}|{d}" for f, t, d in COLORSPACE_DEFINES])
    for n, (filt, defines) in enumerate(RESIZE_DEFINES):
        for (ow, oh) in ((20, 15), (82, 62)):
            dst = np.empty((oh, ow, 4), np.float32)
            assert r.ref_resize_defines(P(src4), W, H, 4, P(dst), ow, oh, filt, defines.encode()) == 0
            util.record("r02b_golden/resizedef", f"{n}/{ow}x{oh}", dst)
    out["resizedef/defines"] = np.array([f"{f}|{d}" for f, d in RESIZE_DEFINES])
    for ch in (3, 4):
        src = source(ch)
        for filt, name in ((13, "jinc"), (16, "kaiser")):
            for (ow, oh) in ((20, 15), (82, 62), (41, 13)):
                dst = np.empty((oh, ow, ch), np.float32)
                assert r.ref_resize(P(src), W, H, ch, P(dst), ow, oh, filt) == 0
                util.record(f"r02b_golden/c{ch}", f"resize_{name}_{ow}x{oh}", dst)
        poster = (np.round(src / 16384.0) * 16384.0).astype(np.float32)     # few levels: tied counts, medians on the extremes
        for typ, tname in ((6, "mode"), (7, "nonpeak")):
            for (ww, wh) in ((3, 3), (5, 5), (4, 2)):
                for image, iname in ((src, "src"), (poster, "poster")):
                    dst = np.empty_like(image)
                    assert r.ref_statistic(P(image), P(dst), W, H, ch, typ, ww, wh) == 0
                    util.record(f"r02b_golden/c{ch}", f"statistic_{tname}_{ww}x{wh}_{iname}", dst)
        for name, cs in HEXCONE.items():
            for frm, to, tag in ((23, cs, f"srgb_{name}"), (cs, 23, f"{name}_srgb")):
                buf = src.copy()
                assert r.ref_colorspace(P(buf), W, H, ch, frm, to) == 0
                util.record(f"r02b_golden/c{ch}", f"colorspace_{tag}", buf)
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), "arrays", OUT.stat().st_size, "bytes,", len(util.REF_STORE.recorded), "digests")


if __name__ == "__main__":
    main()
