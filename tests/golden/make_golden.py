"""Generates the hot-path golden data from the REAL reference (ImageMagick 7.1.1-45 compiled from
source into oracle/_ref/libmagickref.so, oracle/Makefile):   python tests/golden/make_golden.py

The inputs are seeded (test_golden.hot_source); the reference's raw float Quantum outputs are
stored as digests (util.digest) in tests/golden/ref_digests.json under "hotpath_golden/<tag>",
the kernel taps and the known-answer pixel as arrays in tests/golden/hotpath_golden.npz.
tests/test_golden.py pins the oracle (and, on the GPU, the CUDA path through the oracle) to them.
"""
import ctypes as C
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import util  # noqa: E402
from test_golden import hot_source  # noqa: E402

OUT = Path(__file__).resolve().parent / "hotpath_golden.npz"


def main():
    r = util.ref()
    P = util.P
    out = {}
    W, H = 41, 31
    for ch in (1, 2, 3, 4):
        for kind in ("noise", "alpha_blocks"):
            if kind == "alpha_blocks" and ch in (1, 3):
                continue
            tag = f"c{ch}_{kind}"
            src, clamp_src = hot_source(tag)
            record = lambda name, a: util.record(f"hotpath_golden/{tag}", name, a)   # noqa: E731
            for name, fn, args in (("blur_0x2", r.ref_blur, (0.0, 2.0)), ("blur_0x4", r.ref_blur, (0.0, 4.0)),
                                   ("blur_2x1", r.ref_blur, (2.0, 1.0)),
                                   ("gaussian_0x1.5", r.ref_gaussian_blur, (0.0, 1.5)),
                                   ("unsharp_0x2_1.5_0.02", r.ref_unsharp, (0.0, 2.0, 1.5, 0.02)),
                                   ("sharpen_0x1", r.ref_sharpen, (0.0, 1.0)), ("edge_1", r.ref_edge, (1.0,))):
                dst = np.empty_like(src)
                assert fn(P(src), P(dst), W, H, ch, *args) == 0
                record(name, dst)
            for kname in ("Disk:3", "Diamond:2", "Rectangle:5x3+1+2"):
                for method, mname in ((3, "erode"), (4, "dilate"), (8, "open"), (9, "close"), (12, "smooth")):
                    dst = np.empty_like(src)
                    assert r.ref_morphology(P(src), P(dst), W, H, ch, method, 1, kname.encode()) == 0
                    record(f"{mname}_{kname}", dst)
            for method, mname in ((13, "edgein"), (14, "edgeout"), (15, "edge"), (16, "tophat"), (17, "bottomhat")):
                dst = np.empty_like(src)            # morphology.c:3995-4012: ends in CompositeImage(Difference)
                assert r.ref_morphology(P(src), P(dst), W, H, ch, method, 1, b"Disk:3") == 0
                record(f"{mname}_Disk:3", dst)
            for op, thr, spec, tname in ((0, 30000.0, "", "bilevel_30000"), (3, 0.0, "", "clamp"),
                                         (1, 0.0, "40%,50%,60%", "black_40%,50%,60%"), (2, 0.0, "45000", "white_45000")):
                if op in (1, 2) and ch < 3:
                    continue                        # gray images are promoted to sRGB (threshold.c:949)
                buf = clamp_src.copy() if op == 3 else src.copy()
                assert r.ref_threshold(P(buf), W, H, ch, op, thr, spec.encode()) == 0
                record(f"threshold_{tname}", buf)
            dst = np.empty_like(src)
            assert r.ref_convolve(P(src), P(dst), W, H, ch, b"3x3: 1,2,0.5 0,-1,nan 3,0.25,-2") == 0
            record("convolve_user3x3", dst)
            for filt, fname, sizes in ((22, "lanczos", ((20, 15), (21, 16), (82, 62), (41, 13))),
                                       (12, "mitchell", ((20, 15), (60, 40))), (0, "undefined", ((20, 15), (60, 40))),
                                       (3, "triangle", ((13, 31),)), (1, "point", ((20, 15),))):
                for (ow, oh) in sizes:
                    dst = np.empty((oh, ow, ch), np.float32)
                    assert r.ref_resize(P(src), W, H, ch, P(dst), ow, oh, filt) == 0
                    record(f"resize_{fname}_{ow}x{oh}", dst)
            for (ow, oh) in ((20, 15), (97, 50)):
                dst = np.empty((oh, ow, ch), np.float32)
                assert r.ref_sample(P(src), W, H, ch, P(dst), ow, oh) == 0
                record(f"sample_{ow}x{oh}", dst)
            if ch >= 3:
                for frm, to, cname in ((23, 11, "srgb_lab"), (23, 26, "srgb_xyz"), (23, 21, "srgb_rgb"),
                                       (11, 23, "lab_srgb"), (21, 23, "rgb_srgb"), (23, 18, "srgb_ohta"),
                                       (23, 19, "srgb_rec601ycbcr"), (20, 23, "rec709ycbcr_srgb"), (23, 30, "srgb_yiq"),
                                       (32, 23, "yuv_srgb"), (23, 1, "srgb_cmy"), (27, 23, "ycbcr_srgb")):
                    buf = src.copy()
                    assert r.ref_colorspace(P(buf), W, H, ch, frm, to) == 0
                    record(f"colorspace_{cname}", buf)
    # kernel taps as the reference builds them
    for ks in ("blur:0x2", "blur:0x4", "blur:0x4+90", "blur:3x1.5", "gaussian:0x1.5", "gaussian:0x4", "Disk:3",
               "Disk:2.5", "Octagon:3", "Plus:2", "Cross:2", "Diamond:3", "Square:2", "Rectangle:5x3+1+2",
               "dog:0x2,1", "log:0x1.2", "binomial:2", "unity"):
        vals, x, y = util.ref_kernel(ks)
        out[f"kernel/{ks}"] = vals
        out[f"kernel_origin/{ks}"] = np.array([x, y])
    # tests/validate.c:244-259 known-answer (sRGB 0.545877,0.966567,0.463759 -> Lab)
    kat = (np.array([[[0.545877, 0.966567, 0.463759]]]) * 65535.0).astype(np.float32)
    buf = kat.copy()
    assert r.ref_colorspace(P(buf), 1, 1, 3, 23, 11) == 0
    out["kat/srgb"] = kat
    out["kat/lab"] = buf
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, OUT.stat().st_size, "bytes,", len(out), "arrays", len(util.REF_STORE.recorded), "digests",
          r.ref_version())


if __name__ == "__main__":
    main()
