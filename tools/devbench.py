"""Developer micro-benchmark: device-resident timings of the hot-path operators (CUDA events).
usage: python tools/devbench.py [blur|resize|lab|dilate|erode|gauss|conv2d|stencils|hooks|enhance|layout|level|direct|distort|
                                 geometry|threshold|trim|all]
       [size] [ref]   (ref: distort also times the reference's all-core DistortImage / RotateImage, minutes at 8192^2;
                       threshold and trim time the reference's all-core call beside theirs)"""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch
import imagemagick_b200 as im
from imagemagick_b200 import _lib

which = sys.argv[1] if len(sys.argv) > 1 else "all"
size = int(sys.argv[2]) if len(sys.argv) > 2 else 8192
from bench import measured_peak  # noqa: E402
PEAK, PEAK_SOURCE = measured_peak()


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def report(name, ms, npix, bytes_per_px):
    gbs = npix * bytes_per_px / ms / 1e6
    print(f"{name:34s} {ms:9.3f} ms  {npix / ms / 1e3:10.1f} Mpix/s  {gbs:8.1f} GB/s  {gbs / PEAK * 100:5.1f}% of {PEAK:.0f} GB/s HBM", flush=True)


torch.manual_seed(0)
if which in ("blur", "all"):
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    for sigma in (4.0, 2.0):
        ms = timeit(lambda: im.BlurImage(x, 0.0, sigma))
        report(f"BlurImage {size}^2 RGBA sigma={sigma}", ms, size * size, 64)
    k = im.AcquireKernelInfo("blur:0x4")
    ms = timeit(lambda: im.ConvolveImage(x, k)); report("  row pass only (33 taps)", ms, size * size, 32)
    k = im.AcquireKernelInfo("blur:0x4+90")
    ms = timeit(lambda: im.ConvolveImage(x, k)); report("  column pass only (33 taps)", ms, size * size, 32)
    del x
if which == "taps":          # DFMA streaming kernels against the FP64 mma.sync kernels, per window length
    from imagemagick_b200 import _lib
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    for mma in (0, 1):
        _lib.check(_lib.load().mb200_set_option(b"conv_mma", mma))
        for sigma in (1.0, 2.0, 3.0, 4.0):
            ms = timeit(lambda: im.BlurImage(x, 0.0, sigma))
            report(f"mma={mma} BlurImage sigma={sigma}", ms, size * size, 64)
        ms = timeit(lambda: im.GaussianBlurImage(x, 0.0, 4.0)); report(f"mma={mma} GaussianBlurImage(0,4) rank-1", ms, size * size, 32)
        ms = timeit(lambda: im.GaussianBlurImage(x, 0.0, 2.0)); report(f"mma={mma} GaussianBlurImage(0,2) rank-1", ms, size * size, 32)
        ms = timeit(lambda: im.UnsharpMaskImage(x, 0.0, 4.0, 1.5, 0.02)); report(f"mma={mma} UnsharpMaskImage(0,4)", ms, size * size, 80)
        ms = timeit(lambda: im.UnsharpMaskImage(x, 0.0, 2.0, 1.5, 0.02)); report(f"mma={mma} UnsharpMaskImage(0,2)", ms, size * size, 80)
    del x
if which in ("resize", "all"):
    s2 = size * 2 if size <= 8192 else size
    x = im.Image(torch.rand(s2, s2, 4, device="cuda") * 65535)
    ms = timeit(lambda: im.ResizeImage(x, s2 // 2, s2 // 2, im.LanczosFilter))
    report(f"ResizeImage {s2}^2->{s2 // 2}^2 Lanczos", ms, s2 * s2, 36)
    del x
if which in ("lab", "all"):
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    def f():
        x.colorspace = im.sRGBColorspace
        im.TransformImageColorspace(x, im.LabColorspace)
    ms = timeit(f); report(f"sRGB->Lab {size}^2", ms, size * size, 32)
    del x
if which in ("dilate", "all"):
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    k = im.AcquireKernelInfo("Disk:3")
    ms = timeit(lambda: im.MorphologyImage(x, im.DilateMorphology, 1, k)); report(f"Dilate Disk:3 {size}^2", ms, size * size, 32)
    del x
if which in ("erode", "all"):
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    k = im.AcquireKernelInfo("Disk:3")
    ms = timeit(lambda: im.MorphologyImage(x, im.ErodeMorphology, 1, k)); report(f"Erode Disk:3 {size}^2", ms, size * size, 32)
    del x
if which in ("gauss", "all"):
    s = min(size, 4096)
    x = im.Image(torch.rand(s, s, 4, device="cuda") * 65535)
    ms = timeit(lambda: im.GaussianBlurImage(x, 0.0, 4.0), iters=3, warm=1); report(f"GaussianBlurImage 2-D 29x29 {s}^2", ms, s * s, 32)

if which in ("conv2d", "all"):
    hd = im.Image(torch.rand(1080, 1920, 4, device="cuda") * 65535)
    ms = timeit(lambda: im.SharpenImage(hd, 5.0, 2.0), iters=9); report("SharpenImage 5x2 (11x11) 1920x1080", ms, 1920 * 1080, 32)
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    ms = timeit(lambda: im.SharpenImage(x, 5.0, 2.0)); report(f"SharpenImage 5x2 (11x11) {size}^2", ms, size * size, 32)
    ms = timeit(lambda: im.EdgeImage(x, 1.0)); report(f"EdgeImage(1) (3x3) {size}^2", ms, size * size, 32)
    ms = timeit(lambda: im.EmbossImage(x, 0.0, 1.0), iters=3); report(f"EmbossImage(0,1) {size}^2 (conv + equalize)", ms, size * size, 64)
    ms = timeit(lambda: im.ConvolveImage(x, "LoG:0x2")); report(f"ConvolveImage LoG:0x2 {size}^2", ms, size * size, 32)
    del x, hd
if which in ("stencils", "all"):
    s = min(size, 4096)
    x = im.Image(torch.rand(s, s, 4, device="cuda") * 65535)
    ms = timeit(lambda: im.StatisticImage(x, im.MedianStatistic, 3, 3), iters=3); report(f"StatisticImage Median 3x3 {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.StatisticImage(x, im.MeanStatistic, 5, 5), iters=3); report(f"StatisticImage Mean 5x5 {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.BilateralBlurImage(x, 7, 7, 20.0, 2.0), iters=3); report(f"BilateralBlurImage 7x7 {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.SelectiveBlurImage(x, 0.0, 1.5, 6553.5), iters=3); report(f"SelectiveBlurImage 0x1.5 t=10% {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.AdaptiveBlurImage(x, 0.0, 1.5), iters=3); report(f"AdaptiveBlurImage 0x1.5 {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.RotationalBlurImage(x, 5.0), iters=3); report(f"RotationalBlurImage(5) {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.MotionBlurImage(x, 0.0, 4.0, 30.0), iters=3); report(f"MotionBlurImage(0,4,30) {s}^2", ms, s * s, 32)
    ms = timeit(lambda: im.EqualizeImage(x), iters=3); report(f"EqualizeImage {s}^2", ms, s * s, 32)
if which in ("hooks", "all"):
    # the last three accelerate hooks at size^2 RGBA; bytes per pixel are the kernels' unique HBM traffic (DESIGN §5.7)
    import ctypes as C
    from imagemagick_b200 import _lib
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    ms = timeit(lambda: im.DespeckleImage(x), iters=3); report(f"DespeckleImage {size}^2 RGBA", ms, size * size, 128)
    ms = timeit(lambda: im.WaveletDenoiseImage(x, 6553.5, 0.0), iters=3)
    report(f"WaveletDenoiseImage 10% {size}^2 RGBA", ms, size * size, 240)
    rate = C.c_double(0.0)
    _lib.check(_lib.load().mb200_probe_fp64_fma_rate(C.byref(rate)))
    width = int(size * 0.002 * 10.0)
    fmas = 2 * (2 * width - 1) * size * size
    ms = timeit(lambda: im.LocalContrastImage(x, 10.0, 12.5), iters=3)
    print(f"{'LocalContrastImage 10x12.5 ' + str(size) + '^2 RGBA':34s} {ms:9.3f} ms  {fmas / 1e9:.1f} G DFMA  "
          f"{fmas / (ms * 1e-3) / 1e12:.2f} T DFMA/s  {fmas / (ms * 1e-3) / rate.value * 100:5.1f}% of the probed "
          f"{rate.value / 1e12:.2f} T DFMA/s", flush=True)
    del x
if which in ("enhance", "all"):
    # the in-place enhance operators at size^2 RGBA: an in-place pass reads and writes 16 B per pixel (32 B); Grayscale
    # reads 16 B and writes the 4 B gray sample (20 B).  Share of the 3.35 TB/s H100 SXM data-sheet HBM bandwidth.
    DATASHEET = 3350.0
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    for name, fn, bpp in [
            ("ContrastImage(sharpen)", lambda: im.ContrastImage(x, True), 32),
            ("ModulateImage 90,120,130 HSL", lambda: im.ModulateImage(x, "90,120,130"), 32),
            ("ModulateImage 90,120,130 HSB", lambda: im.ModulateImage(x, "90,120,130", {"modulate:colorspace": "HSB"}), 32),
            ("ModulateImage 90,120,130 LCHab", lambda: im.ModulateImage(x, "90,120,130", {"modulate:colorspace": "LCHab"}), 32),
            ("GrayscaleImage Rec709Luma", lambda: im.api._in_place(x, "mb200_grayscale_image_dev", "mb200_grayscale_image",
                                                                   im.Rec709LumaPixelIntensityMethod, im.sRGBColorspace), 20),
            ("GrayscaleImage Rec709Luminance", lambda: im.api._in_place(x, "mb200_grayscale_image_dev", "mb200_grayscale_image",
                                                                        im.Rec709LuminancePixelIntensityMethod, im.sRGBColorspace), 20),
            ("FunctionImage Polynomial 4", lambda: im.FunctionImage(x, im.PolynomialFunction, [0.5, -0.5, 0.75, 0.1]), 32),
            ("FunctionImage Sinusoid", lambda: im.FunctionImage(x, im.SinusoidFunction, [3.0, 45.0]), 32)]:
        x.pixels.copy_(torch.rand(size, size, 4, device="cuda") * 65535)
        ms = timeit(fn, iters=5)
        gbs = size * size * bpp / ms / 1e6
        print(f"{name + ' ' + str(size) + '^2 RGBA':44s} {ms:8.3f} ms  {bpp} B/px  {gbs:7.1f} GB/s  "
              f"{gbs / DATASHEET * 100:5.1f}% of {DATASHEET:.0f} GB/s", flush=True)
    del x
if which in ("layout", "all"):
    # TransformImageColorspace legs that change the channel layout, out of place on device buffers (the entry point
    # itself, without the Python layer's allocation).  Bytes per pixel: what the leg must read plus write; share of the
    # 3.35 TB/s H100 SXM data-sheet HBM bandwidth.
    from imagemagick_b200 import _lib
    DATASHEET = 3350.0
    lib = _lib.load()
    GRAY, LGRAY, CMYK, SRGB, LAB = im.GRAYColorspace, im.LinearGRAYColorspace, im.CMYKColorspace, im.sRGBColorspace, im.LabColorspace
    import ctypes as C
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream or 1)
    bufs = {ch: torch.rand(size, size, ch, device="cuda") * 65535 for ch in (1, 2, 3, 4, 5)}
    for name, frm, to, ich, och, bpp in [
            ("RGBA -> GA", SRGB, GRAY, 4, 2, 24), ("RGBA -> LinearGA", SRGB, LGRAY, 4, 2, 24),
            ("GA -> RGBA", GRAY, SRGB, 2, 4, 24), ("LinearGA -> RGBA", LGRAY, SRGB, 2, 4, 24),
            ("RGBA -> CMYKA", SRGB, CMYK, 4, 5, 36), ("CMYKA -> RGBA", CMYK, SRGB, 5, 4, 36),
            ("RGB -> GRAY", SRGB, GRAY, 3, 1, 16), ("RGB -> CMYK", SRGB, CMYK, 3, 4, 28),
            ("Lab RGBA -> GA (hop)", LAB, GRAY, 4, 2, 88)]:
        src, dst = bufs[ich], bufs[och]
        ms = timeit(lambda: _lib.check(lib.mb200_transform_colorspace_layout_dev(src.data_ptr(), ich, dst.data_ptr(), och, size,
                                                                                   size, frm, to, None, stream)), iters=9)
        gbs = size * size * bpp / ms / 1e6
        print(f"{name + ' ' + str(size) + '^2':44s} {ms:8.3f} ms  {bpp} B/px  {gbs:7.1f} GB/s  "
              f"{gbs / DATASHEET * 100:5.1f}% of {DATASHEET:.0f} GB/s", flush=True)
    del bufs
if which in ("level", "all"):
    # the level and stretch operators at size^2 RGBA, device-resident, with the card and its power limit (part of the
    # numbers).  Floor: the bytes each operator must move -- a histogram pass reads 16 B/px, an in-place pass reads and
    # writes 32 B/px, AutoLevel's range pass reads 16 B/px -- at the 3.35 TB/s H100 SXM data-sheet HBM bandwidth.
    import subprocess
    DATASHEET = 3350.0
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    print(f"level operators on {torch.cuda.get_device_name()} at a power limit of {limit or 'unknown'}", flush=True)
    n = size * size
    x = im.Image(torch.rand(size, size, 4, device="cuda") * 65535)
    for name, fn, bpp in [
            ("LevelImage 1000,60000,1", lambda: im.LevelImage(x, 1000.0, 60000.0, 1.0), 32),
            ("LevelImage 1000,60000,2.2", lambda: im.LevelImage(x, 1000.0, 60000.0, 2.2), 32),
            ("LevelizeImage 1000,60000,0.45", lambda: im.LevelizeImage(x, 1000.0, 60000.0, 0.45), 32),
            ("GammaImage 2.2", lambda: im.GammaImage(x, 2.2), 32),
            ("AutoLevelImage", lambda: im.AutoLevelImage(x), 48),
            ("AutoLevelImage -channel RGB", lambda: im.AutoLevelImage(x, 0b0111), 144),
            ("ContrastStretchImage 1%x97%", lambda: im.ContrastStretchImage(x, 0.01 * n, 0.97 * n), 48),
            ("NormalizeImage -channel RGBA", lambda: im.NormalizeImage(x, 0b1111), 48),
            ("LinearStretchImage 2%x1%", lambda: im.LinearStretchImage(x, 0.02 * n, 0.01 * n), 48)]:
        x.pixels.copy_(torch.rand(size, size, 4, device="cuda") * 65535)
        ms = timeit(fn, iters=5)
        gbs = size * size * bpp / ms / 1e6
        floor = size * size * bpp / DATASHEET / 1e6
        print(f"{name + ' ' + str(size) + '^2 RGBA':44s} {ms:8.3f} ms  floor {floor:6.3f} ms ({bpp} B/px)  {gbs:7.1f} GB/s  "
              f"{gbs / DATASHEET * 100:5.1f}% of {DATASHEET:.0f} GB/s", flush=True)
    del x
if which in ("direct", "all"):
    # Distance / Voronoi morphology at size^2 RGBA, device-resident, with the card and its power limit.  Floor: two
    # passes of 16 B/px read + 16 B/px written (64 B/px) at the 3.35 TB/s H100 SXM data-sheet HBM bandwidth.  Critical
    # path: wavefront steps of the two passes, (rows-1)*skew + columns each (skew = reach right + 1).  Where
    # oracle/_ref is built, the reference's own MorphologyImage runs single-threaded on the same image.
    import ctypes
    import subprocess
    import time
    import numpy as np
    DATASHEET = 3350.0
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    print(f"Distance / Voronoi on {torch.cuda.get_device_name()} at a power limit of {limit or 'unknown'}", flush=True)
    ref_so = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "libmagickref_direct.so"
    ref = ctypes.CDLL(str(ref_so)) if ref_so.exists() else None
    src = (torch.rand(size, size, 4, device="cuda") > 0.02).float() * 65535
    x = im.Image(src)
    host = src.cpu().numpy()
    floor = size * size * 64 / DATASHEET / 1e6
    for method, kernel in [(im.DistanceMorphology, "Euclidean"), (im.DistanceMorphology, "Euclidean:4"),
                           (im.DistanceMorphology, "Chebyshev:2"), (im.VoronoiMorphology, "Euclidean")]:
        vals, kx, ky = im.AcquireKernelInfo(kernel).arrays()[0]
        kh, kw = vals.shape
        steps = (size - 1) * (kx + 1) + size + (size - 1) * (kw - kx) + size
        ms = timeit(lambda: im.MorphologyDirectImage(x, method, kernel), iters=5)
        name = ("Distance " if method == im.DistanceMorphology else "Voronoi ") + kernel
        line = (f"{name + ' ' + str(size) + '^2 RGBA':36s} {ms:9.3f} ms  floor {floor:5.3f} ms = {floor / ms * 100:5.2f}%  "
                f"critical path {steps} steps ({ms * 1e6 / steps:6.1f} ns/step)")
        if ref is not None:
            ref.ref_set_threads(1)
            out = np.empty((size, size, 5), np.float32)
            trait = ctypes.c_int()
            t0 = time.perf_counter()
            rc = ref.ref_morphology_direct(ctypes.c_void_p(host.ctypes.data), ctypes.c_void_p(out.ctypes.data), ctypes.c_size_t(size), ctypes.c_size_t(size),
                                           4, method, ctypes.c_long(1), ctypes.c_char_p(kernel.encode()), ctypes.byref(trait))
            t = time.perf_counter() - t0
            line += f"  reference 1 thread {t * 1e3:9.1f} ms (rc {rc})"
        print(line, flush=True)
    del x

if which in ("distort", "all"):
    # DistortImage / RotateImage at size^2 RGBA, device-resident, with the card and its power limit.  Floor: 16 B/px
    # read + 16 B/px written per output pixel at the 3.35 TB/s H100 SXM data-sheet HBM bandwidth (the source is read
    # about once when the ellipse covers ~1 source pixel per output pixel).  With "ref", the reference itself runs on
    # all cores on the same image (oracle/_ref).
    import ctypes
    import subprocess
    import time
    import numpy as np
    DATASHEET = 3350.0
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    print(f"DistortImage on {torch.cuda.get_device_name()} at a power limit of {limit or 'unknown'}", flush=True)
    with_ref = len(sys.argv) > 3 and sys.argv[3] == "ref"
    ref_so = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "libmagickref_distort.so"
    ref = ctypes.CDLL(str(ref_so)) if with_ref and ref_so.exists() else None
    src = torch.rand(size, size, 4, device="cuda") * 65535
    x = im.Image(src)
    host = src.cpu().numpy()
    c = float(size)
    cases = [("RotateImage 30", 0, [30.0], True),
             ("SRT 0.5x 30deg", im.ScaleRotateTranslateDistortion, [0.5, 30.0], True),
             ("Affine 2x", im.AffineDistortion, [0, 0, 0, 0, c, 0, 2 * c, 0, 0, c, 0, 2 * c], True),
             ("Perspective with horizon", im.PerspectiveProjectionDistortion, [1.0, 0.3, 0.0, 0.0, 1.0, 0.0, 0.0, -0.6 / c],
              False)]
    for name, method, args, bestfit in cases:
        fn = (lambda: im.RotateImage(x, args[0])) if method == 0 else (lambda: im.DistortImage(x, method, args, bestfit))
        out = fn()
        npix = out.columns * out.rows
        ms = timeit(fn, iters=5)
        floor = npix * 32 / DATASHEET / 1e6
        line = (f"{name:26s} -> {out.columns}x{out.rows}  {ms:9.3f} ms  {npix / ms / 1e3:9.1f} Mpix/s  "
                f"floor {floor:6.3f} ms = {floor / ms * 100:5.2f}%")
        if ref is not None:
            buf = np.empty(npix * 4 + (1 << 22), np.float32)
            g = (ctypes.c_long * 4)()
            d = (ctypes.c_double * len(args))(*args)
            bg = (ctypes.c_double * 4)(65535.0, 65535.0, 65535.0, 65535.0)
            mt = (ctypes.c_double * 4)(48573.0, 48573.0, 48573.0, 65535.0)
            t0 = time.perf_counter()
            rc = ref.ref_distort(ctypes.c_void_p(host.ctypes.data), ctypes.c_size_t(size), ctypes.c_size_t(size), 4,
                                 ctypes.c_long(0), ctypes.c_long(0), method, d, ctypes.c_size_t(len(args)), int(bestfit),
                                 0, 0, 0, bg, 0, mt, 0, None, ctypes.c_void_p(buf.ctypes.data),
                                 ctypes.c_size_t(buf.size), g)
            line += f"  reference all cores {(time.perf_counter() - t0) * 1e3:9.1f} ms (rc {rc})"
        print(line, flush=True)
    del x

if which in ("geometry", "all"):
    # The orientation and crop operators at size^2 RGBA, device-resident, with the card and its power limit.  Floor:
    # 16 B/px read + 16 B/px written per output pixel at the 3.35 TB/s H100 SXM data-sheet HBM bandwidth; a plain
    # device-to-device copy of the same image is timed beside them.
    import subprocess
    DATASHEET = 3350.0
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    print(f"geometry operators on {torch.cuda.get_device_name()} at a power limit of {limit or 'unknown'}", flush=True)
    src = torch.rand(size, size, 4, device="cuda") * 65535
    x = im.Image(src)
    cases = [("copy (torch clone)", lambda: src.clone(), size * size),
             ("FlipImage", lambda: im.FlipImage(x), size * size),
             ("FlopImage", lambda: im.FlopImage(x), size * size),
             ("TransposeImage", lambda: im.TransposeImage(x), size * size),
             ("IntegralRotateImage 90", lambda: im.IntegralRotateImage(x, 1), size * size),
             ("CropImage half", lambda: im.CropImage(x, size // 2, size // 2, size // 4, size // 4), (size // 2) ** 2),
             ("RollImage +1000+777", lambda: im.RollImage(x, 1000, 777), size * size)]
    for name, fn, npix in cases:
        ms = timeit(fn, iters=20, warm=3)
        floor = npix * 32 / DATASHEET / 1e6
        print(f"{name:26s} {ms:9.3f} ms  {npix * 32 / ms / 1e6:8.1f} GB/s  floor {floor:6.3f} ms = {floor / ms * 100:5.1f}%",
              flush=True)
    del x, src

if which in ("threshold", "all"):
    # AdaptiveThreshold, AutoThreshold, RangeThreshold and Perceptible at size^2 RGBA, device-resident, with the card, its
    # power limit and max SM clock.  AdaptiveThreshold is bound by its serial chains (h+1 dependent DADDs per pixel and
    # chain, size * 4 chains), not by HBM: the time per dependent step is printed.  The in-place operators are timed on a
    # fresh copy of the source each run; the copy is timed alone and taken off ("operator" column).  With `ref` the
    # reference's all-core time of the same call on the same image is printed beside it (one run each).
    import ctypes
    import subprocess
    import time
    import numpy as np
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    print(f"threshold operators on {torch.cuda.get_device_name()} (power limit, max SM clock: {q or 'unknown'})", flush=True)
    with_ref = len(sys.argv) > 3 and sys.argv[3] == "ref"
    ref_so = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "libmagickref_threshold.so"
    ref = ctypes.CDLL(str(ref_so)) if with_ref and ref_so.exists() else None
    if with_ref and ref is None:
        print("reference not built (oracle/_ref/libmagickref_threshold.so): no reference times", flush=True)
    src = torch.rand(size, size, 4, device="cuda") * 65535
    x = im.Image(src)
    work = im.Image(src.clone())
    host = src.cpu().numpy() if ref is not None else None

    def ref_ms(op, args):
        if ref is None:
            return ""
        buf = np.empty(size * size * 4, np.float32)
        buf[:] = host.reshape(-1)
        a = (ctypes.c_double * 4)(*(list(args) + [0.0] * (4 - len(args))))
        prop = ctypes.create_string_buffer(64)
        t0 = time.perf_counter()
        rc = ref.ref_threshold_op(ctypes.c_void_p(buf.ctypes.data), ctypes.c_size_t(size), ctypes.c_size_t(size), 4, op, a,
                                  ctypes.c_long(-1), prop)
        return f"  reference all cores {(time.perf_counter() - t0) * 1e3:10.1f} ms (rc {rc})"

    def fresh(fn):
        def run():
            work.pixels.copy_(src)
            fn()
        return run
    copy_ms = timeit(lambda: work.pixels.copy_(src), iters=9, warm=2)
    print(f"{'device copy of the image':40s} {copy_ms:9.3f} ms", flush=True)
    for ww in (15, 51):
        for direct in (0, 1):
            _lib.load().mb200_set_option(b"no_adaptive_tile", direct)
            ms = timeit(lambda: im.AdaptiveThresholdImage(x, ww, ww, 65535 * 0.05), iters=7, warm=2)
            fam = "direct" if direct else "auto"
            line = (f"{'AdaptiveThreshold %dx%d+5%% (%s)' % (ww, ww, fam):40s} {ms:9.3f} ms  "
                    f"{ms * 1e6 / (size * (ww + 1)):8.3f} ns per dependent step")
            print(line + (ref_ms(0, (ww, ww, 65535 * 0.05)) if not direct else ""), flush=True)
        _lib.load().mb200_set_option(b"no_adaptive_tile", 0)
    for name, op, args, fn in [
            ("AutoThreshold OTSU", 1, (2,), lambda: im.AutoThresholdImage(work, im.OTSUThresholdMethod)),
            ("RangeThreshold", 2, (10000, 20000, 40000, 50000), lambda: im.RangeThresholdImage(work, 10000, 20000, 40000, 50000)),
            ("Perceptible 1000", 3, (1000.0,), lambda: im.PerceptibleImage(work, 1000.0))]:
        ms = timeit(fresh(fn), iters=9, warm=2)
        print(f"{name:40s} copy + operator {ms:9.3f} ms  operator {ms - copy_ms:7.3f} ms" + ref_ms(op, args), flush=True)
    del x, work, src

if which in ("trim", "all"):
    # GetImageBoundingBox and TrimImage at size^2 RGBA, device-resident, with the card, its power limit and max SM clock:
    # a framed object on a background whose four corners are equal (one comparison per pixel), then four distinct
    # corners (four).  The box call includes its readback of size * 16 B of row summaries and the synchronise.  Floors:
    # 16 B/px read at the 3.35 TB/s H100 SXM data-sheet HBM bandwidth, and the FP64 pipe at its data-sheet 33.5 TFLOP/s
    # (one operation per FP64 instruction: 64 per SM and clock) for the comparisons' FP64 instructions, counted from
    # fuzzy.cuh for RGBA: 4 float -> double conversions per pixel, and per comparison 6 for the alpha term, 1 for the x3
    # rescale and 5 per colour term (sub, mul, mul, add, compare) = 22.  With `ref` the reference's all-core time of the
    # same call on the same image is printed beside it (one run each).
    import ctypes
    import os
    import subprocess
    import time
    import numpy as np
    DATASHEET_BW, DATASHEET_FP64 = 3350.0, 33.5e12
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    print(f"bounding box and trim on {torch.cuda.get_device_name()} (power limit, max SM clock: {q or 'unknown'})",
          flush=True)
    with_ref = len(sys.argv) > 3 and sys.argv[3] == "ref"
    ref_so = Path(__file__).resolve().parent.parent / "oracle" / "_ref" / "libmagickref_trim.so"
    ref = ctypes.CDLL(str(ref_so)) if with_ref and ref_so.exists() else None
    if with_ref and ref is None:
        print("reference not built (oracle/_ref/libmagickref_trim.so): no reference times", flush=True)
    src = torch.full((size, size, 4), 1000.0, device="cuda")
    src[..., 1] = 20000.0
    src[..., 3] = 65535.0
    src[size // 5: size - size // 4, size // 6: size - size // 3] = torch.rand(size - size // 4 - size // 5,
                                                                               size - size // 3 - size // 6, 4,
                                                                               device="cuda") * 65535
    floor_bw = size * size * 16 / DATASHEET_BW / 1e6

    def ref_ms(image, op):
        if ref is None:
            return ""
        host = np.ascontiguousarray(image.cpu().numpy())
        lp = ctypes.c_long * 7
        box, geom, sev = lp(), lp(), ctypes.c_int(0)
        out = np.empty(host.size, np.float32) if op == 1 else np.empty(1, np.float32)
        t0 = time.perf_counter()
        rc = ref.ref_trim(ctypes.c_void_p(host.ctypes.data), ctypes.c_size_t(size), ctypes.c_size_t(size), 4, 0, -1,
                          (ctypes.c_long * 4)(), ctypes.c_double(0.0), None, None, 0, op, box, ctypes.byref(sev),
                          ctypes.c_void_p(out.ctypes.data), ctypes.c_size_t(out.size), geom, os.cpu_count())
        return f"  reference all cores {(time.perf_counter() - t0) * 1e3:9.1f} ms (rc {rc}, {os.cpu_count()} threads)"

    for corners in ("equal corners", "four distinct corners"):
        if corners != "equal corners":
            for k, (y, x) in enumerate([(0, 0), (0, size - 1), (size - 1, 0), (size - 1, size - 1)]):
                src[y, x, 0] = 1000.0 + 3000.0 * k
        x = im.Image(src)
        compares = 1 if corners == "equal corners" else 4
        floor_fp64 = size * size * (4 + 22 * compares) / DATASHEET_FP64 * 1e3
        ms = timeit(lambda: im.GetImageBoundingBox(x), iters=20, warm=3)
        print(f"{'GetImageBoundingBox ' + corners:44s} {ms:8.3f} ms  HBM floor {floor_bw:6.3f} ms ({floor_bw / ms * 100:5.1f}%)"
              f"  FP64 floor {floor_fp64:6.3f} ms ({floor_fp64 / ms * 100:5.1f}%)  box {im.GetImageBoundingBox(x)}"
              + ref_ms(src, 0), flush=True)
        ms = timeit(lambda: im.TrimImage(x), iters=20, warm=3)
        print(f"{'TrimImage ' + corners:44s} {ms:8.3f} ms" + ref_ms(src, 1), flush=True)
    del x, src
