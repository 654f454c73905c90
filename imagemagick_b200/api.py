"""Host-side mirror of the MagickCore entry points of the hot path.

Same names, argument meaning and error behaviour as the reference operators
(MagickCore/effect.c, morphology.c, resize.c, colorspace.c), on top of the C-ABI in
include/magick_b200.h:

    BlurImage, GaussianBlurImage, ConvolveImage, UnsharpMaskImage   effect.c:765/1709/1170/4256
    SharpenImage, EdgeImage, EmbossImage, MotionBlurImage           effect.c:3991/1520/1600/2347
    EqualizeImage                                                   enhance.c:2040
    BilateralBlurImage, RotationalBlurImage                         effect.c:821/3129
    StatisticImage                                                  statistic.c:2918
    DespeckleImage, LocalContrastImage                              effect.c:1308/2013
    WaveletDenoiseImage                                             visual-effects.c:3515
    MorphologyImage, AcquireKernelInfo                              morphology.c:4129/485
    MorphologyDirectImage (MorphologyImage: Distance, Voronoi)      morphology.c:3736-3776
    ResizeImage, SampleImage, ScaleImage, ThumbnailImage (pixel)    resize.c:3761/3907/4106/4591
    TransformImageColorspace                                        colorspace.c:1751
    BilevelImage, BlackThresholdImage, WhiteThresholdImage, ClampImage  threshold.c:805/927/2518/1087
    AdaptiveThresholdImage, AutoThresholdImage, RangeThresholdImage, PerceptibleImage  threshold.c:182/660/2377/2092
    ContrastImage, ModulateImage, GrayscaleImage                    enhance.c:1370/3461/2474
    FunctionImage                                                   statistic.c:1064
    LevelImage, LevelizeImage, GammaImage                           enhance.c:2913/3062/2322
    AutoLevelImage, MinMaxStretchImage                              enhance.c:187, histogram.c:927
    ContrastStretchImage, NormalizeImage, LinearStretchImage        enhance.c:1544/4130/3347
    DistortImage, RotateImage                                       distort.c:1754/2954
    CropImage, ShaveImage, RollImage, AutoOrientImage               transform.c:542/1641/1546/103
    FlipImage, FlopImage, TransposeImage, TransverseImage           transform.c:1194/1329/2127/2265
    IntegralRotateImage                                             shear.c:700
    GetImageBoundingBox, TrimImage                                  attribute.c:391, transform.c:2412

An `Image` wraps the pixel cache: an (rows, columns, channels) float32 array of raw
Quantum values (0..65535), either a NumPy array (host; every call stages through
HBM and back -- the end-to-end path) or a CUDA torch tensor (device-resident; the
kernels run on torch's current stream and the result stays in HBM).

Operators that return `Image *` in the reference return a NEW Image here and never
modify their input; TransformImageColorspace, the threshold operators, Contrast, Modulate,
Grayscale, Function and the level operators work in place and return True (the stretch operators: their
"histogram:*" property value), like the reference.  Failures raise MagickB200Error (the reference returns NULL / MagickFalse
and fills an ExceptionInfo); MB200_EUNSUPPORTED is the "decline" signal on which the
MagickCore shim falls back to the stock CPU path.  Nothing here computes pixels on
the CPU.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Union

import numpy as np

from . import _lib
from ._lib import KernelPtr, MagickB200Error, check

# MagickCore/morphology.h:69-99
UndefinedMorphology, ConvolveMorphology, CorrelateMorphology, ErodeMorphology, DilateMorphology = 0, 1, 2, 3, 4
OpenMorphology, CloseMorphology, SmoothMorphology = 8, 9, 12
EdgeInMorphology, EdgeOutMorphology, EdgeMorphology, TopHatMorphology, BottomHatMorphology = 13, 14, 15, 16, 17
ErodeIntensityMorphology, DilateIntensityMorphology, IterativeDistanceMorphology = 5, 6, 7
OpenIntensityMorphology, CloseIntensityMorphology = 10, 11
HitAndMissMorphology, ThinningMorphology, ThickenMorphology = 18, 19, 20
DistanceMorphology, VoronoiMorphology = 21, 22

# MagickCore/resample.h:32-69
(UndefinedFilter, PointFilter, BoxFilter, TriangleFilter, HermiteFilter, HannFilter, HammingFilter,
 BlackmanFilter, GaussianFilter, QuadraticFilter, CubicFilter, CatromFilter, MitchellFilter, JincFilter,
 SincFilter, SincFastFilter, KaiserFilter, WelchFilter, ParzenFilter, BohmanFilter, BartlettFilter,
 LagrangeFilter, LanczosFilter, LanczosSharpFilter, Lanczos2Filter, Lanczos2SharpFilter, RobidouxFilter,
 RobidouxSharpFilter, CosineFilter, SplineFilter, LanczosRadiusFilter, CubicSplineFilter,
 MagicKernelSharp2013Filter, MagicKernelSharp2021Filter, SentinelFilter) = range(35)

# MagickCore/colorspace.h:27-67
LabColorspace, RGBColorspace, sRGBColorspace, XYZColorspace = 11, 21, 23, 26
CMYColorspace, OHTAColorspace, Rec601YCbCrColorspace, Rec709YCbCrColorspace = 1, 18, 19, 20
YCbCrColorspace, YDbDrColorspace, YIQColorspace, YPbPrColorspace, YUVColorspace = 27, 29, 30, 31, 32
LCHColorspace, LCHabColorspace, LCHuvColorspace, OklabColorspace, OklchColorspace, JzazbzColorspace = 12, 13, 14, 38, 39, 34
LogColorspace, YCCColorspace = 15, 28
LMSColorspace, LuvColorspace, xyYColorspace, DisplayP3Colorspace, Adobe98Colorspace, ProPhotoColorspace, CAT02LMSColorspace = 16, 17, 25, 35, 36, 37, 40
HCLColorspace, HCLpColorspace, HSBColorspace, HSIColorspace, HSLColorspace, HSVColorspace, HWBColorspace = 4, 5, 6, 7, 8, 9, 10
GRAYColorspace, LinearGRAYColorspace = 3, 33
CMYKColorspace = 2
# the colourspaces whose pixel cache has a channel layout of its own: gray (+ alpha), C M Y K (+ alpha)
_LAYOUT_SPACES = {GRAYColorspace, LinearGRAYColorspace, CMYKColorspace}

# MagickCore/pixel.h:110-120
(UndefinedPixelIntensityMethod, AveragePixelIntensityMethod, BrightnessPixelIntensityMethod, LightnessPixelIntensityMethod,
 MSPixelIntensityMethod, Rec601LumaPixelIntensityMethod, Rec601LuminancePixelIntensityMethod, Rec709LumaPixelIntensityMethod,
 Rec709LuminancePixelIntensityMethod, RMSPixelIntensityMethod) = range(10)

# MagickCore/threshold.h AutoThresholdMethod
UndefinedThresholdMethod, KapurThresholdMethod, OTSUThresholdMethod, TriangleThresholdMethod = range(4)

# MagickCore/statistic.h:130-137
UndefinedFunction, ArcsinFunction, ArctanFunction, PolynomialFunction, SinusoidFunction = range(5)

# kernel types of include/magick_b200.h
(UserDefinedKernel, BlurKernel, GaussianKernel, DiskKernel, SquareKernel, DiamondKernel, OctagonKernel,
 PlusKernel, CrossKernel, RectangleKernel, UnityKernel, DoGKernel, LoGKernel, BinomialKernel) = range(14)


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


class Image:
    """The pixel cache of one image: rows x columns x channels float32 Quantum."""

    def __init__(self, pixels, colorspace: int = sRGBColorspace):
        if _is_torch(pixels):
            import torch
            if not pixels.is_cuda:
                raise ValueError("torch pixel caches must live on a CUDA device (use NumPy for host buffers)")
            if pixels.dtype != torch.float32 or pixels.dim() != 3:
                raise ValueError("pixels must be float32 of shape (rows, columns, channels)")
            pixels = pixels.contiguous()
        else:
            pixels = np.ascontiguousarray(pixels, dtype=np.float32)
            if pixels.ndim != 3:
                raise ValueError("pixels must have shape (rows, columns, channels)")
        if not 1 <= pixels.shape[2] <= (5 if colorspace == CMYKColorspace else 4):
            raise ValueError("1..4 channels (Gray, Gray+Alpha, RGB, RGBA), or 5 for CMYK with alpha")
        self.pixels = pixels
        self.colorspace = colorspace
        self.page = (0, 0)                 # the virtual canvas offset (page.x, page.y) DistortImage reads and sets
        self.page_size = (0, 0)            # the virtual canvas size (page.width, page.height); 0 = not set

    rows = property(lambda self: int(self.pixels.shape[0]))
    columns = property(lambda self: int(self.pixels.shape[1]))
    channels = property(lambda self: int(self.pixels.shape[2]))
    on_device = property(lambda self: _is_torch(self.pixels))

    def _ptr(self) -> int:
        return self.pixels.data_ptr() if self.on_device else self.pixels.ctypes.data

    def _new_like(self, rows: Optional[int] = None, columns: Optional[int] = None) -> "Image":
        shape = (rows or self.rows, columns or self.columns, self.channels)
        if self.on_device:
            import torch
            out = torch.empty(shape, dtype=torch.float32, device=self.pixels.device)
        else:
            out = np.empty(shape, dtype=np.float32)
        return Image(out, self.colorspace)


def _stream(image: Image):
    import torch
    handle = torch.cuda.current_stream(image.pixels.device).cuda_stream
    # torch's default stream is the legacy NULL stream; NULL means "library stream" in the
    # C-ABI, so name the legacy stream explicitly (cudaStreamLegacy == 0x1).
    return C.c_void_p(handle if handle else 1)


def _activate(image: Image) -> None:
    if image.on_device:
        import torch
        dev = image.pixels.device.index
        if dev is None:
            dev = torch.cuda.current_device()
        check(_lib.load().mb200_set_device(dev))


class KernelInfo:
    """Owning handle of a KernelInfo list (MagickCore/morphology.h:102-130)."""

    def __init__(self, ptr: KernelPtr):
        if not ptr:
            raise MagickB200Error(_lib.EINVAL, "kernel could not be parsed / built")
        self._ptr = ptr

    def __del__(self):
        ptr, self._ptr = getattr(self, "_ptr", None), None
        if ptr:
            try:
                _lib.load().mb200_destroy_kernel_info(ptr)
            except Exception:
                pass

    def __iter__(self):
        p = self._ptr
        while p:
            yield p.contents
            p = p.contents.next

    def arrays(self):
        """[(values(h,w) float64, x, y), ...] for every kernel of the list."""
        out = []
        for k in self:
            n = k.width * k.height
            vals = np.ctypeslib.as_array(k.values, shape=(n,)).copy().reshape(k.height, k.width)
            out.append((vals, int(k.x), int(k.y)))
        return out


def AcquireKernelInfo(kernel_string: str) -> KernelInfo:
    """MagickCore/morphology.c:485."""
    return KernelInfo(_lib.load().mb200_acquire_kernel_info(kernel_string.encode()))


def AcquireKernelBuiltIn(kernel_type: int, rho: float = 0.0, sigma: float = 0.0, xi: float = 0.0,
                         psi: float = 0.0) -> KernelInfo:
    """MagickCore/morphology.c:950 (GeometryInfo rho, sigma, xi, psi)."""
    return KernelInfo(_lib.load().mb200_acquire_kernel_builtin(kernel_type, rho, sigma, xi, psi))


def _as_kernel(kernel: Union[str, KernelInfo]) -> KernelInfo:
    return AcquireKernelInfo(kernel) if isinstance(kernel, str) else kernel


def _same_size_op(image: Image, dev_fn: str, host_fn: str, *args) -> Image:
    lib = _lib.load()
    out = image._new_like()
    if image.on_device:
        _activate(image)
        check(getattr(lib, dev_fn)(image._ptr(), out._ptr(), image.columns, image.rows, image.channels, *args,
                                   _stream(image)))
    else:
        check(getattr(lib, host_fn)(image._ptr(), out._ptr(), image.columns, image.rows, image.channels, *args))
    return out


def BlurImage(image: Image, radius: float, sigma: float) -> Image:
    """MagickCore/effect.c:765 -- separable Gaussian ("blur:RxS;blur:RxS+90")."""
    return _same_size_op(image, "mb200_blur_image_dev", "mb200_blur_image", float(radius), float(sigma))


def GaussianBlurImage(image: Image, radius: float, sigma: float) -> Image:
    """MagickCore/effect.c:1709 -- true 2-D "gaussian:RxS" kernel."""
    return _same_size_op(image, "mb200_gaussian_blur_image_dev", "mb200_gaussian_blur_image", float(radius),
                         float(sigma))


def ConvolveImage(image: Image, kernel_info: Union[str, KernelInfo]) -> Image:
    """MagickCore/effect.c:1170."""
    k = _as_kernel(kernel_info)
    return _same_size_op(image, "mb200_convolve_image_dev", "mb200_convolve_image", k._ptr)


def MorphologyImage(image: Image, method: int, iterations: int, kernel: Union[str, KernelInfo],
                    bias: float = 0.0) -> Image:
    """MagickCore/morphology.c:4129 (bias == the "convolve:bias" artifact).  Distance and Voronoi are declined
    (MB200_EUNSUPPORTED) here; MorphologyDirectImage runs them."""
    k = _as_kernel(kernel)
    return _same_size_op(image, "mb200_morphology_image_dev", "mb200_morphology_image", int(method),
                         int(iterations), k._ptr, float(bias))


def MorphologyDirectImage(image: Image, method: int, kernel: Union[str, KernelInfo]) -> Image:
    """MorphologyImage with DistanceMorphology or VoronoiMorphology (MagickCore/morphology.c:3736-3776): one forward and
    one reverse sweep with the head kernel of the list -- the reference ignores the iteration count (0 aside) and the
    bias for these methods.  Voronoi needs an image with alpha (its result takes the source's alpha, and the reference
    leaves the alpha trait at Copy); on an image without alpha it raises MB200_EUNSUPPORTED, because the reference's
    result has one channel more."""
    k = _as_kernel(kernel)
    return _same_size_op(image, "mb200_morphology_direct_image_dev", "mb200_morphology_direct_image", int(method),
                         k._ptr)


def UnsharpMaskImage(image: Image, radius: float, sigma: float, gain: float, threshold: float) -> Image:
    """MagickCore/effect.c:4256."""
    return _same_size_op(image, "mb200_unsharp_mask_image_dev", "mb200_unsharp_mask_image", float(radius),
                         float(sigma), float(gain), float(threshold))


def SharpenImage(image: Image, radius: float, sigma: float) -> Image:
    """MagickCore/effect.c:3991 -- ConvolveImage with the inline sharpening kernel."""
    return _same_size_op(image, "mb200_sharpen_image_dev", "mb200_sharpen_image", float(radius), float(sigma))


def EdgeImage(image: Image, radius: float) -> Image:
    """MagickCore/effect.c:1520 -- ConvolveImage with the all -1 / centre n-1 kernel."""
    return _same_size_op(image, "mb200_edge_image_dev", "mb200_edge_image", float(radius))


def EmbossImage(image: Image, radius: float, sigma: float) -> Image:
    """MagickCore/effect.c:1600 -- ConvolveImage with the anti-diagonal emboss kernel, then EqualizeImage."""
    return _same_size_op(image, "mb200_emboss_image_dev", "mb200_emboss_image", float(radius), float(sigma))


def EqualizeImage(image: Image, sync_channels: bool = True) -> bool:
    """MagickCore/enhance.c:2040 -- in place.  sync_channels: the channel mask carries SyncChannels (the default)."""
    return _in_place(image, "mb200_equalize_image_dev", "mb200_equalize_image", int(bool(sync_channels)))


# MagickCore/statistic.h:141-151
(UndefinedStatistic, GradientStatistic, MaximumStatistic, MeanStatistic, MedianStatistic, MinimumStatistic, ModeStatistic,
 NonpeakStatistic, RootMeanSquareStatistic, StandardDeviationStatistic, ContrastStatistic) = range(11)


def StatisticImage(image: Image, statistic_type: int, width: int, height: int) -> Image:
    """MagickCore/statistic.c:2918."""
    return _same_size_op(image, "mb200_statistic_image_dev", "mb200_statistic_image", int(statistic_type), int(width),
                         int(height))


def RotationalBlurImage(image: Image, angle: float) -> Image:
    """MagickCore/effect.c:3129."""
    return _same_size_op(image, "mb200_rotational_blur_image_dev", "mb200_rotational_blur_image", float(angle))


def BilateralBlurImage(image: Image, width: int, height: int, intensity_sigma: float, spatial_sigma: float) -> Image:
    """MagickCore/effect.c:821."""
    return _same_size_op(image, "mb200_bilateral_blur_image_dev", "mb200_bilateral_blur_image", int(width), int(height),
                         float(intensity_sigma), float(spatial_sigma))


def AdaptiveBlurImage(image: Image, radius: float, sigma: float) -> Image:
    """MagickCore/effect.c:128."""
    return _same_size_op(image, "mb200_adaptive_blur_image_dev", "mb200_adaptive_blur_image", float(radius), float(sigma))


def AdaptiveSharpenImage(image: Image, radius: float, sigma: float) -> Image:
    """MagickCore/effect.c:447."""
    return _same_size_op(image, "mb200_adaptive_sharpen_image_dev", "mb200_adaptive_sharpen_image", float(radius), float(sigma))


def SelectiveBlurImage(image: Image, radius: float, sigma: float, threshold: float) -> Image:
    """MagickCore/effect.c:3406 (threshold in quantum units)."""
    return _same_size_op(image, "mb200_selective_blur_image_dev", "mb200_selective_blur_image", float(radius), float(sigma),
                         float(threshold))


def DespeckleImage(image: Image) -> Image:
    """MagickCore/effect.c:1308."""
    return _same_size_op(image, "mb200_despeckle_image_dev", "mb200_despeckle_image")


def LocalContrastImage(image: Image, radius: float, strength: float) -> Image:
    """MagickCore/effect.c:2013 (-local-contrast RxS).  MagickB200Error (EUNSUPPORTED) where the kernel width
    max(columns, rows) * 0.002 * |radius| exceeds columns - 1."""
    return _same_size_op(image, "mb200_local_contrast_image_dev", "mb200_local_contrast_image", float(radius),
                         float(strength))


def WaveletDenoiseImage(image: Image, threshold: float, softness: float = 0.0) -> Image:
    """MagickCore/visual-effects.c:3515 (threshold in quantum units).  MagickB200Error (EUNSUPPORTED) below 32x32."""
    return _same_size_op(image, "mb200_wavelet_denoise_image_dev", "mb200_wavelet_denoise_image", float(threshold),
                         float(softness))


def MotionBlurImage(image: Image, radius: float, sigma: float, angle: float) -> Image:
    """MagickCore/effect.c:2347."""
    return _same_size_op(image, "mb200_motion_blur_image_dev", "mb200_motion_blur_image", float(radius), float(sigma),
                         float(angle))


class FilterOptions(C.Structure):
    """mb200_filter_options: the "filter:*" expert settings of AcquireResizeFilter (MagickCore/resize.c:999-1226) as values."""
    _fields_ = [("set", C.c_uint), ("window", C.c_int), ("keep_filter", C.c_int), ("lobes", C.c_long), ("sigma", C.c_double),
                ("kaiser_beta", C.c_double), ("blur", C.c_double), ("support", C.c_double), ("win_support", C.c_double),
                ("b", C.c_double), ("c", C.c_double)]


_FILTER_NAMES = {n[:-len("Filter")].lower(): v for n, v in list(globals().items())
                 if n.endswith("Filter") and isinstance(v, int)}


def filter_options_from_artifacts(artifacts) -> "FilterOptions | None":
    """What the shim does in C (b200_filter_options): read the -define filter:* strings the way the reference does."""
    if not artifacts:
        return None
    o = FilterOptions()
    truthy = str(artifacts.get("filter:filter", "")).strip().lower() in ("true", "yes", "on", "1")
    w = artifacts.get("filter:window")
    if w is not None and str(w).strip().lower() in _FILTER_NAMES and _FILTER_NAMES[str(w).strip().lower()] > 0:
        o.window, o.keep_filter, o.set = _FILTER_NAMES[str(w).strip().lower()], int(truthy), o.set | 1
    for key, field, bit in (("filter:sigma", "sigma", 2), ("filter:alpha", "kaiser_beta", 4), ("filter:kaiser-beta", "kaiser_beta", 4),
                            ("filter:blur", "blur", 16), ("filter:support", "support", 32), ("filter:win-support", "win_support", 64),
                            ("filter:b", "b", 128), ("filter:c", "c", 256)):
        if key in artifacts:
            setattr(o, field, float(artifacts[key]))
            o.set |= bit
    if "filter:kaiser-alpha" in artifacts:
        o.kaiser_beta, o.set = float(artifacts["filter:kaiser-alpha"]) * 3.14159265358979323846264338327950288419716939937510, o.set | 4
    if "filter:lobes" in artifacts:
        o.lobes, o.set = int(float(artifacts["filter:lobes"])), o.set | 8
    return o if o.set else None


def ResizeImage(image: Image, columns: int, rows: int, filter: int = UndefinedFilter, artifacts=None) -> Image:
    """MagickCore/resize.c:3761.  `artifacts`: the image's "-define filter:*" settings, e.g. {"filter:blur": "0.8"}."""
    if columns <= 0 or rows <= 0:
        raise MagickB200Error(_lib.EINVAL, "NegativeOrZeroImageSize")
    lib = _lib.load()
    out = image._new_like(rows=rows, columns=columns)
    opts = filter_options_from_artifacts(artifacts)
    ref = C.byref(opts) if opts is not None else None
    if image.on_device:
        _activate(image)
        check(lib.mb200_resize_image_ex_dev(image._ptr(), image.columns, image.rows, image.channels, out._ptr(),
                                            columns, rows, int(filter), ref, _stream(image)))
    else:
        check(lib.mb200_resize_image_ex(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns,
                                        rows, int(filter), ref))
    return out


class DistortParams(C.Structure):
    """mb200_distort_params: the reverse map and output geometry mb200_distort_plan / mb200_rotate_plan compute."""
    _fields_ = [("map", C.c_int), ("coeff", C.c_double * 9), ("columns", C.c_size_t), ("rows", C.c_size_t),
                ("page_x", C.c_long), ("page_y", C.c_long), ("output_scaling", C.c_double), ("bestfit", C.c_int),
                ("src_page_x", C.c_long), ("src_page_y", C.c_long)]


class ResampleOptions(C.Structure):
    """mb200_resample_options: the source image's filter, virtual-pixel method, interpolate and colours."""
    _fields_ = [("filter", C.c_int), ("filter_options", C.c_void_p), ("virtual_pixel", C.c_int),
                ("interpolate", C.c_int), ("background", C.c_double * 4), ("matte", C.c_double * 4),
                ("matte_alpha", C.c_int)]


# MagickCore/distort.h DistortMethod; cache-view.h VirtualPixelMethod; pixel.h PixelInterpolateMethod
(AffineDistortion, AffineProjectionDistortion, ScaleRotateTranslateDistortion, PerspectiveDistortion,
 PerspectiveProjectionDistortion) = 1, 2, 3, 4, 5
RigidAffineDistortion = 19
(UndefinedVirtualPixelMethod, BackgroundVirtualPixelMethod, EdgeVirtualPixelMethod, TransparentVirtualPixelMethod,
 BlackVirtualPixelMethod, GrayVirtualPixelMethod, WhiteVirtualPixelMethod) = 0, 1, 3, 7, 9, 10, 11
UndefinedInterpolatePixel, BilinearInterpolatePixel = 0, 5
WHITE = (65535.0, 65535.0, 65535.0)                      # BackgroundColorRGBA (image-private.h:32)
MATTE = (48573.0, 48573.0, 48573.0)                      # MatteColorRGBA #BDBDBD (image-private.h:56)


def DistortPlan(image: Image, method: int, arguments, bestfit: bool = False, viewport=None,
                scale: Optional[float] = None) -> DistortParams:
    """GenerateCoefficients and the output geometry of MagickCore/distort.c:1754 for the affine and perspective methods,
    on the host.  viewport: (width, height, x, y), the "distort:viewport" geometry; scale: "distort:scale"."""
    args = (C.c_double * max(1, len(arguments)))(*[float(a) for a in arguments])
    vp = (C.c_long * 4)(*[int(v) for v in viewport]) if viewport is not None else None
    plan = DistortParams()
    page = getattr(image, "page", (0, 0))
    check(_lib.load().mb200_distort_plan(int(method), args, len(arguments), int(bool(bestfit)), image.columns,
                                         image.rows, int(page[0]), int(page[1]), vp, float("nan") if scale is None else float(scale),
                                         C.byref(plan)))
    return plan


def _opaque_alpha(image: Image) -> Image:
    """The image with an opaque alpha channel appended (Gray -> Gray+Alpha, RGB -> RGBA), page kept."""
    if image.on_device:
        import torch
        a = torch.full((image.rows, image.columns, 1), 65535.0, dtype=torch.float32, device=image.pixels.device)
        out = Image(torch.cat([image.pixels, a], dim=2), image.colorspace)
    else:
        out = Image(np.concatenate([image.pixels, np.full((image.rows, image.columns, 1), 65535.0, np.float32)], axis=2),
                    image.colorspace)
    out.page = getattr(image, "page", (0, 0))
    return out


def _distort(image: Image, plan: DistortParams, filter: int, virtual_pixel: int, interpolate: int, background,
             matte_color, artifacts) -> Image:
    if image.colorspace == CMYKColorspace:
        raise MagickB200Error(_lib.EUNSUPPORTED, "distort: CMYK (its black channel) is not implemented")
    bg = tuple(background) + (65535.0,) * (4 - len(background))
    if image.channels in (1, 2) and not bg[0] == bg[1] == bg[2]:
        raise MagickB200Error(_lib.EUNSUPPORTED, "distort: a gray image with a non-gray background becomes sRGB")
    if image.channels in (1, 3) and len(matte_color) == 4:
        raise MagickB200Error(_lib.EUNSUPPORTED, "distort: a matte colour with alpha adds alpha inside DistortImage")
    if image.channels in (1, 3) and len(background) == 4 and virtual_pixel not in (BackgroundVirtualPixelMethod,
                                                                                    TransparentVirtualPixelMethod):
        raise MagickB200Error(_lib.EUNSUPPORTED, "distort: a background with alpha adds alpha inside DistortImage")
    if image.channels in (1, 3) and ((len(background) == 4 and virtual_pixel == BackgroundVirtualPixelMethod) or
                                     virtual_pixel == TransparentVirtualPixelMethod):
        # SetImageVirtualPixelMethod(Background with alpha / Transparent) gives the source an opaque alpha channel
        # before the reference resamples it (cache.c:5294-5309)
        image = _opaque_alpha(image)
    opts = ResampleOptions(filter=int(filter), virtual_pixel=int(virtual_pixel), interpolate=int(interpolate))
    fo = filter_options_from_artifacts(artifacts)
    opts.filter_options = C.cast(C.byref(fo), C.c_void_p) if fo is not None else None
    opts.background[:] = [float(v) for v in bg]
    opts.matte[:] = [float(v) for v in tuple(matte_color) + (65535.0,) * (4 - len(matte_color))]
    opts.matte_alpha = int(len(matte_color) == 4)
    lib = _lib.load()
    out = image._new_like(rows=plan.rows, columns=plan.columns)
    if image.on_device:
        _activate(image)
        check(lib.mb200_distort_image_dev(image._ptr(), image.columns, image.rows, image.channels, out._ptr(),
                                          C.byref(plan), C.byref(opts), _stream(image)))
    else:
        check(lib.mb200_distort_image(image._ptr(), image.columns, image.rows, image.channels, out._ptr(),
                                      C.byref(plan), C.byref(opts)))
    out.page = (plan.page_x, plan.page_y)
    return out


def DistortImage(image: Image, method: int, arguments, bestfit: bool = False, *, filter: int = UndefinedFilter,
                 virtual_pixel: int = UndefinedVirtualPixelMethod, interpolate: int = UndefinedInterpolatePixel,
                 background=WHITE, matte_color=MATTE, viewport=None, scale: Optional[float] = None,
                 artifacts=None) -> Image:
    """MagickCore/distort.c:1754 with Affine, AffineProjection, ScaleRotateTranslate, RigidAffine, Perspective
    and PerspectiveProjection, through the EWA sampler of resample.c; bit exact.  `image.page` (default (0, 0)) is read and
    the result's page set.  filter / virtual_pixel / interpolate / background / matte_color are the source image's
    settings (a 4-tuple colour has an alpha trait); viewport / scale are "distort:viewport" / "distort:scale" as values,
    artifacts the "filter:*" settings.  As SetImageVirtualPixelMethod does, a Gray or RGB image gains an opaque alpha
    channel for Transparent virtual pixels, or Background ones with a background that has an alpha trait; other
    colours with an alpha trait on such an image (the reference adds alpha inside DistortImage), CMYK, and a Gray image with a non-gray background (the reference turns it into sRGB), raise MB200_EUNSUPPORTED."""
    plan = DistortPlan(image, method, arguments, bestfit, viewport, scale)
    return _distort(image, plan, filter, virtual_pixel, interpolate, background, matte_color, artifacts)


def RotateImage(image: Image, degrees: float, background=WHITE, *, filter: int = UndefinedFilter,
                matte_color=MATTE) -> Image:
    """MagickCore/distort.c:2954 for angles that are not a multiple of 90 degrees (those raise MB200_EUNSUPPORTED):
    DistortImage(ScaleRotateTranslate, bestfit) with Background virtual pixels.  A 4-tuple background has an alpha
    trait: a Gray or RGB image then gains an opaque alpha channel, as SetImageVirtualPixelMethod gives it one."""
    plan = DistortParams()
    page = getattr(image, "page", (0, 0))
    check(_lib.load().mb200_rotate_plan(float(degrees), image.columns, image.rows, int(page[0]), int(page[1]),
                                        C.byref(plan)))
    return _distort(image, plan, filter, BackgroundVirtualPixelMethod, UndefinedInterpolatePixel, background,
                    matte_color, None)


class Page(C.Structure):
    """mb200_page: an image's RectangleInfo page."""
    _fields_ = [("width", C.c_size_t), ("height", C.c_size_t), ("x", C.c_long), ("y", C.c_long)]


class GeometryParams(C.Structure):
    """mb200_geometry_params: the output geometry, page and map mb200_geometry_plan computes."""
    _fields_ = [("map", C.c_int), ("columns", C.c_size_t), ("rows", C.c_size_t), ("page", Page),
                ("src_x", C.c_long), ("src_y", C.c_long), ("roll_x", C.c_long), ("roll_y", C.c_long)]


# mb200_geometry_op (include/magick_b200.h)
(GeometryCrop, GeometryShave, GeometryFlip, GeometryFlop, GeometryTranspose, GeometryTransverse,
 GeometryIntegralRotate, GeometryRoll) = range(8)
# MagickCore/image.h OrientationType
(UndefinedOrientation, TopLeftOrientation, TopRightOrientation, BottomRightOrientation, BottomLeftOrientation,
 LeftTopOrientation, RightTopOrientation, RightBottomOrientation, LeftBottomOrientation) = range(9)


def GeometryPlan(image: Image, op: int, arguments=()) -> GeometryParams:
    """The output geometry, page and map of one orientation or crop operator, on the host (mb200_geometry_plan).
    `image.page` and `image.page_size` are the source's page."""
    page = Page(*getattr(image, "page_size", (0, 0)), *getattr(image, "page", (0, 0)))
    args = (C.c_long * 4)(*[int(a) for a in arguments])
    plan = GeometryParams()
    check(_lib.load().mb200_geometry_plan(int(op), image.columns, image.rows, C.byref(page), args, C.byref(plan)))
    return plan


def _geometry(image: Image, op: int, arguments=()) -> Image:
    return _run_geometry(image, GeometryPlan(image, op, arguments))


def _run_geometry(image: Image, plan: GeometryParams) -> Image:
    lib = _lib.load()
    out = image._new_like(rows=plan.rows, columns=plan.columns)
    if image.on_device:
        _activate(image)
        check(lib.mb200_geometry_image_dev(image._ptr(), image.columns, image.rows, image.channels, out._ptr(),
                                           C.byref(plan), _stream(image)))
    else:
        check(lib.mb200_geometry_image(image._ptr(), image.columns, image.rows, image.channels, out._ptr(),
                                       C.byref(plan)))
    out.page = (plan.page.x, plan.page.y)
    out.page_size = (plan.page.width, plan.page.height)
    return out


def CropImage(image: Image, width: int, height: int, x: int = 0, y: int = 0) -> Image:
    """MagickCore/transform.c:542 with the geometry WxH+X+Y (0 = the page's width / height), against the image's page;
    bit exact.  A crop outside the virtual canvas or of zero area raises MB200_EUNSUPPORTED (the reference warns and
    returns a transparent 1x1 image or none)."""
    return _geometry(image, GeometryCrop, (width, height, x, y))


def ShaveImage(image: Image, width: int, height: int) -> Image:
    """MagickCore/transform.c:1641; shaving half the image or more raises MB200_EUNSUPPORTED, as the reference warns."""
    return _geometry(image, GeometryShave, (width, height))


def FlipImage(image: Image) -> Image:
    """MagickCore/transform.c:1194: the rows in reverse order."""
    return _geometry(image, GeometryFlip)


def FlopImage(image: Image) -> Image:
    """MagickCore/transform.c:1329: the columns in reverse order."""
    return _geometry(image, GeometryFlop)


def TransposeImage(image: Image) -> Image:
    """MagickCore/transform.c:2127: mirrored along the top-left to bottom-right diagonal."""
    return _geometry(image, GeometryTranspose)


def TransverseImage(image: Image) -> Image:
    """MagickCore/transform.c:2265: mirrored along the bottom-left to top-right diagonal."""
    return _geometry(image, GeometryTransverse)


def IntegralRotateImage(image: Image, rotations: int) -> Image:
    """MagickCore/shear.c:700: `rotations` quarter turns clockwise, taken mod 4 (as a size_t: -1 is 3).  0 raises
    MB200_EUNSUPPORTED: the reference returns a clone."""
    return _geometry(image, GeometryIntegralRotate, (rotations,))


def RollImage(image: Image, x_offset: int, y_offset: int) -> Image:
    """MagickCore/transform.c:1546: the image shifted by (x_offset, y_offset), wrapping around its edges."""
    return _geometry(image, GeometryRoll, (x_offset, y_offset))


def AutoOrientImage(image: Image, orientation: int) -> Image:
    """MagickCore/transform.c:103: the image brought to TopLeft from `orientation` (the reference's own dispatch to
    Flop, Flip, Transpose, Transverse and RotateImage by 90, 180 or 270 degrees, which is IntegralRotateImage).
    Undefined and TopLeft raise MB200_EUNSUPPORTED: the reference returns a clone."""
    ops = {TopRightOrientation: (GeometryFlop, ()), BottomRightOrientation: (GeometryIntegralRotate, (2,)),
           BottomLeftOrientation: (GeometryFlip, ()), LeftTopOrientation: (GeometryTranspose, ()),
           RightTopOrientation: (GeometryIntegralRotate, (1,)), RightBottomOrientation: (GeometryTransverse, ()),
           LeftBottomOrientation: (GeometryIntegralRotate, (3,))}
    if orientation not in ops:
        raise MagickB200Error(_lib.EUNSUPPORTED, "auto-orient: already TopLeft (the reference returns a clone)")
    return _geometry(image, *ops[orientation])


# MagickCore/geometry.h GravityType
(UndefinedGravity, NorthWestGravity, NorthGravity, NorthEastGravity, WestGravity, CenterGravity, EastGravity,
 SouthWestGravity, SouthGravity, SouthEastGravity) = range(10)
ForgetGravity = UndefinedGravity
# mb200_trim_edge: the edges a "trim:edges" artifact names
TrimEdgeNorth, TrimEdgeEast, TrimEdgeSouth, TrimEdgeWest = 1, 2, 4, 8
TRIM_EDGES_UNSET = -1


class TrimOptions(C.Structure):
    """mb200_trim_options: the image settings GetImageBoundingBox reads."""
    _fields_ = [("fuzz", C.c_double), ("edges", C.c_int), ("colorspace", C.c_int)]


def trim_edges(artifact: Optional[str]) -> int:
    """The mb200_trim_edge bits of a "trim:edges" artifact, split on ',' and compared without case as attribute.c:444-454
    does (other tokens count for nothing); TRIM_EDGES_UNSET for None."""
    if artifact is None:
        return TRIM_EDGES_UNSET
    bits = {"north": TrimEdgeNorth, "east": TrimEdgeEast, "south": TrimEdgeSouth, "west": TrimEdgeWest}
    edges = 0
    for token in artifact.split(","):
        edges |= bits.get(token.lower(), 0)
    return edges


def BoundingBoxWarning(image: Image, fuzz: float = 0.0, edges: Optional[str] = None):
    """GetImageBoundingBox's box and whether the reference warns GeometryDoesNotContainImage for it (the scan left a
    zero width or height; the final arithmetic can give a zero side without the warning)."""
    options = TrimOptions(float(fuzz), trim_edges(edges), int(image.colorspace))
    box = Page()
    warning = C.c_int(0)
    lib = _lib.load()
    if image.on_device:
        _activate(image)
        check(lib.mb200_bounding_box_dev(image._ptr(), image.columns, image.rows, image.channels, C.byref(options),
                                         C.byref(box), C.byref(warning), _stream(image)))
    else:
        check(lib.mb200_bounding_box(image._ptr(), image.columns, image.rows, image.channels, C.byref(options),
                                     C.byref(box), C.byref(warning)))
    return (int(box.width), int(box.height), int(box.x), int(box.y)), bool(warning.value)


def GetImageBoundingBox(image: Image, fuzz: float = 0.0, edges: Optional[str] = None):
    """MagickCore/attribute.c:391 -- (width, height, x, y) of the region that differs, beyond `fuzz`, from the corner
    pixels; `edges` is the "trim:edges" artifact.  Bit exact, with the reference's single-threaded result.  A box of zero
    width or height is returned as it is (BoundingBoxWarning tells whether the reference warns)."""
    return BoundingBoxWarning(image, fuzz, edges)[0]


def TrimImage(image: Image, fuzz: float = 0.0, edges: Optional[str] = None, min_size=None,
              gravity: int = UndefinedGravity) -> Image:
    """MagickCore/transform.c:2412: CropImage to GetImageBoundingBox, grown to `min_size` (width, height; the
    "trim:minSize" artifact) under `gravity` when both sides of the box are smaller.  Bit exact; one bounding-box scan
    and one crop.  A zero box raises MB200_EUNSUPPORTED (the reference warns and returns a transparent 1x1 image), as do
    the crops CropImage declines."""
    width, height, x, y = GetImageBoundingBox(image, fuzz, edges)
    box = Page(width, height, x, y)
    page = Page(*image.page_size, *image.page)
    size = None if min_size is None else (C.c_size_t * 2)(*[int(v) for v in min_size])
    plan = GeometryParams()
    check(_lib.load().mb200_trim_plan(image.columns, image.rows, C.byref(page), C.byref(box), int(gravity), size,
                                      C.byref(plan)))
    return _run_geometry(image, plan)


def SampleImage(image: Image, columns: int, rows: int) -> Image:
    """MagickCore/resize.c:3907 -- nearest-sample gather."""
    if columns <= 0 or rows <= 0:
        raise MagickB200Error(_lib.EINVAL, "NegativeOrZeroImageSize")
    lib = _lib.load()
    out = image._new_like(rows=rows, columns=columns)
    if image.on_device:
        _activate(image)
        check(lib.mb200_sample_image_dev(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns,
                                         rows, _stream(image)))
    else:
        check(lib.mb200_sample_image(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns, rows))
    return out


def ScaleImage(image: Image, columns: int, rows: int) -> Image:
    """MagickCore/resize.c:4106 -- box scaling."""
    if columns <= 0 or rows <= 0:
        raise MagickB200Error(_lib.EINVAL, "NegativeOrZeroImageSize")
    lib = _lib.load()
    out = image._new_like(rows=rows, columns=columns)
    if image.on_device:
        _activate(image)
        check(lib.mb200_scale_image_dev(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns, rows,
                                        _stream(image)))
    else:
        check(lib.mb200_scale_image(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns, rows))
    return out


def ThumbnailImage(image: Image, columns: int, rows: int, filter: int = UndefinedFilter) -> Image:
    """MagickCore/resize.c:4591 -- pixel path (sample / box / LanczosSharp cascade); `filter` is image->filter."""
    if columns <= 0 or rows <= 0:
        raise MagickB200Error(_lib.EINVAL, "NegativeOrZeroImageSize")
    lib = _lib.load()
    out = image._new_like(rows=rows, columns=columns)
    if image.on_device:
        _activate(image)
        check(lib.mb200_thumbnail_image_dev(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns,
                                            rows, int(filter), _stream(image)))
    else:
        check(lib.mb200_thumbnail_image(image._ptr(), image.columns, image.rows, image.channels, out._ptr(), columns,
                                        rows, int(filter)))
    return out


class ColorspaceOptions(C.Structure):
    """mb200_colorspace_options: the image settings sRGBTransformImage / TransformsRGBImage read (MagickCore/colorspace.c:761,
    :996, :1085-1095) as values."""
    _fields_ = [("set", C.c_uint), ("illuminant", C.c_int), ("white_luminance", C.c_double), ("film_gamma", C.c_double),
                ("reference_black", C.c_double), ("reference_white", C.c_double)]


_ILLUMINANTS = {"a": 0, "b": 1, "c": 2, "d50": 3, "d55": 4, "d65": 5, "d75": 6, "e": 7, "f2": 8, "f7": 9, "f11": 10}


def colorspace_options_from_settings(settings) -> "ColorspaceOptions | None":
    """What the shim does in C (b200_colorspace_options): the "color:illuminant" artifact and the "white-luminance",
    "film-gamma", "reference-black", "reference-white" properties.  An unparsable illuminant selects D65 like the
    reference's UndefinedIlluminant (MagickCore/color.h:42)."""
    if not settings:
        return None
    o = ColorspaceOptions()
    if "color:illuminant" in settings:
        o.illuminant, o.set = _ILLUMINANTS.get(str(settings["color:illuminant"]).strip().lower(), 5), o.set | 1
    for key, field, bit in (("white-luminance", "white_luminance", 2), ("film-gamma", "film_gamma", 4),
                            ("reference-black", "reference_black", 8), ("reference-white", "reference_white", 16)):
        if key in settings:
            setattr(o, field, float(settings[key]))
            o.set |= bit
    return o if o.set else None


def TransformImageColorspace(image: Image, colorspace: int, settings=None) -> bool:
    """MagickCore/colorspace.c:1751 -- in place; updates image.colorspace.  `settings`: the image's artifacts / properties
    the transform reads, e.g. {"color:illuminant": "D50"} or {"reference-white": "700"}."""
    lib = _lib.load()
    if image.colorspace == colorspace:
        return True
    opts = colorspace_options_from_settings(settings)
    ref = C.byref(opts) if opts is not None else None
    if image.colorspace in _LAYOUT_SPACES or colorspace in _LAYOUT_SPACES:
        _transform_colorspace_layout(image, colorspace, ref)
        return True
    if image.on_device:
        _activate(image)
        check(lib.mb200_transform_colorspace_ex_dev(image._ptr(), image.columns, image.rows, image.channels,
                                                    image.colorspace, colorspace, ref, _stream(image)))
    else:
        check(lib.mb200_transform_colorspace_ex(image._ptr(), image.columns, image.rows, image.channels,
                                                image.colorspace, colorspace, ref))
    image.colorspace = colorspace
    return True


def _transform_colorspace_layout(image: Image, colorspace: int, options_ref) -> None:
    """GRAY, LinearGRAY or CMYK on either side: the pixel cache is replaced by one in the target's channel layout (gray
    [+ alpha], C M Y K [+ alpha], or three channels [+ alpha]), on the device or on the host like the source."""
    lib = _lib.load()
    alpha = image.channels - lib.mb200_colorspace_channels(image.colorspace, 0)
    out_ch = lib.mb200_colorspace_channels(colorspace, 1 if alpha == 1 else 0)
    shape = (image.rows, image.columns, out_ch)
    if image.on_device:
        import torch
        out = torch.empty(shape, dtype=torch.float32, device=image.pixels.device)
        _activate(image)
        check(lib.mb200_transform_colorspace_layout_dev(image._ptr(), image.channels, out.data_ptr(), out_ch, image.columns,
                                                        image.rows, image.colorspace, colorspace, options_ref,
                                                        _stream(image)))
    else:
        out = np.empty(shape, dtype=np.float32)
        check(lib.mb200_transform_colorspace_layout(image._ptr(), image.channels, out.ctypes.data, out_ch, image.columns,
                                                    image.rows, image.colorspace, colorspace, options_ref))
    image.pixels = out
    image.colorspace = colorspace


def _in_place(image: Image, dev_fn: str, host_fn: str, *args) -> bool:
    lib = _lib.load()
    if image.on_device:
        _activate(image)
        check(getattr(lib, dev_fn)(image._ptr(), image.columns, image.rows, image.channels, *args, _stream(image)))
    else:
        check(getattr(lib, host_fn)(image._ptr(), image.columns, image.rows, image.channels, *args))
    return True


def BilevelImage(image: Image, threshold: float) -> bool:
    """MagickCore/threshold.c:805 -- in place; a non-gray image is re-tagged sRGB (:827)."""
    ok = _in_place(image, "mb200_bilevel_image_dev", "mb200_bilevel_image", float(threshold))
    if image.channels >= 3:
        image.colorspace = sRGBColorspace
    return ok


def BlackThresholdImage(image: Image, thresholds: str) -> bool:
    """MagickCore/threshold.c:927 -- in place."""
    return _in_place(image, "mb200_black_threshold_image_dev", "mb200_black_threshold_image", int(image.colorspace),
                     thresholds.encode())


def WhiteThresholdImage(image: Image, thresholds: str) -> bool:
    """MagickCore/threshold.c:2518 -- in place."""
    return _in_place(image, "mb200_white_threshold_image_dev", "mb200_white_threshold_image", int(image.colorspace),
                     thresholds.encode())


def ClampImage(image: Image) -> bool:
    """MagickCore/threshold.c:1087 -- in place."""
    return _in_place(image, "mb200_clamp_image_dev", "mb200_clamp_image")


def _update_mask(image: Image, channels: Optional[int]) -> int:
    """The Update channels (bit c = channel c) of a `channels` selection; None = all, alpha included."""
    return (1 << image.channels) - 1 if channels is None else int(channels) & ((1 << image.channels) - 1)


def AdaptiveThresholdImage(image: Image, width: int, height: int, bias: float, channels: Optional[int] = None) -> Image:
    """MagickCore/threshold.c:182 -- a new image: every Update channel := centre <= mean of the width x height window
    + bias ? 0 : QuantumRange (`bias` in quantum units); the other channels of a `channels` selection are copied."""
    return _same_size_op(image, "mb200_adaptive_threshold_image_dev", "mb200_adaptive_threshold_image", int(width),
                         int(height), float(bias), _update_mask(image, channels))


def AutoThresholdImage(image: Image, method: int) -> float:
    """MagickCore/threshold.c:660 -- in place; returns the threshold in percent (the "auto-threshold:threshold" property
    is its "%g%%")."""
    _check_intensity(image, "AutoThresholdImage")
    threshold = C.c_double(0.0)
    _in_place(image, "mb200_auto_threshold_image_dev", "mb200_auto_threshold_image", int(method), C.byref(threshold))
    return float(threshold.value)


def RangeThresholdImage(image: Image, low_black: float, low_white: float, high_white: float, high_black: float,
                        channels: Optional[int] = None) -> bool:
    """MagickCore/threshold.c:2377 -- in place; a gray image is first transformed to sRGB, as the reference does.
    Without `channels` every channel is thresholded on the pixel's intensity, with them each selected channel on its
    own sample."""
    if image.channels <= 2 or image.colorspace in (GRAYColorspace, LinearGRAYColorspace):
        if image.colorspace not in (GRAYColorspace, LinearGRAYColorspace):
            image.colorspace = GRAYColorspace              # a gray (+ alpha) pixel cache
        TransformImageColorspace(image, sRGBColorspace)
    _check_intensity(image, "RangeThresholdImage")
    return _in_place(image, "mb200_range_threshold_image_dev", "mb200_range_threshold_image", float(low_black),
                     float(low_white), float(high_white), float(high_black), 0 if channels is None else 1,
                     _update_mask(image, channels))


def PerceptibleImage(image: Image, epsilon: float, channels: Optional[int] = None) -> bool:
    """MagickCore/threshold.c:2092 -- in place: samples of the Update channels closer to 0 than epsilon become
    +-epsilon."""
    return _in_place(image, "mb200_perceptible_image_dev", "mb200_perceptible_image", float(epsilon),
                     _update_mask(image, channels))


def ContrastImage(image: Image, sharpen: bool) -> bool:
    """MagickCore/enhance.c:1370 -- in place; alpha untouched."""
    return _in_place(image, "mb200_contrast_image_dev", "mb200_contrast_image", 1 if sharpen else 0)


# ParseCommandOption(MagickColorspaceOptions, ...) for the spaces ModulateImage distinguishes (enhance.c:3837-3887)
_MODULATE_SPACES = {"hcl": HCLColorspace, "hclp": HCLpColorspace, "hsb": HSBColorspace, "hsi": HSIColorspace,
                    "hsl": HSLColorspace, "hsv": HSVColorspace, "hwb": HWBColorspace, "lch": LCHColorspace,
                    "lchab": LCHabColorspace, "lchuv": LCHuvColorspace}
# IssRGBCompatibleColorspace (colorspace-private.h:1763): sRGB, RGB, scRGB, Transparent, GRAY, LinearGRAY and the wide-gamut RGBs
_SRGB_COMPATIBLE = {sRGBColorspace, RGBColorspace, 22, 24, GRAYColorspace, LinearGRAYColorspace, Adobe98Colorspace,
                    ProPhotoColorspace, DisplayP3Colorspace}


def _modulate_percentages(modulate: str):
    """The "B[,S[,H]]" geometry of -modulate (ParseGeometry's rho / sigma / xi): 1-3 numbers; the first separator may be
    'x' (rho x sigma), the second is ','."""
    parts = str(modulate).strip().split(",")
    parts = parts[0].split("x", 1) + parts[1:]
    try:
        values = [float(p) for p in parts]
    except ValueError:
        values = []
    if not 1 <= len(values) <= 3:
        raise MagickB200Error(_lib.EINVAL, f"modulate: '{modulate}' is not of the form B[,S[,H]]")
    return (values + [100.0, 100.0])[:3]


def ModulateImage(image: Image, modulate: str, artifacts=None) -> bool:
    """MagickCore/enhance.c:3461 -- in place.  `artifacts`: the image's "modulate:colorspace" (HSL unless one of HCL, HCLp,
    HSB, HSI, HSL, HSV, HWB, LCH, LCHab, LCHuv) and "color:illuminant" (for the LCH spaces; an unparsable one selects HSL,
    :3694-3709).  An image whose colourspace is not sRGB-compatible is re-tagged sRGB first, its pixels unchanged (:3681)."""
    brightness, saturation, hue = _modulate_percentages(modulate)
    artifacts = artifacts or {}
    space = _MODULATE_SPACES.get(str(artifacts.get("modulate:colorspace", "")).strip().lower(), HSLColorspace)
    illuminant = 5
    if "color:illuminant" in artifacts:
        name = str(artifacts["color:illuminant"]).strip().lower()
        illuminant = 5 if name == "undefined" else _ILLUMINANTS.get(name, -1)
        if illuminant < 0:
            illuminant, space = 5, HSLColorspace
    if image.colorspace not in _SRGB_COMPATIBLE:
        image.colorspace = sRGBColorspace
    return _in_place(image, "mb200_modulate_image_dev", "mb200_modulate_image", brightness, saturation, hue, space,
                     illuminant)


def GrayscaleImage(image: Image, method: int) -> bool:
    """MagickCore/enhance.c:2474 -- in place.  The pixel cache is re-laid out to the gray channel (plus alpha) and the
    image re-tagged GRAY, or LinearGRAY for the Luminance methods, as the reference's hook branch does (:2503-2511)."""
    _in_place(image, "mb200_grayscale_image_dev", "mb200_grayscale_image", int(method), int(image.colorspace))
    keep = [0, image.channels - 1] if image.channels in (2, 4) else [0]
    if image.channels > len(keep):
        pixels = image.pixels[:, :, keep]
        image.pixels = pixels.contiguous() if image.on_device else np.ascontiguousarray(pixels)
    luminance = method in (Rec601LuminancePixelIntensityMethod, Rec709LuminancePixelIntensityMethod)
    image.colorspace = LinearGRAYColorspace if luminance else GRAYColorspace
    return True


def FunctionImage(image: Image, function: int, parameters, channels: Optional[int] = None) -> bool:
    """MagickCore/statistic.c:1064 -- in place on the channels with the Update trait: all of them, alpha included, unless
    `channels` (bit c = channel c, a `-channel` selection) says otherwise.  At most 32 parameters."""
    params = [float(p) for p in parameters]
    arr = (C.c_double * max(1, len(params)))(*params)
    mask = (1 << image.channels) - 1 if channels is None else int(channels)
    return _in_place(image, "mb200_function_image_dev", "mb200_function_image", int(function), len(params), arr, mask)


# ---- level and stretch operators (enhance.c) ------------------------------------------------------------------------
# `channels` is a `-channel` selection (bit c = channel c has the Update trait); a selection that is given means the
# image's channel mask is not AllChannels, which switches the histogram operators to per-channel histograms and
# MinMaxStretch to its per-channel loop even when every channel is selected.
# colorspace-private.h IssRGBCompatibleColorspace (scRGB 22, Transparent 24)
_SRGB_COMPATIBLE = (sRGBColorspace, RGBColorspace, DisplayP3Colorspace, Adobe98Colorspace, ProPhotoColorspace, 22, 24,
                    GRAYColorspace, LinearGRAYColorspace)
_LINEAR_INTENSITY = (RGBColorspace, LinearGRAYColorspace)     # GetPixelIntensity's Rec709Luma encodes their gamma


def _level_mask(image: Image, channels: Optional[int]):
    """(update_mask, per_channel) of a `channels` selection."""
    if channels is None:
        return (1 << image.channels) - 1, 0
    return int(channels) & ((1 << image.channels) - 1), 1


def _check_intensity(image: Image, what: str) -> None:
    if image.channels > 1 and image.colorspace in _LINEAR_INTENSITY:
        raise MagickB200Error(_lib.EUNSUPPORTED, f"{what}: the intensity histogram of a linear image is not implemented")


def IdentifyImageGray(image: Image) -> int:
    """The pixel scan of MagickCore/attribute.c:1564 (IsPixelGray / IsPixelMonochrome): 0 not gray, 1 grayscale,
    2 bilevel.  A colourspace that is not sRGB-compatible is never gray."""
    if image.colorspace not in _SRGB_COMPATIBLE:
        return 0
    kind = C.c_int(0)
    lib = _lib.load()
    if image.on_device:
        _activate(image)
        check(lib.mb200_identify_gray_dev(image._ptr(), image.columns, image.rows, image.channels, C.byref(kind),
                                          _stream(image)))
    else:
        check(lib.mb200_identify_gray(image._ptr(), image.columns, image.rows, image.channels, C.byref(kind)))
    return int(kind.value)


def _intensity(v, channels: int) -> float:
    """GetPixelIntensity (pixel.c:2356, Rec709Luma without a gamma step) of a 4-entry array of channel values."""
    red = float(v[0])
    if channels == 1:
        return red
    green, blue = (float(v[1]), float(v[2])) if channels >= 3 else (red, red)
    return 0.212656 * red + 0.715158 * green + 0.072186 * blue


def ContrastStretchImage(image: Image, black_point: float, white_point: float, channels: Optional[int] = None) -> str:
    """MagickCore/enhance.c:1544 -- in place; returns the "histogram:contrast-stretch" property.  A gray-valued image
    (IdentifyImageType, enhance.c:1589-1591) is first re-laid out to the gray channel (plus alpha) and tagged GRAY, as
    GrayscaleImage's re-layout does."""
    update_mask, per_channel = _level_mask(image, channels)
    if IdentifyImageGray(image):
        if image.channels >= 3:
            keep = [0, image.channels - 1] if image.channels == 4 else [0]
            pixels = image.pixels[:, :, keep]
            image.pixels = pixels.contiguous() if image.on_device else np.ascontiguousarray(pixels)
            # the selection follows the channels: gray keeps red's bit, alpha its own
            update_mask = (update_mask & 1) | (2 if len(keep) == 2 and update_mask & 8 else 0)
        image.colorspace = GRAYColorspace
    if not per_channel:
        _check_intensity(image, "contrast stretch")
    black, white = (C.c_float * 4)(), (C.c_float * 4)()
    _in_place(image, "mb200_contrast_stretch_image_dev", "mb200_contrast_stretch_image", float(black_point),
              float(white_point), per_channel, update_mask, black, white)
    quantum_scale = 1.0 / 65535.0
    return "%gx%g%%" % (100.0 * quantum_scale * _intensity(black, image.channels),
                        100.0 * quantum_scale * _intensity(white, image.channels))


def NormalizeImage(image: Image, channels: Optional[int] = None) -> str:
    """MagickCore/enhance.c:4130 -- ContrastStretchImage(0.02 N, 0.99 N) for N pixels."""
    n = image.columns * image.rows
    return ContrastStretchImage(image, 0.02 * n, 0.99 * n, channels)


def LinearStretchImage(image: Image, black_point: float, white_point: float, channels: Optional[int] = None) -> str:
    """MagickCore/enhance.c:3347 -- in place (one intensity histogram, then LevelImage on the selected channels); returns
    the "histogram:linear-stretch" property."""
    update_mask, _ = _level_mask(image, channels)
    _check_intensity(image, "linear stretch")
    black, white = C.c_double(0.0), C.c_double(0.0)
    _in_place(image, "mb200_linear_stretch_image_dev", "mb200_linear_stretch_image", float(black_point),
              float(white_point), update_mask, C.byref(black), C.byref(white))
    return "%gx%g%%" % (100.0 * black.value / 65535, 100.0 * white.value / 65535)


def LevelImage(image: Image, black_point: float, white_point: float, gamma: float,
               channels: Optional[int] = None) -> bool:
    """MagickCore/enhance.c:2913 -- in place, with its closing ClampImage."""
    update_mask, _ = _level_mask(image, channels)
    return _in_place(image, "mb200_level_image_dev", "mb200_level_image", float(black_point), float(white_point),
                     float(gamma), update_mask)


def LevelizeImage(image: Image, black_point: float, white_point: float, gamma: float,
                  channels: Optional[int] = None) -> bool:
    """MagickCore/enhance.c:3062 -- in place, no clamp."""
    update_mask, _ = _level_mask(image, channels)
    return _in_place(image, "mb200_levelize_image_dev", "mb200_levelize_image", float(black_point), float(white_point),
                     float(gamma), update_mask)


def MinMaxStretchImage(image: Image, black: float, white: float, gamma: float, channels: Optional[int] = None) -> bool:
    """MagickCore/histogram.c:927 -- GetImageRange, then LevelImage(min + black, max - white, gamma); with a `channels`
    selection the selected colour channels one at a time.  A CMYK image with a selection is declined: the reference's
    per-channel loop levels K too, and the library's loop takes the gray / RGB layout."""
    update_mask, per_channel = _level_mask(image, channels)
    if per_channel and image.colorspace == CMYKColorspace:
        raise MagickB200Error(_lib.EUNSUPPORTED, "minmax stretch: a per-channel CMYK image is not implemented")
    return _in_place(image, "mb200_minmax_stretch_image_dev", "mb200_minmax_stretch_image", float(black), float(white),
                     float(gamma), per_channel, update_mask)


def AutoLevelImage(image: Image, channels: Optional[int] = None) -> bool:
    """MagickCore/enhance.c:187 -- MinMaxStretchImage(0, 0, 1)."""
    return MinMaxStretchImage(image, 0.0, 0.0, 1.0, channels)


def GammaImage(image: Image, gamma: float, channels: Optional[int] = None) -> bool:
    """MagickCore/enhance.c:2322 -- in place through the reference's 65 536-entry table; nothing for gamma 1.  (The
    reference also multiplies image->gamma; an Image here carries no gamma attribute.)"""
    update_mask, _ = _level_mask(image, channels)
    return _in_place(image, "mb200_gamma_image_dev", "mb200_gamma_image", float(gamma), update_mask)


def MorphologyPrimitive(image: Image, method: int, kernel: Union[str, KernelInfo], bias: float = 0.0):
    """One MorphologyPrimitive pass (MagickCore/morphology.c:2566): returns (Image, changed).
    Device-resident images only (the primitive has no host-buffer entry point)."""
    if not image.on_device:
        raise ValueError("MorphologyPrimitive needs a device-resident Image")
    k = _as_kernel(kernel)
    out = image._new_like()
    changed = C.c_longlong(0)
    _activate(image)
    check(_lib.load().mb200_morphology_primitive_dev(image._ptr(), out._ptr(), image.columns, image.rows,
                                                     image.channels, int(method), k._ptr, float(bias),
                                                     C.byref(changed), _stream(image)))
    return out, int(changed.value)


def launch_count() -> int:
    return int(_lib.load().mb200_launch_count())


def device_count() -> int:
    return int(_lib.load().mb200_device_count())
