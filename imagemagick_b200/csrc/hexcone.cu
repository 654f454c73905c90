// hexcone.cu -- the hue / saturation colourspaces of TransformImageColorspace's generic branch:
// HCL, HCLp, HSB, HSI, HSL, HSV, HWB (MagickCore/colorspace.c:958-1054 forward, :2296-2390 inverse; the per-pixel
// formulae are ConvertRGBTo* / Convert*ToRGB of colorspace-private.h:149-529, :801-1064 and colorspace.c:307, :597).
//
// These transforms are piecewise: which branch a pixel takes depends on comparisons of differences against
// MagickEpsilon and on floor() of a scaled hue, and the branches do not meet continuously (hue jumps by a sector, a
// gray pixel's hue is a constant).  A result that is merely "close in double" can therefore be a different colour, so
// every operation here is the reference's own IEEE double operation, in its order, unfused (__dmul_rn / __dadd_rn /
// __ddiv_rn; nvcc would otherwise contract a*b+c) => bit exact, except HSI whose atan2 / cos come from the CUDA math
// library instead of glibc (<= 1 ULP of the float Quantum, measured 0).
//
// Structure: one thread per pixel, float4 access for RGBA, alpha untouched.  The six-sector fan-out of every inverse
// transform is one permutation table (kSector) applied to the three values the sector formulae produce.
#include "hexcone.cuh"
#include "launch.cuh"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

template <int CH>
__global__ void __launch_bounds__(256) hexcone_kernel(float *buf, size_t npixels, int space, int forward) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float in0, in1, in2, in3 = 0.f;
  if (CH == 4) { const float4 t = *reinterpret_cast<const float4 *>(q); in0 = t.x; in1 = t.y; in2 = t.z; in3 = t.w; }
  else { in0 = q[0]; in1 = q[1]; in2 = q[2]; }
  Triple o;
  if (forward) {                                   // colorspace.c:1038-1043: (float) (QuantumRange * X)
    const double r = in0, g = in1, b = in2;
    switch (space) {
      case kHCL: case kHCLp: o = to_hcl(r, g, b); break;
      case kHSB: o = to_hsb(r, g, b); break;
      case kHSI: o = to_hsi(r, g, b); break;
      case kHSL: o = to_hsl_hsv<false>(r, g, b); break;
      case kHSV: o = to_hsl_hsv<true>(r, g, b); break;
      default: o = to_hwb(r, g, b); break;
    }
    o.x = ml(QR, o.x); o.y = ml(QR, o.y); o.z = ml(QR, o.z);
  } else {                                         // :2373-2379: components arrive as QuantumScale * sample
    const double a = ml(QS, static_cast<double>(in0)), b = ml(QS, static_cast<double>(in1)), c = ml(QS, static_cast<double>(in2));
    switch (space) {
      case kHCL: o = from_hcl<false>(a, b, c); break;
      case kHCLp: o = from_hcl<true>(a, b, c); break;
      case kHSB: o = from_hsb(a, b, c); break;
      case kHSI: o = from_hsi(a, b, c); break;
      case kHSL: o = from_hsl_hsv<false>(a, b, c); break;
      case kHSV: o = from_hsl_hsv<true>(a, b, c); break;
      default: o = from_hwb(a, b, c); break;
    }
  }
  const float o0 = static_cast<float>(o.x), o1 = static_cast<float>(o.y), o2 = static_cast<float>(o.z);
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o0, o1, o2, in3);
  else { q[0] = o0; q[1] = o1; q[2] = o2; }
}

}  // namespace

bool is_hexcone_colorspace(int cs) {
  return cs == kHCL || cs == kHCLp || cs == kHSB || cs == kHSI || cs == kHSL || cs == kHSV || cs == kHWB;
}

int launch_hexcone_leg(float *buf, size_t npixels, int channels, int space, bool forward, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  if (channels == 4) hexcone_kernel<4><<<blocks, 256, 0, s>>>(buf, npixels, space, forward ? 1 : 0);
  else hexcone_kernel<3><<<blocks, 256, 0, s>>>(buf, npixels, space, forward ? 1 : 0);
  return launch_status("hexcone launch");
}

}  // namespace mb200
