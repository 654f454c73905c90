// resize_filter.cpp -- host side of the resize path: the reference's filter table
// and the per-output contribution (start / count / normalised weights) lists.
//
// Behavioural mirror of MagickCore/resize.c: AcquireResizeFilter :803 (mapping table
// :835-876, function table :888-942, sharpening :1064, cubic coefficients :1181-1226),
// GetResizeFilterWeight :1690, GetResizeFilterSupport :1656, and the contribution
// set-up that opens every iteration of HorizontalFilter (:3398-3443) and
// VerticalFilter (:3614-3657).  Orthogonal for ResizeImage (MagickFalse, :3817);
// cylindrical (:995-997, :1033, :1049-1069) for the EWA weight table of
// SetResampleFilter (resample.c:1246-1300), which DistortImage samples through.
//
// Weights are evaluated on the host in double with the same operation order as the
// reference, so the table uploaded to the GPU is bit-identical to what the CPU path
// uses; the device only does the weighted sums.
#include "mb200_internal.h"

#include <cmath>
#include <utility>
#include <vector>

namespace {

constexpr double kEps = 1.0e-12;
constexpr double kPi = 3.1415926535897932384626433832795028841971693993751058209749445923078164062;
constexpr double kPi2 = 1.57079632679489661923132169163975144209858469968755;
constexpr double k2Pi = 6.28318530717958647692528676655900576839433879875020;

inline double perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= kEps ? 1.0 / x : sign / kEps;
}

enum class Fn { Box, Triangle, CubicBC, Hann, Hamming, Blackman, Gaussian, Quadratic, Sinc, SincFast,
                Welch, Bohman, Lagrange, Cosine, CubicSpline, Mks2013, Mks2021, Jinc, Kaiser, Unsupported };

struct FnEntry { Fn fn; double support, scale, B, C; };

// resize.c:888-942, indexed by FilterType
const FnEntry kFunctions[MB200_SentinelFilter] = {
  {Fn::Box, 0.5, 0.5, 0, 0},            // Undefined
  {Fn::Box, 0.0, 0.5, 0, 0},            // Point
  {Fn::Box, 0.5, 0.5, 0, 0},            // Box
  {Fn::Triangle, 1.0, 1.0, 0, 0},       // Triangle
  {Fn::CubicBC, 1.0, 1.0, 0, 0},        // Hermite
  {Fn::Hann, 1.0, 1.0, 0, 0},
  {Fn::Hamming, 1.0, 1.0, 0, 0},
  {Fn::Blackman, 1.0, 1.0, 0, 0},
  {Fn::Gaussian, 2.0, 1.5, 0, 0},
  {Fn::Quadratic, 1.5, 1.5, 0, 0},
  {Fn::CubicBC, 2.0, 2.0, 1.0, 0.0},    // Cubic
  {Fn::CubicBC, 2.0, 1.0, 0.0, 0.5},    // Catrom
  {Fn::CubicBC, 2.0, 8.0 / 7.0, 1. / 3., 1. / 3.},   // Mitchell
  {Fn::Jinc, 3.0, 1.2196698912665045, 0, 0},         // Jinc: 3 lobes, converted to the third zero below
  {Fn::Sinc, 4.0, 1.0, 0, 0},
  {Fn::SincFast, 4.0, 1.0, 0, 0},
  {Fn::Kaiser, 1.0, 1.0, 0, 0},         // Kaiser window (I0)
  {Fn::Welch, 1.0, 1.0, 0, 0},
  {Fn::CubicBC, 2.0, 2.0, 1.0, 0.0},    // Parzen
  {Fn::Bohman, 1.0, 1.0, 0, 0},
  {Fn::Triangle, 1.0, 1.0, 0, 0},       // Bartlett
  {Fn::Lagrange, 2.0, 1.0, 0, 0},
  {Fn::SincFast, 3.0, 1.0, 0, 0},       // Lanczos
  {Fn::SincFast, 3.0, 1.0, 0, 0},       // LanczosSharp
  {Fn::SincFast, 2.0, 1.0, 0, 0},       // Lanczos2
  {Fn::SincFast, 2.0, 1.0, 0, 0},       // Lanczos2Sharp
  {Fn::CubicBC, 2.0, 1.1685777620836932, 0.37821575509399867, 0.31089212245300067},  // Robidoux
  {Fn::CubicBC, 2.0, 1.105822933719019, 0.2620145123990142, 0.3689927438004929},     // RobidouxSharp
  {Fn::Cosine, 1.0, 1.0, 0, 0},
  {Fn::CubicBC, 2.0, 2.0, 1.0, 0.0},    // Spline
  {Fn::SincFast, 3.0, 1.0, 0, 0},       // LanczosRadius
  {Fn::CubicSpline, 2.0, 0.5, 0, 0},
  {Fn::Mks2013, 2.5, 1.0, 0, 0},
  {Fn::Mks2021, 4.5, 1.0, 0, 0},
};

// resize.c:835-876: requested filter -> {weighting function's filter, window's filter}
struct Mapping { int filter, window; };
const Mapping kMapping[MB200_SentinelFilter] = {
  {MB200_UndefinedFilter, MB200_BoxFilter}, {MB200_PointFilter, MB200_BoxFilter},
  {MB200_BoxFilter, MB200_BoxFilter}, {MB200_TriangleFilter, MB200_BoxFilter},
  {MB200_HermiteFilter, MB200_BoxFilter}, {MB200_SincFastFilter, MB200_HannFilter},
  {MB200_SincFastFilter, MB200_HammingFilter}, {MB200_SincFastFilter, MB200_BlackmanFilter},
  {MB200_GaussianFilter, MB200_BoxFilter}, {MB200_QuadraticFilter, MB200_BoxFilter},
  {MB200_CubicFilter, MB200_BoxFilter}, {MB200_CatromFilter, MB200_BoxFilter},
  {MB200_MitchellFilter, MB200_BoxFilter}, {MB200_JincFilter, MB200_BoxFilter},
  {MB200_SincFilter, MB200_BoxFilter}, {MB200_SincFastFilter, MB200_BoxFilter},
  {MB200_SincFastFilter, MB200_KaiserFilter}, {MB200_LanczosFilter, MB200_WelchFilter},
  {MB200_SincFastFilter, MB200_CubicFilter}, {MB200_SincFastFilter, MB200_BohmanFilter},
  {MB200_SincFastFilter, MB200_TriangleFilter}, {MB200_LagrangeFilter, MB200_BoxFilter},
  {MB200_LanczosFilter, MB200_LanczosFilter}, {MB200_LanczosSharpFilter, MB200_LanczosSharpFilter},
  {MB200_Lanczos2Filter, MB200_Lanczos2Filter}, {MB200_Lanczos2SharpFilter, MB200_Lanczos2SharpFilter},
  {MB200_RobidouxFilter, MB200_BoxFilter}, {MB200_RobidouxSharpFilter, MB200_BoxFilter},
  {MB200_LanczosFilter, MB200_CosineFilter}, {MB200_SplineFilter, MB200_BoxFilter},
  {MB200_LanczosRadiusFilter, MB200_LanczosFilter}, {MB200_CubicSplineFilter, MB200_BoxFilter},
  {MB200_MagicKernelSharp2013Filter, MB200_BoxFilter}, {MB200_MagicKernelSharp2021Filter, MB200_BoxFilter},
};

struct ResizeFilter {
  Fn filter = Fn::Box, window = Fn::Box;
  double support = 0, window_support = 0, scale = 1, blur = 1, coefficient[7] = {0};
  bool valid = false;

  // The expert settings take effect in the reference's order (resize.c:999-1226): window override, sharpening, Gaussian
  // sigma (widens the support), Kaiser beta, lobes, Jinc zeros, blur, support, window support, window scale, cubic B / C.
  explicit ResizeFilter(int requested, const mb200_filter_options *opt = nullptr, bool cylindrical = false) {
    if (requested <= MB200_UndefinedFilter || requested >= MB200_SentinelFilter) return;
    const unsigned set = opt ? opt->set : 0u;
    int ft = kMapping[requested].filter, wt = kMapping[requested].window;
    if (cylindrical && ft == MB200_SincFastFilter && requested != MB200_SincFastFilter)
      ft = MB200_JincFilter;                                 // 1-D windowed Sinc => 2-D windowed Jinc (:995-997)
    if ((set & MB200_FO_WINDOW) && opt->window > MB200_UndefinedFilter && opt->window < MB200_SentinelFilter) {
      // a window without a filter: windowed Sinc, or Jinc when cylindrical (:1024-1041)
      if (!opt->keep_filter) ft = cylindrical ? MB200_JincFilter : MB200_SincFastFilter;
      wt = opt->window;
    }
    filter = kFunctions[ft].fn;
    window = kFunctions[wt].fn;
    if (filter == Fn::Unsupported || window == Fn::Unsupported) return;
    support = kFunctions[ft].support;
    scale = kFunctions[wt].scale;
    if (cylindrical) {                                       // :1049-1069
      if (ft == MB200_BoxFilter) support = 0.70710678118654752440;      // MagickSQ1_2
      if (ft == MB200_LanczosFilter || ft == MB200_LanczosSharpFilter || ft == MB200_Lanczos2Filter ||
          ft == MB200_Lanczos2SharpFilter || ft == MB200_LanczosRadiusFilter) {
        filter = window = Fn::Jinc;
        scale = kFunctions[MB200_JincFilter].scale;
      }
    }
    if (ft == MB200_LanczosSharpFilter) blur *= 0.9812505644269356;
    if (ft == MB200_Lanczos2SharpFilter) blur *= 0.9549963639785485;
    if (filter == Fn::Gaussian || window == Fn::Gaussian) {
      const double sigma = (set & MB200_FO_SIGMA) ? opt->sigma : 0.5;
      coefficient[0] = sigma;
      coefficient[1] = perceptible_reciprocal(2.0 * sigma * sigma);
      coefficient[2] = perceptible_reciprocal(k2Pi * sigma * sigma);
      if (sigma > 0.5) support *= 2 * sigma;                 // :1097-1098
    }
    if (filter == Fn::Kaiser || window == Fn::Kaiser) {      // :1104-1120
      const double beta = (set & MB200_FO_KAISER_BETA) ? opt->kaiser_beta : 6.5;
      coefficient[0] = beta;
      coefficient[1] = perceptible_reciprocal(bessel_i0(beta));
    }
    if (set & MB200_FO_LOBES) support = static_cast<double>(opt->lobes < 1 ? 1 : opt->lobes);   // :1123-1133
    if (filter == Fn::Jinc) {                                // :1135-1150 lobes -> support
      support = jinc_zero(static_cast<long>(support));
      if (ft == MB200_LanczosRadiusFilter) blur *= std::floor(support) / support;
    }
    if (set & MB200_FO_BLUR) blur *= opt->blur;              // :1155-1157
    if (blur < kEps) blur = kEps;
    if (set & MB200_FO_SUPPORT) support = std::fabs(opt->support);             // :1163-1165
    window_support = (set & MB200_FO_WIN_SUPPORT) ? std::fabs(opt->win_support) : support;   // :1170-1173
    scale *= perceptible_reciprocal(window_support);
    if (filter == Fn::CubicBC || window == Fn::CubicBC) {
      double B = kFunctions[ft].B, C = kFunctions[ft].C;
      if (kFunctions[wt].fn == Fn::CubicBC) { B = kFunctions[wt].B; C = kFunctions[wt].C; }
      if (set & MB200_FO_B) {                                // :1196-1212: one of them given => a Keys cubic
        B = opt->b;
        C = (1.0 - B) / 2.0;
        if (set & MB200_FO_C) C = opt->c;
      } else if (set & MB200_FO_C) {
        C = opt->c;
        B = 1.0 - 2.0 * C;
      }
      const double twoB = B + B;
      coefficient[0] = 1.0 - (1.0 / 3.0) * B;
      coefficient[1] = -3.0 + twoB + C;
      coefficient[2] = 2.0 - 1.5 * B - C;
      coefficient[3] = (4.0 / 3.0) * B + 4.0 * C;
      coefficient[4] = -8.0 * C - twoB;
      coefficient[5] = B + 5.0 * C;
      coefficient[6] = (-1.0 / 6.0) * B - C;
    }
    valid = true;
  }

  // ---- Bessel functions of the Jinc filter and the Kaiser window (resize.c:1385-1553).  The reference evaluates them
  // with fixed rational approximations; the weights must come out bit-identical, so the coefficient tables and the
  // association of every product are the reference's: p = ((p * u) * u) + c, one table pair per range.
  template <int N>
  static double rational(const double (&num)[N], const double (&den)[N], double u) {
    double p = num[N - 1], q = den[N - 1];
    for (int i = N - 2; i >= 0; --i) {
      p = p * u * u + num[i];
      q = q * u * u + den[i];
    }
    return p / q;
  }
  static double bessel_i0(double x) {          // :1385 power series, terms down to MagickEpsilon
    const double y = x * x / 4.0;
    double sum = 1.0, term = y;
    for (long i = 2; term > kEps; ++i) {
      sum += term;
      term *= y / (static_cast<double>(i) * i);
    }
    return sum;
  }
  static double bessel_j1_signed(double x) {   // :1535 BesselOrderOne
    static const double kJ1Num[9] = {
      0.581199354001606143928050809e+21, -0.6672106568924916298020941484e+20, 0.2316433580634002297931815435e+19,
      -0.3588817569910106050743641413e+17, 0.2908795263834775409737601689e+15, -0.1322983480332126453125473247e+13,
      0.3413234182301700539091292655e+10, -0.4695753530642995859767162166e+7, 0.270112271089232341485679099e+4};
    static const double kJ1Den[9] = {
      0.11623987080032122878585294e+22, 0.1185770712190320999837113348e+20, 0.6092061398917521746105196863e+17,
      0.2081661221307607351240184229e+15, 0.5243710262167649715406728642e+12, 0.1013863514358673989967045588e+10,
      0.1501793594998585505921097578e+7, 0.1606931573481487801970916749e+4, 0.1e+1};
    static const double kP1Num[6] = {
      0.352246649133679798341724373e+5, 0.62758845247161281269005675e+5, 0.313539631109159574238669888e+5,
      0.49854832060594338434500455e+4, 0.2111529182853962382105718e+3, 0.12571716929145341558495e+1};
    static const double kP1Den[6] = {
      0.352246649133679798068390431e+5, 0.626943469593560511888833731e+5, 0.312404063819041039923015703e+5,
      0.4930396490181088979386097e+4, 0.2030775189134759322293574e+3, 0.1e+1};
    static const double kQ1Num[6] = {
      0.3511751914303552822533318e+3, 0.7210391804904475039280863e+3, 0.4259873011654442389886993e+3,
      0.831898957673850827325226e+2, 0.45681716295512267064405e+1, 0.3532840052740123642735e-1};
    static const double kQ1Den[6] = {
      0.74917374171809127714519505e+4, 0.154141773392650970499848051e+5, 0.91522317015169922705904727e+4,
      0.18111867005523513506724158e+4, 0.1038187585462133728776636e+3, 0.1e+1};
    if (x == 0.0) return 0.0;
    const double ax = x < 0.0 ? -x : x;
    if (ax < 8.0) return x * rational(kJ1Num, kJ1Den, ax);
    const double u = 8.0 / ax;
    const double q = std::sqrt(2.0 / (kPi * ax)) *
                     (rational(kP1Num, kP1Den, u) * (1.0 / std::sqrt(2.0) * (std::sin(ax) - std::cos(ax))) -
                      8.0 / ax * rational(kQ1Num, kQ1Den, u) * (-1.0 / std::sqrt(2.0) * (std::sin(ax) + std::cos(ax))));
    return x < 0.0 ? -q : q;
  }
  static double jinc_zero(long lobes) {        // :955-973 first zero crossings of the Jinc function
    static const double kZeros[16] = {
      1.2196698912665045, 2.2331305943815286, 3.2383154841662362, 4.2410628637960699, 5.2427643768701817,
      6.2439216898644877, 7.2447598687199570, 8.2453949139520427, 9.2458926849494673, 10.246293348754916,
      11.246622794877883, 12.246898461138105, 13.247132522181061, 14.247333735806849, 15.247508563037300,
      16.247661874700962};
    return lobes > 16 ? kZeros[15] : kZeros[lobes - 1];
  }

  // resize.c:493-587, Q16 coefficient set (:547-563)
  static double sinc_fast(double x) {
    if (x > 4.0) {
      const double alpha = kPi * x;
      return std::sin(alpha) / alpha;
    }
    static const double c[10] = {
      0.173611107357320220183368594093166520811e-2L, -0.384240921114946632192116762889211361285e-3L,
      0.394201182359318128221229891724947048771e-4L, -0.250963301609117217660068889165550534856e-5L,
      0.111902032818095784414237782071368805120e-6L, -0.372895101408779549368465614321137048875e-8L,
      0.957694196677572570319816780188718518330e-10L, -0.187208577776590710853865174371617338991e-11L,
      0.253524321426864752676094495396308636823e-13L, -0.177084805010701112639035485248501049364e-15L};
    const double xx = x * x;
    double p = c[9];
    for (int i = 8; i >= 0; --i) p = c[i] + xx * p;      // Horner, same association as the reference
    return (xx - 1.0) * (xx - 4.0) * (xx - 9.0) * (xx - 16.0) * p;
  }

  double eval(Fn fn, double x) const {
    switch (fn) {
      case Fn::Box: return 1.0;
      case Fn::Triangle: return x < 1.0 ? 1.0 - x : 0.0;
      case Fn::CubicBC:
        if (x < 1.0) return coefficient[0] + x * (x * (coefficient[1] + x * coefficient[2]));
        if (x < 2.0) return coefficient[3] + x * (coefficient[4] + x * (coefficient[5] + x * coefficient[6]));
        return 0.0;
      case Fn::Hann: { const double c = std::cos(kPi * x); return 0.5 + 0.5 * c; }
      case Fn::Hamming: { const double c = std::cos(kPi * x); return 0.54 + 0.46 * c; }
      case Fn::Blackman: { const double c = std::cos(kPi * x); return 0.34 + c * (0.5 + c * 0.16); }
      case Fn::Gaussian: return std::exp(-coefficient[1] * x * x);
      case Fn::Quadratic:
        if (x < 0.5) return 0.75 - x * x;
        if (x < 1.5) return 0.5 * (x - 1.5) * (x - 1.5);
        return 0.0;
      case Fn::Sinc:
        if (x != 0.0) { const double a = kPi * x; return std::sin(a) / a; }
        return 1.0;
      case Fn::SincFast: return sinc_fast(x);
      case Fn::Welch: return x < 1.0 ? 1.0 - x * x : 0.0;
      case Fn::Bohman: {
        const double c = std::cos(kPi * x);
        const double s = std::sqrt(1.0 - c * c);
        return (1.0 - x) * c + (1.0 / kPi) * s;
      }
      case Fn::Cosine: return std::cos(kPi2 * x);
      case Fn::Lagrange: {
        if (x > support) return 0.0;
        const long order = static_cast<long>(2.0 * window_support);
        const long n = static_cast<long>(window_support + x);
        double value = 1.0f;
        for (long i = 0; i < order; ++i)
          if (i != n) value *= (n - i - x) / (n - i);
        return value;
      }
      case Fn::CubicSpline:   // 2-lobe form; support is never overridden here
        if (x < 1.0) return ((x - 9.0 / 5.0) * x - 1.0 / 5.0) * x + 1.0;
        if (x < 2.0) return ((-1.0 / 3.0 * (x - 1.0) + 4.0 / 5.0) * (x - 1.0) - 7.0 / 15.0) * (x - 1.0);
        return 0.0;
      case Fn::Jinc: return x == 0.0 ? 0.5 * kPi : bessel_j1_signed(kPi * x) / x;                    // :348
      case Fn::Kaiser: return coefficient[1] * bessel_i0(coefficient[0] * std::sqrt(1.0 - x * x));    // :366
      case Fn::Mks2013:
        if (x < 0.5) return 0.625 + 1.75 * (0.5 - x) * (0.5 + x);
        if (x < 1.5) return (1.0 - x) * (1.75 - x);
        if (x < 2.5) return -0.125 * (2.5 - x) * (2.5 - x);
        return 0.0;
      case Fn::Mks2021:
        if (x < 0.5) return 577.0 / 576.0 - 239.0 / 144.0 * x * x;
        if (x < 1.5) return 35.0 / 36.0 * (x - 1.0) * (x - 239.0 / 140.0);
        if (x < 2.5) return 1.0 / 6.0 * (x - 2.0) * (65.0 / 24.0 - x);
        if (x < 3.5) return 1.0 / 36.0 * (x - 3.0) * (x - 3.75);
        if (x < 4.5) return -1.0 / 288.0 * (x - 4.5) * (x - 4.5);
        return 0.0;
      default: return 0.0;
    }
  }

  double weight(double x) const {           // resize.c:1690
    const double x_blur = std::fabs(x) * perceptible_reciprocal(blur);
    double s;
    if (window_support < kEps || window == Fn::Box) s = 1.0;
    else s = eval(window, x_blur * scale);
    return s * eval(filter, x_blur);
  }
  double practical_support() const { return support * blur; }   // resize.c:1656
};

}  // namespace

extern "C" {

double mb200_resize_filter_weight_ex(int filter, const mb200_filter_options *options, double x) {
  ResizeFilter rf(filter, options);
  if (!rf.valid) return std::nan("");
  return rf.weight(x);
}
double mb200_resize_filter_weight(int filter, double x) { return mb200_resize_filter_weight_ex(filter, nullptr, x); }

double mb200_resize_filter_support_ex(int filter, const mb200_filter_options *options) {
  ResizeFilter rf(filter, options);
  if (!rf.valid) return std::nan("");
  return rf.practical_support();
}
double mb200_resize_filter_support(int filter) { return mb200_resize_filter_support_ex(filter, nullptr); }

// SetResampleFilter (resample.c:1246-1300): the cylindrical filter of the image's FilterType (Undefined is Robidoux,
// :1261) sampled at sqrt(Q) * support / sqrt(1024) for the Q = 0..1023 of the EWA's squared-radius index.
int mb200_resample_filter_lut(int filter, const mb200_filter_options *options, double *lut, double *support) {
  if (filter == MB200_UndefinedFilter) filter = MB200_RobidouxFilter;
  if (filter == MB200_PointFilter)
    return mb200::fail(MB200_EUNSUPPORTED, "the Point filter interpolates every pixel instead of sampling an ellipse");
  ResizeFilter rf(filter, options, true);
  if (!rf.valid) return mb200::fail(MB200_EINVAL, "resample filter %d is not a FilterType", filter);
  if (!lut || !support) return mb200::fail(MB200_EINVAL, "resample filter: no output");
  *support = rf.practical_support();
  const double r_scale = *support * std::sqrt(1.0 / static_cast<double>(MB200_RESAMPLE_LUT));
  for (int q = 0; q < MB200_RESAMPLE_LUT; ++q) lut[q] = rf.weight(std::sqrt(static_cast<double>(q)) * r_scale);
  return MB200_OK;
}

long mb200_resize_contributions(int filter, size_t in_n, size_t out_n, double factor, long *start,
                                int *count, double *weights, size_t max_taps) {
  return mb200_resize_contributions_ex(filter, nullptr, in_n, out_n, factor, start, count, weights, max_taps);
}

long mb200_resize_contributions_ex(int filter, const mb200_filter_options *options, size_t in_n, size_t out_n, double factor,
                                   long *start, int *count, double *weights, size_t max_taps) {
  ResizeFilter rf(filter, options);
  if (!rf.valid) return mb200::fail(MB200_EUNSUPPORTED, "resize filter %d is not supported on the 1-D GPU path", filter);
  if (in_n == 0 || out_n == 0 || !(factor > 0.0)) return mb200::fail(MB200_EINVAL, "bad resize geometry");
  // resize.c:3363-3386 / :3578-3601
  double scale = std::fmax(1.0 / factor + kEps, 1.0);
  double support = scale * rf.practical_support();
  if (support < 0.5) { support = 0.5; scale = 1.0; }
  const long need = static_cast<long>(2.0 * support + 3.0);
  if (!start || !count || !weights) return need;
  if (static_cast<long>(max_taps) < need) return mb200::fail(MB200_EINVAL, "max_taps %zu < %ld", max_taps, need);
  scale = perceptible_reciprocal(scale);
  for (size_t o = 0; o < out_n; ++o) {
    const double bisect = static_cast<double>(o + 0.5) / factor + kEps;
    const long first = static_cast<long>(std::fmax(bisect - support + 0.5, 0.0));
    const long last = static_cast<long>(std::fmin(bisect + support + 0.5, static_cast<double>(in_n)));
    const long n = last - first > 0 ? last - first : 0;
    double *w = weights + o * max_taps;
    double density = 0.0;
    for (long j = 0; j < n; ++j) {
      w[j] = rf.weight(scale * (static_cast<double>(first + j) - bisect + 0.5));
      density += w[j];
    }
    if (n > 0 && density != 0.0 && density != 1.0) {
      density = perceptible_reciprocal(density);
      for (long j = 0; j < n; ++j) w[j] *= density;
    }
    for (size_t j = static_cast<size_t>(n); j < max_taps; ++j) w[j] = 0.0;
    start[o] = first;
    count[o] = static_cast<int>(n);
  }
  return need;
}

// ScaleImage (resize.c:4106-4530) is a sequential state machine whose weights do not depend on the pixels: the running
// (span, scale) pairs are simulated here in the reference's own order and arithmetic, and recorded per output as a list of
// (source index, weight) terms in accumulation order.  axis 1 = rows (the y machine pulls source rows per output row,
// :4229-4330), axis 0 = columns (the x machine pushes every source column into the outputs it overlaps, :4378-4440).
// offsets has out_n + 1 entries; index / weight hold offsets[out_n] terms (query the count with index == NULL).
long mb200_scale_contributions(int axis, size_t in_n, size_t out_n, long *offsets, int *index, double *weight, size_t max_terms) {
  if (in_n == 0 || out_n == 0 || !offsets) return mb200::fail(MB200_EINVAL, "bad scale geometry");
  std::vector<std::vector<std::pair<int, double>>> lists(out_n);
  const double factor = static_cast<double>(out_n) / static_cast<double>(in_n);
  if (in_n == out_n) {
    for (size_t o = 0; o < out_n; ++o) lists[o].emplace_back(static_cast<int>(o), 1.0);      // taken as is (:4190, :4336)
  } else if (axis == 1) {
    long number_rows = 0, next = 0;
    int cur = 0;
    bool next_row = true;
    double span = 1.0, scale = factor;
    for (size_t y = 0; y < out_n; ++y) {
      while (scale < span) {
        if (next_row && number_rows < static_cast<long>(in_n)) { cur = static_cast<int>(next++); ++number_rows; }
        lists[y].emplace_back(cur, scale);                       // y_vector += scale.y * x_vector
        span -= scale;
        scale = factor;
        next_row = true;
      }
      if (next_row && number_rows < static_cast<long>(in_n)) { cur = static_cast<int>(next++); ++number_rows; next_row = false; }
      lists[y].emplace_back(cur, span);                          // pixel = y_vector + span.y * x_vector
      scale -= span;
      if (scale <= 0) { scale = factor; next_row = true; }
      span = 1.0;
    }
  } else {
    long t = 0;
    bool next_column = false;
    double span = 1.0;
    auto add = [&](long out, size_t x, double w) { if (out >= 0 && out < static_cast<long>(out_n)) lists[static_cast<size_t>(out)].emplace_back(static_cast<int>(x), w); };
    for (size_t x = 0; x < in_n; ++x) {
      double scale = factor;
      while (scale >= span) {
        if (next_column) ++t;                                    // pixel = 0 for a new output
        add(t, x, span);
        scale -= span;
        span = 1.0;
        next_column = true;
      }
      if (scale > 0) {
        if (next_column) { next_column = false; ++t; }
        add(t, x, scale);
        span -= scale;
      }
    }
    if (span > 0 && !next_column) add(t, in_n - 1, span);         // :4433-4440 (only a still-open output is stored again)
  }
  long total = 0;
  for (size_t o = 0; o < out_n; ++o) { offsets[o] = total; total += static_cast<long>(lists[o].size()); }
  offsets[out_n] = total;
  if (!index || !weight) return total;
  if (static_cast<long>(max_terms) < total) return mb200::fail(MB200_EINVAL, "max_terms %zu < %ld", max_terms, total);
  long k = 0;
  for (size_t o = 0; o < out_n; ++o)
    for (const auto &term : lists[o]) { index[k] = term.first; weight[k] = term.second; ++k; }
  return total;
}

// The source sample a Copy-trait channel takes for every output of one axis (resize.c:3697-3707):
// j = (ssize_t) (min(max(bisect, start), stop - 1) + 0.5), with bisect / start / stop as in the contribution list.
int mb200_resize_nearest(int filter, size_t in_n, size_t out_n, double factor, long *nearest) {
  ResizeFilter rf(filter);
  if (!rf.valid) return mb200::fail(MB200_EUNSUPPORTED, "resize filter %d is not supported on the 1-D GPU path", filter);
  if (in_n == 0 || out_n == 0 || !(factor > 0.0) || !nearest) return mb200::fail(MB200_EINVAL, "bad resize geometry");
  double scale = std::fmax(1.0 / factor + kEps, 1.0);
  double support = scale * rf.practical_support();
  if (support < 0.5) support = 0.5;
  for (size_t o = 0; o < out_n; ++o) {
    const double bisect = static_cast<double>(o + 0.5) / factor + kEps;
    const long first = static_cast<long>(std::fmax(bisect - support + 0.5, 0.0));
    const long last = static_cast<long>(std::fmin(bisect + support + 0.5, static_cast<double>(in_n)));
    nearest[o] = static_cast<long>(std::fmin(std::fmax(bisect, static_cast<double>(first)), static_cast<double>(last) - 1.0) + 0.5);
  }
  return MB200_OK;
}

}  // extern "C"
