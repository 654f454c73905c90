// distort_plan.cpp -- host side of DistortImage / RotateImage: the reverse map and the output geometry.
//
// Behavioural mirror of MagickCore/distort.c: GenerateCoefficients (:380-960) for the six methods that reduce to an
// affine or a perspective map, with matrix.c's LeastSquaresAddTerms (:831) and GaussJordanElimination (:482) in the
// reference's order of operations; the bestfit bounds and fix_bounds rounding (:1827-1990); the viewport (:2033) and
// "distort:scale" (:2393-2410); and RotateImage's angle reduction (:2976-2988).  No device.
#include "mb200_internal.h"

#include <cmath>
#include <vector>

namespace {

constexpr double kEps = 1.0e-12;
constexpr double kPi = 3.14159265358979323846264338327950288419716939937510;

enum { kAffine = 1, kAffineProjection = 2, kSRT = 3, kPerspective = 4, kPerspectiveProjection = 5,
       kRigidAffine = 19 };   // DistortMethod: BilinearDistortion aliases BilinearForward, so RigidAffine is 19

inline double perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= kEps ? 1.0 / x : sign / kEps;
}

struct Matrix {              // AcquireMagickMatrix: rank x rank zeros, plus the right-hand sides
  size_t rank;
  std::vector<std::vector<double>> m;
  explicit Matrix(size_t r) : rank(r), m(r, std::vector<double>(r, 0.0)) {}
};

// LeastSquaresAddTerms (matrix.c:831)
void add_terms(Matrix &a, double **vectors, const double *terms, const double *results, size_t nvec) {
  for (size_t j = 0; j < a.rank; ++j) {
    for (size_t i = 0; i < a.rank; ++i) a.m[i][j] += terms[i] * terms[j];
    for (size_t i = 0; i < nvec; ++i) vectors[i][j] += results[i] * terms[j];
  }
}

inline void gj_swap(double &x, double &y) {      // GaussJordanSwap, arithmetic and all
  if (x != y) { x += y; y = x - y; x = x - y; }
}

// GaussJordanElimination (matrix.c:482)
bool gauss_jordan(Matrix &a, double **vectors, size_t nvec) {
  const long rank = static_cast<long>(a.rank);
  std::vector<long> columns(rank, 0), rows(rank, 0), pivots(rank, 0);
  long column = 0, row = 0;
  auto &m = a.m;
  for (long i = 0; i < rank; ++i) {
    double max = 0.0;
    for (long j = 0; j < rank; ++j)
      if (pivots[j] != 1)
        for (long k = 0; k < rank; ++k)
          if (pivots[k] != 0) {
            if (pivots[k] > 1) return false;
          } else if (std::fabs(m[j][k]) >= max) {
            max = std::fabs(m[j][k]);
            row = j;
            column = k;
          }
    pivots[column]++;
    if (row != column) {
      for (long k = 0; k < rank; ++k) gj_swap(m[row][k], m[column][k]);
      for (size_t k = 0; k < nvec; ++k) gj_swap(vectors[k][row], vectors[k][column]);
    }
    rows[i] = row;
    columns[i] = column;
    if (m[column][column] == 0.0) return false;
    double scale = perceptible_reciprocal(m[column][column]);
    m[column][column] = 1.0;
    for (long j = 0; j < rank; ++j) m[column][j] *= scale;
    for (size_t j = 0; j < nvec; ++j) vectors[j][column] *= scale;
    for (long j = 0; j < rank; ++j)
      if (j != column) {
        scale = m[j][column];
        m[j][column] = 0.0;
        for (long k = 0; k < rank; ++k) m[j][k] -= scale * m[column][k];
        for (size_t k = 0; k < nvec; ++k) vectors[k][j] -= scale * vectors[k][column];
      }
  }
  for (long j = rank - 1; j >= 0; --j)
    if (columns[j] != rows[j])
      for (long i = 0; i < rank; ++i) gj_swap(m[i][rows[j]], m[i][columns[j]]);
  return true;
}

void affine_args_to_coefficients(double *c) {    // :78-84: sx,ry,rx,sy,tx,ty -> c0,c2,c4,c1,c3,c5
  const double t0 = c[1], t1 = c[2], t2 = c[3], t3 = c[4];
  c[3] = t0; c[1] = t1; c[4] = t2; c[2] = t3;
}

void invert_affine(const double *c, double *inv) {          // :94
  const double det = perceptible_reciprocal(c[0] * c[4] - c[1] * c[3]);
  inv[0] = det * c[4];
  inv[1] = det * (-c[1]);
  inv[2] = det * (c[1] * c[5] - c[2] * c[4]);
  inv[3] = det * (-c[3]);
  inv[4] = det * c[0];
  inv[5] = det * (c[2] * c[3] - c[0] * c[5]);
}

void invert_perspective(const double *c, double *inv) {     // :108
  const double det = perceptible_reciprocal(c[0] * c[4] - c[3] * c[1]);
  inv[0] = det * (c[4] - c[7] * c[5]);
  inv[1] = det * (c[7] * c[2] - c[1]);
  inv[2] = det * (c[1] * c[5] - c[4] * c[2]);
  inv[3] = det * (c[6] * c[5] - c[3]);
  inv[4] = det * (c[0] - c[6] * c[2]);
  inv[5] = det * (c[3] * c[2] - c[0] * c[5]);
  inv[6] = det * (c[3] * c[7] - c[6] * c[4]);
  inv[7] = det * (c[6] * c[1] - c[0] * c[7]);
}

// GenerateCoefficients for the six methods: *map receives the reduced method (affine / perspective).
int coefficients(int method, const double *args, size_t n, size_t width, size_t height, long px, long py, double *coeff,
                 int *map) {
  for (int i = 0; i < 9; ++i) coeff[i] = 0.0;
  if (n < 16 && method == kPerspective) method = kAffine;                   // :408-415, cp_size 4
  switch (method) {
    case kAffine: {                                                         // :502-597
      if (n % 4 != 0 || n < 4) return mb200::fail(MB200_EINVAL, "Affine: require at least 1 CPs");
      *map = MB200_DistortAffineMap;
      if (n == 4) {
        coeff[0] = 1.0;
        coeff[2] = args[0] - args[2];
        coeff[4] = 1.0;
        coeff[5] = args[1] - args[3];
        return MB200_OK;
      }
      Matrix a(3);
      double *vectors[2] = {&coeff[0], &coeff[3]};
      double terms[3];
      for (size_t i = 0; i < n; i += 4) {
        terms[0] = args[i + 2];
        terms[1] = args[i + 3];
        terms[2] = 1;
        add_terms(a, vectors, terms, &args[i], 2);
      }
      if (n == 8) {                               // a third point: p1 rotated 90 degrees about p0
        terms[0] = args[2] - (args[4 + 3] - args[3]);
        terms[1] = args[3] + +(args[4 + 2] - args[2]);
        terms[2] = 1;
        const double uv2[2] = {args[0] - args[5] + args[1], args[1] + args[4] - args[0]};
        add_terms(a, vectors, terms, uv2, 2);
      }
      if (!gauss_jordan(a, vectors, 2)) return mb200::fail(MB200_EINVAL, "Affine: Unsolvable Matrix");
      return MB200_OK;
    }
    case kRigidAffine: {                                                    // :611-690
      if (n % 4 != 0 || n < 4) return mb200::fail(MB200_EINVAL, "RigidAffine: require at least 2 CPs");
      *map = MB200_DistortAffineMap;
      Matrix a(4);
      double *vectors[1] = {&coeff[0]};
      double terms[4];
      for (size_t i = 0; i < n; i += 4) {
        terms[0] = args[i + 0]; terms[1] = -args[i + 1]; terms[2] = 1.0; terms[3] = 0.0;
        add_terms(a, vectors, terms, &args[i + 2], 1);
        terms[0] = args[i + 1]; terms[1] = args[i + 0]; terms[2] = 0.0; terms[3] = 1.0;
        add_terms(a, vectors, terms, &args[i + 3], 1);
      }
      if (!gauss_jordan(a, vectors, 1)) return mb200::fail(MB200_EINVAL, "RigidAffine: Unsolvable Matrix");
      double inverse[6] = {coeff[0], coeff[1], -coeff[1], coeff[0], coeff[2], coeff[3]};
      affine_args_to_coefficients(inverse);
      invert_affine(inverse, coeff);
      return MB200_OK;
    }
    case kAffineProjection: {                                               // :691-720
      if (n != 6) return mb200::fail(MB200_EINVAL, "AffineProjection: Needs 6 coeff values");
      *map = MB200_DistortAffineMap;
      double inverse[8];
      for (int i = 0; i < 6; ++i) inverse[i] = args[i];
      affine_args_to_coefficients(inverse);
      invert_affine(inverse, coeff);
      return MB200_OK;
    }
    case kSRT: {                                                            // :721-826
      double x, y, nx, ny, sx = 1.0, sy = 1.0, a;
      x = nx = static_cast<double>(width) / 2.0 + static_cast<double>(px);
      y = ny = static_cast<double>(height) / 2.0 + static_cast<double>(py);
      switch (n) {
        case 0: return mb200::fail(MB200_EINVAL, "ScaleRotateTranslate: Needs at least 1 argument");
        case 1: a = args[0]; break;
        case 2: sx = sy = args[0]; a = args[1]; break;
        default:
          x = nx = args[0];
          y = ny = args[1];
          switch (n) {
            case 3: a = args[2]; break;
            case 4: sx = sy = args[2]; a = args[3]; break;
            case 5: sx = args[2]; sy = args[3]; a = args[4]; break;
            case 6: sx = sy = args[2]; a = args[3]; nx = args[4]; ny = args[5]; break;
            case 7: sx = args[2]; sy = args[3]; a = args[4]; nx = args[5]; ny = args[6]; break;
            default: return mb200::fail(MB200_EINVAL, "ScaleRotateTranslate: Too Many Arguments (7 or less)");
          }
      }
      if (std::fabs(sx) < kEps || std::fabs(sy) < kEps) return mb200::fail(MB200_EINVAL, "ScaleRotateTranslate: Zero Scale Given");
      *map = MB200_DistortAffineMap;
      a = kPi * a / 180.0;                                                  // DegreesToRadians
      const double cosine = std::cos(a), sine = std::sin(a);
      coeff[0] = cosine / sx;
      coeff[1] = sine / sx;
      coeff[2] = x - nx * coeff[0] - ny * coeff[1];
      coeff[3] = (-sine) / sy;
      coeff[4] = cosine / sy;
      coeff[5] = y - nx * coeff[3] - ny * coeff[4];
      return MB200_OK;
    }
    case kPerspective: {                                                    // :827-934
      if (n % 4 != 0) return mb200::fail(MB200_EINVAL, "Perspective: require at least 4 CPs");
      *map = MB200_DistortPerspectiveMap;
      Matrix a(8);
      double *vectors[1] = {&coeff[0]};
      double terms[8];
      for (size_t i = 0; i < n; i += 4) {
        terms[0] = args[i + 2]; terms[1] = args[i + 3]; terms[2] = 1.0;
        terms[3] = 0.0; terms[4] = 0.0; terms[5] = 0.0;
        terms[6] = -terms[0] * args[i + 0];
        terms[7] = -terms[1] * args[i + 0];
        add_terms(a, vectors, terms, &args[i + 0], 1);
        terms[0] = 0.0; terms[1] = 0.0; terms[2] = 0.0;
        terms[3] = args[i + 2]; terms[4] = args[i + 3]; terms[5] = 1.0;
        terms[6] = -terms[3] * args[i + 1];
        terms[7] = -terms[4] * args[i + 1];
        add_terms(a, vectors, terms, &args[i + 1], 1);
      }
      if (!gauss_jordan(a, vectors, 1)) return mb200::fail(MB200_EINVAL, "Perspective: Unsolvable Matrix");
      coeff[8] = coeff[6] * args[2] + coeff[7] * args[3] + 1.0;
      coeff[8] = (coeff[8] < 0.0) ? -1.0 : +1.0;
      return MB200_OK;
    }
    case kPerspectiveProjection: {                                          // :935-960
      if (n != 8) return mb200::fail(MB200_EINVAL, "PerspectiveProjection: Needs 8 coefficient values");
      *map = MB200_DistortPerspectiveMap;
      invert_perspective(args, coeff);
      coeff[8] = coeff[6] * args[2] + coeff[7] * args[5] + 1.0;
      coeff[8] = (coeff[8] < 0.0) ? -1.0 : +1.0;
      return MB200_OK;
    }
    default:
      return mb200::fail(MB200_EUNSUPPORTED, "distort method %d is not implemented on the GPU", method);
  }
}

}  // namespace

extern "C" {

int mb200_distort_plan(int method, const double *args, size_t n, int bestfit, size_t width, size_t height, long px,
                       long py, const long *viewport, double scale, mb200_distort_params *plan) {
  if (!plan || (n && !args) || width == 0 || height == 0) return mb200::fail(MB200_EINVAL, "distort plan: bad arguments");
  mb200_distort_params p = {};
  int rc = coefficients(method, args, n, width, height, px, py, p.coeff, &p.map);
  if (rc) return rc;
  long gx = 0, gy = 0;
  size_t gw = width, gh = height;
  if (bestfit) {                                                            // :1827-1990
    double mnx = 0, mxx = 0, mny = 0, mxy = 0;
    const double sxs[4] = {static_cast<double>(px), static_cast<double>(px) + width, static_cast<double>(px),
                           static_cast<double>(px) + width};
    const double sys[4] = {static_cast<double>(py), static_cast<double>(py), static_cast<double>(py) + height,
                           static_cast<double>(py) + height};
    double inv[8];
    if (p.map == MB200_DistortAffineMap) invert_affine(p.coeff, inv);
    else invert_perspective(p.coeff, inv);
    for (int k = 0; k < 4; ++k) {
      const double sx = sxs[k], sy = sys[k];
      double dx, dy;
      if (p.map == MB200_DistortAffineMap) {
        dx = inv[0] * sx + inv[1] * sy + inv[2];
        dy = inv[3] * sx + inv[4] * sy + inv[5];
      } else {
        const double s = perceptible_reciprocal(inv[6] * sx + inv[7] * sy + 1.0);
        dx = s * (inv[0] * sx + inv[1] * sy + inv[2]);
        dy = s * (inv[3] * sx + inv[4] * sy + inv[5]);
      }
      if (k == 0) { mnx = mxx = dx; mny = mxy = dy; }
      else {                                                                // MagickMin / MagickMax
        mnx = mnx < dx ? mnx : dx; mxx = mxx > dx ? mxx : dx;
        mny = mny < dy ? mny : dy; mxy = mxy > dy ? mxy : dy;
      }
    }
    gx = static_cast<long>(std::floor(mnx - 0.5));
    gy = static_cast<long>(std::floor(mny - 0.5));
    gw = static_cast<size_t>(std::ceil(mxx - gx + 0.5));
    gh = static_cast<size_t>(std::ceil(mxy - gy + 0.5));
  }
  if (viewport) {                                                           // :2033
    gw = static_cast<size_t>(viewport[0]);
    gh = static_cast<size_t>(viewport[1]);
    gx = viewport[2];
    gy = viewport[3];
  }
  p.output_scaling = 1.0;
  if (!std::isnan(scale)) {                                                       // :2393-2410
    p.output_scaling = std::fabs(scale);
    gw = static_cast<size_t>(p.output_scaling * gw + 0.5);
    gh = static_cast<size_t>(p.output_scaling * gh + 0.5);
    gx = static_cast<long>(p.output_scaling * gx + 0.5);
    gy = static_cast<long>(p.output_scaling * gy + 0.5);
    if (p.output_scaling < 0.1) return mb200::fail(MB200_EINVAL, "InvalidArgument: -set option:distort:scale");
    p.output_scaling = 1 / p.output_scaling;
  }
  if (gw == 0 || gh == 0) return mb200::fail(MB200_EINVAL, "NegativeOrZeroImageSize");
  p.columns = gw;
  p.rows = gh;
  p.page_x = gx;
  p.page_y = gy;
  p.bestfit = bestfit ? 1 : 0;
  p.src_page_x = px;
  p.src_page_y = py;
  *plan = p;
  return MB200_OK;
}

int mb200_rotate_plan(double degrees, size_t width, size_t height, long px, long py, mb200_distort_params *plan) {
  double angle = std::fmod(degrees, 360.0);                                 // :2976-2988
  while (angle < -45.0) angle += 360.0;
  while (angle > 45.0) angle -= 90.0;
  const double shear_x = -std::tan(kPi * angle / 180.0 / 2.0);
  const double shear_y = std::sin(kPi * angle / 180.0);
  if (std::fabs(shear_x) < kEps && std::fabs(shear_y) < kEps)
    return mb200::fail(MB200_EUNSUPPORTED, "rotate: %g degrees is an integral rotation", degrees);
  return mb200_distort_plan(kSRT, &degrees, 1, 1, width, height, px, py, nullptr, std::nan(""), plan);
}

}  // extern "C"
