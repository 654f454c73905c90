// kernel_info.cpp -- host side of the convolution / morphology path: builds the
// tap arrays the CUDA kernels consume.
//
// Mirrors (behaviour, not code) MagickCore/morphology.c:
//   AcquireKernelInfo :485, ParseKernelName :372, ParseKernelArray :213,
//   AcquireKernelBuiltIn :950 (Unity :1032, Gaussian/DoG/LoG :1045, Blur :1140,
//   Binomial :1333, Diamond :1537, Square/Rectangle :1560, Octagon :1601, Disk :1625,
//   Plus :1651, Cross :1673), CalcKernelMetaData :2485, ScaleKernelInfo :4571,
//   RotateKernelInfo :4258 and MagickCore/gem.c:262/302 GetOptimalKernelWidth1D/2D.
//
// Taps are generated on the host in double with the host libm `exp`, i.e. with the
// very same arithmetic the reference uses, so they are bit-identical to the
// reference's KernelInfo (tests/test_host_logic.py::test_kernel_strings_match_reference_taps and
// tests/test_golden.py check this against the compiled reference).  Nothing here touches the GPU.
#include "mb200_internal.h"

#include <cctype>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

namespace {

constexpr double kEps = 1.0e-12;                 // MagickEpsilon, magick-type.h:114
constexpr double kQuantumScale = 1.0 / 65535.0;  // magick-type.h:119
constexpr double k2Pi = 6.28318530717958647692528676655900576839433879875020;   // image-private.h:44
constexpr double kSq2Pi = 2.50662827463100024161235523934010416269302368164062; // image-private.h:51
constexpr double kPi = 3.1415926535897932384626433832795028841971693993751058209749445923078164062;

inline double perceptible_reciprocal(double x) {  // pixel-accessor.h:242
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= kEps ? 1.0 / x : sign / kEps;
}

mb200_kernel_info *new_kernel(int type, size_t w, size_t h) {
  auto *k = static_cast<mb200_kernel_info *>(std::calloc(1, sizeof(mb200_kernel_info)));
  if (!k) return nullptr;
  k->type = type;
  k->width = w;
  k->height = h;
  k->values = static_cast<double *>(std::calloc(w * h != 0 ? w * h : 1, sizeof(double)));
  if (!k->values) { std::free(k); return nullptr; }
  return k;
}

void centre_origin(mb200_kernel_info *k) {
  k->x = static_cast<long>((k->width - 1) / 2);
  k->y = static_cast<long>((k->height - 1) / 2);
}

// morphology.c:2485 -- zero tiny taps, accumulate the positive / negative ranges
void calc_meta(mb200_kernel_info *k) {
  k->minimum = k->maximum = 0.0;
  k->negative_range = k->positive_range = 0.0;
  const size_t n = k->width * k->height;
  for (size_t i = 0; i < n; ++i) {
    double &v = k->values[i];
    if (std::fabs(v) < kEps) v = 0.0;
    if (v < 0) k->negative_range += v; else k->positive_range += v;
    if (v < k->minimum) k->minimum = v;
    if (v > k->maximum) k->maximum = v;
  }
}

// Flat ("shape") kernels: every in-shape cell gets `scale`, the rest NaN.
template <typename Pred>
mb200_kernel_info *shape_kernel(int type, size_t w, double scale, Pred inside, bool sum_range) {
  mb200_kernel_info *k = new_kernel(type, w, w);
  if (!k) return nullptr;
  centre_origin(k);
  const double nan = std::numeric_limits<double>::quiet_NaN();
  size_t i = 0;
  for (long v = -k->y; v <= k->y; ++v)
    for (long u = -k->x; u <= k->x; ++u, ++i) {
      if (inside(u, v, k)) {
        k->values[i] = scale;
        if (sum_range) k->positive_range += scale;
      } else {
        k->values[i] = nan;
      }
    }
  k->minimum = k->maximum = scale;
  return k;
}

// Simplified ParseGeometry (geometry.c:922) for kernel arguments:
//   rho [x|,|/] sigma [+|-|,] xi [+|-|,] psi ; flags '@' '>' '<' '!' '%' recorded.
struct Geometry {
  double rho = 0, sigma = 0, xi = 0, psi = 0;
  bool has_rho = false, has_sigma = false, has_xi = false, has_psi = false;
  bool area = false, greater = false, less = false, aspect = false, percent = false;
  bool ok = true;
};

Geometry parse_geometry(const std::string &text) {
  Geometry g;
  std::string s;
  for (char c : text) {
    if (std::isspace(static_cast<unsigned char>(c))) continue;
    switch (c) {
      case '@': g.area = true; break;
      case '>': g.greater = true; break;
      case '<': g.less = true; break;
      case '!': g.aspect = true; break;
      case '%': g.percent = true; break;
      case '(': case ')': break;
      default: s.push_back(c);
    }
  }
  const char *p = s.c_str();
  auto number = [&](double *out) -> bool {
    char *end = nullptr;
    // "0x4" must not be read as a hexadecimal literal (geometry.c:1107)
    if ((p[0] == '0') && (p[1] == 'x' || p[1] == 'X')) { *out = 0.0; p += 1; return true; }
    const double v = std::strtod(p, &end);
    if (end == p) return false;
    *out = v; p = end; return true;
  };
  if (*p == '\0') return g;
  if (*p != '+' && *p != '-' && *p != ',' && *p != 'x' && *p != 'X') {
    if (number(&g.rho)) g.has_rho = true; else { g.ok = false; return g; }
  } else if ((*p == '+' || *p == '-') ) {
    // a leading sign: StringToDouble would consume it as part of rho only if the
    // number is followed by a separator; "+90" alone is an offset (xi)
    const char *save = p; double v;
    char *end = nullptr; v = std::strtod(p, &end);
    if (end != p && (*end == 'x' || *end == 'X' || *end == ',' || *end == '/' || *end == '\0')) {
      g.rho = v; g.has_rho = true; p = end;
    } else p = save;
  }
  if (*p == 'x' || *p == 'X' || *p == ',' || *p == '/') {
    const char sep = *p++;
    if (!((sep == 'x' || sep == 'X') && (*p == '+' || *p == '-'))) {
      if (number(&g.sigma)) g.has_sigma = true;
    }
  }
  auto signed_value = [&](double *out, bool *has) {
    if (*p == ',' || *p == '/') ++p;
    bool neg = false;
    while (*p == '+' || *p == '-') { if (*p == '-') neg = !neg; ++p; }
    double v;
    if (number(&v)) { *out = neg ? -v : v; *has = true; }
  };
  if (*p == '+' || *p == '-' || *p == ',' || *p == '/') {
    signed_value(&g.xi, &g.has_xi);
    if (*p == '+' || *p == '-' || *p == ',' || *p == '/') signed_value(&g.psi, &g.has_psi);
  }
  if (*p != '\0') g.ok = false;
  return g;
}

std::string lower(std::string s) {
  for (char &c : s) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
  return s;
}

void rotate_kernel(mb200_kernel_info *k, double angle);
void expand_rotated(mb200_kernel_info *kernel, double angle);
void expand_mirrored(mb200_kernel_info *kernel);

// morphology.c:213 ParseKernelArray: "WxH+X+Y:v,v,.." or old style "v,v,v,..."
mb200_kernel_info *parse_user_kernel(const std::string &def) {
  std::string body = def;
  int expand = 0;                                        // '@' / '>' / '<' in the size part (:361-366)
  size_t w = 0, h = 0; long ox = -1, oy = -1;
  const size_t colon = def.find(':');
  bool have_geometry = false;
  if (colon != std::string::npos) {
    Geometry g = parse_geometry(def.substr(0, colon));
    if (!g.ok) return nullptr;
    expand = g.area ? 1 : g.greater ? 2 : g.less ? 3 : 0;
    if (!g.has_rho) g.rho = g.sigma;
    if (g.rho < 1.0) g.rho = 1.0;
    if (g.sigma < 1.0) g.sigma = g.rho;
    w = static_cast<size_t>(g.rho); h = static_cast<size_t>(g.sigma);
    if (g.xi < 0.0 || g.psi < 0.0) return nullptr;
    ox = g.has_xi ? static_cast<long>(g.xi) : static_cast<long>((w - 1) / 2);
    oy = g.has_psi ? static_cast<long>(g.psi) : static_cast<long>((h - 1) / 2);
    if (ox >= static_cast<long>(w) || oy >= static_cast<long>(h)) return nullptr;
    body = def.substr(colon + 1);
    have_geometry = true;
  }
  std::vector<double> vals;
  const double nan = std::numeric_limits<double>::quiet_NaN();
  size_t i = 0;
  while (i < body.size()) {
    const char c = body[i];
    if (std::isspace(static_cast<unsigned char>(c)) || c == ',' || c == '\'') { ++i; continue; }
    size_t j = i;
    while (j < body.size() && !std::isspace(static_cast<unsigned char>(body[j])) && body[j] != ',' && body[j] != '\'') ++j;
    const std::string tok = lower(body.substr(i, j - i));
    if (tok == "nan" || tok == "-") vals.push_back(nan);
    else {
      char *end = nullptr;
      const double v = std::strtod(tok.c_str(), &end);
      if (end == tok.c_str() || *end != '\0') return nullptr;
      vals.push_back(v);
    }
    i = j;
  }
  if (!have_geometry) {
    // old odd-square form: size = sqrt(count+1)
    w = h = static_cast<size_t>(std::sqrt(static_cast<double>(vals.size()) + 1.0));
    ox = oy = static_cast<long>((w - 1) / 2);
  }
  if (w * h == 0 || vals.size() != w * h) return nullptr;
  mb200_kernel_info *k = new_kernel(MB200_UserDefinedKernel, w, h);
  if (!k) return nullptr;
  k->x = ox; k->y = oy;
  k->minimum = std::numeric_limits<double>::max();
  k->maximum = -std::numeric_limits<double>::max();
  bool any = false;
  for (size_t n = 0; n < w * h; ++n) {
    k->values[n] = vals[n];
    if (std::isnan(vals[n])) continue;
    any = true;
    if (vals[n] < 0) k->negative_range += vals[n]; else k->positive_range += vals[n];
    if (vals[n] < k->minimum) k->minimum = vals[n];
    if (vals[n] > k->maximum) k->maximum = vals[n];
  }
  if (!any) { mb200_destroy_kernel_info(k); return nullptr; }
  if (expand == 1) expand_rotated(k, 45.0);
  else if (expand == 2) expand_rotated(k, 90.0);
  else if (expand == 3) expand_mirrored(k);
  return k;
}

struct NamedKernel { const char *name; int type; };
const NamedKernel kNames[] = {
  {"blur", MB200_BlurKernel}, {"gaussian", MB200_GaussianKernel}, {"dog", MB200_DoGKernel},
  {"log", MB200_LoGKernel}, {"disk", MB200_DiskKernel}, {"square", MB200_SquareKernel},
  {"diamond", MB200_DiamondKernel}, {"octagon", MB200_OctagonKernel}, {"plus", MB200_PlusKernel},
  {"cross", MB200_CrossKernel}, {"rectangle", MB200_RectangleKernel}, {"unity", MB200_UnityKernel},
  {"binomial", MB200_BinomialKernel}, {"comet", MB200_CometKernel}, {"laplacian", MB200_LaplacianKernel},
  {"sobel", MB200_SobelKernel}, {"freichen", MB200_FreiChenKernel}, {"roberts", MB200_RobertsKernel},
  {"prewitt", MB200_PrewittKernel}, {"compass", MB200_CompassKernel}, {"kirsch", MB200_KirschKernel},
  {"ring", MB200_RingKernel}, {"peaks", MB200_PeaksKernel}, {"edges", MB200_EdgesKernel},
  {"corners", MB200_CornersKernel}, {"diagonals", MB200_DiagonalsKernel}, {"lineends", MB200_LineEndsKernel},
  {"linejunctions", MB200_LineJunctionsKernel}, {"ridges", MB200_RidgesKernel}, {"convexhull", MB200_ConvexHullKernel},
  {"thinse", MB200_ThinSEKernel}, {"skeleton", MB200_SkeletonKernel}, {"chebyshev", MB200_ChebyshevKernel},
  {"manhattan", MB200_ManhattanKernel}, {"octagonal", MB200_OctagonalKernel}, {"euclidean", MB200_EuclideanKernel},
};

// morphology.c:372 ParseKernelName (+ the per-type argument defaults :426-470)
mb200_kernel_info *parse_named_kernel(const std::string &def, bool *was_named) {
  size_t i = 0;
  while (i < def.size() && std::isspace(static_cast<unsigned char>(def[i]))) ++i;
  size_t j = i;
  while (j < def.size() && std::isalpha(static_cast<unsigned char>(def[j]))) ++j;
  const std::string name = lower(def.substr(i, j - i));
  int type = -1;
  // GetNextToken ends the name at white space, ',' or ':' only: "Sobel@" is one token and names no kernel (:395-398)
  const bool clean_end = j >= def.size() || std::isspace(static_cast<unsigned char>(def[j])) || def[j] == ',' || def[j] == ':';
  if (clean_end)
    for (const NamedKernel &n : kNames) if (name == n.name) type = n.type;
  *was_named = (type >= 0);
  if (type < 0) return nullptr;
  while (j < def.size() && (std::isspace(static_cast<unsigned char>(def[j])) || def[j] == ',' || def[j] == ':')) ++j;
  Geometry g = parse_geometry(def.substr(j));
  if (!g.ok) return nullptr;
  switch (type) {
    case MB200_UnityKernel: if (!g.has_rho) g.rho = 1.0; break;
    case MB200_RingKernel: if (!g.has_xi) g.xi = 1.0; break;
    case MB200_ChebyshevKernel: case MB200_ManhattanKernel: case MB200_OctagonalKernel: case MB200_EuclideanKernel:
      if (!g.has_sigma) g.sigma = 100.0;                              // default distance scale (:453-464)
      else if (g.aspect) g.sigma = 65535.0 / (g.sigma + 1);           // '!': the maximum pixel distance
      else if (g.percent) g.sigma *= 65535.0 / 100.0;                 // '%' of the colour range
      break;
    case MB200_SquareKernel: case MB200_DiamondKernel: case MB200_OctagonKernel:
    case MB200_DiskKernel: case MB200_PlusKernel: case MB200_CrossKernel:
      if (!g.has_sigma) g.sigma = 1.0; break;
    case MB200_RectangleKernel:
      if (!g.has_rho) g.rho = g.sigma;
      if (g.rho < 1.0) g.rho = 3;
      if (g.sigma < 1.0) g.sigma = g.rho;
      if (!g.has_xi) g.xi = static_cast<double>((static_cast<long>(g.rho) - 1) / 2);
      if (!g.has_psi) g.psi = static_cast<double>((static_cast<long>(g.sigma) - 1) / 2);
      break;
    default: break;
  }
  mb200_kernel_info *k = mb200_acquire_kernel_builtin(type, g.rho, g.sigma, g.xi, g.psi);
  if (k && k->next == nullptr) {                         // '@' '>' '<': rotated / mirrored lists of a single kernel (:473-481)
    if (g.area) expand_rotated(k, 45.0);
    else if (g.greater) expand_rotated(k, 90.0);
    else if (g.less) expand_mirrored(k);
  }
  return k;
}

// RotateKernelInfo (morphology.c:4258) as what it amounts to for the angles the hot path uses: a rotation by q quarter
// turns, written as ONE index permutation.  With i = column and j = row, a quarter turn maps
//     new(i, j) = old(j, W_new - 1 - i),      origin (x, y) -> (W_new - 1 - y, x),      W_new = H_old,
// which reproduces the reference's three separate mechanisms: the transpose of 1-D kernels (row -> column keeps the tap
// order, column -> row reverses it), the cyclic four-way swap of square kernels and, for q = 2, the plain reversal.
// Like the reference, cylindrical / symmetric built-ins are left alone, a Blur kernel only ever turns by +-90 (a half
// turn of a symmetric 1-D kernel is the identity), a non-square 2-D kernel can only be reflected, and 45-degree steps
// (3x3 only in the reference) are not produced by anything on this path.
void rotate_kernel(mb200_kernel_info *k, double angle) {
  angle = std::fmod(angle, 360.0);
  if (angle < 0) angle += 360.0;
  if (337.5 < angle || angle <= 22.5) return;
  switch (k->type) {                                       // cylindrical / fourfold-symmetric built-ins never turn (:4281-4305)
    case MB200_GaussianKernel: case MB200_DoGKernel: case MB200_LoGKernel: case MB200_DiskKernel:
    case MB200_PeaksKernel: case MB200_LaplacianKernel: case MB200_ChebyshevKernel: case MB200_ManhattanKernel:
    case MB200_EuclideanKernel:
    case MB200_SquareKernel: case MB200_DiamondKernel: case MB200_PlusKernel: case MB200_CrossKernel:
      return;
    case MB200_BlurKernel:
      if (135.0 < angle && angle <= 225.0) return;
      if (225.0 < angle && angle <= 315.0) angle -= 180;
      break;
    default: break;
  }
  // An eighth of a turn exists for 3x3 kernels only (:4307-4340): the eight perimeter cells -- and an origin that sits
  // on the perimeter -- move one place clockwise along the ring.
  const double within = std::fmod(angle, 90.0);
  if (22.5 < within && within <= 67.5) {
    if (k->width == 3 && k->height == 3) {
      static const int ring[8] = {0, 1, 2, 5, 8, 7, 6, 3};
      double old[9];
      for (int i = 0; i < 9; ++i) old[i] = k->values[i];
      for (int i = 0; i < 8; ++i) k->values[ring[(i + 1) % 8]] = old[ring[i]];
      const int at = static_cast<int>(k->x + 3 * k->y);
      if (at != 4)
        for (int i = 0; i < 8; ++i)
          if (ring[i] == at) { const int to = ring[(i + 1) % 8]; k->x = to % 3; k->y = to / 3; break; }
      angle = std::fmod(angle + 315.0, 360.0);
      k->angle = std::fmod(k->angle + 45.0, 360.0);
    }
    // (any other size: the reference prints a complaint and goes on with the quarter turns)
  }
  int q = angle > 45.0 && angle <= 135.0 ? 1 : angle > 135.0 && angle <= 225.0 ? 2 : angle > 225.0 && angle <= 315.0 ? 3 : 0;
  const long W = static_cast<long>(k->width), H = static_cast<long>(k->height);
  if ((q & 1) && W != H && W != 1 && H != 1) return;        // the reference cannot turn such a kernel either
  if (q == 0) return;
  const std::vector<double> old(k->values, k->values + W * H);
  const long Wn = (q & 1) ? H : W, Hn = (q & 1) ? W : H;
  for (long j = 0; j < Hn; ++j)
    for (long i = 0; i < Wn; ++i) {
      long si, sj;                                           // source column / row of new(i, j)
      if (q == 1) { si = j; sj = Wn - 1 - i; }
      else if (q == 2) { si = W - 1 - i; sj = H - 1 - j; }
      else { si = Hn - 1 - j; sj = i; }                      // three quarter turns == one backwards
      k->values[i + j * Wn] = old[si + sj * W];
    }
  const long x = k->x, y = k->y;
  if (q == 1) { k->x = Wn - 1 - y; k->y = x; }
  else if (q == 2) { k->x = W - 1 - x; k->y = H - 1 - y; }
  else { k->x = y; k->y = Hn - 1 - x; }
  k->width = static_cast<size_t>(Wn);
  k->height = static_cast<size_t>(Hn);
  k->angle = std::fmod(k->angle + 90.0 * q, 360.0);
}

void rotate_list(mb200_kernel_info *k, double angle) { for (; k; k = k->next) rotate_kernel(k, angle); }
mb200_kernel_info *last_of(mb200_kernel_info *k) { while (k->next) k = k->next; return k; }

// SameKernelInfo (:2396): same geometry, NaN in the same cells, values within MagickEpsilon
bool same_kernel(const mb200_kernel_info *a, const mb200_kernel_info *b) {
  if (a->width != b->width || a->height != b->height || a->x != b->x || a->y != b->y) return false;
  for (size_t i = 0; i < a->width * a->height; ++i) {
    const bool na = std::isnan(a->values[i]), nb = std::isnan(b->values[i]);
    if (na != nb) return false;
    if (!na && std::fabs(a->values[i] - b->values[i]) >= kEps) return false;
  }
  return true;
}

// ExpandRotateKernelInfo (:2424): append turned copies of the LAST element (the clone carries the rest of the list with
// it, like CloneKernelInfo) until a turn reproduces the first kernel.
void expand_rotated(mb200_kernel_info *kernel, double angle) {
  mb200_kernel_info *last = kernel;
  for (int guard = 0; guard < 64; ++guard) {
    mb200_kernel_info *turned = mb200_clone_kernel_info(last);
    if (!turned) return;
    rotate_list(turned, angle);
    if (same_kernel(kernel, turned)) { mb200_destroy_kernel_info(turned); return; }
    last_of(last)->next = turned;
    last = turned;
  }
}

// ExpandMirrorKernelInfo (:2332): the kernel, its half turn, that one's quarter turn, and the half turn of the latter
void expand_mirrored(mb200_kernel_info *kernel) {
  mb200_kernel_info *last = kernel;
  for (double angle : {180.0, 90.0, 180.0}) {
    mb200_kernel_info *c = mb200_clone_kernel_info(last);
    if (!c) return;
    rotate_list(c, angle);
    last_of(last)->next = c;
    last = c;
  }
}

// ---- kernels the reference defines by a literal array (morphology.c:1333-1535, :1748-2088): the strings are data -------
mb200_kernel_info *from_array(int type, const char *text) {
  mb200_kernel_info *k = parse_user_kernel(text);
  if (k) k->type = type;
  return k;
}
mb200_kernel_info *list_of(int type, std::initializer_list<const char *> texts) {
  mb200_kernel_info *head = nullptr;
  for (const char *t : texts) {
    mb200_kernel_info *k = from_array(type, t);
    if (!k) { mb200_destroy_kernel_info(head); return nullptr; }
    if (!head) head = k; else last_of(head)->next = k;
  }
  return head;
}
void retype(mb200_kernel_info *k, int type) { for (; k; k = k->next) k->type = type; }

const char *laplacian_array(int which) {
  switch (which) {
    case 1: return "3: 0,-1,0  -1,4,-1  0,-1,0";
    case 2: return "3: -2,1,-2  1,4,1  -2,1,-2";
    case 3: return "3: 1,-2,1  -2,4,-2  1,-2,1";
    case 5: return "5: -4,-1,0,-1,-4  -1,2,3,2,-1  0,3,4,3,0  -1,2,3,2,-1  -4,-1,0,-1,-4";
    case 7: return "7:-10,-5,-2,-1,-2,-5,-10 -5,0,3,4,3,0,-5 -2,3,6,7,6,3,-2 -1,4,7,8,7,4,-1 -2,3,6,7,6,3,-2 -5,0,3,4,3,0,-5 -10,-5,-2,-1,-2,-5,-10";
    case 15: return "5: 0,0,-1,0,0  0,-1,-2,-1,0  -1,-2,16,-2,-1  0,-1,-2,-1,0  0,0,-1,0,0";
    case 19: return "9: 0,-1,-1,-2,-2,-2,-1,-1,0  -1,-2,-4,-5,-5,-5,-4,-2,-1  -1,-4,-5,-3,-0,-3,-5,-4,-1  -2,-5,-3,12,24,12,-3,-5,-2  -2,-5,-0,24,40,24,-0,-5,-2  -2,-5,-3,12,24,12,-3,-5,-2  -1,-4,-5,-3,-0,-3,-5,-4,-1  -1,-2,-4,-5,-5,-5,-4,-2,-1  0,-1,-1,-2,-2,-2,-1,-1,0";
    default: return "3: -1,-1,-1  -1,8,-1  -1,-1,-1";
  }
}
const char *thin_se_array(int which) {            // Bloomberg's structuring elements (:1998-2088)
  switch (which) {
    case 41: return "3: -,-,1  0,-,1  -,-,1";
    case 42: return "3: -,-,1  0,-,1  -,0,-";
    case 43: return "3: -,0,-  0,-,1  -,-,1";
    case 44: return "3: -,0,-  0,-,1  -,0,-";
    case 45: return "3: -,0,1  0,-,1  -,0,-";
    case 46: return "3: -,0,-  0,-,1  -,0,1";
    case 47: return "3: -,1,1  0,-,1  -,0,-";
    case 48: return "3: -,-,1  0,-,1  0,-,1";
    case 49: return "3: 0,-,1  0,-,1  -,-,1";
    case 81: return "3: -,1,-  0,-,1  -,1,-";
    case 82: return "3: -,1,-  0,-,1  0,-,-";
    case 83: return "3: 0,-,-  0,-,1  -,1,-";
    case 84: return "3: 0,-,-  0,-,1  0,-,-";
    case 85: return "3: 0,-,1  0,-,1  0,-,-";
    case 86: return "3: 0,-,-  0,-,1  0,-,1";
    case 87: return "3: -,1,-  0,-,1  0,0,-";
    case 88: return "3: -,1,-  0,-,1  0,1,-";
    case 89: return "3: 0,1,-  0,-,1  -,1,-";
    case 423: return "3: -,-,1  0,-,-  -,0,-";
    case 823: return "3: -,1,-  -,-,1  0,-,-";
    case 481: return "3: -,1,1  0,-,1  0,0,-";
    default: return "3: 0,-,1  0,-,1  0,-,1";     // 482, the general edge element
  }
}
mb200_kernel_info *thin_se(int which, double angle, int type) {
  mb200_kernel_info *k = from_array(MB200_ThinSEKernel, thin_se_array(which));
  if (k) { rotate_kernel(k, angle); k->type = type; }
  return k;
}

// FreiChen (:1416-1535): Sobel-like arrays with sqrt(2) written into some cells, most of them rescaled
mb200_kernel_info *frei_chen(double rho, double sigma) {
  constexpr double kSq2 = 1.41421356237309504880168872420969807856967187537695;
  const int which = static_cast<int>(rho);
  struct Variant { const char *text; int plus[2], minus[2]; double scale; };
  auto build = [&](const Variant &v) -> mb200_kernel_info * {
    mb200_kernel_info *k = from_array(MB200_FreiChenKernel, v.text);
    if (!k) return nullptr;
    bool touched = false;
    for (int c : v.plus) if (c >= 0) { k->values[c] = +kSq2; touched = true; }
    for (int c : v.minus) if (c >= 0) { k->values[c] = -kSq2; touched = true; }
    if (touched) calc_meta(k);
    if (v.scale != 0.0) mb200_scale_kernel_info(k, v.scale, 0);
    return k;
  };
  mb200_kernel_info *k = nullptr;
  switch (which) {
    case 2: k = build({"3: 1,2,0  2,0,-2  0,-2,-1", {1, 3}, {5, 7}, 1.0 / 2.0 * kSq2}); break;
    case 10: {
      for (int v = 11; v <= 19; ++v) {
        mb200_kernel_info *one = frei_chen(static_cast<double>(v), 0.0);
        if (!one) { mb200_destroy_kernel_info(k); return nullptr; }
        if (!k) k = one; else last_of(k)->next = one;
      }
      break;
    }
    case 1: case 11: k = build({"3: 1,0,-1  2,0,-2  1,0,-1", {3, -1}, {5, -1}, 1.0 / 2.0 * kSq2}); break;
    case 12: k = build({"3: 1,2,1  0,0,0  1,2,1", {1, 7}, {-1, -1}, 1.0 / 2.0 * kSq2}); break;
    case 13: k = build({"3: 2,-1,0  -1,0,1  0,1,-2", {0, -1}, {8, -1}, 1.0 / 2.0 * kSq2}); break;
    case 14: k = build({"3: 0,1,-2  -1,0,1  2,-1,0", {6, -1}, {2, -1}, 1.0 / 2.0 * kSq2}); break;
    case 15: k = build({"3: 0,-1,0  1,0,1  0,-1,0", {-1, -1}, {-1, -1}, 1.0 / 2.0}); break;
    case 16: k = build({"3: 1,0,-1  0,0,0  -1,0,1", {-1, -1}, {-1, -1}, 1.0 / 2.0}); break;
    case 17: k = build({"3: 1,-2,1  -2,4,-2  -1,-2,1", {-1, -1}, {-1, -1}, 1.0 / 6.0}); break;
    case 18: k = build({"3: -2,1,-2  1,4,1  -2,1,-2", {-1, -1}, {-1, -1}, 1.0 / 6.0}); break;
    case 19: k = build({"3: 1,1,1  1,1,1  1,1,1", {-1, -1}, {-1, -1}, 1.0 / 3.0}); break;
    default: k = build({"3: 1,0,-1  2,0,-2  1,0,-1", {3, -1}, {5, -1}, 0.0}); break;
  }
  if (!k) return nullptr;
  if (std::fabs(sigma) >= kEps) rotate_list(k, sigma);
  else if (rho > 30.0 || rho < -30.0) rotate_list(k, rho);
  return k;
}

}  // namespace

namespace mb200 {
void rotate_kernel_info(mb200_kernel_info *k, double angle) {
  for (; k; k = k->next) rotate_kernel(k, angle);
}

KernelList blur_kernel_pair(double radius, double sigma) {
  KernelList k(mb200_acquire_kernel_builtin(MB200_BlurKernel, radius, sigma, 0.0, 0.0));
  if (k) k->next = mb200_acquire_kernel_builtin(MB200_BlurKernel, radius, sigma, 90.0, 0.0);
  if (k && !k->next) k.reset();
  return k;
}
}  // namespace mb200

extern "C" {

size_t mb200_optimal_kernel_width_1d(double radius, double sigma) {   // gem.c:262
  if (radius > kEps) return static_cast<size_t>(2.0 * std::ceil(radius) + 1.0);
  const double gamma = std::fabs(sigma);
  if (gamma <= kEps) return 3;
  const double alpha = perceptible_reciprocal(2.0 * gamma * gamma);
  const double beta = perceptible_reciprocal(kSq2Pi * gamma);
  size_t width = 5;
  for (;; width += 2) {
    const long j = static_cast<long>(width - 1) / 2;
    double normalize = 0.0;
    for (long i = -j; i <= j; ++i) normalize += std::exp(-(static_cast<double>(i * i)) * alpha) * beta;
    const double value = std::exp(-(static_cast<double>(j * j)) * alpha) * beta / normalize;
    if (value < kQuantumScale || value < kEps) break;
  }
  return width - 2;
}

size_t mb200_optimal_kernel_width_2d(double radius, double sigma) {   // gem.c:302
  if (radius > kEps) return static_cast<size_t>(2.0 * std::ceil(radius) + 1.0);
  const double gamma = std::fabs(sigma);
  if (gamma <= kEps) return 3;
  const double alpha = perceptible_reciprocal(2.0 * gamma * gamma);
  const double beta = perceptible_reciprocal(k2Pi * gamma * gamma);
  size_t width = 5;
  for (;; width += 2) {
    const long j = static_cast<long>(width - 1) / 2;
    double normalize = 0.0;
    for (long v = -j; v <= j; ++v)
      for (long u = -j; u <= j; ++u)
        normalize += std::exp(-(static_cast<double>(u * u + v * v)) * alpha) * beta;
    const double value = std::exp(-(static_cast<double>(j * j)) * alpha) * beta / normalize;
    if (value < kQuantumScale || value < kEps) break;
  }
  return width - 2;
}

void mb200_scale_kernel_info(mb200_kernel_info *kernel, double scaling_factor, int flags) {  // :4571
  if (!kernel) return;
  if (kernel->next) mb200_scale_kernel_info(kernel->next, scaling_factor, flags);
  double pos_scale = 1.0, neg_scale;
  if (flags & 1) {
    if (std::fabs(kernel->positive_range + kernel->negative_range) >= kEps)
      pos_scale = std::fabs(kernel->positive_range + kernel->negative_range);
    else
      pos_scale = kernel->positive_range;
  }
  if (flags & 2) {
    pos_scale = std::fabs(kernel->positive_range) >= kEps ? kernel->positive_range : 1.0;
    neg_scale = std::fabs(kernel->negative_range) >= kEps ? -kernel->negative_range : 1.0;
  } else {
    neg_scale = pos_scale;
  }
  pos_scale = scaling_factor / pos_scale;
  neg_scale = scaling_factor / neg_scale;
  const size_t n = kernel->width * kernel->height;
  for (size_t i = 0; i < n; ++i)
    if (!std::isnan(kernel->values[i])) kernel->values[i] *= (kernel->values[i] >= 0) ? pos_scale : neg_scale;
  kernel->positive_range *= pos_scale;
  kernel->negative_range *= neg_scale;
  kernel->maximum *= (kernel->maximum >= 0.0) ? pos_scale : neg_scale;
  kernel->minimum *= (kernel->minimum >= 0.0) ? pos_scale : neg_scale;
  if (scaling_factor < kEps) {
    std::swap(kernel->positive_range, kernel->negative_range);
    kernel->maximum = kernel->minimum;
    kernel->minimum = 1;
  }
}

mb200_kernel_info *mb200_acquire_kernel_builtin(int type, double rho, double sigma_arg, double xi,
                                               double psi) {
  switch (type) {
    case MB200_UnityKernel: {                                   // :1032
      mb200_kernel_info *k = new_kernel(type, 1, 1);
      if (!k) return nullptr;
      k->maximum = k->values[0] = rho;
      return k;
    }
    case MB200_GaussianKernel: case MB200_DoGKernel: case MB200_LoGKernel: {   // :1045
      double sigma = std::fabs(sigma_arg);
      const double sigma2 = std::fabs(xi);
      size_t w;
      if (rho >= 1.0) w = static_cast<size_t>(rho) * 2 + 1;
      else if (type != MB200_DoGKernel || sigma >= sigma2) w = mb200_optimal_kernel_width_2d(rho, sigma);
      else w = mb200_optimal_kernel_width_2d(rho, sigma2);
      mb200_kernel_info *k = new_kernel(type, w, w);
      if (!k) return nullptr;
      centre_origin(k);
      const long cx = k->x, cy = k->y, W = static_cast<long>(w);
      auto fill = [&](double s, double sign) {
        if (s > kEps) {
          const double A = 1.0 / (2.0 * s * s);
          const double B = 1.0 / (k2Pi * s * s);
          size_t i = 0;
          for (long v = -cy; v <= cy; ++v)
            for (long u = -cx; u <= cx; ++u, ++i) {
              const double g = std::exp(-(static_cast<double>(u * u + v * v)) * A) * B;
              if (sign > 0) k->values[i] = g; else k->values[i] -= g;
            }
        } else {
          if (sign > 0) { std::memset(k->values, 0, w * w * sizeof(double)); k->values[cx + cy * W] = 1.0; }
          else k->values[cx + cy * W] -= 1.0;
        }
      };
      if (type == MB200_GaussianKernel || type == MB200_DoGKernel) fill(sigma, +1.0);
      if (type == MB200_DoGKernel) fill(sigma2, -1.0);
      if (type == MB200_LoGKernel) {
        if (sigma > kEps) {
          const double A = 1.0 / (2.0 * sigma * sigma);
          const double B = 1.0 / (kPi * sigma * sigma * sigma * sigma);
          size_t i = 0;
          for (long v = -cy; v <= cy; ++v)
            for (long u = -cx; u <= cx; ++u, ++i) {
              const double R = (static_cast<double>(u * u + v * v)) * A;
              k->values[i] = (1 - R) * std::exp(-R) * B;
            }
        } else {
          std::memset(k->values, 0, w * w * sizeof(double));
          k->values[cx + cy * W] = 1.0;
        }
      }
      calc_meta(k);
      mb200_scale_kernel_info(k, 1.0, 2);
      return k;
    }
    case MB200_BlurKernel: {                                    // :1140
      double sigma = std::fabs(sigma_arg);
      const size_t w = rho >= 1.0 ? static_cast<size_t>(rho) * 2 + 1 : mb200_optimal_kernel_width_1d(rho, sigma);
      mb200_kernel_info *k = new_kernel(type, w, 1);
      if (!k) return nullptr;
      k->x = static_cast<long>((w - 1) / 2);
      k->y = 0;
      constexpr long kRank = 3;                                 // oversampling, :1161
      const long v = static_cast<long>(w * kRank - 1) / 2;
      if (sigma > kEps) {
        sigma *= kRank;
        const double alpha = 1.0 / (2.0 * sigma * sigma);
        const double beta = 1.0 / (kSq2Pi * sigma);
        for (long u = -v; u <= v; ++u)
          k->values[(u + v) / kRank] += std::exp(-(static_cast<double>(u * u)) * alpha) * beta;
      } else {
        k->values[k->x] = 1.0;
      }
      calc_meta(k);
      mb200_scale_kernel_info(k, 1.0, 2);
      rotate_kernel(k, xi);
      return k;
    }
    case MB200_BinomialKernel: {                                // :1333
      const size_t w = rho < 1.0 ? 3 : static_cast<size_t>(rho) * 2 + 1;
      mb200_kernel_info *k = new_kernel(type, w, w);
      if (!k) return nullptr;
      centre_origin(k);
      // Pascal's triangle row (w-1), outer product, as the reference's fact() ratio
      auto fact = [](size_t n) { size_t f = 1; for (size_t l = 2; l <= n; ++l) f = f * l; return f; };
      const size_t order_f = fact(w - 1);
      size_t i = 0;
      for (size_t v = 0; v < w; ++v) {
        const size_t alpha = order_f / (fact(v) * fact(w - v - 1));
        for (size_t u = 0; u < w; ++u, ++i)
          k->positive_range += k->values[i] =
              static_cast<double>(alpha * order_f / (fact(u) * fact(w - u - 1)));
      }
      k->minimum = 1.0;
      k->maximum = k->values[k->x + k->y * static_cast<long>(w)];
      k->negative_range = 0.0;
      return k;
    }
    case MB200_DiamondKernel: {                                 // :1537
      const size_t w = rho < 1.0 ? 3 : static_cast<size_t>(rho) * 2 + 1;
      return shape_kernel(type, w, sigma_arg,
          [](long u, long v, const mb200_kernel_info *k) { return std::labs(u) + std::labs(v) <= k->x; }, true);
    }
    case MB200_OctagonKernel: {                                 // :1601
      const size_t w = rho < 1.0 ? 5 : static_cast<size_t>(rho) * 2 + 1;
      return shape_kernel(type, w, sigma_arg,
          [](long u, long v, const mb200_kernel_info *k) { return std::labs(u) + std::labs(v) <= k->x + k->x / 2; }, true);
    }
    case MB200_DiskKernel: {                                    // :1625
      long limit = static_cast<long>(rho * rho);
      size_t w;
      if (rho < 0.4) { w = 9; limit = 18; } else w = static_cast<size_t>(std::fabs(rho)) * 2 + 1;
      return shape_kernel(type, w, sigma_arg,
          [limit](long u, long v, const mb200_kernel_info *) { return u * u + v * v <= limit; }, true);
    }
    case MB200_PlusKernel: case MB200_CrossKernel: {            // :1651, :1673
      const size_t w = rho < 1.0 ? 5 : static_cast<size_t>(rho) * 2 + 1;
      mb200_kernel_info *k = (type == MB200_PlusKernel)
          ? shape_kernel(type, w, sigma_arg, [](long u, long v, const mb200_kernel_info *) { return u == 0 || v == 0; }, false)
          : shape_kernel(type, w, sigma_arg, [](long u, long v, const mb200_kernel_info *) { return u == v || u == -v; }, false);
      if (k) k->positive_range = sigma_arg * (k->width * 2.0 - 1.0);
      return k;
    }
    case MB200_SquareKernel: case MB200_RectangleKernel: {      // :1560
      size_t w, h; long ox, oy; double scale;
      if (type == MB200_SquareKernel) {
        w = h = rho < 1.0 ? 3 : static_cast<size_t>(2 * rho + 1);
        ox = oy = static_cast<long>((w - 1) / 2);
        scale = sigma_arg;
      } else {
        if (rho < 1.0 || sigma_arg < 1.0) return nullptr;
        w = static_cast<size_t>(rho); h = static_cast<size_t>(sigma_arg);
        if (xi < 0.0 || xi > static_cast<double>(w) || psi < 0.0 || psi > static_cast<double>(h)) return nullptr;
        ox = static_cast<long>(xi); oy = static_cast<long>(psi);
        scale = 1.0;
      }
      mb200_kernel_info *k = new_kernel(type, w, h);
      if (!k) return nullptr;
      k->x = ox; k->y = oy;
      const long n = static_cast<long>(w * h);
      for (long i = 0; i < n; ++i) k->values[i] = scale;
      k->minimum = k->maximum = scale;
      k->positive_range = scale * n;
      return k;
    }
    case MB200_CometKernel: {                                   // :1228 half a 1-D Gaussian, normalised, turned by xi
      double sigma = std::fabs(sigma_arg);
      const size_t w = rho < 1.0 ? (mb200_optimal_kernel_width_1d(rho, sigma) - 1) / 2 + 1 : static_cast<size_t>(rho);
      mb200_kernel_info *k = new_kernel(type, w, 1);
      if (!k) return nullptr;
      k->x = k->y = 0;
      if (sigma > kEps) {
        constexpr long kRank = 3;
        const long v = static_cast<long>(w) * kRank;
        sigma *= kRank;
        const double A = 1.0 / (2.0 * sigma * sigma);
        for (long u = 0; u < v; ++u) k->values[u / kRank] += std::exp(-(static_cast<double>(u * u)) * A);
        for (size_t i = 0; i < w; ++i) k->positive_range += k->values[i];
      } else {
        k->values[0] = 1.0;
        k->positive_range = 1.0;
      }
      k->minimum = 0.0;
      k->maximum = k->values[0];
      k->negative_range = 0.0;
      mb200_scale_kernel_info(k, 1.0, 1);                       // NormalizeValue
      rotate_kernel(k, xi);
      return k;
    }
    case MB200_LaplacianKernel: return from_array(type, laplacian_array(static_cast<int>(rho)));     // :1333
    case MB200_SobelKernel: case MB200_RobertsKernel: case MB200_PrewittKernel: case MB200_CompassKernel:
    case MB200_KirschKernel: {                                  // :1371-1414: one 3x3 array, turned by rho
      const char *text = type == MB200_SobelKernel ? "3: 1,0,-1  2,0,-2  1,0,-1"
                         : type == MB200_RobertsKernel ? "3: 0,0,0  1,-1,0  0,0,0"
                         : type == MB200_PrewittKernel ? "3: 1,0,-1  1,0,-1  1,0,-1"
                         : type == MB200_CompassKernel ? "3: 1,1,-1  1,-2,-1  1,1,-1" : "3: 5,-3,-3  5,0,-3  5,-3,-3";
      mb200_kernel_info *k = from_array(type, text);
      if (k) rotate_kernel(k, rho);
      return k;
    }
    case MB200_FreiChenKernel: return frei_chen(rho, sigma_arg);
    case MB200_RingKernel: case MB200_PeaksKernel: {            // :1698
      long limit1, limit2;
      size_t w;
      if (rho < sigma_arg) {
        w = static_cast<size_t>(sigma_arg) * 2 + 1;
        limit1 = static_cast<long>(rho * rho); limit2 = static_cast<long>(sigma_arg * sigma_arg);
      } else {
        w = static_cast<size_t>(rho) * 2 + 1;
        limit1 = static_cast<long>(sigma_arg * sigma_arg); limit2 = static_cast<long>(rho * rho);
      }
      if (limit2 <= 0) { w = 7; limit1 = 7; limit2 = 11; }
      const double scale = static_cast<double>(static_cast<long>(type == MB200_PeaksKernel ? 0.0 : xi));
      mb200_kernel_info *k = shape_kernel(type, w, scale, [limit1, limit2](long u, long v, const mb200_kernel_info *) {
        const long r = u * u + v * v;
        return limit1 < r && r <= limit2;
      }, true);
      if (k && type == MB200_PeaksKernel) {
        k->values[k->x + k->y * static_cast<long>(w)] = 1.0;
        k->positive_range = 1.0;
        k->maximum = 1.0;
      }
      return k;
    }
    case MB200_EdgesKernel: {                                   // :1748 the general edge element and its mirror images
      mb200_kernel_info *k = thin_se(482, 0.0, type);
      if (k) expand_mirrored(k);
      return k;
    }
    case MB200_CornersKernel: {                                 // :1757
      mb200_kernel_info *k = thin_se(87, 0.0, type);
      if (k) expand_rotated(k, 90.0);
      return k;
    }
    case MB200_DiagonalsKernel: {                               // :1766
      const int which = static_cast<int>(rho);
      if (which == 1 || which == 2) {
        mb200_kernel_info *k = from_array(type, which == 1 ? "3: 0,0,0  0,-,1  1,1,-" : "3: 0,0,1  0,-,1  0,1,-");
        if (k) rotate_kernel(k, sigma_arg);
        return k;
      }
      mb200_kernel_info *k = list_of(type, {"3: 0,0,0  0,-,1  1,1,-", "3: 0,0,1  0,-,1  0,1,-"});
      if (k) expand_mirrored(k);
      return k;
    }
    case MB200_LineEndsKernel: {                                // :1798
      const char *text = nullptr;
      switch (static_cast<int>(rho)) {
        case 1: text = "3: 0,0,-  0,1,1  0,0,-"; break;
        case 2: text = "3: 0,0,0  0,1,0  0,0,1"; break;
        case 3: text = "3: 0,0,0  0,1,1  0,0,0"; break;
        case 4: text = "3: 0,0,0  0,1,-  0,0,-"; break;
        default: return mb200_acquire_kernel_info("LineEnds:1>;LineEnds:2>");
      }
      mb200_kernel_info *k = from_array(type, text);
      if (k) rotate_kernel(k, sigma_arg);
      return k;
    }
    case MB200_LineJunctionsKernel: {                           // :1828
      const char *text = nullptr;
      switch (static_cast<int>(rho)) {
        case 1: text = "3: 1,-,1  -,1,-  -,1,-"; break;
        case 2: text = "3: 1,-,-  -,1,-  1,-,1"; break;
        case 3: text = "3: -,-,-  1,1,1  -,1,-"; break;
        case 4: text = "3: 1,-,1  -,1,-  1,-,1"; break;
        case 5: text = "3: -,1,-  1,1,1  -,1,-"; break;
        default: return mb200_acquire_kernel_info("LineJunctions:1@;LineJunctions:2>");
      }
      mb200_kernel_info *k = from_array(type, text);
      if (k) rotate_kernel(k, sigma_arg);
      return k;
    }
    case MB200_RidgesKernel: {                                  // :1862
      if (static_cast<int>(rho) == 2) {
        mb200_kernel_info *k = from_array(type, "4x1:0,1,1,0");
        if (!k) return nullptr;
        expand_rotated(k, 90.0);
        mb200_kernel_info *thick = list_of(type, {"4x3+1+1:0,1,1,- -,1,1,- -,1,1,0", "4x3+2+1:0,1,1,- -,1,1,- -,1,1,0",
                                                  "4x3+1+1:-,1,1,0 -,1,1,- 0,1,1,-", "4x3+2+1:-,1,1,0 -,1,1,- 0,1,1,-",
                                                  "3x4+1+1:0,-,- 1,1,1 1,1,1 -,-,0", "3x4+1+2:0,-,- 1,1,1 1,1,1 -,-,0",
                                                  "3x4+1+1:-,-,0 1,1,1 1,1,1 0,-,-", "3x4+1+2:-,-,0 1,1,1 1,1,1 0,-,-"});
        if (!thick) return mb200_destroy_kernel_info(k);
        last_of(k)->next = thick;
        return k;
      }
      mb200_kernel_info *k = from_array(type, "3x1:0,1,0");
      if (k) expand_rotated(k, 90.0);
      return k;
    }
    case MB200_ConvexHullKernel: {                              // :1929 eight kernels: four turns of an element and of its mirror
      mb200_kernel_info *k = from_array(type, "3: 1,1,-  1,0,-  1,-,0");
      mb200_kernel_info *m = from_array(type, "3: 1,1,1  1,0,-  -,-,0");
      if (!k || !m) { mb200_destroy_kernel_info(k); return mb200_destroy_kernel_info(m); }
      expand_rotated(k, 90.0);
      expand_rotated(m, 90.0);
      last_of(k)->next = m;
      return k;
    }
    case MB200_SkeletonKernel: {                                // :1948
      mb200_kernel_info *k = nullptr;
      switch (static_cast<int>(rho)) {
        case 2: {                                               // HIPR variation: the edge element and a corner, four turns
          k = thin_se(482, 0.0, type);
          mb200_kernel_info *c = thin_se(87, 90.0, type);
          if (!k || !c) { mb200_destroy_kernel_info(k); return mb200_destroy_kernel_info(c); }
          k->next = c;
          expand_rotated(k, 90.0);
          break;
        }
        case 3: {                                               // Bloomberg's 4-connected elements and their mirror images
          k = thin_se(41, 0.0, type);
          mb200_kernel_info *b = thin_se(42, 0.0, type), *c = thin_se(43, 0.0, type);
          if (!k || !b || !c) { mb200_destroy_kernel_info(k); mb200_destroy_kernel_info(b); return mb200_destroy_kernel_info(c); }
          k->next = b; b->next = c;
          expand_mirrored(k);
          break;
        }
        default:                                                // the edge element through eight eighth turns
          k = thin_se(482, 0.0, type);
          if (k) expand_rotated(k, 45.0);
          break;
      }
      return k;
    }
    case MB200_ThinSEKernel: return thin_se(static_cast<int>(rho), sigma_arg, type);
    case MB200_ChebyshevKernel: case MB200_ManhattanKernel: case MB200_OctagonalKernel:
    case MB200_EuclideanKernel: {                               // :2090-2178 distance to the origin, scaled by sigma
      const size_t w = type == MB200_OctagonalKernel ? (rho < 2.0 ? 5 : static_cast<size_t>(rho) * 2 + 1)
                                                     : (rho < 1.0 ? 3 : static_cast<size_t>(rho) * 2 + 1);
      mb200_kernel_info *k = new_kernel(type, w, w);
      if (!k) return nullptr;
      centre_origin(k);
      size_t i = 0;
      for (long v = -k->y; v <= k->y; ++v)
        for (long u = -k->x; u <= k->x; ++u, ++i) {
          const double au = std::fabs(static_cast<double>(u)), av = std::fabs(static_cast<double>(v));
          double d;
          if (type == MB200_ChebyshevKernel) d = au > av ? au : av;
          else if (type == MB200_ManhattanKernel) d = static_cast<double>(std::labs(u) + std::labs(v));
          else if (type == MB200_OctagonalKernel) {
            const double r1 = au > av ? au : av, r2 = std::floor(static_cast<double>(std::labs(u) + std::labs(v) + 1) / 1.5);
            d = r1 > r2 ? r1 : r2;
          } else d = std::sqrt(static_cast<double>(u * u + v * v));
          k->positive_range += (k->values[i] = sigma_arg * d);
        }
      k->maximum = k->values[0];
      return k;
    }
    default:
      return nullptr;
  }
}

mb200_kernel_info *mb200_acquire_kernel_info(const char *kernel_string) {   // :485
  if (!kernel_string) return nullptr;
  std::string all(kernel_string);
  mb200_kernel_info *head = nullptr, *tail = nullptr;
  size_t pos = 0;
  while (pos <= all.size()) {
    size_t semi = all.find(';', pos);
    if (semi == std::string::npos) semi = all.size();
    std::string def = all.substr(pos, semi - pos);
    pos = semi + 1;
    bool blank = true;
    for (char c : def) if (!std::isspace(static_cast<unsigned char>(c))) blank = false;
    if (blank) { if (semi == all.size()) break; else continue; }
    size_t first = 0;
    while (first < def.size() && std::isspace(static_cast<unsigned char>(def[first]))) ++first;
    mb200_kernel_info *k = nullptr;
    if (std::isalpha(static_cast<unsigned char>(def[first]))) {
      bool named = false;
      k = parse_named_kernel(def, &named);
      if (!named) k = parse_user_kernel(def);   // e.g. "nan,1,nan,..."
    } else {
      k = parse_user_kernel(def);
    }
    if (!k) { mb200_destroy_kernel_info(head); return nullptr; }
    if (!head) head = k; else tail->next = k;
    tail = k;
    while (tail->next) tail = tail->next;
    if (semi == all.size()) break;
  }
  return head;
}

mb200_kernel_info *mb200_clone_kernel_info(const mb200_kernel_info *kernel) {
  if (!kernel) return nullptr;
  mb200_kernel_info *k = new_kernel(kernel->type, kernel->width, kernel->height);
  if (!k) return nullptr;
  double *vals = k->values;
  *k = *kernel;
  k->values = vals;
  std::memcpy(k->values, kernel->values, kernel->width * kernel->height * sizeof(double));
  k->next = nullptr;
  if (kernel->next) {
    k->next = mb200_clone_kernel_info(kernel->next);
    if (!k->next) return mb200_destroy_kernel_info(k);
  }
  return k;
}

mb200_kernel_info *mb200_destroy_kernel_info(mb200_kernel_info *kernel) {
  while (kernel) {
    mb200_kernel_info *next = kernel->next;
    std::free(kernel->values);
    std::free(kernel);
    kernel = next;
  }
  return nullptr;
}

}  // extern "C"

// ---- effect.c kernels that are built inline by SharpenImage (:3991-4063) and EdgeImage (:1520-1570) ----------
extern "C" {

// SharpenImage: -exp(-(u*u+v*v)/(2 s^2))/(2 pi s^2) everywhere, centre = -2 * sum, then normalised to sum 1.
mb200_kernel_info *mb200_sharpen_kernel(double radius, double sigma) {
  const size_t width = mb200_optimal_kernel_width_2d(radius, sigma);
  mb200_kernel_info *k = new_kernel(MB200_UserDefinedKernel, width, width);
  if (!k) return nullptr;
  centre_origin(k);
  const double s = std::fabs(sigma) < kEps ? kEps : sigma;            // MagickSigma (effect.c)
  double normalize = 0.0;
  const long j = static_cast<long>(width - 1) / 2;
  size_t i = 0;
  for (long v = -j; v <= j; ++v)
    for (long u = -j; u <= j; ++u) {
      k->values[i] = -std::exp(-(static_cast<double>(u * u) + static_cast<double>(v * v)) / (2.0 * s * s)) / (2.0 * kPi * s * s);
      normalize += k->values[i];
      ++i;
    }
  k->values[i / 2] = (-2.0) * normalize;
  normalize = 0.0;
  for (i = 0; i < width * width; ++i) normalize += k->values[i];
  const double gamma = perceptible_reciprocal(normalize);
  for (i = 0; i < width * width; ++i) k->values[i] *= gamma;
  return k;
}

// EmbossImage (effect.c:1632-1665): width = GetOptimalKernelWidth1D(radius, sigma); only the anti-diagonal is non-zero:
// +-8 * exp(-(u*u+v*v)/(2 s^2))/(2 pi s^2), negative where u < 0 or v < 0; normalised to sum 1 (PerceptibleReciprocal).
mb200_kernel_info *mb200_emboss_kernel(double radius, double sigma) {
  const size_t width = mb200_optimal_kernel_width_1d(radius, sigma);
  mb200_kernel_info *k = new_kernel(MB200_UserDefinedKernel, width, width);
  if (!k) return nullptr;
  centre_origin(k);
  const double s = std::fabs(sigma) < kEps ? kEps : sigma;            // MagickSigma
  const long j = static_cast<long>(width - 1) / 2;
  long diag = j;
  size_t i = 0;
  for (long v = -j; v <= j; ++v) {
    for (long u = -j; u <= j; ++u) {
      k->values[i] = ((u < 0 || v < 0) ? -8.0 : 8.0) *
                     std::exp(-(static_cast<double>(u) * static_cast<double>(u) + static_cast<double>(v * v)) / (2.0 * s * s)) /
                     (2.0 * kPi * s * s);
      if (u != diag) k->values[i] = 0.0;
      ++i;
    }
    --diag;
  }
  double normalize = 0.0;
  for (i = 0; i < width * width; ++i) normalize += k->values[i];
  const double gamma = perceptible_reciprocal(normalize);
  for (i = 0; i < width * width; ++i) k->values[i] *= gamma;
  return k;
}

// EdgeImage: width = GetOptimalKernelWidth1D(radius, 0.5); all cells -1, centre = width*height - 1.
mb200_kernel_info *mb200_edge_kernel(double radius) {
  const size_t width = mb200_optimal_kernel_width_1d(radius, 0.5);
  mb200_kernel_info *k = new_kernel(MB200_UserDefinedKernel, width, width);
  if (!k) return nullptr;
  centre_origin(k);
  const size_t n = width * width;
  for (size_t i = 0; i < n; ++i) k->values[i] = -1.0;
  k->values[n / 2] = static_cast<double>(width) * static_cast<double>(width) - 1.0;
  return k;
}

// MotionBlurImage's taps (GetMotionBlurKernel, effect.c:2316-2345) and offsets (:2390-2398).  Returns the tap count
// (GetOptimalKernelWidth1D) or a negative error; arrays hold `max` entries.
long mb200_motion_blur_kernel(double radius, double sigma, double angle, double *taps, long *offset_x, long *offset_y,
                              size_t max) {
  const size_t width = mb200_optimal_kernel_width_1d(radius, sigma);
  if (taps == nullptr || offset_x == nullptr || offset_y == nullptr) return static_cast<long>(width);
  if (width > max) return MB200_EINVAL;
  const double s = std::fabs(sigma) < kEps ? kEps : sigma;            // MagickSigma
  double normalize = 0.0;
  for (size_t i = 0; i < width; ++i) {
    taps[i] = std::exp((-(static_cast<double>(i) * static_cast<double>(i)) / (2.0 * s * s))) / (kSq2Pi * s);
    normalize += taps[i];
  }
  for (size_t i = 0; i < width; ++i) taps[i] /= normalize;
  const double px = static_cast<double>(width) * std::sin(kPi * angle / 180.0);
  const double py = static_cast<double>(width) * std::cos(kPi * angle / 180.0);
  for (size_t i = 0; i < width; ++i) {
    offset_x[i] = static_cast<long>(std::ceil((static_cast<double>(i) * py) / std::hypot(px, py) - 0.5));
    offset_y[i] = static_cast<long>(std::ceil((static_cast<double>(i) * px) / std::hypot(px, py) - 0.5));
  }
  return static_cast<long>(width);
}

}  // extern "C"
