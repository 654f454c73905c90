// geometry_plan.cpp -- host side of the orientation and crop operators: the output geometry, the output page and the
// map the kernel of geometry.cu runs.
//
// Behavioural mirror of MagickCore/transform.c: CropImage's bounding box, clamps and page rule (:580-677), ShaveImage's
// geometry (:1654-1668), the page updates of FlipImage (:1294-1298), FlopImage (:1430-1434), TransposeImage
// (:2230-2234) and TransverseImage (:2372-2380), RollImage's offset normalisation (:1572-1581); and shear.c's
// IntegralRotateImage (rotations mod 4, the page swaps :1060-1092).  Also the host half of GetImageBoundingBox
// (attribute.c:487-560, the serial rule over trim.cu's row summaries) and TrimImage's geometry (transform.c:2445-2509).
// size_t / ssize_t arithmetic is the reference's, wrap-around included.  No device.
#include "mb200_internal.h"

#include <cmath>
#include <climits>
#include <cstdint>
#include <utility>

namespace {

inline size_t cast_double_to_unsigned(double x) {           // CastDoubleToUnsigned (image-private.h:118)
  if (std::isnan(x)) return 0;
  const double value = std::floor(x);
  if (value >= static_cast<double>(SIZE_MAX)) return SIZE_MAX;
  if (value < 0.0) return 0;
  return static_cast<size_t>(value);
}

inline long cast_double_to_long(double x) {                 // CastDoubleToLong (image-private.h:67)
  if (std::isnan(x)) return 0;
  if (x < 0.0) {
    const double value = std::ceil(x);
    return value < static_cast<double>(LONG_MIN) ? LONG_MIN : static_cast<long>(value);
  }
  const double value = std::floor(x);
  return value > static_cast<double>(LONG_MAX) ? LONG_MAX : static_cast<long>(value);
}

// The page of CloneImage(image, columns, rows) for a new size (image.c:896-911): scaled with the image, the offsets by
// one factor when the two are within 2 of each other.  TransposeImage and TransverseImage start from it.
mb200_page clone_page(size_t columns, size_t rows, size_t new_columns, size_t new_rows, const mb200_page &page) {
  double scale_x = static_cast<double>(new_columns) / static_cast<double>(columns);
  double scale_y = static_cast<double>(new_rows) / static_cast<double>(rows);
  mb200_page p;
  p.width = static_cast<size_t>(cast_double_to_long(std::floor(scale_x * page.width + 0.5)));
  p.height = static_cast<size_t>(cast_double_to_long(std::floor(scale_y * page.height + 0.5)));
  if (std::fabs(scale_x - scale_y) < 2.0) scale_x = scale_y = scale_x < scale_y ? scale_x : scale_y;
  p.x = cast_double_to_long(std::ceil(scale_x * page.x - 0.5));
  p.y = cast_double_to_long(std::ceil(scale_y * page.y - 0.5));
  return p;
}

// CropImage (transform.c:542): the source rectangle and the output page; MB200_EUNSUPPORTED where the reference warns
// GeometryDoesNotContainImage.
int crop(size_t columns, size_t rows, const mb200_page &image_page, const mb200_page &geometry, mb200_geometry_params *p) {
  mb200_page bounding_box = image_page;                                      // :580-585
  if (bounding_box.width == 0 || bounding_box.height == 0) {
    bounding_box.width = columns;
    bounding_box.height = rows;
  }
  mb200_page page = geometry;                                                // :586-590
  if (page.width == 0) page.width = bounding_box.width;
  if (page.height == 0) page.height = bounding_box.height;
  if ((static_cast<double>(bounding_box.x) - page.x) >= static_cast<double>(page.width) ||     // :591-615
      (static_cast<double>(bounding_box.y) - page.y) >= static_cast<double>(page.height) ||
      (static_cast<double>(page.x) - bounding_box.x) > static_cast<double>(columns) ||
      (static_cast<double>(page.y) - bounding_box.y) > static_cast<double>(rows))
    return mb200::fail(MB200_EUNSUPPORTED, "crop: GeometryDoesNotContainImage (outside the virtual canvas)");
  if (page.x < 0 && bounding_box.x >= 0) {                                   // :616-643
    page.width = cast_double_to_unsigned(static_cast<double>(page.width) + page.x - bounding_box.x);
    page.x = 0;
  } else {
    page.width = cast_double_to_unsigned(static_cast<double>(page.width) - (bounding_box.x - page.x));
    page.x -= bounding_box.x;
    if (page.x < 0) page.x = 0;
  }
  if (page.y < 0 && bounding_box.y >= 0) {
    page.height = cast_double_to_unsigned(static_cast<double>(page.height) + page.y - bounding_box.y);
    page.y = 0;
  } else {
    page.height = cast_double_to_unsigned(static_cast<double>(page.height) - (bounding_box.y - page.y));
    page.y -= bounding_box.y;
    if (page.y < 0) page.y = 0;
  }
  if (page.x + static_cast<long>(page.width) > static_cast<long>(columns))   // :644-651
    page.width = static_cast<size_t>(static_cast<long>(columns) - page.x);
  if (geometry.width != 0 && page.width > geometry.width) page.width = geometry.width;
  if (page.y + static_cast<long>(page.height) > static_cast<long>(rows))
    page.height = static_cast<size_t>(static_cast<long>(rows) - page.y);
  if (geometry.height != 0 && page.height > geometry.height) page.height = geometry.height;
  bounding_box.x += page.x;                                                  // :652-653
  bounding_box.y += page.y;
  if (page.width == 0 || page.height == 0)                                   // :654-659
    return mb200::fail(MB200_EUNSUPPORTED, "crop: GeometryDoesNotContainImage (zero area)");
  p->map = MB200_MapIdentity;
  p->columns = page.width;
  p->rows = page.height;
  p->page.width = image_page.width;                                          // :666-677
  p->page.height = image_page.height;
  const long offset_x = bounding_box.x + static_cast<long>(bounding_box.width);
  const long offset_y = bounding_box.y + static_cast<long>(bounding_box.height);
  if (offset_x > static_cast<long>(image_page.width) || offset_y > static_cast<long>(image_page.height)) {
    p->page.width = bounding_box.width;
    p->page.height = bounding_box.height;
  }
  p->page.x = bounding_box.x;
  p->page.y = bounding_box.y;
  p->src_x = page.x;
  p->src_y = page.y;
  return MB200_OK;
}

}  // namespace

extern "C" {

int mb200_geometry_plan(int op, size_t columns, size_t rows, const mb200_page *page, const long *args,
                        mb200_geometry_params *plan) {
  if (!plan || !page || columns == 0 || rows == 0 ||
      ((op == MB200_GeometryCrop || op == MB200_GeometryShave || op == MB200_GeometryIntegralRotate ||
        op == MB200_GeometryRoll) && !args))
    return mb200::fail(MB200_EINVAL, "geometry plan: bad arguments");
  mb200_geometry_params p = {};
  p.map = MB200_MapIdentity;
  p.columns = columns;
  p.rows = rows;
  p.page = *page;
  const long cols = static_cast<long>(columns), nrows = static_cast<long>(rows);
  switch (op) {
    case MB200_GeometryCrop: {
      const mb200_page geometry = {static_cast<size_t>(args[0]), static_cast<size_t>(args[1]), args[2], args[3]};
      const int rc = crop(columns, rows, *page, geometry, &p);
      if (rc) return rc;
      break;
    }
    case MB200_GeometryShave: {                                              // transform.c:1641
      const size_t sw = static_cast<size_t>(args[0]), sh = static_cast<size_t>(args[1]);
      if (2 * sw >= columns || 2 * sh >= rows)
        return mb200::fail(MB200_EUNSUPPORTED, "shave: GeometryDoesNotContainImage");
      const mb200_page geometry = {columns - 2 * sw, rows - 2 * sh, static_cast<long>(sw) + page->x,
                                   static_cast<long>(sh) + page->y};
      const int rc = crop(columns, rows, *page, geometry, &p);
      if (rc) return rc;
      p.page.width -= 2 * sw;
      p.page.height -= 2 * sh;
      p.page.x -= static_cast<long>(sw);
      p.page.y -= static_cast<long>(sh);
      break;
    }
    case MB200_GeometryFlip:                                                 // transform.c:1294-1298
      p.map = MB200_MapFlip;
      if (p.page.height != 0) p.page.y = static_cast<long>(p.page.height) - nrows - p.page.y;
      break;
    case MB200_GeometryFlop:                                                 // :1430-1434
      p.map = MB200_MapFlop;
      if (p.page.width != 0) p.page.x = static_cast<long>(p.page.width) - cols - p.page.x;
      break;
    case MB200_GeometryTranspose:                                            // :2230-2234
      p.map = MB200_MapTranspose;
      p.columns = rows;
      p.rows = columns;
      p.page = clone_page(columns, rows, p.columns, p.rows, *page);
      std::swap(p.page.width, p.page.height);
      std::swap(p.page.x, p.page.y);
      break;
    case MB200_GeometryTransverse:                                           // :2372-2380
      p.map = MB200_MapTransverse;
      p.columns = rows;
      p.rows = columns;
      p.page = clone_page(columns, rows, p.columns, p.rows, *page);
      std::swap(p.page.width, p.page.height);
      std::swap(p.page.x, p.page.y);
      if (p.page.width != 0) p.page.x = static_cast<long>(p.page.width) - static_cast<long>(p.columns) - p.page.x;
      if (p.page.height != 0) p.page.y = static_cast<long>(p.page.height) - static_cast<long>(p.rows) - p.page.y;
      break;
    case MB200_GeometryIntegralRotate: {                                     // shear.c:700
      const size_t rotations = static_cast<size_t>(args[0]) % 4;
      if (rotations == 0) return mb200::fail(MB200_EUNSUPPORTED, "integral rotate: 0 rotations is a clone");
      if (rotations == 1) {
        p.map = MB200_MapRotate90;
        p.columns = rows;
        p.rows = columns;
        std::swap(p.page.width, p.page.height);
        std::swap(p.page.x, p.page.y);
        if (p.page.width != 0) p.page.x = static_cast<long>(p.page.width) - static_cast<long>(p.columns) - p.page.x;
      } else if (rotations == 2) {
        p.map = MB200_MapRotate180;
        if (p.page.width != 0) p.page.x = static_cast<long>(p.page.width) - cols - p.page.x;
        if (p.page.height != 0) p.page.y = static_cast<long>(p.page.height) - nrows - p.page.y;
      } else {
        p.map = MB200_MapRotate270;
        p.columns = rows;
        p.rows = columns;
        std::swap(p.page.width, p.page.height);
        std::swap(p.page.x, p.page.y);
        if (p.page.height != 0) p.page.y = static_cast<long>(p.page.height) - static_cast<long>(p.rows) - p.page.y;
      }
      break;
    }
    case MB200_GeometryRoll: {                                               // transform.c:1572-1581, as remainders
      long ox = args[0] % cols, oy = args[1] % nrows;
      if (ox < 0) ox += cols;
      if (oy < 0) oy += nrows;
      p.roll_x = ox;
      p.roll_y = oy;
      break;
    }
    default:
      return mb200::fail(MB200_EINVAL, "geometry plan: unknown operation %d", op);
  }
  *plan = p;
  return MB200_OK;
}

// GetImageBoundingBox's row loop (attribute.c:487-551) run on the row summaries, in the single-threaded order.  Row y
// starts from the bounds the rows before it left, and its updates reduce as follows:
//   - x: the first x that mismatches target 0, when it is below the bounds' x (:517-519);
//   - y: y itself, when some x mismatches target 0 and y is below the bounds' y (:523-525);
//   - width: the last x that mismatches target 1, when it is above the width W the row started with (:520-522).  The
//     target 3 rule (:529-535) can lower the row's width, but only to an x below W, and the merge (:546) keeps the
//     larger of W and the row's width, so a lowered width never survives;
//   - height: y, when y is above the height the row started with and either some x mismatches target 2 (:526-528) or
//     the target 3 rule fires.  That rule fires at most once per row (it sets the height to y), at the first x that
//     mismatches target 3, and only if that x is below W: a target 1 update raises the width to some x' > W, and every
//     later x is above x'.
// Each row reads only the bounds the rows above it left, so the serial order is one pass over the rows.
int mb200_bounding_box_from_rows(const unsigned *summaries, size_t columns, size_t rows, int edges, mb200_page *box,
                                 int *warning) {
  if (!summaries || !box || columns == 0 || rows == 0 || edges < MB200_TRIM_EDGES_UNSET || edges > 15)
    return mb200::fail(MB200_EINVAL, "bounding box: bad arguments");
  const long cols = static_cast<long>(columns), nrows = static_cast<long>(rows);
  long x, y, width, height;                                                  // :423-456
  if (edges == MB200_TRIM_EDGES_UNSET) {
    width = columns == 1 ? 1 : 0;
    height = rows == 1 ? 1 : 0;
    x = cols;
    y = nrows;
  } else {
    width = cols;
    height = nrows;
    x = 0;
    y = 0;
    if (edges & MB200_TrimEdgeNorth) y = nrows;
    if (edges & MB200_TrimEdgeEast) width = 0;
    if (edges & MB200_TrimEdgeSouth) height = 0;
    if (edges & MB200_TrimEdgeWest) x = cols;
  }
  for (long r = 0; r < nrows; ++r) {
    const unsigned *s = summaries + 4 * r;
    const long first0 = s[0] ? cols - static_cast<long>(s[0]) : cols;
    const long last1 = static_cast<long>(s[1]) - 1;
    const long first3 = s[3] ? cols - static_cast<long>(s[3]) : cols;
    if (first0 < x) x = first0;
    if (first0 < cols && r < y) y = r;
    if (r > height && (s[2] != 0 || first3 < width)) height = r;
    if (last1 > width) width = last1;
  }
  box->x = x;
  box->y = y;
  box->width = static_cast<size_t>(width);
  box->height = static_cast<size_t>(height);
  const bool empty = box->width == 0 || box->height == 0;                    // :553-560
  if (!empty) {
    box->width -= static_cast<size_t>(x - 1);
    box->height -= static_cast<size_t>(y - 1);
  }
  if (warning) *warning = empty ? 1 : 0;
  return MB200_OK;
}

int mb200_trim_plan(size_t columns, size_t rows, const mb200_page *page, const mb200_page *box, int gravity,
                    const size_t *min_size, mb200_geometry_params *plan) {
  if (!page || !box || !plan || gravity < MB200_UndefinedGravity || gravity > MB200_SouthEastGravity)
    return mb200::fail(MB200_EINVAL, "trim plan: bad arguments");
  if (box->width == 0 || box->height == 0)                                   // transform.c:2429-2444
    return mb200::fail(MB200_EUNSUPPORTED, "trim: GeometryDoesNotContainImage (the reference returns a 1x1 clone)");
  mb200_page geometry = *box;
  if (min_size && geometry.width < min_size[0] && geometry.height < min_size[1]) {   // :2445-2507
    const long dw = static_cast<long>(min_size[0]) - static_cast<long>(geometry.width);
    const long dh = static_cast<long>(min_size[1]) - static_cast<long>(geometry.height);
    switch (gravity) {
      case MB200_CenterGravity: geometry.x -= dw / 2; geometry.y -= dh / 2; break;
      case MB200_NorthWestGravity: geometry.x -= dw; geometry.y -= dh; break;
      case MB200_NorthGravity: geometry.x -= dw / 2; geometry.y -= dh; break;
      case MB200_NorthEastGravity: geometry.y -= dh; break;
      case MB200_EastGravity: geometry.y -= dh / 2; break;
      case MB200_SouthGravity: geometry.x -= dw / 2; break;
      case MB200_SouthWestGravity: geometry.x -= dw; break;
      case MB200_WestGravity: geometry.x -= dw; geometry.y -= dh / 2; break;
      default: break;                                                        // SouthEast, Undefined
    }
    geometry.width = min_size[0];
    geometry.height = min_size[1];
  }
  geometry.x += page->x;                                                     // :2508-2510
  geometry.y += page->y;
  const long args[4] = {static_cast<long>(geometry.width), static_cast<long>(geometry.height), geometry.x, geometry.y};
  return mb200_geometry_plan(MB200_GeometryCrop, columns, rows, page, args, plan);
}

}  // extern "C"
