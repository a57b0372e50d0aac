// boundary.cuh -- vision_tools::computeObjectMaskBoundaryMask on a provided motion mask (VisionTools.cc:361-449), as
// FeatureTracker::objectDetection calls it (FeatureTracker.cc:1151-1210), stated as integer rules that host and device share.
//
// The reference, per object label j of the int32 motion mask M: D_j = dilate(M == j, MORPH_RECT 1x11); drawContours of every
// RETR_TREE contour of D_j, FILLED with j, into a u8 image T; bb_j = the union of the contours' bounding rects.  Then
// outer = dilate(T, ELLIPSE(2t+1)) - T, inner = T - erode(T, ELLIPSE(21)), boundary = 255 with 0 where outer or inner is
// non-zero, and inner_bb_j = findObjectBoundingBox(erode(T), j).  Restated:
//   T(x, y)       = max { M(x, y+d) : |d| <= 5, inside the image }   (filling D_j's contours gives back D_j; labels are drawn
//                   in ascending order, so the largest label wins where dilations overlap -- the reference's order is that of an
//                   unordered_set, i.e. unspecified);
//   outer(p)      <=> max over E_t(p) of T > T(p),   inner(p) <=> min over E_10(p) of T < T(p), E_r the rows of
//                   cv::getStructuringElement(MORPH_ELLIPSE, (2r+1, 2r+1)) centred on p, pixels outside the image never winning
//                   (OpenCV's default morphology border);
//   bb_j          = x extent of M == j, y extent widened by 5 rows and clipped to the image; inner_bb_j likewise over
//                   erode(T) == j, (0, 0, 0, 0) when that set is empty.
// Everything is integer max / min / compare, so any evaluation order gives the same result.
#pragma once
#include <cmath>
#include <cstdint>

#define BOUNDARY_MAX_LABEL 255        // CHECK_LE(object_id, 255) (VisionTools.cc:394): T is a u8 image
#define BOUNDARY_MAX_THICKNESS 127    // the scaled thickness of objectDetection up to 2560 x 1440 is 120
#define BOUNDARY_INNER 10             // inner_thickness (VisionTools.cc:412)
#define BOUNDARY_PAD 5                // the 1x11 rectangle of findObjectBoundingBox: +-5 rows

// objectDetection's scaled_boarder_thickness for a W x H image (FeatureTracker.cc:1159-1164), in the reference's operation order
__host__ __device__ inline int boundary_thickness(int W, int H) {
  const double image_ratio = static_cast<double>(W*H)/(640.0*480.0);
  return (int)::round(image_ratio*640.0/480.0*7.51);
}

// half width of row dy (|dy| <= r) of cv::getStructuringElement(MORPH_ELLIPSE, Size(2r+1, 2r+1)): OpenCV's
// saturate_cast<int>(c*sqrt((r*r - dy*dy)*inv_r2)) (round half to even), clipped to the element
__host__ __device__ inline int boundary_ellipse_hw(int r, int dy) {
  const double inv_r2 = r ? 1.0/((double)r*r) : 0.0;
  const int dx = (int)::rint(r*::sqrt((r*r - dy*dy)*inv_r2));
  return dx < r ? dx : r;
}

// the sparse-table level that covers a run of 2w+1 pixels with two overlapping windows of 2^level pixels
__host__ __device__ inline int boundary_level(int w) {
  int k = 0;
  while ((2 << k) <= 2*w + 1) k++;
  return k;
}

// T at (x, y): the largest label of the 1x11 column window (ascending drawContours: the last writer is the largest label)
__host__ __device__ inline int boundary_column_max(const int32_t* M, int W, int H, int x, int y) {
  int best = 0;
  for (int d = -BOUNDARY_PAD; d <= BOUNDARY_PAD; d++) {
    const int yy = y + d;
    if (yy < 0 || yy >= H) continue;
    const int v = M[(size_t)yy*W + x];
    if (v > best) best = v;
  }
  return best;
}

__host__ __device__ inline bool boundary_label_ok(int32_t v) { return v >= 0 && v <= BOUNDARY_MAX_LABEL; }

// the boundary mask at a pixel from T, the max of T over E_t and the min of T over E_10 (both include the pixel)
__host__ __device__ inline uint8_t boundary_value(int t_p, int dil, int ero) { return (dil > t_p || ero < t_p) ? 0 : 255; }

// Raw per-label extents, as the device tables hold them: every field is combined with max, so a zeroed table is empty and
// (W - x_min, H - y_min, x_max + 1, y_max + 1) are stored.
__host__ __device__ inline void boundary_extent_add(int* e, int W, int H, int x, int y) {
  if (W - x > e[0]) e[0] = W - x;
  if (H - y > e[1]) e[1] = H - y;
  if (x + 1 > e[2]) e[2] = x + 1;
  if (y + 1 > e[3]) e[3] = y + 1;
}

// cv::Rect (x, y, w, h) of findObjectBoundingBox from a raw extent: the 1x11 dilation widens the rows by pad, clipped to the
// image; (0, 0, 0, 0) for an empty extent
__host__ __device__ inline void boundary_rect(const int* e, int W, int H, int pad, int32_t* r) {
  if (e[2] == 0) { r[0] = r[1] = r[2] = r[3] = 0; return; }
  const int x0 = W - e[0], x1 = e[2] - 1;
  const int y0 = (H - e[1]) - pad < 0 ? 0 : (H - e[1]) - pad;
  const int y1 = (e[3] - 1) + pad > H - 1 ? H - 1 : (e[3] - 1) + pad;
  r[0] = x0; r[1] = y0; r[2] = x1 - x0 + 1; r[3] = y1 - y0 + 1;
}

// ObjectBoundaryMaskResult's lists from the two extent tables ([256][4] each): the labels present in M in ascending order,
// bb and inner_bb; the first min(n, capacity) rows are written.  Returns n.
inline int boundary_finish(const int* bb_ext, const int* inner_ext, int W, int H, int capacity, int32_t* objects, int32_t* bb,
                           int32_t* inner_bb) {
  int n = 0;
  for (int j = 1; j <= BOUNDARY_MAX_LABEL; j++) {
    if (bb_ext[4*j + 2] == 0) continue;
    if (n < capacity) {
      objects[n] = j;
      boundary_rect(bb_ext + 4*j, W, H, BOUNDARY_PAD, bb + 4*n);
      boundary_rect(inner_ext + 4*j, W, H, BOUNDARY_PAD, inner_bb + 4*n);
    }
    n++;
  }
  return n;
}

// The whole call, sequentially, for the host build (tests/capi/boundary_host.cu): M (labels already checked), thickness t.
// T and the boundary mask are u8[H][W]; bb_ext / inner_ext are zeroed [256][4] tables.
inline void boundary_seq(const int32_t* M, int W, int H, int t, uint8_t* T, uint8_t* boundary, int* bb_ext, int* inner_ext) {
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      T[(size_t)y*W + x] = (uint8_t)boundary_column_max(M, W, H, x, y);
      const int j = M[(size_t)y*W + x];
      if (j > 0) boundary_extent_add(bb_ext + 4*j, W, H, x, y);
    }
  for (int y = 0; y < H; y++)
    for (int x = 0; x < W; x++) {
      int dil = 0, ero = 255;
      for (int dy = -t; dy <= t; dy++) {
        const int yy = y + dy, w = boundary_ellipse_hw(t, dy < 0 ? -dy : dy);
        if (yy < 0 || yy >= H) continue;
        for (int xx = x - w; xx <= x + w; xx++)
          if (xx >= 0 && xx < W && T[(size_t)yy*W + xx] > dil) dil = T[(size_t)yy*W + xx];
      }
      for (int dy = -BOUNDARY_INNER; dy <= BOUNDARY_INNER; dy++) {
        const int yy = y + dy, w = boundary_ellipse_hw(BOUNDARY_INNER, dy < 0 ? -dy : dy);
        for (int xx = x - w; xx <= x + w; xx++) {
          int v;
          if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;     // outside the image: never the minimum
          v = T[(size_t)yy*W + xx];
          if (v < ero) ero = v;
        }
      }
      const int tp = T[(size_t)y*W + x];
      boundary[(size_t)y*W + x] = boundary_value(tp, dil, ero);
      if (ero > 0) boundary_extent_add(inner_ext + 4*ero, W, H, x, y);
    }
}
