/* CPU checker — TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * The 3-D mask editor of invesalius_rs, restated line for line in C (float64 in the reference's
 * operation order, -ffp-contract=off):
 *   polygon2mask_rs  polygon_mask_py.rs:7-27 -> polygon_mask.rs:4-79
 *   mask_cut         mask_cut_py.rs:8-69 -> mask_cut.rs:7-62
 *   brush_mask_rs    brush_mask_py.rs:7-28 -> brush_mask.rs:5-71
 * Integer conversions are those of the crate's release build: `as isize` / `as usize` saturate
 * (NaN -> 0), isize `+ 1` / `- 1` and usize `w - 1` wrap.
 * The reference holds no test or golden vector for these functions: PARITY UNPINNED. nalgebra's
 * Matrix4 * Vector4 is taken to sum every row as ((m0 p0 + m1 p1) + m2 p2) + m3 p3 (column-axpy
 * order); nalgebra's source is not part of the reference checkout, so that order is an assumption. */
#include <math.h>
#include <stdint.h>

#define IDX3(z, y, x, s) ((z) * (s)[0] + (y) * (s)[1] + (x) * (s)[2])

static int64_t as_isize(double v) {
  if (v != v) return 0;
  if (v >= 9223372036854775808.0) return INT64_MAX;
  if (v < -9223372036854775808.0) return INT64_MIN;
  return (int64_t)v;
}
static uint64_t as_usize(double v) {
  if (!(v > 0.0)) return 0;
  if (v >= 18446744073709551616.0) return UINT64_MAX;
  return (uint64_t)v;
}
static int64_t isize_add(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
static uint64_t usize_min(uint64_t a, uint64_t b) { return a < b ? a : b; }
static int64_t isize_max0(int64_t a) { return a > 0 ? a : 0; }

/* out: dense [w][h] uint8, written completely (1 = true). pts: n (x, y) pairs, dense. */
void orc_polygon2mask(int64_t w, int64_t h, const double* pts, int64_t n, uint8_t* out) {
  for (int64_t i = 0; i < w * h; ++i) out[i] = 0;
  if (n == 0 || w == 0 || h == 0) return;
  double min_px = 1.7976931348623157e308, max_px = -1.7976931348623157e308;
  double min_py = 1.7976931348623157e308, max_py = -1.7976931348623157e308;
  for (int64_t k = 0; k < n; ++k) {
    const double* p = pts + 2 * k;
    if (p[0] < min_px) min_px = p[0];
    if (p[0] > max_px) max_px = p[0];
    if (p[1] < min_py) min_py = p[1];
    if (p[1] > max_py) max_py = p[1];
  }
  uint64_t min_x_idx = (uint64_t)isize_max0(isize_add(as_isize(floor(min_px)), -1));
  uint64_t max_x_idx = (uint64_t)isize_max0(isize_add(as_isize(ceil(max_px)), 1));
  min_x_idx = usize_min(min_x_idx, (uint64_t)w);
  max_x_idx = usize_min(max_x_idx, (uint64_t)w);
  uint64_t min_y_idx = (uint64_t)isize_max0(isize_add(as_isize(floor(min_py)), -1));
  uint64_t max_y_idx = (uint64_t)isize_max0(isize_add(as_isize(ceil(max_py)), 1));
  min_y_idx = usize_min(min_y_idx, (uint64_t)h);
  max_y_idx = usize_min(max_y_idx, (uint64_t)h);

  for (uint64_t r = 0; r < (uint64_t)w; ++r) {
    if (r >= min_x_idx && r <= max_x_idx) {
      const double px = (double)r;
      for (uint64_t c = 0; c < (uint64_t)h; ++c) {
        if (c >= min_y_idx && c <= max_y_idx) {
          const double py = (double)c;
          int inside = 0;
          int64_t j = n - 1;
          for (int64_t i = 0; i < n; ++i) {
            const double xi = pts[2 * i], yi = pts[2 * i + 1];
            const double xj = pts[2 * j], yj = pts[2 * j + 1];
            const int intersect = ((yi > py) != (yj > py)) && (px < (xj - xi) * (py - yi) / (yj - yi) + xi);
            if (intersect) inside = !inside;
            j = i;
          }
          out[r * (uint64_t)h + c] = (uint8_t)inside;
        }
      }
    }
  }
}

static void matvec(const double* m, const double p[4], double q[4]) {
  for (int i = 0; i < 4; ++i) q[i] = ((m[4 * i] * p[0] + m[4 * i + 1] * p[1]) + m[4 * i + 2] * p[2]) + m[4 * i + 3] * p[3];
}

/* mask: [h][w] bool (uint8) with element strides ms; out: [dz][dy][dx] uint8 with element strides os;
 * m, mv: 16 doubles row-major (Matrix4::from_row_slice). */
void orc_mask_cut(double sx, double sy, double sz, double max_depth, const uint8_t* mask, const int64_t* ms,
                  int64_t h, int64_t w, const double* m, const double* mv, uint8_t* out, const int64_t* os,
                  int64_t dz, int64_t dy, int64_t dx, int32_t edit_mode) {
  for (int64_t z = 0; z < dz; ++z)
    for (int64_t y = 0; y < dy; ++y)
      for (int64_t x = 0; x < dx; ++x) {
        uint8_t* val = out + IDX3(z, y, x, os);
        if ((int32_t)*val > 127) {
          const double p[4] = {(double)x * sx, (double)y * sy, (double)z * sz, 1.0};
          double q_[4];
          matvec(m, p, q_);
          if (q_[3] > 0.0) {
            double q[4], c_[4], c[4];
            for (int i = 0; i < 4; ++i) q[i] = q_[i] / q_[3];
            matvec(mv, p, c_);
            for (int i = 0; i < 4; ++i) c[i] = c_[i] / c_[3];
            const double dist = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
            if (dist <= max_depth) {
              const double px = (q[0] / 2.0 + 0.5) * (double)((uint64_t)w - 1);
              const double py = (q[1] / 2.0 + 0.5) * (double)((uint64_t)h - 1);
              if (px >= 0.0 && px < (double)w && py >= 0.0 && py < (double)h) {
                if (mask[(int64_t)as_usize(py) * ms[0] + (int64_t)as_usize(px) * ms[1]]) *val = 0;
              } else if (edit_mode == 0) {
                *val = 0;
              }
            }
          }
        }
      }
}

/* out, orig (or NULL): [d][h][w] uint8 with element strides os / gs. */
void orc_brush_mask(uint8_t* out, const int64_t* os, const uint8_t* orig, const int64_t* gs, int64_t d, int64_t h,
                    int64_t w, double sx, double sy, double sz, double cx, double cy, double cz, double radius,
                    int32_t edit_mode) {
  const uint64_t min_x = as_usize(fmax(floor((cx - radius) / sx), 0.0));
  const uint64_t max_x = as_usize(fmin(fmax(ceil((cx + radius) / sx), 0.0), (double)((uint64_t)w - 1)));
  const uint64_t min_y = as_usize(fmax(floor((cy - radius) / sy), 0.0));
  const uint64_t max_y = as_usize(fmin(fmax(ceil((cy + radius) / sy), 0.0), (double)((uint64_t)h - 1)));
  const uint64_t min_z = as_usize(fmax(floor((cz - radius) / sz), 0.0));
  const uint64_t max_z = as_usize(fmin(fmax(ceil((cz + radius) / sz), 0.0), (double)((uint64_t)d - 1)));
  const double radius_sq = radius * radius;

  for (uint64_t z = 0; z < (uint64_t)d; ++z)
    for (uint64_t y = 0; y < (uint64_t)h; ++y)
      for (uint64_t x = 0; x < (uint64_t)w; ++x) {
        uint8_t* val = out + IDX3((int64_t)z, (int64_t)y, (int64_t)x, os);
        if (z >= min_z && z <= max_z && y >= min_y && y <= max_y && x >= min_x && x <= max_x) {
          if (edit_mode == 1) {
            if ((int32_t)*val > 0) {
              const double ddx = (double)x * sx - cx;
              const double ddy = (double)y * sy - cy;
              const double ddz = (double)z * sz - cz;
              const double dist_sq = ddx * ddx + ddy * ddy + ddz * ddz;
              if (dist_sq <= radius_sq) *val = 0;
            }
          } else if (edit_mode == 0) {
            const double ddx = (double)x * sx - cx;
            const double ddy = (double)y * sy - cy;
            const double ddz = (double)z * sz - cz;
            const double dist_sq = ddx * ddx + ddy * ddy + ddz * ddz;
            if (dist_sq <= radius_sq) {
              if (orig) {
                const uint8_t orig_val = orig[IDX3((int64_t)z, (int64_t)y, (int64_t)x, gs)];
                if ((int32_t)orig_val > 0) *val = orig_val;
              } else {
                *val = 255;
              }
            }
          }
        }
      }
}
