/* CPU checker — TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * apply_view_matrix_transform: invesalius_rs/src/transforms_py.rs:12-49,96-148 ->
 * transforms.rs:9-55 -> interpolation.rs:6-188, restated line for line in C (float64 arithmetic in
 * the reference's operation order, -ffp-contract=off). The reference holds no test or golden vector
 * for this function: PARITY UNPINNED (the restatement is what the device kernels are checked against).
 * nalgebra's Matrix4 * Vector4 accumulates column by column, i.e. every row as
 * ((m0 c0 + m1 c1) + m2 c2) + m3 c3.
 *
 * Returns 0, 3 when a cast to the output type would have panicked (NumCast::from(..).unwrap()), or 4
 * when a Lanczos-4 tap is still outside the volume after get_value's one-step wrap (an axis of 2
 * voxels: ndarray's index panics). Such a sample reads nothing and is written as 0. */
#include <math.h>
#include <stdint.h>

#define IDX3(z, y, x, s) ((z) * (s)[0] + (y) * (s)[1] + (x) * (s)[2])

static inline int cast_i16(double v, int16_t* o) { if (!(v > -32769.0 && v < 32768.0)) return 0; *o = (int16_t)v; return 1; }
static inline int cast_u8(double v, uint8_t* o) { if (!(v > -1.0 && v < 256.0)) return 0; *o = (uint8_t)v; return 1; }
static inline int cast_f64(double v, double* o) { *o = v; return 1; }

static double cubic_interpolate(const double p[4], double x) {
  return p[1] + 0.5 * x * (p[2] - p[0] + x * (2.0 * p[0] - 5.0 * p[1] + 4.0 * p[2] - p[3] + x * (3.0 * (p[1] - p[2]) + p[3] - p[0])));
}
static double bicubic_interpolate(double p[4][4], double x, double y) {
  double arr[4];
  for (int i = 0; i < 4; ++i) arr[i] = cubic_interpolate(p[i], y);
  return cubic_interpolate(arr, x);
}
/* every tap lo .. hi lands in [0, n) after the one-step wrap */
static int taps_wrap_inside(int64_t lo, int64_t hi, int64_t n) { return (lo >= 0 || lo + n >= 0) && (hi < n || hi - n < n); }
static double lanczos_kernel(double x, int a) {
  if (x == 0.0) return 1.0;
  if (-(double)a <= x && x < (double)a) {
    double a_f = (double)a;
    return (a_f * sin(M_PI * x) * sin(M_PI * (x / a_f))) / (M_PI * M_PI * x * x);
  }
  return 0.0;
}

#define DEF_AVMT(NAME, T, CAST)                                                                                  \
  static inline double NAME##_get(const T* v, const int64_t* s, int64_t dz, int64_t dy, int64_t dx, int64_t x,  \
                                  int64_t y, int64_t z) {                                                        \
    if (x < 0) x += dx; else if (x >= dx) x -= dx;                                                               \
    if (y < 0) y += dy; else if (y >= dy) y -= dy;                                                               \
    if (z < 0) z += dz; else if (z >= dz) z -= dz;                                                               \
    return (double)v[IDX3(z, y, x, s)];                                                                          \
  }                                                                                                              \
  int NAME(const T* vol, const int64_t* vs, int64_t dz, int64_t dy, int64_t dx, const double* spacing,          \
           const double* m, int64_t n, int orientation, int minterpol, T cval, T* out, const int64_t* os,        \
           int64_t odz, int64_t ody, int64_t odx) {                                                              \
    const double sx = spacing[0], sy = spacing[1], sz = spacing[2];                                              \
    int bad = 0;                                                                                                 \
    for (int64_t cz = 0; cz < odz; ++cz)                                                                         \
      for (int64_t cy = 0; cy < ody; ++cy)                                                                       \
        for (int64_t cx = 0; cx < odx; ++cx) {                                                                   \
          int64_t z = cz, y = cy, x = cx;                                                                        \
          if (orientation == 0) z = n + cz; else if (orientation == 1) y = n + cy; else if (orientation == 2) x = n + cx; \
          const double c[4] = {(double)z * sz, (double)y * sy, (double)x * sx, 1.0};                            \
          double nc[4];                                                                                          \
          for (int i = 0; i < 4; ++i) nc[i] = ((m[4 * i] * c[0] + m[4 * i + 1] * c[1]) + m[4 * i + 2] * c[2]) + m[4 * i + 3] * c[3]; \
          const double fz = (nc[0] / nc[3]) / sz, fy = (nc[1] / nc[3]) / sy, fx = (nc[2] / nc[3]) / sx;          \
          T val = cval;                                                                                          \
          if (fz >= 0.0 && fz < (double)dz - 1.0 && fy >= 0.0 && fy < (double)dy - 1.0 && fx >= 0.0 &&           \
              fx < (double)dx - 1.0) {                                                                           \
            if (minterpol == 0) {                                                                                \
              val = vol[IDX3((int64_t)fz, (int64_t)fy, (int64_t)fx, vs)];                                        \
            } else if (minterpol == 1) {                                                                         \
              const int64_t x0 = (int64_t)floor(fx), y0 = (int64_t)floor(fy), z0 = (int64_t)floor(fz);           \
              const int64_t x1 = x0 + 1, y1 = y0 + 1, z1 = z0 + 1;                                               \
              const double xd = fx - (double)x0, yd = fy - (double)y0, zd = fz - (double)z0;                     \
              const double v000 = NAME##_get(vol, vs, dz, dy, dx, x0, y0, z0), v100 = NAME##_get(vol, vs, dz, dy, dx, x1, y0, z0), \
                           v010 = NAME##_get(vol, vs, dz, dy, dx, x0, y1, z0), v001 = NAME##_get(vol, vs, dz, dy, dx, x0, y0, z1), \
                           v110 = NAME##_get(vol, vs, dz, dy, dx, x1, y1, z0), v101 = NAME##_get(vol, vs, dz, dy, dx, x1, y0, z1), \
                           v011 = NAME##_get(vol, vs, dz, dy, dx, x0, y1, z1), v111 = NAME##_get(vol, vs, dz, dy, dx, x1, y1, z1); \
              const double c00 = v000 * (1.0 - xd) + v100 * xd, c10 = v010 * (1.0 - xd) + v110 * xd,             \
                           c01 = v001 * (1.0 - xd) + v101 * xd, c11 = v011 * (1.0 - xd) + v111 * xd;             \
              const double c0 = c00 * (1.0 - yd) + c10 * yd, c1 = c01 * (1.0 - yd) + c11 * yd;                   \
              if (!CAST(c0 * (1.0 - zd) + c1 * zd, &val)) { bad |= 1; val = 0; }                                  \
            } else if (minterpol == 2) {                                                                         \
              const int64_t xi = (int64_t)floor(fx), yi = (int64_t)floor(fy), zi = (int64_t)floor(fz);           \
              double p[4][4][4];                                                                                 \
              for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) for (int k = 0; k < 4; ++k)                \
                p[i][j][k] = NAME##_get(vol, vs, dz, dy, dx, xi + i - 1, yi + j - 1, zi + k - 1);                \
              double r[4];                                                                                       \
              for (int i = 0; i < 4; ++i) r[i] = bicubic_interpolate(p[i], fy - (double)yi, fz - (double)zi);    \
              if (!CAST(cubic_interpolate(r, fx - (double)xi), &val)) { bad |= 1; val = 0; }                      \
              else if (val < cval) val = cval;                                                                   \
            } else {                                                                                             \
              const int a = 4;                                                                                   \
              const int64_t xd = (int64_t)floor(fx), yd = (int64_t)floor(fy), zd = (int64_t)floor(fz);           \
              const int64_t xi = xd - a + 1, xf = xd + a, yi = yd - a + 1, yf = yd + a, zi = zd - a + 1, zf = zd + a; \
              if (!taps_wrap_inside(xi, xf - 1, dx) || !taps_wrap_inside(yi, yf - 1, dy) ||                      \
                  !taps_wrap_inside(zi, zf - 1, dz)) {                                                           \
                bad |= 2;                                                                                        \
                out[IDX3(cz, cy, cx, os)] = 0;                                                                   \
                continue;                                                                                        \
              }                                                                                                  \
              double tx[7][7], ty[7];                                                                            \
              for (int64_t kk = zi; kk < zf; ++kk)                                                               \
                for (int64_t jj = yi; jj < yf; ++jj) {                                                           \
                  double lx = 0.0;                                                                               \
                  for (int64_t ii = xi; ii < xf; ++ii)                                                           \
                    lx += NAME##_get(vol, vs, dz, dy, dx, ii, jj, kk) * lanczos_kernel(fx - (double)ii, a);      \
                  tx[kk - zi][jj - yi] = lx;                                                                     \
                }                                                                                                \
              for (int64_t kk = zi; kk < zf; ++kk) {                                                             \
                double ly = 0.0;                                                                                 \
                for (int64_t jj = yi; jj < yf; ++jj) ly += tx[kk - zi][jj - yi] * lanczos_kernel(fy - (double)jj, a); \
                ty[kk - zi] = ly;                                                                                \
              }                                                                                                  \
              double lz = 0.0;                                                                                   \
              for (int64_t kk = zi; kk < zf; ++kk) lz += ty[kk - zi] * lanczos_kernel(fz - (double)kk, a);       \
              if (!CAST(lz, &val)) { bad |= 1; val = 0; }                                                         \
              else if (val < cval) val = cval;                                                                   \
            }                                                                                                    \
          }                                                                                                      \
          out[IDX3(cz, cy, cx, os)] = val;                                                                       \
        }                                                                                                        \
    return (bad & 2) ? 4 : bad ? 3 : 0;                                                                          \
  }
DEF_AVMT(orc_avmt_i16, int16_t, cast_i16)
DEF_AVMT(orc_avmt_u8, uint8_t, cast_u8)
DEF_AVMT(orc_avmt_f64, double, cast_f64)
