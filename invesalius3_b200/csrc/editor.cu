// The 3-D mask editor (invesalius/data/mask3d_editor_state.py): polygon2mask_rs
// (polygon_mask_py.rs:7-27 -> polygon_mask.rs:4-79), mask_cut (mask_cut_py.rs:8-69 -> mask_cut.rs:7-62) and
// brush_mask_rs (brush_mask_py.rs:7-28 -> brush_mask.rs:5-71).
//
// All arithmetic is float64 in the reference's order (-fmad=false; IEEE division, sqrt.rn). Integer
// conversions follow the release build of the crate: `as isize` / `as usize` saturate, `+ 1` / `- 1` on
// isize wrap, and `(w - 1)` on a zero usize wraps.
//
//   k_polygon2mask  one thread per cell of the polygon's bounding box; the vertices are staged through
//                   shared memory in chunks, so any vertex count works. Issue-bound on the edge loop.
//   k_mask_cut      16 voxels per thread with 128-bit loads; a group without a selected voxel (> 127)
//                   returns at once, only changed groups are stored. The products m_i1 p1, m_i2 p2 and
//                   m_i3 are fixed along an x-row and hoisted; the row sums keep nalgebra's order
//                   ((m_i0 p0 + m_i1 p1) + m_i2 p2) + m_i3 p3. Row 2 of M is never read.
//   k_brush_mask    one thread per voxel of the brush's bounding box, through row / plane pitches so the
//                   same kernel edits a whole resident volume or a dense copy of just the box.
#include <math.h>

#include "b2v_common.cuh"

namespace {

struct Mat4 { double m[16]; };

// ---- Rust release-build integer conversions ---------------------------------------------------
int64_t isize_sat(double v) {               // `v as isize`
  if (v != v) return 0;
  if (v >= 9223372036854775808.0) return INT64_MAX;
  if (v < -9223372036854775808.0) return INT64_MIN;
  return (int64_t)v;
}
uint64_t usize_sat(double v) {              // `v as usize`
  if (!(v > 0.0)) return 0;
  if (v >= 18446744073709551616.0) return UINT64_MAX;
  return (uint64_t)v;
}
int64_t wrap_add(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }

// polygon_mask.rs:26-34: (f(v) as isize + d).max(0) as usize, then .min(n)
int64_t poly_bound(double fv, int64_t d, int64_t n) {
  int64_t v = wrap_add(isize_sat(fv), d);
  if (v < 0) v = 0;
  return v < n ? v : n;
}

// ---- polygon2mask ----------------------------------------------------------------------------
constexpr int kPolyChunk = 512;   // vertices per shared-memory chunk (8 KiB, plus the closing vertex)

__global__ void __launch_bounds__(256) k_polygon2mask(const double2* __restrict__ pts, long long n, long long h,
                                                      long long r0, long long nrows, long long c0, long long ncols,
                                                      uint8_t* __restrict__ out) {
  __shared__ double2 s[kPolyChunk + 1];
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const long long cc = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  // the row loop bound is uniform over the block, so every thread reaches every __syncthreads
  for (long long rb = (long long)blockIdx.y * blockDim.y; rb < nrows; rb += (long long)gridDim.y * blockDim.y) {
    const long long rr = rb + threadIdx.y;
    const bool live = rr < nrows && cc < ncols;
    const double px = (double)(r0 + rr), py = (double)(c0 + cc);
    bool inside = false;
    for (long long base = 0; base < n; base += kPolyChunk) {
      const int cnt = (int)(n - base < kPolyChunk ? n - base : kPolyChunk);
      __syncthreads();
      for (int t = tid; t <= cnt; t += blockDim.x * blockDim.y)   // s[0] = vertex j of the chunk's first edge
        s[t] = pts[t == 0 ? (base == 0 ? n - 1 : base - 1) : base + t - 1];
      __syncthreads();
      if (live) {
#pragma unroll 1   // unrolled, the division's slow-path call spills
        for (int k = 0; k < cnt; ++k) {
          const double2 pj = s[k], pi = s[k + 1];
          if (((pi.y > py) != (pj.y > py)) && (px < (pj.x - pi.x) * (py - pi.y) / (pj.y - pi.y) + pi.x)) inside = !inside;
        }
      }
    }
    if (live) out[(r0 + rr) * h + (c0 + cc)] = inside ? 1 : 0;
  }
}

// ---- mask_cut --------------------------------------------------------------------------------
struct CutParams {
  Mat4 M, MV;
  double sx, sy, sz, max_depth;
  double wm1, hm1, wf, hf;          // (w - 1) as f64, (h - 1) as f64, w as f64, h as f64
  long long dy, dx, h, w, n;
  int edit_mode;
};

__device__ __forceinline__ uint32_t byte_mask(uint32_t nibble) {   // bit k -> 0xff in byte k
  return (nibble & 1u ? 0xffu : 0u) | (nibble & 2u ? 0xff00u : 0u) | (nibble & 4u ? 0xff0000u : 0u) |
         (nibble & 8u ? 0xff000000u : 0u);
}

__global__ void __launch_bounds__(256) k_mask_cut(uint8_t* __restrict__ vol, const uint8_t* __restrict__ filt,
                                                  const CutParams P) {
  const long long ngroups = (P.n + 15) / 16;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < ngroups; g += stride) {
    const long long i0 = g * 16;
    const int cnt = P.n - i0 < 16 ? (int)(P.n - i0) : 16;
    uint32_t wd[4] = {0u, 0u, 0u, 0u};
    if (cnt == 16) {
      const uint4 v = ld_stream(reinterpret_cast<const uint4*>(vol + i0));
      wd[0] = v.x; wd[1] = v.y; wd[2] = v.z; wd[3] = v.w;
    } else {
      for (int k = 0; k < cnt; ++k) {
        const uint32_t b = vol[i0 + k];
        if (k < 4) wd[0] |= b << (8 * k);
        else if (k < 8) wd[1] |= b << (8 * (k - 4));
        else if (k < 12) wd[2] |= b << (8 * (k - 8));
        else wd[3] |= b << (8 * (k - 12));
      }
    }
    // bit k of sel: byte k is > 127
    uint32_t sel = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) sel |= flags_to_nibble(wd[j] & 0x80808080u) << (4 * j);
    if (!sel) continue;

    const long long x0 = i0 % P.dx, row0 = i0 / P.dx;
    long long row = -1;
    double a[14];                   // per x-row: m_i1 p1, m_i2 p2 for rows 0, 1, 3 of M and 0..3 of MV
    uint32_t clr = 0;
    while (sel) {
      const int k = __ffs(sel) - 1;
      sel &= sel - 1;
      long long x = x0 + k, r = row0;
      if (x >= P.dx) { r += x / P.dx; x %= P.dx; }
      if (r != row) {
        row = r;
        const double p1 = (double)(r % P.dy) * P.sy, p2 = (double)(r / P.dy) * P.sz;
        const int rows[7] = {0, 1, 3, 0, 1, 2, 3};
#pragma unroll
        for (int i = 0; i < 7; ++i) {
          const double* mi = (i < 3 ? P.M.m : P.MV.m) + 4 * rows[i];
          a[2 * i] = mi[1] * p1;
          a[2 * i + 1] = mi[2] * p2;
        }
      }
      const double p0 = (double)x * P.sx;
      const double* M = P.M.m;
      const double q3 = ((M[12] * p0 + a[4]) + a[5]) + M[15];
      if (!(q3 > 0.0)) continue;
      const double q0 = ((M[0] * p0 + a[0]) + a[1]) + M[3];
      const double q1 = ((M[4] * p0 + a[2]) + a[3]) + M[7];
      const double* V = P.MV.m;
      const double c0 = ((V[0] * p0 + a[6]) + a[7]) + V[3];
      const double c1 = ((V[4] * p0 + a[8]) + a[9]) + V[7];
      const double c2 = ((V[8] * p0 + a[10]) + a[11]) + V[11];
      const double c3 = ((V[12] * p0 + a[12]) + a[13]) + V[15];
      const double qx = q0 / q3, qy = q1 / q3;
      const double cx = c0 / c3, cy = c1 / c3, cz = c2 / c3;
      const double dist = sqrt((cx * cx + cy * cy) + cz * cz);
      if (!(dist <= P.max_depth)) continue;
      const double px = (qx / 2.0 + 0.5) * P.wm1, py = (qy / 2.0 + 0.5) * P.hm1;
      bool zero;
      if (px >= 0.0 && px < P.wf && py >= 0.0 && py < P.hf) zero = __ldg(filt + (long long)py * P.w + (long long)px) != 0;
      else zero = P.edit_mode == 0;
      if (zero) clr |= 1u << k;
    }
    if (!clr) continue;
    if (cnt == 16) {
      uint4 v;
      v.x = wd[0] & ~byte_mask(clr & 15u);
      v.y = wd[1] & ~byte_mask((clr >> 4) & 15u);
      v.z = wd[2] & ~byte_mask((clr >> 8) & 15u);
      v.w = wd[3] & ~byte_mask((clr >> 12) & 15u);
      st_stream(reinterpret_cast<uint4*>(vol + i0), v);
    } else {
      for (int k = 0; k < cnt; ++k)
        if (clr & (1u << k)) vol[i0 + k] = 0;
    }
  }
}

// ---- brush -----------------------------------------------------------------------------------
struct BrushParams {
  double sx, sy, sz, cx, cy, cz, radius_sq;
  long long z0, y0, x0, bz, by, bx;     // box origin and extent (volume indices)
  long long oz, oy, ox, row_pitch, plane_pitch;
  int edit_mode;
};

__global__ void __launch_bounds__(256) k_brush_mask(uint8_t* __restrict__ out, const uint8_t* __restrict__ orig,
                                                    const BrushParams P) {
  const long long total = P.bz * P.by * P.bx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long x = P.x0 + i % P.bx, r = i / P.bx, y = P.y0 + r % P.by, z = P.z0 + r / P.by;
    const long long off = (z - P.oz) * P.plane_pitch + (y - P.oy) * P.row_pitch + (x - P.ox);
    if (P.edit_mode == 1 && out[off] == 0) continue;
    const double dx = (double)x * P.sx - P.cx, dy = (double)y * P.sy - P.cy, dz = (double)z * P.sz - P.cz;
    const double dist_sq = (dx * dx + dy * dy) + dz * dz;
    if (!(dist_sq <= P.radius_sq)) continue;
    if (P.edit_mode == 1) {
      out[off] = 0;
    } else if (orig) {
      const uint8_t o = orig[off];
      if (o > 0) out[off] = o;
    } else {
      out[off] = 255;
    }
  }
}

// brush_mask.rs:24-31, one axis: [floor((c - r)/s).max(0), ceil((c + r)/s).max(0).min(n - 1)] as usize.
// Returns false when the range is empty.
bool brush_axis(double c, double r, double s, int64_t n, int64_t* lo, int64_t* hi) {
  if (n <= 0) return false;
  const uint64_t a = usize_sat(fmax(floor((c - r) / s), 0.0));
  const uint64_t b = usize_sat(fmin(fmax(ceil((c + r) / s), 0.0), (double)(n - 1)));
  if (a > b) return false;
  *lo = (int64_t)a;
  *hi = (int64_t)b;
  return true;
}

bool brush_box(int64_t dz, int64_t dy, int64_t dx, const double* sp, const double* c, double r, int64_t box[6]) {
  return brush_axis(c[2], r, sp[2], dz, &box[0], &box[3]) && brush_axis(c[1], r, sp[1], dy, &box[1], &box[4]) &&
         brush_axis(c[0], r, sp[0], dx, &box[2], &box[5]);
}

}  // namespace

extern "C" int b2v_polygon2mask(const double* polygon_host, int64_t n, int64_t w, int64_t h, uint8_t* out,
                                void* workspace, void* stream) {
  B2V_REQUIRE(n >= 0 && w >= 0 && h >= 0, B2V_ERR_ARG, "polygon2mask: negative size");
  B2V_REQUIRE(w == 0 || h == 0 || out, B2V_ERR_ARG, "polygon2mask: null output");
  B2V_REQUIRE(n == 0 || (polygon_host && workspace), B2V_ERR_ARG, "polygon2mask: null polygon or workspace");
  cudaStream_t s = (cudaStream_t)stream;
  double min_px = 1.7976931348623157e308, max_px = -1.7976931348623157e308;
  double min_py = min_px, max_py = max_px;
  for (int64_t i = 0; i < n; ++i) {
    const double x = polygon_host[2 * i], y = polygon_host[2 * i + 1];
    B2V_REQUIRE(isfinite(x) && isfinite(y), B2V_ERR_ARG, "polygon2mask: vertex %lld is not finite", (long long)i);
    if (x < min_px) min_px = x;
    if (x > max_px) max_px = x;
    if (y < min_py) min_py = y;
    if (y > max_py) max_py = y;
  }
  if (w == 0 || h == 0) return B2V_OK;
  B2V_CUDA(cudaMemsetAsync(out, 0, (size_t)(w * h), s));
  if (n == 0) return B2V_OK;
  const int64_t rx0 = poly_bound(floor(min_px), -1, w), rx1 = poly_bound(ceil(max_px), 1, w);
  const int64_t cy0 = poly_bound(floor(min_py), -1, h), cy1 = poly_bound(ceil(max_py), 1, h);
  const int64_t nrows = (rx1 < w - 1 ? rx1 : w - 1) - rx0 + 1, ncols = (cy1 < h - 1 ? cy1 : h - 1) - cy0 + 1;
  if (nrows <= 0 || ncols <= 0) return B2V_OK;
  B2V_CUDA(cudaMemcpyAsync(workspace, polygon_host, (size_t)n * 2 * sizeof(double), cudaMemcpyHostToDevice, s));
  const dim3 block(32, 8);
  const long long gx = ceil_div64(ncols, 32), gy = ceil_div64(nrows, 8);
  B2V_REQUIRE(gx <= 0x7fffffffLL, B2V_ERR_ARG, "polygon2mask: viewport too large");
  const dim3 grid((unsigned)gx, (unsigned)(gy < 65535 ? gy : 65535));
  k_polygon2mask<<<grid, block, 0, s>>>((const double2*)workspace, n, h, rx0, nrows, cy0, ncols, out);
  return b2v_check_launch("k_polygon2mask");
}

extern "C" int b2v_mask_cut(uint8_t* out, int64_t dz, int64_t dy, int64_t dx, const double* spacing_host,
                            double max_depth, const uint8_t* filter, int64_t h, int64_t w, const double* m_host,
                            const double* mv_host, int edit_mode, void* stream) {
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0 && h >= 0 && w >= 0, B2V_ERR_ARG, "mask_cut: negative size");
  B2V_REQUIRE(spacing_host && m_host && mv_host, B2V_ERR_ARG, "mask_cut: null host argument");
  const long long n = dz * dy * dx;
  if (n == 0) return B2V_OK;
  B2V_REQUIRE(out && (h * w == 0 || filter), B2V_ERR_ARG, "mask_cut: null device pointer");
  B2V_REQUIRE(b2v_aligned16(out), B2V_ERR_ARG, "mask_cut: the mask must be 16-byte aligned");
  CutParams P;
  for (int k = 0; k < 16; ++k) { P.M.m[k] = m_host[k]; P.MV.m[k] = mv_host[k]; }
  P.sx = spacing_host[0]; P.sy = spacing_host[1]; P.sz = spacing_host[2];
  P.max_depth = max_depth;
  P.wm1 = (double)(uint64_t)(w - 1);    // usize arithmetic: wraps when w == 0 (every voxel is off-screen then)
  P.hm1 = (double)(uint64_t)(h - 1);
  P.wf = (double)w; P.hf = (double)h;
  P.dy = dy; P.dx = dx; P.h = h; P.w = w; P.n = n;
  P.edit_mode = edit_mode;
  cudaStream_t s = (cudaStream_t)stream;
  k_mask_cut<<<b2v_grid(ceil_div64(n, 16), 256, 64), 256, 0, s>>>(out, filter, P);
  return b2v_check_launch("k_mask_cut");
}

extern "C" int b2v_brush_mask_box(int64_t dz, int64_t dy, int64_t dx, const double* spacing_host,
                                  const double* center_host, double radius, int64_t* box_host) {
  B2V_REQUIRE(spacing_host && center_host && box_host, B2V_ERR_ARG, "brush_mask_box: null host argument");
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0, B2V_ERR_ARG, "brush_mask_box: negative size");
  if (!brush_box(dz, dy, dx, spacing_host, center_host, radius, box_host)) {
    box_host[0] = box_host[1] = box_host[2] = 0;
    box_host[3] = box_host[4] = box_host[5] = -1;
  }
  return B2V_OK;
}

extern "C" int b2v_brush_mask(uint8_t* out, const uint8_t* orig, int64_t dz, int64_t dy, int64_t dx, int64_t oz,
                              int64_t oy, int64_t ox, int64_t row_pitch, int64_t plane_pitch,
                              const double* spacing_host, const double* center_host, double radius, int edit_mode,
                              void* stream) {
  B2V_REQUIRE(spacing_host && center_host, B2V_ERR_ARG, "brush_mask: null host argument");
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0, B2V_ERR_ARG, "brush_mask: negative size");
  int64_t box[6];
  if (edit_mode != 0 && edit_mode != 1) return B2V_OK;           // brush_mask.rs: any other mode edits nothing
  if (!brush_box(dz, dy, dx, spacing_host, center_host, radius, box)) return B2V_OK;
  B2V_REQUIRE(out, B2V_ERR_ARG, "brush_mask: null output");
  B2V_REQUIRE(oz <= box[0] && oy <= box[1] && ox <= box[2] && oz >= 0 && oy >= 0 && ox >= 0, B2V_ERR_ARG,
              "brush_mask: the buffer starts after the brush box");
  B2V_REQUIRE(row_pitch > 0 && plane_pitch > 0, B2V_ERR_ARG, "brush_mask: bad pitches");
  BrushParams P;
  P.sx = spacing_host[0]; P.sy = spacing_host[1]; P.sz = spacing_host[2];
  P.cx = center_host[0]; P.cy = center_host[1]; P.cz = center_host[2];
  P.radius_sq = radius * radius;
  P.z0 = box[0]; P.y0 = box[1]; P.x0 = box[2];
  P.bz = box[3] - box[0] + 1; P.by = box[4] - box[1] + 1; P.bx = box[5] - box[2] + 1;
  P.oz = oz; P.oy = oy; P.ox = ox; P.row_pitch = row_pitch; P.plane_pitch = plane_pitch;
  P.edit_mode = edit_mode;
  cudaStream_t s = (cudaStream_t)stream;
  k_brush_mask<<<b2v_grid(P.bz * P.by * P.bx, 256, 16), 256, 0, s>>>(out, orig, P);
  return b2v_check_launch("k_brush_mask");
}
