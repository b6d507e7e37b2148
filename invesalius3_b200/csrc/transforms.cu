// apply_view_matrix_transform: invesalius_rs/src/transforms_py.rs:12-49,96-148 -> transforms.rs:9-55 ->
// interpolation.rs:6-188. The step before every projection when the volume is rotated
// (invesalius/data/slice_.py:864-874, 949, 1036) and the body of apply_reorientation (:1980, :2038):
// every output voxel maps its index through the 4x4 view matrix (float64, the reference's
// operation order: no FMA, nalgebra's row sums left to right) and samples the volume with nearest /
// trilinear / tricubic / Lanczos-4 interpolation, indices wrapping once at the faces like get_value.
// One thread per output voxel; gather-bound (8 / 64 / 343 reads per voxel through L1 / L2).
// Bit-exact against the CPU restatement for modes 0-2; mode 3 goes through sin(): libm and the
// device differ by an ulp on rare inputs, which may move a truncated value by one unit.
// Reads stay inside [0, d) on every axis: a sample is interpolated only when 0 <= f < d - 1 on all
// three axes (so d >= 2). Nearest and trilinear read floor(f) and floor(f) + 1 <= d - 1; tricubic's
// taps floor(f) - 1 .. floor(f) + 2 lie in [-1, d] and the one-step wrap brings them into [0, d).
// Lanczos-4's taps floor(f) - 3 .. floor(f) + 3 do too when d >= 3, but on a 2-voxel axis the tap
// -3 is still -1 after the wrap: the reference's ndarray index panics there, and so does this
// kernel (status word, nothing read, B2V_ERR_RANGE).
#include <math.h>

#include "b2v_common.cuh"

namespace {

struct Mat4 { double m[16]; };
struct VDims { long long dz, dy, dx; };

// bits of the status word
enum { kStatusCast = 1, kStatusIndex = 2 };

// true when every tap lo .. hi (lo <= hi) lands in [0, n) after get_value's one-step wrap
__device__ __forceinline__ bool taps_wrap_inside(long long lo, long long hi, long long n) {
  return (lo >= 0 || lo + n >= 0) && (hi < n || hi - n < n);
}

template <typename T> __device__ __forceinline__ bool cast_f64(double v, T* o);
template <> __device__ __forceinline__ bool cast_f64<int16_t>(double v, int16_t* o) {
  if (!(v > -32769.0 && v < 32768.0)) return false;
  *o = (int16_t)v;
  return true;
}
template <> __device__ __forceinline__ bool cast_f64<uint8_t>(double v, uint8_t* o) {
  if (!(v > -1.0 && v < 256.0)) return false;
  *o = (uint8_t)v;
  return true;
}
template <> __device__ __forceinline__ bool cast_f64<double>(double v, double* o) { *o = v; return true; }

template <typename T>
__device__ __forceinline__ double get_value(const T* __restrict__ v, const VDims& d, long long x, long long y, long long z) {
  if (x < 0) x += d.dx; else if (x >= d.dx) x -= d.dx;
  if (y < 0) y += d.dy; else if (y >= d.dy) y -= d.dy;
  if (z < 0) z += d.dz; else if (z >= d.dz) z -= d.dz;
  return (double)v[(z * d.dy + y) * d.dx + x];
}

__device__ __forceinline__ double cubic(const double p[4], double x) {
  return p[1] + 0.5 * x * (p[2] - p[0] + x * (2.0 * p[0] - 5.0 * p[1] + 4.0 * p[2] - p[3] + x * (3.0 * (p[1] - p[2]) + p[3] - p[0])));
}

__device__ __forceinline__ double lanczos_kernel(double x, int a) {
  const double kPi = 3.14159265358979323846;
  if (x == 0.0) return 1.0;
  if (-(double)a <= x && x < (double)a) {
    const double a_f = (double)a;
    return (a_f * sin(kPi * x) * sin(kPi * (x / a_f))) / (kPi * kPi * x * x);
  }
  return 0.0;
}

template <typename T>
__global__ void __launch_bounds__(256) k_view_transform(const T* __restrict__ vol, VDims d, double sx, double sy, double sz,
                                                        Mat4 M, long long n, int orientation, int minterpol, T cval,
                                                        T* __restrict__ out, VDims od, int* status) {
  const long long total = od.dz * od.dy * od.dx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long cx = i % od.dx, r = i / od.dx, cy = r % od.dy, cz = r / od.dy;
    long long z = cz, y = cy, x = cx;
    if (orientation == 0) z = n + cz; else if (orientation == 1) y = n + cy; else if (orientation == 2) x = n + cx;
    const double c0 = (double)z * sz, c1 = (double)y * sy, c2 = (double)x * sx;
    double nc[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) nc[k] = ((M.m[4 * k] * c0 + M.m[4 * k + 1] * c1) + M.m[4 * k + 2] * c2) + M.m[4 * k + 3] * 1.0;
    const double fz = (nc[0] / nc[3]) / sz, fy = (nc[1] / nc[3]) / sy, fx = (nc[2] / nc[3]) / sx;
    T val = cval;
    if (fz >= 0.0 && fz < (double)d.dz - 1.0 && fy >= 0.0 && fy < (double)d.dy - 1.0 && fx >= 0.0 && fx < (double)d.dx - 1.0) {
      if (minterpol == 0) {
        val = vol[((long long)fz * d.dy + (long long)fy) * d.dx + (long long)fx];
      } else if (minterpol == 1) {
        const long long x0 = (long long)floor(fx), y0 = (long long)floor(fy), z0 = (long long)floor(fz);
        const double xd = fx - (double)x0, yd = fy - (double)y0, zd = fz - (double)z0;
        const double v000 = get_value(vol, d, x0, y0, z0), v100 = get_value(vol, d, x0 + 1, y0, z0),
                     v010 = get_value(vol, d, x0, y0 + 1, z0), v001 = get_value(vol, d, x0, y0, z0 + 1),
                     v110 = get_value(vol, d, x0 + 1, y0 + 1, z0), v101 = get_value(vol, d, x0 + 1, y0, z0 + 1),
                     v011 = get_value(vol, d, x0, y0 + 1, z0 + 1), v111 = get_value(vol, d, x0 + 1, y0 + 1, z0 + 1);
        const double c00 = v000 * (1.0 - xd) + v100 * xd, c10 = v010 * (1.0 - xd) + v110 * xd,
                     c01 = v001 * (1.0 - xd) + v101 * xd, c11 = v011 * (1.0 - xd) + v111 * xd;
        const double e0 = c00 * (1.0 - yd) + c10 * yd, e1 = c01 * (1.0 - yd) + c11 * yd;
        if (!cast_f64<T>(e0 * (1.0 - zd) + e1 * zd, &val)) { atomicOr(status, kStatusCast); val = 0; }
      } else if (minterpol == 2) {
        const long long xi = (long long)floor(fx), yi = (long long)floor(fy), zi = (long long)floor(fz);
        const double ty = fy - (double)yi, tz = fz - (double)zi;
        double rr[4];
        for (int a = 0; a < 4; ++a) {            // p[a][b][c] = value at (xi + a - 1, yi + b - 1, zi + c - 1)
          double arr[4];
          for (int b = 0; b < 4; ++b) {
            double p[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) p[c] = get_value(vol, d, xi + a - 1, yi + b - 1, zi + c - 1);
            arr[b] = cubic(p, tz);               // bicubic_interpolate(p[a], y - yi, z - zi): inner along its 2nd argument
          }
          rr[a] = cubic(arr, ty);
        }
        if (!cast_f64<T>(cubic(rr, fx - (double)xi), &val)) { atomicOr(status, kStatusCast); val = 0; }
        else if (val < cval) val = cval;
      } else {
        const int a = 4;
        const long long xd = (long long)floor(fx), yd = (long long)floor(fy), zd = (long long)floor(fz);
        const long long xi = xd - a + 1, yi = yd - a + 1, zi = zd - a + 1;
        if (!taps_wrap_inside(xi, xd + a - 1, d.dx) || !taps_wrap_inside(yi, yd + a - 1, d.dy) ||
            !taps_wrap_inside(zi, zd + a - 1, d.dz)) {
          atomicOr(status, kStatusIndex);
          out[i] = 0;
          continue;
        }
        double kx[7], ky[7], kz[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) {
          kx[k] = lanczos_kernel(fx - (double)(xi + k), a);
          ky[k] = lanczos_kernel(fy - (double)(yi + k), a);
          kz[k] = lanczos_kernel(fz - (double)(zi + k), a);
        }
        double lz = 0.0;
        for (int kk = 0; kk < 7; ++kk) {
          double ly = 0.0;
          for (int jj = 0; jj < 7; ++jj) {
            double lx = 0.0;
#pragma unroll
            for (int ii = 0; ii < 7; ++ii) lx += get_value(vol, d, xi + ii, yi + jj, zi + kk) * kx[ii];
            ly += lx * ky[jj];
          }
          lz += ly * kz[kk];
        }
        if (!cast_f64<T>(lz, &val)) { atomicOr(status, kStatusCast); val = 0; }
        else if (val < cval) val = cval;
      }
    }
    out[i] = val;
  }
}

template <typename T>
int run_view_transform(const void* vol, VDims d, const double* sp, const Mat4& M, long long n, int orientation,
                       int minterpol, double cval, void* out, VDims od, int* status, cudaStream_t s) {
  long long total = od.dz * od.dy * od.dx;
  long long blocks = ceil_div64(total, 256);
  long long cap = (long long)b2v_sm_count() * 32;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  k_view_transform<T><<<(unsigned)blocks, 256, 0, s>>>((const T*)vol, d, sp[0], sp[1], sp[2], M, n, orientation, minterpol,
                                                      (T)cval, (T*)out, od, status);
  return b2v_check_launch("k_view_transform");
}

}  // namespace

extern "C" int b2v_apply_view_matrix_transform(const void* volume, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                               const double* spacing_host, const double* m_host, int64_t n,
                                               int orientation, int minterpol, double cval, void* out, int64_t odz,
                                               int64_t ody, int64_t odx, void* workspace, void* stream) {
  B2V_REQUIRE(volume && out && spacing_host && m_host && workspace, B2V_ERR_ARG, "apply_view_matrix_transform: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0 && odz > 0 && ody > 0 && odx > 0 && n >= 0, B2V_ERR_ARG,
              "apply_view_matrix_transform: bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  int* status = (int*)workspace;
  B2V_CUDA(cudaMemsetAsync(status, 0, sizeof(int), s));
  Mat4 M;
  for (int k = 0; k < 16; ++k) M.m[k] = m_host[k];
  VDims d = {dz, dy, dx}, od = {odz, ody, odx};
  int rc;
  if (dtype == B2V_I16) rc = run_view_transform<int16_t>(volume, d, spacing_host, M, n, orientation, minterpol, cval, out, od, status, s);
  else if (dtype == B2V_U8) rc = run_view_transform<uint8_t>(volume, d, spacing_host, M, n, orientation, minterpol, cval, out, od, status, s);
  else if (dtype == B2V_F64) rc = run_view_transform<double>(volume, d, spacing_host, M, n, orientation, minterpol, cval, out, od, status, s);
  else B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid volume or output type");
  if (rc) return rc;
  int st = 0;
  B2V_CUDA(cudaMemcpyAsync(&st, status, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!(st & kStatusIndex), B2V_ERR_RANGE,
              "apply_view_matrix_transform: a Lanczos-4 tap lies outside the volume after the one-step wrap "
              "(an axis of 2 voxels): index out of bounds, the reference's ndarray indexing panics here");
  B2V_REQUIRE(st == 0, B2V_ERR_RANGE,
              "apply_view_matrix_transform: an interpolated value is not representable in the output type (the reference panics here)");
  return B2V_OK;
}
