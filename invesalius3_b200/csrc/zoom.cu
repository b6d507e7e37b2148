// scipy.ndimage.zoom(input, zoom, output, order <= 3, mode 'constant' | 'mirror') with prefilter=True and
// grid_mode=False: the resample behind imagedata_utils.resize_image_array / resize_slice (imagedata_utils.py:109-139)
// and the thumbnails (:271-284). Bit-exact against SciPy: every step is float64 in SciPy's evaluation order, no FMA
// (the library builds with -fmad=false).
//
//   prefilter (orders 2, 3)  spline_filter(input, order, float64, mode): per axis, in axis order z, y, x, each line
//                            runs gain, causal init (mirror boundary), forward recursion, anticausal init, backward
//                            recursion. The gain is applied where a sample is read (g * c[i] is the value SciPy
//                            stores before the recursions), so a line costs three reads and two writes.
//     k_prefilter_strided<T> z and y axes: one thread per line; neighbouring threads hold neighbouring x lines, so
//                            every access of a warp is coalesced. The z pass reads the input dtype and writes the
//                            float64 workspace; the y pass works in place.
//     k_prefilter_rows       x axis: one warp per 32 rows. Rows move through shared memory in 32 x 16 tiles (two rows
//                            of 128 bytes per load), each lane walks its row inside the tile.
//   k_zoom_gather<T, ORDER>  one thread per output voxel: coordinate o * step per axis, B-spline weights, taps folded
//                            by mirror, sum over the (ORDER + 1)^rank taps in row-major order, each value multiplied
//                            by the axis weights in axis order. In 'constant' mode a coordinate past n - 1 (the last
//                            sample's o * step can round just above it) writes cval, as SciPy does. Integer outputs
//                            round half away from zero and clip to the type's range.
#include <math.h>

#include <type_traits>

#include "b2v_common.cuh"

namespace {

// sqrt(8) - 3 and sqrt(3) - 2, correctly rounded (SciPy's constants; computing them in float64 loses 7 and 2 ulps)
constexpr double kPole2 = -0.171572875253809902396622551580603843;
constexpr double kPole3 = -0.267949192431122706472553658494127633;

struct Pole {
  double z, gain, zn1;   // zn1 = z^(n - 1) for the axis' line length n (host libm pow, as SciPy computes it)
};

template <typename T>
__device__ __forceinline__ double to_f64(T v) { return (double)v; }

// ---- prefilter: z and y axes --------------------------------------------------------------------
// Line L starts at (L / inner) * n * inner + L % inner and steps by `inner` (the product of the later dims).
template <typename T>
__global__ void __launch_bounds__(256) k_prefilter_strided(const T* src, double* dst, int64_t n,
                                                           int64_t inner, int64_t nlines, Pole P) {
  const int64_t L = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (L >= nlines) return;
  const int64_t base = (L / inner) * n * inner + L % inner;
  const T* s = src + base;
  double* d = dst + base;
  if (n == 1) {
    d[0] = to_f64(s[0]);
    return;
  }
  const double z = P.z, g = P.gain, zn1 = P.zn1;
  double c0 = g * to_f64(s[0]) + zn1 * (g * to_f64(s[(n - 1) * inner]));
  double zi = z;
  for (int64_t i = 1; i < n - 1; ++i) {
    c0 += zi * (g * to_f64(s[i * inner]) + zn1 * (g * to_f64(s[(n - 1 - i) * inner])));
    zi *= z;
  }
  c0 /= 1.0 - zn1 * zn1;
  // `src` may alias `dst` (in place): sample j is read before it is written, and only by this thread
  double prev2 = 0.0, prev = c0;
  d[0] = c0;
  for (int64_t j = 1; j < n; ++j) {
    const double v = g * to_f64(s[j * inner]) + z * prev;
    d[j * inner] = v;
    prev2 = prev;
    prev = v;
  }
  double next = (z * prev2 + prev) * z / (z * z - 1.0);
  d[(n - 1) * inner] = next;
  for (int64_t j = n - 2; j >= 0; --j) {
    next = z * (next - d[j * inner]);
    d[j * inner] = next;
  }
}

// ---- prefilter: x axis (contiguous rows) ----------------------------------------------------------
constexpr int kRowWarps = 4;
constexpr int kCols = 16;   // tile width: 16 doubles = 128 bytes per row segment

// tile[r][k] <- row (row0 + r), column (col0 + k); out-of-range entries are left as they are
__device__ __forceinline__ void tile_load(double (*tile)[kCols + 1], const double* c, int64_t row0, int64_t nrows,
                                          int64_t n, int64_t col0, int lane) {
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int r = 2 * k + (lane >> 4), col = lane & 15;
    const int64_t x = col0 + col;
    if (row0 + r < nrows && x >= 0 && x < n) tile[r][col] = c[(row0 + r) * n + x];
  }
  __syncwarp();
}

__device__ __forceinline__ void tile_store(double (*tile)[kCols + 1], double* c, int64_t row0, int64_t nrows, int64_t n,
                                           int64_t col0, int lane) {
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int r = 2 * k + (lane >> 4), col = lane & 15;
    const int64_t x = col0 + col;
    if (row0 + r < nrows && x >= 0 && x < n) c[(row0 + r) * n + x] = tile[r][col];
  }
  __syncwarp();
}

__global__ void __launch_bounds__(32 * kRowWarps) k_prefilter_rows(double* c, int64_t n, int64_t nrows, Pole P) {
  __shared__ double s_a[kRowWarps][32][kCols + 1];
  __shared__ double s_b[kRowWarps][32][kCols + 1];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t row0 = ((int64_t)blockIdx.x * kRowWarps + w) * 32;
  if (row0 >= nrows) return;   // whole warps only: the tiles are per warp
  double(*A)[kCols + 1] = s_a[w];
  double(*B)[kCols + 1] = s_b[w];
  const double z = P.z, g = P.gain, zn1 = P.zn1;

  // causal init: sample i pairs with sample n - 1 - i, so tile B holds the mirrored columns of tile A
  tile_load(A, c, row0, nrows, n, 0, lane);
  tile_load(B, c, row0, nrows, n, n - kCols, lane);
  double c0 = g * A[lane][0] + zn1 * (g * B[lane][kCols - 1]);
  double zi = z;
  for (int64_t i0 = 0; i0 < n; i0 += kCols) {
    if (i0 > 0) {
      __syncwarp();
      tile_load(A, c, row0, nrows, n, i0, lane);
      tile_load(B, c, row0, nrows, n, n - i0 - kCols, lane);
    }
    for (int k = 0; k < kCols; ++k) {
      const int64_t i = i0 + k;
      if (i >= 1 && i < n - 1) {
        c0 += zi * (g * A[lane][k] + zn1 * (g * B[lane][kCols - 1 - k]));
        zi *= z;
      }
    }
  }
  c0 /= 1.0 - zn1 * zn1;

  // forward recursion
  double prev2 = 0.0, prev = c0;
  for (int64_t i0 = 0; i0 < n; i0 += kCols) {
    __syncwarp();
    tile_load(A, c, row0, nrows, n, i0, lane);
    for (int k = 0; k < kCols; ++k) {
      const int64_t j = i0 + k;
      if (j == 0) {
        A[lane][0] = c0;
      } else if (j < n) {
        const double v = g * A[lane][k] + z * prev;
        A[lane][k] = v;
        prev2 = prev;
        prev = v;
      }
    }
    tile_store(A, c, row0, nrows, n, i0, lane);
  }

  // anticausal init and backward recursion, last tile first
  double next = (z * prev2 + prev) * z / (z * z - 1.0);
  for (int64_t i0 = ((n - 1) / kCols) * kCols; i0 >= 0; i0 -= kCols) {
    tile_load(A, c, row0, nrows, n, i0, lane);
    for (int k = kCols - 1; k >= 0; --k) {
      const int64_t j = i0 + k;
      if (j == n - 1) {
        A[lane][k] = next;
      } else if (j < n - 1) {
        next = z * (next - A[lane][k]);
        A[lane][k] = next;
      }
    }
    tile_store(A, c, row0, nrows, n, i0, lane);
  }
}

// ---- gather ---------------------------------------------------------------------------------------
struct Axis {
  int64_t n_in, n_out;
  double step;   // (n_in - 1) / (n_out - 1), or 1 when n_out == 1
};

struct GatherParams {
  Axis ax[3];    // z, y, x; a 2-D zoom leaves the z axis unused
  int rank3, mirror, out_dtype;
  double cval;
};

__device__ __forceinline__ int64_t fold_mirror(int64_t i, int64_t n) {
  if (n == 1) return 0;
  const int64_t p = 2 * n - 2;
  int64_t m = i % p;
  if (m < 0) m += p;
  return m >= n ? p - m : m;
}

// Coordinate, weights and folded tap indices of output index o along one axis; false where 'constant' mode
// writes cval.
template <int ORDER>
__device__ __forceinline__ bool axis_taps(const Axis& A, int64_t o, bool mirror, double* w, int64_t* idx) {
  double cc = (double)o * A.step;
  if (cc > (double)(A.n_in - 1)) {
    if (!mirror) return false;
    if (A.n_in == 1) {
      cc = 0.0;
    } else {
      const double p = (double)(2 * A.n_in - 2);
      cc -= p * (double)(int64_t)(cc / p);
      if (cc >= (double)A.n_in) cc = p - cc;
    }
  }
  const double f = (ORDER & 1) ? floor(cc) : floor(cc + 0.5);
  const double t = cc - f;
  if (ORDER == 1) {
    w[0] = 1.0 - t;
  } else if (ORDER == 2) {
    w[1] = 0.75 - t * t;
    const double h = 0.5 - t;
    w[0] = 0.5 * h * h;
  } else if (ORDER == 3) {
    const double u = 1.0 - t;
    w[0] = u * u * u / 6.0;
    w[1] = (t * t * (t - 2.0) * 3.0 + 4.0) / 6.0;
    w[2] = (u * u * (u - 2.0) * 3.0 + 4.0) / 6.0;
  }
  double last = 1.0;   // the weights sum to one: the last is what the others leave, subtracted in order
#pragma unroll
  for (int k = 0; k < ORDER; ++k) last -= w[k];
  w[ORDER] = last;
  const int64_t start = (int64_t)f - ORDER / 2;
#pragma unroll
  for (int k = 0; k <= ORDER; ++k) idx[k] = fold_mirror(start + k, A.n_in);
  return true;
}

template <typename T>
__device__ __forceinline__ void store_rounded(void* out, int64_t i, double t) {
  if (t > 0.0) t += 0.5;
  else t = (T)-1 < (T)0 ? t - 0.5 : 0.0;   // unsigned: everything up to 0 becomes 0
  const double lo = (double)((T)-1 < (T)0 ? (T)(1 << (8 * sizeof(T) - 1)) : (T)0);
  const double hi = (double)((T)-1 < (T)0 ? (T)((1 << (8 * sizeof(T) - 1)) - 1) : (T)-1);
  t = t > hi ? hi : t;
  t = t < lo ? lo : t;
  ((T*)out)[i] = (T)t;   // truncation
}

template <typename T, int ORDER>
__global__ void __launch_bounds__(256) k_zoom_gather(const T* __restrict__ src, GatherParams P, void* out) {
  const Axis &AZ = P.ax[0], &AY = P.ax[1], &AX = P.ax[2];
  const int64_t total = AZ.n_out * AY.n_out * AX.n_out;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int kz_taps = P.rank3 ? ORDER + 1 : 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t ox = i % AX.n_out, r = i / AX.n_out, oy = r % AY.n_out, oz = r / AY.n_out;
    double wz[ORDER + 1], wy[ORDER + 1], wx[ORDER + 1];
    int64_t iz[ORDER + 1], iy[ORDER + 1], ix[ORDER + 1];
    bool inside = axis_taps<ORDER>(AY, oy, P.mirror, wy, iy) && axis_taps<ORDER>(AX, ox, P.mirror, wx, ix);
    if (P.rank3) {
      inside = axis_taps<ORDER>(AZ, oz, P.mirror, wz, iz) && inside;
    } else {
      iz[0] = 0;
    }
    double t = P.cval;
    if (inside) {
      t = 0.0;
#pragma unroll
      for (int a = 0; a <= ORDER; ++a) {
        if (a == kz_taps) break;
        const T* pz = src + iz[a] * AY.n_in * AX.n_in;
#pragma unroll
        for (int b = 0; b <= ORDER; ++b) {
          const T* py = pz + iy[b] * AX.n_in;
#pragma unroll
          for (int c = 0; c <= ORDER; ++c) {
            double v = to_f64(py[ix[c]]);
            if (ORDER > 0) {
              if (P.rank3) v *= wz[a];
              v *= wy[b];
              v *= wx[c];
            }
            t += v;
          }
        }
      }
    }
    switch (P.out_dtype) {
      case B2V_I16: store_rounded<int16_t>(out, i, t); break;
      case B2V_U8: store_rounded<uint8_t>(out, i, t); break;
      case B2V_F32: ((float*)out)[i] = (float)t; break;
      default: ((double*)out)[i] = t; break;
    }
  }
}

int dtype_size(int dtype) {
  switch (dtype) {
    case B2V_I16: return 2;
    case B2V_U8: return 1;
    case B2V_F32: return 4;
    case B2V_F64: return 8;
    default: return 0;
  }
}

Pole make_pole(int order, int64_t n) {
  Pole P;
  P.z = order == 2 ? kPole2 : kPole3;
  P.gain = (1.0 - P.z) * (1.0 - 1.0 / P.z);
  P.zn1 = pow(P.z, (double)(n - 1));
  return P;
}

template <typename T>
int prefilter_first(const void* in, double* ws, int64_t n, int64_t inner, int order, cudaStream_t s) {
  const int64_t nlines = inner;
  k_prefilter_strided<T><<<(unsigned)ceil_div64(nlines, 256), 256, 0, s>>>((const T*)in, ws, n, inner, nlines,
                                                                           make_pole(order, n));
  return b2v_check_launch("k_prefilter_strided");
}

template <typename T, int ORDER>
int gather_launch(const void* src, const GatherParams& P, void* out, cudaStream_t s) {
  const int64_t total = P.ax[0].n_out * P.ax[1].n_out * P.ax[2].n_out;
  int64_t blocks = ceil_div64(total, 256);
  const int64_t cap = (int64_t)b2v_sm_count() * 16;
  if (blocks > cap) blocks = cap;
  k_zoom_gather<T, ORDER><<<(unsigned)blocks, 256, 0, s>>>((const T*)src, P, out);
  return b2v_check_launch("k_zoom_gather");
}

// orders 2 and 3 gather from the float64 prefilter output only
template <typename T>
int gather_order(const void* src, int order, const GatherParams& P, void* out, cudaStream_t s) {
  if constexpr (std::is_same<T, double>::value) {
    if (order == 2) return gather_launch<T, 2>(src, P, out, s);
    if (order == 3) return gather_launch<T, 3>(src, P, out, s);
  }
  return order == 0 ? gather_launch<T, 0>(src, P, out, s) : gather_launch<T, 1>(src, P, out, s);
}

}  // namespace

extern "C" int64_t b2v_zoom_workspace_bytes(int64_t nz, int64_t ny, int64_t nx, int order) {
  if (order < 2 || nz < 0 || ny < 0 || nx < 0) return 0;
  return nz * ny * nx * (int64_t)sizeof(double);
}

extern "C" int b2v_zoom(const void* in, int in_dtype, int ndim, int64_t nz, int64_t ny, int64_t nx, int64_t out_nz,
                        int64_t out_ny, int64_t out_nx, int order, int mode, double cval, void* out, int out_dtype,
                        void* workspace, void* stream) {
  B2V_REQUIRE(dtype_size(in_dtype) && dtype_size(out_dtype), B2V_ERR_ARG, "zoom: bad dtype code (%d, %d)", in_dtype,
              out_dtype);
  B2V_REQUIRE(order >= 0 && order <= 3, B2V_ERR_ARG, "zoom: spline order %d not built (0-3)", order);
  B2V_REQUIRE(mode == B2V_ZOOM_CONSTANT || mode == B2V_ZOOM_MIRROR, B2V_ERR_ARG, "zoom: bad mode %d", mode);
  B2V_REQUIRE(ndim == 2 || ndim == 3, B2V_ERR_ARG, "zoom: ndim must be 2 or 3");
  B2V_REQUIRE(ndim == 3 || (nz == 1 && out_nz == 1), B2V_ERR_ARG, "zoom: a 2-D zoom takes nz = out_nz = 1");
  B2V_REQUIRE(nz >= 1 && ny >= 1 && nx >= 1, B2V_ERR_ARG, "zoom: empty input");
  B2V_REQUIRE(out_nz >= 0 && out_ny >= 0 && out_nx >= 0, B2V_ERR_ARG, "zoom: negative output size");
  if (out_nz * out_ny * out_nx == 0) return B2V_OK;
  B2V_REQUIRE(in && out, B2V_ERR_ARG, "zoom: null pointer");
  B2V_REQUIRE(order < 2 || workspace, B2V_ERR_ARG, "zoom: orders 2 and 3 need the workspace");
  cudaStream_t s = (cudaStream_t)stream;

  const void* src = in;
  int src_dtype = in_dtype;
  if (order >= 2) {
    double* ws = (double*)workspace;
    int rc;
    switch (in_dtype) {   // z pass: input dtype -> float64
      case B2V_I16: rc = prefilter_first<int16_t>(in, ws, nz, ny * nx, order, s); break;
      case B2V_U8: rc = prefilter_first<uint8_t>(in, ws, nz, ny * nx, order, s); break;
      case B2V_F32: rc = prefilter_first<float>(in, ws, nz, ny * nx, order, s); break;
      default: rc = prefilter_first<double>(in, ws, nz, ny * nx, order, s); break;
    }
    if (rc) return rc;
    if (ny > 1) {
      const int64_t nlines = nz * nx;
      k_prefilter_strided<double><<<(unsigned)ceil_div64(nlines, 256), 256, 0, s>>>(ws, ws, ny, nx, nlines,
                                                                                   make_pole(order, ny));
      if ((rc = b2v_check_launch("k_prefilter_strided"))) return rc;
    }
    if (nx > 1) {
      const int64_t nrows = nz * ny;
      k_prefilter_rows<<<(unsigned)ceil_div64(nrows, 32 * kRowWarps), 32 * kRowWarps, 0, s>>>(ws, nx, nrows,
                                                                                              make_pole(order, nx));
      if ((rc = b2v_check_launch("k_prefilter_rows"))) return rc;
    }
    src = ws;
    src_dtype = B2V_F64;
  }

  GatherParams P;
  const int64_t n_in[3] = {nz, ny, nx}, n_out[3] = {out_nz, out_ny, out_nx};
  for (int a = 0; a < 3; ++a) {
    P.ax[a].n_in = n_in[a];
    P.ax[a].n_out = n_out[a];
    P.ax[a].step = n_out[a] > 1 ? (double)(n_in[a] - 1) / (double)(n_out[a] - 1) : 1.0;
  }
  P.rank3 = ndim == 3;
  P.mirror = mode == B2V_ZOOM_MIRROR;
  P.out_dtype = out_dtype;
  P.cval = cval;
  switch (src_dtype) {
    case B2V_I16: return gather_order<int16_t>(src, order, P, out, s);
    case B2V_U8: return gather_order<uint8_t>(src, order, P, out, s);
    case B2V_F32: return gather_order<float>(src, order, P, out, s);
    default: return gather_order<double>(src, order, P, out, s);
  }
}
