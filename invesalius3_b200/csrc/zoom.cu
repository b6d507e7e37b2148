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
//   k_resample<T, ORDER>     one thread per output voxel, one output slice per grid row: coordinate o * step - off
//                            per axis, B-spline weights, taps folded by mirror, sum over the (ORDER + 1)^rank taps in
//                            row-major order, each value multiplied by the axis weights in axis order. SciPy's 3-D
//                            sum for volumes, its 2-D sum for a stack of slices, each slice with its own optional
//                            (y, x) offset. 'constant' mode writes cval at a coordinate outside [0, n - 1] (the
//                            last zoom sample's o * step can round just above n - 1), as SciPy does. Integer
//                            outputs round half away from zero and clip to the type's range.
//
// scipy.ndimage.shift(input, shift, output, order <= 3, mode) with prefilter=True shares SciPy's routine with zoom
// (zoom_shift): the same prefilter and the same gather, with coordinate o - shift per axis (step 1, off = shift)
// where zoom has o * step (off 0). Shift coordinates can be negative, so 'mirror' folds negative coordinates as
// SciPy's map_coordinate does; zoom coordinates never are, so that branch leaves zoom results unchanged.
//
// imagedata_utils.FixGantryTilt (imagedata_utils.py:143-154) shifts slice n of an int16 volume in place along y at
// order 3 with cval = matrix.min() of the partly shifted volume. b2v_gantry_tilt evaluates it without the
// sequential loop: cval[n] = min(min of original slices n.., min of shifted slices ..n-1), where a shifted slice's
// minimum is the minimum of its in-range outputs (independent of cval), lowered to cval[k] if it has out-of-range
// outputs (a property of its shift alone). So every slice is interpolated at once, then a scan over nz scalars
// gives the cvals, then the out-of-range outputs are filled.
//   k_slice_min_i16          per-slice minimum of the original volume, before any slice is overwritten
//   (prefilter, slab by slab) y then x passes over a slab of slices into a float64 workspace of the slab's size
//   k_resample<double, 3>    writes the in-range outputs in place, records per-slice in-range minima (warp
//                            min-reduce, one int atomicMin per warp: order-independent) and out-of-range flags
//   k_tilt_cval_chain        the scan over nz scalars (one thread)
//   k_tilt_fill              writes each slice's cval into its out-of-range outputs
#include <limits.h>
#include <math.h>

#include <algorithm>
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
// Output index o of an axis samples input coordinate o * step - off. Zoom sets off = 0 and step = (n_in - 1) /
// (n_out - 1); shift sets step = 1, off = shift and n_out = n_in. Both are exact in float64, so each keeps SciPy's
// coordinate bit for bit: x - 0.0 == x (+0 included), o * 1.0 == o, and the library builds with -fmad=false, so
// the multiply and the subtract are never fused.
struct Axis {
  int64_t n_in, n_out;
  double step, off;
};

struct ResampleParams {
  Axis ax[3];                // z, y, x; a stack of 2-D slices when rank3 is 0 (a 2-D zoom: one slice)
  const double* slice_off;   // stack of slices: per-slice (y, x) offsets on the device, or null (ax[1].off, ax[2].off)
  int rank3, mirror, out_dtype;
  double cval;
  // Stack of slices with int16 output (gantry tilt): out-of-range outputs are left unwritten; slice_min receives
  // the per-slice minimum of the in-range outputs and slice_out is set where a slice has an out-of-range output.
  int* slice_min;
  int* slice_out;
};

__device__ __forceinline__ int64_t fold_mirror(int64_t i, int64_t n) {
  if (n == 1) return 0;
  const int64_t p = 2 * n - 2;
  int64_t m = i % p;
  if (m < 0) m += p;
  return m >= n ? p - m : m;
}

// 'constant' mode writes cval at a coordinate outside [0, n - 1] (SciPy's test is strict on both sides)
__device__ __forceinline__ bool outside_axis(double cc, int64_t n) { return cc < 0.0 || cc > (double)(n - 1); }

// Weights and folded tap indices at coordinate cc of an axis of n_in samples; false where 'constant' mode writes
// cval.
template <int ORDER>
__device__ __forceinline__ bool taps_at(double cc, int64_t n_in, bool mirror, double* w, int64_t* idx) {
  if (outside_axis(cc, n_in)) {
    if (!mirror) return false;
    if (n_in == 1) {
      cc = 0.0;
    } else if (cc < 0.0) {   // SciPy's map_coordinate, in its operation order
      const int64_t p = 2 * n_in - 2;
      cc = (double)(p * (int64_t)(-cc / (double)p)) + cc;
      cc = cc <= (double)(1 - n_in) ? cc + (double)p : -cc;
    } else {
      const double p = (double)(2 * n_in - 2);
      cc -= p * (double)(int64_t)(cc / p);
      if (cc >= (double)n_in) cc = p - cc;
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
  for (int k = 0; k <= ORDER; ++k) idx[k] = fold_mirror(start + k, n_in);
  return true;
}

// Weights and folded tap indices of output index o along one axis, at offset off
template <int ORDER>
__device__ __forceinline__ bool axis_taps(const Axis& A, int64_t o, double off, bool mirror, double* w, int64_t* idx) {
  return taps_at<ORDER>((double)o * A.step - off, A.n_in, mirror, w, idx);
}

template <typename T>
__device__ __forceinline__ T round_clip(double t) {
  if (t > 0.0) t += 0.5;
  else t = (T)-1 < (T)0 ? t - 0.5 : 0.0;   // unsigned: everything up to 0 becomes 0
  const double lo = (double)((T)-1 < (T)0 ? (T)(1 << (8 * sizeof(T) - 1)) : (T)0);
  const double hi = (double)((T)-1 < (T)0 ? (T)((1 << (8 * sizeof(T) - 1)) - 1) : (T)-1);
  t = t > hi ? hi : t;
  t = t < lo ? lo : t;
  return (T)t;   // truncation
}

__device__ __forceinline__ void store_out(int out_dtype, void* out, int64_t i, double t) {
  switch (out_dtype) {
    case B2V_I16: ((int16_t*)out)[i] = round_clip<int16_t>(t); break;
    case B2V_U8: ((uint8_t*)out)[i] = round_clip<uint8_t>(t); break;
    case B2V_F32: ((float*)out)[i] = (float)t; break;
    default: ((double*)out)[i] = t; break;
  }
}

// Orders 0 and 1 are held to four blocks per SM (64 registers), which ptxas's own choice reaches only by spilling;
// a minimum of 0 leaves orders 2 and 3 to ptxas.
template <typename T, int ORDER>
__global__ void __launch_bounds__(256, ORDER < 2 ? 4 : 0) k_resample(const T* __restrict__ src, ResampleParams P,
                                                                    void* out) {
  const Axis &AZ = P.ax[0], &AY = P.ax[1], &AX = P.ax[2];
  const int64_t in_area = AY.n_in * AX.n_in, area = AY.n_out * AX.n_out;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int kz_taps = P.rank3 ? ORDER + 1 : 1;
  for (int64_t oz = blockIdx.y; oz < AZ.n_out; oz += gridDim.y) {   // uniform across the block
    double wz[ORDER + 1];
    int64_t iz[ORDER + 1];
    bool z_inside = true;
    double offy = AY.off, offx = AX.off;
    const T* plane = src;
    iz[0] = 0;
    if (P.rank3) {
      z_inside = axis_taps<ORDER>(AZ, oz, AZ.off, P.mirror, wz, iz);
    } else {
      plane = src + oz * in_area;
      if (P.slice_off) {
        offy = P.slice_off[2 * oz];
        offx = P.slice_off[2 * oz + 1];
      }
    }
    int vmin = INT_MAX;
    bool any_out = false;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < area; i += stride) {
      const int64_t ox = i % AX.n_out, oy = i / AX.n_out, o = oz * area + i;
      double wy[ORDER + 1], wx[ORDER + 1];
      int64_t iy[ORDER + 1], ix[ORDER + 1];
      const bool inside = z_inside && axis_taps<ORDER>(AY, oy, offy, P.mirror, wy, iy) &&
                          axis_taps<ORDER>(AX, ox, offx, P.mirror, wx, ix);
      if (!inside) {
        if (P.slice_min) any_out = true;
        else store_out(P.out_dtype, out, o, P.cval);
        continue;
      }
      double t = 0.0;
#pragma unroll
      for (int a = 0; a <= ORDER; ++a) {
        if (a == kz_taps) break;
        const T* pz = plane + iz[a] * in_area;
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
      if (P.slice_min) {
        const int16_t r = round_clip<int16_t>(t);
        ((int16_t*)out)[o] = r;
        vmin = min(vmin, (int)r);
      } else {
        store_out(P.out_dtype, out, o, t);
      }
    }
    if (P.slice_min) {
      vmin = __reduce_min_sync(0xffffffffu, vmin);
      any_out = __any_sync(0xffffffffu, any_out);
      if ((threadIdx.x & 31) == 0) {
        atomicMin(P.slice_min + oz, vmin);
        if (any_out) P.slice_out[oz] = 1;
      }
    }
  }
}

// per-slice minimum of a [nz][area] int16 volume into slice_min (initialised above every int16)
__global__ void __launch_bounds__(256) k_slice_min_i16(const int16_t* __restrict__ vol, int64_t nz, int64_t area,
                                                       int* slice_min) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t oz = blockIdx.y; oz < nz; oz += gridDim.y) {
    int vmin = INT_MAX;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < area; i += stride)
      vmin = min(vmin, (int)vol[oz * area + i]);
    vmin = __reduce_min_sync(0xffffffffu, vmin);
    if ((threadIdx.x & 31) == 0) atomicMin(slice_min + oz, vmin);
  }
}

// cval[n] = min(min of original slices n.., min of shifted slices ..n-1), where shifted slice k's minimum is its
// in-range minimum, lowered to cval[k] if it has out-of-range outputs. One thread: nz scalars.
__global__ void k_tilt_cval_chain(int64_t nz, const int* orig_min, const int* inrange_min, const int* slice_out,
                                  int* cval, int16_t* cval_out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int suffix = INT_MAX;
  for (int64_t n = nz - 1; n >= 0; --n) {
    suffix = min(suffix, orig_min[n]);
    cval[n] = suffix;
  }
  int shifted = INT_MAX;
  for (int64_t n = 0; n < nz; ++n) {
    const int c = min(cval[n], shifted);
    cval[n] = c;
    if (cval_out) cval_out[n] = (int16_t)c;
    shifted = min(shifted, slice_out[n] ? min(inrange_min[n], c) : inrange_min[n]);
  }
}

// writes cval[z] into the outputs of slice z whose coordinate is outside the input (the gather's test)
__global__ void __launch_bounds__(256) k_tilt_fill(int16_t* vol, int64_t nz, int64_t ny, int64_t nx,
                                                   const double* slice_shift, const int* slice_out, const int* cval) {
  const int64_t area = ny * nx, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t oz = blockIdx.y; oz < nz; oz += gridDim.y) {
    if (!slice_out[oz]) continue;
    const double sy = slice_shift[2 * oz], sx = slice_shift[2 * oz + 1];
    const int16_t c = (int16_t)cval[oz];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < area; i += stride) {
      const int64_t ox = i % nx, oy = i / nx;
      if (outside_axis((double)oy - sy, ny) || outside_axis((double)ox - sx, nx)) vol[oz * area + i] = c;
    }
  }
}

// one grid row per slice (grid-stride beyond 65535 slices), blocks across the slice
dim3 slice_grid(int64_t nz, int64_t area) {
  return dim3((unsigned)std::min<int64_t>(ceil_div64(area, 256), 1024), (unsigned)std::min<int64_t>(nz, 65535));
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

// first prefilter pass: input dtype -> float64 along lines of length n, stride `inner`
template <typename T>
int prefilter_first(const void* in, double* ws, int64_t n, int64_t inner, int64_t nlines, int order, cudaStream_t s) {
  k_prefilter_strided<T><<<(unsigned)ceil_div64(nlines, 256), 256, 0, s>>>((const T*)in, ws, n, inner, nlines,
                                                                           make_pole(order, n));
  return b2v_check_launch("k_prefilter_strided");
}

int prefilter_rows(double* ws, int64_t nx, int64_t nrows, int order, cudaStream_t s) {
  if (nx == 1) return B2V_OK;
  k_prefilter_rows<<<(unsigned)ceil_div64(nrows, 32 * kRowWarps), 32 * kRowWarps, 0, s>>>(ws, nx, nrows,
                                                                                          make_pole(order, nx));
  return b2v_check_launch("k_prefilter_rows");
}

// spline_filter(in, order, float64) of a [nz][ny][nx] volume into ws, axes z, y, x (nz = 1: a 2-D image)
int prefilter_volume(const void* in, int in_dtype, int64_t nz, int64_t ny, int64_t nx, int order, double* ws,
                     cudaStream_t s) {
  int rc;
  switch (in_dtype) {   // z pass: input dtype -> float64
    case B2V_I16: rc = prefilter_first<int16_t>(in, ws, nz, ny * nx, ny * nx, order, s); break;
    case B2V_U8: rc = prefilter_first<uint8_t>(in, ws, nz, ny * nx, ny * nx, order, s); break;
    case B2V_F32: rc = prefilter_first<float>(in, ws, nz, ny * nx, ny * nx, order, s); break;
    default: rc = prefilter_first<double>(in, ws, nz, ny * nx, ny * nx, order, s); break;
  }
  if (rc) return rc;
  if (ny > 1) {
    const int64_t nlines = nz * nx;
    k_prefilter_strided<double><<<(unsigned)ceil_div64(nlines, 256), 256, 0, s>>>(ws, ws, ny, nx, nlines,
                                                                                 make_pole(order, ny));
    if ((rc = b2v_check_launch("k_prefilter_strided"))) return rc;
  }
  return prefilter_rows(ws, nx, nz * ny, order, s);
}

// One grid row per output slice, and across the rows about as many blocks as a grid-stride launch over every
// output takes: a thread then loops over several outputs of its slice, which spreads its set-up over them.
template <typename T, int ORDER>
int resample_launch(const void* src, const ResampleParams& P, void* out, cudaStream_t s) {
  const int64_t nz = P.ax[0].n_out, rows = std::min<int64_t>(nz, 65535);
  const int blocks = b2v_grid(nz * P.ax[1].n_out * P.ax[2].n_out, 256, 64);
  k_resample<T, ORDER><<<dim3((unsigned)ceil_div64(blocks, rows), (unsigned)rows), 256, 0, s>>>((const T*)src, P, out);
  return b2v_check_launch("k_resample");
}

// orders 2 and 3 gather from the float64 prefilter output only
template <typename T>
int resample_order(const void* src, int order, const ResampleParams& P, void* out, cudaStream_t s) {
  if constexpr (std::is_same<T, double>::value) {
    if (order == 2) return resample_launch<T, 2>(src, P, out, s);
    if (order == 3) return resample_launch<T, 3>(src, P, out, s);
  }
  return order == 0 ? resample_launch<T, 0>(src, P, out, s) : resample_launch<T, 1>(src, P, out, s);
}

// zoom and shift once their arguments are checked and P's axes filled in: the prefilter into the workspace at
// orders 2 and 3, then the gather from the input's dtype or from the float64 workspace
int resample(const void* in, int in_dtype, int order, const ResampleParams& P, void* out, void* workspace,
             cudaStream_t s) {
  if (order >= 2) {
    const int rc =
        prefilter_volume(in, in_dtype, P.ax[0].n_in, P.ax[1].n_in, P.ax[2].n_in, order, (double*)workspace, s);
    if (rc) return rc;
    return resample_order<double>(workspace, order, P, out, s);
  }
  switch (in_dtype) {
    case B2V_I16: return resample_order<int16_t>(in, order, P, out, s);
    case B2V_U8: return resample_order<uint8_t>(in, order, P, out, s);
    case B2V_F32: return resample_order<float>(in, order, P, out, s);
    default: return resample_order<double>(in, order, P, out, s);
  }
}

constexpr int64_t kTiltSlabBytes = int64_t(1) << 30;   // default float64 workspace of the gantry-tilt slab

int64_t tilt_slab(int64_t nz, int64_t ny, int64_t nx, int64_t slab) {
  if (slab <= 0) slab = std::max<int64_t>(1, kTiltSlabBytes / (ny * nx * (int64_t)sizeof(double)));
  return std::min(slab, nz);
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

  ResampleParams P = {};
  const int64_t n_in[3] = {nz, ny, nx}, n_out[3] = {out_nz, out_ny, out_nx};
  for (int a = 0; a < 3; ++a) {
    const double step = n_out[a] > 1 ? (double)(n_in[a] - 1) / (double)(n_out[a] - 1) : 1.0;
    P.ax[a] = {n_in[a], n_out[a], step, 0.0};
  }
  P.rank3 = ndim == 3;
  P.mirror = mode == B2V_ZOOM_MIRROR;
  P.out_dtype = out_dtype;
  P.cval = cval;
  return resample(in, in_dtype, order, P, out, workspace, (cudaStream_t)stream);
}

extern "C" int64_t b2v_shift_workspace_bytes(int64_t nz, int64_t ny, int64_t nx, int order) {
  return b2v_zoom_workspace_bytes(nz, ny, nx, order);
}

extern "C" int b2v_shift(const void* in, int in_dtype, int ndim, int64_t nz, int64_t ny, int64_t nx,
                         const double* shift, int order, int mode, double cval, void* out, int out_dtype,
                         void* workspace, void* stream) {
  B2V_REQUIRE(dtype_size(in_dtype) && dtype_size(out_dtype), B2V_ERR_ARG, "shift: bad dtype code (%d, %d)",
              in_dtype, out_dtype);
  B2V_REQUIRE(order >= 0 && order <= 3, B2V_ERR_ARG, "shift: spline order %d not built (0-3)", order);
  B2V_REQUIRE(mode == B2V_ZOOM_CONSTANT || mode == B2V_ZOOM_MIRROR, B2V_ERR_ARG, "shift: bad mode %d", mode);
  B2V_REQUIRE(ndim == 2 || ndim == 3, B2V_ERR_ARG, "shift: ndim must be 2 or 3");
  B2V_REQUIRE(ndim == 3 || nz == 1, B2V_ERR_ARG, "shift: a 2-D shift takes nz = 1");
  B2V_REQUIRE(nz >= 0 && ny >= 0 && nx >= 0, B2V_ERR_ARG, "shift: negative size");
  if (nz * ny * nx == 0) return B2V_OK;
  B2V_REQUIRE(in && out && shift, B2V_ERR_ARG, "shift: null pointer");
  B2V_REQUIRE(in != out, B2V_ERR_ARG, "shift: the output must not be the input");
  B2V_REQUIRE(order < 2 || workspace, B2V_ERR_ARG, "shift: orders 2 and 3 need the workspace");

  ResampleParams P = {};
  const int64_t n[3] = {nz, ny, nx};
  const double off[3] = {ndim == 3 ? shift[0] : 0.0, shift[ndim - 2], shift[ndim - 1]};
  for (int a = 0; a < 3; ++a) P.ax[a] = {n[a], n[a], 1.0, off[a]};
  P.rank3 = ndim == 3;
  P.mirror = mode == B2V_ZOOM_MIRROR;
  P.out_dtype = out_dtype;
  P.cval = cval;
  return resample(in, in_dtype, order, P, out, workspace, (cudaStream_t)stream);
}

// workspace: [slab][ny][nx] float64 coefficients, nz (y, x) shifts, then four int arrays of nz
extern "C" int64_t b2v_gantry_tilt_workspace_bytes(int64_t nz, int64_t ny, int64_t nx, int64_t slab) {
  if (nz <= 0 || ny <= 0 || nx <= 0) return 0;
  return tilt_slab(nz, ny, nx, slab) * ny * nx * (int64_t)sizeof(double) + nz * 2 * (int64_t)sizeof(double) +
         nz * 4 * (int64_t)sizeof(int);
}

extern "C" int b2v_gantry_tilt(int16_t* vol, int64_t nz, int64_t ny, int64_t nx, const double* shifts, int64_t slab,
                               void* workspace, int16_t* cvals, void* stream) {
  B2V_REQUIRE(nz >= 0 && ny >= 0 && nx >= 0, B2V_ERR_ARG, "gantry_tilt: negative size");
  if (nz * ny * nx == 0) return B2V_OK;
  B2V_REQUIRE(vol && shifts && workspace, B2V_ERR_ARG, "gantry_tilt: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t area = ny * nx;
  slab = tilt_slab(nz, ny, nx, slab);
  double* ws = (double*)workspace;
  double* d_shift = ws + slab * area;
  int* orig_min = (int*)(d_shift + 2 * nz);
  int* inrange_min = orig_min + nz;
  int* slice_out = inrange_min + nz;
  int* cval = slice_out + nz;

  cudaError_t e = cudaMemcpyAsync(d_shift, shifts, nz * 2 * sizeof(double), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(orig_min, 0x7f, nz * 2 * sizeof(int), s);   // above every int16
  if (e == cudaSuccess) e = cudaMemsetAsync(slice_out, 0, nz * sizeof(int), s);
  B2V_REQUIRE(e == cudaSuccess, B2V_ERR_CUDA, "gantry_tilt: %s", cudaGetErrorString(e));
  int rc;
  k_slice_min_i16<<<slice_grid(nz, area), 256, 0, s>>>(vol, nz, area, orig_min);
  if ((rc = b2v_check_launch("k_slice_min_i16"))) return rc;

  ResampleParams P = {};
  P.ax[1] = {ny, ny, 1.0, 0.0};
  P.ax[2] = {nx, nx, 1.0, 0.0};
  P.out_dtype = B2V_I16;
  for (int64_t z0 = 0; z0 < nz; z0 += slab) {
    const int64_t n = std::min(slab, nz - z0);
    int16_t* sv = vol + z0 * area;   // the slab's slices are read by the prefilter before the gather overwrites them
    if ((rc = prefilter_first<int16_t>(sv, ws, ny, nx, n * nx, 3, s))) return rc;
    if ((rc = prefilter_rows(ws, nx, n * ny, 3, s))) return rc;
    P.ax[0] = {n, n, 1.0, 0.0};
    P.slice_off = d_shift + 2 * z0;
    P.slice_min = inrange_min + z0;
    P.slice_out = slice_out + z0;
    if ((rc = resample_launch<double, 3>(ws, P, sv, s))) return rc;
  }
  k_tilt_cval_chain<<<1, 32, 0, s>>>(nz, orig_min, inrange_min, slice_out, cval, cvals);
  if ((rc = b2v_check_launch("k_tilt_cval_chain"))) return rc;
  k_tilt_fill<<<slice_grid(nz, area), 256, 0, s>>>(vol, nz, ny, nx, d_shift, slice_out, cval);
  return b2v_check_launch("k_tilt_fill");
}

