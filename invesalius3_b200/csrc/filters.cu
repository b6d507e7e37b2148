// Whole-volume pre-filters and mask algebra (SURVEY 8f-4): the step before threshold
// (invesalius/data/filters.py:5-66 driven by slice_.py:2330-2432) and elementwise mask operations.
//   b2v_boolean_op          Slice.do_boolean_op                   slice_.py:1906-1916
//   b2v_convolve_non_zero   invesalius_rs.convolve_non_zero       transforms_py.rs:52-93 (calc_mask_area, slice_.py:2299-2322)
//   b2v_median_filter_i16   ndimage.median_filter(matrix, size)   filters.py:9-12 (size 3, 4 or 5, mode 'reflect')
//   b2v_uniform_filter_i16  ndimage.uniform_filter(matrix, size)  filters.py:15-18 (separable; every pass stores
//                           trunc(sum / size) in int16 like SciPy's NI_UniformFilter1D writing into an int16 output)
//   *_slices_i16, b2v_slice_minmax  the "2D" branch of slice_.py:2363-2422: every slice along one axis filtered in
//                           the same launches, no pass along the slice axis, per-slice statistics on the device
//   b2v_histogram_i16       np.histogram(matrix, max - min, (min, max))   slice_.py:190-192, 2490-2493
// All integer results are bit-exact against SciPy / NumPy; convolve_non_zero sums in the reference's
// loop order (k, j, i) in float64 without FMA.
#include "b2v_common.cuh"

namespace {

__device__ __forceinline__ long long reflect_idx(long long i, long long n) {   // scipy mode='reflect': (d c b a | a b c d | d c b a)
  if (n == 1) return 0;
  const long long period = 2 * n;
  i %= period;
  if (i < 0) i += period;
  return i < n ? i : period - 1 - i;
}

// double -> int16 like the x86 code NumPy / SciPy compile to: truncate into int32, keep the low 16 bits
// (CUDA's direct double -> short conversion would saturate instead); identical for values in range
template <typename TO> __device__ __forceinline__ TO cast_out(double v);
template <> __device__ __forceinline__ int16_t cast_out<int16_t>(double v) { return (int16_t)(int)v; }
template <> __device__ __forceinline__ double cast_out<double>(double v) { return v; }
template <> __device__ __forceinline__ float cast_out<float>(double v) { return (float)v; }

// op: 0 union, 1 difference, 2 intersection, 3 xor; selected <=> value > 2 (slice_.py:1906-1916)
__global__ void __launch_bounds__(256) k_boolean_op(const uint8_t* __restrict__ m1, const uint8_t* __restrict__ m2, long long n,
                                                    int op, uint8_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool a = m1[i] > 2, b = m2[i] > 2;
    bool r;
    if (op == 0) r = a || b;
    else if (op == 1) r = a != (a && b);
    else if (op == 2) r = a && b;
    else r = a != b;
    out[i] = r ? 255 : 0;
  }
}

__global__ void __launch_bounds__(256) k_convolve_non_zero(const double* __restrict__ vol, int sz, int sy, int sx,
                                                           const double* __restrict__ ker, int skz, int sky, int skx,
                                                           double cval, double* __restrict__ out) {
  const long long n = (long long)sz * sy * sx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int x = (int)(p % sx);
    const long long r = p / sx;
    const int y = (int)(r % sy), z = (int)(r / sy);
    double sum = 0.0;
    if (vol[p] != 0.0) {
      for (int k = 0; k < skz; ++k) {
        const int kz = z - skz / 2 + k;
        for (int j = 0; j < sky; ++j) {
          const int ky = y - sky / 2 + j;
          for (int i = 0; i < skx; ++i) {
            const int kx = x - skx / 2 + i;
            const double v = (kz >= 0 && kz < sz && ky >= 0 && ky < sy && kx >= 0 && kx < sx)
                                 ? vol[((long long)kz * sy + ky) * sx + kx] : cval;
            sum += v * ker[(k * sky + j) * skx + i];
          }
        }
      }
    }
    out[p] = sum;
  }
}

// median of the WZ x WY x WX neighbourhood (reflect borders; window [i - W/2, i - W/2 + W) per axis and
// rank N / 2 as scipy.ndimage.median_filter takes them, even sizes included): radix select on the
// order-preserving unsigned image of the int16 values, 16 counting passes over the window kept in
// registers / local memory. <S, S, S> is the 3-D filter; a window of 1 along one axis is the 2-D filter of
// every slice along that axis (median_filter(vol, size=(1, S, S)) == the per-slice loop, for axis 0).
template <int WZ, int WY, int WX>
__global__ void __launch_bounds__(128) k_median_i16(const int16_t* __restrict__ in, int nz, int ny, int nx,
                                                    int16_t* __restrict__ out) {
  constexpr int N = WZ * WY * WX, R = N / 2;
  const long long n = (long long)nz * ny * nx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int x = (int)(p % nx);
    const long long r = p / nx;
    const int y = (int)(r % ny), z = (int)(r / ny);
    unsigned short w[N];
    int c = 0;
#pragma unroll
    for (int kz = 0; kz < WZ; ++kz) {
      const long long zz = reflect_idx(z - WZ / 2 + kz, nz);
#pragma unroll
      for (int ky = 0; ky < WY; ++ky) {
        const long long yy = reflect_idx(y - WY / 2 + ky, ny);
        const int16_t* row = in + (zz * ny + yy) * nx;
#pragma unroll
        for (int kx = 0; kx < WX; ++kx) w[c++] = (unsigned short)((int)row[reflect_idx(x - WX / 2 + kx, nx)] + 32768);
      }
    }
    // the largest value v such that at least N - R window entries are >= v  ==  the entry of rank R (0-based, ascending)
    unsigned int v = 0;
#pragma unroll 1
    for (int bit = 15; bit >= 0; --bit) {
      const unsigned int cand = v | (1u << bit);
      int ge = 0;
#pragma unroll
      for (int k = 0; k < N; ++k) ge += (unsigned int)w[k] >= cand;
      if (ge >= N - R) v = cand;
    }
    out[p] = (int16_t)((int)v - 32768);
  }
}

// one separable pass of uniform_filter along `axis`: out = trunc(window sum / size), int16 -> int16
__global__ void __launch_bounds__(256) k_uniform1d_i16(const int16_t* __restrict__ in, int nz, int ny, int nx, int axis,
                                                       int size, int16_t* __restrict__ out) {
  const long long n = (long long)nz * ny * nx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int len = axis == 0 ? nz : (axis == 1 ? ny : nx);
  const long long step = axis == 0 ? (long long)ny * nx : (axis == 1 ? nx : 1);
  const int lo = size / 2;        // window [i - size/2, i + size - 1 - size/2] (origin 0)
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int x = (int)(p % nx);
    const long long r = p / nx;
    const int y = (int)(r % ny), z = (int)(r / ny);
    const int i = axis == 0 ? z : (axis == 1 ? y : x);
    const long long base = p - (long long)i * step;
    long long sum = 0;
    for (int k = 0; k < size; ++k) sum += in[base + reflect_idx(i - lo + k, len) * step];
    out[p] = cast_out<int16_t>((double)sum / (double)size);     // NI_UniformFilter1D: tmp / filter_size in double, C cast
  }
}

// scipy.ndimage.correlate1d for symmetric (sym = +1) / antisymmetric (sym = -1) odd kernels, exactly as
// NI_Correlate1D evaluates them: tmp = x[c] * w[0]; for jj = -r .. -1: tmp += (x[c + jj] (+/-) x[c - jj]) * w[jj],
// float64, 'reflect' borders; an int16 output receives the C cast of tmp (truncation), as SciPy's line
// buffer does. w: centred weights on the device (w[r] is the centre).
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) k_correlate1d(const TI* __restrict__ in, int nz, int ny, int nx, int axis,
                                                     const double* __restrict__ w, int r, int sym, TO* __restrict__ out) {
  const long long n = (long long)nz * ny * nx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int len = axis == 0 ? nz : (axis == 1 ? ny : nx);
  const long long step = axis == 0 ? (long long)ny * nx : (axis == 1 ? nx : 1);
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int x = (int)(p % nx);
    const long long rr = p / nx;
    const int y = (int)(rr % ny), z = (int)(rr / ny);
    const int c = axis == 0 ? z : (axis == 1 ? y : x);
    const long long base = p - (long long)c * step;
    double tmp = (double)in[p] * w[r];
    for (int jj = -r; jj < 0; ++jj) {
      const double lo = (double)in[base + reflect_idx(c + jj, len) * step];
      const double hi = (double)in[base + reflect_idx(c - jj, len) * step];
      tmp += (sym > 0 ? lo + hi : lo - hi) * w[r + jj];
    }
    out[p] = cast_out<TO>(tmp);
  }
}

// Where the elementwise kernels below take their per-voxel constants: one set for the whole volume, or
// one set per slice along an axis, read from [min, max] pairs of b2v_slice_minmax on the device.
struct SliceOf {       // slice index of flat voxel p: (p / div) % n
  long long div;
  int n;
  __device__ __forceinline__ int operator()(long long p) const { return (int)((p / div) % n); }
};

SliceOf slice_of(int64_t ny, int64_t nx, int axis, int64_t nz) {
  if (axis == 0) return {ny * nx, (int)nz};
  if (axis == 1) return {nx, (int)ny};
  return {1, (int)nx};
}

struct ClipWhole {
  double lo, hi;
  __device__ __forceinline__ void operator()(long long, double& l, double& h) const { l = lo; h = hi; }
};

struct ClipPerSlice {  // the slice's own [min, max]
  const double* __restrict__ mm;
  SliceOf sl;
  __device__ __forceinline__ void operator()(long long p, double& l, double& h) const {
    const int s = sl(p);
    l = mm[2 * s];
    h = mm[2 * s + 1];
  }
};

// sharpening_filter (filters.py:21-29): clip(f + (value * 0.5) * (f - blurred), min, max).astype(int16)
template <typename Clip>
__global__ void __launch_bounds__(256) k_sharpen(const int16_t* __restrict__ img, const double* __restrict__ blurred, long long n,
                                                 double half_value, Clip clip, int16_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double f = (double)img[i];
    double lo, hi;
    clip(i, lo, hi);
    double s = f + half_value * (f - blurred[i]);
    s = s < lo ? lo : (s > hi ? hi : s);
    out[i] = cast_out<int16_t>(s);
  }
}

// border_detection_filter (filters.py:45-55): sqrt(sx**2 + sy**2 + sz**2) on a volume, sqrt(sx**2 + sy**2)
// on a slice (c == nullptr), in place into a
__global__ void __launch_bounds__(256) k_sobel_magnitude(double* a, const double* __restrict__ b, const double* __restrict__ c,
                                                         long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    a[i] = c ? sqrt((a[i] * a[i] + b[i] * b[i]) + c[i] * c[i]) : sqrt(a[i] * a[i] + b[i] * b[i]);
}

struct Rescale {
  int on;
  double mag_min, mag_range, span, min_val;
};

struct RescaleWhole {
  Rescale r;
  __device__ __forceinline__ Rescale operator()(long long) const { return r; }
};

struct RescalePerSlice {  // filters.py:60-66 on the slice: its own magnitude range and image range
  const double* __restrict__ mag_mm;
  const double* __restrict__ img_mm;
  SliceOf sl;
  __device__ __forceinline__ Rescale operator()(long long p) const {
    const int s = sl(p);
    const double mag_min = mag_mm[2 * s], mag_range = mag_mm[2 * s + 1] - mag_min;
    const double min_val = img_mm[2 * s], max_val = img_mm[2 * s + 1];
    return {mag_range > 0, mag_min, mag_range, max_val - min_val, min_val};
  }
};

// (magnitude - mag_min) / mag_range * span + min_val, cast to int16 (filters.py:56-66); on = 0: plain cast
template <typename Scale>
__global__ void __launch_bounds__(256) k_rescale_cast(const double* __restrict__ m, long long n, Scale scale,
                                                      int16_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v = m[i];
    const Rescale c = scale(i);
    if (c.on) v = (v - c.mag_min) / c.mag_range * c.span + c.min_val;
    out[i] = cast_out<int16_t>(v);
  }
}

// ---- per-slice [min, max]: order-preserving uint64 keys reduced with atomicMin; the max is kept as the
// min of the complemented key, so one 0xFF fill initialises both slots
__device__ __forceinline__ unsigned long long order_key(double v) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ double from_order_key(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__device__ __forceinline__ void block_minmax_to(double lo, double hi, unsigned long long* slot) {
  __shared__ double s_lo[32], s_hi[32];
  for (int o = 16; o > 0; o >>= 1) {
    lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  const int tid = threadIdx.x + threadIdx.y * blockDim.x, nw = (blockDim.x * blockDim.y) >> 5;
  if ((tid & 31) == 0) { s_lo[tid >> 5] = lo; s_hi[tid >> 5] = hi; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < nw; ++w) { lo = fmin(lo, s_lo[w]); hi = fmax(hi, s_hi[w]); }
    atomicMin(slot, order_key(lo));
    atomicMin(slot + 1, ~order_key(hi));
  }
}

// slices along axis 0 or 1: block (slice s, part); slice element j is (y, x) for axis 0, (z, x) for axis 1
template <typename T>
__global__ void __launch_bounds__(256) k_slice_minmax_rows(const T* __restrict__ in, int nz, int ny, int nx, int axis,
                                                           unsigned long long* __restrict__ keys) {
  const int s = blockIdx.x;
  const long long plane = (long long)ny * nx;
  const long long m = axis == 0 ? plane : (long long)nz * nx;
  double lo = INFINITY, hi = -INFINITY;
  for (long long j = (long long)blockIdx.y * blockDim.x + threadIdx.x; j < m; j += (long long)gridDim.y * blockDim.x) {
    const long long p = axis == 0 ? s * plane + j : (j / nx) * plane + (long long)s * nx + j % nx;
    const double v = (double)in[p];
    lo = fmin(lo, v);
    hi = fmax(hi, v);
  }
  block_minmax_to(lo, hi, keys + 2 * s);
}

// slices along axis 2: block of 32 columns x 8 row lanes, each thread keeps one column's extremes over its rows
template <typename T>
__global__ void __launch_bounds__(256) k_slice_minmax_cols(const T* __restrict__ in, long long rows, int nx,
                                                           unsigned long long* __restrict__ keys) {
  __shared__ double s_lo[8][32], s_hi[8][32];
  const int x = blockIdx.x * 32 + threadIdx.x;
  double lo = INFINITY, hi = -INFINITY;
  if (x < nx)
    for (long long r = (long long)blockIdx.y * 8 + threadIdx.y; r < rows; r += (long long)gridDim.y * 8) {
      const double v = (double)in[r * nx + x];
      lo = fmin(lo, v);
      hi = fmax(hi, v);
    }
  s_lo[threadIdx.y][threadIdx.x] = lo;
  s_hi[threadIdx.y][threadIdx.x] = hi;
  __syncthreads();
  if (threadIdx.y == 0 && x < nx) {
    for (int k = 1; k < 8; ++k) { lo = fmin(lo, s_lo[k][threadIdx.x]); hi = fmax(hi, s_hi[k][threadIdx.x]); }
    atomicMin(keys + 2 * x, order_key(lo));
    atomicMin(keys + 2 * x + 1, ~order_key(hi));
  }
}

__global__ void k_slice_minmax_finish(unsigned long long* kv, int ns) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * ns; i += gridDim.x * blockDim.x) {
    const unsigned long long k = kv[i];
    reinterpret_cast<double*>(kv)[i] = from_order_key(i & 1 ? ~k : k);
  }
}

// np.histogram(a, bins, (lo, lo + bins)) of int16 a: count k = #(a == lo + k), the last bin also takes lo + bins,
// values outside [lo, lo + bins] are not counted. SHARED: per-block uint32 counts in dynamic shared memory,
// added to the int64 counts at the end (the caller keeps each block under 2^32 values)
template <bool SHARED>
__global__ void __launch_bounds__(1024) k_histogram_i16(const int16_t* __restrict__ a, long long n, int lo, int bins,
                                                        unsigned long long* __restrict__ counts) {
  extern __shared__ unsigned int h[];
  if (SHARED) {
    for (int k = threadIdx.x; k < bins; k += blockDim.x) h[k] = 0;
    __syncthreads();
  }
  auto add = [&](int v) {
    const int k = v - lo;
    if (k >= 0 && k <= bins) {
      const int b = k == bins ? bins - 1 : k;
      if (SHARED) atomicAdd(&h[b], 1u);
      else atomicAdd(&counts[b], 1ull);
    }
  };
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = (reinterpret_cast<uintptr_t>(a) & 7) ? 0 : n / 4;   // four values per 8-byte load
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const short4 q = reinterpret_cast<const short4*>(a)[i];
    add(q.x); add(q.y); add(q.z); add(q.w);
  }
  for (long long i = 4 * n4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) add(a[i]);
  if (SHARED) {
    __syncthreads();
    for (int k = threadIdx.x; k < bins; k += blockDim.x)
      if (h[k]) atomicAdd(&counts[k], (unsigned long long)h[k]);
  }
}

}  // namespace

extern "C" int b2v_boolean_op(const uint8_t* m1, const uint8_t* m2, int64_t n, int op, uint8_t* out, void* stream) {
  B2V_REQUIRE(m1 && m2 && out && n > 0 && op >= 0 && op <= 3, B2V_ERR_ARG, "boolean_op: bad arguments");
  k_boolean_op<<<b2v_grid(n, 1024, 32), 256, 0, (cudaStream_t)stream>>>(m1, m2, n, op, out);
  return b2v_check_launch("k_boolean_op");
}

extern "C" int b2v_convolve_non_zero(const double* volume, int64_t sz, int64_t sy, int64_t sx, const double* kernel_dev,
                                     int64_t skz, int64_t sky, int64_t skx, double cval, double* out, void* stream) {
  B2V_REQUIRE(volume && kernel_dev && out && sz > 0 && sy > 0 && sx > 0 && skz > 0 && sky > 0 && skx > 0, B2V_ERR_ARG,
              "convolve_non_zero: bad arguments");
  B2V_REQUIRE(sz < (1ll << 30) && sy < (1ll << 30) && sx < (1ll << 30) && skz * sky * skx < (1ll << 20), B2V_ERR_ARG,
              "convolve_non_zero: shape too large");
  k_convolve_non_zero<<<b2v_grid(sz * sy * sx, 256, 32), 256, 0, (cudaStream_t)stream>>>(volume, (int)sz, (int)sy, (int)sx, kernel_dev,
                                                                                         (int)skz, (int)sky, (int)skx, cval, out);
  return b2v_check_launch("k_convolve_non_zero");
}

namespace {

// axis -1: the S^3 window; axis 0, 1, 2: the S x S window of every slice along that axis
template <int S>
void launch_median(const int16_t* in, int nz, int ny, int nx, int axis, int16_t* out, cudaStream_t s) {
  const int g = b2v_grid((long long)nz * ny * nx, 128, 32);
  if (axis < 0) k_median_i16<S, S, S><<<g, 128, 0, s>>>(in, nz, ny, nx, out);
  else if (axis == 0) k_median_i16<1, S, S><<<g, 128, 0, s>>>(in, nz, ny, nx, out);
  else if (axis == 1) k_median_i16<S, 1, S><<<g, 128, 0, s>>>(in, nz, ny, nx, out);
  else k_median_i16<S, S, 1><<<g, 128, 0, s>>>(in, nz, ny, nx, out);
}

int median_filter(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int axis, int16_t* out, void* stream) {
  B2V_REQUIRE(in && out && in != out && nz > 0 && ny > 0 && nx > 0 && nz * ny * nx < (1ll << 40), B2V_ERR_ARG,
              "median_filter: bad arguments");
  B2V_REQUIRE(size >= 3 && size <= 5, B2V_ERR_ARG, "median_filter: size must be 3, 4 or 5 (filters.py:11 keeps it there)");
  cudaStream_t s = (cudaStream_t)stream;
  if (size == 3) launch_median<3>(in, (int)nz, (int)ny, (int)nx, axis, out, s);
  else if (size == 4) launch_median<4>(in, (int)nz, (int)ny, (int)nx, axis, out, s);
  else launch_median<5>(in, (int)nz, (int)ny, (int)nx, axis, out, s);
  return b2v_check_launch("k_median_i16");
}

bool valid_slice_axis(int axis) { return axis >= 0 && axis <= 2; }

}  // namespace

extern "C" int b2v_median_filter_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int16_t* out,
                                     void* stream) {
  return median_filter(in, nz, ny, nx, size, -1, out, stream);
}

extern "C" int b2v_median_filter_slices_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int axis,
                                            int16_t* out, void* stream) {
  B2V_REQUIRE(valid_slice_axis(axis), B2V_ERR_ARG, "median_filter_slices: axis must be 0, 1 or 2");
  return median_filter(in, nz, ny, nx, size, axis, out, stream);
}

extern "C" int b2v_uniform_filter_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int16_t* out,
                                      int16_t* tmp, void* stream) {
  B2V_REQUIRE(in && out && tmp && in != out && in != tmp && out != tmp && nz > 0 && ny > 0 && nx > 0 && size >= 1,
              B2V_ERR_ARG, "uniform_filter: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = nz * ny * nx;
  int rc;
  // SciPy filters axis 0 first (input -> output), then axes 1, 2 in place on the int16 output
  k_uniform1d_i16<<<b2v_grid(n, 256, 32), 256, 0, s>>>(in, (int)nz, (int)ny, (int)nx, 0, size, out);
  if ((rc = b2v_check_launch("k_uniform1d_i16"))) return rc;
  k_uniform1d_i16<<<b2v_grid(n, 256, 32), 256, 0, s>>>(out, (int)nz, (int)ny, (int)nx, 1, size, tmp);
  if ((rc = b2v_check_launch("k_uniform1d_i16"))) return rc;
  k_uniform1d_i16<<<b2v_grid(n, 256, 32), 256, 0, s>>>(tmp, (int)nz, (int)ny, (int)nx, 2, size, out);
  return b2v_check_launch("k_uniform1d_i16");
}

extern "C" int b2v_uniform_filter_slices_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int axis,
                                             int16_t* out, int16_t* tmp, void* stream) {
  B2V_REQUIRE(in && out && tmp && in != out && in != tmp && out != tmp && nz > 0 && ny > 0 && nx > 0 && size >= 1 &&
                  valid_slice_axis(axis),
              B2V_ERR_ARG, "uniform_filter_slices: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = nz * ny * nx;
  const int a0 = axis == 0 ? 1 : 0, a1 = axis == 2 ? 1 : 2;   // the in-slice axes, ascending, as SciPy runs them
  int rc;
  k_uniform1d_i16<<<b2v_grid(n, 256, 32), 256, 0, s>>>(in, (int)nz, (int)ny, (int)nx, a0, size, tmp);
  if ((rc = b2v_check_launch("k_uniform1d_i16"))) return rc;
  k_uniform1d_i16<<<b2v_grid(n, 256, 32), 256, 0, s>>>(tmp, (int)nz, (int)ny, (int)nx, a1, size, out);
  return b2v_check_launch("k_uniform1d_i16");
}

extern "C" int b2v_slice_minmax(const void* in, int dtype, int64_t nz, int64_t ny, int64_t nx, int axis, double* minmax_out,
                                void* stream) {
  B2V_REQUIRE(in && minmax_out && nz > 0 && ny > 0 && nx > 0 && valid_slice_axis(axis) && (dtype == B2V_I16 || dtype == B2V_F64),
              B2V_ERR_ARG, "slice_minmax: bad arguments");
  B2V_REQUIRE(nz < (1ll << 30) && ny < (1ll << 30) && nx < (1ll << 30), B2V_ERR_ARG, "slice_minmax: shape too large");
  cudaStream_t s = (cudaStream_t)stream;
  const int ns = (int)(axis == 0 ? nz : (axis == 1 ? ny : nx));
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(minmax_out);
  B2V_CUDA(cudaMemsetAsync(keys, 0xff, sizeof(double) * 2 * ns, s));
  const long long target = (long long)b2v_sm_count() * 16;      // blocks in flight over the whole launch
  if (axis == 2) {
    const long long rows = nz * ny;
    const int gx = (int)ceil_div64(nx, 32);
    const int gy = (int)std::max<long long>(1, std::min<long long>(ceil_div64(rows, 64), ceil_div64(target, gx)));
    const dim3 grid(gx, gy), block(32, 8);
    if (dtype == B2V_I16) k_slice_minmax_cols<<<grid, block, 0, s>>>((const int16_t*)in, rows, (int)nx, keys);
    else k_slice_minmax_cols<<<grid, block, 0, s>>>((const double*)in, rows, (int)nx, keys);
  } else {
    const long long m = axis == 0 ? ny * nx : nz * nx;          // voxels per slice
    const int gy = (int)std::max<long long>(1, std::min<long long>(ceil_div64(m, 256 * 8), ceil_div64(target, ns)));
    const dim3 grid(ns, gy);
    if (dtype == B2V_I16) k_slice_minmax_rows<<<grid, 256, 0, s>>>((const int16_t*)in, (int)nz, (int)ny, (int)nx, axis, keys);
    else k_slice_minmax_rows<<<grid, 256, 0, s>>>((const double*)in, (int)nz, (int)ny, (int)nx, axis, keys);
  }
  int rc;
  if ((rc = b2v_check_launch("k_slice_minmax"))) return rc;
  k_slice_minmax_finish<<<(int)ceil_div64(2 * ns, 256), 256, 0, s>>>(keys, ns);
  return b2v_check_launch("k_slice_minmax_finish");
}

extern "C" int b2v_histogram_i16(const int16_t* a, int64_t n, int lo, int bins, int64_t* counts, void* stream) {
  B2V_REQUIRE(a && counts && n > 0 && bins >= 1 && bins <= 65535, B2V_ERR_ARG, "histogram: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  unsigned long long* c = reinterpret_cast<unsigned long long*>(counts);
  B2V_CUDA(cudaMemsetAsync(c, 0, sizeof(int64_t) * bins, s));
  int dev = 0, optin = 0;
  B2V_CUDA(cudaGetDevice(&dev));
  B2V_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t smem = sizeof(unsigned int) * (size_t)bins;
  if (smem <= (size_t)optin) {
    B2V_CUDA(cudaFuncSetAttribute(k_histogram_i16<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2V_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_histogram_i16<true>, 1024, smem));
    // one resident wave, and at least enough blocks that none counts 2^31 values into its uint32 bins
    const long long g = std::max<long long>((long long)b2v_sm_count() * std::max(per_sm, 1), ceil_div64(n, 1ll << 31));
    k_histogram_i16<true><<<(int)g, 1024, smem, s>>>(a, n, lo, bins, c);
  } else {
    k_histogram_i16<false><<<b2v_grid(n, 1024, 32), 1024, 0, s>>>(a, n, lo, bins, c);
  }
  return b2v_check_launch("k_histogram_i16");
}

// dtype pairs (B2V_I16, B2V_I16), (B2V_I16, B2V_F64), (B2V_F64, B2V_F64), (B2V_F32, B2V_F32); in != out
extern "C" int b2v_correlate1d(const void* in, int in_dtype, int64_t nz, int64_t ny, int64_t nx, int axis,
                               const double* weights_dev, int radius, int symmetry, void* out, int out_dtype, void* stream) {
  B2V_REQUIRE(in && out && in != out && weights_dev && nz > 0 && ny > 0 && nx > 0 && axis >= 0 && axis <= 2 && radius >= 0 &&
                  (symmetry == 1 || symmetry == -1),
              B2V_ERR_ARG, "correlate1d: bad arguments");
  B2V_REQUIRE(nz < (1ll << 30) && ny < (1ll << 30) && nx < (1ll << 30), B2V_ERR_ARG, "correlate1d: shape too large");
  cudaStream_t s = (cudaStream_t)stream;
  const int g = b2v_grid(nz * ny * nx, 256, 32);
  if (in_dtype == B2V_I16 && out_dtype == B2V_I16)
    k_correlate1d<int16_t, int16_t><<<g, 256, 0, s>>>((const int16_t*)in, (int)nz, (int)ny, (int)nx, axis, weights_dev, radius, symmetry, (int16_t*)out);
  else if (in_dtype == B2V_I16 && out_dtype == B2V_F64)
    k_correlate1d<int16_t, double><<<g, 256, 0, s>>>((const int16_t*)in, (int)nz, (int)ny, (int)nx, axis, weights_dev, radius, symmetry, (double*)out);
  else if (in_dtype == B2V_F64 && out_dtype == B2V_F64)
    k_correlate1d<double, double><<<g, 256, 0, s>>>((const double*)in, (int)nz, (int)ny, (int)nx, axis, weights_dev, radius, symmetry, (double*)out);
  else if (in_dtype == B2V_F32 && out_dtype == B2V_F32)
    k_correlate1d<float, float><<<g, 256, 0, s>>>((const float*)in, (int)nz, (int)ny, (int)nx, axis, weights_dev, radius, symmetry, (float*)out);
  else B2V_REQUIRE(false, B2V_ERR_ARG, "correlate1d: dtype pair must be (int16,int16), (int16,float64), (float64,float64) or (float32,float32)");
  return b2v_check_launch("k_correlate1d");
}

extern "C" int b2v_sharpen_i16(const int16_t* img, const double* blurred, int64_t n, double value, double lo, double hi,
                               int16_t* out, void* stream) {
  B2V_REQUIRE(img && blurred && out && n > 0, B2V_ERR_ARG, "sharpen: bad arguments");
  k_sharpen<<<b2v_grid(n, 256, 32), 256, 0, (cudaStream_t)stream>>>(img, blurred, n, value * 0.5, ClipWhole{lo, hi}, out);
  return b2v_check_launch("k_sharpen");
}

extern "C" int b2v_sharpen_slices_i16(const int16_t* img, const double* blurred, int64_t nz, int64_t ny, int64_t nx, int axis,
                                      double value, const double* minmax_dev, int16_t* out, void* stream) {
  B2V_REQUIRE(img && blurred && minmax_dev && out && nz > 0 && ny > 0 && nx > 0 && valid_slice_axis(axis), B2V_ERR_ARG,
              "sharpen_slices: bad arguments");
  const long long n = nz * ny * nx;
  k_sharpen<<<b2v_grid(n, 256, 32), 256, 0, (cudaStream_t)stream>>>(img, blurred, n, value * 0.5,
                                                                    ClipPerSlice{minmax_dev, slice_of(ny, nx, axis, nz)}, out);
  return b2v_check_launch("k_sharpen");
}

extern "C" int b2v_sobel_magnitude(double* sx_inout, const double* sy, const double* sz, int64_t n, void* stream) {
  B2V_REQUIRE(sx_inout && sy && n > 0, B2V_ERR_ARG, "sobel_magnitude: bad arguments");
  k_sobel_magnitude<<<b2v_grid(n, 256, 32), 256, 0, (cudaStream_t)stream>>>(sx_inout, sy, sz, n);
  return b2v_check_launch("k_sobel_magnitude");
}

extern "C" int b2v_rescale_cast_i16(const double* m, int64_t n, int rescale, double mag_min, double mag_range, double span,
                                    double min_val, int16_t* out, void* stream) {
  B2V_REQUIRE(m && out && n > 0, B2V_ERR_ARG, "rescale_cast: bad arguments");
  k_rescale_cast<<<b2v_grid(n, 256, 32), 256, 0, (cudaStream_t)stream>>>(m, n, RescaleWhole{{rescale, mag_min, mag_range, span, min_val}},
                                                                         out);
  return b2v_check_launch("k_rescale_cast");
}

extern "C" int b2v_rescale_cast_slices_i16(const double* m, int64_t nz, int64_t ny, int64_t nx, int axis,
                                           const double* mag_minmax_dev, const double* img_minmax_dev, int16_t* out,
                                           void* stream) {
  B2V_REQUIRE(m && mag_minmax_dev && img_minmax_dev && out && nz > 0 && ny > 0 && nx > 0 && valid_slice_axis(axis),
              B2V_ERR_ARG, "rescale_cast_slices: bad arguments");
  const long long n = nz * ny * nx;
  k_rescale_cast<<<b2v_grid(n, 256, 32), 256, 0, (cudaStream_t)stream>>>(
      m, n, RescalePerSlice{mag_minmax_dev, img_minmax_dev, slice_of(ny, nx, axis, nz)}, out);
  return b2v_check_launch("k_rescale_cast");
}
