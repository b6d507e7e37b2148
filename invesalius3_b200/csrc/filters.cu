// Whole-volume pre-filters and mask algebra (SURVEY 8f-4): the step before threshold
// (invesalius/data/filters.py:5-66 driven by slice_.py:2330-2432) and elementwise mask operations.
//   b2v_boolean_op          Slice.do_boolean_op                   slice_.py:1906-1916
//   b2v_convolve_non_zero   invesalius_rs.convolve_non_zero       transforms_py.rs:52-93 (calc_mask_area, slice_.py:2299-2322)
//   b2v_median_filter_i16   ndimage.median_filter(matrix, size)   filters.py:9-12 (size 3, 4 or 5, mode 'reflect')
//   b2v_uniform_filter_i16  ndimage.uniform_filter(matrix, size)  filters.py:15-18 (separable; every pass stores
//                           trunc(sum / size) in int16 like SciPy's NI_UniformFilter1D writing into an int16 output)
// All integer results are bit-exact against SciPy / NumPy; convolve_non_zero sums in the reference's
// loop order (k, j, i) in float64 without FMA.
#include "b2v_common.cuh"

namespace {

int fgrid(long long n, int per = 256) {
  long long blocks = ceil_div64(n, per);
  long long cap = (long long)b2v_sm_count() * 32;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

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

// median of the S^3 neighbourhood (reflect borders; window [i - S/2, i - S/2 + S) and rank S^3 / 2 as
// scipy.ndimage.median_filter takes them, even sizes included): radix select on the order-preserving
// unsigned image of the int16 values, 16 counting passes over the window kept in registers / local memory
template <int S>
__global__ void __launch_bounds__(128) k_median_i16(const int16_t* __restrict__ in, int nz, int ny, int nx,
                                                    int16_t* __restrict__ out) {
  constexpr int N = S * S * S, R = N / 2, H = S / 2;
  const long long n = (long long)nz * ny * nx;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
    const int x = (int)(p % nx);
    const long long r = p / nx;
    const int y = (int)(r % ny), z = (int)(r / ny);
    unsigned short w[N];
    int c = 0;
#pragma unroll
    for (int kz = 0; kz < S; ++kz) {
      const long long zz = reflect_idx(z - H + kz, nz);
#pragma unroll
      for (int ky = 0; ky < S; ++ky) {
        const long long yy = reflect_idx(y - H + ky, ny);
        const int16_t* row = in + (zz * ny + yy) * nx;
#pragma unroll
        for (int kx = 0; kx < S; ++kx) w[c++] = (unsigned short)((int)row[reflect_idx(x - H + kx, nx)] + 32768);
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

// sharpening_filter (filters.py:21-29): clip(f + (value * 0.5) * (f - blurred), min, max).astype(int16)
__global__ void __launch_bounds__(256) k_sharpen(const int16_t* __restrict__ img, const double* __restrict__ blurred, long long n,
                                                 double half_value, double lo, double hi, int16_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double f = (double)img[i];
    double s = f + half_value * (f - blurred[i]);
    s = s < lo ? lo : (s > hi ? hi : s);
    out[i] = cast_out<int16_t>(s);
  }
}

// border_detection_filter (filters.py:45-51): sqrt(sx**2 + sy**2 + sz**2), in place into a
__global__ void __launch_bounds__(256) k_sobel_magnitude(double* a, const double* __restrict__ b, const double* __restrict__ c,
                                                         long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    a[i] = sqrt((a[i] * a[i] + b[i] * b[i]) + c[i] * c[i]);
}

// (magnitude - mag_min) / mag_range * span + min_val, cast to int16 (filters.py:56-66); scale = 0: plain cast
__global__ void __launch_bounds__(256) k_rescale_cast(const double* __restrict__ m, long long n, int rescale, double mag_min,
                                                      double mag_range, double span, double min_val, int16_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v = m[i];
    if (rescale) v = (v - mag_min) / mag_range * span + min_val;
    out[i] = cast_out<int16_t>(v);
  }
}

}  // namespace

extern "C" int b2v_boolean_op(const uint8_t* m1, const uint8_t* m2, int64_t n, int op, uint8_t* out, void* stream) {
  B2V_REQUIRE(m1 && m2 && out && n > 0 && op >= 0 && op <= 3, B2V_ERR_ARG, "boolean_op: bad arguments");
  k_boolean_op<<<fgrid(n, 1024), 256, 0, (cudaStream_t)stream>>>(m1, m2, n, op, out);
  return b2v_check_launch("k_boolean_op");
}

extern "C" int b2v_convolve_non_zero(const double* volume, int64_t sz, int64_t sy, int64_t sx, const double* kernel_dev,
                                     int64_t skz, int64_t sky, int64_t skx, double cval, double* out, void* stream) {
  B2V_REQUIRE(volume && kernel_dev && out && sz > 0 && sy > 0 && sx > 0 && skz > 0 && sky > 0 && skx > 0, B2V_ERR_ARG,
              "convolve_non_zero: bad arguments");
  B2V_REQUIRE(sz < (1ll << 30) && sy < (1ll << 30) && sx < (1ll << 30) && skz * sky * skx < (1ll << 20), B2V_ERR_ARG,
              "convolve_non_zero: shape too large");
  k_convolve_non_zero<<<fgrid(sz * sy * sx), 256, 0, (cudaStream_t)stream>>>(volume, (int)sz, (int)sy, (int)sx, kernel_dev,
                                                                             (int)skz, (int)sky, (int)skx, cval, out);
  return b2v_check_launch("k_convolve_non_zero");
}

extern "C" int b2v_median_filter_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int16_t* out,
                                     void* stream) {
  B2V_REQUIRE(in && out && in != out && nz > 0 && ny > 0 && nx > 0 && nz * ny * nx < (1ll << 40), B2V_ERR_ARG,
              "median_filter: bad arguments");
  B2V_REQUIRE(size >= 3 && size <= 5, B2V_ERR_ARG, "median_filter: size must be 3, 4 or 5 (filters.py:11 keeps it there)");
  cudaStream_t s = (cudaStream_t)stream;
  if (size == 3) k_median_i16<3><<<fgrid(nz * ny * nx, 128), 128, 0, s>>>(in, (int)nz, (int)ny, (int)nx, out);
  else if (size == 4) k_median_i16<4><<<fgrid(nz * ny * nx, 128), 128, 0, s>>>(in, (int)nz, (int)ny, (int)nx, out);
  else k_median_i16<5><<<fgrid(nz * ny * nx, 128), 128, 0, s>>>(in, (int)nz, (int)ny, (int)nx, out);
  return b2v_check_launch("k_median_i16");
}

extern "C" int b2v_uniform_filter_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int16_t* out,
                                      int16_t* tmp, void* stream) {
  B2V_REQUIRE(in && out && tmp && in != out && in != tmp && out != tmp && nz > 0 && ny > 0 && nx > 0 && size >= 1,
              B2V_ERR_ARG, "uniform_filter: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const long long n = nz * ny * nx;
  int rc;
  // SciPy filters axis 0 first (input -> output), then axes 1, 2 in place on the int16 output
  k_uniform1d_i16<<<fgrid(n), 256, 0, s>>>(in, (int)nz, (int)ny, (int)nx, 0, size, out);
  if ((rc = b2v_check_launch("k_uniform1d_i16"))) return rc;
  k_uniform1d_i16<<<fgrid(n), 256, 0, s>>>(out, (int)nz, (int)ny, (int)nx, 1, size, tmp);
  if ((rc = b2v_check_launch("k_uniform1d_i16"))) return rc;
  k_uniform1d_i16<<<fgrid(n), 256, 0, s>>>(tmp, (int)nz, (int)ny, (int)nx, 2, size, out);
  return b2v_check_launch("k_uniform1d_i16");
}

// dtype pairs (B2V_I16, B2V_I16), (B2V_I16, B2V_F64), (B2V_F64, B2V_F64), (B2V_F32, B2V_F32); in != out
extern "C" int b2v_correlate1d(const void* in, int in_dtype, int64_t nz, int64_t ny, int64_t nx, int axis,
                               const double* weights_dev, int radius, int symmetry, void* out, int out_dtype, void* stream) {
  B2V_REQUIRE(in && out && in != out && weights_dev && nz > 0 && ny > 0 && nx > 0 && axis >= 0 && axis <= 2 && radius >= 0 &&
                  (symmetry == 1 || symmetry == -1),
              B2V_ERR_ARG, "correlate1d: bad arguments");
  B2V_REQUIRE(nz < (1ll << 30) && ny < (1ll << 30) && nx < (1ll << 30), B2V_ERR_ARG, "correlate1d: shape too large");
  cudaStream_t s = (cudaStream_t)stream;
  const int g = fgrid(nz * ny * nx);
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
  k_sharpen<<<fgrid(n), 256, 0, (cudaStream_t)stream>>>(img, blurred, n, value * 0.5, lo, hi, out);
  return b2v_check_launch("k_sharpen");
}

extern "C" int b2v_sobel_magnitude(double* sx_inout, const double* sy, const double* sz, int64_t n, void* stream) {
  B2V_REQUIRE(sx_inout && sy && sz && n > 0, B2V_ERR_ARG, "sobel_magnitude: bad arguments");
  k_sobel_magnitude<<<fgrid(n), 256, 0, (cudaStream_t)stream>>>(sx_inout, sy, sz, n);
  return b2v_check_launch("k_sobel_magnitude");
}

extern "C" int b2v_rescale_cast_i16(const double* m, int64_t n, int rescale, double mag_min, double mag_range, double span,
                                    double min_val, int16_t* out, void* stream) {
  B2V_REQUIRE(m && out && n > 0, B2V_ERR_ARG, "rescale_cast: bad arguments");
  k_rescale_cast<<<fgrid(n), 256, 0, (cudaStream_t)stream>>>(m, n, rescale, mag_min, mag_range, span, min_val, out);
  return b2v_check_launch("k_rescale_cast");
}
