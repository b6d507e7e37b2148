// Error plumbing, launch accounting, strided host<->device packing, global min/max.
#include <stdarg.h>
#include <string.h>

#include "b2v_common.cuh"

static thread_local char g_err[512] = "";
static thread_local int64_t g_launches = 0;

void b2v_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int b2v_check_launch(const char* what) {
  g_launches++;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    b2v_set_error("launch of %s failed: %s", what, cudaGetErrorString(e));
    return B2V_ERR_CUDA;
  }
  return B2V_OK;
}

int b2v_sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B2V_SM_COUNT_FALLBACK;
  if (dev != cached_dev) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = B2V_SM_COUNT_FALLBACK;
    cached = n;
    cached_dev = dev;
  }
  return cached;
}

extern "C" const char* b2v_last_error(void) { return g_err; }
extern "C" int b2v_version(void) { return 100; }
extern "C" int64_t b2v_launch_count(void) { return g_launches; }
extern "C" void b2v_launch_count_reset(void) { g_launches = 0; }

// ---- strided host views -----------------------------------------------------
static int copy3d(void* dst, int64_t dpitch, int64_t dslice_rows, const void* src, int64_t spitch,
                  int64_t sslice_rows, int64_t dz, int64_t dy, int64_t dx_bytes, cudaMemcpyKind kind,
                  cudaStream_t s) {
  if (dz == 1 && dy == 1) {  // flat run: plain async copy (no pitch limit, fastest DMA path)
    B2V_CUDA(cudaMemcpyAsync(dst, src, (size_t)dx_bytes, kind, s));
    return B2V_OK;
  }
  cudaMemcpy3DParms p;
  memset(&p, 0, sizeof(p));
  p.srcPtr = make_cudaPitchedPtr(const_cast<void*>(src), (size_t)spitch, (size_t)dx_bytes, (size_t)sslice_rows);
  p.dstPtr = make_cudaPitchedPtr(dst, (size_t)dpitch, (size_t)dx_bytes, (size_t)dslice_rows);
  p.extent = make_cudaExtent((size_t)dx_bytes, (size_t)dy, (size_t)dz);
  p.kind = kind;
  B2V_CUDA(cudaMemcpy3DAsync(&p, s));
  return B2V_OK;
}

extern "C" int b2v_copy3d_h2d(void* dst_dev, const void* src_host, int64_t dz, int64_t dy, int64_t dx,
                              int64_t elem, int64_t src_row_pitch, int64_t src_plane_pitch, void* stream) {
  B2V_REQUIRE(dst_dev && src_host, B2V_ERR_ARG, "copy3d_h2d: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0 && elem > 0, B2V_ERR_ARG, "copy3d_h2d: empty box");
  B2V_REQUIRE(src_row_pitch >= dx * elem && src_plane_pitch % src_row_pitch == 0 &&
                  src_plane_pitch / src_row_pitch >= dy,
              B2V_ERR_ARG, "copy3d_h2d: plane pitch must be a whole number of rows >= dy");
  return copy3d(dst_dev, dx * elem, dy, src_host, src_row_pitch, src_plane_pitch / src_row_pitch, dz, dy,
                dx * elem, cudaMemcpyHostToDevice, (cudaStream_t)stream);
}

extern "C" int b2v_copy3d_d2h(void* dst_host, const void* src_dev, int64_t dz, int64_t dy, int64_t dx,
                              int64_t elem, int64_t dst_row_pitch, int64_t dst_plane_pitch, void* stream) {
  B2V_REQUIRE(dst_host && src_dev, B2V_ERR_ARG, "copy3d_d2h: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0 && elem > 0, B2V_ERR_ARG, "copy3d_d2h: empty box");
  B2V_REQUIRE(dst_row_pitch >= dx * elem && dst_plane_pitch % dst_row_pitch == 0 &&
                  dst_plane_pitch / dst_row_pitch >= dy,
              B2V_ERR_ARG, "copy3d_d2h: plane pitch must be a whole number of rows >= dy");
  return copy3d(dst_host, dst_row_pitch, dst_plane_pitch / dst_row_pitch, src_dev, dx * elem, dy, dz, dy,
                dx * elem, cudaMemcpyDeviceToHost, (cudaStream_t)stream);
}

// ---- global min/max as float32 ------------------------------------------------
// Two launches: per-block partial (min,max) pairs, then one block folds them.
// float min/max of values converted to f32 is order-independent (no NaN in int data;
// for f64 inputs NaN handling follows f32::min/f32::max: NaN operands are ignored).
template <typename T>
__device__ __forceinline__ float to_f32(T v) {
  return (float)v;
}

__device__ __forceinline__ void warp_minmax(float& mn, float& mx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
}

__device__ __forceinline__ void block_minmax_store(float mn, float mx, float2* dst) {
  __shared__ float smn[32], smx[32];
  warp_minmax(mn, mx);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    smn[w] = mn;
    smx[w] = mx;
  }
  __syncthreads();
  if (w == 0) {
    int nw = (blockDim.x + 31) >> 5;
    mn = l < nw ? smn[l] : __int_as_float(0x7f800000);
    mx = l < nw ? smx[l] : __int_as_float(0xff800000);
    warp_minmax(mn, mx);
    if (l == 0) *dst = make_float2(mn, mx);
  }
}

// int16 fast path: 8 voxels per 128-bit load, packed min/max.
__global__ void __launch_bounds__(256) k_minmax_i16_vec(const int4* __restrict__ img, int64_t nvec,
                                                        float2* __restrict__ partial) {
  uint32_t mn = 0x7fff7fffu, mx = 0x80008000u;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    int4 a = ld_stream(img + i), b = ld_stream(img + i + stride), c = ld_stream(img + i + 2 * stride),
         d = ld_stream(img + i + 3 * stride);
    uint32_t m0 = min_s16x2(min_s16x2(a.x, a.y), min_s16x2(a.z, a.w));
    uint32_t m1 = min_s16x2(min_s16x2(b.x, b.y), min_s16x2(b.z, b.w));
    uint32_t m2 = min_s16x2(min_s16x2(c.x, c.y), min_s16x2(c.z, c.w));
    uint32_t m3 = min_s16x2(min_s16x2(d.x, d.y), min_s16x2(d.z, d.w));
    mn = min_s16x2(mn, min_s16x2(min_s16x2(m0, m1), min_s16x2(m2, m3)));
    uint32_t x0 = max_s16x2(max_s16x2(a.x, a.y), max_s16x2(a.z, a.w));
    uint32_t x1 = max_s16x2(max_s16x2(b.x, b.y), max_s16x2(b.z, b.w));
    uint32_t x2 = max_s16x2(max_s16x2(c.x, c.y), max_s16x2(c.z, c.w));
    uint32_t x3 = max_s16x2(max_s16x2(d.x, d.y), max_s16x2(d.z, d.w));
    mx = max_s16x2(mx, max_s16x2(max_s16x2(x0, x1), max_s16x2(x2, x3)));
  }
  for (; i < nvec; i += stride) {
    int4 a = ld_stream(img + i);
    mn = min_s16x2(mn, min_s16x2(min_s16x2(a.x, a.y), min_s16x2(a.z, a.w)));
    mx = max_s16x2(mx, max_s16x2(max_s16x2(a.x, a.y), max_s16x2(a.z, a.w)));
  }
  int lo = min((int)(int16_t)(mn & 0xffff), (int)(int16_t)(mn >> 16));
  int hi = max((int)(int16_t)(mx & 0xffff), (int)(int16_t)(mx >> 16));
  block_minmax_store((float)lo, (float)hi, partial + blockIdx.x);
}

template <typename T>
__global__ void __launch_bounds__(256) k_minmax_scalar(const T* __restrict__ img, int64_t n,
                                                       float2* __restrict__ partial) {
  float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float v = to_f32(img[i]);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  block_minmax_store(mn, mx, partial + blockIdx.x);
}

// Folds `nparts` partial pairs plus an optional scalar tail [tail0, n) of the image.
template <typename T>
__global__ void __launch_bounds__(256) k_minmax_final(const float2* __restrict__ partial, int nparts,
                                                      const T* __restrict__ img, int64_t tail0, int64_t n,
                                                      float* __restrict__ out) {
  float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
    float2 p = partial[i];
    mn = fminf(mn, p.x);
    mx = fmaxf(mx, p.y);
  }
  for (int64_t i = tail0 + threadIdx.x; i < n; i += blockDim.x) {
    float v = to_f32(img[i]);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  __shared__ float2 res;
  block_minmax_store(mn, mx, &res);
  __syncthreads();
  if (threadIdx.x == 0) {
    out[0] = res.x;
    out[1] = res.y;
  }
}

// one partial per block: the workspace size and the launch must agree
static int minmax_blocks(int64_t n) { return b2v_grid(n, 256 * 16, 8); }

extern "C" int64_t b2v_minmax_workspace_bytes(int64_t n) { return (int64_t)minmax_blocks(n) * sizeof(float2); }

extern "C" int b2v_minmax_f32(const void* img, int dtype, int64_t n, float* minmax_out, void* workspace,
                              void* stream) {
  B2V_REQUIRE(img && minmax_out && workspace, B2V_ERR_ARG, "minmax: null pointer");
  B2V_REQUIRE(n > 0, B2V_ERR_ARG, "minmax: empty input");
  cudaStream_t s = (cudaStream_t)stream;
  float2* partial = (float2*)workspace;
  int blocks = minmax_blocks(n);
  int rc;
  if (dtype == B2V_I16) {
    const int16_t* p = (const int16_t*)img;
    if (b2v_aligned16(p) && n >= 8) {
      int64_t nvec = n / 8;
      k_minmax_i16_vec<<<blocks, 256, 0, s>>>((const int4*)p, nvec, partial);
      if ((rc = b2v_check_launch("k_minmax_i16_vec"))) return rc;
      k_minmax_final<int16_t><<<1, 256, 0, s>>>(partial, blocks, p, nvec * 8, n, minmax_out);
    } else {
      k_minmax_scalar<int16_t><<<blocks, 256, 0, s>>>(p, n, partial);
      if ((rc = b2v_check_launch("k_minmax_scalar"))) return rc;
      k_minmax_final<int16_t><<<1, 256, 0, s>>>(partial, blocks, p, n, n, minmax_out);
    }
  } else if (dtype == B2V_U8) {
    const uint8_t* p = (const uint8_t*)img;
    k_minmax_scalar<uint8_t><<<blocks, 256, 0, s>>>(p, n, partial);
    if ((rc = b2v_check_launch("k_minmax_scalar"))) return rc;
    k_minmax_final<uint8_t><<<1, 256, 0, s>>>(partial, blocks, p, n, n, minmax_out);
  } else if (dtype == B2V_F64) {
    const double* p = (const double*)img;
    k_minmax_scalar<double><<<blocks, 256, 0, s>>>(p, n, partial);
    if ((rc = b2v_check_launch("k_minmax_scalar"))) return rc;
    k_minmax_final<double><<<1, 256, 0, s>>>(partial, blocks, p, n, n, minmax_out);
  } else {
    B2V_REQUIRE(false, B2V_ERR_ARG, "minmax: unknown dtype code %d", dtype);
  }
  return b2v_check_launch("k_minmax_final");
}
