// Ray-sequential projections: MIDA, LMIP and the contour-enhanced variants.
// Reference semantics: invesalius_rs/src/mips.rs
//   mida_internal               :102-168 (+ get_opacity :88-100)     b2v_mida
//   lmip                        :7-86                                 b2v_lmip
//   fast_countour_mip_internal  :215-279 (finite_difference :170-195,
//                               calc_fcm_intensity :197-213)          b2v_fast_countour_mip
// All float arithmetic is float32 with the reference's operation order and no FMA
// (explicit __f*_rn intrinsics); casts to the output type truncate toward zero and a value
// that does not fit (NaN included) is reported as B2V_ERR_RANGE, where the reference panics.
//
// One ray per thread; MIDA and LMIP are operators (MidaOp, LmipOp) run by the same ray kernels.
// Rays along z or y (axis 0/1) keep x contiguous across the threads of a warp, so every step is
// a coalesced row access; rays along x (axis 2) are staged through a padded shared-memory tile
// (128 rays x 32 samples) that is loaded row-wise (coalesced) and walked column-wise (bank-conflict
// free). A block stops loading as soon as all of its rays have terminated (alpha >= 1 in MIDA,
// first local maximum in LMIP).
// HBM: 2 B/voxel for the ray pass + 2 B/voxel for the global min/max pass MIDA needs.
//
// The contour variants do as the reference does: k_fcm_volume materialises the contour volume,
// which b2v_mip, b2v_lmip or b2v_mida then projects. The *_z_partial entry points walk the rays
// along z through one Z shard at a time, handing each ray's state on to the next shard.
#include <math.h>

#include "b2v_common.cuh"

namespace {

struct Dims {
  int64_t nz, ny, nx;
};

template <typename T> __device__ __forceinline__ float wrapdiff(T a, T b);
template <> __device__ __forceinline__ float wrapdiff<int16_t>(int16_t a, int16_t b) {
  return (float)(int16_t)((int)a - (int)b);
}
template <> __device__ __forceinline__ float wrapdiff<uint8_t>(uint8_t a, uint8_t b) {
  return (float)(uint8_t)((int)a - (int)b);
}

template <> __device__ __forceinline__ float wrapdiff<double>(double a, double b) {
  return (float)(a - b);   // f64 difference, then to_f32 (mips.rs:190-192 on ArrayView3<f64>)
}

template <typename T> __device__ __forceinline__ bool cast_f32(float f, T* o);
template <> __device__ __forceinline__ bool cast_f32<double>(float f, double* o) {
  *o = (double)f;
  return true;
}
template <> __device__ __forceinline__ bool cast_f32<int16_t>(float f, int16_t* o) {
  if (!(f > -32769.0f && f < 32768.0f)) return false;
  *o = (int16_t)f;
  return true;
}
template <> __device__ __forceinline__ bool cast_f32<uint8_t>(float f, uint8_t* o) {
  if (!(f > -1.0f && f < 256.0f)) return false;
  *o = (uint8_t)f;
  return true;
}

// ---- per-ray operators --------------------------------------------------------------------
// An operator is copied into every thread, which calls init() once, first() with the ray's first
// sample, step() with every sample from the first on until it reports the ray finished, and
// result() at the end.

// get_opacity (mips.rs:88-100). The window bounds are ray-invariant: computed once per thread
// (same float32 operations, so the same values) instead of once per sample.
struct Window {
  float mn, mx, den;
  __device__ __forceinline__ void set(float wl, float ww) {
    float half = __fdiv_rn(ww, 2.0f);
    mn = __fsub_rn(wl, half);
    mx = __fadd_rn(wl, half);
    den = __fsub_rn(mx, mn);
  }
  __device__ __forceinline__ float opacity(float vl) const {
    if (vl < mn) return 0.0f;
    if (vl > mx) return 1.0f;
    return __fdiv_rn(__fsub_rn(vl, mn), den);
  }
};

template <typename T, typename U>
struct MidaOp {
  // The (min, max) pair of the volume stays on the device (b2v_minmax_f32 or the caller wrote
  // it): every thread derives (min, range, 1/range) from it in init() instead of the host
  // synchronising to read it.
  const float* mm;
  float wl, ww;
  float img_min, range, inv;
  float fmax, alpha_p, colour_p, final_colour;
  Window win;
  __device__ __forceinline__ void init() {
    img_min = mm[0];
    range = __fsub_rn(mm[1], mm[0]);
    inv = __fdiv_rn(1.0f, range);
    fmax = alpha_p = colour_p = final_colour = 0.0f;
    win.set(wl, ww);
  }
  __device__ __forceinline__ void first(T) {}
  // returns true when the ray is finished
  __device__ __forceinline__ bool step(T raw) {
    float vl = (float)raw;
    float fpi = __fmul_rn(inv, __fsub_rn(vl, img_min));
    float dl = 0.0f;
    if (fpi > fmax) {
      dl = __fsub_rn(fpi, fmax);
      fmax = fpi;
    }
    float bt = __fsub_rn(1.0f, dl);
    float alpha = win.opacity(vl);
    float one_m = __fsub_rn(1.0f, __fmul_rn(bt, alpha_p));
    float colour = __fadd_rn(__fmul_rn(bt, colour_p), __fmul_rn(__fmul_rn(one_m, fpi), alpha));
    float cur = __fadd_rn(__fmul_rn(bt, alpha_p), __fmul_rn(one_m, alpha));
    colour_p = colour;
    alpha_p = cur;
    final_colour = colour;
    return cur >= 1.0f;
  }
  __device__ __forceinline__ bool result(U* o) const {
    return cast_result(__fadd_rn(__fmul_rn(range, final_colour), img_min), o);
  }
  // ray state handed from one Z shard to the next: (fmax, alpha, colour) as three planes of
  // 32-bit words; final_colour always equals colour_p, and the ray is finished exactly when
  // the accumulated alpha reached 1 (the value step() tested)
  __device__ __forceinline__ void load(const uint32_t* st, int64_t i, int64_t plane, bool* done) {
    fmax = __uint_as_float(st[i]);
    alpha_p = __uint_as_float(st[plane + i]);
    colour_p = final_colour = __uint_as_float(st[2 * plane + i]);
    *done = alpha_p >= 1.0f;
  }
  __device__ __forceinline__ void store(uint32_t* st, int64_t i, int64_t plane, bool) const {
    st[i] = __float_as_uint(fmax);
    st[plane + i] = __float_as_uint(alpha_p);
    st[2 * plane + i] = __float_as_uint(colour_p);
  }
  __device__ __forceinline__ static bool cast_result(float f, int16_t* o) { return cast_f32<int16_t>(f, o); }
  __device__ __forceinline__ static bool cast_result(float f, uint8_t* o) { return cast_f32<uint8_t>(f, o); }
};

template <typename T>
struct LmipOp {
  T tmin, tmax, max_val;
  bool start;
  __device__ __forceinline__ void init() {}
  __device__ __forceinline__ void first(T v) {
    max_val = v;
    start = v >= tmin && v <= tmax;
  }
  __device__ __forceinline__ bool step(T val) {
    if (val > max_val) max_val = val;
    else if (val < max_val && start) return true;
    if (val >= tmin && val <= tmax) start = true;
    return false;
  }
  __device__ __forceinline__ bool result(T* o) const {
    *o = max_val;
    return true;
  }
  // ray state across Z shards: the running maximum (two words: a double needs both), then
  // bit 0 = inside [tmin, tmax] seen, bit 1 = ray finished
  __device__ __forceinline__ void load(const uint32_t* st, int64_t i, int64_t plane, bool* done) {
    if (sizeof(T) == 8) {
      const unsigned long long b = (unsigned long long)st[i] | ((unsigned long long)st[plane + i] << 32);
      max_val = (T)__longlong_as_double((long long)b);
    } else {
      max_val = (T)(int)st[i];
    }
    const uint32_t f = st[2 * plane + i];
    start = f & 1u;
    *done = (f & 2u) != 0;
  }
  __device__ __forceinline__ void store(uint32_t* st, int64_t i, int64_t plane, bool done) const {
    if (sizeof(T) == 8) {
      const unsigned long long b = (unsigned long long)__double_as_longlong((double)max_val);
      st[i] = (uint32_t)b;
      st[plane + i] = (uint32_t)(b >> 32);
    } else {
      st[i] = (uint32_t)(int)max_val;
      st[plane + i] = 0u;
    }
    st[2 * plane + i] = (start ? 1u : 0u) | (done ? 2u : 0u);
  }
};

// ---- ray kernels ---------------------------------------------------------------------------
// One ray of a keep-x kernel (axis 0: along z, axis 1: along y): a pointer advanced by a constant
// stride. kBatch samples are fetched before any of them is consumed, because the recurrence is a
// long dependent chain the loads must not wait for. The walk stops at the first sample whose
// step() reports the ray finished.
constexpr int kBatch = 8;

template <typename T, typename Op>
__device__ __forceinline__ bool walk_keepx(const T* __restrict__ vol, Dims d, int axis, int64_t r, int64_t x,
                                           int64_t n_l, Op& op) {
  const int64_t plane = d.ny * d.nx;
  const int64_t stride = axis == 0 ? plane : d.nx;
  const T* __restrict__ p = vol + (axis == 0 ? r * d.nx + x : r * plane + x);
  int64_t l0 = 0;
  for (; l0 + kBatch <= n_l; l0 += kBatch) {
    T v[kBatch];
#pragma unroll
    for (int k = 0; k < kBatch; ++k) v[k] = p[k * stride];
    p += kBatch * stride;
#pragma unroll
    for (int k = 0; k < kBatch; ++k)
      if (op.step(v[k])) return true;
  }
  for (; l0 < n_l; ++l0, p += stride)
    if (op.step(*p)) return true;
  return false;
}

// axis 0: out[y][x], ray along z; axis 1: out[z][x], ray along y. One thread per (r, x).
template <typename T, typename U, typename Op>
__global__ void __launch_bounds__(128) k_rays_keepx(const T* __restrict__ vol, Dims d, int axis, Op op0,
                                                    U* __restrict__ out, int* status) {
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = blockIdx.y;
  if (x >= d.nx) return;
  const int64_t n_l = axis == 0 ? d.nz : d.ny;
  Op op = op0;
  op.init();
  op.first(vol[axis == 0 ? r * d.nx + x : r * d.ny * d.nx + x]);
  walk_keepx<T>(vol, d, axis, r, x, n_l, op);
  U o;
  if (op.result(&o)) out[r * d.nx + x] = o; else *status = B2V_ERR_RANGE;
}

// axis 2: out[z][y], ray along x. 128 rays per block, 32 samples per tile.
constexpr int kRays = 128, kChunk = 32;
template <typename T> struct Pitch;
template <> struct Pitch<int16_t> { static constexpr int value = kChunk + 2; };   // 17 words
template <> struct Pitch<uint8_t> { static constexpr int value = kChunk + 4; };   // 9 words
template <> struct Pitch<double> { static constexpr int value = kChunk + 1; };

// Stage the 32-sample segments [x0, x0+32) of kRays consecutive rows in shared memory. An int16
// volume with even rows moves two samples per lane (half a warp per row, 64 B each); otherwise
// one sample per lane (a warp per row).
template <typename T>
__device__ __forceinline__ void load_tile(const T* __restrict__ vol, Dims d, T (*tile)[Pitch<T>::value], int64_t row0,
                                          int64_t nrows, int64_t x0, int lane, int warp) {
  if constexpr (sizeof(T) == 2) {
    if ((d.nx & 1) == 0 && (reinterpret_cast<uintptr_t>(vol) & 3) == 0) {
      const int half = lane >> 4, l16 = lane & 15;
      const int64_t x = x0 + 2 * l16;
      const bool xin = x < d.nx;
      const T* p = vol + (row0 + warp * 2 + half) * d.nx + x;
      const int64_t step = (int64_t)(kRays / 16) * d.nx;
#pragma unroll
      for (int rr = warp * 2 + half; rr < kRays; rr += kRays / 16, p += step) {
        uint32_t w = 0;
        if (row0 + rr < nrows && xin) w = *reinterpret_cast<const uint32_t*>(p);
        *reinterpret_cast<uint32_t*>(&tile[rr][2 * l16]) = w;
      }
      return;
    }
  }
  for (int rr = warp; rr < kRays; rr += kRays / 32) {
    const int64_t row = row0 + rr;
    const int64_t x = x0 + lane;
    T v = 0;
    if (row < nrows && x < d.nx) v = vol[row * d.nx + x];
    tile[rr][lane] = v;
  }
}

// Feed one thread's staged samples to its operator; true when the ray is finished.
template <typename T, typename Op>
__device__ __forceinline__ bool consume_tile(const T* row, int lim, Op& op) {
  if (lim == kChunk) {
    if constexpr (sizeof(T) == 2) {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(row);   // rows are 4-byte aligned
#pragma unroll
      for (int k = 0; k < kChunk / 2; ++k) {
        const uint32_t pair = w[k];
        if (op.step((T)(pair & 0xffffu))) return true;
        if (op.step((T)(pair >> 16))) return true;
      }
    } else {
#pragma unroll
      for (int k = 0; k < kChunk; ++k)
        if (op.step(row[k])) return true;
    }
    return false;
  }
  for (int k = 0; k < lim; ++k)
    if (op.step(row[k])) return true;
  return false;
}

template <typename T, typename U, typename Op>
__global__ void __launch_bounds__(kRays) k_rays_alongx(const T* __restrict__ vol, Dims d, Op op0, U* __restrict__ out,
                                                       int* status) {
  __shared__ __align__(16) T tile[kRays][Pitch<T>::value];
  const int64_t nrows = d.nz * d.ny;
  const int64_t row0 = (int64_t)blockIdx.x * kRays;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t myrow = row0 + tid;
  const bool live = myrow < nrows;
  Op op = op0;
  op.init();
  bool done = !live;
  for (int64_t x0 = 0; x0 < d.nx; x0 += kChunk) {
    load_tile<T>(vol, d, tile, row0, nrows, x0, lane, warp);
    __syncthreads();
    if (!done) {
      if (x0 == 0) op.first(tile[tid][0]);
      int lim = (int)((d.nx - x0) < kChunk ? (d.nx - x0) : kChunk);
      done = consume_tile<T>(tile[tid], lim, op);
    }
    if (__syncthreads_and(done)) break;
  }
  if (live) {
    U o;
    if (op.result(&o)) out[myrow] = o; else *status = B2V_ERR_RANGE;
  }
}

// ---- rays along z over ONE Z shard (dist: MIDA / LMIP with rays that cross the shards) ------
// The ray of pixel (y, x) starts from the state the previous shard left (or is started here),
// walks this slab and leaves its state for the next shard; the last shard writes the pixel.
// The per-ray operation order is that of the whole-volume walk, so the result is bit-exact.
template <typename T, typename U, typename Op>
__global__ void __launch_bounds__(128) k_rays_z_partial(const T* __restrict__ vol, Dims d, Op op, uint32_t* state,
                                                        int first, int last, U* __restrict__ out, int* status) {
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t y = blockIdx.y;
  if (x >= d.nx) return;
  const int64_t plane = d.ny * d.nx, i = y * d.nx + x;
  bool done = false;
  op.init();
  if (first) op.first(vol[i]);
  else op.load(state, i, plane, &done);
  if (!done) done = walk_keepx<T>(vol, d, 0, y, x, d.nz, op);
  op.store(state, i, plane, done);
  if (last) {
    U o;
    if (op.result(&o)) out[i] = o; else *status = B2V_ERR_RANGE;
  }
}

__global__ void k_status_init(int* status) { *status = 0; }

// `what` names the projection in the error message.
template <typename T, typename U, typename Op>
int launch_rays(const T* vol, Dims d, int axis, Op op, U* out, int* status, cudaStream_t s, const char* what) {
  if (axis == 2) {
    k_rays_alongx<T, U, Op><<<(unsigned)ceil_div64(d.nz * d.ny, kRays), kRays, 0, s>>>(vol, d, op, out, status);
    return b2v_check_launch("k_rays_alongx");
  }
  int64_t nr = axis == 0 ? d.ny : d.nz;
  B2V_REQUIRE(nr <= 65535, B2V_ERR_ARG, "%s: more than 65535 output rows", what);
  dim3 grid((unsigned)ceil_div64(d.nx, 128), (unsigned)nr);
  k_rays_keepx<T, U, Op><<<grid, 128, 0, s>>>(vol, d, axis, op, out, status);
  return b2v_check_launch("k_rays_keepx");
}

template <typename T, typename U, typename Op>
int launch_z_partial(const T* vol, Dims d, Op op, uint32_t* state, int first, int last, U* out, int* status,
                     cudaStream_t s) {
  const dim3 grid((unsigned)ceil_div64(d.nx, 128), (unsigned)d.ny);
  k_rays_z_partial<T, U, Op><<<grid, 128, 0, s>>>(vol, d, op, state, first, last, out, status);
  return b2v_check_launch("k_rays_z_partial");
}

// ---- dtype dispatch: launch(vol, out, op) with the typed pointers and the operator -----------
// MIDA's (image, output) dtype pairs (mips_py.rs:161-202); wl and ww are taken as the image type
// (mips_py.rs:174-175). mm is the device (min, max) pair.
template <typename Launch>
int dispatch_mida(const void* img, int dtype, void* out, int out_dtype, double wl, double ww, const float* mm,
                  Launch&& launch) {
  auto with = [&](auto t, auto u) {
    using T = decltype(t);
    using U = decltype(u);
    return launch((const T*)img, (U*)out, MidaOp<T, U>{mm, (float)(T)wl, (float)(T)ww});
  };
  if (dtype == B2V_I16 && out_dtype == B2V_I16) return with(int16_t(), int16_t());
  if (dtype == B2V_U8 && out_dtype == B2V_U8) return with(uint8_t(), uint8_t());
  if (dtype == B2V_F64 && out_dtype == B2V_U8) return with(double(), uint8_t());
  B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
}

// LMIP takes int16, uint8 or float64, the output of the same dtype, tmin and tmax as that dtype.
template <typename Launch>
int dispatch_lmip(const void* img, int dtype, void* out, double tmin, double tmax, Launch&& launch) {
  auto with = [&](auto t) {
    using T = decltype(t);
    return launch((const T*)img, (T*)out, LmipOp<T>{(T)tmin, (T)tmax});
  };
  if (dtype == B2V_I16) return with(int16_t());
  if (dtype == B2V_U8) return with(uint8_t());
  if (dtype == B2V_F64) return with(double());
  B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
}

int finish_status(int* status_dev, cudaStream_t s, const char* what) {
  int st = 0;
  B2V_CUDA(cudaMemcpyAsync(&st, status_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(st == 0, B2V_ERR_RANGE, "%s: a value is not representable in the output type (the reference panics here)",
              what);
  return B2V_OK;
}

struct ProjWs {
  float* mm_f;   // [2]
  int* mm_i;     // [2]
  int* status;   // [1]
  void* minmax_ws;
};
ProjWs carve(void* ws) {
  ProjWs w;
  char* p = (char*)ws;
  w.mm_f = (float*)p;
  w.mm_i = (int*)(p + 64);
  w.status = (int*)(p + 128);
  w.minmax_ws = p + 256;
  return w;
}

bool check_axis_dims(int64_t dz, int64_t dy, int64_t dx, int axis) {
  return dz > 0 && dy > 0 && dx > 0 && axis >= 0 && axis <= 2;
}

}  // namespace

extern "C" int64_t b2v_proj_workspace_bytes(int64_t n) { return 256 + b2v_minmax_workspace_bytes(n); }

static int mida_impl(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double wl, double ww,
                     const float* minmax_dev, void* out, int out_dtype, void* workspace, void* stream) {
  B2V_REQUIRE(img && out && workspace, B2V_ERR_ARG, "mida: null pointer");
  B2V_REQUIRE(check_axis_dims(dz, dy, dx, axis), B2V_ERR_ARG, "mida: bad shape or axis");
  cudaStream_t s = (cudaStream_t)stream;
  ProjWs w = carve(workspace);
  Dims d = {dz, dy, dx};
  int rc;
  k_status_init<<<1, 1, 0, s>>>(w.status);
  if ((rc = b2v_check_launch("k_status_init"))) return rc;
  if (minmax_dev) {
    // the caller already knows the (global) min / max: a Z shard after its all_reduce
    B2V_CUDA(cudaMemcpyAsync(w.mm_f, minmax_dev, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  } else if ((rc = b2v_minmax_f32(img, dtype, dz * dy * dx, w.mm_f, w.minmax_ws, stream))) {
    return rc;
  }
  rc = dispatch_mida(img, dtype, out, out_dtype, wl, ww, w.mm_f, [&](auto* vol, auto* o, auto op) {
    return launch_rays(vol, d, axis, op, o, w.status, s, "mida");
  });
  if (rc) return rc;
  return finish_status(w.status, s, "mida");
}

extern "C" int b2v_mida(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double wl,
                        double ww, void* out, int out_dtype, void* workspace, void* stream) {
  return mida_impl(img, dtype, dz, dy, dx, axis, wl, ww, nullptr, out, out_dtype, workspace, stream);
}

extern "C" int b2v_mida_minmax(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double wl,
                               double ww, const float* minmax_dev, void* out, int out_dtype, void* workspace,
                               void* stream) {
  B2V_REQUIRE(minmax_dev, B2V_ERR_ARG, "mida_minmax: null min/max pointer");
  return mida_impl(img, dtype, dz, dy, dx, axis, wl, ww, minmax_dev, out, out_dtype, workspace, stream);
}

extern "C" int b2v_lmip(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double tmin,
                        double tmax, void* out, void* workspace, void* stream) {
  B2V_REQUIRE(img && out && workspace, B2V_ERR_ARG, "lmip: null pointer");
  B2V_REQUIRE(check_axis_dims(dz, dy, dx, axis), B2V_ERR_ARG, "lmip: bad shape or axis");
  cudaStream_t s = (cudaStream_t)stream;
  ProjWs w = carve(workspace);
  Dims d = {dz, dy, dx};
  int rc;
  k_status_init<<<1, 1, 0, s>>>(w.status);
  if ((rc = b2v_check_launch("k_status_init"))) return rc;
  return dispatch_lmip(img, dtype, out, tmin, tmax, [&](auto* vol, auto* o, auto op) {
    return launch_rays(vol, d, axis, op, o, w.status, s, "projection");
  });
}

// ---- the contour volume itself (mips.rs:238-242: tmp[z, y, x] = T(calc_fcm_intensity)) -------------
// One pass over the volume, HBM-bound on paper (sizeof(T) read + sizeof(T) written per voxel) and
// in practice bounded by the IEEE sqrt and division of every sample. A block owns a 64 x 8 (x, y)
// column and marches along z: the plane being differentiated sits in shared memory with its x / y
// halo (every voxel is read from global memory once, plus 1.3 halo reads per 64 x 8 plane), the
// z neighbours of a voxel are the thread's own previous / next values (registers). Central
// differences clamp at the volume faces exactly as finite_difference does (mips.rs:182-187).
constexpr int kFcmX = 64, kFcmY = 8, kFcmThreads = kFcmX * kFcmY;
constexpr int kFcmAhead = 2;   // planes in flight per block

template <typename T>
__global__ void __launch_bounds__(kFcmThreads, 3) k_fcm_volume(const T* __restrict__ vol, Dims d, float n, float dirx,
                                                           float diry, float dirz, int zchunk, T* __restrict__ out,
                                                           int* status) {
  __shared__ T s[2][kFcmY + 2][kFcmX + 2];
  const int tid = threadIdx.x, tx = tid % kFcmX, ty = tid / kFcmX;
  const int64_t x = (int64_t)blockIdx.x * kFcmX + tx, y = (int64_t)blockIdx.y * kFcmY + ty;
  const bool active = x < d.nx && y < d.ny;
  const int64_t cx = x < d.nx ? x : d.nx - 1, cy = y < d.ny ? y : d.ny - 1;
  const int64_t z0 = (int64_t)blockIdx.z * zchunk;
  const int64_t z1 = z0 + zchunk < d.nz ? z0 + zchunk : d.nz;
  if (z0 >= z1) return;
  // halo cell of this thread (the first 2 * 64 + 2 * 8 threads): row above / below, column left / right
  int hy = -1, hx = -1;   // shared-memory coordinates
  if (tid < kFcmX) { hy = 0; hx = tid + 1; }
  else if (tid < 2 * kFcmX) { hy = kFcmY + 1; hx = tid - kFcmX + 1; }
  else if (tid < 2 * kFcmX + kFcmY) { hy = tid - 2 * kFcmX + 1; hx = 0; }
  else if (tid < 2 * kFcmX + 2 * kFcmY) { hy = tid - 2 * kFcmX - kFcmY + 1; hx = kFcmX + 1; }
  int64_t gy = (int64_t)blockIdx.y * kFcmY + hy - 1, gx = (int64_t)blockIdx.x * kFcmX + hx - 1;
  gy = gy < 0 ? 0 : (gy > d.ny - 1 ? d.ny - 1 : gy);
  gx = gx < 0 ? 0 : (gx > d.nx - 1 ? d.nx - 1 : gx);
  const int64_t plane = d.ny * d.nx;
  const int64_t own = cy * d.nx + cx, hal = gy * d.nx + gx;
  // software pipeline: planes z + 1 .. z + kFcmAhead travel in registers (own voxel + halo cell of
  // each); the loads of plane z + kFcmAhead + 1 are issued before plane z is differentiated. The
  // kernel is bound by instruction issue (IEEE sqrt and division per sample: ~75 instructions per
  // voxel), not by bandwidth: pointers advance by one plane per step, no 64-bit products in the loop.
  T prev = vol[(z0 > 0 ? z0 - 1 : 0) * plane + own];
  T cur = vol[z0 * plane + own];
  T pf[kFcmAhead], hpf[kFcmAhead];
  int64_t zl = z0;                               // plane the read pointers stand on
  const T* p_own = vol + z0 * plane + own;
  const T* p_hal = vol + z0 * plane + hal;
  auto advance = [&]() { if (zl + 1 < d.nz) { ++zl; p_own += plane; p_hal += plane; } };   // clamps at the last plane
#pragma unroll
  for (int k = 0; k < kFcmAhead; ++k) {
    advance();
    pf[k] = *p_own;
    hpf[k] = 0;
    if (hy >= 0) hpf[k] = *p_hal;
  }
  int b = 0;
  s[0][ty + 1][tx + 1] = cur;
  if (hy >= 0) s[0][hy][hx] = vol[z0 * plane + hal];
  __syncthreads();
  T* p_out = out + z0 * plane + y * d.nx + x;
  for (int64_t z = z0; z < z1; ++z, p_out += plane) {
    advance();
    const T nn = *p_own;
    T hnn = 0;
    if (hy >= 0) hnn = *p_hal;
    const T nxt = pf[0];
    if (active) {
      const float gxf = __fmul_rn(wrapdiff<T>(s[b][ty + 1][tx + 2], s[b][ty + 1][tx]), 0.5f);   // / (2.0 * h), h = 1
      const float gyf = __fmul_rn(wrapdiff<T>(s[b][ty + 2][tx + 1], s[b][ty][tx + 1]), 0.5f);
      const float gzf = __fmul_rn(wrapdiff<T>(nxt, prev), 0.5f);
      const float gm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gxf, gxf), __fmul_rn(gyf, gyf)), __fmul_rn(gzf, gzf)));
      float val = 0.0f;
      if (gm != 0.0f) {
        const float dd = __fadd_rn(__fadd_rn(__fmul_rn(gxf, dirx), __fmul_rn(gyf, diry)), __fmul_rn(gzf, dirz));
        const float base = __fsub_rn(1.0f, fabsf(__fdiv_rn(dd, gm)));
        // powf of the reference is libm's (<1 ulp); a double pow rounded once is within the same ulp;
        // n == 1 (InVesalius' default border size) is exact in any libm; n == 2 is x * x here (glibc: <= 1 ulp off)
        const float sf = n == 1.0f ? base : (n == 2.0f ? __fmul_rn(base, base) : (float)pow((double)base, (double)n));
        val = __fmul_rn(gm, sf);
      }
      T o = 0;
      if (!cast_f32<T>(val, &o)) *status = B2V_ERR_RANGE;
      *p_out = o;
    }
    s[b ^ 1][ty + 1][tx + 1] = nxt;
    if (hy >= 0) s[b ^ 1][hy][hx] = hpf[0];
    __syncthreads();
    b ^= 1;
    prev = cur;
    cur = nxt;
#pragma unroll
    for (int k = 0; k + 1 < kFcmAhead; ++k) { pf[k] = pf[k + 1]; hpf[k] = hpf[k + 1]; }
    pf[kFcmAhead - 1] = nn;
    hpf[kFcmAhead - 1] = hnn;
  }
}

template <typename T>
int launch_fcm_volume(const T* img, Dims d, float n, int axis, T* tmp, int* status, cudaStream_t s) {
  const int64_t gx = ceil_div64(d.nx, kFcmX), gy = ceil_div64(d.ny, kFcmY);
  B2V_REQUIRE(gy <= 65535, B2V_ERR_ARG, "fcm_volume: more than 524280 rows");
  int64_t nchunk = ceil_div64((int64_t)b2v_sm_count() * 4 * 16, gx * gy);   // >= 16 waves of blocks: short tail
  if (nchunk < 1) nchunk = 1;
  if (nchunk > d.nz) nchunk = d.nz;
  const int zchunk = (int)ceil_div64(d.nz, nchunk);
  nchunk = ceil_div64(d.nz, zchunk);
  B2V_REQUIRE(nchunk <= 65535, B2V_ERR_ARG, "fcm_volume: too many z chunks");
  k_fcm_volume<T><<<dim3((unsigned)gx, (unsigned)gy, (unsigned)nchunk), kFcmThreads, 0, s>>>(
      img, d, n, axis == 2 ? 1.0f : 0.0f, axis == 1 ? 1.0f : 0.0f, axis == 0 ? 1.0f : 0.0f, zchunk, tmp, status);
  return b2v_check_launch("k_fcm_volume");
}

static int fcm_volume_impl(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, float n, int axis, void* tmp,
                           int* status, cudaStream_t s) {
  Dims d = {dz, dy, dx};
  if (dtype == B2V_I16) return launch_fcm_volume<int16_t>((const int16_t*)img, d, n, axis, (int16_t*)tmp, status, s);
  if (dtype == B2V_U8) return launch_fcm_volume<uint8_t>((const uint8_t*)img, d, n, axis, (uint8_t*)tmp, status, s);
  if (dtype == B2V_F64) return launch_fcm_volume<double>((const double*)img, d, n, axis, (double*)tmp, status, s);
  B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
}

extern "C" int b2v_fcm_volume(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, float n, int axis,
                              void* tmp, void* workspace, void* stream) {
  B2V_REQUIRE(img && tmp && workspace, B2V_ERR_ARG, "fcm_volume: null pointer");
  B2V_REQUIRE(check_axis_dims(dz, dy, dx, axis), B2V_ERR_ARG, "fcm_volume: bad shape or axis");
  cudaStream_t s = (cudaStream_t)stream;
  ProjWs w = carve(workspace);
  int rc;
  k_status_init<<<1, 1, 0, s>>>(w.status);
  if ((rc = b2v_check_launch("k_status_init"))) return rc;
  if ((rc = fcm_volume_impl(img, dtype, dz, dy, dx, n, axis, tmp, w.status, s))) return rc;
  return finish_status(w.status, s, "fast_countour_mip");
}

static int64_t dtype_bytes(int dtype) { return dtype == B2V_I16 ? 2 : (dtype == B2V_U8 ? 1 : 8); }

// workspace of b2v_fast_countour_mip: [projection workspace | contour volume | MaxIP workspace]
extern "C" int64_t b2v_fcm_workspace_bytes(int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, int tmip) {
  if (dz <= 0 || dy <= 0 || dx <= 0) return 0;
  const int64_t n = dz * dy * dx;
  return align256(b2v_proj_workspace_bytes(n)) + align256(n * dtype_bytes(dtype)) +
         (tmip == 0 ? align256(b2v_mip_workspace_bytes(dtype, dz, dy, dx, axis, 0)) : 0) + 256;
}

extern "C" int b2v_fast_countour_mip(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, float n,
                                     int axis, double wl, double ww, int tmip, void* out, void* workspace,
                                     void* stream) {
  // As the reference does (mips.rs:236-278): the contour volume first, then the projection of it.
  // workspace: b2v_fcm_workspace_bytes.
  B2V_REQUIRE(img && out && workspace, B2V_ERR_ARG, "fast_countour_mip: null pointer");
  B2V_REQUIRE(check_axis_dims(dz, dy, dx, axis), B2V_ERR_ARG, "fast_countour_mip: bad shape or axis");
  B2V_REQUIRE(tmip >= 0 && tmip <= 2, B2V_ERR_ARG, "fast_countour_mip: tmip must be 0, 1 or 2");
  B2V_REQUIRE(dtype == B2V_I16 || dtype == B2V_U8 || dtype == B2V_F64, B2V_ERR_ARG, "Invalid image or output type");
  // lmip(tmp, axis, 700, 3033): NumCast::from(700) does not fit uint8 -> the reference panics
  B2V_REQUIRE(!(tmip == 1 && dtype == B2V_U8), B2V_ERR_RANGE, "fast_countour_mip: LMIP bounds 700/3033 do not fit uint8");
  B2V_REQUIRE(!(tmip == 2 && dtype == B2V_F64), B2V_ERR_ARG,
              "fast_countour_mip: float64 contour-MIDA (float64 output) is not supported on the device");
  const int64_t nvox = dz * dy * dx;
  char* p = (char*)workspace;
  void* proj_ws = p;
  void* tmp = p + align256(b2v_proj_workspace_bytes(nvox));
  void* mip_ws = (char*)tmp + align256(nvox * dtype_bytes(dtype));
  int rc;
  if ((rc = b2v_fcm_volume(img, dtype, dz, dy, dx, n, axis, tmp, proj_ws, stream))) return rc;
  if (tmip == 0) return b2v_mip(tmp, dtype, dz, dy, dx, axis, 0 /* max */, out, mip_ws, stream);
  if (tmip == 1) return b2v_lmip(tmp, dtype, dz, dy, dx, axis, 700.0, 3033.0, out, proj_ws, stream);
  return b2v_mida(tmp, dtype, dz, dy, dx, axis, wl, ww, out, dtype, proj_ws, stream);
}

extern "C" int b2v_mida_z_partial(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, double wl, double ww,
                                  const float* minmax_dev, uint32_t* state, int first, int last, void* out,
                                  int out_dtype, void* workspace, void* stream) {
  B2V_REQUIRE(img && workspace && minmax_dev && state && (out || !last), B2V_ERR_ARG, "mida_z_partial: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG, "mida_z_partial: empty slab");
  B2V_REQUIRE(dy <= 65535, B2V_ERR_ARG, "mida_z_partial: more than 65535 output rows");
  cudaStream_t s = (cudaStream_t)stream;
  ProjWs w = carve(workspace);
  Dims d = {dz, dy, dx};
  int rc;
  k_status_init<<<1, 1, 0, s>>>(w.status);
  if ((rc = b2v_check_launch("k_status_init"))) return rc;
  B2V_CUDA(cudaMemcpyAsync(w.mm_f, minmax_dev, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  rc = dispatch_mida(img, dtype, out, out_dtype, wl, ww, w.mm_f, [&](auto* vol, auto* o, auto op) {
    return launch_z_partial(vol, d, op, state, first, last, o, w.status, s);
  });
  if (rc) return rc;
  return finish_status(w.status, s, "mida_z_partial");
}

extern "C" int b2v_lmip_z_partial(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, double tmin,
                                  double tmax, uint32_t* state, int first, int last, void* out, void* workspace,
                                  void* stream) {
  B2V_REQUIRE(img && workspace && state && (out || !last), B2V_ERR_ARG, "lmip_z_partial: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG, "lmip_z_partial: empty slab");
  B2V_REQUIRE(dy <= 65535, B2V_ERR_ARG, "lmip_z_partial: more than 65535 output rows");
  cudaStream_t s = (cudaStream_t)stream;
  ProjWs w = carve(workspace);
  Dims d = {dz, dy, dx};
  int rc;
  k_status_init<<<1, 1, 0, s>>>(w.status);
  if ((rc = b2v_check_launch("k_status_init"))) return rc;
  return dispatch_lmip(img, dtype, out, tmin, tmax, [&](auto* vol, auto* o, auto op) {
    return launch_z_partial(vol, d, op, state, first, last, o, w.status, s);
  });
}
