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
// One ray per thread. Rays along z or y (axis 0/1) keep x contiguous across the threads
// of a warp, so every step is a coalesced row access; rays along x (axis 2) are staged
// through a padded shared-memory tile (128 rays x 32 samples) that is loaded row-wise
// (coalesced) and walked column-wise (bank-conflict free). A block stops loading as soon
// as all of its rays have terminated (alpha >= 1 in MIDA, first local maximum in LMIP).
// HBM: 2 B/voxel for the ray pass + 2 B/voxel for the global min/max pass MIDA needs.
//
// The contour variants never materialise the reference's temp volume: a sampler computes
// the T-typed contour intensity of a voxel on the fly from its six neighbours.
#include <math.h>
#include <stdlib.h>

#include "b2v_common.cuh"

namespace {

struct Dims {
  int64_t nz, ny, nx;
};

// ---- samplers -----------------------------------------------------------------------------
template <typename T>
struct PlainSampler {
  static constexpr int kBatch = 8;   // samples fetched ahead of the recurrence (plain loads)
  static constexpr bool kLinear = true;   // a sample is vol[flat index]: rays advance a pointer
  const T* __restrict__ vol;
  Dims d;
  __device__ __forceinline__ T at(int64_t z, int64_t y, int64_t x, int* status) const {
    return vol[(z * d.ny + y) * d.nx + x];
  }
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
  float img_min, range, inv, wl, ww;
  float fmax, alpha_p, colour_p, final_colour;
  Window win;
  __device__ __forceinline__ void init() {
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

template <typename T>
struct MaxOp {  // fold_axis with Bounded::min_value() (mips.rs:250-254)
  T m;
  __device__ __forceinline__ void init() {}
  __device__ __forceinline__ void first(T v) { m = v; }
  __device__ __forceinline__ bool step(T v) {
    if (v > m) m = v;
    return false;
  }
  __device__ __forceinline__ bool result(T* o) const {
    *o = m;
    return true;
  }
};

// ---- ray walkers ---------------------------------------------------------------------------
// One ray of a keep-x kernel (axis 0: along z, axis 1: along y). For a plain volume the ray is
// a pointer advanced by a constant stride; kBatch samples are fetched before any of them is
// consumed, because the recurrence is a long dependent chain the loads must not wait for. The
// walk stops at the first sample whose step() reports the ray finished.
template <typename T, typename S, typename Op>
__device__ __forceinline__ bool walk_keepx(const S& smp, int axis, int64_t r, int64_t x, int64_t n_l, Op& op, int* st) {
  if constexpr (S::kLinear) {
    constexpr int B = S::kBatch;
    const int64_t plane = smp.d.ny * smp.d.nx;
    const int64_t stride = axis == 0 ? plane : smp.d.nx;
    const T* __restrict__ p = smp.vol + (axis == 0 ? r * smp.d.nx + x : r * plane + x);
    int64_t l0 = 0;
    for (; l0 + B <= n_l; l0 += B) {
      T v[B];
#pragma unroll
      for (int k = 0; k < B; ++k) v[k] = p[k * stride];
      p += B * stride;
#pragma unroll
      for (int k = 0; k < B; ++k)
        if (op.step(v[k])) return true;
    }
    for (; l0 < n_l; ++l0, p += stride)
      if (op.step(*p)) return true;
  } else {
    for (int64_t l = 0; l < n_l; ++l) {
      const T v = axis == 0 ? smp.at(l, r, x, st) : smp.at(r, l, x, st);
      if (op.step(v)) return true;
    }
  }
  return false;
}

// axis 0: out[y][x], ray along z; axis 1: out[z][x], ray along y. One thread per (r, x).
template <typename T, typename U, typename S, typename Op>
__global__ void __launch_bounds__(128) k_rays_keepx(S smp, int axis, Op op0, U* __restrict__ out, int* status) {
  const Dims d = smp.d;
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = blockIdx.y;
  if (x >= d.nx) return;
  const int64_t n_l = axis == 0 ? d.nz : d.ny;
  Op op = op0;
  op.init();
  int st = 0;
  {
    T v0 = axis == 0 ? smp.at(0, r, x, &st) : smp.at(r, 0, x, &st);
    op.first(v0);
  }
  walk_keepx<T>(smp, axis, r, x, n_l, op, &st);
  U o;
  if (op.result(&o)) out[r * d.nx + x] = o; else st = B2V_ERR_RANGE;
  if (st) *status = st;
}

// axis 2: out[z][y], ray along x. 128 rays per block, 32 samples per tile.
constexpr int kRays = 128, kChunk = 32;
template <typename T> struct Pitch { static constexpr int value = kChunk + 4 / sizeof(T) * 1; };
template <> struct Pitch<int16_t> { static constexpr int value = kChunk + 2; };   // 17 words
template <> struct Pitch<uint8_t> { static constexpr int value = kChunk + 4; };   // 9 words
template <> struct Pitch<double> { static constexpr int value = kChunk + 1; };

// Stage the 32-sample segments [x0, x0+32) of kRays consecutive rows in shared memory. A plain
// int16 volume with even rows moves two samples per lane (half a warp per row, 64 B each);
// otherwise one sample per lane (a warp per row), through the sampler.
template <typename T, typename S>
__device__ __forceinline__ void load_tile(const S& smp, T (*tile)[Pitch<T>::value], int64_t row0, int64_t nrows,
                                          int64_t x0, int lane, int warp, int* st) {
  const Dims d = smp.d;
  if constexpr (S::kLinear && sizeof(T) == 2) {
    if ((d.nx & 1) == 0 && (reinterpret_cast<uintptr_t>(smp.vol) & 3) == 0) {
      const int half = lane >> 4, l16 = lane & 15;
      const int64_t x = x0 + 2 * l16;
      const bool xin = x < d.nx;
      const T* p = smp.vol + (row0 + warp * 2 + half) * d.nx + x;
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
    if (row < nrows && x < d.nx) {
      if constexpr (S::kLinear) {
        v = smp.vol[row * d.nx + x];
      } else {
        const int64_t z = row / d.ny, y = row - z * d.ny;
        v = smp.at(z, y, x, st);
      }
    }
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

template <typename T, typename U, typename S, typename Op>
__global__ void __launch_bounds__(kRays) k_rays_alongx(S smp, Op op0, U* __restrict__ out, int* status) {
  __shared__ __align__(16) T tile[kRays][Pitch<T>::value];
  const Dims d = smp.d;
  const int64_t nrows = d.nz * d.ny;
  const int64_t row0 = (int64_t)blockIdx.x * kRays;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t myrow = row0 + tid;
  const bool live = myrow < nrows;
  Op op = op0;
  op.init();
  int st = 0;
  bool done = !live;
  for (int64_t x0 = 0; x0 < d.nx; x0 += kChunk) {
    load_tile<T>(smp, tile, row0, nrows, x0, lane, warp, &st);
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
    if (op.result(&o)) out[myrow] = o; else st = B2V_ERR_RANGE;
  }
  if (st) *status = st;
}

// ---- rays along x, int16: rows staged by the TMA engine ---------------------------------------------
// cp.async.bulk (1-D bulk tensor copy, global -> shared, completion counted on an mbarrier): every
// thread asks the copy engine for the next 64-sample segment (128 B) of ITS ray and goes back to
// the float32 recurrence; no thread spends issue slots on loads, and the segment after next is in
// flight while the current one is consumed (two stages). Rows sit 144 B apart in shared memory, so
// the 16-byte reads of eight consecutive threads fall into eight different bank groups.
// Needs 16-byte aligned rows (nx % 8 == 0, aligned base); otherwise the lane-load kernels above run.
constexpr int kTmaChunk = 64;                                  // samples per stage and ray
constexpr int kTmaPitch = kTmaChunk * 2 + 16;                  // bytes between rows in shared memory

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  }
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// the block's 128 rays through `op` (one per thread); returns false if a result does not fit
template <typename U, typename Op>
__device__ __forceinline__ void rays_alongx_tma(const int16_t* __restrict__ vol, Dims d, Op& op, bool call_first,
                                                U* __restrict__ out, int* status) {
  __shared__ __align__(16) unsigned char stage[2][kRays * kTmaPitch];
  __shared__ __align__(8) uint64_t bar[2];
  const int64_t nrows = d.nz * d.ny;
  const int tid = threadIdx.x;
  const int64_t myrow = (int64_t)blockIdx.x * kRays + tid;
  const bool live = myrow < nrows;
  const int nchunks = (int)ceil_div64(d.nx, kTmaChunk);
  if (tid == 0) {
    mbar_init(&bar[0], kRays);
    mbar_init(&bar[1], kRays);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int16_t* row = vol + (live ? myrow : 0) * d.nx;
  auto issue = [&](int k) {
    const int b = k & 1;
    const int64_t x0 = (int64_t)k * kTmaChunk;
    const uint32_t bytes = live ? (uint32_t)(((d.nx - x0) < kTmaChunk ? (d.nx - x0) : kTmaChunk) * 2) : 0u;
    mbar_arrive_expect_tx(&bar[b], bytes);
    if (bytes) tma_load_1d(&stage[b][tid * kTmaPitch], row + x0, bytes, &bar[b]);
  };
  issue(0);
  if (nchunks > 1) issue(1);
  int issued = nchunks > 1 ? 2 : 1, waited = 0;
  int st = 0;
  bool done = !live;
  for (int k = 0; k < nchunks; ++k) {
    const int b = k & 1;
    mbar_wait(&bar[b], (uint32_t)((k >> 1) & 1));
    ++waited;
    if (!done) {
      const uint4* w = reinterpret_cast<const uint4*>(&stage[b][tid * kTmaPitch]);
      const int lim = (int)((d.nx - (int64_t)k * kTmaChunk) < kTmaChunk ? (d.nx - (int64_t)k * kTmaChunk) : kTmaChunk);
      if (k == 0 && call_first) op.first((int16_t)(w[0].x & 0xffffu));
      for (int j = 0; j < kTmaChunk / 8 && !done; ++j) {
        const uint4 q = w[j];
        const uint32_t ww4[4] = {q.x, q.y, q.z, q.w};
        const int base = j * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (!done && base + e < lim) done = op.step((int16_t)((e & 1) ? (ww4[e >> 1] >> 16) : (ww4[e >> 1] & 0xffffu)));
        }
        if (base + 8 >= lim) break;
      }
    }
    const bool all_done = __syncthreads_and(done);   // also: everyone has finished reading stage b
    if (all_done) break;
    if (k + 2 < nchunks) { issue(k + 2); ++issued; }
  }
  // a segment may still be in flight when the rays ended early: let it land before the block leaves
  for (int k = waited; k < issued; ++k) mbar_wait(&bar[k & 1], (uint32_t)((k >> 1) & 1));
  if (live) {
    U o;
    if (op.result(&o)) out[myrow] = o; else st = B2V_ERR_RANGE;
  }
  if (st) *status = st;
}

template <typename U, typename Op>
__global__ void __launch_bounds__(kRays) k_rays_alongx_tma(const int16_t* __restrict__ vol, Dims d, Op op0,
                                                           U* __restrict__ out, int* status) {
  Op op = op0;
  op.init();
  rays_alongx_tma<U, Op>(vol, d, op, true, out, status);
}

// Measured at 1024^3, rays along x (tools/mida_axis2.py, two alternating runs on one H100 80GB HBM3 at
// a 400 W power limit): MIDA full rays 2.42-2.43 ms (TMA rows) vs 2.36-2.46 ms (lane loads), LMIP
// 0.13-0.19 vs 0.10-0.11 ms — 128-byte bulk copies per thread are too small for the copy engine to
// beat 32-bit lane loads here, and the rays are bound by the recurrence, not by the loads. The lane-load kernels stay the default; b2v_proj_set_tma(1) (or B2V_TMA=1) selects this path.
int g_proj_tma = -1;
inline bool tma_rows_ok(const void* vol, const Dims& d) {
  if (g_proj_tma < 0) g_proj_tma = getenv("B2V_TMA") != nullptr ? 1 : 0;
  return g_proj_tma == 1 && d.nx % 8 == 0 && (reinterpret_cast<uintptr_t>(vol) & 15u) == 0;
}

__global__ void k_status_init(int* status) { *status = 0; }

template <typename T, typename U, typename S, typename Op>
int launch_rays(S smp, int axis, Op op, U* out, int* status, cudaStream_t s) {
  const Dims d = smp.d;
  if (axis == 2) {
    int64_t nrows = d.nz * d.ny;
    if constexpr (S::kLinear && sizeof(T) == 2) {
      if (tma_rows_ok(smp.vol, d)) {
        k_rays_alongx_tma<U, Op><<<(unsigned)ceil_div64(nrows, kRays), kRays, 0, s>>>((const int16_t*)smp.vol, d, op, out,
                                                                                     status);
        return b2v_check_launch("k_rays_alongx_tma");
      }
    }
    k_rays_alongx<T, U, S, Op><<<(unsigned)ceil_div64(nrows, kRays), kRays, 0, s>>>(smp, op, out, status);
    return b2v_check_launch("k_rays_alongx");
  }
  int64_t nr = axis == 0 ? d.ny : d.nz;
  B2V_REQUIRE(nr <= 65535, B2V_ERR_ARG, "projection: more than 65535 output rows");
  dim3 grid((unsigned)ceil_div64(d.nx, 128), (unsigned)nr);
  k_rays_keepx<T, U, S, Op><<<grid, 128, 0, s>>>(smp, axis, op, out, status);
  return b2v_check_launch("k_rays_keepx");
}

// MidaOp needs (min, range, 1/range) which live on the device: a tiny kernel finishes the
// operator there instead of synchronising.
template <typename T, typename U, typename S>
__global__ void __launch_bounds__(128) k_mida_keepx(S smp, int axis, const float* __restrict__ mm, float wl, float ww,
                                                    U* __restrict__ out, int* status);

template <typename T, typename U>
__device__ __forceinline__ MidaOp<T, U> make_mida(const float* mm, float wl, float ww) {
  MidaOp<T, U> op;
  op.img_min = mm[0];
  op.range = __fsub_rn(mm[1], mm[0]);
  op.inv = __fdiv_rn(1.0f, op.range);
  op.wl = wl;
  op.ww = ww;
  return op;
}

template <typename T, typename U, typename S>
__global__ void __launch_bounds__(128) k_mida_keepx(S smp, int axis, const float* __restrict__ mm, float wl, float ww,
                                                    U* __restrict__ out, int* status) {
  const Dims d = smp.d;
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = blockIdx.y;
  if (x >= d.nx) return;
  const int64_t n_l = axis == 0 ? d.nz : d.ny;
  MidaOp<T, U> op = make_mida<T, U>(mm, wl, ww);
  op.init();
  int st = 0;
  walk_keepx<T>(smp, axis, r, x, n_l, op, &st);
  U o;
  if (op.result(&o)) out[r * d.nx + x] = o; else st = B2V_ERR_RANGE;
  if (st) *status = st;
}

template <typename T, typename U, typename S>
__global__ void __launch_bounds__(kRays) k_mida_alongx(S smp, const float* __restrict__ mm, float wl, float ww,
                                                       U* __restrict__ out, int* status) {
  __shared__ __align__(16) T tile[kRays][Pitch<T>::value];
  const Dims d = smp.d;
  const int64_t nrows = d.nz * d.ny;
  const int64_t row0 = (int64_t)blockIdx.x * kRays;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t myrow = row0 + tid;
  const bool live = myrow < nrows;
  MidaOp<T, U> op = make_mida<T, U>(mm, wl, ww);
  op.init();
  int st = 0;
  bool done = !live;
  for (int64_t x0 = 0; x0 < d.nx; x0 += kChunk) {
    load_tile<T>(smp, tile, row0, nrows, x0, lane, warp, &st);
    __syncthreads();
    if (!done) {
      int lim = (int)((d.nx - x0) < kChunk ? (d.nx - x0) : kChunk);
      done = consume_tile<T>(tile[tid], lim, op);
    }
    if (__syncthreads_and(done)) break;
  }
  if (live) {
    U o;
    if (op.result(&o)) out[myrow] = o; else st = B2V_ERR_RANGE;
  }
  if (st) *status = st;
}

template <typename U>
__global__ void __launch_bounds__(kRays) k_mida_alongx_tma(const int16_t* __restrict__ vol, Dims d,
                                                           const float* __restrict__ mm, float wl, float ww,
                                                           U* __restrict__ out, int* status) {
  MidaOp<int16_t, U> op = make_mida<int16_t, U>(mm, wl, ww);
  op.init();
  rays_alongx_tma<U, MidaOp<int16_t, U>>(vol, d, op, false, out, status);
}

template <typename T, typename U, typename S>
int launch_mida(S smp, int axis, const float* mm, float wl, float ww, U* out, int* status, cudaStream_t s) {
  const Dims d = smp.d;
  if (axis == 2) {
    if constexpr (S::kLinear && sizeof(T) == 2) {
      if (tma_rows_ok(smp.vol, d)) {
        k_mida_alongx_tma<U><<<(unsigned)ceil_div64(d.nz * d.ny, kRays), kRays, 0, s>>>((const int16_t*)smp.vol, d, mm, wl,
                                                                                      ww, out, status);
        return b2v_check_launch("k_mida_alongx_tma");
      }
    }
    k_mida_alongx<T, U, S><<<(unsigned)ceil_div64(d.nz * d.ny, kRays), kRays, 0, s>>>(smp, mm, wl, ww, out, status);
    return b2v_check_launch("k_mida_alongx");
  }
  int64_t nr = axis == 0 ? d.ny : d.nz;
  B2V_REQUIRE(nr <= 65535, B2V_ERR_ARG, "mida: more than 65535 output rows");
  dim3 grid((unsigned)ceil_div64(d.nx, 128), (unsigned)nr);
  k_mida_keepx<T, U, S><<<grid, 128, 0, s>>>(smp, axis, mm, wl, ww, out, status);
  return b2v_check_launch("k_mida_keepx");
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

// ---- rays along z over ONE Z shard (dist: MIDA / LMIP with rays that cross the shards) ------
// The ray of pixel (y, x) starts from the state the previous shard left (or is started here),
// walks this slab and leaves its state for the next shard; the last shard writes the pixel.
// The per-ray operation order is that of the whole-volume walk, so the result is bit-exact.
template <typename T, typename U, typename Op>
__device__ __forceinline__ void ray_z_partial(const PlainSampler<T>& smp, Op& op, uint32_t* state, int first, int last,
                                              U* out, int* status) {
  const Dims d = smp.d;
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t y = blockIdx.y;
  if (x >= d.nx) return;
  const int64_t plane = d.ny * d.nx, i = y * d.nx + x;
  int st = 0;
  bool done = false;
  op.init();
  if (first) op.first(smp.vol[i]);
  else op.load(state, i, plane, &done);
  if (!done) done = walk_keepx<T>(smp, 0, y, x, d.nz, op, &st);
  op.store(state, i, plane, done);
  if (last) {
    U o;
    if (op.result(&o)) out[i] = o; else st = B2V_ERR_RANGE;
  }
  if (st) *status = st;
}

template <typename T, typename U>
__global__ void __launch_bounds__(128) k_mida_z_partial(PlainSampler<T> smp, const float* __restrict__ mm, float wl,
                                                        float ww, uint32_t* state, int first, int last,
                                                        U* __restrict__ out, int* status) {
  MidaOp<T, U> op = make_mida<T, U>(mm, wl, ww);
  ray_z_partial<T, U>(smp, op, state, first, last, out, status);
}

template <typename T>
__global__ void __launch_bounds__(128) k_lmip_z_partial(PlainSampler<T> smp, LmipOp<T> op0, uint32_t* state, int first,
                                                        int last, T* __restrict__ out, int* status) {
  LmipOp<T> op = op0;
  ray_z_partial<T, T>(smp, op, state, first, last, out, status);
}

}  // namespace

extern "C" void b2v_proj_set_tma(int on) { g_proj_tma = on ? 1 : 0; }

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
  if (dtype == B2V_I16 && out_dtype == B2V_I16) {
    PlainSampler<int16_t> smp = {(const int16_t*)img, d};
    rc = launch_mida<int16_t, int16_t>(smp, axis, w.mm_f, (float)(int16_t)wl, (float)(int16_t)ww, (int16_t*)out,
                                       w.status, s);
  } else if (dtype == B2V_U8 && out_dtype == B2V_U8) {
    PlainSampler<uint8_t> smp = {(const uint8_t*)img, d};
    rc = launch_mida<uint8_t, uint8_t>(smp, axis, w.mm_f, (float)(uint8_t)wl, (float)(uint8_t)ww, (uint8_t*)out,
                                       w.status, s);
  } else if (dtype == B2V_F64 && out_dtype == B2V_U8) {
    PlainSampler<double> smp = {(const double*)img, d};
    rc = launch_mida<double, uint8_t>(smp, axis, w.mm_f, (float)wl, (float)ww, (uint8_t*)out, w.status, s);
  } else {
    B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
  }
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
  if (dtype == B2V_I16) {
    PlainSampler<int16_t> smp = {(const int16_t*)img, d};
    LmipOp<int16_t> op;
    op.tmin = (int16_t)tmin; op.tmax = (int16_t)tmax;
    rc = launch_rays<int16_t, int16_t>(smp, axis, op, (int16_t*)out, w.status, s);
  } else if (dtype == B2V_U8) {
    PlainSampler<uint8_t> smp = {(const uint8_t*)img, d};
    LmipOp<uint8_t> op;
    op.tmin = (uint8_t)tmin; op.tmax = (uint8_t)tmax;
    rc = launch_rays<uint8_t, uint8_t>(smp, axis, op, (uint8_t*)out, w.status, s);
  } else if (dtype == B2V_F64) {
    PlainSampler<double> smp = {(const double*)img, d};
    LmipOp<double> op;
    op.tmin = tmin; op.tmax = tmax;
    rc = launch_rays<double, double>(smp, axis, op, (double*)out, w.status, s);
  } else {
    B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
  }
  return rc;
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
static int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }

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
  const dim3 grid((unsigned)ceil_div64(dx, 128), (unsigned)dy);
  if (dtype == B2V_I16 && out_dtype == B2V_I16) {
    PlainSampler<int16_t> smp = {(const int16_t*)img, d};
    k_mida_z_partial<int16_t, int16_t><<<grid, 128, 0, s>>>(smp, w.mm_f, (float)(int16_t)wl, (float)(int16_t)ww, state,
                                                            first, last, (int16_t*)out, w.status);
  } else if (dtype == B2V_U8 && out_dtype == B2V_U8) {
    PlainSampler<uint8_t> smp = {(const uint8_t*)img, d};
    k_mida_z_partial<uint8_t, uint8_t><<<grid, 128, 0, s>>>(smp, w.mm_f, (float)(uint8_t)wl, (float)(uint8_t)ww, state,
                                                          first, last, (uint8_t*)out, w.status);
  } else if (dtype == B2V_F64 && out_dtype == B2V_U8) {
    PlainSampler<double> smp = {(const double*)img, d};
    k_mida_z_partial<double, uint8_t><<<grid, 128, 0, s>>>(smp, w.mm_f, (float)wl, (float)ww, state, first, last,
                                                         (uint8_t*)out, w.status);
  } else {
    B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
  }
  if ((rc = b2v_check_launch("k_mida_z_partial"))) return rc;
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
  const dim3 grid((unsigned)ceil_div64(dx, 128), (unsigned)dy);
  if (dtype == B2V_I16) {
    PlainSampler<int16_t> smp = {(const int16_t*)img, d};
    LmipOp<int16_t> op;
    op.tmin = (int16_t)tmin; op.tmax = (int16_t)tmax;
    k_lmip_z_partial<int16_t><<<grid, 128, 0, s>>>(smp, op, state, first, last, (int16_t*)out, w.status);
  } else if (dtype == B2V_U8) {
    PlainSampler<uint8_t> smp = {(const uint8_t*)img, d};
    LmipOp<uint8_t> op;
    op.tmin = (uint8_t)tmin; op.tmax = (uint8_t)tmax;
    k_lmip_z_partial<uint8_t><<<grid, 128, 0, s>>>(smp, op, state, first, last, (uint8_t*)out, w.status);
  } else if (dtype == B2V_F64) {
    PlainSampler<double> smp = {(const double*)img, d};
    LmipOp<double> op;
    op.tmin = tmin; op.tmax = tmax;
    k_lmip_z_partial<double><<<grid, 128, 0, s>>>(smp, op, state, first, last, (double*)out, w.status);
  } else {
    B2V_REQUIRE(false, B2V_ERR_ARG, "Invalid image or output type");
  }
  return b2v_check_launch("k_lmip_z_partial");
}
