// b2v — volumetric compute core for the H100 (sm_90a).
// Shared device/host helpers for every translation unit of libb2v.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b2v.h"

#define B2V_SM_COUNT_FALLBACK 132

// ---- error plumbing -------------------------------------------------------
void b2v_set_error(const char* fmt, ...);
int b2v_check_launch(const char* what);  // cudaGetLastError -> status
int b2v_sm_count();                      // cached SM count of the current device

#define B2V_REQUIRE(cond, code, ...)   \
  do {                                 \
    if (!(cond)) {                     \
      b2v_set_error(__VA_ARGS__);      \
      return (code);                   \
    }                                  \
  } while (0)

#define B2V_CUDA(call)                                                        \
  do {                                                                        \
    cudaError_t e__ = (call);                                                 \
    if (e__ != cudaSuccess) {                                                 \
      b2v_set_error("%s failed: %s", #call, cudaGetErrorString(e__));         \
      return B2V_ERR_CUDA;                                                    \
    }                                                                         \
  } while (0)

static inline bool b2v_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- streaming 128-bit accessors -------------------------------------------
// Volumes are swept once per op: bypass L1 allocation on the read side and
// keep stores out of the way of whatever L2 still holds.
__device__ __forceinline__ int4 ld_stream(const int4* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ld_stream(const uint2* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_stream(uint2* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

// ---- packed int16 arithmetic (two voxels per 32-bit lane) -------------------
__device__ __forceinline__ uint32_t max_s16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("max.s16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ uint32_t min_s16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("min.s16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// four packed bytes -> 0x80 in every byte that is >= the (per-byte constant) threshold t4.
// Low seven bits: (x | 0x80) - t7 keeps bit 7 exactly when x7 >= t7 and never borrows across
// bytes; the top bit of x then decides alone (t >= 128: both needed, t < 128: either).
__device__ __forceinline__ uint32_t ge_flags_u8x4(uint32_t x, uint32_t t7, bool t_high) {
  const uint32_t d = (x | 0x80808080u) - t7;
  return (t_high ? (x & d) : (x | d)) & 0x80808080u;
}
// 0x80-per-byte flags -> 4 bits (byte 0 -> bit 0)
__device__ __forceinline__ uint32_t flags_to_nibble(uint32_t f) { return (((f >> 7) * 0x01020408u) >> 24) & 0xfu; }

// two packed int16 -> 0x8000 in every half that lies in [lo, hi] (lo2 / hi2 = the bound in both halves)
__device__ __forceinline__ uint32_t inrange_flags_s16x2(uint32_t w, uint32_t lo2, uint32_t hi2) {
  const uint32_t d = max_s16x2(min_s16x2(w, hi2), lo2) ^ w;   // half == 0  <=>  in range
  const uint32_t t = (d & 0x7fff7fffu) + 0x7fff7fffu;
  return ~(t | d | 0x7fff7fffu);
}
// four packed bytes -> 0x80 in every non-zero byte
__device__ __forceinline__ uint32_t nonzero_flags_u8x4(uint32_t x) {
  return (((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x) & 0x80808080u;
}

__host__ __device__ __forceinline__ int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- launch shapes and workspace layout -----------------------------------------
// Blocks for a grid-stride launch over `items` at `per_block` items a block: enough to cover them once,
// at most per_sm blocks per SM, and never 0 (a launch of 0 blocks fails).
static inline int b2v_grid(int64_t items, int per_block, int per_sm) {
  int64_t blocks = ceil_div64(items, per_block);
  const int64_t cap = (int64_t)b2v_sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

// workspace buffers start on 256-byte boundaries
static inline int64_t align256(int64_t bytes) { return (bytes + 255) & ~(int64_t)255; }

__device__ __forceinline__ int64_t gtid() { return (int64_t)blockIdx.x * blockDim.x + threadIdx.x; }
__device__ __forceinline__ int64_t gstride() { return (int64_t)gridDim.x * blockDim.x; }

namespace {
// a[0, n) = v, grid-stride (each translation unit has its own instantiations)
template <typename T>
__global__ void __launch_bounds__(256) k_fill(T* a, int64_t n, T v) {
  for (int64_t i = gtid(); i < n; i += gstride()) a[i] = v;
}
}  // namespace

// Block-wide sum of a block of 256 threads, returned to thread 0 (the other threads get 0). Every thread of
// the block calls it; s_w holds 8 words.
template <typename T>
__device__ __forceinline__ T block_sum(T x, T* s_w) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = x;
  __syncthreads();
  T t = 0;
  if (threadIdx.x == 0)
    for (int k = 0; k < 8; ++k) t += s_w[k];
  return t;
}

// Block-wide exclusive scan: returns x's prefix and stores the block total. Every thread of the block calls
// it; blockDim.x is a multiple of 32, and s_w holds blockDim.x / 32 words. A kernel whose blocks have fewer
// than 32 warps may say so in MaxWarps (a power of two), which shortens the scan of the warp sums.
template <typename T, int MaxWarps = 32>
__device__ __forceinline__ T block_exscan(T x, T* s_w, T* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T inc = x;
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s_w[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const int nw = blockDim.x >> 5;
    T v = lane < nw ? s_w[lane] : 0;
    for (int o = 1; o < MaxWarps; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += y;
    }
    if (lane < nw) s_w[lane] = v;
  }
  __syncthreads();
  const T base = wid ? s_w[wid - 1] : 0;
  *total = s_w[(blockDim.x >> 5) - 1];
  __syncthreads();
  return base + inc - x;
}

// ---- imagedata_utils.image_normalize ---------------------------------------------------
// One voxel of (image - imin) * scale + min_ in T's arithmetic (NumPy's, for a float32 or float64 image and
// Python-scalar bounds), stored with the C cast: truncated into int32, low 16 bits kept (the x86 cast).
template <typename T>
__device__ __forceinline__ int16_t normalize_i16(T v, T imin, T scale, T min_f) {
  return (int16_t)(int)((v - imin) * scale + min_f);
}

// ---- 3x3x3 structuring elements ---------------------------------------------------------
// A uint8 element [odz][ody][odx] of at most 3 voxels on each axis, centred at (odz / 2, ody / 2, odx / 2), as
// a 27-bit mask: bit (oz+1)*9 + (oy+1)*3 + (ox+1) stands for the offset (oz, oy, ox); bit 13 is the centre.
static inline uint32_t strct_mask(const uint8_t* st, int64_t odz, int64_t ody, int64_t odx) {
  uint32_t sb = 0;
  for (int64_t kk = 0; kk < odz; ++kk)
    for (int64_t jj = 0; jj < ody; ++jj)
      for (int64_t ii = 0; ii < odx; ++ii)
        if (st[(kk * ody + jj) * odx + ii]) {
          const int oz = (int)(kk - odz / 2), oy = (int)(jj - ody / 2), ox = (int)(ii - odx / 2);
          sb |= 1u << ((oz + 1) * 9 + (oy + 1) * 3 + (ox + 1));
        }
  return sb;
}

// the six face neighbours (0,0,+-1), (0,+-1,0), (+-1,0,0): generate_binary_structure(3, 1) without its centre
constexpr uint32_t kSB6 = (1u << 12) | (1u << 14) | (1u << 10) | (1u << 16) | (1u << 4) | (1u << 22);

// ---- triangle faces ---------------------------------------------------------------
// int32 or int64 ids, [T,3] or [T,4] with a leading 3 (the Mesh form), every id in [0, nv)
struct Faces {
  const void* p;
  int64_t nt;
  int cols;    // 3, or 4 with a leading 3
  int i64;
  int64_t nv;
};

enum : uint32_t { ST_BAD_FACE = 1u };   // status bit: some face failed load_face

// the three vertex ids of face t; false when the face is malformed (an index outside [0, nv) or a leading
// entry other than 3 in the [T, 4] form)
__device__ __forceinline__ bool load_face(const Faces& F, int64_t t, int64_t v[3]) {
  const int64_t base = t * F.cols;
  const int off = F.cols == 4 ? 1 : 0;
  if (F.i64) {
    const int64_t* f = (const int64_t*)F.p + base;
    if (off && f[0] != 3) return false;
    v[0] = f[off]; v[1] = f[off + 1]; v[2] = f[off + 2];
  } else {
    const int32_t* f = (const int32_t*)F.p + base;
    if (off && f[0] != 3) return false;
    v[0] = f[off]; v[1] = f[off + 1]; v[2] = f[off + 2];
  }
  return v[0] >= 0 && v[0] < F.nv && v[1] >= 0 && v[1] < F.nv && v[2] >= 0 && v[2] < F.nv;
}
