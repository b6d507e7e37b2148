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
