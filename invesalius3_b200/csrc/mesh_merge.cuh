// vtkCleanPolyData's point merge at tolerance 0 (vtkMergePoints), shared by the surface tools that renumber
// a mesh's points (visibility.cu, clean.cu). Every name is in an anonymous namespace, so each translation unit
// has its own copy.
//
//   merge_slots      the size of the open-addressing table: a power of two, at least 2 V and 1024.
//   k_merge_insert   one thread per point: exactly coincident points share one slot of the table (keys: the
//                    coordinate bits with -0 read as +0, compared with float ==, so a point with a NaN
//                    coordinate merges with no other point); rep[k] is point k's slot.
//   note_first_use   atomicMin of a corner index on its point's slot: after a pass over the corners, first[s]
//                    is the first corner (in traversal order) that uses slot s.
//   is_first_use     whether a corner is that first corner. Exclusive scans of these flags, in corner order,
//                    number the output points in order of first use.
#pragma once
#include "b2v_common.cuh"

namespace {

inline uint64_t merge_slots(int64_t nv) {
  uint64_t h = 1024;
  while (h < 2 * (uint64_t)nv) h <<= 1;
  return h;
}

__device__ __forceinline__ uint32_t canon_bits(float f) { return __float_as_uint(f == 0.0f ? 0.0f : f); }

__device__ __forceinline__ uint64_t vhash(uint32_t a, uint32_t b, uint32_t c) {
  uint64_t h = (uint64_t)a * 0x9E3779B97F4A7C15ull ^ (uint64_t)b * 0xC2B2AE3D27D4EB4Full ^ (uint64_t)c * 0x165667B19E3779F9ull;
  h ^= h >> 31;
  h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 29;
  return h;
}

// slots [hmask + 1] start at -1 (merge_reset)
__global__ void __launch_bounds__(256) k_merge_insert(const float* __restrict__ v, int64_t nv, uint64_t hmask,
                                                      int32_t* slots, uint32_t* __restrict__ rep) {
  for (int64_t k = gtid(); k < nv; k += gstride()) {
    const float x = v[3 * k], y = v[3 * k + 1], z = v[3 * k + 2];
    uint64_t h = vhash(canon_bits(x), canon_bits(y), canon_bits(z)) & hmask;
    for (;;) {
      const int32_t old = atomicCAS(&slots[h], -1, (int32_t)k);
      if (old == -1) break;
      if (v[3 * (int64_t)old] == x && v[3 * (int64_t)old + 1] == y && v[3 * (int64_t)old + 2] == z) break;
      h = (h + 1) & hmask;
    }
    rep[k] = (uint32_t)h;
  }
}

__device__ __forceinline__ void note_first_use(unsigned long long* first, uint32_t slot, unsigned long long corner) {
  unsigned long long* f = first + slot;
  if (corner < *f) atomicMin(f, corner);
}

__device__ __forceinline__ bool is_first_use(const unsigned long long* __restrict__ first, uint32_t slot,
                                             unsigned long long corner) {
  return first[slot] == corner;
}

// empties the table (slots [H] = -1) and the first uses (first [H] = ~0: no corner yet)
inline int merge_reset(int32_t* slots, unsigned long long* first, uint64_t H, cudaStream_t s) {
  B2V_CUDA(cudaMemsetAsync(slots, 0xff, H * 4, s));
  B2V_CUDA(cudaMemsetAsync(first, 0xff, H * 8, s));
  return B2V_OK;
}

// merges the points v [nv][3] into slots / rep (nv > 0)
inline int merge_points(const float* v, int64_t nv, uint64_t hmask, int32_t* slots, uint32_t* rep, cudaStream_t s) {
  k_merge_insert<<<b2v_grid(nv, 256, 16), 256, 0, s>>>(v, nv, hmask, slots, rep);
  return b2v_check_launch("k_merge_insert");
}

}  // namespace
