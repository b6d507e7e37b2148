// Threshold: int16 volume -> uint8 mask (255 inside [lo, hi], 0 outside), optionally
// keeping edit/watershed marker values of the previous mask.
// Reference semantics: invesalius/data/slice_.py:1238-1246 and :1722-1769.
//
// HBM-bound elementwise sweep: every thread turns 16 voxels (two 128-bit loads) into
// one 128-bit store; four such groups are in flight per thread. 3 B/voxel (4 B with
// marker preservation).
#include "b2v_common.cuh"

namespace {

// 0xFF in every byte of `x` that is zero, 0x00 elsewhere
__device__ __forceinline__ uint32_t zero_bytes_ff(uint32_t x) {
  return ((nonzero_flags_u8x4(x) ^ 0x80808080u) >> 7) * 0xffu;
}

// bytes of `m` equal to 1, 2, 253 or 254 -> 0xFF
__device__ __forceinline__ uint32_t marker_bytes_ff(uint32_t m) {
  uint32_t hi = (m >> 7) & 0x01010101u;
  uint32_t f = m ^ (hi * 0xffu);                            // 253->2, 254->1, byte < 128 now
  uint32_t h = ((f + 0x01010101u) >> 1) & 0x7f7f7f7fu;      // {1,2} -> 1
  return zero_bytes_ff(h ^ 0x01010101u);
}

// two packed int16 voxels -> 0xFFFF per half that lies in [lo, hi]
__device__ __forceinline__ uint32_t inrange_s16x2(uint32_t w, uint32_t lo2, uint32_t hi2) {
  return (inrange_flags_s16x2(w, lo2, hi2) >> 15) * 0xffffu;
}

__device__ __forceinline__ uint32_t thr4(uint32_t w0, uint32_t w1, uint32_t lo2, uint32_t hi2) {
  // bytes: voxel0 = low half of w0, voxel1 = high half of w0, voxel2/3 from w1
  return __byte_perm(inrange_s16x2(w0, lo2, hi2), inrange_s16x2(w1, lo2, hi2), 0x6420);
}

template <bool PRESERVE>
__device__ __forceinline__ uint4 thr16(const int4& a, const int4& b, uint32_t lo2, uint32_t hi2, uint32_t keep,
                                       const uint4& old) {
  uint4 r;
  r.x = thr4(a.x, a.y, lo2, hi2) & keep;
  r.y = thr4(a.z, a.w, lo2, hi2) & keep;
  r.z = thr4(b.x, b.y, lo2, hi2) & keep;
  r.w = thr4(b.z, b.w, lo2, hi2) & keep;
  if (PRESERVE) {
    uint32_t s;
    s = marker_bytes_ff(old.x); r.x = (r.x & ~s) | (old.x & s);
    s = marker_bytes_ff(old.y); r.y = (r.y & ~s) | (old.y & s);
    s = marker_bytes_ff(old.z); r.z = (r.z & ~s) | (old.z & s);
    s = marker_bytes_ff(old.w); r.w = (r.w & ~s) | (old.w & s);
  }
  return r;
}

__device__ __forceinline__ uint8_t thr1(int v, int lo, int hi, bool preserve, uint8_t old) {
  uint8_t r = (v >= lo && v <= hi) ? 255 : 0;
  if (preserve && (old == 1 || old == 2 || old == 253 || old == 254)) r = old;
  return r;
}

constexpr int kGroupsPerThread = 4;  // 4 x 16 voxels in flight per thread

template <bool PRESERVE>
__global__ void __launch_bounds__(256) k_threshold_vec(const int4* __restrict__ img, uint4* __restrict__ mask,
                                                       int64_t ngroups, uint32_t lo2, uint32_t hi2,
                                                       uint32_t keep) {
  // group g = 16 voxels = img[2g], img[2g+1] -> mask[g]
  int64_t base = (int64_t)blockIdx.x * (256 * kGroupsPerThread) + threadIdx.x;
  int4 a[kGroupsPerThread], b[kGroupsPerThread];
  uint4 o[kGroupsPerThread] = {};
#pragma unroll
  for (int k = 0; k < kGroupsPerThread; ++k) {
    int64_t g = base + (int64_t)k * 256;
    if (g < ngroups) {
      a[k] = ld_stream(img + 2 * g);
      b[k] = ld_stream(img + 2 * g + 1);
      if (PRESERVE) o[k] = ld_stream(reinterpret_cast<const uint4*>(mask) + g);
    }
  }
#pragma unroll
  for (int k = 0; k < kGroupsPerThread; ++k) {
    int64_t g = base + (int64_t)k * 256;
    if (g < ngroups) st_stream(mask + g, thr16<PRESERVE>(a[k], b[k], lo2, hi2, keep, o[k]));
  }
}

// scalar sweep over [i0, n): tails and unaligned buffers
__global__ void __launch_bounds__(256) k_threshold_scalar(const int16_t* __restrict__ img,
                                                          uint8_t* __restrict__ mask, int64_t i0, int64_t n,
                                                          int lo, int hi, int preserve) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = i0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    mask[i] = thr1(img[i], lo, hi, preserve, preserve ? mask[i] : 0);
}

// Padded Mask layout [dz+1][dy+1][dx+1]: one warp per image row, rows of one slice
// are consecutive in both arrays. The destination row start is byte-misaligned
// ((dx+1) pitch, +1 column), so lanes write single bytes; full 32-byte sectors are
// still assembled in L2 because a warp covers 32 consecutive bytes per step.
__global__ void __launch_bounds__(256) k_threshold_masklayout(const int16_t* __restrict__ img,
                                                              uint8_t* __restrict__ mask, int64_t dz, int64_t dy,
                                                              int64_t dx, int lo, int hi, int preserve,
                                                              int only_dirty) {
  int64_t nrows = dz * dy;
  int lane = threadIdx.x & 31;
  int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t prow = dx + 1, pplane = (dy + 1) * (dx + 1);
  for (int64_t r = warp; r < nrows; r += nwarps) {
    int64_t z = r / dy, y = r - z * dy;
    uint8_t* flag = mask + (z + 1) * pplane;
    if (only_dirty && *(volatile uint8_t*)flag != 0) continue;
    const int16_t* src = img + r * dx;
    uint8_t* dst = flag + (y + 1) * prow + 1;
    for (int64_t x = lane; x < dx; x += 32) dst[x] = thr1(src[x], lo, hi, preserve, preserve ? dst[x] : 0);
  }
}

// flags are written after every row of the pass has tested them
__global__ void k_set_axial_flags(uint8_t* mask, int64_t dz, int64_t pplane) {
  int64_t z = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (z < dz) mask[(z + 1) * pplane] = 1;
}

struct Range {
  int lo, hi;
  bool none;
};
Range clamp_range(int32_t lo, int32_t hi) {
  Range r;
  r.none = lo > hi || lo > 32767 || hi < -32768;
  r.lo = lo < -32768 ? -32768 : lo;
  r.hi = hi > 32767 ? 32767 : hi;
  if (r.none) {
    r.lo = 0;
    r.hi = 0;
  }
  return r;
}

}  // namespace

extern "C" int b2v_threshold_i16(const int16_t* img, int64_t n, int32_t lo, int32_t hi, uint8_t* mask,
                                 int preserve_markers, void* stream) {
  B2V_REQUIRE(img && mask, B2V_ERR_ARG, "threshold: null pointer");
  B2V_REQUIRE(n >= 0, B2V_ERR_ARG, "threshold: negative size");
  if (n == 0) return B2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  Range r = clamp_range(lo, hi);
  int rc;
  int64_t done = 0;
  if (b2v_aligned16(img) && b2v_aligned16(mask) && n >= 16) {
    int64_t ngroups = n / 16;
    uint32_t lo2 = (uint32_t)(uint16_t)r.lo * 0x00010001u, hi2 = (uint32_t)(uint16_t)r.hi * 0x00010001u;
    uint32_t keep = r.none ? 0u : 0xffffffffu;
    int64_t blocks = ceil_div64(ngroups, 256 * kGroupsPerThread);
    B2V_REQUIRE(blocks < (1ll << 31), B2V_ERR_ARG, "threshold: volume too large for one launch");
    if (preserve_markers)
      k_threshold_vec<true><<<(unsigned)blocks, 256, 0, s>>>((const int4*)img, (uint4*)mask, ngroups, lo2, hi2, keep);
    else
      k_threshold_vec<false><<<(unsigned)blocks, 256, 0, s>>>((const int4*)img, (uint4*)mask, ngroups, lo2, hi2, keep);
    if ((rc = b2v_check_launch("k_threshold_vec"))) return rc;
    done = ngroups * 16;
  }
  if (done < n) {
    // an empty range is expressed to the scalar kernel as lo > hi
    k_threshold_scalar<<<b2v_grid(n - done, 256, 16), 256, 0, s>>>(img, mask, done, n, r.none ? 1 : r.lo,
                                                                   r.none ? 0 : r.hi, preserve_markers);
    if ((rc = b2v_check_launch("k_threshold_scalar"))) return rc;
  }
  return B2V_OK;
}

extern "C" int b2v_threshold_i16_masklayout(const int16_t* img, int64_t dz, int64_t dy, int64_t dx, int32_t lo,
                                            int32_t hi, uint8_t* mask_padded, int preserve_markers,
                                            int only_dirty, void* stream) {
  B2V_REQUIRE(img && mask_padded, B2V_ERR_ARG, "threshold_masklayout: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG, "threshold_masklayout: empty volume");
  cudaStream_t s = (cudaStream_t)stream;
  Range r = clamp_range(lo, hi);
  k_threshold_masklayout<<<b2v_grid(dz * dy, 8, 32), 256, 0, s>>>(img, mask_padded, dz, dy, dx, r.none ? 1 : r.lo,
                                                                  r.none ? 0 : r.hi, preserve_markers, only_dirty);
  int rc;
  if ((rc = b2v_check_launch("k_threshold_masklayout"))) return rc;
  k_set_axial_flags<<<(unsigned)ceil_div64(dz, 256), 256, 0, s>>>(mask_padded, dz, (dy + 1) * (dx + 1));
  return b2v_check_launch("k_set_axial_flags");
}
