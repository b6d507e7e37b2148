// b2v — the bit volume: one bit per voxel of a [rows][dx] volume, packed 32 voxels per uint32 along x.
// A row holds wx = ceil(dx / 32) words; voxel (row, x) is bit x % 32 of word row * wx + x / 32 (row = z * dy + y),
// and the padding bits of a row's last word are 0. The flood fill's passable bits and marching cubes' inside
// bits are both built here, in one HBM-bound pass over the volume (and over `other`, when it is given).
#pragma once
#include <type_traits>

#include "b2v_common.cuh"

namespace {

// lo <= v <= hi and, with OTHER, other[i] != other_fill
template <typename B, bool OTHER>
struct InRange {
  static constexpr bool kOther = OTHER;
  B lo, hi;
  const uint8_t* other;
  uint8_t other_fill;
  __device__ __forceinline__ bool operator()(B v, int64_t i) const {
    return v >= lo && v <= hi && (!OTHER || other[i] != other_fill);
  }
};

// one warp per word, one lane per voxel: any dtype, any alignment, any predicate p(value, index)
template <typename T, typename Pred>
__global__ void __launch_bounds__(256) k_pack_ballot(const T* __restrict__ data, int64_t rows, int64_t dx, Pred p,
                                                     uint32_t* __restrict__ bits, uint32_t* __restrict__ zero) {
  const int lane = threadIdx.x & 31;
  const int64_t wx = (dx + 31) >> 5, nwords = rows * wx;
  for (int64_t wi = gtid() >> 5; wi < nwords; wi += gstride() >> 5) {
    const int64_t row = wi / wx, x = (wi - row * wx) * 32 + lane, i = row * dx + x;
    const uint32_t word = __ballot_sync(0xffffffffu, x < dx && p(data[i], i));
    if (lane == 0) {
      bits[wi] = word;
      if (zero) zero[wi] = 0;
    }
  }
}

// InRange on int16 or uint8 data, lo <= hi inside T's range, dx a multiple of the group and rows 16-byte aligned
// (`other` aligned to its load): each lane packs a group, one 128-bit load of data (8 int16 or 16 uint8 voxels)
// and with OTHER one 64- or 128-bit load of `other`, into as many bits; 4 or 2 lanes make a word, and four groups
// per thread are in flight. LINEAR: dx % 32 == 0, so rows hold no padding groups and group g is part of word
// g / lanes: no 64-bit division per group.
template <typename T, bool OTHER, bool LINEAR>
__global__ void __launch_bounds__(256) k_pack_vec(const T* __restrict__ data, const uint8_t* __restrict__ other,
                                                  uint8_t other_fill, int64_t rows, int64_t dx, int lo, int hi,
                                                  uint32_t* __restrict__ bits, uint32_t* __restrict__ zero) {
  constexpr int G = 16 / sizeof(T);      // voxels per group
  constexpr int LS = G == 8 ? 2 : 1;     // log2 of the lanes per word
  typedef typename std::conditional<G == 8, uint2, uint4>::type OtherVec;
  const int wx = (int)((dx + 31) >> 5);
  const int gx = wx << LS;               // groups per row (padded)
  const int64_t ngroups = rows * gx;
  const int64_t stride = gstride() * 4;
  const int lane = threadIdx.x & 31;
  const uint32_t fill4 = (uint32_t)other_fill * 0x01010101u;
  // int16: the bounds in both halves; uint8: the byte-compare constants of lo and, below 255, of hi + 1
  const uint32_t lo2 = ((uint32_t)lo & 0xffffu) * 0x00010001u, hi2 = ((uint32_t)hi & 0xffffu) * 0x00010001u;
  const uint32_t lo7 = ((uint32_t)lo & 0x7fu) * 0x01010101u, hi7 = ((uint32_t)(hi + 1) & 0x7fu) * 0x01010101u;
  const bool lo_high = lo >= 128, hi_high = hi + 1 >= 128, capped = hi < 255;
  for (int64_t g0 = (int64_t)blockIdx.x * blockDim.x * 4; g0 < ngroups; g0 += stride) {
    uint4 v[4];
    OtherVec o[4];
    int64_t row[4];
    int q[4];
    bool ok[4], in[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t g = g0 + k * blockDim.x + threadIdx.x;
      ok[k] = g < ngroups;
      row[k] = LINEAR || !ok[k] ? 0 : g / gx;
      q[k] = LINEAR || !ok[k] ? 0 : (int)(g - row[k] * gx);
      in[k] = ok[k] && (LINEAR || (int64_t)q[k] * G < dx);   // a padding group packs zero bits
      v[k] = make_uint4(0u, 0u, 0u, 0u);
      o[k] = OtherVec{};
      if (in[k]) {
        const int64_t i = LINEAR ? g * G : row[k] * dx + (int64_t)q[k] * G;
        v[k] = ld_stream((const uint4*)(data + i));
        if (OTHER) o[k] = ld_stream((const OtherVec*)(other + i));
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t b = 0;
      if (in[k]) {
        if constexpr (G == 8) {
          // voxels 0..3 / 4..7 as 0x80-per-byte flags
          uint32_t a = __byte_perm(inrange_flags_s16x2(v[k].x, lo2, hi2), inrange_flags_s16x2(v[k].y, lo2, hi2), 0x7531);
          uint32_t c = __byte_perm(inrange_flags_s16x2(v[k].z, lo2, hi2), inrange_flags_s16x2(v[k].w, lo2, hi2), 0x7531);
          if (OTHER) {
            a &= nonzero_flags_u8x4(o[k].x ^ fill4);
            c &= nonzero_flags_u8x4(o[k].y ^ fill4);
          }
          b = flags_to_nibble(a) | (flags_to_nibble(c) << 4);
        } else {
          const uint32_t d[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
          const uint32_t e[4] = {o[k].x, o[k].y, o[k].z, o[k].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint32_t f = ge_flags_u8x4(d[j], lo7, lo_high);
            if (capped) f &= ~ge_flags_u8x4(d[j], hi7, hi_high);
            if (OTHER) f &= nonzero_flags_u8x4(e[j] ^ fill4);
            b |= flags_to_nibble(f) << (4 * j);
          }
        }
      }
      uint32_t word = b << (G * (lane & ((1 << LS) - 1)));
#pragma unroll
      for (int m = 1; m < (1 << LS); m <<= 1) word |= __shfl_xor_sync(0xffffffffu, word, m);
      if ((lane & ((1 << LS) - 1)) == 0 && ok[k]) {
        const int64_t wi = LINEAR ? (g0 + k * blockDim.x + threadIdx.x) >> LS : row[k] * wx + (q[k] >> LS);
        bits[wi] = word;
        if (zero) zero[wi] = 0;
      }
    }
  }
}

template <typename Pred>
constexpr bool kIntRange = std::is_same<Pred, InRange<int, false>>::value || std::is_same<Pred, InRange<int, true>>::value;

// Packs p over the rows x dx voxels of data into bits, and stores 0 into zero[w] beside every word w when zero is
// given. InRange with int bounds on int16 or uint8 data takes k_pack_vec when dx is a multiple of the group and
// data (and `other`) are aligned to their loads; every other case takes k_pack_ballot.
template <typename T, typename Pred>
int pack_bits(const T* data, int64_t rows, int64_t dx, Pred p, uint32_t* bits, uint32_t* zero, cudaStream_t s) {
  const int64_t nwords = rows * ceil_div64(dx, 32);
  if constexpr (kIntRange<Pred>) {
    static_assert(std::is_same<T, int16_t>::value || std::is_same<T, uint8_t>::value, "int bounds: int16 or uint8 data");
    constexpr int G = 16 / sizeof(T), tmin = sizeof(T) == 2 ? -32768 : 0, tmax = sizeof(T) == 2 ? 32767 : 255;
    if (p.lo < tmin) p.lo = tmin;
    if (p.hi > tmax) p.hi = tmax;
    if (p.lo > p.hi) {   // no voxel can be in range
      B2V_CUDA(cudaMemsetAsync(bits, 0, (size_t)nwords * 4, s));
      if (zero) B2V_CUDA(cudaMemsetAsync(zero, 0, (size_t)nwords * 4, s));
      return B2V_OK;
    }
    if (dx % G == 0 && b2v_aligned16(data) && ((uintptr_t)p.other & (G - 1)) == 0) {
      const int grid = b2v_grid(nwords * (32 / G), 1024, 16);
      if (dx % 32 == 0)
        k_pack_vec<T, Pred::kOther, true><<<grid, 256, 0, s>>>(data, p.other, p.other_fill, rows, dx, p.lo, p.hi, bits,
                                                               zero);
      else
        k_pack_vec<T, Pred::kOther, false><<<grid, 256, 0, s>>>(data, p.other, p.other_fill, rows, dx, p.lo, p.hi,
                                                                bits, zero);
      return b2v_check_launch("k_pack_vec");
    }
  }
  k_pack_ballot<T, Pred><<<b2v_grid(nwords, 8, 16), 256, 0, s>>>(data, rows, dx, p, bits, zero);
  return b2v_check_launch("k_pack_ballot");
}

}  // namespace
