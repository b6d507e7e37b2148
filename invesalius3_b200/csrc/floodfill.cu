// Seeded flood fill / region grow on a bit-packed volume.
// Reference semantics: invesalius_rs/src/floodfill.rs
//   generic_floodfill_threshold          :96-166   (b2v_floodfill_threshold)
//   generic_floodfill_threshold_inplace  :168-237  (b2v_floodfill_threshold_inplace)
//   floodfill_internal                   :5-49     (b2v_floodfill_equal)
//   fill_holes_automatically_internal    :51-94    (b2v_fill_holes)
//
// The reference is a serial stack walk; its RESULT is order independent: the set reachable
// from the valid seeds through "passable" voxels (value in [t0,t1] and out != fill) using
// the structuring-element offsets. We compute that set in three steps:
//   1. build   (HBM-bound, 3 B/voxel): one pass over data (+out) packs `passable` into a
//              bit volume, 32 voxels per word along x (bitpack.cuh). 512^3 voxels -> 16 MiB, i.e. the
//              whole working set of step 2 lives in the H100's 50 MB L2.
//   2. flood   (L2 / shared-memory latency-bound): tiles of the two bit volumes are pulled
//              into shared memory, swept once along x (run fill by the carry trick), y and
//              z, written back; the tiles that can gain from a grown tile are activated for
//              the next round. Rounds ~ geodesic length measured in tiles, not voxels; all
//              rounds run inside one persistent cooperative launch.
//   3. write   (sparse): reached bits are expanded to `fill` stores into out.
#include <cooperative_groups.h>
#include <stdlib.h>
#include <string.h>

#include "b2v_common.cuh"
#include "bitpack.cuh"
#include "peer.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kTileWords = 4096;   // interior words of the largest tile (16 x 16 rows x 16 words = 131 072 voxels)
constexpr int kMaxRounds = 1 << 16;
constexpr int kFloodThreads = 1024;  // one thread per tile word: short dependent chains, 32 warps to overlap them

struct BitVol {
  int64_t dz, dy, dx;
  int wx;              // words per row
  int tz, ty, tw;      // tile dims (rows, rows, words), powers of two
  int ntz, nty, ntw;   // tile grid
  int ltw, lty;        // log2(tw), log2(ty)
  uint32_t m_pw, m_pp; // ceil(2^24 / (tw+2)), ceil(2^24 / ((tw+2)(ty+2))): exact division for i < 2^12
};

int pow2ceil(int64_t v, int cap) {
  int p = 1;
  while (p < v && p < cap) p <<= 1;
  return p;
}

// Tuning knob (results identical either way), read from the environment ONCE per process:
// B2V_FF_GRID=n caps the persistent grid at n blocks.
struct FloodKnobs {
  int grid = 0;
  FloodKnobs() {
    if (const char* e = getenv("B2V_FF_GRID")) { int v = atoi(e); if (v > 0) grid = v; }
  }
};
const FloodKnobs& knobs() {
  static const FloodKnobs k;
  return k;
}

BitVol make_bitvol(int64_t dz, int64_t dy, int64_t dx) {
  BitVol b;
  b.dz = dz; b.dy = dy; b.dx = dx;
  b.wx = (int)ceil_div64(dx, 32);
  // Tile edge (rows): 16 halves the number of rounds of a flood (one tile hop per round)
  // against 8 for about twice the work per visit.
  b.tw = pow2ceil(b.wx, 16);
  b.ty = pow2ceil(dy, 16);
  b.tz = pow2ceil(dz, kTileWords / (b.tw * b.ty));
  // reached + passable tiles with halo must fit the 48 KB of default shared memory
  while (b.tz > 1 && (int64_t)(b.tz + 2) * (b.ty + 2) * (b.tw + 2) * 8 > 48 * 1024) b.tz >>= 1;
  b.ntz = (int)ceil_div64(dz, b.tz);
  b.nty = (int)ceil_div64(dy, b.ty);
  b.ntw = (int)ceil_div64(b.wx, b.tw);
  b.ltw = 0; while ((1 << b.ltw) < b.tw) ++b.ltw;
  b.lty = 0; while ((1 << b.lty) < b.ty) ++b.lty;
  const uint32_t pw = b.tw + 2, pp = (b.tw + 2) * (b.ty + 2);
  b.m_pw = ((1u << 24) + pw - 1) / pw;
  b.m_pp = ((1u << 24) + pp - 1) / pp;
  return b;
}

struct Workspace {
  uint32_t* fg;
  uint32_t* reach;
  uint8_t* active[2];
  int* flags;        // flags[r] != 0  <=>  some tile is active in round r
  int* lists;        // persistent engine: three rotating bitmaps of active tiles [3][ceil(ntiles / 32)]
  int* ctl;          // persistent engine: [3] error, [7] rounds, [16..18] peer exchange (k_ff_persistent)
  int64_t* seeds;    // device copy, 3 per seed
  int64_t bytes;
};

Workspace carve(void* base, const BitVol& b, int64_t nseeds) {
  Workspace w;
  int64_t nwords = b.dz * b.dy * b.wx;
  int64_t ntiles = (int64_t)b.ntz * b.nty * b.ntw;
  auto align = [](int64_t v) { return (v + 255) & ~(int64_t)255; };
  char* p = (char*)base;
  int64_t off = 0;
  w.fg = (uint32_t*)(p + off); off += align(nwords * 4);
  w.reach = (uint32_t*)(p + off); off += align(nwords * 4);
  w.active[0] = (uint8_t*)(p + off); off += align(ntiles);
  w.active[1] = (uint8_t*)(p + off); off += align(ntiles);
  w.flags = (int*)(p + off); off += align((int64_t)(kMaxRounds + 2) * 4);
  w.lists = (int*)(p + off); off += align(3 * ((ntiles + 31) / 32) * 4);
  w.ctl = (int*)(p + off); off += 256;
  w.seeds = (int64_t*)(p + off); off += align((nseeds > 0 ? nseeds : 1) * 24);
  w.bytes = off;
  return w;
}

// ---- passable predicates ----------------------------------------------------------
template <typename T> struct Thr { typedef int type; };
template <> struct Thr<double> { typedef double type; };

enum { MODE_THRESHOLD = 0, MODE_INPLACE = 1, MODE_EQUAL = 2 };

// MODE_THRESHOLD: t0 <= data <= t1 && out != fill          (floodfill.rs:154-157)
// MODE_INPLACE  : t0 <= data <= t1 && data != fill         (floodfill.rs:225-228)
// MODE_EQUAL    : data == t0       && out != fill          (floodfill.rs:25)
// The first and the last are InRange (bitpack.cuh) with `out` as its other stream; the in-place test is this one.
template <typename B>
struct InRangeNotFill {
  B lo, hi, fill;
  __device__ __forceinline__ bool operator()(B v, int64_t) const { return v >= lo && v <= hi && v != fill; }
};

// seeds: (x, y, z) triples, already bounds-checked on the host. A valid seed is reached
// and passable even if out already holds `fill` there (floodfill.rs:121-127); force=1
// marks the seed unconditionally (floodfill.rs:21).
template <typename T>
__global__ void k_ff_seeds(const T* __restrict__ data, BitVol b, const int64_t* __restrict__ seeds, int64_t nseeds,
                           typename Thr<T>::type t0, typename Thr<T>::type t1, int force, uint32_t* fg,
                           uint32_t* reach, uint8_t* active, int* flags) {
  typedef typename Thr<T>::type TT;
  int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseeds) return;
  int64_t x = seeds[3 * s], y = seeds[3 * s + 1], z = seeds[3 * s + 2];
  TT v = (TT)data[(z * b.dy + y) * b.dx + x];
  if (!force && !(v >= t0 && v <= t1)) return;
  int64_t wi = (z * b.dy + y) * b.wx + (x >> 5);
  uint32_t bit = 1u << (x & 31);
  atomicOr(&fg[wi], bit);
  atomicOr(&reach[wi], bit);
  int tile = ((int)(z / b.tz) * b.nty + (int)(y / b.ty)) * b.ntw + (int)((x >> 5) / b.tw);
  active[tile] = 1;
  flags[0] = 1;
}

// ---- the flood round ------------------------------------------------------------------
// run fill: every run of ones in `m` that contains a bit of `s` (s subset of m) is filled.
__device__ __forceinline__ uint32_t run_fill(uint32_t s, uint32_t m) {
  uint32_t up = (((m + s) ^ m) & m) | s;
  uint32_t rm = __brev(m), rs = __brev(s);
  uint32_t dn = __brev(((rm + rs) ^ rm) & rm);
  return up | dn;
}

// sb: 27 structuring-element bits, index (oz+1)*9 + (oy+1)*3 + (ox+1); the flood moves
// from p to p + (oz, oy, ox).
// One tile of the bit volume relaxed to local convergence in shared memory; grown words are
// written back. Returns (uniformly over the block) the 27-bit mask of neighbour tiles that
// can gain reached bits from this tile (bit (oz+1)*9 + (oy+1)*3 + (ow+1)).
// Axis sweep of one column of words: v[k] = (v[k] | v[k-1]) & f[k] along +axis (and the
// mirror image along -axis), rows held in registers eight at a time; the ends are fed by
// the read-only halo words. Returns whether anything changed.
__device__ __forceinline__ int sweep_column(uint32_t* sR, const uint32_t* sF, int base, int stride, int n, bool fwd,
                                            bool bwd) {
  int changed = 0;
  if (fwd) {
    uint32_t prev = sR[base];
    for (int c0 = 0; c0 < n; c0 += 8) {
      uint32_t r[8], f[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        r[k] = c0 + k < n ? sR[base + (c0 + k + 1) * stride] : 0u;
        f[k] = c0 + k < n ? sF[base + (c0 + k + 1) * stride] : 0u;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        uint32_t v = (r[k] | prev) & f[k];
        if (c0 + k < n) {
          if (v != r[k]) { sR[base + (c0 + k + 1) * stride] = v; changed = 1; }
          prev = v;
        }
      }
    }
  }
  if (bwd) {
    uint32_t prev = sR[base + (n + 1) * stride];
    for (int c1 = n; c1 > 0; c1 -= 8) {
      uint32_t r[8], f[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        r[k] = c1 - 1 - k >= 0 ? sR[base + (c1 - k) * stride] : 0u;
        f[k] = c1 - 1 - k >= 0 ? sF[base + (c1 - k) * stride] : 0u;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        uint32_t v = (r[k] | prev) & f[k];
        if (c1 - 1 - k >= 0) {
          if (v != r[k]) { sR[base + (c1 - k) * stride] = v; changed = 1; }
          prev = v;
        }
      }
    }
  }
  return changed;
}

// SBC != 0 fixes the structuring element at compile time (6-, 18-, 26-connectivity): the
// stencil loops lose their dead rows and, for axis-only elements, the generic hop vanishes
// (the three sweeps already cover every offset).
constexpr uint32_t kSB26 = 0x7ffffffu & ~(1u << 13);
constexpr uint32_t kSB18 = kSB26 & ~((1u << 0) | (1u << 2) | (1u << 6) | (1u << 8) | (1u << 18) | (1u << 20) |
                                     (1u << 24) | (1u << 26));

// ---- 6-connected, canonical tiles (2^LZ x 2^LY rows x 16 words) ------------------------------
// The common case (InVesalius floods with the 6-neighbourhood) with every index a
// compile-time constant: K = tile words / 1024 words per thread for the loads, the write-back
// and the change detection; the three axis sweeps as register chains.

// One row of 16 words swept along x by one thread: the run fill of a word (carry trick of
// run_fill) plus the carry into the next word, towards higher x and then towards lower x.
// The filled words of the first pass seed the second, so every run that holds a reached bit
// ends up full across word boundaries. first = the row's word 0 in the haloed tile.
__device__ __forceinline__ void sweep_row_x(uint32_t* sR, const uint32_t* sF, int first) {
  uint32_t m[16], v[16];
#pragma unroll
  for (int w = 0; w < 16; ++w) { m[w] = sF[first + w]; v[w] = sR[first + w]; }
  uint32_t cin = sR[first - 1] >> 31;           // last bit of the word before the row (halo)
#pragma unroll
  for (int w = 0; w < 16; ++w) {
    const uint32_t sd = v[w] | (cin & m[w]);
    v[w] = (((m[w] + sd) ^ m[w]) & m[w]) | sd;
    cin = v[w] >> 31;
  }
  cin = sR[first + 16] & 1u;                    // first bit of the word after the row (halo)
#pragma unroll
  for (int w = 15; w >= 0; --w) {
    const uint32_t sd = v[w] | ((cin << 31) & m[w]);
    const uint32_t rm = __brev(m[w]), rs = __brev(sd);
    v[w] = __brev(((rm + rs) ^ rm) & rm) | sd;
    cin = v[w] & 1u;
  }
#pragma unroll
  for (int w = 0; w < 16; ++w) sR[first + w] = v[w];
}

// One column of N words swept along y or z by one thread: v[j] |= v[j-1] & m[j] down the
// column, then the mirror image up; the ends are fed by the read-only halo words.
// halo0 = the halo word before the column, stride = distance between column neighbours.
template <int N>
__device__ __forceinline__ void sweep_col(uint32_t* sR, const uint32_t* sF, int halo0, int stride) {
  uint32_t m[N], v[N];
#pragma unroll
  for (int j = 0; j < N; ++j) { m[j] = sF[halo0 + (j + 1) * stride]; v[j] = sR[halo0 + (j + 1) * stride]; }
  uint32_t prev = sR[halo0];
#pragma unroll
  for (int j = 0; j < N; ++j) { v[j] |= prev & m[j]; prev = v[j]; }
  prev = sR[halo0 + (N + 1) * stride];
#pragma unroll
  for (int j = N - 1; j >= 0; --j) { v[j] |= prev & m[j]; prev = v[j]; }
#pragma unroll
  for (int j = 0; j < N; ++j) sR[halo0 + (j + 1) * stride] = v[j];
}

template <int LZ, int LY>
__device__ __forceinline__ int ff_process_tile_sb6(const uint32_t* __restrict__ fg, uint32_t* reach, const BitVol& b,
                                                   int tile, uint32_t* sR, int* s_faces) {
  constexpr int TZ = 1 << LZ, TY = 1 << LY, PW = 18, PY = TY + 2, NH = (TZ + 2) * PY * PW;
  constexpr int K = TZ * TY * 16 / kFloodThreads;          // words per thread
  constexpr int NL = (NH + kFloodThreads - 1) / kFloodThreads;
  const int tid = threadIdx.x;
  const int twi = tile % b.ntw, tyi = (tile / b.ntw) % b.nty, tzi = tile / (b.ntw * b.nty);
  // 32-bit indices: the word count of a bit volume is below 2^31 (checked on entry)
  const int z0 = tzi * TZ, y0 = tyi * TY, w0 = twi * 16;
  const int dz = (int)b.dz, dy = (int)b.dy;
  uint32_t* sF = sR + NH;
  if (tid == 0) *s_faces = 0;
  {
    uint32_t v[NL], f[NL];
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      const int i = tid + k * kFloodThreads;
      v[k] = 0; f[k] = 0;
      if (i < NH) {
        const int hz = i / (PW * PY), rem = i - hz * (PW * PY), hy = rem / PW, hw = rem - hy * PW;
        const int z = z0 + hz - 1, y = y0 + hy - 1, w = w0 + hw - 1;
        if ((unsigned)z < (unsigned)dz && (unsigned)y < (unsigned)dy && (unsigned)w < (unsigned)b.wx) {
          const int gi = (z * dy + y) * b.wx + w;
          v[k] = __ldcg(&reach[gi]);
          f[k] = __ldg(&fg[gi]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      const int i = tid + k * kFloodThreads;
      if (i < NH) { sR[i] = v[k]; sF[i] = f[k]; }
    }
  }
  __syncthreads();
  // owner role: word i = tid + k * 1024 -> (iz, iy, iw), iw fastest (a 16-lane group = a row)
  uint32_t f[K], r0[K], r[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int i = tid + k * kFloodThreads;
    const int h = (((i >> (4 + LY)) + 1) * PY + (((i >> 4) & (TY - 1)) + 1)) * PW + (i & 15) + 1;
    f[k] = sF[h];
    r0[k] = r[k] = sR[h];
  }
  const int iw = tid & 15;
  // Each sweep is a serial chain in the registers of ONE thread per row / column (a few
  // hundred threads busy, a few hundred cycles): far fewer instructions than a
  // word-per-thread scan, and the block is latency-bound here, not width-bound.
  if (tid < TZ * TY)        // x: row (z = tid >> LY, y = tid & (TY-1))
    sweep_row_x(sR, sF, (((tid >> LY) + 1) * PY + ((tid & (TY - 1)) + 1)) * PW + 1);
  __syncthreads();
  if (tid < TZ * 16)        // y: column (z = tid >> 4, w = tid & 15), halo row y = -1 first
    sweep_col<TY>(sR, sF, ((tid >> 4) + 1) * PY * PW + (tid & 15) + 1, PW);
  __syncthreads();
  if (tid < TY * 16)        // z: column (y = tid >> 4, w = tid & 15), halo plane z = -1 first
    sweep_col<TZ>(sR, sF, ((tid >> 4) + 1) * PW + (tid & 15) + 1, PY * PW);
  __syncthreads();
  int moved = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int i = tid + k * kFloodThreads;
    const int h = (((i >> (4 + LY)) + 1) * PY + (((i >> 4) & (TY - 1)) + 1)) * PW + iw + 1;
    const uint32_t v = sR[h];
    moved |= v != r[k];
    r[k] = v;
  }
  // one sweep set per visit: a tile that changed may not be settled yet and re-queues itself
  const bool unfinished = __syncthreads_or(moved) != 0;
  int grew = 0;
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (r[k] != r0[k]) {   // r != 0 only inside the volume: out-of-volume words have no passable bit
      const int i = tid + k * kFloodThreads;
      __stcg(&reach[((z0 + (i >> (4 + LY))) * dy + (y0 + ((i >> 4) & (TY - 1)))) * b.wx + (w0 + iw)], r[k]);
      grew = 1;
    }
  grew = __syncthreads_or(grew);
  // which of the six face neighbours can gain a bit from this tile's interior? One face word
  // per thread: passable-but-unreached bits of the halo word against the reached bits of the
  // interior word next to it (same bit across y / z, the adjacent bit across a word boundary).
  // Every face is a multiple of 32 words, so a warp votes for one face.
  constexpr int NYF = TZ * 16, NZF = TY * 16, NXF = TZ * TY, TOT = 2 * (NYF + NZF + NXF);
  for (int t = tid; t < TOT; t += kFloodThreads) {
    bool gain;
    int bit;
    if (t < 2 * NYF) {
      const int hi = t >= NYF, u = t - hi * NYF, a = u >> 4, bw = u & 15;
      const int h = ((a + 1) * PY + (hi ? TY + 1 : 0)) * PW + bw + 1, src = hi ? h - PW : h + PW;
      bit = hi ? 16 : 10;
      gain = (sF[h] & ~sR[h] & sR[src]) != 0;
    } else if (t < 2 * NYF + 2 * NZF) {
      const int u0 = t - 2 * NYF, hi = u0 >= NZF, u = u0 - hi * NZF, a = u >> 4, bw = u & 15;
      const int h = ((hi ? TZ + 1 : 0) * PY + a + 1) * PW + bw + 1, src = hi ? h - PY * PW : h + PY * PW;
      bit = hi ? 22 : 4;
      gain = (sF[h] & ~sR[h] & sR[src]) != 0;
    } else {
      const int u0 = t - 2 * NYF - 2 * NZF, hi = u0 >= NXF, u = u0 - hi * NXF;
      const int row = (((u >> LY) + 1) * PY + ((u & (TY - 1)) + 1)) * PW;
      bit = hi ? 14 : 12;
      gain = hi ? ((sF[row + 17] & ~sR[row + 17]) & (sR[row + 16] >> 31) & 1u) != 0
                : (((sF[row] & ~sR[row]) >> 31) & sR[row + 1] & 1u) != 0;
    }
    if (__any_sync(0xffffffffu, gain) && (tid & 31) == 0) atomicOr(s_faces, 1 << bit);
  }
  if (unfinished && tid == 0) atomicOr(s_faces, 1 << 13);   // (0,0,0): re-queue this tile itself
  __syncthreads();
  return *s_faces;
}

template <uint32_t SBC>
__device__ __forceinline__ int ff_process_tile(const uint32_t* __restrict__ fg, uint32_t* reach, const BitVol& b,
                                               uint32_t sb_rt, int tile, uint32_t* sR, int* s_faces) {
  if constexpr (SBC == kSB6) {
    if (b.tw == 16 && b.ty == 16 && b.tz == 16) return ff_process_tile_sb6<4, 4>(fg, reach, b, tile, sR, s_faces);
  }
  const uint32_t sb = SBC ? SBC : sb_rt;
  // the x sweep needs both x offsets; a one-sided x offset is left to the generic hop
  const bool axis_only = (sb & ~kSB6) == 0 && (((sb >> 12) & 1u) == ((sb >> 14) & 1u));
  const int tid = threadIdx.x;
  const int tw = b.tw, ty = b.ty, tz = b.tz;
  const int pw = tw + 2, py = ty + 2;
  const int twi = tile % b.ntw, tyi = (tile / b.ntw) % b.nty, tzi = tile / (b.ntw * b.nty);
  const int64_t z0 = (int64_t)tzi * tz, y0 = (int64_t)tyi * ty;
  const int w0 = twi * tw;
  if (tid == 0) *s_faces = 0;
  // halo load (zero outside the volume); the passable bits ride along (halo words are
  // never written)
  const int nh = (tz + 2) * py * pw;
  uint32_t* sF = sR + nh;
  // all loads of a batch are issued before the first shared store: the L2 round trips of a
  // thread overlap
  for (int i0 = 0; i0 < nh; i0 += 4 * kFloodThreads) {
    uint32_t v[4], f[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = i0 + k * kFloodThreads + tid;
      v[k] = 0; f[k] = 0;
      if (i < nh) {
        const int hz = (int)(((unsigned long long)i * b.m_pp) >> 24);
        const int rem = i - hz * (pw * py);
        const int hy = (int)(((unsigned long long)rem * b.m_pw) >> 24);
        const int hw = rem - hy * pw;
        const int64_t z = z0 + hz - 1, y = y0 + hy - 1;
        const int w = w0 + hw - 1;
        if (z >= 0 && z < b.dz && y >= 0 && y < b.dy && w >= 0 && w < b.wx) {
          const int64_t gi = (z * b.dy + y) * b.wx + w;
          v[k] = __ldcg(&reach[gi]);
          f[k] = __ldg(&fg[gi]);   // halo words included: they decide which neighbour tiles can gain
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = i0 + k * kFloodThreads + tid;
      if (i < nh) { sR[i] = v[k]; sF[i] = f[k]; }
    }
  }
  // owned words: fg and the initial reach value stay in registers
  constexpr int kOwn = kTileWords / kFloodThreads;
  uint32_t fgr[kOwn], r0[kOwn];
  int hidx[kOwn];
  const int nint = tz * ty * tw;
#pragma unroll
  for (int k = 0; k < kOwn; ++k) {
    int i = tid + k * kFloodThreads;
    fgr[k] = 0; r0[k] = 0; hidx[k] = -1;
    if (i < nint) {
      int iw = i & (tw - 1), iy = (i >> b.ltw) & (ty - 1), iz = i >> (b.ltw + b.lty);
      int64_t z = z0 + iz, y = y0 + iy;
      int w = w0 + iw;
      if (z < b.dz && y < b.dy && w < b.wx) {
        hidx[k] = ((iz + 1) * py + (iy + 1)) * pw + (iw + 1);
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kOwn; ++k)
    if (hidx[k] >= 0) {
      r0[k] = sR[hidx[k]];
      fgr[k] = sF[hidx[k]];
    }

  const bool xfill = ((sb >> 12) & 1u) && ((sb >> 14) & 1u);  // (0,0,-1) and (0,0,+1)
  // axis-aligned offsets present in the structuring element (flood moves p -> p + off)
  const bool yfwd = (sb >> 16) & 1u, ybwd = (sb >> 10) & 1u;   // (0,+1,0), (0,-1,0)
  const bool zfwd = (sb >> 22) & 1u, zbwd = (sb >> 4) & 1u;    // (+1,0,0), (-1,0,0)
  int changed = 0;
  // ---- directional sweeps: each carries reached bits across the whole tile along one
  // axis in O(1) dependent steps (a Jacobi step moves them by one row / one word only)
  if (xfill) {
    // Along x a row is a chain of words. Per word: fill the runs that already hold a
    // reached bit; g = "the fill reaches the word's last bit" (carry generate), p = "the
    // word is all passable" (carry propagate). The carries into every word of the row
    // are then one integer addition (carry-lookahead): (a + b + c0) ^ a ^ b with
    // a = g | p, b = g. Same towards lower x on the bit-reversed masks.
    const int lane = tid & 31;
    const int grp = lane >> b.ltw;                   // tw is a power of two <= 16
    const uint32_t gmask = (tw == 32) ? 0xffffffffu : ((1u << tw) - 1u);
    for (int i0 = 0; i0 < nint || i0 == 0; i0 += kFloodThreads) {
      const int i = i0 + tid;
      const bool live = i < nint;
      const int row = live ? i >> b.ltw : 0, w = live ? i & (tw - 1) : 0;
      const int base = (((row >> b.lty) + 1) * py + ((row & (ty - 1)) + 1)) * pw + 1;
      uint32_t f = 0, cur = 0, filled = 0;
      if (live) {
        f = sF[base + w];
        cur = sR[base + w];
        filled = (f && cur) ? run_fill(cur & f, f) : 0u;
      }
      const bool pfull = live && f == 0xffffffffu;
      const uint32_t gu = (__ballot_sync(0xffffffffu, filled >> 31) >> (grp * tw)) & gmask;
      const uint32_t gd = (__ballot_sync(0xffffffffu, filled & 1u) >> (grp * tw)) & gmask;
      const uint32_t pm = (__ballot_sync(0xffffffffu, pfull) >> (grp * tw)) & gmask;
      if (live) {
        // up: carry into word k = bit k of the carry vector; the left halo word feeds bit 0
        const uint32_t c0 = sR[base - 1] >> 31;
        const uint32_t au = gu | pm, bu = gu;
        const uint32_t cu = ((au + bu + c0) ^ au ^ bu);
        // down: reverse the word order so that the same adder runs towards lower x
        const uint32_t gdr = __brev(gd) >> (32 - tw), pmr = __brev(pm) >> (32 - tw);
        const uint32_t c1 = sR[base + tw] & 1u;
        const uint32_t ad = gdr | pmr, bd = gdr;
        const uint32_t cd = ((ad + bd + c1) ^ ad ^ bd);
        const uint32_t cin_lo = (cu >> w) & 1u;                 // enters at bit 0
        const uint32_t cin_hi = (cd >> (tw - 1 - w)) & 1u;      // enters at bit 31
        const uint32_t seed = (cur | cin_lo | (cin_hi << 31)) & f;
        const uint32_t v = seed ? run_fill(seed, f) : 0u;
        if (v != cur) { sR[base + w] = v; changed = 1; }
      }
    }
    __syncthreads();
  }
  if (yfwd || ybwd) {
    // one thread per (z, word) column
    for (int c = tid; c < tz * tw; c += kFloodThreads) {
      const int base = (((c >> b.ltw) + 1) * py) * pw + ((c & (tw - 1)) + 1);  // halo row hy = 0
      changed |= sweep_column(sR, sF, base, pw, ty, yfwd, ybwd);
    }
    __syncthreads();
  }
  if (zfwd || zbwd) {
    // one thread per (y, word) column
    for (int c = tid; c < ty * tw; c += kFloodThreads) {
      const int base = ((c >> b.ltw) + 1) * pw + ((c & (tw - 1)) + 1);         // halo plane hz = 0
      changed |= sweep_column(sR, sF, base, py * pw, tz, zfwd, zbwd);
    }
    __syncthreads();
  }
  // ---- generic step: every offset of the structuring element, one hop
  if (!axis_only)
#pragma unroll
  for (int k = 0; k < kOwn; ++k) {
    if (hidx[k] < 0 || fgr[k] == 0) continue;
    uint32_t cur = sR[hidx[k]];
    if (cur == fgr[k]) continue;  // saturated
    uint32_t acc = cur;
#pragma unroll
    for (int oz = -1; oz <= 1; ++oz) {
#pragma unroll
      for (int oy = -1; oy <= 1; ++oy) {
        uint32_t xm = (sb >> ((oz + 1) * 9 + (oy + 1) * 3)) & 7u;
        if (xm == 0) continue;
        int src = hidx[k] - (oz * py + oy) * pw;  // row (z - oz, y - oy)
        uint32_t c = sR[src];
        if (xm & 2u) acc |= c;
        if (xm & 4u) acc |= (c << 1) | (sR[src - 1] >> 31);  // ox = +1
        if (xm & 1u) acc |= (c >> 1) | (sR[src + 1] << 31);  // ox = -1
      }
    }
    acc &= fgr[k];
    if (xfill && acc) acc = run_fill(acc, fgr[k]);
    if (acc != cur) {
      sR[hidx[k]] = acc;
      changed = 1;
    }
  }
  // one sweep set per visit: a tile that changed may not be settled yet and re-queues itself
  const bool unfinished = __syncthreads_or(changed) != 0;

  // write back what grew
  int grew = 0;
#pragma unroll
  for (int k = 0; k < kOwn; ++k) {
    if (hidx[k] < 0) continue;
    uint32_t v = sR[hidx[k]];
    if (v != r0[k]) {
      int i = tid + k * kFloodThreads;
      int iw = i & (tw - 1), iy = (i >> b.ltw) & (ty - 1), iz = i >> (b.ltw + b.lty);
      int64_t z = z0 + iz, y = y0 + iy;
      __stcg(&reach[(z * b.dy + y) * b.wx + (w0 + iw)], v);
      grew = 1;
    }
  }
  // Which neighbour tiles would gain a bit from this tile's state? For every halo word with
  // passable-but-unreached bits, apply one hop of the structuring element from the tile
  // box; a non-empty gain marks the tile that owns the word (bit (oz+1)*9+(oy+1)*3+(ow+1)).
  int nbmask = 0;
  // (checked even without growth: a lone seed on a tile face must still wake its neighbour)
  grew = __syncthreads_or(grew);
  {
    const int hzmax = tz + 1, hymax = ty + 1, hwmax = tw + 1;
    for (int i = tid; i < nh; i += kFloodThreads) {
      const int hz = (int)(((unsigned long long)i * b.m_pp) >> 24);
      const int rem = i - hz * (pw * py);
      const int hy = (int)(((unsigned long long)rem * b.m_pw) >> 24);
      const int hw = rem - hy * pw;
      const int tz_o = hz == 0 ? -1 : (hz == hzmax ? 1 : 0);
      const int ty_o = hy == 0 ? -1 : (hy == hymax ? 1 : 0);
      const int tw_o = hw == 0 ? -1 : (hw == hwmax ? 1 : 0);
      if (tz_o == 0 && ty_o == 0 && tw_o == 0) continue;  // interior
      const uint32_t want = sF[i] & ~sR[i];
      if (want == 0) continue;
      uint32_t acc = 0;
#pragma unroll
      for (int oz = -1; oz <= 1; ++oz) {
#pragma unroll
        for (int oy = -1; oy <= 1; ++oy) {
          uint32_t xm = (sb >> ((oz + 1) * 9 + (oy + 1) * 3)) & 7u;
          if (xm == 0) continue;
          const int sz = hz - oz, sy = hy - oy;  // source row (z - oz, y - oy)
          if (sz < 0 || sz > hzmax || sy < 0 || sy > hymax) continue;
          const int src = (sz * py + sy) * pw + hw;
          const uint32_t c = sR[src];
          if (xm & 2u) acc |= c;
          if (xm & 4u) acc |= (c << 1) | (hw > 0 ? (sR[src - 1] >> 31) : 0u);
          if (xm & 1u) acc |= (c >> 1) | (hw < hwmax ? (sR[src + 1] << 31) : 0u);
        }
      }
      if (acc & want) nbmask |= 1 << ((tz_o + 1) * 9 + (ty_o + 1) * 3 + (tw_o + 1));
    }
  }
  if (unfinished && tid == 0) nbmask |= 1 << 13;   // (0,0,0): re-queue this tile itself
  if (nbmask) atomicOr(s_faces, nbmask);
  __syncthreads();
  return *s_faces;
}

template <uint32_t SBC>
__global__ void __launch_bounds__(kFloodThreads)
    k_ff_round(const uint32_t* __restrict__ fg, uint32_t* reach, BitVol b, uint32_t sb, uint8_t* active_cur,
               uint8_t* active_next, int* flags, int round) {
  if (flags[round] == 0) return;
  const int tile = blockIdx.x;
  // consistent decision for the whole block before thread 0 clears the entry
  if (!__syncthreads_or(active_cur[tile] != 0)) return;
  extern __shared__ uint32_t sR[];  // [(tz+2)][(ty+2)][(tw+2)] reached + same for passable
  __shared__ int s_faces;
  const int tid = threadIdx.x;
  if (tid == 0) active_cur[tile] = 0;  // this buffer becomes `next` of the following round
  const int twi = tile % b.ntw, tyi = (tile / b.ntw) % b.nty, tzi = tile / (b.ntw * b.nty);
  const int nbmask = ff_process_tile<SBC>(fg, reach, b, sb, tile, sR, &s_faces);
  if (nbmask == 0) return;
  __threadfence();
  // activate the neighbour tiles that can gain from this one
  if (tid < 27 && ((nbmask >> tid) & 1)) {
    int oz = tid / 9 - 1, oy = (tid / 3) % 3 - 1, ow = tid % 3 - 1;
    int nz = tzi + oz, ny = tyi + oy, nw = twi + ow;
    if (nz >= 0 && nz < b.ntz && ny >= 0 && ny < b.nty && nw >= 0 && nw < b.ntw) {
      active_next[(nz * b.nty + ny) * b.ntw + nw] = 1;
      flags[round + 1] = 1;
    }
  }
}

// ---- persistent variant: all rounds in ONE cooperative launch ------------------------------
// The host-driven rounds above pay for a launch of every tile's block per round although a
// few dozen tiles are active. Here the active tiles of a round are a bitmap (one bit per
// tile); a persistent grid reads it after the grid-wide barrier, every block ranks the set
// bits with a block scan and takes the tiles whose rank is congruent to its index, and a
// tile that can gain is posted to the next round's bitmap with one fire-and-forget atomic OR
// (no list slot to reserve, no duplicate to filter: the per-round critical path is one
// bitmap read, one tile visit and the barrier). Three bitmaps rotate so that the one being
// posted to was cleared a full round earlier.
constexpr int kMaxMine = 256;    // tiles one block may own in a round (host falls back to launches beyond)

__global__ void k_ff_lists_init(const uint8_t* __restrict__ active, uint8_t* active_clr, int ntiles, uint32_t* bm,
                                int nbw) {
  for (int wi = threadIdx.x; wi < nbw; wi += blockDim.x) {
    uint32_t w = 0;
    for (int j = 0; j < 32; ++j) {
      const int t = wi * 32 + j;
      if (t < ntiles && active[t]) { w |= 1u << j; active_clr[t] = 0; }
    }
    bm[wi] = w;
    bm[nbw + wi] = 0;
    bm[2 * nbw + wi] = 0;
  }
}

// Rank the set bits of the bitmap; the tiles of rank bid, bid + nblocks, ... go to mine[].
// Returns the number of set bits (uniform over the block).
__device__ __forceinline__ int ff_select_tiles(const uint32_t* bm, int nbw, int bid, int nblocks, int* mine,
                                               int* s_wsum) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (nbw <= 32) {   // up to 1024 tiles: one warp ranks the whole bitmap, one block barrier
    if (warp == 0) {
      const uint32_t w = lane < nbw ? __ldcg(&bm[lane]) : 0u;
      const int c = __popc(w);
      int incl = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += v;
      }
      const int rank = incl - c;
      if (c) {
        int slot = rank > bid ? (rank - bid + nblocks - 1) / nblocks : 0;
        for (int q = bid + slot * nblocks; q < rank + c; q += nblocks, ++slot)
          if (slot < kMaxMine) mine[slot] = lane * 32 + (int)__fns(w, 0, q - rank + 1);
      }
      if (lane == 31) s_wsum[0] = incl;
    }
    __syncthreads();
    return s_wsum[0];
  }
  int base = 0;
  for (int i0 = 0; i0 < nbw; i0 += kFloodThreads) {
    const int i = i0 + tid;
    uint32_t w = i < nbw ? __ldcg(&bm[i]) : 0u;
    const int c = __popc(w);
    int incl = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += v;
    }
    if (lane == 31) s_wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int ws = s_wsum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, ws, d);
        if (lane >= d) ws += v;
      }
      s_wsum[lane] = ws;   // inclusive over warps
    }
    __syncthreads();
    int rank = base + (warp ? s_wsum[warp - 1] : 0) + incl - c;
    const int total = s_wsum[31];
    // ranks [rank, rank + c) sit in this word: those of the form bid + slot * nblocks are mine
    if (c) {
      int slot = rank > bid ? (rank - bid + nblocks - 1) / nblocks : 0;
      for (int q = bid + slot * nblocks; q < rank + c; q += nblocks, ++slot)
        if (slot < kMaxMine) mine[slot] = i * 32 + (int)__fns(w, 0, q - rank + 1);
    }
    base += total;
    __syncthreads();   // s_wsum is reused by the next chunk
  }
  return base;
}

// CANON = 4: 6-connected flood on the canonical 16 x 16 rows x 16 words tile only
// (ff_process_tile_sb6, no generic path); 0 = any tile, any element.
// (Two co-resident blocks per SM at 32 registers were measured slower: the barrier doubles
// and the visits of the two blocks contend.)
// PEER: the slab is one Z shard of a larger volume (extended by one halo plane per inner side).
// After local convergence the shard pushes the reached bits of the two planes around each inner
// boundary into its neighbours' mailboxes over NVLink, merges what the neighbours pushed, and all
// ranks agree (flag words written into every mailbox) whether anyone gained a bit; if so the
// rounds resume. The whole sharded flood is this ONE launch per GPU: no host round trip, no
// NCCL call. ctl[3] error (1 round cap, 2 peer timeout), ctl[7] rounds, ctl[18] exchanges.
template <uint32_t SBC, int CANON, bool PEER>
__global__ void __launch_bounds__(kFloodThreads)
    k_ff_persistent(const uint32_t* __restrict__ fg, uint32_t* reach, BitVol b, uint32_t sb, uint32_t* bm, int nbw,
                    int* ctl, int max_rounds, PeerSet ps) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ uint32_t sR[];
  __shared__ int s_faces;
  __shared__ int s_wsum[32];
  __shared__ int s_mine[kMaxMine];
  const int tid = threadIdx.x;
  int r = 0, outer = 0;
  for (;;) {
  for (;; ++r) {
    const int cur = r % 3, nxt = (r + 1) % 3, old = (r + 2) % 3;
    const int n = ff_select_tiles(bm + (size_t)cur * nbw, nbw, blockIdx.x, gridDim.x, s_mine, s_wsum);
    if (n == 0) break;
    if (r >= max_rounds) { if (blockIdx.x == 0 && tid == 0) ctl[3] = 1; break; }
    // `old` was read by everyone before the last barrier and is posted to from the next round on
    for (int i = blockIdx.x * kFloodThreads + tid; i < nbw; i += gridDim.x * kFloodThreads) bm[(size_t)old * nbw + i] = 0;
    int nmine = n > (int)blockIdx.x ? (n - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    int keep = -1;
    if (nmine == 2) {
      // a few tiles more than blocks: pass them on to the next round instead of making every
      // block wait for a second visit (always the cheaper of the two while n <= 2 x blocks)
      // (alternating which of the two waits, so that no tile waits twice in a row)
      const int t = s_mine[(r & 1) ? 0 : 1];
      keep = s_mine[(r & 1) ? 1 : 0];
      if (tid == 0) atomicOr(&bm[(size_t)nxt * nbw + (t >> 5)], 1u << (t & 31));
      nmine = 1;
    }
    for (int k = 0; k < nmine; ++k) {
      const int tile = keep >= 0 ? keep : s_mine[k];
      int nbmask;
      if constexpr (CANON != 0) nbmask = ff_process_tile_sb6<CANON, CANON>(fg, reach, b, tile, sR, &s_faces);
      else nbmask = ff_process_tile<SBC>(fg, reach, b, sb, tile, sR, &s_faces);
      if (tid < 27 && ((nbmask >> tid) & 1)) {
        const int twi = tile % b.ntw, tyi = (tile / b.ntw) % b.nty, tzi = tile / (b.ntw * b.nty);
        int oz = tid / 9 - 1, oy = (tid / 3) % 3 - 1, ow = tid % 3 - 1;
        int nz = tzi + oz, ny = tyi + oy, nw = twi + ow;
        if (nz >= 0 && nz < b.ntz && ny >= 0 && ny < b.nty && nw >= 0 && nw < b.ntw) {
          const int nb = (nz * b.nty + ny) * b.ntw + nw;
          atomicOr(&bm[(size_t)nxt * nbw + (nb >> 5)], 1u << (nb & 31));
        }
      }
      __syncthreads();   // s_faces / shared tile are reused by the next tile of this block
    }
    grid.sync();   // orders every thread's writes (reach words, next bitmap) before the next round's reads
  }
  if constexpr (!PEER) {
    break;
  } else {
    // ---- exchange with the neighbour shards (every rank takes part in every exchange, in lockstep)
    const uint32_t ep = ps.epoch + (uint32_t)outer;
    const int par = (int)(ep & 1u);
    const bool has_lo = ps.rank > 0, has_hi = ps.rank + 1 < ps.world;
    const int pw = (int)b.dy * b.wx;                    // words per plane (checked on the host: fits the mailbox)
    const int gt = blockIdx.x * kFloodThreads + tid, gs = gridDim.x * kFloodThreads;
    // 1. push [halo, first own] down and [last own, halo] up
    if (has_lo) {
      uint32_t* dst = ps.of(ps.rank - 1).ff_from_hi();
      for (int i = gt; i < 2 * pw; i += gs) dst[i] = __ldcg(reach + i);
    }
    if (has_hi) {
      uint32_t* dst = ps.of(ps.rank + 1).ff_from_lo();
      const uint32_t* src = reach + (size_t)(b.dz - 2) * pw;
      for (int i = gt; i < 2 * pw; i += gs) dst[i] = __ldcg(src + i);
    }
    __threadfence_system();
    grid.sync();
    if (blockIdx.x == 0 && tid == 0) {
      if (has_lo) st_release_sys(ps.of(ps.rank - 1).sig(PB_SIG_FF_FROM_HI), ep);
      if (has_hi) st_release_sys(ps.of(ps.rank + 1).sig(PB_SIG_FF_FROM_LO), ep);
      bool ok = true;
      if (has_lo) ok = peer_wait_eq(ps.mine().sig(PB_SIG_FF_FROM_LO), ep, ps.timeout) && ok;
      if (has_hi) ok = peer_wait_eq(ps.mine().sig(PB_SIG_FF_FROM_HI), ep, ps.timeout) && ok;
      if (!ok) ctl[3] = 2;
      ctl[16] = 0;
      __threadfence();
    }
    grid.sync();
    // 2. merge what the neighbours pushed; a word that gains bits re-activates its tile for round r
    {
      int changed = 0;
      uint32_t* bmr = bm + (size_t)(r % 3) * nbw;
      for (int side = 0; side < 2; ++side) {
        if (side == 0 ? !has_lo : !has_hi) continue;
        const uint32_t* in = side == 0 ? ps.mine().ff_from_lo() : ps.mine().ff_from_hi();
        const int z0 = side == 0 ? 0 : (int)b.dz - 2;
        for (int i = gt; i < 2 * pw; i += gs) {
          const size_t wi = (size_t)z0 * pw + i;
          const uint32_t c = __ldcg(reach + wi);
          const uint32_t nwv = c | (ld_relaxed_sys_u32(in + i) & __ldg(fg + wi));
          if (nwv != c) {
            __stcg(reach + wi, nwv);
            const int z = z0 + i / pw, rem = i % pw, y = rem / b.wx, w = rem - y * b.wx;
            const int tile = ((z / b.tz) * b.nty + y / b.ty) * b.ntw + w / b.tw;
            atomicOr(&bmr[tile >> 5], 1u << (tile & 31));
            changed = 1;
          }
        }
      }
      if (__syncthreads_or(changed) && tid == 0) atomicOr(&ctl[16], 1);
    }
    __threadfence();
    grid.sync();
    // 3. did any shard gain a bit? every rank writes its flag into every mailbox
    if (blockIdx.x == 0) {
      bool ok = true;
      uint32_t got = 0;
      if (tid < ps.world) {
        const uint32_t tag = ep * 2u + (uint32_t)(__ldcg(&ctl[16]) != 0);
        st_release_sys(ps.of(tid).flags(par) + ps.rank, tag);
        const uint32_t* mine = ps.mine().flags(par) + tid;
        const long long t0 = clock64();
        uint32_t v;
        while (((v = ld_acquire_sys(mine)) >> 1) != ep) {
          if (clock64() - t0 > ps.timeout) { ok = false; break; }
          __nanosleep(64);
        }
        got = ok ? (v & 1u) : 0u;
      }
      const int any = __syncthreads_or((int)got);
      ok = __syncthreads_and(ok);
      if (tid == 0) {
        if (!ok) ctl[3] = 2;
        ctl[17] = (ok && any && __ldcg(&ctl[3]) == 0) ? 1 : 0;
        __threadfence();
      }
    }
    grid.sync();
    ++outer;
    if (__ldcg(&ctl[17]) != 1) break;
  }
  }
  if (blockIdx.x == 0 && tid == 0) {
    ctl[7] = r;
    ctl[18] = outer;
  }
}

// ---- write back ----------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_ff_write(const uint32_t* __restrict__ reach, BitVol b, T fill,
                                                  T* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t nwords = b.dz * b.dy * b.wx;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t wi0 = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; wi0 < nwords; wi0 += nwarps * 32) {
    // each lane fetches one word, then the warp expands the non-zero ones together
    int64_t mine = wi0 + lane;
    uint32_t w = mine < nwords ? __ldcg(&reach[mine]) : 0u;
    uint32_t nz = __ballot_sync(0xffffffffu, w != 0);
    while (nz) {
      int src = __ffs(nz) - 1;
      nz &= nz - 1;
      uint32_t bits = __shfl_sync(0xffffffffu, w, src);
      int64_t wi = wi0 + src;
      int64_t row = wi / b.wx;
      int64_t x = (wi - row * b.wx) * 32 + lane;
      if ((bits >> lane) & 1u) out[row * b.dx + x] = fill;
    }
  }
}

int strct_bits(const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, uint32_t* sb) {
  B2V_REQUIRE(strct_host && odz >= 1 && ody >= 1 && odx >= 1, B2V_ERR_ARG, "floodfill: bad structuring element");
  B2V_REQUIRE(odz <= 3 && ody <= 3 && odx <= 3, B2V_ERR_ARG,
              "floodfill: structuring elements larger than 3x3x3 are not supported (got %lldx%lldx%lld)",
              (long long)odz, (long long)ody, (long long)odx);
  // the centre offset moves nothing: drop it so that the standard elements match the compile-time
  // specialisations
  *sb = strct_mask(strct_host, odz, ody, odx) & ~(1u << 13);
  return B2V_OK;
}

int check_seeds(const int64_t* seeds_host, int64_t nseeds, int64_t dz, int64_t dy, int64_t dx) {
  B2V_REQUIRE(nseeds >= 0 && (nseeds == 0 || seeds_host), B2V_ERR_ARG, "floodfill: bad seed list");
  for (int64_t s = 0; s < nseeds; ++s) {
    int64_t x = seeds_host[3 * s], y = seeds_host[3 * s + 1], z = seeds_host[3 * s + 2];
    B2V_REQUIRE(x >= 0 && y >= 0 && z >= 0 && x < dx && y < dy && z < dz, B2V_ERR_RANGE,
                "floodfill: seed (%lld, %lld, %lld) outside the volume (the reference panics here)", (long long)x,
                (long long)y, (long long)z);
  }
  return B2V_OK;
}

// rounds until no tile is active. Synchronises the stream (reads one flag per batch).
int run_rounds(const BitVol& b, const Workspace& w, uint32_t sb, cudaStream_t s, int r0, int* rounds_out) {
  const int ntiles = b.ntz * b.nty * b.ntw;
  const size_t smem = 2 * (size_t)(b.tz + 2) * (b.ty + 2) * (b.tw + 2) * sizeof(uint32_t);
  int r = r0, batch = 4, rc;
  B2V_REQUIRE(r0 >= 0 && r0 + batch < kMaxRounds, B2V_ERR_NOCONV, "floodfill: round counter exhausted (%d)", r0);
  {
    const void* kr = sb == kSB6 ? (const void*)k_ff_round<kSB6> : sb == kSB26 ? (const void*)k_ff_round<kSB26>
                   : sb == kSB18 ? (const void*)k_ff_round<kSB18> : (const void*)k_ff_round<0u>;
    B2V_CUDA(cudaFuncSetAttribute(kr, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  while (true) {
    for (int k = 0; k < batch; ++k, ++r) {
#define B2V_FF_ROUND(SBC)                                                                                     \
  k_ff_round<SBC><<<ntiles, kFloodThreads, smem, s>>>(w.fg, w.reach, b, sb, w.active[r & 1], w.active[(r + 1) & 1], \
                                                      w.flags, r)
      if (sb == kSB6) B2V_FF_ROUND(kSB6);
      else if (sb == kSB26) B2V_FF_ROUND(kSB26);
      else if (sb == kSB18) B2V_FF_ROUND(kSB18);
      else B2V_FF_ROUND(0u);
#undef B2V_FF_ROUND
      if ((rc = b2v_check_launch("k_ff_round"))) return rc;
    }
    int more = 0;
    B2V_CUDA(cudaMemcpyAsync(&more, w.flags + r, sizeof(int), cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    if (!more) break;
    if (batch < 32) batch *= 2;
    B2V_REQUIRE(r + batch < kMaxRounds, B2V_ERR_NOCONV, "floodfill: no convergence after %d rounds", r);
  }
  if (rounds_out) *rounds_out = r;
  return B2V_OK;
}

// Persistent convergence: the tiles active for round r0 (seeds, merged planes) seed the first
// list; one cooperative launch runs every round to the fixed point. Synchronises the stream.
static thread_local int g_last_rounds = 0;
static thread_local int g_last_exchanges = 0;
static int g_flood_engine = 1;   // 1 persistent (default), 0 host-driven rounds

// Fetch the persistent kernel's verdict (synchronises the stream).
int persistent_verdict(const Workspace& w, cudaStream_t s) {
  int ctlh[20];
  memset(ctlh, 0, sizeof(ctlh));
  B2V_CUDA(cudaMemcpyAsync(ctlh, w.ctl, sizeof(ctlh), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  g_last_rounds = ctlh[7];
  g_last_exchanges = ctlh[18];
  B2V_REQUIRE(ctlh[3] != 2, B2V_ERR_NOCONV,
              "floodfill: a neighbour shard did not answer within the time-out (exchange %d): ranks out of step?",
              ctlh[18]);
  B2V_REQUIRE(ctlh[3] == 0, B2V_ERR_NOCONV, "floodfill: no convergence after %d rounds", ctlh[7]);
  return B2V_OK;
}

// *verdict_later: the caller queues more work behind the kernel and calls persistent_verdict()
// itself (one host round trip per flood instead of two). Cleared when the host-driven rounds ran
// instead: they have checked convergence already, and the unlaunched kernel's verdict would report 0 rounds.
int run_persistent(const BitVol& b, const Workspace& w, uint32_t sb, cudaStream_t s, int r0, int* rounds_out,
                   bool* verdict_later, const PeerSet* peer = nullptr) {
  int ntiles = b.ntz * b.nty * b.ntw;
  const size_t smem = 2 * (size_t)(b.tz + 2) * (b.ty + 2) * (b.tw + 2) * sizeof(uint32_t);
  int rc;
  const int nbw = (int)((ntiles + 31) / 32);
  uint32_t* bm = (uint32_t*)w.lists;   // three rotating tile bitmaps [3][nbw]
  const bool canon = sb == kSB6 && b.tw == 16 && b.ty == 16 && b.tz == 16;
  void* kern = peer ? (canon ? (void*)k_ff_persistent<kSB6, 4, true>
                      : sb == kSB6 ? (void*)k_ff_persistent<kSB6, 0, true>
                      : sb == kSB26 ? (void*)k_ff_persistent<kSB26, 0, true>
                      : sb == kSB18 ? (void*)k_ff_persistent<kSB18, 0, true> : (void*)k_ff_persistent<0u, 0, true>)
                    : (canon ? (void*)k_ff_persistent<kSB6, 4, false>
                      : sb == kSB6 ? (void*)k_ff_persistent<kSB6, 0, false>
                      : sb == kSB26 ? (void*)k_ff_persistent<kSB26, 0, false>
                      : sb == kSB18 ? (void*)k_ff_persistent<kSB18, 0, false> : (void*)k_ff_persistent<0u, 0, false>);
  B2V_CUDA(cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  B2V_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)kern, kFloodThreads, smem));
  B2V_REQUIRE(per_sm >= 1, B2V_ERR_CUDA, "floodfill: persistent kernel does not fit on an SM");
  int grid = per_sm * b2v_sm_count();        // every co-resident slot: one tile per block per round
  if (knobs().grid > 0 && knobs().grid < grid) grid = knobs().grid;   // tuning knob
  if (grid > ntiles) grid = (int)ntiles;
  // a block keeps at most kMaxMine tiles of a round in shared memory (4.4 G voxels at 132 blocks and 16^3-word tiles)
  if ((int64_t)grid * kMaxMine < ntiles) {
    B2V_REQUIRE(!peer, B2V_ERR_ARG, "floodfill: shard too large for the fused peer exchange (%d tiles)", ntiles);
    *verdict_later = false;
    return run_rounds(b, w, sb, s, r0, rounds_out);
  }
  k_ff_lists_init<<<1, 1024, 0, s>>>(w.active[r0 & 1], w.active[r0 & 1], (int)ntiles, bm, nbw);
  if ((rc = b2v_check_launch("k_ff_lists_init"))) return rc;
  const uint32_t* fg = w.fg;
  uint32_t* reach = w.reach;
  BitVol bb = b;
  int* ctl = w.ctl;
  int max_rounds = kMaxRounds;
  int nbw_arg = nbw;
  PeerSet pset;
  if (peer) pset = *peer; else memset(&pset, 0, sizeof(pset));
  void* args[] = {&fg, &reach, &bb, &sb, &bm, &nbw_arg, &ctl, &max_rounds, &pset};
  B2V_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kFloodThreads), args, smem, s));
  if ((rc = b2v_check_launch("k_ff_persistent"))) return rc;
  // the round flag of r0 was consumed; the next merge raises flags[r0 + 1]
  B2V_CUDA(cudaMemsetAsync(w.flags + r0, 0, sizeof(int), s));
  if (rounds_out) *rounds_out = r0 + 1;
  return *verdict_later ? B2V_OK : persistent_verdict(w, s);
}

enum { STAGE_BEGIN = 1, STAGE_CONVERGE = 2, STAGE_FINISH = 4, STAGE_ALL = 7 };

// stages: BEGIN builds the bit volumes and plants the seeds; CONVERGE runs rounds from
// *round_io until no tile is active (and stores the next free round there); FINISH writes
// `fill` into every reached voxel. The one-shot entry points run all three.
template <typename T, int MODE>
int flood(T* data, uint8_t* out, int64_t dz, int64_t dy, int64_t dx, const int64_t* seeds_host, int64_t nseeds,
          typename Thr<T>::type t0, typename Thr<T>::type t1, typename Thr<T>::type fill_t, uint8_t fill_o,
          uint32_t sb, void* workspace, cudaStream_t s, int stages, int* round_io, const PeerSet* peer = nullptr) {
  B2V_REQUIRE(data && workspace && (MODE == MODE_INPLACE || out), B2V_ERR_ARG, "floodfill: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG, "floodfill: empty volume");
  B2V_REQUIRE(dz * dy * ceil_div64(dx, 32) < (1ll << 31), B2V_ERR_ARG, "floodfill: volume too large");
  int rc;
  bool verdict_due = false;
  BitVol b = make_bitvol(dz, dy, dx);
  Workspace w = carve(workspace, b, nseeds);
  const int64_t nwords = dz * dy * b.wx;
  if (stages & STAGE_BEGIN) {
    if ((rc = check_seeds(seeds_host, nseeds, dz, dy, dx))) return rc;
    if (round_io) *round_io = 0;
    if (nseeds == 0 && stages == STAGE_ALL && !peer) return B2V_OK;
    // control region (active flags, round flags) starts clean
    B2V_CUDA(cudaMemsetAsync(w.active[0], 0, (size_t)((char*)w.seeds - (char*)w.active[0]), s));
    if (nseeds) B2V_CUDA(cudaMemcpyAsync(w.seeds, seeds_host, (size_t)nseeds * 24, cudaMemcpyHostToDevice, s));
    typedef typename Thr<T>::type TT;
    if (MODE == MODE_INPLACE)
      rc = pack_bits<T>(data, dz * dy, dx, InRangeNotFill<TT>{t0, t1, fill_t}, w.fg, w.reach, s);
    else
      rc = pack_bits<T>(data, dz * dy, dx, InRange<TT, true>{t0, MODE == MODE_EQUAL ? t0 : t1, out, fill_o}, w.fg,
                        w.reach, s);
    if (rc) return rc;
    if (nseeds) {
      k_ff_seeds<T><<<(unsigned)ceil_div64(nseeds, 128), 128, 0, s>>>(data, b, w.seeds, nseeds, t0, t1,
                                                                      MODE == MODE_EQUAL ? 1 : 0, w.fg, w.reach,
                                                                      w.active[0], w.flags);
      if ((rc = b2v_check_launch("k_ff_seeds"))) return rc;
    }
  }
  if (stages & STAGE_CONVERGE) {
    int r0 = round_io ? *round_io : 0, r1 = r0;
    verdict_due = (g_flood_engine || peer) && (stages & STAGE_FINISH);
    if (peer) {
      B2V_REQUIRE(b.dz >= 2 && b.dy * (int64_t)b.wx * 4 <= peer->pc, B2V_ERR_ARG,
                  "floodfill: the shard's planes do not fit the peer mailboxes (or the slab has < 2 planes)");
    }
    if ((rc = (g_flood_engine || peer) ? run_persistent(b, w, sb, s, r0, &r1, &verdict_due, peer)
                                       : run_rounds(b, w, sb, s, r0, &r1)))
      return rc;
    if (round_io) *round_io = r1;
  }
  if (stages & STAGE_FINISH) {
    if (MODE == MODE_INPLACE)
      k_ff_write<T><<<b2v_grid(nwords, 8, 16), 256, 0, s>>>(w.reach, b, (T)fill_t, data);
    else
      k_ff_write<uint8_t><<<b2v_grid(nwords, 8, 16), 256, 0, s>>>(w.reach, b, fill_o, out);
    if ((rc = b2v_check_launch("k_ff_write"))) return rc;
  }
  if (verdict_due) {
    if ((rc = persistent_verdict(w, s))) return rc;
    if (round_io && stages == STAGE_ALL) *round_io = g_last_rounds;
  }
  return B2V_OK;
}

// OR an externally supplied plane of reached bits (a neighbour shard's copy of the same
// voxels) into plane z; tiles that gain bits become active for round `round`.
__global__ void __launch_bounds__(256) k_ff_merge_plane(const uint32_t* __restrict__ fg, uint32_t* reach, BitVol b,
                                                        int64_t z, const uint32_t* __restrict__ ext,
                                                        uint8_t* active, int* flags, int round) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t plane = b.dy * b.wx;
  if (i >= plane) return;
  int64_t wi = z * plane + i;
  uint32_t cur = reach[wi];
  uint32_t nw = cur | (ext[i] & fg[wi]);
  if (nw != cur) {
    reach[wi] = nw;
    int64_t y = i / b.wx;
    int w = (int)(i - y * b.wx);
    int tile = ((int)(z / b.tz) * b.nty + (int)(y / b.ty)) * b.ntw + w / b.tw;
    active[tile] = 1;
    flags[round] = 1;
    // the tiles sharing this word's faces must look again as well
    int tz = (int)(z / b.tz), ty = (int)(y / b.ty), tw = w / b.tw;
    for (int oz = -1; oz <= 1; ++oz)
      for (int oy = -1; oy <= 1; ++oy)
        for (int ow = -1; ow <= 1; ++ow) {
          int nz = tz + oz, ny = ty + oy, nwi = tw + ow;
          if (nz >= 0 && nz < b.ntz && ny >= 0 && ny < b.nty && nwi >= 0 && nwi < b.ntw)
            active[(nz * b.nty + ny) * b.ntw + nwi] = 1;
        }
  }
}

template <int MODE>
int flood_dispatch(void* data, int dtype, uint8_t* out, int64_t dz, int64_t dy, int64_t dx, const int64_t* seeds_host,
                   int64_t nseeds, double t0, double t1, double fill_t, uint8_t fill_o, uint32_t sb, void* workspace,
                   cudaStream_t s, int stages, int* round_io, const PeerSet* peer = nullptr) {
  B2V_REQUIRE(t0 == t0 && t1 == t1 && fill_t == fill_t, B2V_ERR_ARG, "floodfill: NaN threshold");
  if (dtype == B2V_I16 || dtype == B2V_U8) {
    // Inclusive bounds on integer data: a fractional bound is equivalent to ceil(t0) / floor(t1)
    // (MODE_EQUAL: a non-integer value matches nothing); clamped well inside int32 so the casts
    // are defined for +-inf and huge values.
    const double lim = 1073741824.0;   // 2^30
    double a = MODE == MODE_EQUAL ? t0 : ceil(t0), b = MODE == MODE_EQUAL ? t0 : floor(t1);
    if (MODE == MODE_EQUAL && t0 != floor(t0)) { a = lim; b = lim; }   // matches no integer voxel
    a = a < -lim ? -lim : (a > lim ? lim : a);
    b = b < -lim ? -lim : (b > lim ? lim : b);
    const double f = fill_t < -lim ? -lim : (fill_t > lim ? lim : fill_t);
    if (dtype == B2V_I16)
      return flood<int16_t, MODE>((int16_t*)data, out, dz, dy, dx, seeds_host, nseeds, (int)a, (int)b, (int)f,
                                  fill_o, sb, workspace, s, stages, round_io, peer);
    return flood<uint8_t, MODE>((uint8_t*)data, out, dz, dy, dx, seeds_host, nseeds, (int)a, (int)b, (int)f,
                                fill_o, sb, workspace, s, stages, round_io, peer);
  }
  if (dtype == B2V_F64)
    return flood<double, MODE>((double*)data, out, dz, dy, dx, seeds_host, nseeds, t0, t1, fill_t, fill_o, sb,
                               workspace, s, stages, round_io, peer);
  B2V_REQUIRE(false, B2V_ERR_ARG, "floodfill: unknown dtype code %d", dtype);
}

}  // namespace

extern "C" void b2v_floodfill_set_engine(int persistent) { g_flood_engine = persistent ? 1 : 0; }

extern "C" int64_t b2v_floodfill_workspace_bytes(int64_t dz, int64_t dy, int64_t dx, int64_t nseeds) {
  if (dz <= 0 || dy <= 0 || dx <= 0) return 0;
  BitVol b = make_bitvol(dz, dy, dx);
  return carve(nullptr, b, nseeds).bytes;
}

extern "C" int b2v_floodfill_threshold(const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                       const int64_t* seeds_host, int64_t nseeds, double t0, double t1, uint8_t fill,
                                       const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx,
                                       uint8_t* out, void* workspace, void* stream, int* rounds_out) {
  uint32_t sb;
  int rc;
  if ((rc = strct_bits(strct_host, odz, ody, odx, &sb))) return rc;
  if (rounds_out) *rounds_out = 0;
  return flood_dispatch<MODE_THRESHOLD>(const_cast<void*>(data), dtype, out, dz, dy, dx, seeds_host, nseeds, t0, t1,
                                        0.0, fill, sb, workspace, (cudaStream_t)stream, STAGE_ALL, rounds_out);
}

extern "C" int b2v_floodfill_threshold_inplace(void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                               const int64_t* seeds_host, int64_t nseeds, double t0, double t1,
                                               double fill, const uint8_t* strct_host, int64_t odz, int64_t ody,
                                               int64_t odx, void* workspace, void* stream, int* rounds_out) {
  uint32_t sb;
  int rc;
  if ((rc = strct_bits(strct_host, odz, ody, odx, &sb))) return rc;
  if (rounds_out) *rounds_out = 0;
  return flood_dispatch<MODE_INPLACE>(data, dtype, nullptr, dz, dy, dx, seeds_host, nseeds, t0, t1, fill, 0, sb,
                                      workspace, (cudaStream_t)stream, STAGE_ALL, rounds_out);
}

extern "C" int b2v_floodfill_equal(const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx, int64_t i,
                                   int64_t j, int64_t k, double v, uint8_t fill, uint8_t* out, void* workspace,
                                   void* stream, int* rounds_out) {
  const uint32_t sb = kSB6;
  int64_t seed[3] = {i, j, k};
  if (rounds_out) *rounds_out = 0;
  return flood_dispatch<MODE_EQUAL>(const_cast<void*>(data), dtype, out, dz, dy, dx, seed, 1, v, v, 0.0, fill, sb,
                                    workspace, (cudaStream_t)stream, STAGE_ALL, rounds_out);
}

// ---- staged interface for Z-sharded volumes (dist.py) ---------------------------------------
extern "C" int b2v_floodfill_threshold_staged(int stages, const void* data, int dtype, int64_t dz, int64_t dy,
                                              int64_t dx, const int64_t* seeds_host, int64_t nseeds, double t0,
                                              double t1, uint8_t fill, const uint8_t* strct_host, int64_t odz,
                                              int64_t ody, int64_t odx, uint8_t* out, void* workspace, void* stream,
                                              int* round_io) {
  uint32_t sb;
  int rc;
  if ((rc = strct_bits(strct_host, odz, ody, odx, &sb))) return rc;
  B2V_REQUIRE(stages > 0 && stages <= STAGE_ALL && round_io, B2V_ERR_ARG, "floodfill_staged: bad stage mask");
  return flood_dispatch<MODE_THRESHOLD>(const_cast<void*>(data), dtype, out, dz, dy, dx, seeds_host, nseeds, t0, t1,
                                        0.0, fill, sb, workspace, (cudaStream_t)stream, stages, round_io);
}

// One Z shard of a sharded flood with the boundary exchange fused into the persistent kernel
// (peer mailboxes over NVLink, csrc/peer.cuh). data / out are the EXTENDED slab (own planes plus
// one halo plane per inner side, halo planes of `data` valid), seeds are local to it. Every rank
// of the job must make this call with the same `epoch`; *epochs_used_out tells how many
// exchanges (epochs) the call consumed — the same number on every rank. Synchronises the stream.
extern "C" int b2v_floodfill_threshold_peer(const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                            const int64_t* seeds_host, int64_t nseeds, double t0, double t1,
                                            uint8_t fill, const uint8_t* strct_host, int64_t odz, int64_t ody,
                                            int64_t odx, uint8_t* out, void* workspace, void* stream, int rank,
                                            int world, const void* const* mailboxes_host, int64_t mailbox_plane_bytes,
                                            uint32_t epoch, int* rounds_out, int* epochs_used_out) {
  uint32_t sb;
  int rc;
  if ((rc = strct_bits(strct_host, odz, ody, odx, &sb))) return rc;
  B2V_REQUIRE(epoch >= 1 && epochs_used_out, B2V_ERR_ARG, "floodfill_peer: epochs start at 1");
  PeerSet ps;
  if ((rc = peer_make_set(rank, world, mailboxes_host, mailbox_plane_bytes, epoch, &ps))) return rc;
  int rounds = 0;
  *epochs_used_out = 0;
  rc = flood_dispatch<MODE_THRESHOLD>(const_cast<void*>(data), dtype, out, dz, dy, dx, seeds_host, nseeds, t0, t1, 0.0,
                                      fill, sb, workspace, (cudaStream_t)stream, STAGE_ALL, &rounds, &ps);
  *epochs_used_out = g_last_exchanges;
  if (rounds_out) *rounds_out = rounds;
  return rc;
}

extern "C" int b2v_floodfill_layout(int64_t dz, int64_t dy, int64_t dx, int64_t nseeds, int64_t* layout_out) {
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0 && layout_out, B2V_ERR_ARG, "floodfill_layout: bad arguments");
  BitVol b = make_bitvol(dz, dy, dx);
  Workspace w = carve(nullptr, b, nseeds);
  layout_out[0] = (int64_t)((char*)w.fg - (char*)nullptr);
  layout_out[1] = (int64_t)((char*)w.reach - (char*)nullptr);
  layout_out[2] = (int64_t)((char*)w.flags - (char*)nullptr);
  layout_out[3] = (int64_t)b.dy * b.wx * 4;  // bytes per z-plane of a bit volume
  layout_out[4] = (int64_t)b.ntz * b.nty * b.ntw;
  layout_out[5] = kMaxRounds;
  layout_out[6] = (int64_t)((char*)w.ctl - (char*)nullptr);  // int32 ctl[]: [7] rounds of the persistent kernel
  return B2V_OK;
}

extern "C" int b2v_floodfill_merge_plane(int64_t dz, int64_t dy, int64_t dx, int64_t nseeds, void* workspace,
                                         int64_t z, const uint32_t* plane_bits, int round, void* stream) {
  B2V_REQUIRE(workspace && plane_bits && z >= 0 && z < dz && round >= 0 && round < kMaxRounds, B2V_ERR_ARG,
              "floodfill_merge_plane: bad arguments");
  BitVol b = make_bitvol(dz, dy, dx);
  Workspace w = carve(workspace, b, nseeds);
  int64_t plane = b.dy * b.wx;
  k_ff_merge_plane<<<(unsigned)ceil_div64(plane, 256), 256, 0, (cudaStream_t)stream>>>(
      w.fg, w.reach, b, z, plane_bits, w.active[round & 1], w.flags, round);
  return b2v_check_launch("k_ff_merge_plane");
}

// ---- fill holes -------------------------------------------------------------------------------
// fill_holes_automatically_internal, floodfill.rs:51-94: histogram the labels, then every
// voxel whose label has at most max_size voxels becomes 254 (label 0 included).
namespace {

__global__ void __launch_bounds__(256) k_fh_hist(const uint32_t* __restrict__ labels, int64_t n, uint32_t nlabels,
                                                 uint32_t* sizes, int* status) {
  // runs of equal labels are common (label images are piecewise constant along x):
  // each thread folds its 8 consecutive voxels into runs before touching global atomics
  int64_t stride = (int64_t)gridDim.x * blockDim.x * 8;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8; i0 < n; i0 += stride) {
    uint32_t cur = 0xffffffffu, cnt = 0;
    int64_t i1 = i0 + 8 < n ? i0 + 8 : n;
    for (int64_t i = i0; i < i1; ++i) {
      uint32_t l = labels[i];
      if (l == cur) { ++cnt; continue; }
      if (cnt) atomicAdd(&sizes[cur], cnt);
      if (l > nlabels) { *status = 1; cur = 0xffffffffu; cnt = 0; continue; }
      cur = l; cnt = 1;
    }
    if (cnt) atomicAdd(&sizes[cur], cnt);
  }
}

__global__ void __launch_bounds__(256) k_fh_any(const uint32_t* __restrict__ sizes, int64_t nbins, uint32_t max_size,
                                                int* modified) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool hit = i < nbins && sizes[i] > 0 && sizes[i] <= max_size;
  if (__syncthreads_or(hit) && threadIdx.x == 0) *modified = 1;
}

__global__ void __launch_bounds__(256) k_fh_apply(const uint32_t* __restrict__ labels, int64_t n,
                                                  const uint32_t* __restrict__ sizes, uint32_t nlabels,
                                                  uint32_t max_size, const int* __restrict__ ctrl,
                                                  uint8_t* __restrict__ mask) {
  // ctrl[0] = something qualifies, ctrl[1] = a label exceeded nlabels (reported as B2V_ERR_RANGE:
  // the mask is left untouched and no size is read out of bounds)
  if (ctrl[0] == 0 || ctrl[1] != 0) return;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t l = labels[i];
    if (l <= nlabels && __ldg(&sizes[l]) <= max_size) mask[i] = 254;
  }
}

}  // namespace

extern "C" int64_t b2v_fill_holes_workspace_bytes(uint32_t nlabels) { return ((int64_t)nlabels + 1) * 4 + 256; }

// stages (bit mask): 1 HISTOGRAM (label sizes of this buffer into the workspace: uint32 [nlabels + 1]
// at byte offset 256 — a Z shard all-reduces them with its peers before stage 2), 2 APPLY (qualify,
// write 254, report). The one-shot entry runs both.
extern "C" int b2v_fill_holes_staged(int stages, uint8_t* mask, const uint32_t* labels, int64_t n, uint32_t nlabels,
                                     uint32_t max_size, void* workspace, void* stream, int* modified_out) {
  B2V_REQUIRE(mask && labels && workspace && modified_out, B2V_ERR_ARG, "fill_holes: null pointer");
  B2V_REQUIRE(n >= 0, B2V_ERR_ARG, "fill_holes: negative size");
  cudaStream_t s = (cudaStream_t)stream;
  int* ctrl = (int*)workspace;            // [0] modified, [1] status
  uint32_t* sizes = (uint32_t*)((char*)workspace + 256);
  int64_t nbins = (int64_t)nlabels + 1;
  int rc;
  if (stages & 1) {
    B2V_CUDA(cudaMemsetAsync(workspace, 0, (size_t)(256 + nbins * 4), s));
    if (n > 0) {
      k_fh_hist<<<b2v_grid(n, 256 * 8, 16), 256, 0, s>>>(labels, n, nlabels, sizes, ctrl + 1);
      if ((rc = b2v_check_launch("k_fh_hist"))) return rc;
    }
  }
  if (stages & 2) {
    k_fh_any<<<(unsigned)ceil_div64(nbins, 256), 256, 0, s>>>(sizes, nbins, max_size, ctrl);
    if ((rc = b2v_check_launch("k_fh_any"))) return rc;
    if (n > 0) {
      k_fh_apply<<<b2v_grid(n, 256, 16), 256, 0, s>>>(labels, n, sizes, nlabels, max_size, ctrl, mask);
      if ((rc = b2v_check_launch("k_fh_apply"))) return rc;
    }
    int host[2] = {0, 0};
    B2V_CUDA(cudaMemcpyAsync(host, ctrl, sizeof(host), cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    B2V_REQUIRE(host[1] == 0, B2V_ERR_RANGE, "fill_holes: a label exceeds nlabels (the reference panics here)");
    *modified_out = host[0];
  }
  return B2V_OK;
}

extern "C" int b2v_fill_holes(uint8_t* mask, const uint32_t* labels, int64_t n, uint32_t nlabels, uint32_t max_size,
                              void* workspace, void* stream, int* modified_out) {
  return b2v_fill_holes_staged(3, mask, labels, n, nlabels, max_size, workspace, stream, modified_out);
}
