// Marching cubes: classify -> scan -> emit, on a bit-packed inside volume.
// Replaces the per-piece vtkContourFilter step of invesalius/data/surface_process.py:71-201
// (geometry: converters.py:34-101). Canonical output order is defined in DESIGN.md and
// restated by the CPU checker; VTK itself is not available, so parity to VTK is unpinned.
//
//   1. bits   (HBM-bound, the only pass over the volume: 1 B/voxel uint8, 2 B/voxel int16):
//             inside(p) = S[p] >= iso packed 32 voxels per word along x (bitpack.cuh).
//   2. classify + compact (on bits, L2 resident, ONE pass): per word the crossing masks towards
//             +x/+y/+z, the owned vertices (popcounts) and the triangles of its active cells;
//             non-empty words are appended in word order to two compact lists, the running
//             offsets carried from tile to tile by a chained (decoupled look-back) scan.
//   3. emit   one thread per vertex and one thread per active cell over the compact lists; a
//             vertex id is  voff[owner word] + popcounts below the owner bit, each owner
//             record fetched once per cell.
#include "b2v_common.cuh"
#include "bitpack.cuh"
#include "peer.cuh"
#define B2V_MC_QUAL __device__
#include "mc_tables.h"

namespace {

struct McGeom {
  int64_t nz, ny, nx;
  int wx;           // words per row
  int64_t nwords;   // < 2^31 (checked on entry): word indices and dims fit 32 bits in the kernels
  int inz, iny;     // 32-bit copies
  int wx_sh, ny_sh; // log2 when a power of two (the usual case), else -1
};

McGeom make_geom(int64_t nz, int64_t ny, int64_t nx) {
  McGeom g;
  g.nz = nz; g.ny = ny; g.nx = nx;
  g.wx = (int)ceil_div64(nx, 32);
  g.nwords = nz * ny * g.wx;
  g.inz = (int)nz; g.iny = (int)ny;
  auto lg = [](int64_t v) { int s = 0; while ((1ll << s) < v) ++s; return (1ll << s) == v ? s : -1; };
  g.wx_sh = lg(g.wx);
  g.ny_sh = lg(ny);
  return g;
}

// word index -> (z, y, w) in 32-bit arithmetic, shifts when the dims are powers of two
__device__ __forceinline__ void split_word(const McGeom& g, uint32_t wi, int& z, int& y, int& w) {
  uint32_t row;
  if (g.wx_sh >= 0) { row = wi >> g.wx_sh; w = (int)(wi & (uint32_t)(g.wx - 1)); }
  else { row = wi / (uint32_t)g.wx; w = (int)(wi - row * (uint32_t)g.wx); }
  if (g.ny_sh >= 0) { z = (int)(row >> g.ny_sh); y = (int)(row & (uint32_t)(g.iny - 1)); }
  else { z = (int)(row / (uint32_t)g.iny); y = (int)(row - (uint32_t)z * (uint32_t)g.iny); }
}

constexpr int kTileThreads = 256;
constexpr int kWPT = 4;                              // words per thread
constexpr int kTileWords = kTileThreads * kWPT;      // one tile = 1024 consecutive words
constexpr int kTileShift = 10;

struct McWs {
  uint32_t* bits;    // [nwords] inside bits
  uint4* vrec;       // [ntiles * 1024] per word (cx, cy, cz, exclusive vertex offset INSIDE its tile); written for
                     // the tiles that hold vertices only
  uint4* tcnt;       // [ntiles] per tile (vertices, active cells, triangles, 0)
  uint4* toff;       // [ntiles] their exclusive prefixes over the tiles
  uint4* plane0;     // [ny * wx] dense records of plane 0 with GLOBAL vertex offsets (Z-sharded volumes)
  unsigned long long* totals;  // [0] V, [1] T, [2] active cells
  unsigned int* ticket;        // tiles done (the last one scans the tile counts)
  int64_t ctl_bytes; // totals + ticket: zeroed before every classify
  int64_t bytes;
};

McWs carve(void* base, const McGeom& g) {
  McWs w;
  char* p = (char*)base;
  int64_t off = 0;
  const int64_t ntiles = ceil_div64(g.nwords, kTileWords);
  w.bits = (uint32_t*)(p + off); off += align256(g.nwords * 4 + 64);
  w.vrec = (uint4*)(p + off); off += align256(ntiles * kTileWords * 16);
  w.tcnt = (uint4*)(p + off); off += align256(ntiles * 16);
  w.toff = (uint4*)(p + off); off += align256(ntiles * 16);
  w.plane0 = (uint4*)(p + off); off += align256(g.ny * g.wx * 16);
  const int64_t ctl0 = off;
  w.totals = (unsigned long long*)(p + off); off += 256;
  w.ticket = (unsigned int*)(p + off); off += 256;
  w.ctl_bytes = off - ctl0;
  w.bytes = off;
  return w;
}

// ---- 2. classify (one pass over the bits, per-TILE counts, scan of the tile counts) ----------
// The surface touches a few per cent of the words. A tile is 1024 consecutive words (4 per
// thread). One pass classifies every word (crossing masks towards +x/+y/+z, active cells,
// triangle count); a tile that holds nothing writes one zero count and leaves. The others scan
// their words' vertex counts inside the block and write the dense per-word records
// vrec[word] = (cx, cy, cz, exclusive vertex offset inside the tile): what a triangle corner
// needs to turn "crossing edge owned by word W, bit b" into a vertex id. Only per-TILE counts
// are scanned across the volume (4096 entries at 512^3): the last tile to finish does it in the
// same launch. The emit kernels re-derive everything else from the bits.
struct Rows {       // the four bit rows a cell row touches, word w and bit 0 of word w+1
  uint32_t i00, i01, i10, i11;  // [cz][cy]
  uint32_t n00, n01, n10, n11;  // next word in x (0 past the row end)
};

// bit i of the result = bit i+1 of the 64-bit (hi:lo)
__device__ __forceinline__ uint32_t shift_in(uint32_t lo, uint32_t hi) { return (lo >> 1) | (hi << 31); }

// bits i with x = 32 w + i and x + 1 < nx
__device__ __forceinline__ uint32_t valid_x1(const McGeom& g, int w) {
  const int rem = (int)g.nx - 1 - w * 32;  // number of valid bits
  return rem >= 32 ? 0xffffffffu : (rem <= 0 ? 0u : ((1u << rem) - 1u));
}

__device__ __forceinline__ int cell_case(const Rows& r, int i) {
  uint32_t a = __funnelshift_r(r.i00, r.n00, i) & 3u;
  uint32_t b = __funnelshift_r(r.i01, r.n01, i) & 3u;
  uint32_t c = __funnelshift_r(r.i10, r.n10, i) & 3u;
  uint32_t d = __funnelshift_r(r.i11, r.n11, i) & 3u;
  return (int)(a | (b << 2) | (c << 4) | (d << 6));
}

__device__ __forceinline__ Rows load_rows(const uint32_t* __restrict__ bits, const McGeom& g, int z, int y, int w) {
  Rows r;
  const bool hy = y + 1 < g.iny, hz = z + 1 < g.inz, hn = w + 1 < g.wx;
  const uint32_t b00 = ((uint32_t)z * (uint32_t)g.iny + (uint32_t)y) * (uint32_t)g.wx + (uint32_t)w;
  const uint32_t b01 = b00 + (uint32_t)g.wx, b10 = b00 + (uint32_t)g.iny * (uint32_t)g.wx, b11 = b10 + (uint32_t)g.wx;
  r.i00 = __ldg(bits + b00);
  r.i01 = hy ? __ldg(bits + b01) : 0u;
  r.i10 = hz ? __ldg(bits + b10) : 0u;
  r.i11 = (hy && hz) ? __ldg(bits + b11) : 0u;
  r.n00 = hn ? __ldg(bits + b00 + 1) : 0u;
  r.n01 = (hn && hy) ? __ldg(bits + b01 + 1) : 0u;
  r.n10 = (hn && hz) ? __ldg(bits + b10 + 1) : 0u;
  r.n11 = (hn && hy && hz) ? __ldg(bits + b11 + 1) : 0u;
  return r;
}

// The four words of one thread: rows, position, validity. VEC (wx % 4 == 0): the four words lie
// in one row and every bit row is one aligned 128-bit load.
struct Word4 {
  Rows r[kWPT];
  int z[kWPT], y[kWPT], w[kWPT];
  bool ok[kWPT];
};

template <bool VEC>
__device__ __forceinline__ void load_word4(const uint32_t* __restrict__ bits, const McGeom& g, uint32_t wi0,
                                           Word4& q) {
  const uint32_t nwords = (uint32_t)g.nwords;
  if (VEC) {
    const bool ok = wi0 < nwords;
    int z = 0, y = 0, w0 = 0;
    uint32_t a00[kWPT + 1] = {0, 0, 0, 0, 0}, a01[kWPT + 1] = {0, 0, 0, 0, 0}, a10[kWPT + 1] = {0, 0, 0, 0, 0},
             a11[kWPT + 1] = {0, 0, 0, 0, 0};
    if (ok) {
      split_word(g, wi0, z, y, w0);
      const bool hy = y + 1 < g.iny, hz = z + 1 < g.inz;
      const uint32_t b00 = wi0, b01 = b00 + (uint32_t)g.wx, b10 = b00 + (uint32_t)g.iny * (uint32_t)g.wx,
                     b11 = b10 + (uint32_t)g.wx;
      const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
      const uint4 q00 = __ldg((const uint4*)(bits + b00));
      const uint4 q01 = hy ? __ldg((const uint4*)(bits + b01)) : z4;
      const uint4 q10 = hz ? __ldg((const uint4*)(bits + b10)) : z4;
      const uint4 q11 = (hy && hz) ? __ldg((const uint4*)(bits + b11)) : z4;
      a00[0] = q00.x; a00[1] = q00.y; a00[2] = q00.z; a00[3] = q00.w;
      a01[0] = q01.x; a01[1] = q01.y; a01[2] = q01.z; a01[3] = q01.w;
      a10[0] = q10.x; a10[1] = q10.y; a10[2] = q10.z; a10[3] = q10.w;
      a11[0] = q11.x; a11[1] = q11.y; a11[2] = q11.z; a11[3] = q11.w;
    }
    // the word after my four is the first word of the next lane (same row unless mine end it)
    {
      const int lane = threadIdx.x & 31;
      const uint32_t s00 = __shfl_down_sync(0xffffffffu, a00[0], 1), s01 = __shfl_down_sync(0xffffffffu, a01[0], 1),
                     s10 = __shfl_down_sync(0xffffffffu, a10[0], 1), s11 = __shfl_down_sync(0xffffffffu, a11[0], 1);
      if (ok && w0 + kWPT < g.wx) {
        if (lane < 31) { a00[kWPT] = s00; a01[kWPT] = s01; a10[kWPT] = s10; a11[kWPT] = s11; }
        else {
          const bool hy = y + 1 < g.iny, hz = z + 1 < g.inz;
          const uint32_t b00 = wi0 + kWPT, b01 = b00 + (uint32_t)g.wx, b10 = b00 + (uint32_t)g.iny * (uint32_t)g.wx,
                         b11 = b10 + (uint32_t)g.wx;
          a00[kWPT] = __ldg(bits + b00);
          a01[kWPT] = hy ? __ldg(bits + b01) : 0u;
          a10[kWPT] = hz ? __ldg(bits + b10) : 0u;
          a11[kWPT] = (hy && hz) ? __ldg(bits + b11) : 0u;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kWPT; ++j) {
      q.r[j] = Rows{a00[j], a01[j], a10[j], a11[j], a00[j + 1], a01[j + 1], a10[j + 1], a11[j + 1]};
      q.z[j] = z; q.y[j] = y; q.w[j] = w0 + j; q.ok[j] = ok;
    }
  } else {
#pragma unroll
    for (int j = 0; j < kWPT; ++j) {
      q.ok[j] = wi0 + j < nwords;
      q.z[j] = q.y[j] = q.w[j] = 0;
      q.r[j] = Rows{0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
      if (q.ok[j]) {
        split_word(g, wi0 + j, q.z[j], q.y[j], q.w[j]);
        q.r[j] = load_rows(bits, g, q.z[j], q.y[j], q.w[j]);
      }
    }
  }
}

// a word whose whole 2 x 2-row neighbourhood is uniform (most of the volume) holds nothing: all
// outside (missing rows / words read as 0), or all inside with every neighbour present
__device__ __forceinline__ bool word_uniform(const Rows& r, const McGeom& g, int z, int y, int w) {
  const uint32_t o_ = r.i00 | r.i01 | r.i10 | r.i11 | ((r.n00 | r.n01 | r.n10 | r.n11) & 1u);
  if (o_ == 0u) return true;
  return y + 1 < g.iny && z + 1 < g.inz && w + 1 < g.wx && (r.i00 & r.i01 & r.i10 & r.i11) == 0xffffffffu &&
         ((r.n00 & r.n01 & r.n10 & r.n11) & 1u);
}

// active cells of a word: corners neither all outside nor all inside
__device__ __forceinline__ uint32_t active_cells(const Rows& r, uint32_t vx) {
  const uint32_t s00 = shift_in(r.i00, r.n00), s01 = shift_in(r.i01, r.n01), s10 = shift_in(r.i10, r.n10),
                 s11 = shift_in(r.i11, r.n11);
  const uint32_t any = r.i00 | r.i01 | r.i10 | r.i11 | s00 | s01 | s10 | s11;
  const uint32_t all = r.i00 & r.i01 & r.i10 & r.i11 & s00 & s01 & s10 & s11;
  return any & ~all & vx;
}

// block-wide exclusive scan of a 64-bit value (256 threads); returns the exclusive prefix, *total = block sum.
// s_w: 8 words of shared scratch; two barriers.
__device__ __forceinline__ unsigned long long block_scan_u64(unsigned long long x, unsigned long long* s_w,
                                                             unsigned long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long ix = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long p = __shfl_up_sync(0xffffffffu, ix, o);
    if (lane >= o) ix += p;
  }
  __syncthreads();            // s_w free (previous use read)
  if (lane == 31) s_w[warp] = ix;
  __syncthreads();
  unsigned long long before = 0, tot = 0;
#pragma unroll
  for (int k = 0; k < kTileThreads / 32; ++k) {
    const unsigned long long v = s_w[k];
    if (k < warp) before += v;
    tot += v;
  }
  *total = tot;
  return before + ix - x;
}

// same for a 32-bit value (s_w: 8 words)
__device__ __forceinline__ uint32_t block_scan_u32(uint32_t x, uint32_t* s_w, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t ix = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t p = __shfl_up_sync(0xffffffffu, ix, o);
    if (lane >= o) ix += p;
  }
  __syncthreads();
  if (lane == 31) s_w[warp] = ix;
  __syncthreads();
  uint32_t before = 0, tot = 0;
#pragma unroll
  for (int k = 0; k < kTileThreads / 32; ++k) {
    const uint32_t v = s_w[k];
    if (k < warp) before += v;
    tot += v;
  }
  *total = tot;
  return before + ix - x;
}

// position of the n-th (0-based) set bit of m (n < popc(m))
__device__ __forceinline__ int nth_set_bit(uint32_t m, int n) {
  int pos = 0;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const int c = __popc((m >> pos) & ((1u << s) - 1u));
    if (n >= c) { n -= c; pos += s; }
  }
  return pos;
}

template <bool VEC>
__global__ void __launch_bounds__(kTileThreads, 4) k_mc_classify(const uint32_t* __restrict__ bits, McGeom g,
                                                              int skip_last, uint4* __restrict__ vrec,
                                                              uint4* tcnt, uint4* toff, unsigned int* ticket,
                                                              unsigned long long* totals, int ntiles) {
  __shared__ unsigned char s_ntri[256];
  __shared__ unsigned long long s_w[kTileThreads / 32];
  __shared__ unsigned long long s_carry[3];
  __shared__ int s_last;
  const int tid = threadIdx.x;
  s_ntri[tid] = B2V_MC_NTRI[tid];
  __syncthreads();
  const int tile = blockIdx.x;
  const uint32_t wi0 = ((uint32_t)tile * kTileThreads + tid) * kWPT;
  Word4 q;
  load_word4<VEC>(bits, g, wi0, q);
  uint32_t cx[kWPT], cy[kWPT], cz[kWPT], nv[kWPT];
  // packed thread sums: vertices (bits 0..19) | active cells (20..39) | triangles (40..63)
  unsigned long long X = 0;
#pragma unroll
  for (int j = 0; j < kWPT; ++j) {
    cx[j] = cy[j] = cz[j] = nv[j] = 0u;
    if (!q.ok[j] || word_uniform(q.r[j], g, q.z[j], q.y[j], q.w[j])) continue;
    const Rows& r = q.r[j];
    const bool hy = q.y[j] + 1 < g.iny, hz = q.z[j] + 1 < g.inz;
    const uint32_t vx = valid_x1(g, q.w[j]);
    cx[j] = (r.i00 ^ shift_in(r.i00, r.n00)) & vx;
    cy[j] = hy ? (r.i00 ^ r.i01) : 0u;
    cz[j] = hz ? (r.i00 ^ r.i10) : 0u;
    // a Z shard does not own the vertices of its last (shared) plane: the next shard does
    const bool own = !(skip_last && q.z[j] == g.inz - 1);
    nv[j] = own ? __popc(cx[j]) + __popc(cy[j]) + __popc(cz[j]) : 0;
    uint32_t nt = 0, act = 0;
    if (hy && hz) {
      act = active_cells(r, vx);
      for (uint32_t m = act; m; m &= m - 1) nt += s_ntri[cell_case(r, __ffs(m) - 1)];
    }
    X += (unsigned long long)nv[j] | ((unsigned long long)__popc(act) << 20) | ((unsigned long long)nt << 40);
  }
  if (__syncthreads_or(X != 0ull)) {
    unsigned long long tot;
    const unsigned long long ex = block_scan_u64(X, s_w, &tot);
    const uint32_t tv = (uint32_t)(tot & 0xfffffu);
    if (tv) {   // the records are read by the vertex emitter (this tile) and by triangle corners (any tile)
      uint32_t run = (uint32_t)(ex & 0xfffffu);
#pragma unroll
      for (int j = 0; j < kWPT; ++j) {
        vrec[wi0 + j] = make_uint4(cx[j], cy[j], cz[j], run);
        run += nv[j];
      }
    }
    if (tid == 0) tcnt[tile] = make_uint4(tv, (uint32_t)((tot >> 20) & 0xfffffu), (uint32_t)(tot >> 40), 0u);
  } else if (tid == 0) {
    tcnt[tile] = make_uint4(0u, 0u, 0u, 0u);
  }
  // the last tile to finish turns the tile counts into exclusive prefixes (thread 0 wrote this
  // tile's count: its fence orders that store before the ticket)
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(ticket, 1u) == (unsigned)(ntiles - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (tid < 3) s_carry[tid] = 0ull;
  constexpr int kPer = 8;
  for (int base = 0; base < ntiles; base += kTileThreads * kPer) {
    uint4 c[kPer];
    unsigned long long sv = 0, sc = 0, st = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int i = base + tid * kPer + k;
      c[k] = i < ntiles ? __ldcg(tcnt + i) : make_uint4(0u, 0u, 0u, 0u);
      sv += c[k].x; sc += c[k].y; st += c[k].z;
    }
    unsigned long long tv, tc, tt;
    unsigned long long ev = block_scan_u64(sv, s_w, &tv);
    unsigned long long ec = block_scan_u64(sc, s_w, &tc);
    unsigned long long et = block_scan_u64(st, s_w, &tt);
    ev += s_carry[0]; ec += s_carry[1]; et += s_carry[2];
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
      const int i = base + tid * kPer + k;
      if (i < ntiles) toff[i] = make_uint4((uint32_t)ev, (uint32_t)ec, (uint32_t)et, 0u);
      ev += c[k].x; ec += c[k].y; et += c[k].z;
    }
    __syncthreads();
    if (tid == 0) { s_carry[0] += tv; s_carry[1] += tc; s_carry[2] += tt; }
    __syncthreads();
  }
  if (tid == 0) { totals[0] = s_carry[0]; totals[1] = s_carry[2]; totals[2] = s_carry[1]; }
}

// dense per-word records (cx, cy, cz, GLOBAL exclusive vertex offset) of plane 0: what the shard
// BELOW needs to number the vertices of the plane it shares with this one (b2v_mc_emit_shard)
__global__ void __launch_bounds__(256) k_mc_plane0(const uint32_t* __restrict__ bits, McGeom g,
                                                   const uint4* __restrict__ vrec, const uint4* __restrict__ tcnt,
                                                   const uint4* __restrict__ toff, uint4* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.iny * g.wx) return;
  const int y = i / g.wx;
  const int w = i - y * g.wx;
  const Rows r = load_rows(bits, g, 0, y, w);
  const uint32_t cx = (r.i00 ^ shift_in(r.i00, r.n00)) & valid_x1(g, w);
  const uint32_t cy = y + 1 < g.iny ? (r.i00 ^ r.i01) : 0u;
  const uint32_t cz = g.inz > 1 ? (r.i00 ^ r.i10) : 0u;
  const int t = i >> kTileShift;
  const uint32_t voff = ((cx | cy | cz) && __ldg(&tcnt[t].x)) ? __ldg(&toff[t].x) + __ldg(&vrec[i].w) : 0u;
  out[i] = make_uint4(cx, cy, cz, voff);
}

// ---- 3. emit ---------------------------------------------------------------------------------
// One block per tile that holds something; one thread per VERTEX and one thread per ACTIVE CELL
// (the surface touches a few cells per word: a warp-per-word emitter leaves most lanes idle). A
// thread finds its word by bisecting the tile's 1024 exclusive offsets in shared memory, then its
// voxel / cell by popcounts. Outputs of consecutive threads are consecutive in memory.
struct McXform {
  float sx, sy, sz;
  int ox, oy, oz;
  int flip_y;
  float iso;
};

__device__ __forceinline__ uint32_t below(int i) { return i >= 32 ? 0xffffffffu : ((1u << i) - 1u); }

// largest l in [0, 1024) with key[l] <= k (key non-decreasing, key[0] <= k)
template <typename F>
__device__ __forceinline__ int tile_locate(uint32_t k, F key) {
  int lo = 0;
#pragma unroll
  for (int step = kTileWords / 2; step > 0; step >>= 1)
    if (key(lo + step) <= k) lo += step;
  return lo;
}

template <typename T>
__global__ void __launch_bounds__(kTileThreads) k_mc_emit_verts(const T* __restrict__ vol, McGeom g,
                                                                const uint4* __restrict__ vrec,
                                                                const uint4* __restrict__ tcnt,
                                                                const uint4* __restrict__ toff, int ntiles,
                                                                McXform xf, float* __restrict__ verts) {
  __shared__ uint4 s_rec[kTileWords];
  const int tid = threadIdx.x;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const uint32_t V = __ldg(&tcnt[tile].x);
    if (V == 0u) continue;
    const uint32_t vbase = __ldg(&toff[tile].x);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kWPT; ++k) s_rec[tid + k * kTileThreads] = __ldg(vrec + ((size_t)tile << kTileShift) + tid + k * kTileThreads);
    __syncthreads();
    for (uint32_t k = tid; k < V; k += kTileThreads) {
      const int l = tile_locate(k, [&](int i) { return s_rec[i].w; });
      const uint4 inf = s_rec[l];
      const uint32_t wi = ((uint32_t)tile << kTileShift) + (uint32_t)l;
      const uint32_t r = k - inf.w;
      // voxel: largest i with (#vertices of voxels below i) <= r
      int i = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const uint32_t m = below(i + step);
        if ((uint32_t)(__popc(inf.x & m) + __popc(inf.y & m) + __popc(inf.z & m)) <= r) i += step;
      }
      const uint32_t m = below(i);
      int rr = (int)(r - (uint32_t)(__popc(inf.x & m) + __popc(inf.y & m) + __popc(inf.z & m)));
      const int bx = (inf.x >> i) & 1, by = (inf.y >> i) & 1;
      // rr-th crossing edge of the voxel in x, y, z order
      int axis;
      if (bx && rr == 0) axis = 0;
      else { rr -= bx; if (by && rr == 0) axis = 1; else axis = 2; }
      int z, y, w;
      split_word(g, wi, z, y, w);
      const int x = w * 32 + i;
      const int64_t p = ((int64_t)z * g.iny + y) * g.nx + x;
      const int64_t step = axis == 0 ? 1 : (axis == 1 ? g.nx : g.nx * g.ny);
      const float s0 = (float)vol[p], s1 = (float)vol[p + step];
      const float t = __fdiv_rn(__fsub_rn(xf.iso, s0), __fsub_rn(s1, s0));
      float fx = (float)(x + xf.ox), fy = (float)(y + xf.oy), fz = (float)(z + xf.oz);
      if (axis == 0) fx = __fadd_rn(fx, t); else if (axis == 1) fy = __fadd_rn(fy, t); else fz = __fadd_rn(fz, t);
      const float py = __fmul_rn(fy, xf.sy);
      float* o = verts + 3ll * (vbase + k);
      o[0] = __fmul_rn(fx, xf.sx);
      o[1] = xf.flip_y ? -py : py;
      o[2] = __fmul_rn(fz, xf.sz);
    }
  }
}

// Crossing edges of a cell are owned by seven of its corner voxels, which live in FOUR bit rows:
// row (y + oy, z + oz) holds the owners at bit i (ox = 0) and bit i + 1 (ox = 1; bit 0 of the next
// word when i = 31). One record per row resolves all of the row's edges:
//   id(bit b, axis a) = vertex base of the word + #crossings below bit b + #crossings of bit b on axes < a.
// Edge ids (axis*4 + cu + 2*cv as in mc_tables.h) per row:
//   (y, z):     0 (x@i)  4 (y@i)  8 (z@i)  5 (y@i+1)  9 (z@i+1)
//   (y+1, z):   1 (x@i)  10 (z@i)  11 (z@i+1)
//   (y, z+1):   2 (x@i)  6 (y@i)   7 (y@i+1)
//   (y+1, z+1): 3 (x@i)
// All twelve ids go to shared memory ([edge][thread]; the ones of non-crossing edges are never
// read) and every triangle corner is a lookup by edge id.
// the triangle table as the emitter wants it: 16 bytes per case (15 edge ids + the triangle count),
// filled once per process from mc_tables.h (mc_tables_ready)
__device__ uint4 g_tri_packed[256];

struct RowIds { int x0, y0, z0, y1, z1; };   // ids at bit i (x, y, z) and at bit i + 1 (y, z)

template <bool VEC>
__global__ void __launch_bounds__(kTileThreads) k_mc_emit_tris(McGeom g, const uint32_t* __restrict__ bits,
                                                               const uint4* __restrict__ vrec,
                                                               const uint4* __restrict__ tcnt,
                                                               const uint4* __restrict__ toff, int ntiles,
                                                               int flip_y, int skip_last, int vbase,
                                                               const uint4* __restrict__ foreign, int foreign_base,
                                                               int* __restrict__ tris) {
  __shared__ __align__(16) signed char s_tri[256][16];  // 15 edge ids + triangle count
  __shared__ int s_id[12 * kTileThreads];  // [edge][thread]
  __shared__ uint32_t s_act[kTileWords];
  __shared__ uint32_t s_coff[kTileWords];
  __shared__ uint32_t s_w[kTileThreads / 32];
  const int tid = threadIdx.x;
  bool tables = false;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const uint32_t C = __ldg(&tcnt[tile].y);
    if (C == 0u) continue;     // most tiles: nothing but this load
    if (!tables) {             // (made visible by the barriers of the scan below)
      reinterpret_cast<uint4*>(&s_tri[0][0])[tid] = g_tri_packed[tid];   // 16 bytes per case, one load per thread
      tables = true;
    }
    uint32_t tbase = __ldg(&toff[tile].z);
    // active-cell masks of the tile's words and their exclusive offsets
    const uint32_t wi0 = ((uint32_t)tile * kTileThreads + tid) * kWPT;
    {
      Word4 q;
      load_word4<VEC>(bits, g, wi0, q);
      uint32_t act[kWPT], nc = 0;
#pragma unroll
      for (int j = 0; j < kWPT; ++j) {
        act[j] = 0u;
        if (q.ok[j] && q.y[j] + 1 < g.iny && q.z[j] + 1 < g.inz && !word_uniform(q.r[j], g, q.z[j], q.y[j], q.w[j]))
          act[j] = active_cells(q.r[j], valid_x1(g, q.w[j]));
        nc += __popc(act[j]);
      }
      uint32_t tot;
      uint32_t run = block_scan_u32(nc, s_w, &tot);   // barriers inside: s_act / s_coff free
#pragma unroll
      for (int j = 0; j < kWPT; ++j) {
        s_act[tid * kWPT + j] = act[j];
        s_coff[tid * kWPT + j] = run;
        run += __popc(act[j]);
      }
    }
    __syncthreads();
    for (uint32_t k0 = 0; k0 < C; k0 += kTileThreads) {
      const uint32_t k = k0 + tid;
      const bool valid = k < C;
      int i = 0, c = 0, ntri = 0, z = 0, y = 0, w = 0;
      if (valid) {
        const int l = tile_locate(k, [&](int j) { return s_coff[j]; });
        i = nth_set_bit(s_act[l], (int)(k - s_coff[l]));   // this thread's cell bit
        split_word(g, ((uint32_t)tile << kTileShift) + (uint32_t)l, z, y, w);
        const Rows r = load_rows(bits, g, z, y, w);
        c = cell_case(r, i);
        ntri = s_tri[c][15];
      }
      // triangles of the cells before mine: scan over the chunk, running base across chunks
      uint32_t tot;
      const uint32_t tex = block_scan_u32((uint32_t)ntri, s_w, &tot);
      if (valid) {
        const uint32_t ol = (1u << i) - 1u;
        const uint32_t row0 = ((uint32_t)z * (uint32_t)g.iny + (uint32_t)y) * (uint32_t)g.wx + (uint32_t)w;
        // one row: record of word (row, w), ids at bit i and bit i + 1
        auto row_ids = [&](uint32_t ow, bool is_foreign) -> RowIds {
          uint4 oi;
          int v;
          if (is_foreign) {   // owned by the next shard: its records of that plane, its numbering
            oi = __ldg(foreign + (ow - (uint32_t)(g.inz - 1) * (uint32_t)g.iny * (uint32_t)g.wx));
            v = foreign_base;
          } else {
            oi = __ldg(vrec + ow);
            v = vbase + (int)__ldg(&toff[ow >> kTileShift].x);
          }
          RowIds o;
          const int bx = (oi.x >> i) & 1, by = (oi.y >> i) & 1, bz = (oi.z >> i) & 1;
          o.x0 = v + (int)(oi.w + __popc(oi.x & ol) + __popc(oi.y & ol) + __popc(oi.z & ol));
          o.y0 = o.x0 + bx;
          o.z0 = o.y0 + by;
          int n1, bx1;
          if (i < 31) {
            n1 = o.z0 + bz;
            bx1 = (oi.x >> (i + 1)) & 1;
            o.y1 = n1 + bx1;
            o.z1 = o.y1 + (int)((oi.y >> (i + 1)) & 1);
          } else {            // bit 0 of the next word of the row
            uint4 on;
            int vn;
            if (is_foreign) {
              on = __ldg(foreign + (ow + 1u - (uint32_t)(g.inz - 1) * (uint32_t)g.iny * (uint32_t)g.wx));
              vn = foreign_base;
            } else {
              on = __ldg(vrec + ow + 1u);
              vn = vbase + (int)__ldg(&toff[(ow + 1u) >> kTileShift].x);
            }
            n1 = vn + (int)on.w;
            o.y1 = n1 + (int)(on.x & 1u);
            o.z1 = o.y1 + (int)(on.y & 1u);
          }
          return o;
        };
        const bool f0 = skip_last && z == g.inz - 1, f1 = skip_last && z + 1 == g.inz - 1;
        const uint32_t dy = (uint32_t)g.wx, dz = (uint32_t)g.iny * (uint32_t)g.wx;
        const RowIds r00 = row_ids(row0, f0), r01 = row_ids(row0 + dy, f0), r10 = row_ids(row0 + dz, f1),
                     r11 = row_ids(row0 + dz + dy, f1);
        int* sid = s_id + tid;
        sid[0 * kTileThreads] = r00.x0; sid[4 * kTileThreads] = r00.y0; sid[8 * kTileThreads] = r00.z0;
        sid[5 * kTileThreads] = r00.y1; sid[9 * kTileThreads] = r00.z1;
        sid[1 * kTileThreads] = r01.x0; sid[10 * kTileThreads] = r01.z0; sid[11 * kTileThreads] = r01.z1;
        sid[2 * kTileThreads] = r10.x0; sid[6 * kTileThreads] = r10.y0; sid[7 * kTileThreads] = r10.y1;
        sid[3 * kTileThreads] = r11.x0;
        int* o = tris + 3ll * (tbase + tex);
        for (int t = 0; t < ntri; ++t, o += 3) {
          const int i0 = sid[s_tri[c][3 * t] * kTileThreads], i1 = sid[s_tri[c][3 * t + 1] * kTileThreads],
                    i2 = sid[s_tri[c][3 * t + 2] * kTileThreads];
          o[0] = i0;
          o[1] = flip_y ? i2 : i1;
          o[2] = flip_y ? i1 : i2;
        }
      }
      tbase += tot;
    }
    __syncthreads();   // s_act / s_coff are rewritten by the next tile
  }
}

__global__ void k_mc_pack_tables() {
  signed char e[16];
  for (int k = 0; k < 15; ++k) e[k] = B2V_MC_TRI[threadIdx.x][k];
  e[15] = (signed char)B2V_MC_NTRI[threadIdx.x];
  uint4 v;
  memcpy(&v, e, 16);
  g_tri_packed[threadIdx.x] = v;
}

int mc_tables_ready(cudaStream_t s) {
  static int done_for_device[64] = {0};
  int devi = 0;
  B2V_CUDA(cudaGetDevice(&devi));
  if (devi >= 0 && devi < 64 && done_for_device[devi]) return B2V_OK;
  k_mc_pack_tables<<<1, 256, 0, s>>>();
  int rc = b2v_check_launch("k_mc_pack_tables");
  if (rc) return rc;
  if (devi >= 0 && devi < 64) done_for_device[devi] = 1;
  return B2V_OK;
}

// inside(p) <=> (double)S >= iso  <=>  S >= ceil(iso) for integer S
int int_threshold(double iso, int lo, int hi) {
  double c = ceil(iso);
  if (c <= (double)lo) return lo;          // everything inside
  if (c > (double)hi) return hi + 1;       // nothing inside
  return (int)c;
}

}  // namespace

extern "C" int64_t b2v_mc_workspace_bytes(int64_t nz, int64_t ny, int64_t nx) {
  if (nz <= 0 || ny <= 0 || nx <= 0) return 0;
  return carve(nullptr, make_geom(nz, ny, nx)).bytes;
}

static int mc_count_impl(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso, int skip_last,
                         int shard, void* workspace, void* stream, int64_t* nverts_host, int64_t* ntris_host,
                         bool no_sync = false) {
  B2V_REQUIRE(vol && workspace && nverts_host && ntris_host, B2V_ERR_ARG, "mc_count: null pointer");
  B2V_REQUIRE(nz > 0 && ny > 0 && nx > 0, B2V_ERR_ARG, "mc_count: empty volume");
  B2V_REQUIRE(dtype == B2V_U8 || dtype == B2V_I16, B2V_ERR_ARG, "mc_count: dtype must be uint8 or int16");
  B2V_REQUIRE(iso == iso, B2V_ERR_ARG, "mc_count: iso is NaN");
  McGeom g = make_geom(nz, ny, nx);
  B2V_REQUIRE(g.nwords < (1ll << 31), B2V_ERR_ARG, "mc_count: volume too large for one call; shard along z");
  McWs w = carve(workspace, g);
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  B2V_CUDA(cudaMemsetAsync(w.totals, 0, (size_t)w.ctl_bytes, s));
  // inside <=> S >= int_threshold(iso) <=> S in [int_threshold(iso), dtype max]
  if (dtype == B2V_U8)
    rc = pack_bits((const uint8_t*)vol, nz * ny, nx, InRange<int, false>{int_threshold(iso, 0, 255), 255, nullptr, 0},
                   w.bits, nullptr, s);
  else
    rc = pack_bits((const int16_t*)vol, nz * ny, nx,
                   InRange<int, false>{int_threshold(iso, -32768, 32767), 32767, nullptr, 0}, w.bits, nullptr, s);
  if (rc) return rc;
  const int ntiles = (int)ceil_div64(g.nwords, kTileWords);
  if (g.wx % 4 == 0)
    k_mc_classify<true><<<ntiles, kTileThreads, 0, s>>>(w.bits, g, skip_last, w.vrec, w.tcnt, w.toff, w.ticket,
                                                         w.totals, ntiles);
  else
    k_mc_classify<false><<<ntiles, kTileThreads, 0, s>>>(w.bits, g, skip_last, w.vrec, w.tcnt, w.toff, w.ticket,
                                                          w.totals, ntiles);
  if ((rc = b2v_check_launch("k_mc_classify"))) return rc;
  if (shard) {
    k_mc_plane0<<<(unsigned)ceil_div64(g.ny * g.wx, 256), 256, 0, s>>>(w.bits, g, w.vrec, w.tcnt, w.toff, w.plane0);
    if ((rc = b2v_check_launch("k_mc_plane0"))) return rc;
  }
  if (no_sync) return B2V_OK;   // the caller queues the peer exchange behind and reads everything at once
  unsigned long long tot[6] = {0, 0, 0, 0, 0, 0};
  B2V_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(tot[0] < (1ull << 31) && tot[1] < (1ull << 31) && tot[2] < (1ull << 31), B2V_ERR_RANGE,
              "mc_count: %llu vertices / %llu triangles exceed int32 indices; shard along z", tot[0], tot[1]);
  *nverts_host = (int64_t)tot[0];
  *ntris_host = (int64_t)tot[1];
  return B2V_OK;
}

static int mc_emit_impl(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                        const void* workspace, float sx, float sy, float sz, int32_t ox, int32_t oy, int32_t oz,
                        int flip_y, int skip_last, int32_t vbase, const void* foreign, int32_t foreign_base,
                        float* verts, int32_t* tris, void* stream) {
  B2V_REQUIRE(vol && workspace, B2V_ERR_ARG, "mc_emit: null pointer");
  B2V_REQUIRE(dtype == B2V_U8 || dtype == B2V_I16, B2V_ERR_ARG, "mc_emit: dtype must be uint8 or int16");
  B2V_REQUIRE(!skip_last || foreign, B2V_ERR_ARG, "mc_emit: a shard that skips its last plane needs the next shard's records");
  McGeom g = make_geom(nz, ny, nx);
  McWs w = carve(const_cast<void*>(workspace), g);
  cudaStream_t s = (cudaStream_t)stream;
  McXform xf = {sx, sy, sz, ox, oy, oz, flip_y ? 1 : 0, (float)iso};
  const int ntiles = (int)ceil_div64(g.nwords, kTileWords);   // one block per tile; empty tiles leave at once
  int rc;
  if ((rc = mc_tables_ready(s))) return rc;
  if (verts) {
    if (dtype == B2V_U8)
      k_mc_emit_verts<uint8_t><<<ntiles, kTileThreads, 0, s>>>((const uint8_t*)vol, g, w.vrec, w.tcnt, w.toff, ntiles,
                                                               xf, verts);
    else
      k_mc_emit_verts<int16_t><<<ntiles, kTileThreads, 0, s>>>((const int16_t*)vol, g, w.vrec, w.tcnt, w.toff, ntiles,
                                                               xf, verts);
    if ((rc = b2v_check_launch("k_mc_emit_verts"))) return rc;
  }
  if (tris) {
    if (g.wx % 4 == 0)
      k_mc_emit_tris<true><<<ntiles, kTileThreads, 0, s>>>(g, w.bits, w.vrec, w.tcnt, w.toff, ntiles, flip_y ? 1 : 0,
                                                           skip_last, vbase, (const uint4*)foreign, foreign_base, tris);
    else
      k_mc_emit_tris<false><<<ntiles, kTileThreads, 0, s>>>(g, w.bits, w.vrec, w.tcnt, w.toff, ntiles, flip_y ? 1 : 0,
                                                            skip_last, vbase, (const uint4*)foreign, foreign_base, tris);
    if ((rc = b2v_check_launch("k_mc_emit_tris"))) return rc;
  }
  return B2V_OK;
}

// ---- Z shards over peer mailboxes (csrc/peer.cuh) ----------------------------------------------
// After classify: publish this shard's (V, T) into every rank's mailbox, push the dense plane-0
// records into the LOWER neighbour's (it numbers the vertices of the shared plane from them), and
// wait until every rank's counts (and with them the upper neighbour's records) have arrived. One
// small launch replaces an all_gather, a device->host copy and a send/recv pair.
__global__ void __launch_bounds__(1024) k_mc_peer_exchange(PeerSet ps, const unsigned long long* __restrict__ totals,
                                                           const uint4* __restrict__ plane0, int nrec, int* ok_dev) {
  const int tid = threadIdx.x, par = (int)(ps.epoch & 1u);
  if (ps.rank > 0) {
    uint4* dst = ps.of(ps.rank - 1).mc_from_hi(par);
    for (int i = tid; i < nrec; i += blockDim.x) dst[i] = plane0[i];
  }
  __threadfence_system();
  __syncthreads();
  bool ok = true;
  if (tid < ps.world) {
    PeerBox box = ps.of(tid);
    st_relaxed_sys_s64(box.counts(par) + 2 * ps.rank, (long long)totals[0]);
    st_relaxed_sys_s64(box.counts(par) + 2 * ps.rank + 1, (long long)totals[1]);
    __threadfence_system();
    st_release_sys(box.cnt_tag(par) + ps.rank, ps.epoch);
    ok = peer_wait_eq(ps.mine().cnt_tag(par) + tid, ps.epoch, ps.timeout);
  }
  ok = __syncthreads_and(ok);
  if (tid == 0) *ok_dev = ok ? 1 : 0;
}

extern "C" int64_t b2v_peer_mc_inbox_offset(int64_t plane_bytes, uint32_t epoch) {
  return kPbData + 4 * plane_bytes + (int64_t)(epoch & 1u) * 4 * plane_bytes;
}

extern "C" int b2v_mc_count_shard_peer(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                                       int skip_last_plane, void* workspace, void* stream, int rank, int world,
                                       const void* const* mailboxes_host, int64_t mailbox_plane_bytes, uint32_t epoch,
                                       int64_t* counts_host /*[world][2]: (V, T) of every rank*/) {
  B2V_REQUIRE(counts_host && epoch >= 1, B2V_ERR_ARG, "mc_count_shard_peer: bad arguments");
  PeerSet ps;
  int rc = peer_make_set(rank, world, mailboxes_host, mailbox_plane_bytes, epoch, &ps);
  if (rc) return rc;
  McGeom g = make_geom(nz, ny, nx);
  B2V_REQUIRE(g.ny * g.wx * 16 <= 4 * ps.pc, B2V_ERR_ARG, "mc_count_shard_peer: plane records do not fit the mailbox");
  int64_t nv = 0, nt = 0;
  if ((rc = mc_count_impl(vol, dtype, nz, ny, nx, iso, skip_last_plane ? 1 : 0, 1, workspace, stream, &nv, &nt, true)))
    return rc;
  McWs w = carve(workspace, g);
  cudaStream_t s = (cudaStream_t)stream;
  int* ok_dev = (int*)(w.totals + 8);
  k_mc_peer_exchange<<<1, 1024, 0, s>>>(ps, w.totals, w.plane0, (int)(g.ny * g.wx), ok_dev);
  if ((rc = b2v_check_launch("k_mc_peer_exchange"))) return rc;
  int ok = 0;
  unsigned long long tot[6] = {0, 0, 0, 0, 0, 0};
  B2V_CUDA(cudaMemcpyAsync(counts_host, ps.mine().counts((int)(epoch & 1u)), (size_t)world * 16, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(&ok, ok_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(ok == 1, B2V_ERR_NOCONV, "mc_count_shard_peer: a rank did not publish its counts in time (epoch %u)", epoch);
  B2V_REQUIRE(tot[0] < (1ull << 31) && tot[1] < (1ull << 31) && tot[2] < (1ull << 31), B2V_ERR_RANGE,
              "mc_count: %llu vertices / %llu triangles exceed int32 indices; shard along z", tot[0], tot[1]);
  return B2V_OK;
}

extern "C" int b2v_mc_count(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                            void* workspace, void* stream, int64_t* nverts_host, int64_t* ntris_host) {
  return mc_count_impl(vol, dtype, nz, ny, nx, iso, 0, 0, workspace, stream, nverts_host, ntris_host);
}

extern "C" int b2v_mc_emit(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                           const void* workspace, float sx, float sy, float sz, int32_t ox, int32_t oy, int32_t oz,
                           int flip_y, float* verts, int32_t* tris, void* stream) {
  return mc_emit_impl(vol, dtype, nz, ny, nx, iso, workspace, sx, sy, sz, ox, oy, oz, flip_y, 0, 0, nullptr, 0, verts,
                      tris, stream);
}

// ---- Z-sharded variants (dist.py): the slab passed in ends with the plane it shares with
// the next shard; that plane's vertices belong to the next shard (skip_last_plane).
extern "C" int b2v_mc_count_shard(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                                  int skip_last_plane, void* workspace, void* stream, int64_t* nverts_host,
                                  int64_t* ntris_host) {
  return mc_count_impl(vol, dtype, nz, ny, nx, iso, skip_last_plane ? 1 : 0, 1, workspace, stream, nverts_host,
                       ntris_host);
}

extern "C" int b2v_mc_emit_shard(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                                 const void* workspace, float sx, float sy, float sz, int32_t ox, int32_t oy,
                                 int32_t oz, int flip_y, int skip_last_plane, int32_t vertex_base,
                                 const void* next_shard_plane0_records, int32_t next_shard_vertex_base, float* verts,
                                 int32_t* tris, void* stream) {
  return mc_emit_impl(vol, dtype, nz, ny, nx, iso, workspace, sx, sy, sz, ox, oy, oz, flip_y, skip_last_plane ? 1 : 0,
                      vertex_base, next_shard_plane0_records, next_shard_vertex_base, verts, tris, stream);
}

extern "C" int b2v_mc_layout(int64_t nz, int64_t ny, int64_t nx, int64_t* layout_out) {
  B2V_REQUIRE(nz > 0 && ny > 0 && nx > 0 && layout_out, B2V_ERR_ARG, "mc_layout: bad arguments");
  McGeom g = make_geom(nz, ny, nx);
  McWs w = carve(nullptr, g);
  layout_out[0] = (int64_t)((char*)w.plane0 - (char*)nullptr);   // byte offset of the dense plane-0 records
  layout_out[1] = (int64_t)ny * g.wx * 16;                        // their size in bytes
  layout_out[2] = (int64_t)((char*)w.totals - (char*)nullptr);   // uint64 totals: [0] V, [1] T (device)
  return B2V_OK;
}
