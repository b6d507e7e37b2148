// Marker-based watershed, 6-connected: the persistent engine behind b2v_ws_flood (do_watershed,
// invesalius/data/watershed_process.py:19-60; cost models and labelling rule: watershed.cu).
//
// Same two phases as the generic kernels of watershed.cu (exact minimax cost field, then labels
// along cost-optimal edges with the label-set that marks order-dependent voxels), but
//   * ONE cooperative launch per phase: the active tiles of a round are a compact list (a tile
//     is appended the first time a neighbour posts it: bitmap + list, three sets rotate), the
//     blocks stride over the list, one grid barrier per round, no host round trip;
//   * inside a 16^3 tile the relaxation is a set of six DIRECTIONAL SWEEPS (+x, -x, +y, -y,
//     +z, -z), each a serial chain in the registers of one thread per row / column:
//     c[j] = min(c[j], max(c[j-1], w(j-1, j))) carries a value across the whole tile in one
//     pass where a Jacobi iteration moves it by one voxel (2-3 sweep sets instead of 30-50
//     iterations);
//   * phase 2 reads a per-voxel ADMISSIBILITY byte (which of the six neighbours is a
//     cost-optimal predecessor: fixed once the costs are final) instead of re-deriving it from
//     costs and intensities in every relaxation.
// Z-sharded volumes (dist.watershed): the slab's halo planes are FROZEN (never relaxed locally,
// only overwritten by the neighbour shard's values through b2v_ws_plane); a frozen plane that
// improves re-activates the tiles next to it.
#include <cooperative_groups.h>
#include <stdlib.h>

#include "b2v_common.cuh"
#include "watershed.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kT = 16;                 // tile edge
constexpr int kH = kT + 2;             // with halo
constexpr int kP = kH + 1;             // padded row pitch (words): conflict-free column walks
constexpr int kCells = kH * kH * kP;   // 6156
constexpr int kThreads = 256;
constexpr int kMaxSets = 8;            // sweep sets per visit before the tile re-queues itself
constexpr uint32_t kInfC = 0xffffffffu;
constexpr unsigned long long kInfK = ~0ull;
// label SET of a voxel (watershed.cu): uint32, code = label + 32768 for one label, kSetEmpty = nothing
// yet (the code of label 0, which no marker carries), kSetMulti = two different labels. Every int16
// label is a legal code, so "two labels" lives above the 16-bit code range (DESIGN.md section 6).
constexpr uint32_t kSetEmpty = 32768, kSetMulti = 0x10000;
// phase-2 key: hops above the label. 64 bits hold any label (uint16 code) and any hop count; when
// the markers carry at most 256 distinct labels the key is hops << 8 | rank of the label (32 bits):
// half the chain instructions, shared memory and traffic. kKeyFull32: keys at or above it mean the
// hop count is about to overflow (the caller falls back to 64-bit keys).
template <typename K> struct KeyT;
template <> struct KeyT<unsigned long long> {
  static constexpr unsigned long long inf = ~0ull, hop = 1ull << 32;
};
template <> struct KeyT<uint32_t> {
  static constexpr uint32_t inf = 0xffffffffu, hop = 1u << 8;
};
constexpr uint32_t kKeyFull32 = 0xff000000u;
enum { F_ZLO = 1, F_ZHI = 2, F_YLO = 4, F_YHI = 8, F_XLO = 16, F_XHI = 32 };
// admissibility bits: predecessor at x-1, x+1, y-1, y+1, z-1, z+1
enum { A_XM = 1, A_XP = 2, A_YM = 4, A_YP = 8, A_ZM = 16, A_ZP = 32 };

struct FGrid {
  int nz, ny, nx;
  int ntz, nty, ntx, ntiles;
  long long n;
  int fz0, fz1;      // planes [fz0, fz1) are relaxed; the others are frozen halo planes
  int mode;          // 0: flat-array neighbourhood of scipy.ndimage.watershed_ift; 1: proper bounds
  int vec;           // rows of full tiles are 16-byte aligned in every array (nx % 16 == 0, aligned bases)
};

struct Lists {
  uint32_t* bm;   // [3][nbw] tile bitmaps
  int* list;      // [3][ntiles]
  int* cnt;       // [3] + [3] spare; cnt[4] = error, cnt[5] = rounds, cnt[6] = plane-merge changed flag,
                  // cnt[8 + (r & 1)] = a 32-bit key of round r reached kKeyFull32
  int nbw;
};

struct FastWs {
  uint32_t* cost;
  unsigned long long* key;
  uint32_t* lset;
  uint8_t* adm;
  uint32_t* key32;      // phase-2 keys when the markers carry <= 256 distinct labels
  uint32_t* present;    // [2048] which label codes occur among the markers (bitmap over uint16)
  uint32_t* prefix;     // [2048] label codes below each bitmap word
  uint32_t* inv;        // [256] rank -> label code; inv[256] = number of distinct labels
  Lists L;
  int* init_list;   // marker tiles (both phases start from them)
  int* init_cnt;
  char* lists_begin;
  int64_t lists_bytes;
  int64_t bytes;
};

FGrid make_fgrid(int64_t nz, int64_t ny, int64_t nx, int mode, int frozen_lo, int frozen_hi) {
  FGrid g;
  g.nz = (int)nz; g.ny = (int)ny; g.nx = (int)nx;
  g.ntz = (int)ceil_div64(nz, kT); g.nty = (int)ceil_div64(ny, kT); g.ntx = (int)ceil_div64(nx, kT);
  g.ntiles = g.ntz * g.nty * g.ntx;
  g.n = (long long)nz * ny * nx;
  g.fz0 = frozen_lo ? 1 : 0;
  g.fz1 = frozen_hi ? (int)nz - 1 : (int)nz;
  g.mode = mode;
  g.vec = (nx % 16 == 0) ? 1 : 0;
  return g;
}

FastWs fcarve(void* base, int64_t nz, int64_t ny, int64_t nx) {
  FastWs w;
  const int64_t n = nz * ny * nx;
  const int64_t nt = ceil_div64(nz, kT) * ceil_div64(ny, kT) * ceil_div64(nx, kT);
  const int64_t nbw = (nt + 31) / 32;
  char* p = (char*)base;
  int64_t off = 0;
  w.key = (unsigned long long*)(p + off); off += align256(n * 8);
  w.cost = (uint32_t*)(p + off); off += align256(n * 4);
  w.lset = (uint32_t*)(p + off); off += align256(n * 4);
  w.adm = (uint8_t*)(p + off); off += align256(n);
  w.key32 = (uint32_t*)(p + off); off += align256(n * 4);
  w.present = (uint32_t*)(p + off); off += 2048 * 4;
  w.prefix = (uint32_t*)(p + off); off += 2048 * 4;
  w.inv = (uint32_t*)(p + off); off += align256(257 * 4);
  w.init_list = (int*)(p + off); off += align256(nt * 4);
  w.init_cnt = (int*)(p + off); off += 256;
  w.lists_begin = p + off;
  w.L.bm = (uint32_t*)(p + off); off += align256(3 * nbw * 4);
  w.L.cnt = (int*)(p + off); off += 256;
  w.lists_bytes = (p + off) - w.lists_begin;
  w.L.list = (int*)(p + off); off += align256(3 * nt * 4);
  w.L.nbw = (int)nbw;
  w.bytes = off;
  return w;
}

__device__ __forceinline__ void post_tile(const Lists& L, int ntiles, int set, int tile) {
  const uint32_t bit = 1u << (tile & 31);
  const uint32_t old = atomicOr(&L.bm[(size_t)set * L.nbw + (tile >> 5)], bit);
  if (!(old & bit)) L.list[(size_t)set * ntiles + atomicAdd(&L.cnt[set], 1)] = tile;
}

// flat index of (z, y, x), coordinates possibly one step outside the volume; -1 if the voxel does
// not exist. mode 0: SciPy walks the volume as a flat array, a neighbour is flat index + offset if
// that lies in [0, N): the last voxel of a row touches the first of the next row, a plane's last
// row the next plane's first (verified against SciPy 1.18.1, tools/probe_scipy_ift.py).
__device__ __forceinline__ long long flat_or_invalid(const FGrid& g, int z, int y, int x) {
  if (g.mode == 0) {
    const long long p = ((long long)z * g.ny + y) * g.nx + x;
    return (p >= 0 && p < g.n) ? p : -1;
  }
  return (z >= 0 && z < g.nz && y >= 0 && y < g.ny && x >= 0 && x < g.nx) ? ((long long)z * g.ny + y) * g.nx + x : -1;
}

// ---- init -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_wsf_init(const uint16_t* __restrict__ img, const int16_t* __restrict__ markers,
                                                  FGrid g, uint32_t* __restrict__ cost,
                                                  unsigned long long* __restrict__ key, uint32_t* __restrict__ lset,
                                                  Lists L, int* init_list, int* init_cnt, uint32_t* present) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += stride) {
    const int m = markers[i];
    if (m != 0) {
      const uint32_t code = (uint32_t)(m + 32768);
      if (!((present[code >> 5] >> (code & 31)) & 1u)) atomicOr(&present[code >> 5], 1u << (code & 31));
      cost[i] = g.mode == 0 ? 0u : (uint32_t)img[i];
      key[i] = (unsigned long long)(uint32_t)(m + 32768);
      lset[i] = code;
      const int x = (int)(i % g.nx);
      const long long r = i / g.nx;
      const int y = (int)(r % g.ny), z = (int)(r / g.ny);
      const int tile = ((z / kT) * g.nty + (y / kT)) * g.ntx + (x / kT);
      const uint32_t bit = 1u << (tile & 31);
      const uint32_t old = atomicOr(&L.bm[tile >> 5], bit);     // set 0
      if (!(old & bit)) {
        L.list[atomicAdd(&L.cnt[0], 1)] = tile;
        init_list[atomicAdd(init_cnt, 1)] = tile;
      }
    } else {
      cost[i] = kInfC;
      key[i] = kInfK;
      lset[i] = kSetEmpty;
    }
  }
}

// marker tiles -> set 0 (start of phase 2; the sets were cleared by the host)
__global__ void k_wsf_seed_lists(Lists L, const int* __restrict__ init_list, const int* __restrict__ init_cnt) {
  const int n = *init_cnt;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int tile = init_list[i];
    atomicOr(&L.bm[tile >> 5], 1u << (tile & 31));
    L.list[i] = tile;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) L.cnt[0] = n;
}

// ---- label ranks (32-bit keys) ------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_wsf_ranks(const uint32_t* __restrict__ present, uint32_t* prefix, uint32_t* inv) {
  __shared__ uint32_t s_w[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t w0 = present[2 * tid], w1 = present[2 * tid + 1];
  const uint32_t c = __popc(w0) + __popc(w1);
  uint32_t incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_w[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t v = s_w[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    s_w[lane] = v;
  }
  __syncthreads();
  const uint32_t before = (warp ? s_w[warp - 1] : 0u) + incl - c;
  prefix[2 * tid] = before;
  prefix[2 * tid + 1] = before + __popc(w0);
  uint32_t r = before;
  for (uint32_t m = w0; m; m &= m - 1, ++r) if (r < 256) inv[r] = (uint32_t)(2 * tid) * 32 + (uint32_t)(__ffs(m) - 1);
  for (uint32_t m = w1; m; m &= m - 1, ++r) if (r < 256) inv[r] = (uint32_t)(2 * tid + 1) * 32 + (uint32_t)(__ffs(m) - 1);
  if (tid == 1023) inv[256] = s_w[31];
}

__global__ void __launch_bounds__(256) k_wsf_key32_init(const unsigned long long* __restrict__ key, long long n,
                                                        const uint32_t* __restrict__ present,
                                                        const uint32_t* __restrict__ prefix, uint32_t* __restrict__ key32) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long k = key[i];
    uint32_t v = 0xffffffffu;
    if (k != kInfK && (k >> 32) == 0) {     // a marker: rank of its label code
      const uint32_t code = (uint32_t)k;
      v = prefix[code >> 5] + __popc(present[code >> 5] & ((1u << (code & 31)) - 1u));
    }
    key32[i] = v;
  }
}

__global__ void __launch_bounds__(256) k_wsf_labels32(const uint32_t* __restrict__ key32, const uint32_t* __restrict__ lset,
                                                      const uint32_t* __restrict__ inv, long long n,
                                                      int16_t* __restrict__ labels, uint8_t* __restrict__ ambiguous) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t k = key32[i];
    labels[i] = k == 0xffffffffu ? (int16_t)0 : (int16_t)((int)inv[k & 0xffu] - 32768);
    if (ambiguous) ambiguous[i] = lset[i] == kSetMulti ? 1 : 0;
  }
}

// ---- admissible predecessors (phase 2 input) -------------------------------------------------------
// mode 0: v -> p is cost-optimal iff max(C(v), |I(v) - I(p)|) == C(p); mode 1 (labels given at push
// time): p inherits from the neighbours flooded first, i.e. those with the smallest cost among
// ALL its neighbours. Markers and unreached voxels admit nobody; frozen planes are not relaxed.
__global__ void __launch_bounds__(256) k_wsf_adm(const uint16_t* __restrict__ img, const uint32_t* __restrict__ cost,
                                                 const unsigned long long* __restrict__ key, FGrid g,
                                                 uint8_t* __restrict__ adm) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < g.n; i += stride) {
    const int x = (int)(i % g.nx);
    const long long r = i / g.nx;
    const int y = (int)(r % g.ny), z = (int)(r / g.ny);
    const uint32_t c = cost[i];
    uint32_t a = 0;
    if (c != kInfC && (key[i] >> 32) != 0 && z >= g.fz0 && z < g.fz1) {
      const int ip = img[i];
      const int dz[6] = {0, 0, 0, 0, -1, 1}, dy[6] = {0, 0, -1, 1, 0, 0}, dx[6] = {-1, 1, 0, 0, 0, 0};
      uint32_t cv[6];
      uint32_t cmin = kInfC;
#pragma unroll
      for (int d = 0; d < 6; ++d) {
        const long long q = flat_or_invalid(g, z + dz[d], y + dy[d], x + dx[d]);
        cv[d] = kInfC;
        if (q >= 0) {
          const uint32_t cq = cost[q];
          if (g.mode == 0) {
            if (cq != kInfC) {
              const uint32_t w = (uint32_t)abs((int)img[q] - ip);
              cv[d] = cq > w ? cq : w;    // cost of reaching p through q
            }
          } else {
            cv[d] = cq;
          }
        }
        cmin = cv[d] < cmin ? cv[d] : cmin;
      }
      const uint32_t want = g.mode == 0 ? c : cmin;
#pragma unroll
      for (int d = 0; d < 6; ++d)
        if (cv[d] != kInfC && cv[d] == want) a |= 1u << d;
    }
    adm[i] = (uint8_t)a;
  }
}

// ---- tile visits ---------------------------------------------------------------------------------
// diagnostics: [0..2] phase 1 visits / sweep sets / visits that changed, [4..6] the same for phase 2,
// [3] visits that re-queued their own tile (not settled within kMaxSets sweep sets, either phase),
// [7] phase-2 runs on 32-bit keys stopped for the 64-bit re-run
__device__ int g_stats[8];

struct TileGeom {
  int tz, ty, tx, z0, y0, x0;
  int vz, vy, vx;      // valid own cells per axis
  int uz0, uz1;        // own planes hz in [uz0, uz1) are relaxed (1-based like hz)
};

__device__ __forceinline__ TileGeom tile_geom(const FGrid& g, int tile) {
  TileGeom t;
  t.tx = tile % g.ntx; t.ty = (tile / g.ntx) % g.nty; t.tz = tile / (g.ntx * g.nty);
  t.z0 = t.tz * kT; t.y0 = t.ty * kT; t.x0 = t.tx * kT;
  t.vz = min(kT, g.nz - t.z0); t.vy = min(kT, g.ny - t.y0); t.vx = min(kT, g.nx - t.x0);
  t.uz0 = max(g.fz0 - t.z0, 0) + 1;
  t.uz1 = min(g.fz1 - t.z0, t.vz) + 1;
  return t;
}

__device__ __forceinline__ int cell_index(int hz, int hy, int hx) { return (hz * kH + hy) * kP + hx; }

// the neighbours a tile has to wake when cells on its faces changed (faces: F_* bits); mode 0 adds
// the tiles that hold the flat-array neighbours across the x / y borders of the volume
__device__ __forceinline__ void post_neighbours(const FGrid& g, const Lists& L, int nxt, const TileGeom& t, int faces) {
  const int tid = threadIdx.x;
  if (tid < 6) {
    const int f = 1 << tid;
    if (faces & f) {
      int nz = t.tz, ny = t.ty, nx = t.tx;
      if (f == F_ZLO) --nz; else if (f == F_ZHI) ++nz; else if (f == F_YLO) --ny; else if (f == F_YHI) ++ny;
      else if (f == F_XLO) --nx; else ++nx;
      if (nz >= 0 && nz < g.ntz && ny >= 0 && ny < g.nty && nx >= 0 && nx < g.ntx)
        post_tile(L, g.ntiles, nxt, (nz * g.nty + ny) * g.ntx + nx);
    }
  } else if (g.mode == 0 && tid < 10) {
    // wrapped neighbours: (z, y, nx-1) <-> (z, y+1, 0) [(z+1, 0, 0) after the last row];
    //                     (z, ny-1, x) <-> (z+1, 0, x)
    if (tid == 6 && (faces & F_XHI) && t.tx == g.ntx - 1) {
      // rows y0+1 .. y0+vy of the same planes, or row 0 of planes z+1 (tiles tz and tz+1) after the last row
      post_tile(L, g.ntiles, nxt, (t.tz * g.nty + t.ty) * g.ntx + 0);
      if (t.ty + 1 < g.nty) post_tile(L, g.ntiles, nxt, (t.tz * g.nty + t.ty + 1) * g.ntx + 0);
      else {
        post_tile(L, g.ntiles, nxt, (t.tz * g.nty + 0) * g.ntx + 0);
        if (t.tz + 1 < g.ntz) post_tile(L, g.ntiles, nxt, ((t.tz + 1) * g.nty + 0) * g.ntx + 0);
      }
    }
    if (tid == 7 && (faces & F_XLO) && t.tx == 0) {
      const int lx = g.ntx - 1;
      post_tile(L, g.ntiles, nxt, (t.tz * g.nty + t.ty) * g.ntx + lx);
      if (t.ty > 0) post_tile(L, g.ntiles, nxt, (t.tz * g.nty + t.ty - 1) * g.ntx + lx);
      else {
        post_tile(L, g.ntiles, nxt, (t.tz * g.nty + g.nty - 1) * g.ntx + lx);
        if (t.tz > 0) post_tile(L, g.ntiles, nxt, ((t.tz - 1) * g.nty + g.nty - 1) * g.ntx + lx);
      }
    }
    if (tid == 8 && (faces & F_YHI) && t.ty == g.nty - 1) {
      post_tile(L, g.ntiles, nxt, (t.tz * g.nty + 0) * g.ntx + t.tx);
      if (t.tz + 1 < g.ntz) post_tile(L, g.ntiles, nxt, ((t.tz + 1) * g.nty + 0) * g.ntx + t.tx);
    }
    if (tid == 9 && (faces & F_YLO) && t.ty == 0) {
      post_tile(L, g.ntiles, nxt, (t.tz * g.nty + g.nty - 1) * g.ntx + t.tx);
      if (t.tz > 0) post_tile(L, g.ntiles, nxt, ((t.tz - 1) * g.nty + g.nty - 1) * g.ntx + t.tx);
    }
  }
}

// faces touched by a change in the line of a sweep thread
__device__ __forceinline__ int line_faces(int axis, int a, int b, bool any, bool first, bool last, const TileGeom& t) {
  // axis 0: line along x at (hy = a + 1, hz = b + 1); axis 1: along y at (hx = a + 1, hz = b + 1);
  // axis 2: along z at (hx = a + 1, hy = b + 1). first / last: the cell at the line's low / high end
  // of the TILE changed (for z lines the ends of the relaxed range count only if they are the tile's).
  if (!any) return 0;
  int f = 0;
  if (axis == 0) {
    if (first) f |= F_XLO; if (last) f |= F_XHI;
    if (a == 0) f |= F_YLO; if (a == t.vy - 1) f |= F_YHI;
    if (b == 0) f |= F_ZLO; if (b == t.vz - 1) f |= F_ZHI;
  } else if (axis == 1) {
    if (first) f |= F_YLO; if (last) f |= F_YHI;
    if (a == 0) f |= F_XLO; if (a == t.vx - 1) f |= F_XHI;
    if (b == 0) f |= F_ZLO; if (b == t.vz - 1) f |= F_ZHI;
  } else {
    if (first) f |= F_ZLO; if (last) f |= F_ZHI;
    if (a == 0) f |= F_XLO; if (a == t.vx - 1) f |= F_XHI;
    if (b == 0) f |= F_YLO; if (b == t.vy - 1) f |= F_YHI;
  }
  return f;
}

// ---- full tiles (16^3 relaxed cells, aligned rows): vector loads, register chains -------------------
__device__ __forceinline__ bool tile_full(const FGrid& g, const TileGeom& t) {
  return g.vec && t.vx == kT && t.vy == kT && t.vz == kT && t.uz0 == 1 && t.uz1 == kT + 1;
}

// one line of 16 cells + its two ends in registers; forward and backward pass; changed cells stored
template <int MODE, int S>
__device__ __forceinline__ void line_full_cost(uint32_t* sC, const uint16_t* sI, int base, bool& ch, bool& first,
                                               bool& last) {
  uint32_t c[kT + 2], n[kT + 2];
  int iv[kT + 2];
#pragma unroll
  for (int j = 0; j < kT + 2; ++j) { c[j] = sC[base + (j - 1) * S]; iv[j] = sI[base + (j - 1) * S]; n[j] = c[j]; }
#pragma unroll
  for (int j = 1; j <= kT; ++j) {
    const uint32_t w = MODE == 0 ? (uint32_t)abs(iv[j] - iv[j - 1]) : (uint32_t)iv[j];
    const uint32_t cand = n[j - 1] > w ? n[j - 1] : w;
    n[j] = cand < n[j] ? cand : n[j];
  }
#pragma unroll
  for (int j = kT; j >= 1; --j) {
    const uint32_t w = MODE == 0 ? (uint32_t)abs(iv[j] - iv[j + 1]) : (uint32_t)iv[j];
    const uint32_t cand = n[j + 1] > w ? n[j + 1] : w;
    n[j] = cand < n[j] ? cand : n[j];
  }
#pragma unroll
  for (int j = 1; j <= kT; ++j)
    if (n[j] != c[j]) { sC[base + (j - 1) * S] = n[j]; ch = true; }
  first = n[1] != c[1];
  last = n[kT] != c[kT];
}

__device__ __forceinline__ uint32_t set_join(uint32_t a, uint32_t b) {   // b != empty
  return a == kSetEmpty ? b : (a == b ? a : kSetMulti);
}

template <typename K, bool WITH_SET, int S>
__device__ __forceinline__ void line_full_label(K* sK, uint32_t* sA, const uint8_t* sD, int base,
                                                uint32_t from_lo, uint32_t from_hi, bool& ch, bool& first, bool& last) {
  K k[kT + 2];
  uint32_t av[kT + 2], d[kT + 2];
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < kT + 2; ++j) {
    k[j] = sK[base + (j - 1) * S];
    av[j] = WITH_SET ? sA[base + (j - 1) * S] : kSetEmpty;
    d[j] = (j >= 1 && j <= kT) ? sD[base + (j - 1) * S] : 0u;
  }
  // branch-free steps (selects): the lanes of a warp walk different lines
#pragma unroll
  for (int j = 1; j <= kT; ++j) {
    const bool ok = (d[j] & from_lo) != 0u && k[j - 1] != KeyT<K>::inf;
    const K cand = k[j - 1] + KeyT<K>::hop;
    const bool better = ok && cand < k[j];
    k[j] = better ? cand : k[j];
    uint32_t ch1 = better ? 1u : 0u;
    if (WITH_SET) {
      const uint32_t j1 = set_join(av[j], av[j - 1]);
      const bool grow = ok && av[j - 1] != kSetEmpty && j1 != av[j];
      av[j] = grow ? j1 : av[j];
      ch1 |= grow ? 1u : 0u;
    }
    m |= ch1 << j;
  }
#pragma unroll
  for (int j = kT; j >= 1; --j) {
    const bool ok = (d[j] & from_hi) != 0u && k[j + 1] != KeyT<K>::inf;
    const K cand = k[j + 1] + KeyT<K>::hop;
    const bool better = ok && cand < k[j];
    k[j] = better ? cand : k[j];
    uint32_t ch1 = better ? 1u : 0u;
    if (WITH_SET) {
      const uint32_t j1 = set_join(av[j], av[j + 1]);
      const bool grow = ok && av[j + 1] != kSetEmpty && j1 != av[j];
      av[j] = grow ? j1 : av[j];
      ch1 |= grow ? 1u : 0u;
    }
    m |= ch1 << j;
  }
#pragma unroll
  for (int j = 1; j <= kT; ++j)
    if ((m >> j) & 1u) {
      sK[base + (j - 1) * S] = k[j];
      if (WITH_SET) sA[base + (j - 1) * S] = av[j];
    }
  ch = m != 0;
  first = (m >> 1) & 1u;
  last = (m >> kT) & 1u;
}

// the six halo cells of a thread in a full tile: index 0/1 x ends of row (y = a, z = b), 2/3 y ends
// of column (x = a, z = b), 4/5 z ends of column (x = a, y = b). Returns flat index (or -1) and the
// shared-memory cell.
__device__ __forceinline__ long long halo_cell(const FGrid& g, const TileGeom& t, int which, int a, int b, int* ci) {
  int hz, hy, hx;
  switch (which) {
    case 0: hz = b + 1; hy = a + 1; hx = 0; break;
    case 1: hz = b + 1; hy = a + 1; hx = kT + 1; break;
    case 2: hz = b + 1; hy = 0; hx = a + 1; break;
    case 3: hz = b + 1; hy = kT + 1; hx = a + 1; break;
    case 4: hz = 0; hy = b + 1; hx = a + 1; break;
    default: hz = kT + 1; hy = b + 1; hx = a + 1; break;
  }
  *ci = cell_index(hz, hy, hx);
  return flat_or_invalid(g, t.z0 + hz - 1, t.y0 + hy - 1, t.x0 + hx - 1);
}

// PHASE 1: one tile visit. Returns (block-uniform) 0 nothing changed, 1 changed, 2 changed and not
// converged within kMaxSets sweep sets. *faces_out: faces whose cells changed.
template <int MODE>
__device__ int visit_cost(const uint16_t* __restrict__ img, uint32_t* cost, const FGrid& g, const TileGeom& t,
                          uint32_t* sC, uint16_t* sI, int* s_faces) {
  const int tid = threadIdx.x;
  if (tid == 0) *s_faces = 0;
  const bool full = tile_full(g, t);
  if (full) {
    const int a = tid & 15, b = tid >> 4;
    const long long p0 = ((long long)(t.z0 + b) * g.ny + (t.y0 + a)) * g.nx + t.x0;
    uint4 c4[4], i4[2];
#pragma unroll
    for (int k = 0; k < 4; ++k) c4[k] = __ldcg((const uint4*)(cost + p0) + k);
#pragma unroll
    for (int k = 0; k < 2; ++k) i4[k] = __ldg((const uint4*)(img + p0) + k);
    long long hp[6];
    int hc[6];
    uint32_t hcost[6];
    uint16_t himg[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      hp[k] = halo_cell(g, t, k, a, b, &hc[k]);
      hcost[k] = kInfC; himg[k] = 0;
      if (hp[k] >= 0) { hcost[k] = __ldcg(&cost[hp[k]]); himg[k] = img[hp[k]]; }
    }
    const int r0 = cell_index(b + 1, a + 1, 1);
    const uint32_t cc[16] = {c4[0].x, c4[0].y, c4[0].z, c4[0].w, c4[1].x, c4[1].y, c4[1].z, c4[1].w,
                             c4[2].x, c4[2].y, c4[2].z, c4[2].w, c4[3].x, c4[3].y, c4[3].z, c4[3].w};
    const uint32_t ii[8] = {i4[0].x, i4[0].y, i4[0].z, i4[0].w, i4[1].x, i4[1].y, i4[1].z, i4[1].w};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      sC[r0 + k] = cc[k];
      sI[r0 + k] = (uint16_t)((k & 1) ? (ii[k >> 1] >> 16) : (ii[k >> 1] & 0xffffu));
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) { sC[hc[k]] = hcost[k]; sI[hc[k]] = himg[k]; }
  } else {
// load the tile with its six halo faces (edges / corners of the halo are not needed)
    for (int i = tid; i < kH * kH * kH; i += kThreads) {
      const int hx = i % kH, hy = (i / kH) % kH, hz = i / (kH * kH);
      if (hz > t.vz + 1 || hy > t.vy + 1 || hx > t.vx + 1) continue;
      const int nh = (hz == 0 || hz == t.vz + 1) + (hy == 0 || hy == t.vy + 1) + (hx == 0 || hx == t.vx + 1);
      if (nh > 1) continue;
      const long long p = flat_or_invalid(g, t.z0 + hz - 1, t.y0 + hy - 1, t.x0 + hx - 1);
      uint32_t c = kInfC;
      uint16_t v = 0;
      if (p >= 0) { c = __ldcg(&cost[p]); v = img[p]; }
      const int ci = cell_index(hz, hy, hx);
      sC[ci] = c;
      sI[ci] = v;
    }
  }
  __syncthreads();
  const int a = tid & 15, b = tid >> 4;
  int faces = 0, any = 0, changed, sets = 0;
  // a directional pass over one line: cells base + j * s, j in [0, len); the value before the first
  // cell is at base - s (forward) / after the last at base + len * s (backward)
  auto line = [&](int base, int s, int len, bool& ch, bool& first, bool& last) {
    {
      uint32_t cp = sC[base - s];
      int ip = sI[base - s];
      for (int j = 0; j < len; ++j) {
        const int idx = base + j * s;
        uint32_t c = sC[idx];
        const int iv = sI[idx];
        const uint32_t w = MODE == 0 ? (uint32_t)abs(iv - ip) : (uint32_t)iv;
        const uint32_t cand = cp > w ? cp : w;
        if (cand < c) { c = cand; sC[idx] = c; ch = true; first |= j == 0; last |= j == len - 1; }
        cp = c; ip = iv;
      }
    }
    {
      uint32_t cp = sC[base + len * s];
      int ip = sI[base + len * s];
      for (int j = len - 1; j >= 0; --j) {
        const int idx = base + j * s;
        uint32_t c = sC[idx];
        const int iv = sI[idx];
        const uint32_t w = MODE == 0 ? (uint32_t)abs(iv - ip) : (uint32_t)iv;
        const uint32_t cand = cp > w ? cp : w;
        if (cand < c) { c = cand; sC[idx] = c; ch = true; first |= j == 0; last |= j == len - 1; }
        cp = c; ip = iv;
      }
    }
  };
  if (full) {
    // passes x, y, z, x, ... until three in a row (one per axis) change nothing
    int clean = 0, pass = 0;
    changed = 0;
    while (clean < 3 && pass < 3 * kMaxSets) {
      bool ch = false, first = false, last = false;
      const int axis = pass % 3;
      if (axis == 0) line_full_cost<MODE, 1>(sC, sI, cell_index(b + 1, a + 1, 1), ch, first, last);
      else if (axis == 1) line_full_cost<MODE, kP>(sC, sI, cell_index(b + 1, 1, a + 1), ch, first, last);
      else line_full_cost<MODE, kH * kP>(sC, sI, cell_index(1, b + 1, a + 1), ch, first, last);
      if (ch) faces |= line_faces(axis, a, b, true, first, last, t);
      changed = __syncthreads_or(ch ? 1 : 0);
      any |= changed;
      clean = changed ? 0 : clean + 1;
      ++pass;
    }
    sets = (pass + 2) / 3;
    changed = clean < 3;   // pass cap hit before three clean passes: the tile re-queues itself
  } else {
  do {
    changed = 0;
    // x lines: (hy = a + 1, hz = b + 1)
    if (a < t.vy && b + 1 >= t.uz0 && b + 1 < t.uz1) {
      bool ch = false, first = false, last = false;
      line(cell_index(b + 1, a + 1, 1), 1, t.vx, ch, first, last);
      if (ch) { changed = 1; faces |= line_faces(0, a, b, true, first, last, t); }
    }
    __syncthreads();
    // y lines: (hx = a + 1, hz = b + 1)
    if (a < t.vx && b + 1 >= t.uz0 && b + 1 < t.uz1) {
      bool ch = false, first = false, last = false;
      line(cell_index(b + 1, 1, a + 1), kP, t.vy, ch, first, last);
      if (ch) { changed = 1; faces |= line_faces(1, a, b, true, first, last, t); }
    }
    __syncthreads();
    // z lines: (hx = a + 1, hy = b + 1), relaxed planes only
    if (a < t.vx && b < t.vy) {
      bool ch = false, first = false, last = false;
      line(cell_index(t.uz0, b + 1, a + 1), kH * kP, t.uz1 - t.uz0, ch, first, last);
      if (ch) { changed = 1; faces |= line_faces(2, a, b, true, first && t.uz0 == 1, last && t.uz1 == t.vz + 1, t); }
    }
    changed = __syncthreads_or(changed);
    any |= changed;
    ++sets;
  } while (changed && sets < kMaxSets);
  }
  if (tid == 0) { atomicAdd(&g_stats[0], 1); atomicAdd(&g_stats[1], sets); if (any) atomicAdd(&g_stats[2], 1); }
  if (!any) return 0;
  // write the relaxed planes back (whole rows: the cells that did not change keep their value)
  if (full) {
    const long long p0 = ((long long)(t.z0 + b) * g.ny + (t.y0 + a)) * g.nx + t.x0;
    const int c0 = cell_index(b + 1, a + 1, 1);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      __stcg((uint4*)(cost + p0) + k, make_uint4(sC[c0 + 4 * k], sC[c0 + 4 * k + 1], sC[c0 + 4 * k + 2], sC[c0 + 4 * k + 3]));
  } else if (a < t.vy && b + 1 >= t.uz0 && b + 1 < t.uz1) {
    const long long p0 = ((long long)(t.z0 + b) * g.ny + (t.y0 + a)) * g.nx + t.x0;
    const int c0 = cell_index(b + 1, a + 1, 1);
    for (int x = 0; x < t.vx; ++x) __stcg(&cost[p0 + x], sC[c0 + x]);
  }
  if (faces) atomicOr(s_faces, faces);
  __syncthreads();
  return changed ? 2 : 1;
}

// PHASE 2: keys (hops << 32 | label) and label sets along admissible edges
template <typename K, bool WITH_SET>
__device__ int visit_label(const uint8_t* __restrict__ adm, K* key, uint32_t* lset, const FGrid& g,
                           const TileGeom& t, K* sK, uint32_t* sA, uint8_t* sD, int* s_faces, int* err) {
  constexpr bool K64 = sizeof(K) == 8;
  constexpr int KV = K64 ? 8 : 4;     // 128-bit vectors per row of 16 keys
  const int tid = threadIdx.x;
  if (tid == 0) *s_faces = 0;
  const bool full = tile_full(g, t);
  if (full) {
    const int a = tid & 15, b = tid >> 4;
    const long long p0 = ((long long)(t.z0 + b) * g.ny + (t.y0 + a)) * g.nx + t.x0;
    uint4 k4[KV], a4[4], d4;
#pragma unroll
    for (int k = 0; k < KV; ++k) k4[k] = __ldcg((const uint4*)(key + p0) + k);
    if (WITH_SET) {
#pragma unroll
      for (int k = 0; k < 4; ++k) a4[k] = __ldcg((const uint4*)(lset + p0) + k);
    }
    d4 = __ldg((const uint4*)(adm + p0));
    long long hp[6];
    int hc[6];
    K hk[6];
    uint32_t hs[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      hp[k] = halo_cell(g, t, k, a, b, &hc[k]);
      hk[k] = KeyT<K>::inf; hs[k] = kSetEmpty;
      if (hp[k] >= 0) { hk[k] = __ldcg(&key[hp[k]]); if (WITH_SET) hs[k] = __ldcg(&lset[hp[k]]); }
    }
    const int r0 = cell_index(b + 1, a + 1, 1);
    const uint32_t aa[16] = {a4[0].x, a4[0].y, a4[0].z, a4[0].w, a4[1].x, a4[1].y, a4[1].z, a4[1].w,
                             a4[2].x, a4[2].y, a4[2].z, a4[2].w, a4[3].x, a4[3].y, a4[3].z, a4[3].w};
    const uint32_t dd[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      if constexpr (K64) {
        const uint4 q = k4[k >> 1];
        sK[r0 + k] = (k & 1) ? (((unsigned long long)q.w << 32) | q.z) : (((unsigned long long)q.y << 32) | q.x);
      } else {
        const uint4 q = k4[k >> 2];
        sK[r0 + k] = (k & 3) == 0 ? q.x : ((k & 3) == 1 ? q.y : ((k & 3) == 2 ? q.z : q.w));
      }
      if (WITH_SET) sA[r0 + k] = aa[k];
      sD[r0 + k] = (uint8_t)((dd[k >> 2] >> (8 * (k & 3))) & 0xffu);
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) { sK[hc[k]] = hk[k]; if (WITH_SET) sA[hc[k]] = hs[k]; sD[hc[k]] = 0; }
  } else {
for (int i = tid; i < kH * kH * kH; i += kThreads) {
      const int hx = i % kH, hy = (i / kH) % kH, hz = i / (kH * kH);
      if (hz > t.vz + 1 || hy > t.vy + 1 || hx > t.vx + 1) continue;
      const int nh = (hz == 0 || hz == t.vz + 1) + (hy == 0 || hy == t.vy + 1) + (hx == 0 || hx == t.vx + 1);
      if (nh > 1) continue;
      const long long p = flat_or_invalid(g, t.z0 + hz - 1, t.y0 + hy - 1, t.x0 + hx - 1);
      K k = KeyT<K>::inf;
      uint32_t s = kSetEmpty;
      uint8_t d = 0;
      if (p >= 0) {
        k = __ldcg(&key[p]);
        if (WITH_SET) s = __ldcg(&lset[p]);
        if (nh == 0) d = adm[p];
      }
      const int ci = cell_index(hz, hy, hx);
      sK[ci] = k;
      if (WITH_SET) sA[ci] = s;
      sD[ci] = d;
    }
  }
  __syncthreads();
  const int a = tid & 15, b = tid >> 4;
  int faces = 0, any = 0, changed, sets = 0;
  auto line = [&](int base, int s, int len, uint32_t from_lo, uint32_t from_hi, bool& ch, bool& first, bool& last) {
    {
      K kp = sK[base - s];
      uint32_t ap = WITH_SET ? sA[base - s] : kSetEmpty;
      for (int j = 0; j < len; ++j) {
        const int idx = base + j * s;
        K k = sK[idx];
        uint32_t av = WITH_SET ? sA[idx] : kSetEmpty;
        if ((sD[idx] & from_lo) && kp != KeyT<K>::inf) {
          bool c = false;
          const K cand = kp + KeyT<K>::hop;
          if (cand < k) { k = cand; sK[idx] = k; c = true; }
          if (WITH_SET && ap != kSetEmpty) {
            const uint32_t j1 = set_join(av, ap);
            if (j1 != av) { av = j1; sA[idx] = av; c = true; }
          }
          if (c) { ch = true; first |= j == 0; last |= j == len - 1; }
        }
        kp = k; ap = av;
      }
    }
    {
      K kp = sK[base + len * s];
      uint32_t ap = WITH_SET ? sA[base + len * s] : kSetEmpty;
      for (int j = len - 1; j >= 0; --j) {
        const int idx = base + j * s;
        K k = sK[idx];
        uint32_t av = WITH_SET ? sA[idx] : kSetEmpty;
        if ((sD[idx] & from_hi) && kp != KeyT<K>::inf) {
          bool c = false;
          const K cand = kp + KeyT<K>::hop;
          if (cand < k) { k = cand; sK[idx] = k; c = true; }
          if (WITH_SET && ap != kSetEmpty) {
            const uint32_t j1 = set_join(av, ap);
            if (j1 != av) { av = j1; sA[idx] = av; c = true; }
          }
          if (c) { ch = true; first |= j == 0; last |= j == len - 1; }
        }
        kp = k; ap = av;
      }
    }
  };
  if (full) {
    int clean = 0, pass = 0;
    changed = 0;
    while (clean < 3 && pass < 3 * kMaxSets) {
      bool ch = false, first = false, last = false;
      const int axis = pass % 3;
      if (axis == 0) line_full_label<K, WITH_SET, 1>(sK, sA, sD, cell_index(b + 1, a + 1, 1), A_XM, A_XP, ch, first, last);
      else if (axis == 1) line_full_label<K, WITH_SET, kP>(sK, sA, sD, cell_index(b + 1, 1, a + 1), A_YM, A_YP, ch, first, last);
      else line_full_label<K, WITH_SET, kH * kP>(sK, sA, sD, cell_index(1, b + 1, a + 1), A_ZM, A_ZP, ch, first, last);
      if (ch) faces |= line_faces(axis, a, b, true, first, last, t);
      changed = __syncthreads_or(ch ? 1 : 0);
      any |= changed;
      clean = changed ? 0 : clean + 1;
      ++pass;
    }
    sets = (pass + 2) / 3;
    changed = clean < 3;   // pass cap hit before three clean passes: the tile re-queues itself
  } else
  do {
    changed = 0;
    if (a < t.vy && b + 1 >= t.uz0 && b + 1 < t.uz1) {
      bool ch = false, first = false, last = false;
      line(cell_index(b + 1, a + 1, 1), 1, t.vx, A_XM, A_XP, ch, first, last);
      if (ch) { changed = 1; faces |= line_faces(0, a, b, true, first, last, t); }
    }
    __syncthreads();
    if (a < t.vx && b + 1 >= t.uz0 && b + 1 < t.uz1) {
      bool ch = false, first = false, last = false;
      line(cell_index(b + 1, 1, a + 1), kP, t.vy, A_YM, A_YP, ch, first, last);
      if (ch) { changed = 1; faces |= line_faces(1, a, b, true, first, last, t); }
    }
    __syncthreads();
    if (a < t.vx && b < t.vy) {
      bool ch = false, first = false, last = false;
      line(cell_index(t.uz0, b + 1, a + 1), kH * kP, t.uz1 - t.uz0, A_ZM, A_ZP, ch, first, last);
      if (ch) { changed = 1; faces |= line_faces(2, a, b, true, first && t.uz0 == 1, last && t.uz1 == t.vz + 1, t); }
    }
    changed = __syncthreads_or(changed);
    any |= changed;
    ++sets;
  } while (changed && sets < kMaxSets);
  if (tid == 0) { atomicAdd(&g_stats[4], 1); atomicAdd(&g_stats[5], sets); if (any) atomicAdd(&g_stats[6], 1); }
  if (!any) return 0;
  if (full) {
    const long long p0 = ((long long)(t.z0 + b) * g.ny + (t.y0 + a)) * g.nx + t.x0;
    const int c0 = cell_index(b + 1, a + 1, 1);
    if constexpr (K64) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const unsigned long long k0 = sK[c0 + 2 * k], k1 = sK[c0 + 2 * k + 1];
        __stcg((uint4*)(key + p0) + k, make_uint4((uint32_t)k0, (uint32_t)(k0 >> 32), (uint32_t)k1, (uint32_t)(k1 >> 32)));
      }
    } else {
      bool full32 = false;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint4 q = make_uint4(sK[c0 + 4 * k], sK[c0 + 4 * k + 1], sK[c0 + 4 * k + 2], sK[c0 + 4 * k + 3]);
        full32 |= (q.x != KeyT<K>::inf && q.x >= kKeyFull32) || (q.y != KeyT<K>::inf && q.y >= kKeyFull32) ||
                  (q.z != KeyT<K>::inf && q.z >= kKeyFull32) || (q.w != KeyT<K>::inf && q.w >= kKeyFull32);
        __stcg((uint4*)(key + p0) + k, q);
      }
      if (full32) *err = 2;     // hop count about to overflow 24 bits: the host re-runs phase 2 with 64-bit keys
    }
    if (WITH_SET) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        __stcg((uint4*)(lset + p0) + k, make_uint4(sA[c0 + 4 * k], sA[c0 + 4 * k + 1], sA[c0 + 4 * k + 2], sA[c0 + 4 * k + 3]));
    }
  } else if (a < t.vy && b + 1 >= t.uz0 && b + 1 < t.uz1) {
    const long long p0 = ((long long)(t.z0 + b) * g.ny + (t.y0 + a)) * g.nx + t.x0;
    const int c0 = cell_index(b + 1, a + 1, 1);
    for (int x = 0; x < t.vx; ++x) {
      if (!K64 && sK[c0 + x] != KeyT<K>::inf && sK[c0 + x] >= (K)kKeyFull32) *err = 2;
      __stcg(&key[p0 + x], sK[c0 + x]);
      if (WITH_SET) __stcg(&lset[p0 + x], sA[c0 + x]);
    }
  }
  if (faces) atomicOr(s_faces, faces);
  __syncthreads();
  return changed ? 2 : 1;
}

// ---- the persistent kernels ---------------------------------------------------------------------
// PHASE 1 (cost) / PHASE 2 (labels). Rounds until the list of a round is empty. L.cnt[4] error,
// L.cnt[5] rounds.
template <int PHASE, int MODE, bool WITH_SET, typename K>
__global__ void __launch_bounds__(kThreads, (PHASE == 1 || !WITH_SET || sizeof(K) == 4) ? 3 : 2)
    k_wsf_persistent(const uint16_t* __restrict__ img, uint32_t* cost, K* key, uint32_t* lset,
                     const uint8_t* __restrict__ adm, FGrid g, Lists L, int max_rounds) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ unsigned long long s_raw[];
  __shared__ int s_faces;
  // phase 1: cost u32 + intensity u16; phase 2: key (u64 or u32) + set u32 + admissibility u8
  uint32_t* sC = (uint32_t*)s_raw;
  uint16_t* sI = (uint16_t*)(sC + kCells);
  K* sK = (K*)s_raw;
  uint32_t* sA = (uint32_t*)(sK + kCells);
  uint8_t* sD = WITH_SET ? (uint8_t*)(sA + kCells) : (uint8_t*)(sK + kCells);
  const int tid = threadIdx.x;
  int r = 0;
  for (;; ++r) {
    const int cur = r % 3, nxt = (r + 1) % 3, old = (r + 2) % 3;
    // 32-bit keys: a hop count that reached kKeyFull32 in the last round ends the phase at this
    // barrier (the host re-runs it on 64-bit keys; relaxing on would wrap keys modulo 2^32). The
    // flag of round r lives in cnt[8 + (r & 1)]: written during round r only, read by every block
    // between the barriers of rounds r and r + 1, so all blocks take the same decision.
    if (sizeof(K) == 4 && r > 0 && __ldcg(&L.cnt[8 + ((r - 1) & 1)]) != 0) {
      if (blockIdx.x == 0 && tid == 0) { L.cnt[4] = 2; atomicAdd(&g_stats[7], 1); }
      break;
    }
    const int n = __ldcg(&L.cnt[cur]);
    if (n == 0) break;
    if (r >= max_rounds) { if (blockIdx.x == 0 && tid == 0) L.cnt[4] = 1; break; }
    // `old` was read by everyone before the last barrier and is posted to from the next round on
    for (int i = blockIdx.x * kThreads + tid; i < L.nbw; i += gridDim.x * kThreads) L.bm[(size_t)old * L.nbw + i] = 0;
    if (blockIdx.x == 0 && tid == 0) L.cnt[old] = 0;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
      const int tile = __ldcg(&L.list[(size_t)cur * g.ntiles + i]);
      const TileGeom t = tile_geom(g, tile);
      if (t.uz0 >= t.uz1) continue;
      int res;
      if (PHASE == 1) res = visit_cost<MODE>(img, cost, g, t, sC, sI, &s_faces);
      else res = visit_label<K, WITH_SET>(adm, key, lset, g, t, sK, sA, sD, &s_faces, &L.cnt[8 + (r & 1)]);
      if (res) {
        __threadfence();
        post_neighbours(g, L, nxt, t, s_faces);
        if (res == 2 && tid == 32) { post_tile(L, g.ntiles, nxt, tile); atomicAdd(&g_stats[3], 1); }
      }
      __syncthreads();   // the shared tile is reused by the next visit
    }
    grid.sync();
  }
  if (blockIdx.x == 0 && tid == 0) L.cnt[5] = r;
}

__global__ void __launch_bounds__(256) k_wsf_labels(const unsigned long long* __restrict__ key,
                                                    const uint32_t* __restrict__ lset, long long n,
                                                    int16_t* __restrict__ labels, uint8_t* __restrict__ ambiguous) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long k = key[i];
    labels[i] = k == kInfK ? (int16_t)0 : (int16_t)((int)(uint32_t)(k & 0xffffffffu) - 32768);
    if (ambiguous) ambiguous[i] = lset[i] == kSetMulti ? 1 : 0;
  }
}

// ---- frozen planes (Z shards): read a plane / merge a neighbour's plane --------------------------
// what = 0: cost (uint32 per voxel); what = 1: key (uint64) followed by the label sets (uint16)
__global__ void __launch_bounds__(256) k_wsf_plane_get(const uint32_t* __restrict__ cost,
                                                       const unsigned long long* __restrict__ key,
                                                       const uint32_t* __restrict__ lset, FGrid g, int z, int what,
                                                       void* out) {
  const int pn = g.ny * g.nx;
  const long long base = (long long)z * pn;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pn; i += gridDim.x * blockDim.x) {
    if (what == 0) ((uint32_t*)out)[i] = cost[base + i];
    else {
      ((unsigned long long*)out)[i] = key[base + i];
      ((uint32_t*)((unsigned long long*)out + pn))[i] = lset[base + i];
    }
  }
}

__global__ void __launch_bounds__(256) k_wsf_plane_merge(uint32_t* cost, unsigned long long* key, uint32_t* lset,
                                                         FGrid g, int z, int what, const void* in, Lists L) {
  const int pn = g.ny * g.nx;
  const long long base = (long long)z * pn;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pn; i += gridDim.x * blockDim.x) {
    bool ch = false;
    if (what == 0) {
      const uint32_t v = ((const uint32_t*)in)[i];
      if (v < cost[base + i]) { cost[base + i] = v; ch = true; }
    } else {
      const unsigned long long k = ((const unsigned long long*)in)[i];
      const uint32_t s = ((const uint32_t*)((const unsigned long long*)in + pn))[i];
      if (k < key[base + i]) { key[base + i] = k; ch = true; }
      if (s != kSetEmpty) {
        const uint32_t j = set_join(lset[base + i], s);
        if (j != lset[base + i]) { lset[base + i] = j; ch = true; }
      }
    }
    if (ch) {
      const int y = i / g.nx, x = i - y * g.nx;
      // the tiles whose relaxed cells touch this voxel: its own tile and the ones above / below
      for (int dz = -1; dz <= 1; ++dz) {
        const int zz = z + dz;
        if (zz < 0 || zz >= g.nz) continue;
        post_tile(L, g.ntiles, 0, ((zz / kT) * g.nty + y / kT) * g.ntx + x / kT);
      }
      L.cnt[6] = 1;
    }
  }
}

template <typename K>
int launch_persistent(K kern, size_t smem, const uint16_t* img, FastWs& w, FGrid g, cudaStream_t s, void* keyptr = nullptr) {
  B2V_CUDA(cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  B2V_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)kern, kThreads, smem));
  B2V_REQUIRE(per_sm >= 1, B2V_ERR_CUDA, "watershed: persistent kernel does not fit on an SM");
  int grid = per_sm * b2v_sm_count();
  if (grid > g.ntiles) grid = g.ntiles;
  uint32_t* cost = w.cost;
  void* key = keyptr ? keyptr : (void*)w.key;
  uint32_t* lset = w.lset;
  const uint8_t* adm = w.adm;
  Lists L = w.L;
  int max_rounds = 1 << 20;
  void* args[] = {&img, &cost, &key, &lset, &adm, &g, &L, &max_rounds};
  B2V_CUDA(cudaLaunchCooperativeKernel((const void*)kern, dim3(grid), dim3(kThreads), args, smem, s));
  return b2v_check_launch("k_wsf_persistent");
}

int read_ctl(FastWs& w, cudaStream_t s, int* rounds, int* changed, int* key_overflow = nullptr) {
  int ctl[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  B2V_CUDA(cudaMemcpyAsync(ctl, w.L.cnt, sizeof(ctl), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  if (key_overflow) *key_overflow = ctl[4] == 2;
  B2V_REQUIRE(ctl[4] == 0 || (ctl[4] == 2 && key_overflow), B2V_ERR_NOCONV, "watershed: no convergence within the round cap");
  if (rounds) *rounds += ctl[5];
  if (changed) *changed = ctl[6];
  return B2V_OK;
}

}  // namespace

int64_t b2v_wsf_workspace_bytes(int64_t nz, int64_t ny, int64_t nx) { return fcarve(nullptr, nz, ny, nx).bytes; }

// stages (bit mask), in this order:
//    1 INIT            costs / keys from the markers, marker tiles -> phase-1 list
//    2 COST_CONVERGE   phase-1 rounds from the current list (after INIT or after plane merges)
//    4 LABEL_BEGIN     admissibility bytes, marker tiles -> phase-2 list
//    8 LABEL_CONVERGE  phase-2 rounds from the current list
//   16 FINISH          labels (and the ambiguous mask) out
int b2v_wsf_run(int stages, const uint16_t* img, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx, int mode,
                int frozen_lo, int frozen_hi, int16_t* labels, uint8_t* ambiguous, int with_set, void* workspace,
                void* stream, int* rounds_io, int allow_key32) {
  B2V_REQUIRE(img && workspace, B2V_ERR_ARG, "ws_flood: null pointer");
  B2V_REQUIRE(nz > 0 && ny > 0 && nx > 0 && nz * ny * nx < (1ll << 40), B2V_ERR_ARG, "ws_flood: bad volume shape");
  B2V_REQUIRE(mode == 0 || mode == 1, B2V_ERR_ARG, "ws_flood: mode must be 0 (IFT) or 1 (value flood)");
  B2V_REQUIRE(nz - (frozen_lo ? 1 : 0) - (frozen_hi ? 1 : 0) >= 1, B2V_ERR_ARG, "ws_flood: slab has no plane of its own");
  cudaStream_t s = (cudaStream_t)stream;
  FGrid g = make_fgrid(nz, ny, nx, mode, frozen_lo, frozen_hi);
  if (((uintptr_t)img & 15u) || ((uintptr_t)workspace & 15u)) g.vec = 0;
  FastWs w = fcarve(workspace, nz, ny, nx);
  int rc;
  if (stages & 1) {
    B2V_REQUIRE(markers, B2V_ERR_ARG, "ws_flood: null markers");
    B2V_CUDA(cudaMemsetAsync(w.init_cnt, 0, 256 + (size_t)w.lists_bytes, s));
    B2V_CUDA(cudaMemsetAsync(w.present, 0, 2048 * 4, s));
    k_wsf_init<<<b2v_grid(g.n, 256 * 4, 16), 256, 0, s>>>(img, markers, g, w.cost, w.key, w.lset, w.L, w.init_list,
                                                          w.init_cnt, w.present);
    if ((rc = b2v_check_launch("k_wsf_init"))) return rc;
    k_wsf_ranks<<<1, 1024, 0, s>>>(w.present, w.prefix, w.inv);
    if ((rc = b2v_check_launch("k_wsf_ranks"))) return rc;
  }
  // 32-bit keys: one-shot runs only (the staged / sharded protocol exchanges 64-bit keys), markers
  // with at most 256 distinct labels
  bool use32 = false;
  if (allow_key32 && stages == 31 && !getenv("B2V_WS_KEY64")) {
    uint32_t nlab = 0;
    B2V_CUDA(cudaMemcpyAsync(&nlab, w.inv + 256, 4, cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    use32 = nlab <= 256;
  }
  if (stages & 2) {
    const size_t smem = (size_t)kCells * 6;
    rc = mode == 0 ? launch_persistent(k_wsf_persistent<1, 0, false, unsigned long long>, smem, img, w, g, s)
                   : launch_persistent(k_wsf_persistent<1, 1, false, unsigned long long>, smem, img, w, g, s);
    if (rc) return rc;
    if ((rc = read_ctl(w, s, rounds_io, nullptr))) return rc;
    B2V_CUDA(cudaMemsetAsync(w.lists_begin, 0, (size_t)w.lists_bytes, s));
  }
  if (stages & 4) {
    B2V_CUDA(cudaMemsetAsync(w.lists_begin, 0, (size_t)w.lists_bytes, s));
    k_wsf_adm<<<b2v_grid(g.n, 256 * 4, 16), 256, 0, s>>>(img, w.cost, w.key, g, w.adm);
    if ((rc = b2v_check_launch("k_wsf_adm"))) return rc;
    k_wsf_seed_lists<<<8, 256, 0, s>>>(w.L, w.init_list, w.init_cnt);
    if ((rc = b2v_check_launch("k_wsf_seed_lists"))) return rc;
  }
  if ((stages & 8) && use32) {
    k_wsf_key32_init<<<b2v_grid(g.n, 256 * 4, 16), 256, 0, s>>>(w.key, g.n, w.present, w.prefix, w.key32);
    if ((rc = b2v_check_launch("k_wsf_key32_init"))) return rc;
    const size_t smem = (size_t)kCells * (with_set ? 9 : 5) + 16;
    rc = with_set ? launch_persistent(k_wsf_persistent<2, 0, true, uint32_t>, smem, img, w, g, s, w.key32)
                  : launch_persistent(k_wsf_persistent<2, 0, false, uint32_t>, smem, img, w, g, s, w.key32);
    if (rc) return rc;
    int overflow = 0;
    if ((rc = read_ctl(w, s, rounds_io, nullptr, &overflow))) return rc;
    B2V_CUDA(cudaMemsetAsync(w.lists_begin, 0, (size_t)w.lists_bytes, s));
    if (overflow) {      // more than 2^24 hops: start phase 2 again with 64-bit keys (the sets only grow)
      use32 = false;
      k_wsf_seed_lists<<<8, 256, 0, s>>>(w.L, w.init_list, w.init_cnt);
      if ((rc = b2v_check_launch("k_wsf_seed_lists"))) return rc;
    }
  }
  if ((stages & 8) && !use32) {
    const size_t smem = (size_t)kCells * (with_set ? 13 : 9) + 16;
    rc = with_set ? launch_persistent(k_wsf_persistent<2, 0, true, unsigned long long>, smem, img, w, g, s)
                  : launch_persistent(k_wsf_persistent<2, 0, false, unsigned long long>, smem, img, w, g, s);
    if (rc) return rc;
    if ((rc = read_ctl(w, s, rounds_io, nullptr))) return rc;
    B2V_CUDA(cudaMemsetAsync(w.lists_begin, 0, (size_t)w.lists_bytes, s));
  }
  if (stages & 16) {
    B2V_REQUIRE(labels, B2V_ERR_ARG, "ws_flood: null labels");
    B2V_REQUIRE(!ambiguous || with_set, B2V_ERR_ARG, "ws_flood: the ambiguous mask needs the label sets");
    if (use32) k_wsf_labels32<<<b2v_grid(g.n, 256 * 4, 16), 256, 0, s>>>(w.key32, w.lset, w.inv, g.n, labels,
                                                                         ambiguous);
    else k_wsf_labels<<<b2v_grid(g.n, 256 * 4, 16), 256, 0, s>>>(w.key, w.lset, g.n, labels, ambiguous);
    if ((rc = b2v_check_launch("k_wsf_labels"))) return rc;
  }
  return B2V_OK;
}

extern "C" int b2v_ws_flood_staged(int stages, const uint16_t* img, const int16_t* markers, int64_t nz, int64_t ny,
                                   int64_t nx, int mode, int frozen_lo, int frozen_hi, int16_t* labels,
                                   uint8_t* ambiguous, void* workspace, void* stream, int* rounds_io) {
  return b2v_wsf_run(stages, img, markers, nz, ny, nx, mode, frozen_lo, frozen_hi, labels, ambiguous, 1, workspace,
                     stream, rounds_io, 0);
}

extern "C" int b2v_ws_stats(int* out8, int reset) {
  if (out8) B2V_CUDA(cudaMemcpyFromSymbol(out8, g_stats, sizeof(int) * 8));
  if (reset) { int z[8] = {0, 0, 0, 0, 0, 0, 0, 0}; B2V_CUDA(cudaMemcpyToSymbol(g_stats, z, sizeof(z))); }
  return B2V_OK;
}

extern "C" int64_t b2v_ws_plane_bytes(int64_t ny, int64_t nx, int what) {
  return what == 0 ? ny * nx * 4 : ny * nx * 12;
}

extern "C" int b2v_ws_plane(int merge, int what, int64_t nz, int64_t ny, int64_t nx, int mode, int frozen_lo,
                            int frozen_hi, int64_t z, void* plane, void* workspace, void* stream, int* changed_host) {
  B2V_REQUIRE(plane && workspace && z >= 0 && z < nz && (what == 0 || what == 1), B2V_ERR_ARG, "ws_plane: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  FGrid g = make_fgrid(nz, ny, nx, mode, frozen_lo, frozen_hi);
  FastWs w = fcarve(workspace, nz, ny, nx);
  const int grid = (int)ceil_div64(ny * nx, 256 * 4);
  if (!merge) {
    k_wsf_plane_get<<<grid, 256, 0, s>>>(w.cost, w.key, w.lset, g, (int)z, what, plane);
    return b2v_check_launch("k_wsf_plane_get");
  }
  B2V_CUDA(cudaMemsetAsync(w.L.cnt + 6, 0, sizeof(int), s));
  k_wsf_plane_merge<<<grid, 256, 0, s>>>(w.cost, w.key, w.lset, g, (int)z, what, plane, w.L);
  int rc;
  if ((rc = b2v_check_launch("k_wsf_plane_merge"))) return rc;
  if (changed_host) {
    int ch = 0;
    B2V_CUDA(cudaMemcpyAsync(&ch, w.L.cnt + 6, sizeof(int), cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    *changed_host = ch;
  }
  return B2V_OK;
}
