// Marker-based watershed: do_watershed, invesalius/data/watershed_process.py:19-60.
//   b2v_ws_lut_i16            get_LUT_value(image, ww, wl).astype(uint16)      imagedata_utils.py:555-564
//   b2v_ws_shift_i16          (image - image.min()).astype(uint16)             watershed_process.py:50,55
//   b2v_ws_morph_gradient_u16 ndimage.morphological_gradient(pre, size)       watershed_process.py:36,49
//   b2v_ws_flood              the flood itself, two cost models:
//        mode 0 "IFT"   (scipy.ndimage.watershed_ift): path cost = max |I(a) - I(b)| over its edges
//        mode 1 "value" (skimage.segmentation.watershed): path cost = max I over its voxels
//
// Both reference floods are sequential priority-queue walks whose tie-breaking is an artefact
// of queue order (LIFO buckets in SciPy, (value, age) heap in skimage). What is order
// independent is the minimax COST of every voxel; we compute it exactly, then label:
//   phase 1  C(p) = min over markers and paths of the path cost (Bellman-Ford on (min, max),
//            tiles of 16^3 voxels relaxed to local convergence in shared memory, neighbour
//            tiles re-activated round by round, as in floodfill.cu);
//   phase 2  labels spread from the markers along cost-optimal edges only
//            (max(C(v), w(v,p)) == C(p)); where several labels reach a voxel the one with
//            fewer hops wins, then the smaller label (shortest path on key = hops<<32 | label,
//            same tiled relaxation).
// Wherever the reference's result does not depend on its queue order (no cost ties between
// different labels) this is exactly the reference's labelling; on plateaus it is a
// deterministic geodesic split instead of the reference's order artefact (see DESIGN.md §6).
#include <stdlib.h>

#include "b2v_common.cuh"
#include "watershed.cuh"

namespace {

// ---- pre-processing ---------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ws_lut(const int16_t* __restrict__ img, int64_t n, double window,
                                                double level, uint16_t* __restrict__ out) {
  const double lo = level - 0.5 - (window - 1.0) / 2.0;
  const double hi = level - 0.5 + (window - 1.0) / 2.0;
  const double c = level - 0.5;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v = (double)img[i];
    int16_t r;
    if (v <= lo) r = 0;
    else if (v > hi) r = (int16_t)(long long)window;                 // np.piecewise keeps int16
    else r = (int16_t)(long long)(((v - c) / (window - 1.0) + 0.5) * window);  // C cast: truncation
    out[i] = (uint16_t)r;
  }
}

__global__ void __launch_bounds__(256) k_ws_shift(const int16_t* __restrict__ img, int64_t n,
                                                  const float* __restrict__ minmax, uint16_t* __restrict__ out) {
  const int mn = (int)minmax[0];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = (uint16_t)(int16_t)((int)img[i] - mn);  // int16 arithmetic wraps like NumPy's
}

__device__ __forceinline__ int64_t reflect(int64_t i, int64_t n) {
  // scipy mode='reflect': (d c b a | a b c d | d c b a)
  if (n == 1) return 0;
  const int64_t period = 2 * n;
  i %= period;
  if (i < 0) i += period;
  return i < n ? i : period - 1 - i;
}

// dilation window [i - s/2 + e, i + (s-1-s/2) + e] with e = 1 for even s (grey_dilation
// mirrors the footprint and shifts the origin), erosion window [i - s/2, i + (s-1-s/2)].
__global__ void __launch_bounds__(256) k_ws_morph_gradient(const uint16_t* __restrict__ in, int64_t nz, int64_t ny,
                                                           int64_t nx, int sz, int sy, int sx,
                                                           uint16_t* __restrict__ out) {
  const int64_t n = nz * ny * nx;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int ez = (sz & 1) ? 0 : 1, ey = (sy & 1) ? 0 : 1, ex = (sx & 1) ? 0 : 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    int64_t x = i % nx, r = i / nx, y = r % ny, z = r / ny;
    int mn = 65535, mx = 0, dmx = 0;
    for (int kz = 0; kz < sz + ez; ++kz) {
      int64_t zz = reflect(z - sz / 2 + kz, nz);
      for (int ky = 0; ky < sy + ey; ++ky) {
        int64_t yy = reflect(y - sy / 2 + ky, ny);
        for (int kx = 0; kx < sx + ex; ++kx) {
          int64_t xx = reflect(x - sx / 2 + kx, nx);
          int v = in[(zz * ny + yy) * nx + xx];
          bool in_ero = kz < sz && ky < sy && kx < sx;
          bool in_dil = kz >= ez && ky >= ey && kx >= ex;
          if (in_ero) mn = min(mn, v);
          if (in_dil) dmx = max(dmx, v);
        }
      }
    }
    mx = dmx;
    out[i] = (uint16_t)(mx - mn);
  }
}

// Same result, far fewer loads: a thread owns one (y, x) column and marches along z. Per plane it
// reduces the 2-D window (sy x sx values, neighbours' loads hit L1) to the plane's erosion minimum
// and dilation maximum, keeps the last W plane results in registers and combines them: sy * sx
// loads per voxel instead of sz * sy * sx, no 64-bit division per voxel. W = window length along z
// (sz, + 1 for even sizes).
template <int W>
__global__ void __launch_bounds__(256) k_ws_morph_gradient_cols(const uint16_t* __restrict__ in, int nz, int ny, int nx,
                                                                int sz, int sy, int sx, int zchunk,
                                                                uint16_t* __restrict__ out) {
  const int x = blockIdx.x * 64 + (threadIdx.x & 63);
  const int y = blockIdx.y * 4 + (threadIdx.x >> 6);
  const int z_begin = blockIdx.z * zchunk, z_end = min(nz, z_begin + zchunk);
  if (x >= nx || y >= ny) return;
  const int ez = (sz & 1) ? 0 : 1, ey = (sy & 1) ? 0 : 1, ex = (sx & 1) ? 0 : 1;
  const int lo = sz / 2;                      // window along z: offsets [-lo, W - 1 - lo]
  // column / row indices of the 2-D window, reflected once (they do not depend on z)
  int pmin[W], pmax[W];
  auto plane = [&](int zz, int& mn, int& mx) {
    const uint16_t* pl = in + (size_t)reflect(zz, nz) * ny * nx;
    mn = 65535; mx = 0;
    for (int ky = 0; ky < sy + ey; ++ky) {
      const uint16_t* row = pl + (size_t)reflect(y - sy / 2 + ky, ny) * nx;
      const bool ero_y = ky < sy, dil_y = ky >= ey;
      for (int kx = 0; kx < sx + ex; ++kx) {
        const int v = row[reflect(x - sx / 2 + kx, nx)];
        if (ero_y && kx < sx) mn = min(mn, v);
        if (dil_y && kx >= ex) mx = max(mx, v);
      }
    }
  };
  // ring: entry k holds plane z - lo + k
#pragma unroll
  for (int k = 1; k < W; ++k) plane(z_begin - lo + k - 1, pmin[k], pmax[k]);
  for (int z = z_begin; z < z_end; ++z) {
#pragma unroll
    for (int k = 0; k < W - 1; ++k) { pmin[k] = pmin[k + 1]; pmax[k] = pmax[k + 1]; }
    plane(z - lo + W - 1, pmin[W - 1], pmax[W - 1]);
    int mn = 65535, mx = 0;
#pragma unroll
    for (int k = 0; k < W; ++k) {
      if (k < sz) mn = min(mn, pmin[k]);        // erosion: offsets [-lo, sz - 1 - lo]
      if (k >= ez) mx = max(mx, pmax[k]);       // dilation: shifted by one for even sizes
    }
    out[((size_t)z * ny + y) * nx + x] = (uint16_t)(mx - mn);
  }
}

// ---- tiled relaxation --------------------------------------------------------------------
constexpr int kT = 16;            // tile edge (voxels)
constexpr int kH = kT + 2;        // with halo
constexpr int kCells = kH * kH * kH;
constexpr int kThreads = 512;
constexpr int kOwn = kT * kT * kT / kThreads;  // 8
constexpr int kMaxRounds = 1 << 16;
constexpr uint32_t kInfC = 0xffffffffu;
constexpr unsigned long long kInfK = ~0ull;
// label SET of a voxel (phase 2): which labels can reach it along cost-optimal edges, whatever
// the reference's queue order. uint32: code = label + 32768 for one label (every int16 label is a
// legal code); kSetEmpty = nothing yet (the code of label 0, which no marker carries); kSetMulti =
// two different labels (the reference's answer there is an artefact of its queue order), above the
// 16-bit code range.
constexpr uint32_t kSetEmpty = 32768, kSetMulti = 0x10000;

struct Grid {
  int64_t nz, ny, nx;
  int ntz, nty, ntx;
};
Grid make_grid(int64_t nz, int64_t ny, int64_t nx) {
  Grid g;
  g.nz = nz; g.ny = ny; g.nx = nx;
  g.ntz = (int)ceil_div64(nz, kT); g.nty = (int)ceil_div64(ny, kT); g.ntx = (int)ceil_div64(nx, kT);
  return g;
}

struct WsWs {
  uint32_t* cost;
  unsigned long long* key;
  uint32_t* lset;
  uint8_t* active[2];
  int* flags;
  int64_t bytes;
};
WsWs carve(void* base, const Grid& g) {
  WsWs w;
  int64_t n = g.nz * g.ny * g.nx, nt = (int64_t)g.ntz * g.nty * g.ntx;
  char* p = (char*)base;
  int64_t off = 0;
  w.key = (unsigned long long*)(p + off); off += align256(n * 8);
  w.cost = (uint32_t*)(p + off); off += align256(n * 4);
  w.lset = (uint32_t*)(p + off); off += align256(n * 4);
  w.active[0] = (uint8_t*)(p + off); off += align256(nt);
  w.active[1] = (uint8_t*)(p + off); off += align256(nt);
  w.flags = (int*)(p + off); off += align256((int64_t)(kMaxRounds + 2) * 4);
  w.bytes = off;
  return w;
}

// markers: cost 0 (IFT) or I (value flood), key = label (hops 0); others: infinity. Every
// tile holding a marker is active in round 0.
__global__ void __launch_bounds__(256) k_ws_init(const uint16_t* __restrict__ img, const int16_t* __restrict__ markers,
                                                 Grid g, int mode, uint32_t* __restrict__ cost,
                                                 unsigned long long* __restrict__ key, uint32_t* __restrict__ lset,
                                                 uint8_t* active, int* flags) {
  const int64_t n = g.nz * g.ny * g.nx;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    int m = markers[i];
    if (m != 0) {
      cost[i] = mode == 0 ? 0u : (uint32_t)img[i];
      key[i] = (unsigned long long)(uint32_t)(m + 32768);
      lset[i] = (uint32_t)(m + 32768);
      int64_t x = i % g.nx, r = i / g.nx, y = r % g.ny, z = r / g.ny;
      active[((int)(z / kT) * g.nty + (int)(y / kT)) * g.ntx + (int)(x / kT)] = 1;
      flags[0] = 1;
    } else {
      cost[i] = kInfC;
      key[i] = kInfK;
      lset[i] = kSetEmpty;
    }
  }
}

__global__ void k_ws_activate_all(uint8_t* active, int64_t ntiles, int* flags, int round) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < ntiles) active[i] = 1;
  if (i == 0) flags[round] = 1;
}

// PHASE 1: relax costs. PHASE 2: relax (hops, label) keys along cost-optimal edges.
// MODE 0: edge weight |I(v) - I(p)|; MODE 1: weight I(p).
template <int PHASE, int MODE>
__global__ void __launch_bounds__(kThreads) k_ws_round(const uint16_t* __restrict__ img, uint32_t* cost,
                                                       unsigned long long* key, uint32_t* lset, Grid g, uint32_t sb,
                                                       uint8_t* active_cur, uint8_t* active_next, int* flags,
                                                       int round) {
  if (flags[round] == 0) return;
  const int tile = blockIdx.x;
  if (!__syncthreads_or(active_cur[tile] != 0)) return;
  extern __shared__ unsigned char smem_raw[];
  unsigned long long* sK = (unsigned long long*)smem_raw;                    // PHASE 2 only
  uint32_t* sA = (uint32_t*)(smem_raw + kCells * 8);                         // PHASE 2 only
  uint32_t* sC = (uint32_t*)(smem_raw + (PHASE == 2 ? kCells * 12 : 0));
  uint16_t* sI = (uint16_t*)((unsigned char*)sC + kCells * 4);
  __shared__ int s_faces;
  const int tid = threadIdx.x;
  const int tx = tile % g.ntx, ty = (tile / g.ntx) % g.nty, tz = tile / (g.ntx * g.nty);
  const int64_t z0 = (int64_t)tz * kT, y0 = (int64_t)ty * kT, x0 = (int64_t)tx * kT;
  if (tid == 0) {
    active_cur[tile] = 0;
    s_faces = 0;
  }
  for (int i = tid; i < kCells; i += kThreads) {
    int hx = i % kH, hy = (i / kH) % kH, hz = i / (kH * kH);
    int64_t z = z0 + hz - 1, y = y0 + hy - 1, x = x0 + hx - 1;
    uint32_t c = kInfC;
    unsigned long long k = kInfK;
    uint16_t v = 0;
    uint32_t a = kSetEmpty;
    // MODE 0 reproduces scipy.ndimage.watershed_ift's neighbourhood: the volume is walked as
    // a flat array, a neighbour is any flat index + structure offset inside [0, N), so rows
    // and planes wrap into each other at the volume faces (verified against SciPy 1.18.1).
    const int64_t p = (z * g.ny + y) * g.nx + x;
    const bool valid = MODE == 0 ? (p >= 0 && p < g.nz * g.ny * g.nx)
                                 : (z >= 0 && z < g.nz && y >= 0 && y < g.ny && x >= 0 && x < g.nx);
    if (valid) {
      c = __ldcg(&cost[p]);
      v = img[p];
      if (PHASE == 2) { k = __ldcg(&key[p]); a = __ldcg(&lset[p]); }
    }
    sC[i] = c;
    sI[i] = v;
    if (PHASE == 2) { sK[i] = k; sA[i] = a; }
  }
  __syncthreads();
  int hidx[kOwn];
  bool any_own_changed = false;
#pragma unroll
  for (int k = 0; k < kOwn; ++k) {
    int i = tid + k * kThreads;
    int lx = i % kT, ly = (i / kT) % kT, lz = i / (kT * kT);
    bool in = z0 + lz < g.nz && y0 + ly < g.ny && x0 + lx < g.nx;
    hidx[k] = in ? ((lz + 1) * kH + (ly + 1)) * kH + (lx + 1) : -1;
  }
  uint32_t cmask = 0;  // which of my cells changed
  int changed, iters = 0;
  do {
    changed = 0;
#pragma unroll
    for (int k = 0; k < kOwn; ++k) {
      const int h = hidx[k];
      if (h < 0) continue;
      const int ip = sI[h];
      if (PHASE == 1) {
        uint32_t c = sC[h], best = c;
        if (c == 0 || (MODE == 1 && c == (uint32_t)ip)) continue;  // cannot improve
#pragma unroll
        for (int oz = -1; oz <= 1; ++oz)
#pragma unroll
          for (int oy = -1; oy <= 1; ++oy)
#pragma unroll
            for (int ox = -1; ox <= 1; ++ox) {
              if (!((sb >> ((oz + 1) * 9 + (oy + 1) * 3 + (ox + 1))) & 1u)) continue;
              const int v = h - ((oz * kH + oy) * kH + ox);  // the voxel that reaches p by +off
              uint32_t cv = sC[v];
              if (cv == kInfC) continue;
              uint32_t w = MODE == 0 ? (uint32_t)abs((int)sI[v] - ip) : (uint32_t)ip;
              uint32_t cand = cv > w ? cv : w;
              best = cand < best ? cand : best;
            }
        if (best < c) {
          sC[h] = best;
          changed = 1;
          cmask |= 1u << k;
        }
      } else {
        unsigned long long kk = sK[h], best = kk;
        if ((kk >> 32) == 0) continue;  // a marker keeps its label
        const uint32_t c = sC[h];
        if (c == kInfC) continue;
        const uint32_t a0 = sA[h];
        uint32_t a1 = a0;
        // MODE 1 (label at push time): the voxel inherits from the neighbour that is flooded
        // first, i.e. one with the smallest cost among ALL its neighbours.
        uint32_t cmin = kInfC;
        if (MODE == 1) {
#pragma unroll
          for (int oz = -1; oz <= 1; ++oz)
#pragma unroll
            for (int oy = -1; oy <= 1; ++oy)
#pragma unroll
              for (int ox = -1; ox <= 1; ++ox) {
                if (!((sb >> ((oz + 1) * 9 + (oy + 1) * 3 + (ox + 1))) & 1u)) continue;
                uint32_t cv = sC[h - ((oz * kH + oy) * kH + ox)];
                cmin = cv < cmin ? cv : cmin;
              }
        }
#pragma unroll
        for (int oz = -1; oz <= 1; ++oz)
#pragma unroll
          for (int oy = -1; oy <= 1; ++oy)
#pragma unroll
            for (int ox = -1; ox <= 1; ++ox) {
              if (!((sb >> ((oz + 1) * 9 + (oy + 1) * 3 + (ox + 1))) & 1u)) continue;
              const int v = h - ((oz * kH + oy) * kH + ox);
              unsigned long long kv = sK[v];
              if (kv == kInfK) continue;
              uint32_t cv = sC[v];
              if (MODE == 0) {
                uint32_t w = (uint32_t)abs((int)sI[v] - ip);
                uint32_t via = cv > w ? cv : w;
                if (via != c) continue;  // not a cost-optimal edge
              } else {
                if (cv != cmin) continue;  // not among the first-flooded neighbours
              }
              unsigned long long cand = kv + (1ull << 32);
              best = cand < best ? cand : best;
              // join of the label sets of every admissible predecessor
              const uint32_t av = sA[v];
              if (av != kSetEmpty) a1 = (a1 == kSetEmpty) ? av : (a1 == av ? a1 : kSetMulti);
            }
        if (best < kk || a1 != a0) {
          sK[h] = best;
          sA[h] = a1;
          changed = 1;
          cmask |= 1u << k;
        }
      }
    }
    changed = __syncthreads_or(changed);
    ++iters;
  } while (changed && iters < 4 * kT);
  const bool unfinished = changed != 0;  // iteration cap hit: come back next round

  int faces = 0;
#pragma unroll
  for (int k = 0; k < kOwn; ++k) {
    if (!((cmask >> k) & 1u)) continue;
    any_own_changed = true;
    int i = tid + k * kThreads;
    int lx = i % kT, ly = (i / kT) % kT, lz = i / (kT * kT);
    int64_t p = ((z0 + lz) * g.ny + (y0 + ly)) * g.nx + (x0 + lx);
    if (PHASE == 1) __stcg(&cost[p], sC[hidx[k]]);
    else { __stcg(&key[p], sK[hidx[k]]); __stcg(&lset[p], sA[hidx[k]]); }
    faces |= 64;
    if (lz == 0) faces |= 1;
    if (lz == kT - 1) faces |= 2;
    if (ly == 0) faces |= 4;
    if (ly == kT - 1 || y0 + ly == g.ny - 1) faces |= 8;
    if (lx == 0) faces |= 16;
    if (lx == kT - 1 || x0 + lx == g.nx - 1) faces |= 32;
  }
  (void)any_own_changed;
  if (faces) atomicOr(&s_faces, faces);
  __syncthreads();
  faces = s_faces;
  if (unfinished && tid == 0) {
    active_next[tile] = 1;
    flags[round + 1] = 1;
  }
  if ((faces & 63) == 0) return;
  __threadfence();
  if (MODE == 0) {
    // wrapped neighbours live in tiles on the opposite x / y border (a row end touches the
    // next row's start, a plane's last row the next plane's first): wake those up too
    const bool xb = ((faces & 16) && tx == 0) || ((faces & 32) && tx == g.ntx - 1);
    const bool yb = ((faces & 4) && ty == 0) || ((faces & 8) && ty == g.nty - 1);
    if (xb)
      for (int i = tid; i < 2 * 5 * g.nty; i += kThreads) {
        int side = i % 2, dzt = (i / 2) % 5 - 2, yy = i / 10;
        int nz = tz + dzt, nx = side ? g.ntx - 1 : 0;
        if (nz >= 0 && nz < g.ntz) { active_next[(nz * g.nty + yy) * g.ntx + nx] = 1; flags[round + 1] = 1; }
      }
    if (yb)
      for (int i = tid; i < 2 * 5 * g.ntx; i += kThreads) {
        int side = i % 2, dzt = (i / 2) % 5 - 2, xx = i / 10;
        int nz = tz + dzt, ny = side ? g.nty - 1 : 0;
        if (nz >= 0 && nz < g.ntz) { active_next[(nz * g.nty + ny) * g.ntx + xx] = 1; flags[round + 1] = 1; }
      }
  }
  if (tid < 27) {
    int oz = tid / 9 - 1, oy = (tid / 3) % 3 - 1, ox = tid % 3 - 1;
    if (oz == 0 && oy == 0 && ox == 0) return;
    bool need = true;
    if (oz == -1) need = need && (faces & 1);
    if (oz == 1) need = need && (faces & 2);
    if (oy == -1) need = need && (faces & 4);
    if (oy == 1) need = need && (faces & 8);
    if (ox == -1) need = need && (faces & 16);
    if (ox == 1) need = need && (faces & 32);
    int nz = tz + oz, ny = ty + oy, nx = tx + ox;
    if (need && nz >= 0 && nz < g.ntz && ny >= 0 && ny < g.nty && nx >= 0 && nx < g.ntx) {
      active_next[(nz * g.nty + ny) * g.ntx + nx] = 1;
      flags[round + 1] = 1;
    }
  }
}

__global__ void __launch_bounds__(256) k_ws_labels(const unsigned long long* __restrict__ key,
                                                   const uint32_t* __restrict__ lset, int64_t n,
                                                   int16_t* __restrict__ labels, uint8_t* __restrict__ ambiguous) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    unsigned long long k = key[i];
    labels[i] = k == kInfK ? (int16_t)0 : (int16_t)((int)(uint32_t)(k & 0xffffffffu) - 32768);
    if (ambiguous) ambiguous[i] = lset[i] == kSetMulti ? 1 : 0;
  }
}

template <int PHASE, int MODE>
int run_phase(const uint16_t* img, const WsWs& w, const Grid& g, uint32_t sb, cudaStream_t s, int* round_io) {
  const int ntiles = g.ntz * g.nty * g.ntx;
  const size_t smem = (size_t)kCells * (PHASE == 2 ? 18 : 6);
  auto kern = k_ws_round<PHASE, MODE>;
  B2V_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int r = *round_io, batch = 4, rc;
  while (true) {
    B2V_REQUIRE(r + batch < kMaxRounds, B2V_ERR_NOCONV, "watershed: no convergence after %d rounds", r);
    for (int k = 0; k < batch; ++k, ++r) {
      kern<<<ntiles, kThreads, smem, s>>>(img, w.cost, w.key, w.lset, g, sb, w.active[r & 1], w.active[(r + 1) & 1],
                                          w.flags, r);
      if ((rc = b2v_check_launch("k_ws_round"))) return rc;
    }
    int more = 0;
    B2V_CUDA(cudaMemcpyAsync(&more, w.flags + r, sizeof(int), cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    if (!more) break;
    if (batch < 32) batch *= 2;
  }
  *round_io = r;
  return B2V_OK;
}

int ws_strct_bits(const uint8_t* st, int64_t odz, int64_t ody, int64_t odx, uint32_t* sb) {
  B2V_REQUIRE(st && odz >= 1 && ody >= 1 && odx >= 1 && odz <= 3 && ody <= 3 && odx <= 3 && (odz & 1) && (ody & 1) &&
                  (odx & 1),
              B2V_ERR_ARG, "watershed: the structuring element must be 1 or 3 wide on every axis");
  *sb = strct_mask(st, odz, ody, odx) & ~(1u << 13);   // without the centre
  return B2V_OK;
}

}  // namespace

extern "C" int b2v_ws_lut_i16(const int16_t* img, int64_t n, double window, double level, uint16_t* out,
                              void* stream) {
  B2V_REQUIRE(img && out && n > 0, B2V_ERR_ARG, "ws_lut: bad arguments");
  k_ws_lut<<<b2v_grid(n, 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(img, n, window, level, out);
  return b2v_check_launch("k_ws_lut");
}

extern "C" int b2v_ws_shift_i16(const int16_t* img, int64_t n, uint16_t* out, void* workspace, void* stream) {
  B2V_REQUIRE(img && out && workspace && n > 0, B2V_ERR_ARG, "ws_shift: bad arguments");
  float* mm = (float*)workspace;
  int rc = b2v_minmax_f32(img, B2V_I16, n, mm, (char*)workspace + 256, stream);
  if (rc) return rc;
  k_ws_shift<<<b2v_grid(n, 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(img, n, mm, out);
  return b2v_check_launch("k_ws_shift");
}

extern "C" int b2v_ws_shift_i16_with(const int16_t* img, int64_t n, const float* minmax_dev, uint16_t* out, void* stream) {
  B2V_REQUIRE(img && out && minmax_dev && n > 0, B2V_ERR_ARG, "ws_shift: bad arguments");
  k_ws_shift<<<b2v_grid(n, 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(img, n, minmax_dev, out);
  return b2v_check_launch("k_ws_shift");
}

extern "C" int b2v_ws_morph_gradient_u16(const uint16_t* in, int64_t nz, int64_t ny, int64_t nx, int sz, int sy,
                                         int sx, uint16_t* out, void* stream) {
  B2V_REQUIRE(in && out && nz > 0 && ny > 0 && nx > 0, B2V_ERR_ARG, "ws_morph_gradient: bad arguments");
  B2V_REQUIRE(sz >= 1 && sy >= 1 && sx >= 1 && sz <= 31 && sy <= 31 && sx <= 31, B2V_ERR_ARG,
              "ws_morph_gradient: size must be in 1..31");
  const int W = sz + ((sz & 1) ? 0 : 1);
  if (W <= 6 && nz < (1ll << 30) && ny < (1ll << 30) && nx < (1ll << 30)) {
    int zchunk = 64;
    dim3 grid((unsigned)ceil_div64(nx, 64), (unsigned)ceil_div64(ny, 4), (unsigned)ceil_div64(nz, zchunk));
    cudaStream_t s = (cudaStream_t)stream;
#define B2V_MG(WW) k_ws_morph_gradient_cols<WW><<<grid, 256, 0, s>>>(in, (int)nz, (int)ny, (int)nx, sz, sy, sx, zchunk, out)
    switch (W) {
      case 1: B2V_MG(1); break;
      case 2: B2V_MG(2); break;
      case 3: B2V_MG(3); break;
      case 4: B2V_MG(4); break;
      case 5: B2V_MG(5); break;
      default: B2V_MG(6); break;
    }
#undef B2V_MG
    return b2v_check_launch("k_ws_morph_gradient_cols");
  }
  k_ws_morph_gradient<<<b2v_grid(nz * ny * nx, 256 * 4, 16), 256, 0, (cudaStream_t)stream>>>(in, nz, ny, nx, sz, sy, sx,
                                                                                             out);
  return b2v_check_launch("k_ws_morph_gradient");
}

extern "C" int64_t b2v_ws_workspace_bytes(int64_t nz, int64_t ny, int64_t nx) {
  if (nz <= 0 || ny <= 0 || nx <= 0) return 0;
  int64_t a = carve(nullptr, make_grid(nz, ny, nx)).bytes;
  int64_t b = 256 + b2v_minmax_workspace_bytes(nz * ny * nx);
  int64_t c = b2v_wsf_workspace_bytes(nz, ny, nx);
  a = a > b ? a : b;
  return a > c ? a : c;
}

extern "C" int b2v_ws_flood(const uint16_t* img, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                            const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, int mode,
                            int16_t* labels, uint8_t* ambiguous, void* workspace, void* stream, int* rounds_out) {
  B2V_REQUIRE(img && markers && labels && workspace, B2V_ERR_ARG, "ws_flood: null pointer");
  B2V_REQUIRE(nz > 0 && ny > 0 && nx > 0, B2V_ERR_ARG, "ws_flood: empty volume");
  B2V_REQUIRE(mode == 0 || mode == 1, B2V_ERR_ARG, "ws_flood: mode must be 0 (IFT) or 1 (value flood)");
  uint32_t sb;
  int rc;
  if ((rc = ws_strct_bits(strct_host, odz, ody, odx, &sb))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  {
    // 6-connected (the InVesalius default, generate_binary_structure(3, 1)): the persistent engine.
    // Offsets along an axis of extent 1 never apply, so they do not count.
    const uint32_t zb = (1u << 4) | (1u << 22), yb = (1u << 10) | (1u << 16), xb = (1u << 12) | (1u << 14);
    uint32_t eff = sb | (nz == 1 ? zb : 0u) | (ny == 1 ? yb : 0u) | (nx == 1 ? xb : 0u);
    if (eff == kSB6 && !getenv("B2V_WS_GENERIC")) {
      int rounds = 0;
      rc = b2v_wsf_run(31, img, markers, nz, ny, nx, mode, 0, 0, labels, ambiguous, ambiguous ? 1 : 0, workspace, stream,
                       &rounds, 1);
      if (rounds_out) *rounds_out = rounds;
      return rc;
    }
  }
  Grid g = make_grid(nz, ny, nx);
  WsWs w = carve(workspace, g);
  const int64_t n = nz * ny * nx;
  const int64_t ntiles = (int64_t)g.ntz * g.nty * g.ntx;
  B2V_CUDA(cudaMemsetAsync(w.active[0], 0, (size_t)((char*)w.flags - (char*)w.active[0]) + (kMaxRounds + 2) * 4, s));
  k_ws_init<<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>(img, markers, g, mode, w.cost, w.key, w.lset, w.active[0],
                                                     w.flags);
  if ((rc = b2v_check_launch("k_ws_init"))) return rc;
  int round = 0;
  rc = mode == 0 ? run_phase<1, 0>(img, w, g, sb, s, &round) : run_phase<1, 1>(img, w, g, sb, s, &round);
  if (rc) return rc;
  // phase 2 starts with every tile active (markers seed the keys; costs are final)
  k_ws_activate_all<<<(unsigned)ceil_div64(ntiles, 256), 256, 0, s>>>(w.active[round & 1], ntiles, w.flags, round);
  if ((rc = b2v_check_launch("k_ws_activate_all"))) return rc;
  rc = mode == 0 ? run_phase<2, 0>(img, w, g, sb, s, &round) : run_phase<2, 1>(img, w, g, sb, s, &round);
  if (rc) return rc;
  k_ws_labels<<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>(w.key, w.lset, n, labels, ambiguous);
  if ((rc = b2v_check_launch("k_ws_labels"))) return rc;
  if (rounds_out) *rounds_out = round;
  return B2V_OK;
}
