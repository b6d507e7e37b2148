// The point -> cell links of a triangle mesh (vtkCellLinks), and the stable radix sort they are built with
// (the scan is scan.cuh's). Shared by the surface tools that walk a mesh through its links (connectivity.cu,
// smoothing.cu, fill_holes.cu, normals.cu); every name is in an anonymous namespace, so each translation unit
// has its own copy.
//
//   k_conn_load   faces -> int32 [T][3] (a bad face sets ST_BAD_FACE), link counts per point.
//   lstart        an exclusive scan of the counts: point p's links are links[lstart[p], lstart[p + 1]).
//   links         the corners (in corner order, i.e. ascending cell) stably sorted by point id: each point's
//                 cells in ascending id, a degenerate triangle once per corner it occupies.
//   edge_neighbors  GetCellEdgeNeighbors through those links.
//   uf_find / uf_unite  a lock-free union-find whose roots are the lowest ids of their sets.
//
// Stable sorts are LSD radix passes of 8 bits (per-block digit histograms, one scan, a scatter ranked by
// warp match), only over the bits the largest key needs.
#pragma once
#include "b2v_common.cuh"
#include "scan.cuh"

namespace {

constexpr int kBlock = 256;
constexpr int kMaxBlocksPerSm = 2;                 // blocks per SM of a cooperative launch, at most

// ---- stable LSD radix sort of (key, value) pairs, 8 bits a pass -------------------------------------------
__global__ void __launch_bounds__(kBlock) k_rs_hist(const uint32_t* __restrict__ keys, int64_t n, int shift,
                                                    int64_t nb, unsigned long long* hist) {
  __shared__ uint32_t s_c[256];
  s_c[threadIdx.x] = 0;
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i < n) atomicAdd(&s_c[(keys[i] >> shift) & 255u], 1u);
  __syncthreads();
  hist[(int64_t)threadIdx.x * nb + blockIdx.x] = s_c[threadIdx.x];
}

__global__ void __launch_bounds__(kBlock) k_rs_scatter(const uint32_t* __restrict__ kin,
                                                       const uint32_t* __restrict__ vin, int64_t n, int shift,
                                                       int64_t nb, const unsigned long long* __restrict__ hist,
                                                       uint32_t* __restrict__ kout, uint32_t* __restrict__ vout) {
  __shared__ uint32_t s_c[kBlock / 32][256];
  for (int k = threadIdx.x; k < (kBlock / 32) * 256; k += kBlock) (&s_c[0][0])[k] = 0;
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t key = i < n ? kin[i] : 0u;
  const uint32_t d = i < n ? (key >> shift) & 255u : 256u;   // 256: no item
  const uint32_t peers = __match_any_sync(0xffffffffu, d);
  const uint32_t below = peers & ((1u << lane) - 1u);
  if (d < 256u && below == 0) s_c[wid][d] = __popc(peers);
  __syncthreads();
  if (d >= 256u) return;
  uint32_t r = __popc(below);
  for (int w = 0; w < wid; ++w) r += s_c[w][d];
  const unsigned long long pos = hist[(int64_t)d * nb + blockIdx.x] + r;
  kout[pos] = key;
  vout[pos] = vin[i];
}

// Sorts (w.ka, w.va)[0..n) stably by key < 2^keybits; the result is in (ka, va) or (kb, vb): *out_v says
// which. W is a workspace record with the four [n] ping-pong arrays ka, va, kb, vb, hist
// [256 ceil(n / kBlock) + 1] and scratch [scan_blocks(that) + 1].
template <typename W>
int sort_pairs(W& w, int64_t n, int keybits, uint32_t** out_v, cudaStream_t s) {
  uint32_t *ki = w.ka, *vi = w.va, *ko = w.kb, *vo = w.vb;
  const int64_t nb = ceil_div64(n, kBlock);
  for (int shift = 0; shift < keybits && n > 1; shift += 8) {
    k_rs_hist<<<(unsigned)nb, kBlock, 0, s>>>(ki, n, shift, nb, w.hist);
    if (int rc = b2v_check_launch("k_rs_hist")) return rc;
    if (int rc = scan(w.hist, 256 * nb, w.scratch, nullptr, s)) return rc;
    k_rs_scatter<<<(unsigned)nb, kBlock, 0, s>>>(ki, vi, n, shift, nb, w.hist, ko, vo);
    if (int rc = b2v_check_launch("k_rs_scatter")) return rc;
    uint32_t* t = ki; ki = ko; ko = t;
    t = vi; vi = vo; vo = t;
  }
  *out_v = vi;
  return B2V_OK;
}

int bits_for(int64_t max_key) {
  int b = 0;
  while (b < 32 && (max_key >> b) > 0) ++b;
  return b;
}

// ---- faces and links -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_conn_load(Faces F, int32_t* __restrict__ tri, unsigned long long* deg,
                                                     uint32_t* ka, uint32_t* va, uint32_t* status) {
  for (int64_t t = gtid(); t < F.nt; t += gstride()) {
    int64_t v[3];
    if (!load_face(F, t, v)) {
      atomicOr(status, ST_BAD_FACE);
      v[0] = v[1] = v[2] = 0;
    }
    for (int j = 0; j < 3; ++j) {
      tri[3 * t + j] = (int32_t)v[j];
      atomicAdd(&deg[v[j]], 1ull);
      ka[3 * t + j] = (uint32_t)v[j];
      va[3 * t + j] = (uint32_t)t;
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_copy_i32(const uint32_t* __restrict__ in, int64_t n, int32_t* out) {
  for (int64_t i = gtid(); i < n; i += gstride()) out[i] = (int32_t)in[i];
}

// GetCellEdgeNeighbors(c, p1, p2) over the links: the cells d != c in p1's links that contain p2, in link
// order, duplicates included. Returns their number; *first becomes the first of them and *lowest the lowest
// (both unchanged when there is none).
__device__ __forceinline__ int64_t edge_neighbors(const int32_t* __restrict__ tri,
                                                  const unsigned long long* __restrict__ lstart,
                                                  const int32_t* __restrict__ links, int64_t c, int32_t p1,
                                                  int32_t p2, int64_t* first, int64_t* lowest) {
  int64_t num = 0;
  for (unsigned long long k = lstart[p1]; k < lstart[p1 + 1]; ++k) {
    const int32_t d = links[k];
    if (d == c) continue;
    if (tri[3 * (int64_t)d] == p2 || tri[3 * (int64_t)d + 1] == p2 || tri[3 * (int64_t)d + 2] == p2) {
      if (num == 0) *first = d;
      ++num;
      if (d < *lowest) *lowest = d;
    }
  }
  return num;
}

// ---- union-find over int32 ids: a root is the lowest id of its set --------------------------------------
__device__ __forceinline__ int32_t uf_find(const int32_t* parent, int32_t x) {
  const volatile int32_t* p = parent;
  int32_t y = p[x];
  while (y != x) { x = y; y = p[x]; }
  return x;
}

__device__ __forceinline__ void uf_unite(int32_t* parent, int32_t a, int32_t b) {
  for (;;) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a > b) { const int32_t t = a; a = b; b = t; }
    const int32_t old = atomicCAS(&parent[b], b, a);   // hook the larger root under the smaller
    if (old == b) return;
    b = old;
  }
}

// Loads the faces into w.tri and builds w.lstart [V + 1] and w.links [3T] (nt > 0). W also holds status and
// the sort buffers of sort_pairs, with room for 3T items. A bad face is B2V_ERR_ARG, reported as
// "<what>: a face has an index ...". Synchronises the stream.
template <typename W>
int build_links(W& w, const Faces& F, const char* what, cudaStream_t s) {
  const int64_t nv = F.nv, C3 = 3 * F.nt;
  B2V_CUDA(cudaMemsetAsync(w.status, 0, 16, s));
  B2V_CUDA(cudaMemsetAsync(w.lstart, 0, (size_t)(nv + 1) * 8, s));
  k_conn_load<<<b2v_grid(F.nt, kBlock, 16), kBlock, 0, s>>>(F, w.tri, w.lstart, w.ka, w.va, w.status);
  if (int rc = b2v_check_launch("k_conn_load")) return rc;
  uint32_t status = 0;
  B2V_CUDA(cudaMemcpyAsync(&status, w.status, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!(status & ST_BAD_FACE), B2V_ERR_ARG,
              "%s: a face has an index outside [0, V) (or a leading entry other than 3)", what);
  if (int rc = scan(w.lstart, nv + 1, w.scratch, nullptr, s)) return rc;
  uint32_t* lv = nullptr;
  if (int rc = sort_pairs(w, C3, bits_for(nv - 1), &lv, s)) return rc;
  k_copy_i32<<<b2v_grid(C3, kBlock, 16), kBlock, 0, s>>>(lv, C3, w.links);
  return b2v_check_launch("k_copy_i32");
}

// A cooperative launch of fn with kBlock threads and as many blocks as fit at once, at most kMaxBlocksPerSm
// per SM. A kernel that does not fit is B2V_ERR_CUDA, reported as "<op>: <what> does not fit on an SM".
inline int launch_coop(const void* fn, void** args, cudaStream_t s, const char* op, const char* what) {
  int per_sm = 0;
  B2V_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kBlock, 0));
  B2V_REQUIRE(per_sm >= 1, B2V_ERR_CUDA, "%s: %s does not fit on an SM", op, what);
  if (per_sm > kMaxBlocksPerSm) per_sm = kMaxBlocksPerSm;
  B2V_CUDA(cudaLaunchCooperativeKernel(fn, dim3(per_sm * b2v_sm_count()), dim3(kBlock), args, 0, s));
  return b2v_check_launch(what);
}

}  // namespace
