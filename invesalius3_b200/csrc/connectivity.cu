// The surface connectivity tools on the device: vtkPolyDataConnectivityFilter on triangles, as InVesalius's
// "Select largest surface", "Split all disconnected surfaces" and "Select regions of interest..." use it
// (polydata_utils.py:206-278). The contract is restated once, in the C checker's header (connectivity.c,
// DESIGN.md §3 "Surface connectivity"): regions in
// the order of their lowest cell, cells marked in VTK's wave order, points numbered in order of first use.
// Every step below reproduces that order exactly, with no per-wave host round trip.
//
//   build_links          faces -> int32 [T][3] and the point -> cell links of vtkCellLinks, duplicates of
//                        degenerate triangles included (mesh_links.cuh).
//   k_cc_*               union-find over the triangle-point incidence (hook, then compress); each
//                        component's minimum cell; a scan of the "minimum cell" flags numbers the regions
//                        and lists their first cells: wave 0 of every region at once.
//   k_waves<ConnNb>      one persistent cooperative launch runs every wave of every region (waves.cuh): the
//                        appended list of wave L+1 is laid out by a scan over wave L (parent order, then j,
//                        then link order), each unmarked candidate takes the atomicMin of its positions, and
//                        a second scan compacts the winners in position order. That is VTK's processing
//                        order, in linear work and without a sort.
//   sort by region       the processed sequence (wave-major) stably sorted by region: region-major ranks.
//   k_conn_first_use     each point takes the atomicMin of (rank, j) over its corners; a scan of the
//                        first-use flags is PointMap, region by region.
//   faces                the visited cells, in ascending id, stably sorted by region.
//
// Stable sorts are the radix sort of mesh_links.cuh.
#include <string.h>

#include "b2v_common.cuh"
#include "mesh_links.cuh"
#include "waves.cuh"

namespace {

struct ConnWs {
  long long* ctl;                  // [0..15]: two state records for the persistent launch, then results
  uint32_t* status;
  unsigned long long* totals;      // [8] scan totals
  int32_t* tri;                    // [T][3]
  unsigned long long* lstart;      // [V + 1] link offsets
  int32_t* links;                  // [3T]
  uint32_t *ka, *va, *kb, *vb;     // [3T] sort ping-pong
  unsigned long long* hist;        // [256 * nb3 + 1]
  unsigned long long* scratch;     // scan block sums
  int32_t* parent;                 // [V]
  uint32_t* cmin;                  // [V]
  unsigned long long* tflag;       // [T + 1]
  int32_t* reg;                    // [T]
  unsigned long long* best;        // [T]
  int32_t* seq;                    // [T] processed cells, wave-major
  int64_t* seeds;                  // [nseeds]
  unsigned long long *loc1, *loc2; // [max(T, nseeds)]
  unsigned long long* btot;        // [2][kMaxGrid]
  unsigned long long* celloff;     // [T + 2]
  int32_t* rank;                   // [T] processed cells, region-major
  unsigned long long* fu;          // [V] first-use corner
  unsigned long long* cflag;       // [3T + 1]
  int32_t* pmap;                   // [V]
  int32_t* inv;                    // [V]
  int32_t* cells;                  // [T] visited cells, grouped by region
  unsigned long long* ptoff;       // [T + 2]
  int64_t nb3;
  size_t bytes;
};

ConnWs carve(void* base, int64_t nv, int64_t nt, int64_t nseeds) {
  ConnWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const size_t V = (size_t)nv, T = (size_t)nt, C3 = 3 * T;
  const size_t items = T > (size_t)nseeds ? T : (size_t)nseeds;
  w.nb3 = ceil_div64((int64_t)(C3 > 0 ? C3 : 1), kBlock);
  const int64_t hist_n = 256 * w.nb3 + 1;
  int64_t longest = hist_n;
  if ((int64_t)C3 + 1 > longest) longest = (int64_t)C3 + 1;
  if ((int64_t)V + 1 > longest) longest = (int64_t)V + 1;
  w.ctl = (long long*)take(16 * 8);
  w.status = (uint32_t*)take(16);
  w.totals = (unsigned long long*)take(8 * 8);
  w.tri = (int32_t*)take(C3 * 4);
  w.lstart = (unsigned long long*)take((V + 1) * 8);
  w.links = (int32_t*)take(C3 * 4);
  w.ka = (uint32_t*)take(C3 * 4);
  w.va = (uint32_t*)take(C3 * 4);
  w.kb = (uint32_t*)take(C3 * 4);
  w.vb = (uint32_t*)take(C3 * 4);
  w.hist = (unsigned long long*)take((size_t)hist_n * 8);
  w.scratch = (unsigned long long*)take((size_t)(scan_blocks(longest) + 1) * 8);
  w.parent = (int32_t*)take(V * 4);
  w.cmin = (uint32_t*)take(V * 4);
  w.tflag = (unsigned long long*)take((T + 1) * 8);
  w.reg = (int32_t*)take(T * 4);
  w.best = (unsigned long long*)take(T * 8);
  w.seq = (int32_t*)take(T * 4);
  w.seeds = (int64_t*)take((size_t)nseeds * 8);
  w.loc1 = (unsigned long long*)take(items * 8);
  w.loc2 = (unsigned long long*)take(items * 8);
  w.btot = (unsigned long long*)take(2 * kMaxGrid * 8);
  w.celloff = (unsigned long long*)take((T + 2) * 8);
  w.rank = (int32_t*)take(T * 4);
  w.fu = (unsigned long long*)take(V * 8);
  w.cflag = (unsigned long long*)take((C3 + 1) * 8);
  w.pmap = (int32_t*)take(V * 4);
  w.inv = (int32_t*)take(V * 4);
  w.cells = (int32_t*)take(T * 4);
  w.ptoff = (unsigned long long*)take((T + 2) * 8);
  w.bytes = o;
  return w;
}

// ---- union-find partition (uf_find / uf_unite: mesh_links.cuh) ------------------------------------------
__global__ void __launch_bounds__(kBlock) k_cc_init(int32_t* parent, uint32_t* cmin, int64_t nv) {
  for (int64_t p = gtid(); p < nv; p += gstride()) { parent[p] = (int32_t)p; cmin[p] = 0xffffffffu; }
}

__global__ void __launch_bounds__(kBlock) k_cc_hook(const int32_t* __restrict__ tri, int64_t nt, int32_t* parent) {
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    uf_unite(parent, tri[3 * t], tri[3 * t + 1]);
    uf_unite(parent, tri[3 * t], tri[3 * t + 2]);
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_compress(int32_t* parent, int64_t nv) {
  for (int64_t p = gtid(); p < nv; p += gstride()) parent[p] = uf_find(parent, (int32_t)p);
}

__global__ void __launch_bounds__(kBlock) k_cc_min(const int32_t* __restrict__ tri, int64_t nt,
                                                   const int32_t* __restrict__ parent, uint32_t* cmin) {
  for (int64_t t = gtid(); t < nt; t += gstride()) atomicMin(&cmin[parent[tri[3 * t]]], (uint32_t)t);
}

__global__ void __launch_bounds__(kBlock) k_cc_flags(const int32_t* __restrict__ tri, int64_t nt,
                                                     const int32_t* __restrict__ parent,
                                                     const uint32_t* __restrict__ cmin, unsigned long long* flag,
                                                     int32_t* reg, unsigned long long* best) {
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    flag[t] = cmin[parent[tri[3 * t]]] == (uint32_t)t ? 1ull : 0ull;
    reg[t] = -1;
    best[t] = kInf;
  }
}

// wave 0 of every region: its lowest cell, at the region's number
__global__ void __launch_bounds__(kBlock) k_cc_starts(const int32_t* __restrict__ tri, int64_t nt,
                                                      const int32_t* __restrict__ parent,
                                                      const uint32_t* __restrict__ cmin,
                                                      const unsigned long long* __restrict__ regno, int32_t* seq,
                                                      int32_t* reg, unsigned long long* best) {
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    if (cmin[parent[tri[3 * t]]] != (uint32_t)t) continue;
    const int32_t r = (int32_t)regno[t];
    seq[r] = (int32_t)t;
    reg[t] = r;
    best[t] = 0;
  }
}

__global__ void __launch_bounds__(kBlock) k_conn_reset(int32_t* reg, unsigned long long* best, int64_t nt) {
  for (int64_t t = gtid(); t < nt; t += gstride()) { reg[t] = -1; best[t] = kInf; }
}

// ---- the waves: TraverseAndMark's enumeration for waves.cuh -----------------------------------------------
// An item is a cell of seq, or in the seed wave a seed point; its entries are the link lists of its points,
// in point order j, then link order. A winner inherits the region of the item that claimed it.
struct ConnNb {
  const int32_t* tri;
  const unsigned long long* lstart;
  const int32_t* links;
  const int64_t* seeds;
  const int32_t* seq;
  int32_t* reg;

  __device__ __forceinline__ int points(const State& st, int64_t i, int32_t pts[3]) const {
    if (st.seed) {
      const int64_t s = seeds[i];
      pts[0] = (int32_t)s;
      return s >= 0 ? 1 : 0;
    }
    const int32_t c = seq[st.cur + i];
    pts[0] = tri[3 * c]; pts[1] = tri[3 * c + 1]; pts[2] = tri[3 * c + 2];
    return 3;
  }
  __device__ __forceinline__ unsigned long long count(const State& st, int64_t i) const {
    int32_t pts[3];
    const int np = points(st, i, pts);
    unsigned long long c = 0;
    for (int j = 0; j < np; ++j) c += lstart[pts[j] + 1] - lstart[pts[j]];
    return c;
  }
  template <class F>
  __device__ __forceinline__ void each(const State& st, int64_t i, F f) const {
    int32_t pts[3];
    const int np = points(st, i, pts);
    for (int j = 0; j < np; ++j)
      for (unsigned long long k = lstart[pts[j]]; k < lstart[pts[j] + 1]; ++k) f(links[k], j);
  }
  __device__ __forceinline__ void win(const State& st, int64_t i, int, int32_t d) const {
    reg[d] = st.seed ? 0 : reg[seq[st.cur + i]];
  }
};

// ---- ranks, PointMap, faces --------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_conn_sizes(const int32_t* __restrict__ seq, int64_t n,
                                                       const int32_t* __restrict__ reg, unsigned long long* cnt,
                                                       uint32_t* ka, uint32_t* va) {
  for (int64_t g = gtid(); g < n; g += gstride()) {
    const int32_t c = seq[g], r = reg[c];
    atomicAdd(&cnt[r], 1ull);
    ka[g] = (uint32_t)r;
    va[g] = (uint32_t)c;
  }
}

// the largest region: the highest size, ties to the lowest number
__global__ void __launch_bounds__(kBlock) k_conn_largest(const unsigned long long* __restrict__ size, int64_t nr,
                                                         unsigned long long* best) {
  for (int64_t r = gtid(); r < nr; r += gstride()) atomicMax(best, (size[r] << 32) | (0xffffffffull - (uint64_t)r));
}

__global__ void __launch_bounds__(kBlock) k_conn_first_use(const int32_t* __restrict__ rank, int64_t n,
                                                           const int32_t* __restrict__ tri, unsigned long long* fu) {
  for (int64_t k = gtid(); k < n; k += gstride()) {
    const int32_t c = rank[k];
    for (int j = 0; j < 3; ++j) atomicMin(&fu[tri[3 * c + j]], (unsigned long long)(3 * k + j));
  }
}

__global__ void __launch_bounds__(kBlock) k_conn_flags(const int32_t* __restrict__ rank, int64_t n,
                                                       const int32_t* __restrict__ tri,
                                                       const unsigned long long* __restrict__ fu,
                                                       unsigned long long* cflag) {
  for (int64_t k = gtid(); k < n; k += gstride()) {
    const int32_t c = rank[k];
    for (int j = 0; j < 3; ++j) cflag[3 * k + j] = fu[tri[3 * c + j]] == (unsigned long long)(3 * k + j);
  }
}

__global__ void __launch_bounds__(kBlock) k_conn_pointmap(const int32_t* __restrict__ rank, int64_t n,
                                                          const int32_t* __restrict__ tri,
                                                          const unsigned long long* __restrict__ fu,
                                                          const unsigned long long* __restrict__ cnum, int32_t* pmap,
                                                          int32_t* inv) {
  for (int64_t k = gtid(); k < n; k += gstride()) {
    const int32_t c = rank[k];
    for (int j = 0; j < 3; ++j) {
      const int32_t p = tri[3 * c + j];
      if (fu[p] != (unsigned long long)(3 * k + j)) continue;
      const int32_t m = (int32_t)cnum[3 * k + j];
      pmap[p] = m;
      inv[m] = p;
    }
  }
}

// point offsets of the regions: the first-use count before each region's first rank
__global__ void __launch_bounds__(kBlock) k_conn_ptoff(const unsigned long long* __restrict__ celloff, int64_t nr,
                                                       const unsigned long long* __restrict__ cnum,
                                                       unsigned long long* ptoff) {
  for (int64_t r = gtid(); r <= nr; r += gstride()) ptoff[r] = cnum[3 * celloff[r]];
}

__global__ void __launch_bounds__(kBlock) k_conn_visited(const int32_t* __restrict__ reg, int64_t nt,
                                                         unsigned long long* flag) {
  for (int64_t t = gtid(); t < nt; t += gstride()) flag[t] = reg[t] >= 0;
}

__global__ void __launch_bounds__(kBlock) k_conn_compact(const int32_t* __restrict__ reg, int64_t nt,
                                                         const unsigned long long* __restrict__ idx, uint32_t* ka,
                                                         uint32_t* va) {
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    if (reg[t] < 0) continue;
    ka[idx[t]] = (uint32_t)reg[t];
    va[idx[t]] = (uint32_t)t;
  }
}

__global__ void __launch_bounds__(kBlock) k_conn_emit_faces(const int32_t* __restrict__ cells, int64_t n,
                                                            const int32_t* __restrict__ tri,
                                                            const int32_t* __restrict__ pmap, int32_t* faces_out,
                                                            int32_t* cell_ids) {
  for (int64_t i = gtid(); i < n; i += gstride()) {
    const int32_t c = cells[i];
    cell_ids[i] = c;
    for (int j = 0; j < 3; ++j) faces_out[3 * i + j] = pmap[tri[3 * c + j]];
  }
}

__global__ void __launch_bounds__(kBlock) k_conn_emit_points(const float* __restrict__ verts,
                                                             const int32_t* __restrict__ inv, int64_t n,
                                                             float* verts_out, int32_t* point_ids) {
  for (int64_t m = gtid(); m < n; m += gstride()) {
    const int32_t p = inv[m];
    point_ids[m] = p;
    verts_out[3 * m] = verts[3 * (int64_t)p];
    verts_out[3 * m + 1] = verts[3 * (int64_t)p + 1];
    verts_out[3 * m + 2] = verts[3 * (int64_t)p + 2];
  }
}

__global__ void k_conn_offsets(const unsigned long long* __restrict__ celloff,
                               const unsigned long long* __restrict__ ptoff, int64_t nr, int64_t* cell_off,
                               int64_t* point_off) {
  for (int64_t r = gtid(); r <= nr; r += gstride()) {
    cell_off[r] = (int64_t)celloff[r];
    point_off[r] = (int64_t)ptoff[r];
  }
}

int check_args(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
               int64_t nseeds, const char* what) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL && nt >= 0 && nt <= 0x7fffffffLL, B2V_ERR_ARG,
              "%s: need V < 2^31 and T < 2^31", what);
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "%s: faces must be [T,3] or [T,4]", what);
  B2V_REQUIRE(faces_i64 == 0 || faces_i64 == 1, B2V_ERR_ARG, "%s: faces_i64 must be 0 or 1", what);
  B2V_REQUIRE(nt == 0 || nv > 0, B2V_ERR_ARG, "%s: faces without vertices", what);
  B2V_REQUIRE((nv == 0 || verts) && (nt == 0 || faces), B2V_ERR_ARG, "%s: null device pointer", what);
  B2V_REQUIRE(nseeds >= 0, B2V_ERR_ARG, "%s: negative seed count", what);
  return B2V_OK;
}

}  // namespace

extern "C" int64_t b2v_conn_workspace_bytes(int64_t nv, int64_t nt, int64_t nseeds) {
  if (nv < 0 || nt < 0 || nseeds < 0) return -1;
  return (int64_t)carve(nullptr, nv, nt, nseeds).bytes;
}

extern "C" int b2v_conn_layout(int64_t nv, int64_t nt, int64_t nseeds, int64_t* layout_out) {
  B2V_REQUIRE(nv >= 0 && nt >= 0 && nseeds >= 0 && layout_out, B2V_ERR_ARG, "conn_layout: bad arguments");
  const ConnWs w = carve(nullptr, nv, nt, nseeds);
  layout_out[0] = (int64_t)((char*)w.reg - (char*)nullptr);    // int32 [T]: region of each cell, -1 unvisited
  layout_out[1] = (int64_t)((char*)w.pmap - (char*)nullptr);   // int32 [V]: PointMap, -1 unnumbered
  layout_out[2] = (int64_t)((char*)w.seq - (char*)nullptr);    // int32 [C]: visited cells in wave order
  layout_out[3] = (int64_t)((char*)w.rank - (char*)nullptr);   // int32 [C]: visited cells, region-major
  layout_out[4] = (int64_t)((char*)w.links - (char*)nullptr);  // int32 [3T]: point -> cell links
  layout_out[5] = (int64_t)((char*)w.lstart - (char*)nullptr); // uint64 [V + 1]: their offsets
  return B2V_OK;
}

extern "C" int b2v_conn_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                              int faces_i64, int seeded, const int64_t* seeds_host, int64_t nseeds, void* workspace,
                              void* stream, int64_t* counts_host) {
  if (int rc = check_args(verts, nv, faces, nt, face_cols, faces_i64, seeded ? nseeds : 0, "conn_count")) return rc;
  B2V_REQUIRE(workspace && counts_host && (!seeded || nseeds == 0 || seeds_host), B2V_ERR_ARG,
              "conn_count: null argument");
  if (seeded)
    for (int64_t i = 0; i < nseeds; ++i)
      B2V_REQUIRE(seeds_host[i] < nv, B2V_ERR_ARG, "connectivity: seed %lld is not a point id (V = %lld)",
                  (long long)seeds_host[i], (long long)nv);
  if (!seeded) nseeds = 0;
  for (int k = 0; k < 4; ++k) counts_host[k] = 0;
  counts_host[4] = -1;
  if (seeded) counts_host[0] = 1;
  if (nt == 0) return B2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  ConnWs w = carve(workspace, nv, nt, nseeds);
  B2V_CUDA(cudaMemsetAsync(w.totals, 0, 64, s));

  // faces, link counts and offsets, the links themselves (corners stably sorted by point)
  const Faces F{faces, nt, face_cols, faces_i64, nv};
  if (int rc = build_links(w, F, "connectivity", s)) return rc;

  // wave 0 and the starting state
  long long st[6] = {0, 0, 1, 0, 0, 0};
  if (seeded) {
    k_conn_reset<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.reg, w.best, nt);
    if (int rc = b2v_check_launch("k_conn_reset")) return rc;
    if (nseeds) B2V_CUDA(cudaMemcpyAsync(w.seeds, seeds_host, (size_t)nseeds * 8, cudaMemcpyHostToDevice, s));
    st[0] = nseeds;
    st[5] = 1;
  } else {
    k_cc_init<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(w.parent, w.cmin, nv);
    if (int rc = b2v_check_launch("k_cc_init")) return rc;
    k_cc_hook<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.tri, nt, w.parent);
    if (int rc = b2v_check_launch("k_cc_hook")) return rc;
    k_cc_compress<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(w.parent, nv);
    if (int rc = b2v_check_launch("k_cc_compress")) return rc;
    k_cc_min<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.tri, nt, w.parent, w.cmin);
    if (int rc = b2v_check_launch("k_cc_min")) return rc;
    k_cc_flags<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.tri, nt, w.parent, w.cmin, w.tflag, w.reg, w.best);
    if (int rc = b2v_check_launch("k_cc_flags")) return rc;
    if (int rc = scan(w.tflag, nt, w.scratch, w.totals, s)) return rc;
    k_cc_starts<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.tri, nt, w.parent, w.cmin, w.tflag, w.seq, w.reg, w.best);
    if (int rc = b2v_check_launch("k_cc_starts")) return rc;
    unsigned long long nreg = 0;
    B2V_CUDA(cudaMemcpyAsync(&nreg, w.totals, 8, cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    st[0] = (long long)nreg;
    st[3] = nreg > 0;
    st[4] = (long long)nreg;
  }
  B2V_CUDA(cudaMemcpyAsync(w.ctl, st, sizeof(st), cudaMemcpyHostToDevice, s));

  // every wave of every region: one persistent cooperative launch
  const ConnNb E{w.tri, w.lstart, w.links, w.seeds, w.seq, w.reg};
  const WaveBufs B{w.seq, w.best, w.loc1, w.loc2, w.btot};
  if (int rc = launch_waves(E, B, w.ctl, s, "connectivity")) return rc;
  long long res[2] = {0, 0};
  B2V_CUDA(cudaMemcpyAsync(res, w.ctl + W_DEPTH, sizeof(res), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  const long long depth = res[0], ncells = res[1];
  const long long nreg = seeded ? 1 : st[0];

  // region sizes and offsets, the largest region, the region-major ranks
  B2V_CUDA(cudaMemsetAsync(w.celloff, 0, (size_t)(nreg + 1) * 8, s));
  B2V_CUDA(cudaMemsetAsync(w.fu, 0xff, (size_t)nv * 8, s));
  B2V_CUDA(cudaMemsetAsync(w.pmap, 0xff, (size_t)nv * 4, s));
  if (ncells > 0) {
    k_conn_sizes<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(w.seq, ncells, w.reg, w.celloff, w.ka, w.va);
    if (int rc = b2v_check_launch("k_conn_sizes")) return rc;
    k_conn_largest<<<b2v_grid(nreg, kBlock, 16), kBlock, 0, s>>>(w.celloff, nreg, w.totals + 1);
    if (int rc = b2v_check_launch("k_conn_largest")) return rc;
  }
  if (int rc = scan(w.celloff, nreg + 1, w.scratch, nullptr, s)) return rc;
  uint32_t* rv = nullptr;
  if (int rc = sort_pairs(w, ncells, bits_for(nreg - 1), &rv, s)) return rc;
  if (ncells > 0) {
    k_copy_i32<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(rv, ncells, w.rank);
    if (int rc = b2v_check_launch("k_copy_i32")) return rc;
    // PointMap: first use over (rank, j), numbered by a scan of the first-use flags
    k_conn_first_use<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(w.rank, ncells, w.tri, w.fu);
    if (int rc = b2v_check_launch("k_conn_first_use")) return rc;
    k_conn_flags<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(w.rank, ncells, w.tri, w.fu, w.cflag);
    if (int rc = b2v_check_launch("k_conn_flags")) return rc;
  }
  B2V_CUDA(cudaMemsetAsync(w.cflag + 3 * ncells, 0, 8, s));
  if (int rc = scan(w.cflag, 3 * ncells + 1, w.scratch, w.totals + 2, s)) return rc;
  if (ncells > 0) {
    k_conn_pointmap<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(w.rank, ncells, w.tri, w.fu, w.cflag, w.pmap,
                                                                    w.inv);
    if (int rc = b2v_check_launch("k_conn_pointmap")) return rc;
  }
  k_conn_ptoff<<<b2v_grid(nreg + 1, kBlock, 16), kBlock, 0, s>>>(w.celloff, nreg, w.cflag, w.ptoff);
  if (int rc = b2v_check_launch("k_conn_ptoff")) return rc;

  // the visited cells in ascending id, stably grouped by region
  k_conn_visited<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.reg, nt, w.tflag);
  if (int rc = b2v_check_launch("k_conn_visited")) return rc;
  if (int rc = scan(w.tflag, nt, w.scratch, nullptr, s)) return rc;
  k_conn_compact<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.reg, nt, w.tflag, w.ka, w.va);
  if (int rc = b2v_check_launch("k_conn_compact")) return rc;
  uint32_t* cv = nullptr;
  if (int rc = sort_pairs(w, ncells, bits_for(nreg - 1), &cv, s)) return rc;
  if (ncells > 0) {
    k_copy_i32<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(cv, ncells, w.cells);
    if (int rc = b2v_check_launch("k_copy_i32")) return rc;
  }

  unsigned long long tot[3] = {0, 0, 0};
  B2V_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  counts_host[0] = nreg;
  counts_host[1] = (int64_t)tot[2];
  counts_host[2] = ncells;
  counts_host[3] = depth;
  counts_host[4] = ncells > 0 ? (int64_t)(0xffffffffull - (tot[1] & 0xffffffffull)) : -1;
  return B2V_OK;
}

extern "C" int b2v_conn_emit(const float* verts, int64_t nv, int64_t nt, int64_t nseeds, const int64_t* counts_host,
                             void* workspace, float* verts_out, int32_t* point_ids, int32_t* faces_out,
                             int32_t* cell_ids, int64_t* point_offsets, int64_t* cell_offsets, void* stream) {
  B2V_REQUIRE(nv >= 0 && nt >= 0 && nseeds >= 0 && counts_host && workspace, B2V_ERR_ARG, "conn_emit: bad arguments");
  const int64_t nreg = counts_host[0], npts = counts_host[1], ncells = counts_host[2];
  B2V_REQUIRE(nreg >= 0 && nreg <= (nt > 1 ? nt : 1) && npts >= 0 && npts <= nv && ncells >= 0 && ncells <= nt,
              B2V_ERR_ARG, "conn_emit: counts do not come from b2v_conn_count on this mesh");
  B2V_REQUIRE((npts == 0 || (verts && verts_out && point_ids)) && (ncells == 0 || (faces_out && cell_ids)) &&
                  (point_offsets && cell_offsets),
              B2V_ERR_ARG, "conn_emit: null output");
  cudaStream_t s = (cudaStream_t)stream;
  if (nt == 0) {
    B2V_CUDA(cudaMemsetAsync(point_offsets, 0, (size_t)(nreg + 1) * 8, s));
    B2V_CUDA(cudaMemsetAsync(cell_offsets, 0, (size_t)(nreg + 1) * 8, s));
    return B2V_OK;
  }
  const ConnWs w = carve(workspace, nv, nt, nseeds);
  if (npts > 0) {
    k_conn_emit_points<<<b2v_grid(npts, kBlock, 16), kBlock, 0, s>>>(verts, w.inv, npts, verts_out, point_ids);
    if (int rc = b2v_check_launch("k_conn_emit_points")) return rc;
  }
  if (ncells > 0) {
    k_conn_emit_faces<<<b2v_grid(ncells, kBlock, 16), kBlock, 0, s>>>(w.cells, ncells, w.tri, w.pmap, faces_out,
                                                                      cell_ids);
    if (int rc = b2v_check_launch("k_conn_emit_faces")) return rc;
  }
  k_conn_offsets<<<b2v_grid(nreg + 1, kBlock, 16), kBlock, 0, s>>>(w.celloff, w.ptoff, nreg, cell_offsets,
                                                                   point_offsets);
  return b2v_check_launch("k_conn_offsets");
}
