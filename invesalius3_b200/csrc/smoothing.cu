// Laplacian surface smoothing on the device: vtkSmoothPolyDataFilter on triangles, as InVesalius's "Smooth
// surface" (polydata_utils.py:85-107), decimate_polydata (surface.py:1162-1203) and the marker surface
// geometry (markers/surface_geometry.py:106-122) use it. The contract is restated once, in the C checker's
// header (smoothing.c, DESIGN.md §3 "Surface smoothing"). VTK moves the points in place, in ascending id
// (Gauss-Seidel); every step below reproduces that order exactly.
//
//   build_links      faces -> int32 [T][3] and the point -> cell links (mesh_links.cuh).
//   k_sm_edges       one thread per (cell, edge): GetCellEdgeNeighbors through p1's links, the edge's type
//                    (simple, boundary, feature, or skipped as already visited), and the two events it
//                    sends: p1's (with p2 as the other end), then p2's (with p1).
//   sort by point    the events, keyed by point and numbered (cell, edge, p1 before p2), stably sorted by
//                    point: each point's events in VTK's sweep order.
//   k_sm_state       one thread per point runs VTK's per-vertex state machine over its own events, then the
//                    post-pass (boundary smoothing, list length, edge angle). The edge list is kept in the
//                    point's slice of the event array.
//   k_sm_pairs       the dependency graph: an edge lo -> hi for every list entry between two movable points.
//   k_sm_levels      levels by Kahn's peeling in one persistent cooperative launch: a point's level is one
//                    more than the deepest of its lower-id dependencies, i.e. the longest path to it.
//   k_sm_sweep       every iteration runs the levels in order, one barrier apart, moving the points in place.
//                    A point reads its lower-id list entries after they moved (lower level, earlier step)
//                    and its higher-id ones before they move (higher level, later step); two points of one
//                    level never read each other. That is exactly the sequential order. The largest move
//                    of an iteration is reduced before the next one starts, so VTK's early stop is exact.
//
// Runs of levels of at most kSmallLevels / kSmallSweep points run in block 0 alone, with block barriers.
// A call synchronises the host three times: the face check in build_links, the analysis' counts and
// bounds, and the run's iteration count.
#include <cooperative_groups.h>
#include <math.h>
#include <string.h>

#include "b2v_common.cuh"
#include "mesh_links.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int64_t kSmallLevels = 2048;             // peeling rounds this small run in one block
constexpr int64_t kSmallSweep = 512;               // sweep levels this small run in one block
enum : uint8_t { SIMPLE = 0, FIXED = 1, FEATURE = 2, BOUNDARY = 3, SKIPPED = 255 };   // VTK's vertex codes

struct SmWs {
  long long* ctl;                  // [32]: counters, hand-over record, results
  uint32_t* status;
  int32_t* tri;                    // [T][3]
  unsigned long long* lstart;      // [V + 1] link offsets
  int32_t* links;                  // [3T]
  uint32_t *ka, *va, *kb, *vb;     // [6T] sort ping-pong
  unsigned long long* hist;        // [256 * nb6 + 1]
  unsigned long long* scratch;     // scan block sums
  uint8_t* etype;                  // [3T] edge type per (cell, edge)
  unsigned long long* evstart;     // [V + 1] event offsets; a point's edge list is the head of its slice
  int32_t* lists;                  // [6T]
  int32_t* nlist;                  // [V]
  int8_t* types;                   // [V]
  uint32_t* bounds;                // [6] order-preserving encodings of the used points' bounds
  unsigned long long* sstart;      // [V + 1] dependency (successor) offsets
  unsigned long long* scur;        // [V]
  int32_t* indeg;                  // [V]
  int32_t* succ;                   // [6T]
  int32_t* order;                  // [V] movable points, level by level
  unsigned long long* loff;        // [V + 1] level offsets
  unsigned long long* lcnt;        // [V + 2] points per level, appended while the level before is expanded
  size_t bytes;
};

SmWs carve(void* base, int64_t nv, int64_t nt) {
  SmWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const size_t V = (size_t)nv, T = (size_t)nt, C3 = 3 * T, C6 = 6 * T;
  const int64_t nb6 = ceil_div64((int64_t)(C6 > 0 ? C6 : 1), kBlock);
  const int64_t hist_n = 256 * nb6 + 1;
  const int64_t longest = hist_n > (int64_t)V + 1 ? hist_n : (int64_t)V + 1;
  w.ctl = (long long*)take(32 * 8);
  w.status = (uint32_t*)take(16);
  w.tri = (int32_t*)take(C3 * 4);
  w.lstart = (unsigned long long*)take((V + 1) * 8);
  w.links = (int32_t*)take(C3 * 4);
  w.ka = (uint32_t*)take(C6 * 4);
  w.va = (uint32_t*)take(C6 * 4);
  w.kb = (uint32_t*)take(C6 * 4);
  w.vb = (uint32_t*)take(C6 * 4);
  w.hist = (unsigned long long*)take((size_t)hist_n * 8);
  w.scratch = (unsigned long long*)take((size_t)(scan_blocks(longest) + 1) * 8);
  w.etype = (uint8_t*)take(C3);
  w.evstart = (unsigned long long*)take((V + 1) * 8);
  w.lists = (int32_t*)take(C6 * 4);
  w.nlist = (int32_t*)take(V * 4);
  w.types = (int8_t*)take(V);
  w.bounds = (uint32_t*)take(6 * 4);
  w.sstart = (unsigned long long*)take((V + 1) * 8);
  w.scur = (unsigned long long*)take(V * 8);
  w.indeg = (int32_t*)take(V * 4);
  w.succ = (int32_t*)take(C6 * 4);
  w.order = (int32_t*)take(V * 4);
  w.loff = (unsigned long long*)take((V + 1) * 8);
  w.lcnt = (unsigned long long*)take((V + 2) * 8);
  w.bytes = o;
  return w;
}

// ctl words
enum { C_NLEV = 0,      // levels
       C_LBAR = 1,      // grid barriers of the peeling
       C_MOV = 2,       // movable points
       C_MD = 3,        // [3, 6): largest squared move of an iteration, a ring of three (double bits)
       C_ITERS = 6,     // iterations done
       C_SBAR = 7 };    // grid barriers of the sweep

// ---- topology ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void load3(const float* P, int32_t p, double x[3]) {
  x[0] = (double)P[3 * (int64_t)p]; x[1] = (double)P[3 * (int64_t)p + 1]; x[2] = (double)P[3 * (int64_t)p + 2];
}

// vtkPolygon::ComputeNormal of a triangle (vtkTriangle::ComputeNormal)
__device__ void tri_normal(const float* P, const int32_t* t, double n[3]) {
  double v1[3], v2[3], v3[3];
  load3(P, t[0], v1); load3(P, t[1], v2); load3(P, t[2], v3);
  const double ax = v3[0] - v2[0], ay = v3[1] - v2[1], az = v3[2] - v2[2];
  const double bx = v1[0] - v2[0], by = v1[1] - v2[1], bz = v1[2] - v2[2];
  n[0] = ay * bz - az * by;
  n[1] = az * bx - ax * bz;
  n[2] = ax * by - ay * bx;
  const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  if (len != 0.0) { n[0] /= len; n[1] /= len; n[2] /= len; }
}

__global__ void __launch_bounds__(kBlock) k_sm_edges(const float* __restrict__ P, const int32_t* __restrict__ tri,
                                                     const unsigned long long* __restrict__ lstart,
                                                     const int32_t* __restrict__ links, int64_t nt, int64_t nv,
                                                     int feature_smoothing, double cos_feature, uint8_t* etype,
                                                     unsigned long long* evdeg, uint32_t* ka, uint32_t* va) {
  for (int64_t q = gtid(); q < 3 * nt; q += gstride()) {
    const int64_t c = q / 3;
    const int i = (int)(q - 3 * c);
    const int32_t p1 = tri[q], p2 = tri[3 * c + (i + 1) % 3];
    int64_t lowest = INT64_MAX, nei = -1;
    const int64_t num = edge_neighbors(tri, lstart, links, c, p1, p2, &nei, &lowest);
    uint8_t e = SIMPLE;
    if (num == 0) {
      e = BOUNDARY;
    } else if (num >= 2) {
      if (lowest > c) e = FEATURE;
    } else if (nei > c) {
      if (feature_smoothing) {
        double n[3], m[3];
        tri_normal(P, tri + 3 * c, n);
        tri_normal(P, tri + 3 * nei, m);
        if (n[0] * m[0] + n[1] * m[1] + n[2] * m[2] <= cos_feature) e = FEATURE;
      }
    } else {
      e = SKIPPED;
    }
    etype[q] = e;
    const bool sent = e != SKIPPED;
    if (sent) { atomicAdd(&evdeg[p1], 1ull); atomicAdd(&evdeg[p2], 1ull); }
    ka[2 * q] = sent ? (uint32_t)p1 : (uint32_t)nv;        // nv: no event, sorts last
    ka[2 * q + 1] = sent ? (uint32_t)p2 : (uint32_t)nv;
    va[2 * q] = (uint32_t)(2 * q);
    va[2 * q + 1] = (uint32_t)(2 * q + 1);
  }
}

__device__ __forceinline__ uint32_t f2ord(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(kBlock) k_sm_state(const float* __restrict__ P, const int32_t* __restrict__ tri,
                                                     const unsigned long long* __restrict__ lstart,
                                                     const uint8_t* __restrict__ etype,
                                                     const unsigned long long* __restrict__ evstart,
                                                     const uint32_t* __restrict__ ev, int64_t nv,
                                                     int boundary_smoothing, double cos_edge, int32_t* lists,
                                                     int32_t* nlist, int8_t* types, uint32_t* bounds) {
  for (int64_t v = gtid(); v < nv; v += gstride()) {
    const unsigned long long base = evstart[v], end = evstart[v + 1];
    uint8_t type = SIMPLE;
    int32_t n = 0;
    for (unsigned long long k = base; k < end; ++k) {
      const uint32_t s = ev[k];
      const int64_t q = s >> 1, c = q / 3;
      const int i = (int)(q - 3 * c);
      const int32_t other = (s & 1u) ? tri[q] : tri[3 * c + (i + 1) % 3];
      const uint8_t e = etype[q];
      if (e != SIMPLE && type == SIMPLE) {
        lists[base] = other;
        n = 1;
        type = e;
      } else if ((e != SIMPLE && (type == BOUNDARY || type == FEATURE)) || (e == SIMPLE && type == SIMPLE)) {
        lists[base + n++] = other;
        if (type != SIMPLE && n > 2) type = FIXED;
      }
    }
    if (type == FEATURE || type == BOUNDARY) {
      if (!boundary_smoothing && type == BOUNDARY) {
        type = FIXED;
      } else if (n != 2) {
        type = FIXED;
      } else {
        double x1[3], x2[3], x3[3], l1[3], l2[3];
        load3(P, lists[base], x1); load3(P, (int32_t)v, x2); load3(P, lists[base + 1], x3);
        for (int k = 0; k < 3; ++k) { l1[k] = x2[k] - x1[k]; l2[k] = x3[k] - x2[k]; }
        const double d1 = sqrt(l1[0] * l1[0] + l1[1] * l1[1] + l1[2] * l1[2]);
        if (d1 != 0.0) for (int k = 0; k < 3; ++k) l1[k] /= d1;
        const double d2 = sqrt(l2[0] * l2[0] + l2[1] * l2[1] + l2[2] * l2[2]);
        if (d2 != 0.0) for (int k = 0; k < 3; ++k) l2[k] /= d2;
        if (d1 >= 0.0 && d2 >= 0.0 && l1[0] * l2[0] + l1[1] * l2[1] + l1[2] * l2[2] < cos_edge) type = FIXED;
      }
    }
    types[v] = (int8_t)type;
    nlist[v] = n;
    if (lstart[v + 1] > lstart[v])   // a point some cell uses: it counts towards the bounds
      for (int a = 0; a < 3; ++a) {
        const uint32_t o = f2ord(P[3 * v + a]);
        atomicMin(&bounds[2 * a], o);
        atomicMax(&bounds[2 * a + 1], o);
      }
  }
}

__device__ __forceinline__ bool movable(const int8_t* types, const int32_t* nlist, int32_t p) {
  return types[p] != FIXED && nlist[p] > 0;
}

// pass 0 counts the dependencies (lo -> hi) of every movable pair; pass 1 writes them
template <int kPass>
__global__ void __launch_bounds__(kBlock) k_sm_pairs(const unsigned long long* __restrict__ evstart,
                                                     const int32_t* __restrict__ lists,
                                                     const int32_t* __restrict__ nlist,
                                                     const int8_t* __restrict__ types, int64_t nv,
                                                     unsigned long long* sdeg, int32_t* indeg,
                                                     const unsigned long long* __restrict__ sstart, int32_t* succ) {
  for (int64_t v = gtid(); v < nv; v += gstride()) {
    if (!movable(types, nlist, (int32_t)v)) continue;
    const int32_t* L = lists + evstart[v];
    for (int k = 0; k < nlist[v]; ++k) {
      const int32_t j = L[k];
      if (j == v || !movable(types, nlist, j)) continue;
      const int32_t lo = j < v ? j : (int32_t)v, hi = j < v ? (int32_t)v : j;
      if (kPass == 0) {
        atomicAdd(&sdeg[lo], 1ull);
        atomicAdd(&indeg[hi], 1);
      } else {
        succ[sstart[lo] + atomicAdd(&sdeg[lo], 1ull)] = hi;
      }
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_sm_roots(const int32_t* __restrict__ nlist,
                                                     const int8_t* __restrict__ types,
                                                     const int32_t* __restrict__ indeg, int64_t nv, int32_t* order,
                                                     unsigned long long* cnt) {
  for (int64_t v = gtid(); v < nv; v += gstride())
    if (movable(types, nlist, (int32_t)v) && indeg[v] == 0) order[atomicAdd(cnt, 1ull)] = (int32_t)v;
}

// ---- levels -------------------------------------------------------------------------------------------------
struct Pk {
  const unsigned long long* sstart;
  const int32_t* succ;
  int32_t* indeg;
  int32_t* order;
  unsigned long long* loff;
  unsigned long long* lcnt;
  unsigned long long* ctl;
};

// expands level lev = order[b, e): a successor whose last dependency this is joins level lev + 1
__device__ __forceinline__ void expand(const Pk& K, unsigned long long b, unsigned long long e, long long lev,
                                       long long tid, long long nthreads) {
  if (tid == 0) K.loff[lev] = b;
  unsigned long long* cnt = K.lcnt + lev + 1;
  for (unsigned long long i = b + tid; i < e; i += nthreads) {
    const int32_t v = K.order[i];
    for (unsigned long long k = K.sstart[v]; k < K.sstart[v + 1]; ++k) {
      const int32_t w = K.succ[k];
      if (atomicSub(&K.indeg[w], 1) == 1) K.order[e + atomicAdd(cnt, 1ull)] = w;
    }
  }
}

__device__ __forceinline__ unsigned long long read_cnt(const Pk& K, long long lev) {
  return ((volatile const unsigned long long*)K.lcnt)[lev];
}

// Ordering: lcnt is zeroed before the launch, lcnt[0] (the roots) is written by the kernel before, and lcnt[L]
// is only written while level L - 1 is expanded. So after the barrier that ends that expansion, lcnt[L] is
// final: no word is ever cleared or reused, and every block derives the same (begin, end, level) from the
// counts alone. After a single-block stretch the other blocks replay block 0's loop over the final counts;
// no hand-over record is needed.
__global__ void __launch_bounds__(kBlock) k_sm_levels(Pk K) {
  cg::grid_group g = cg::this_grid();
  unsigned long long b = 0, e = read_cnt(K, 0);
  long long lev = 0, bars = 0;
  while (e > b) {
    if (e - b <= kSmallLevels) {
      if (blockIdx.x == 0)
        do {
          expand(K, b, e, lev, threadIdx.x, blockDim.x);
          __syncthreads();
          const unsigned long long n = read_cnt(K, lev + 1);
          b = e; e += n; ++lev;
        } while (e > b && e - b <= kSmallLevels);
      g.sync();
      ++bars;
      if (blockIdx.x != 0)
        do {
          const unsigned long long n = read_cnt(K, lev + 1);
          b = e; e += n; ++lev;
        } while (e > b && e - b <= kSmallLevels);
      continue;
    }
    expand(K, b, e, lev, gtid(), gstride());
    g.sync();
    ++bars;
    const unsigned long long n = read_cnt(K, lev + 1);
    b = e; e += n; ++lev;
  }
  if (gtid() == 0) { K.loff[lev] = b; K.ctl[C_NLEV] = lev; K.ctl[C_LBAR] = bars; K.ctl[C_MOV] = b; }
}

// ---- the sweep ----------------------------------------------------------------------------------------------
struct Sw {
  float* P;                            // moved in place: never read through the non-coherent path
  const int32_t* order;
  const unsigned long long* loff;
  const unsigned long long* evstart;
  const int32_t* lists;
  const int32_t* nlist;
  unsigned long long* ctl;             // holds the level count from the analysis
  long long iterations;
  double relax;
  double conv;
};

// one point of the sweep, in VTK's arithmetic: double sums of (y - x) / n in list order, x + relax * d, the
// squared distance of the move, the result stored as float32
__device__ __forceinline__ void move_point(const Sw& S, int32_t v, double& dmax) {
  const int32_t n = S.nlist[v];
  const int32_t* L = S.lists + S.evstart[v];
  double x[3], d[3] = {0.0, 0.0, 0.0};
  load3(S.P, v, x);
  const double dn = (double)n;
  for (int k = 0; k < n; ++k) {
    double y[3];
    load3(S.P, L[k], y);
    for (int a = 0; a < 3; ++a) d[a] += (y[a] - x[a]) / dn;
  }
  double y[3];
  for (int a = 0; a < 3; ++a) y[a] = x[a] + S.relax * d[a];
  const double e0 = x[0] - y[0], e1 = x[1] - y[1], e2 = x[2] - y[2];
  const double dist = e0 * e0 + e1 * e1 + e2 * e2;
  if (dist > dmax) dmax = dist;
  for (int a = 0; a < 3; ++a) S.P[3 * (int64_t)v + a] = (float)y[a];
}

// With no level (nothing movable) every iteration measures no move: the first one stops the sweep, as in VTK.
__global__ void __launch_bounds__(kBlock, kMaxBlocksPerSm) k_sm_sweep(Sw S) {
  cg::grid_group g = cg::this_grid();
  const long long nlev = (long long)S.ctl[C_NLEV];
  long long t = 0, bars = 0;
  for (; t < S.iterations; ++t) {
    if (gtid() == 0) S.ctl[C_MD + (t + 1) % 3] = 0;   // last read two barriers ago
    double dmax = 0.0;
    long long r = 0;
    while (r < nlev) {
      if ((long long)(S.loff[r + 1] - S.loff[r]) <= kSmallSweep) {
        long long r2 = r;
        while (r2 < nlev && (long long)(S.loff[r2 + 1] - S.loff[r2]) <= kSmallSweep) ++r2;
        if (blockIdx.x == 0)
          for (; r < r2; ++r) {
            for (unsigned long long i = S.loff[r] + threadIdx.x; i < S.loff[r + 1]; i += blockDim.x)
              move_point(S, S.order[i], dmax);
            __syncthreads();
          }
        r = r2;
      } else {
        for (unsigned long long i = S.loff[r] + gtid(); i < S.loff[r + 1]; i += gstride())
          move_point(S, S.order[i], dmax);
        ++r;
      }
      if (r == nlev && dmax > 0.0) atomicMax(&S.ctl[C_MD + t % 3], (unsigned long long)__double_as_longlong(dmax));
      g.sync();
      ++bars;
    }
    const double md = __longlong_as_double((long long)((volatile unsigned long long*)S.ctl)[C_MD + t % 3]);
    if (!(sqrt(md) > S.conv)) { ++t; break; }
  }
  if (gtid() == 0) { S.ctl[C_ITERS] = t; S.ctl[C_SBAR] = bars; }
}

int check_sizes(int64_t nv, int64_t nt, const char* what) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL && nt >= 0 && nt <= 0x7fffffffLL / 3, B2V_ERR_ARG,
              "%s: need V < 2^31 and 6T < 2^32", what);
  return B2V_OK;
}

}  // namespace

extern "C" int64_t b2v_smooth_workspace_bytes(int64_t nv, int64_t nt) {
  if (nv < 0 || nt < 0) return -1;
  return (int64_t)carve(nullptr, nv, nt).bytes;
}

extern "C" int b2v_smooth_layout(int64_t nv, int64_t nt, int64_t* layout_out) {
  B2V_REQUIRE(nv >= 0 && nt >= 0 && layout_out, B2V_ERR_ARG, "smooth_layout: bad arguments");
  const SmWs w = carve(nullptr, nv, nt);
  layout_out[0] = (int64_t)((char*)w.types - (char*)nullptr);     // int8 [V]: VTK's vertex type
  layout_out[1] = (int64_t)((char*)w.nlist - (char*)nullptr);     // int32 [V]: edge list lengths
  layout_out[2] = (int64_t)((char*)w.evstart - (char*)nullptr);   // uint64 [V + 1]: where each list starts
  layout_out[3] = (int64_t)((char*)w.lists - (char*)nullptr);     // int32 [6T]: the lists
  layout_out[4] = (int64_t)((char*)w.order - (char*)nullptr);     // int32 [M]: movable points, level by level
  layout_out[5] = (int64_t)((char*)w.loff - (char*)nullptr);      // uint64 [levels + 1]: level offsets
  return B2V_OK;
}

extern "C" int b2v_smooth_analyse(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                                  int faces_i64, double cos_feature, double cos_edge, int feature_edge_smoothing,
                                  int boundary_smoothing, void* workspace, void* stream, double* bounds_host,
                                  int64_t* counts_host) {
  if (int rc = check_sizes(nv, nt, "smooth_analyse")) return rc;
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "smooth_analyse: faces must be [T,3] or [T,4]");
  B2V_REQUIRE(faces_i64 == 0 || faces_i64 == 1, B2V_ERR_ARG, "smooth_analyse: faces_i64 must be 0 or 1");
  B2V_REQUIRE(nt == 0 || nv > 0, B2V_ERR_ARG, "smooth_analyse: faces without vertices");
  B2V_REQUIRE((nv == 0 || verts) && (nt == 0 || faces) && workspace && bounds_host && counts_host, B2V_ERR_ARG,
              "smooth_analyse: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  SmWs w = carve(workspace, nv, nt);
  B2V_CUDA(cudaMemsetAsync(w.ctl, 0, 32 * 8, s));
  B2V_CUDA(cudaMemsetAsync(w.types, 0, (size_t)nv, s));
  B2V_CUDA(cudaMemsetAsync(w.nlist, 0, (size_t)nv * 4, s));
  B2V_CUDA(cudaMemsetAsync(w.evstart, 0, (size_t)(nv + 1) * 8, s));
  for (int k = 0; k < 6; ++k) bounds_host[k] = 0.0;
  counts_host[0] = counts_host[1] = counts_host[2] = 0;
  if (nt == 0) return B2V_OK;

  const Faces F{faces, nt, face_cols, faces_i64, nv};
  if (int rc = build_links(w, F, "smoothing", s)) return rc;

  // edges, events in sweep order per point, the state machine and post-pass
  const int64_t C6 = 6 * nt;
  k_sm_edges<<<b2v_grid(3 * nt, kBlock, 16), kBlock, 0, s>>>(verts, w.tri, w.lstart, w.links, nt, nv,
                                                             feature_edge_smoothing, cos_feature, w.etype,
                                                             w.evstart, w.ka, w.va);
  if (int rc = b2v_check_launch("k_sm_edges")) return rc;
  if (int rc = scan(w.evstart, nv + 1, w.scratch, nullptr, s)) return rc;
  uint32_t* ev = nullptr;
  if (int rc = sort_pairs(w, C6, bits_for(nv), &ev, s)) return rc;
  const uint32_t binit[6] = {~0u, 0u, ~0u, 0u, ~0u, 0u};
  B2V_CUDA(cudaMemcpyAsync(w.bounds, binit, sizeof(binit), cudaMemcpyHostToDevice, s));
  k_sm_state<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(verts, w.tri, w.lstart, w.etype, w.evstart, ev, nv,
                                                         boundary_smoothing, cos_edge, w.lists, w.nlist, w.types,
                                                         w.bounds);
  if (int rc = b2v_check_launch("k_sm_state")) return rc;

  // the dependency graph and its levels
  B2V_CUDA(cudaMemsetAsync(w.sstart, 0, (size_t)(nv + 1) * 8, s));
  B2V_CUDA(cudaMemsetAsync(w.indeg, 0, (size_t)nv * 4, s));
  B2V_CUDA(cudaMemsetAsync(w.scur, 0, (size_t)nv * 8, s));
  k_sm_pairs<0><<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(w.evstart, w.lists, w.nlist, w.types, nv, w.sstart,
                                                            w.indeg, nullptr, nullptr);
  if (int rc = b2v_check_launch("k_sm_pairs")) return rc;
  if (int rc = scan(w.sstart, nv + 1, w.scratch, nullptr, s)) return rc;
  k_sm_pairs<1><<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(w.evstart, w.lists, w.nlist, w.types, nv, w.scur,
                                                            nullptr, w.sstart, w.succ);
  if (int rc = b2v_check_launch("k_sm_pairs")) return rc;
  B2V_CUDA(cudaMemsetAsync(w.lcnt, 0, (size_t)(nv + 2) * 8, s));
  k_sm_roots<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(w.nlist, w.types, w.indeg, nv, w.order, w.lcnt);
  if (int rc = b2v_check_launch("k_sm_roots")) return rc;
  Pk K{w.sstart, w.succ, w.indeg, w.order, w.loff, w.lcnt, (unsigned long long*)w.ctl};
  void* args[] = {&K};
  if (int rc = launch_coop((const void*)k_sm_levels, args, s, "smoothing", "k_sm_levels")) return rc;

  long long ctl[3];
  uint32_t b[6];
  B2V_CUDA(cudaMemcpyAsync(ctl, w.ctl, sizeof(ctl), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(b, w.bounds, sizeof(b), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  for (int k = 0; k < 6; ++k) {
    const uint32_t o = b[k], u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    float f;
    memcpy(&f, &u, 4);
    bounds_host[k] = (double)f;
  }
  counts_host[0] = ctl[C_MOV];
  counts_host[1] = ctl[C_NLEV];
  counts_host[2] = ctl[C_LBAR];
  return B2V_OK;
}

extern "C" int b2v_smooth_run(const float* verts, int64_t nv, int64_t nt, int64_t iterations, double relaxation,
                              double conv, void* workspace, float* verts_out, void* stream, int64_t* counts_host) {
  if (int rc = check_sizes(nv, nt, "smooth_run")) return rc;
  B2V_REQUIRE(iterations >= 0, B2V_ERR_ARG, "smoothing: negative number of iterations");
  B2V_REQUIRE((nv == 0 || (verts && verts_out)) && workspace && counts_host, B2V_ERR_ARG,
              "smooth_run: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  counts_host[0] = counts_host[1] = counts_host[2] = 0;
  if (nv > 0)
    B2V_CUDA(cudaMemcpyAsync(verts_out, verts, (size_t)nv * 12, cudaMemcpyDeviceToDevice, s));
  if (iterations == 0 || relaxation == 0.0 || nt == 0) return B2V_OK;   // VTK passes the points through
  SmWs w = carve(workspace, nv, nt);
  Sw S{verts_out, w.order, w.loff, w.evstart, w.lists, w.nlist, (unsigned long long*)w.ctl, iterations,
       relaxation, conv};
  B2V_CUDA(cudaMemsetAsync(w.ctl + C_MD, 0, (C_SBAR + 1 - C_MD) * 8, s));
  void* args[] = {&S};
  if (int rc = launch_coop((const void*)k_sm_sweep, args, s, "smoothing", "k_sm_sweep")) return rc;
  long long ctl[C_SBAR + 1];
  B2V_CUDA(cudaMemcpyAsync(ctl, w.ctl, sizeof(ctl), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  counts_host[0] = ctl[C_ITERS];
  counts_host[1] = ctl[C_ITERS] * ctl[C_NLEV];
  counts_host[2] = ctl[C_SBAR];
  return B2V_OK;
}
