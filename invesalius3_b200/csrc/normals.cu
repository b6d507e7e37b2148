// Surface normals, volume and area on the device: vtkPolyDataNormals on triangles with consistency,
// splitting and non-manifold traversal on (every InVesalius caller: surface_process.py:272-280 and :419-436,
// surface.py, viewer_volume.py, brainmesh_handler.py), and vtkMassProperties' volume and area
// (surface_process.py:455-461). The contract is restated once, in the C checker's header (DESIGN.md §3
// "Surface normals"); every step below reproduces its sequential result bit for bit.
//
//   build_links        faces -> int32 [T][3] and the point -> cell links (mesh_links.cuh).
//   k_nm_hook          union-find over the cells across every edge (p1, p2) with p1 != p2: such an edge
//                      neighbour relation is symmetric, so the sets are the regions a traversal covers.
//   k_nm_cross         an edge (a, a) of a cell with a repeated point reaches every cell at a. When one reaches
//                      another set, where a traversal starts decides what it covers, and the regions are
//                      run one at a time in the checker's order (below); otherwise every set is a region
//                      and all of them run at once.
//   seeds              without auto_orient, each set's root (its lowest cell). With auto_orient, rounds of
//                      k_ao_first / k_ao_decide: each undecided set finds its first point in pop order (x,
//                      then id) where it has a cell with |n.x| > 0; a point is decided once every set with
//                      such a cell there has it as its first point, and its best cell seeds its set; the
//                      other sets go on from the next point. The smallest first point is always decided.
//   k_waves<NmNb>      TraverseAndOrder (waves.cuh): the entries of a cell are the edge neighbours of its
//                      current edges, and a winner is reversed unless it runs the shared edge backwards.
//   k_nm_cell_normals  the cell normals of the final order.
//   k_nm_split         one thread per point runs MarkAndSplit over its link slots; a scan of groups - 1
//                      numbers the new points in creation order.
//   k_nm_points / k_nm_faces  (emit) the points and their normals, summed through the links in ascending
//                      cell id; the corners rewritten to their group's point.
//   k_mp_*             per-triangle mass terms in parallel, then summed in cell order by one thread of one
//                      block from coalesced shared-memory tiles: the checker's sums bit for bit. A parallel
//                      tree differs from that sequential sum by more than 1e-12 relative on surfaces of
//                      millions of triangles (8e-12 on the 512^3 phantom's bone), so the order is kept.
//
// b2v_normals_count synchronises the host for the face check, the cross-set test, each auto-orient round
// and each region run one at a time. b2v_normals_emit does not synchronise.
#include <math.h>

#include "b2v_common.cuh"
#include "mesh_links.cuh"
#include "waves.cuh"

namespace {

struct NmWs {
  long long* ctl;                  // [W_CTL] the wave state
  unsigned long long* cnt;         // [16] counters
  uint32_t* status;
  int32_t* tri;                    // [T][3] input order
  unsigned long long* lstart;      // [V + 1]
  int32_t* links;                  // [3T]
  uint32_t *ka, *va, *kb, *vb;     // [3T] sort ping-pong
  unsigned long long* hist;
  unsigned long long* scratch;
  int32_t* parent;                 // [T] union-find over cells
  unsigned long long* best;        // [T] wave claims
  int32_t* seq;                    // [T] cells in wave order
  unsigned long long *loc1, *loc2; // [T]
  unsigned long long* btot;        // [2 kMaxGrid]
  uint8_t* fl;                     // [T] 1: reversed
  unsigned long long* tflag;       // [T + 1] seed flags, scanned
  unsigned long long* lb;          // [T] auto-orient: per set, the first point key still open
  unsigned long long* gk;          // [T]                    its first candidate point key this round
  int32_t* stt;                    // [T]                    -1 undecided, -2 never seeded, else its seed
  int32_t* res;                    // [T]                    this round's decision
  float* cn;                       // [T][3] cell normals
  int32_t* grp;                    // [3T] group of each link slot at its point
  int32_t* ngrp;                   // [V] groups per point (0: unused point)
  unsigned long long* noff;        // [V + 1] new points before each point's
  double* terms;                   // [T][4] mass: area, x, y, z volume terms
  int8_t* cls;                     // [T] mass: normal class
  double* part;                    // [4] mass: the sums
  unsigned long long* ccount;      // [8] class counts
  size_t bytes;
};

NmWs carve(void* base, int64_t nv, int64_t nt) {
  NmWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const size_t V = (size_t)nv, T = (size_t)nt, C3 = 3 * T;
  const int64_t nb3 = ceil_div64((int64_t)(C3 > 0 ? C3 : 1), kBlock);
  const int64_t hist_n = 256 * nb3 + 1;
  int64_t longest = hist_n;
  if ((int64_t)T + 1 > longest) longest = (int64_t)T + 1;
  if ((int64_t)V + 1 > longest) longest = (int64_t)V + 1;
  w.ctl = (long long*)take(W_CTL * 8);
  w.cnt = (unsigned long long*)take(16 * 8);
  w.status = (uint32_t*)take(16);
  w.tri = (int32_t*)take(C3 * 4);
  w.lstart = (unsigned long long*)take((V + 1) * 8);
  w.links = (int32_t*)take(C3 * 4);
  w.ka = (uint32_t*)take(C3 * 4);
  w.va = (uint32_t*)take(C3 * 4);
  w.kb = (uint32_t*)take(C3 * 4);
  w.vb = (uint32_t*)take(C3 * 4);
  w.hist = (unsigned long long*)take((size_t)hist_n * 8);
  w.scratch = (unsigned long long*)take((size_t)(scan_blocks(longest) + 1) * 8);
  w.parent = (int32_t*)take(T * 4);
  w.best = (unsigned long long*)take(T * 8);
  w.seq = (int32_t*)take(T * 4);
  w.loc1 = (unsigned long long*)take(T * 8);
  w.loc2 = (unsigned long long*)take(T * 8);
  w.btot = (unsigned long long*)take(2 * kMaxGrid * 8);
  w.fl = (uint8_t*)take(T);
  w.tflag = (unsigned long long*)take((T + 1) * 8);
  w.lb = (unsigned long long*)take(T * 8);
  w.gk = (unsigned long long*)take(T * 8);
  w.stt = (int32_t*)take(T * 4);
  w.res = (int32_t*)take(T * 4);
  w.cn = (float*)take(T * 12);
  w.grp = (int32_t*)take(C3 * 4);
  w.ngrp = (int32_t*)take(V * 4);
  w.noff = (unsigned long long*)take((V + 1) * 8);
  w.terms = (double*)take(T * 32);
  w.cls = (int8_t*)take(T);
  w.part = (double*)take(4 * 8);
  w.ccount = (unsigned long long*)take(8 * 8);
  w.bytes = o;
  return w;
}

// cnt words
enum { C_CROSS = 0,     // a cell's (a, a) edge reaches another set
       C_PENDING = 1,   // auto-orient: sets still undecided after a round
       C_FLIPS = 2,     // reversed cells
       C_NEW = 3,       // new points
       C_NEXT = 4,      // one at a time: the next seed's key (cell id, or point key)
       C_FOUND = 5 };   // one at a time: 1 when a region was seeded

// ---- geometry ------------------------------------------------------------------------------------------
// vtkTriangle::ComputeNormal in double of corners (a, b, c): (c - b) x (a - b), normalised when non-zero
__device__ __forceinline__ void tri_normal(const float* P, int32_t a, int32_t b, int32_t c, double n[3]) {
  double v1[3], v2[3], v3[3];
  for (int k = 0; k < 3; ++k) {
    v1[k] = (double)P[3 * (int64_t)a + k];
    v2[k] = (double)P[3 * (int64_t)b + k];
    v3[k] = (double)P[3 * (int64_t)c + k];
  }
  const double ax = v3[0] - v2[0], ay = v3[1] - v2[1], az = v3[2] - v2[2];
  const double bx = v1[0] - v2[0], by = v1[1] - v2[1], bz = v1[2] - v2[2];
  n[0] = ay * bz - az * by;
  n[1] = az * bx - ax * bz;
  n[2] = ax * by - ay * bx;
  const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  if (len != 0.0) { n[0] /= len; n[1] /= len; n[2] /= len; }
}

// x of the normal of cell c in its input order
__device__ __forceinline__ double normal_x(const float* P, const int32_t* tri, int64_t c) {
  double n[3];
  tri_normal(P, tri[3 * c], tri[3 * c + 1], tri[3 * c + 2], n);
  return n[0];
}

// pop order of the points: (x, id), -0 as +0, NaN after everything
__device__ __forceinline__ unsigned long long point_key(const float* P, int32_t p) {
  const float x = P[3 * (int64_t)p];
  uint32_t u = __float_as_uint(x == 0.0f ? 0.0f : x);
  u = x != x ? 0xffffffffu : ((u & 0x80000000u) ? ~u : (u | 0x80000000u));
  return ((unsigned long long)u << 32) | (uint32_t)p;
}

__device__ __forceinline__ bool has(const int32_t* t, int32_t p) { return t[0] == p || t[1] == p || t[2] == p; }

// a cell's corners in its current order
__device__ __forceinline__ void corners(const int32_t* tri, const uint8_t* fl, int64_t c, int32_t pts[3]) {
  const int32_t* t = tri + 3 * c;
  if (fl[c]) { pts[0] = t[2]; pts[1] = t[1]; pts[2] = t[0]; }
  else { pts[0] = t[0]; pts[1] = t[1]; pts[2] = t[2]; }
}

// ---- regions ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_nm_init(int32_t* parent, unsigned long long* best, uint8_t* fl,
                                                    int32_t* stt, unsigned long long* lb, int64_t nt) {
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    parent[t] = (int32_t)t;
    best[t] = kInf;
    fl[t] = 0;
    stt[t] = -1;
    lb[t] = 0;
  }
}

__global__ void __launch_bounds__(kBlock) k_nm_hook(const int32_t* __restrict__ tri,
                                                    const unsigned long long* __restrict__ lstart,
                                                    const int32_t* __restrict__ links, int64_t nt, int32_t* parent) {
  for (int64_t q = gtid(); q < 3 * nt; q += gstride()) {
    const int64_t c = q / 3;
    const int32_t p1 = tri[q], p2 = tri[3 * c + (q - 3 * c + 1) % 3];
    if (p1 == p2) continue;
    int64_t first = -1, lowest = INT64_MAX;
    if (edge_neighbors(tri, lstart, links, c, p1, p2, &first, &lowest)) uf_unite(parent, (int32_t)c, (int32_t)first);
  }
}

__global__ void __launch_bounds__(kBlock) k_nm_compress(int32_t* parent, int64_t nt) {
  for (int64_t t = gtid(); t < nt; t += gstride()) parent[t] = uf_find(parent, (int32_t)t);
}

__global__ void __launch_bounds__(kBlock) k_nm_cross(const int32_t* __restrict__ tri,
                                                     const unsigned long long* __restrict__ lstart,
                                                     const int32_t* __restrict__ links,
                                                     const int32_t* __restrict__ parent, int64_t nt,
                                                     unsigned long long* cnt) {
  for (int64_t q = gtid(); q < 3 * nt; q += gstride()) {
    const int64_t c = q / 3;
    const int32_t a = tri[q];
    if (a != tri[3 * c + (q - 3 * c + 1) % 3]) continue;
    for (unsigned long long k = lstart[a]; k < lstart[a + 1]; ++k)
      if (parent[links[k]] != parent[c]) { atomicOr(&cnt[C_CROSS], 1ull); break; }
  }
}

// every set at once: seed flags (roots, or decided auto-orient seeds), scanned into wave 0
__global__ void __launch_bounds__(kBlock) k_nm_seed_flags(const int32_t* __restrict__ parent,
                                                          const int32_t* __restrict__ stt, int auto_orient,
                                                          int64_t nt, unsigned long long* flag) {
  for (int64_t t = gtid(); t < nt; t += gstride())
    flag[t] = parent[t] == (int32_t)t && (!auto_orient || stt[t] >= 0);
}

__global__ void __launch_bounds__(kBlock) k_nm_seeds(const int32_t* __restrict__ parent,
                                                     const int32_t* __restrict__ stt, int auto_orient,
                                                     const unsigned long long* __restrict__ pos, int64_t nt,
                                                     int32_t* seq, unsigned long long* best) {
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    if (parent[t] != (int32_t)t || (auto_orient && stt[t] < 0)) continue;
    const int32_t s = auto_orient ? stt[t] : (int32_t)t;
    seq[pos[t]] = s;
    best[s] = 0;
  }
}

// auto-orient round, part 1: each undecided set's first candidate point at or after its bound
__global__ void __launch_bounds__(kBlock) k_ao_first(const float* __restrict__ P, const int32_t* __restrict__ tri,
                                                     const int32_t* __restrict__ parent,
                                                     const int32_t* __restrict__ stt,
                                                     const unsigned long long* __restrict__ lb, int64_t nt,
                                                     unsigned long long* gk) {
  for (int64_t c = gtid(); c < nt; c += gstride()) {
    const int32_t r = parent[c];
    if (stt[r] != -1 || !(fabs(normal_x(P, tri, c)) > 0.0)) continue;
    for (int j = 0; j < 3; ++j) {
      const unsigned long long k = point_key(P, tri[3 * c + j]);
      if (k >= lb[r]) atomicMin(&gk[r], k);
    }
  }
}

// part 2: per undecided set, its decision at that point: res -2 never seeded, -3 not decidable yet,
// -1 lost, else the seed (reversed when its normal's x is positive)
__global__ void __launch_bounds__(kBlock) k_ao_decide(const float* __restrict__ P, const int32_t* __restrict__ tri,
                                                      const unsigned long long* __restrict__ lstart,
                                                      const int32_t* __restrict__ links,
                                                      const int32_t* __restrict__ parent,
                                                      const int32_t* __restrict__ stt,
                                                      const unsigned long long* __restrict__ gk, int64_t nt,
                                                      int32_t* res, uint8_t* fl) {
  for (int64_t r = gtid(); r < nt; r += gstride()) {
    if (parent[r] != (int32_t)r || stt[r] != -1) continue;
    const unsigned long long key = gk[r];
    if (key == kInf) { res[r] = -2; continue; }
    const int32_t p = (int32_t)(key & 0xffffffffull);
    double bestx = 0.0, nx0 = 0.0;
    int32_t cell = -1, out = 0;
    for (unsigned long long k = lstart[p]; k < lstart[p + 1]; ++k) {
      const int32_t d = links[k];
      const double nx = normal_x(P, tri, d);
      if (!(fabs(nx) > 0.0)) continue;
      const int32_t q = parent[d];
      if (stt[q] >= 0) continue;                       // seeded in an earlier round: before this point
      if (gk[q] != key) { out = -3; break; }           // that set may still be seeded before this point
      if (fabs(nx) > bestx) { bestx = fabs(nx); cell = d; nx0 = nx; }
    }
    if (out == 0) out = parent[cell] == (int32_t)r ? cell : -1;
    if (out >= 0) fl[out] = nx0 > 0.0;
    res[r] = out;
  }
}

// part 3: apply the decisions; count the sets still open
__global__ void __launch_bounds__(kBlock) k_ao_apply(const int32_t* __restrict__ parent,
                                                     const int32_t* __restrict__ res,
                                                     const unsigned long long* __restrict__ gk, int64_t nt,
                                                     int32_t* stt, unsigned long long* lb, unsigned long long* cnt) {
  for (int64_t r = gtid(); r < nt; r += gstride()) {
    if (parent[r] != (int32_t)r || stt[r] != -1) continue;
    const int32_t d = res[r];
    if (d >= 0 || d == -2) { stt[r] = d; continue; }
    if (d == -1) lb[r] = gk[r] + 1;
    atomicAdd(&cnt[C_PENDING], 1ull);
  }
}

// one region at a time, part 1: the next seed's key over the unvisited cells
__global__ void __launch_bounds__(kBlock) k_nm_next(const float* __restrict__ P, const int32_t* __restrict__ tri,
                                                    const unsigned long long* __restrict__ best, int auto_orient,
                                                    unsigned long long after, int64_t nt, unsigned long long* cnt) {
  for (int64_t c = gtid(); c < nt; c += gstride()) {
    if (best[c] != kInf) continue;
    if (!auto_orient) { atomicMin(&cnt[C_NEXT], (unsigned long long)c); continue; }
    if (!(fabs(normal_x(P, tri, c)) > 0.0)) continue;
    for (int j = 0; j < 3; ++j) {
      const unsigned long long k = point_key(P, tri[3 * c + j]);
      if (k + 1 > after) atomicMin(&cnt[C_NEXT], k);
    }
  }
}

// part 2 (one thread): the seed, and the starting state of its traversal after ctl's last one
__global__ void k_nm_seed_one(const float* __restrict__ P, const int32_t* __restrict__ tri,
                              const unsigned long long* __restrict__ lstart, const int32_t* __restrict__ links,
                              int auto_orient, long long* ctl, unsigned long long* cnt, int32_t* seq,
                              unsigned long long* best, uint8_t* fl) {
  const unsigned long long key = cnt[C_NEXT];
  long long* st = ctl;
  const long long total = ctl[W_TOTAL], base = ctl[W_BASE];
  st[0] = 0;
  cnt[C_FOUND] = 0;
  if (key == kInf) return;
  int32_t cell = (int32_t)key;
  if (auto_orient) {
    const int32_t p = (int32_t)(key & 0xffffffffull);
    double bestx = 0.0, nx0 = 0.0;
    cell = -1;
    for (unsigned long long k = lstart[p]; k < lstart[p + 1]; ++k) {
      const int32_t d = links[k];
      if (best[d] != kInf) continue;
      const double nx = normal_x(P, tri, d);
      if (fabs(nx) > bestx) { bestx = fabs(nx); cell = d; nx0 = nx; }
    }
    fl[cell] = nx0 > 0.0;
  }
  seq[total] = cell;
  best[cell] = 0;
  st[0] = 1; st[1] = total; st[2] = base; st[3] = 1; st[4] = total + 1; st[5] = 0;
  cnt[C_FOUND] = 1;
}

// ---- TraverseAndOrder's enumeration for waves.cuh ---------------------------------------------------------
// An item is a cell of seq; its entries are GetCellEdgeNeighbors over its current edges j = 0, 1, 2. A winner
// is reversed unless its first corner at p2 is followed by p1.
struct NmNb {
  const int32_t* tri;
  const unsigned long long* lstart;
  const int32_t* links;
  const int32_t* seq;
  uint8_t* fl;

  template <class F>
  __device__ __forceinline__ void each(const State& st, int64_t i, F f) const {
    const int32_t c = seq[st.cur + i];
    int32_t pts[3];
    corners(tri, fl, c, pts);
    for (int j = 0; j < 3; ++j) {
      const int32_t p1 = pts[j], p2 = pts[j == 2 ? 0 : j + 1];
      for (unsigned long long k = lstart[p1]; k < lstart[p1 + 1]; ++k) {
        const int32_t d = links[k];
        if (d != c && has(tri + 3 * (int64_t)d, p2)) f(d, j);
      }
    }
  }
  __device__ __forceinline__ unsigned long long count(const State& st, int64_t i) const {
    unsigned long long n = 0;
    each(st, i, [&](int32_t, int) { ++n; });
    return n;
  }
  __device__ __forceinline__ void win(const State& st, int64_t i, int j, int32_t d) const {
    int32_t pts[3];
    corners(tri, fl, seq[st.cur + i], pts);
    const int32_t p1 = pts[j], p2 = pts[j == 2 ? 0 : j + 1];
    const int32_t* t = tri + 3 * (int64_t)d;
    const int l = t[0] == p2 ? 0 : (t[1] == p2 ? 1 : 2);
    fl[d] = t[l == 2 ? 0 : l + 1] != p1;
  }
};

// ---- normals and splitting -----------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_nm_cell_normals(const float* __restrict__ P,
                                                            const int32_t* __restrict__ tri,
                                                            const uint8_t* __restrict__ fl, int64_t nt, float* cn,
                                                            unsigned long long* cnt) {
  __shared__ unsigned long long s_w[8];
  unsigned long long flips = 0;
  for (int64_t c = gtid(); c < nt; c += gstride()) {
    int32_t pts[3];
    corners(tri, fl, c, pts);
    double n[3];
    tri_normal(P, pts[0], pts[1], pts[2], n);
    for (int k = 0; k < 3; ++k) cn[3 * c + k] = (float)n[k];
    flips += fl[c];
  }
  const unsigned long long s = block_sum(flips, s_w);
  if (threadIdx.x == 0 && s) atomicAdd(&cnt[C_FLIPS], s);
}

// the first link slot of cell d in [lo, hi) (the links are in ascending cell id)
__device__ __forceinline__ unsigned long long slot_of(const int32_t* links, unsigned long long lo,
                                                      unsigned long long hi, int32_t d) {
  while (lo < hi) {
    const unsigned long long m = lo + (hi - lo) / 2;
    if (links[m] < d) lo = m + 1; else hi = m;
  }
  return lo;
}

// MarkAndSplit of point p over its link slots: grp[k] is the group of slot k's cell
__global__ void __launch_bounds__(kBlock) k_nm_split(const int32_t* __restrict__ tri,
                                                     const unsigned long long* __restrict__ lstart,
                                                     const int32_t* __restrict__ links, const float* __restrict__ cn,
                                                     double cos_angle, int64_t nv, int32_t* grp, int32_t* ngrp,
                                                     unsigned long long* noff) {
  for (int64_t pp = gtid(); pp < nv; pp += gstride()) {
    const int32_t p = (int32_t)pp;
    const unsigned long long lo = lstart[p], hi = lstart[p + 1];
    for (unsigned long long k = lo; k < hi; ++k) grp[k] = 0;
    int32_t ng = hi > lo ? 1 : 0;
    if (hi - lo > 1) {
      for (unsigned long long k = lo; k < hi; ++k) grp[k] = -1;
      ng = 0;
      for (unsigned long long k0 = lo; k0 < hi; ++k0) {
        const int32_t c0 = links[k0];
        if (grp[slot_of(links, lo, hi, c0)] >= 0) continue;
        grp[slot_of(links, lo, hi, c0)] = ng;
        const int32_t* t = tri + 3 * (int64_t)c0;
        const int s = t[0] == p ? 0 : (t[1] == p ? 1 : 2);
        for (int i = 0; i < 2; ++i) {
          int64_t c = c0;
          int32_t nei = i == 0 ? (s == 1 ? t[2] : t[1]) : (s == 0 ? t[2] : t[0]);
          while (c >= 0) {
            int64_t d = -1, lowest = INT64_MAX;
            if (edge_neighbors(tri, lstart, links, c, p, nei, &d, &lowest) != 1) break;
            const unsigned long long ks = slot_of(links, lo, hi, (int32_t)d);
            if (grp[ks] >= 0) break;
            const float *x = cn + 3 * c, *y = cn + 3 * d;
            const double dot = (double)x[0] * (double)y[0] + (double)x[1] * (double)y[1] + (double)x[2] * (double)y[2];
            if (!(dot > cos_angle)) break;
            grp[ks] = ng;
            c = d;
            const int32_t* u = tri + 3 * c;
            const int su = u[0] == p ? 0 : (u[1] == p ? 1 : 2);
            if (su == 0) nei = u[1] != nei ? u[1] : u[2];
            else if (su == 2) nei = u[1] != nei ? u[1] : u[0];
            else nei = u[2] != nei ? u[2] : u[0];
          }
        }
        ++ng;
      }
      for (unsigned long long k = lo + 1; k < hi; ++k)      // a cell twice at p: both slots in its group
        if (links[k] == links[k - 1]) grp[k] = grp[k - 1];
    }
    ngrp[p] = ng;
    noff[p] = ng > 1 ? (unsigned long long)(ng - 1) : 0ull;
  }
}

__device__ __forceinline__ int64_t out_id(int32_t p, int32_t g, int64_t nv, const unsigned long long* noff) {
  return g == 0 ? (int64_t)p : nv + (int64_t)noff[p] + g - 1;
}

__global__ void __launch_bounds__(kBlock) k_nm_points(const float* __restrict__ P,
                                                      const unsigned long long* __restrict__ lstart,
                                                      const int32_t* __restrict__ links,
                                                      const int32_t* __restrict__ grp,
                                                      const int32_t* __restrict__ ngrp,
                                                      const unsigned long long* __restrict__ noff,
                                                      const float* __restrict__ cn, int64_t nv, float* pts_out,
                                                      float* pn_out) {
  for (int64_t pp = gtid(); pp < nv; pp += gstride()) {
    const int32_t p = (int32_t)pp;
    const int32_t ng = ngrp[p] > 0 ? ngrp[p] : 1;
    for (int32_t g = 0; g < ng; ++g) {
      float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;
      for (unsigned long long k = lstart[p]; k < lstart[p + 1]; ++k) {
        if (grp[k] != g) continue;
        const float* n = cn + 3 * (int64_t)links[k];
        s0 += n[0]; s1 += n[1]; s2 += n[2];
      }
      const float den = sqrtf(s0 * s0 + s1 * s1 + s2 * s2);
      if (den != 0.0f) { s0 /= den; s1 /= den; s2 /= den; }
      const int64_t q = out_id(p, g, nv, noff);
      pn_out[3 * q] = s0; pn_out[3 * q + 1] = s1; pn_out[3 * q + 2] = s2;
      for (int k = 0; k < 3; ++k) pts_out[3 * q + k] = P[3 * pp + k];
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_nm_faces(const int32_t* __restrict__ tri, const uint8_t* __restrict__ fl,
                                                     const unsigned long long* __restrict__ lstart,
                                                     const int32_t* __restrict__ links,
                                                     const int32_t* __restrict__ grp,
                                                     const unsigned long long* __restrict__ noff,
                                                     const float* __restrict__ cn, int64_t nv, int64_t nt, int cols,
                                                     int i64, void* faces_out, float* cn_out) {
  for (int64_t c = gtid(); c < nt; c += gstride()) {
    int32_t pts[3];
    corners(tri, fl, c, pts);
    int64_t id[3];
    for (int j = 0; j < 3; ++j) {
      const int32_t p = pts[j];
      id[j] = out_id(p, grp[slot_of(links, lstart[p], lstart[p + 1], (int32_t)c)], nv, noff);
    }
    const int c0 = cols == 4 ? 1 : 0;
    if (i64) {
      int64_t* f = (int64_t*)faces_out + c * cols;
      if (c0) f[0] = 3;
      for (int j = 0; j < 3; ++j) f[c0 + j] = id[j];
    } else {
      int32_t* f = (int32_t*)faces_out + c * cols;
      if (c0) f[0] = 3;
      for (int j = 0; j < 3; ++j) f[c0 + j] = (int32_t)id[j];
    }
    for (int k = 0; k < 3; ++k) cn_out[3 * c + k] = cn[3 * c + k];
  }
}

// ---- mass properties -----------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_mp_terms(const float* __restrict__ P, Faces F, double* terms,
                                                     int8_t* cls, unsigned long long* ccount, uint32_t* status) {
  for (int64_t t = gtid(); t < F.nt; t += gstride()) {
    int64_t v[3];
    if (!load_face(F, t, v)) { atomicOr(status, ST_BAD_FACE); v[0] = v[1] = v[2] = 0; }
    double x[3], y[3], z[3];
    for (int c = 0; c < 3; ++c) {
      x[c] = (double)P[3 * v[c]]; y[c] = (double)P[3 * v[c] + 1]; z[c] = (double)P[3 * v[c] + 2];
    }
    double i[3], j[3], k[3], u[3];
    i[0] = x[1] - x[0]; j[0] = y[1] - y[0]; k[0] = z[1] - z[0];
    i[1] = x[2] - x[0]; j[1] = y[2] - y[0]; k[1] = z[2] - z[0];
    i[2] = x[2] - x[1]; j[2] = y[2] - y[1]; k[2] = z[2] - z[1];
    u[0] = j[0] * k[1] - k[0] * j[1];
    u[1] = k[0] * i[1] - i[0] * k[1];
    u[2] = i[0] * j[1] - j[0] * i[1];
    const double length = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
    if (length != 0.0) { u[0] /= length; u[1] /= length; u[2] /= length; }
    else { u[0] = u[1] = u[2] = 0.0; }
    const double a0 = fabs(u[0]), a1 = fabs(u[1]), a2 = fabs(u[2]);
    int8_t c = -1;
    if (a0 > a1 && a0 > a2) c = 0;
    else if (a1 > a0 && a1 > a2) c = 1;
    else if (a2 > a0 && a2 > a1) c = 2;
    else if (a0 == a1 && a0 == a2) c = 3;
    else if (a0 == a1 && a0 > a2) c = 4;
    else if (a0 == a2 && a0 > a1) c = 5;
    else if (a1 == a2 && a0 < a2) c = 6;
    if (c >= 0) atomicAdd(&ccount[c], 1ull);
    const double a = sqrt(i[1] * i[1] + j[1] * j[1] + k[1] * k[1]);
    const double b = sqrt(i[0] * i[0] + j[0] * j[0] + k[0] * k[0]);
    const double cc = sqrt(i[2] * i[2] + j[2] * j[2] + k[2] * k[2]);
    const double s = 0.5 * (a + b + cc);
    const double area = sqrt(fabs(s * (s - a) * (s - b) * (s - cc)));
    const double zavg = (z[0] + z[1] + z[2]) / 3.0;
    const double yavg = (y[0] + y[1] + y[2]) / 3.0;
    const double xavg = (x[0] + x[1] + x[2]) / 3.0;
    terms[4 * t] = area;
    terms[4 * t + 1] = area * u[0] * xavg;
    terms[4 * t + 2] = area * u[1] * yavg;
    terms[4 * t + 3] = area * u[2] * zavg;
    cls[t] = c;
  }
}

// the sums in cell order, as the checker adds them: the block stages coalesced tiles of terms in shared
// memory and one thread adds them in order (four independent chains), so the totals are its bits
__global__ void __launch_bounds__(kBlock) k_mp_sum(const double* __restrict__ terms, int64_t nt, double* sum) {
  __shared__ double s_t[kBlock * 4];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t t0 = 0; t0 < nt; t0 += kBlock) {
    const int64_t n = nt - t0 < kBlock ? nt - t0 : kBlock;
    for (int64_t k = threadIdx.x; k < 4 * n; k += kBlock) s_t[k] = terms[4 * t0 + k];
    __syncthreads();
    if (threadIdx.x == 0)
      for (int64_t i = 0; i < n; ++i)
        for (int k = 0; k < 4; ++k) acc[k] += s_t[4 * i + k];
    __syncthreads();
  }
  if (threadIdx.x == 0)
    for (int k = 0; k < 4; ++k) sum[k] = acc[k];
}

int check_args(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
               const char* what) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL && nt >= 0 && nt <= 0x7fffffffLL / 3, B2V_ERR_ARG,
              "%s: need V < 2^31 and 3T < 2^31", what);
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "%s: faces must be [T,3] or [T,4]", what);
  B2V_REQUIRE(faces_i64 == 0 || faces_i64 == 1, B2V_ERR_ARG, "%s: faces_i64 must be 0 or 1", what);
  B2V_REQUIRE(nt == 0 || nv > 0, B2V_ERR_ARG, "%s: faces without vertices", what);
  B2V_REQUIRE((nv == 0 || verts) && (nt == 0 || faces), B2V_ERR_ARG, "%s: null device pointer", what);
  return B2V_OK;
}

}  // namespace

extern "C" int64_t b2v_normals_workspace_bytes(int64_t nv, int64_t nt) {
  if (nv < 0 || nt < 0) return -1;
  return (int64_t)carve(nullptr, nv, nt).bytes;
}

extern "C" int b2v_normals_layout(int64_t nv, int64_t nt, int64_t* layout_out) {
  B2V_REQUIRE(nv >= 0 && nt >= 0 && layout_out, B2V_ERR_ARG, "normals_layout: bad arguments");
  const NmWs w = carve(nullptr, nv, nt);
  layout_out[0] = (int64_t)((char*)w.fl - (char*)nullptr);      // uint8 [T]: 1 where the cell was reversed
  layout_out[1] = (int64_t)((char*)w.seq - (char*)nullptr);     // int32 [traversed]: cells in wave order
  layout_out[2] = (int64_t)((char*)w.terms - (char*)nullptr);   // float64 [T][4]: mass terms (area, x, y, z)
  layout_out[3] = (int64_t)((char*)w.cls - (char*)nullptr);     // int8 [T]: their normal class
  return B2V_OK;
}

extern "C" int b2v_normals_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                                 int faces_i64, double feature_angle, int auto_orient, void* workspace,
                                 void* stream, int64_t* counts_host) {
  if (int rc = check_args(verts, nv, faces, nt, face_cols, faces_i64, "normals_count")) return rc;
  B2V_REQUIRE(!(feature_angle != feature_angle), B2V_ERR_ARG, "normals_count: the feature angle is NaN");
  B2V_REQUIRE(workspace && counts_host, B2V_ERR_ARG, "normals_count: null argument");
  auto_orient = auto_orient ? 1 : 0;
  for (int k = 0; k < 4; ++k) counts_host[k] = 0;
  cudaStream_t s = (cudaStream_t)stream;
  NmWs w = carve(workspace, nv, nt);
  const double a = feature_angle < 0.0 ? 0.0 : (feature_angle > 180.0 ? 180.0 : feature_angle);
  const double cos_angle = cos(a * 0.017453292519943295);
  if (nt == 0) {
    if (nv > 0) {
      B2V_CUDA(cudaMemsetAsync(w.lstart, 0, (size_t)(nv + 1) * 8, s));
      B2V_CUDA(cudaMemsetAsync(w.ngrp, 0, (size_t)nv * 4, s));
      B2V_CUDA(cudaMemsetAsync(w.noff, 0, (size_t)(nv + 1) * 8, s));
    }
    return B2V_OK;
  }
  B2V_CUDA(cudaMemsetAsync(w.cnt, 0, 16 * 8, s));
  const Faces F{faces, nt, face_cols, faces_i64, nv};
  if (int rc = build_links(w, F, "normals", s)) return rc;

  // the sets of the symmetric edge relation, and whether an (a, a) edge reaches across them
  const unsigned gt = b2v_grid(nt, kBlock, 16), g3 = b2v_grid(3 * nt, kBlock, 16);
  k_nm_init<<<gt, kBlock, 0, s>>>(w.parent, w.best, w.fl, w.stt, w.lb, nt);
  if (int rc = b2v_check_launch("k_nm_init")) return rc;
  k_nm_hook<<<g3, kBlock, 0, s>>>(w.tri, w.lstart, w.links, nt, w.parent);
  if (int rc = b2v_check_launch("k_nm_hook")) return rc;
  k_nm_compress<<<gt, kBlock, 0, s>>>(w.parent, nt);
  if (int rc = b2v_check_launch("k_nm_compress")) return rc;
  k_nm_cross<<<g3, kBlock, 0, s>>>(w.tri, w.lstart, w.links, w.parent, nt, w.cnt);
  if (int rc = b2v_check_launch("k_nm_cross")) return rc;
  unsigned long long cross = 0;
  B2V_CUDA(cudaMemcpyAsync(&cross, w.cnt + C_CROSS, 8, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));

  const NmNb E{w.tri, w.lstart, w.links, w.seq, w.fl};
  const WaveBufs B{w.seq, w.best, w.loc1, w.loc2, w.btot};
  long long regions = 0, waves = 0;
  if (!cross) {
    // every set is a region: seed them all, then one traversal
    if (auto_orient) {
      for (;;) {
        B2V_CUDA(cudaMemsetAsync(w.gk, 0xff, (size_t)nt * 8, s));
        B2V_CUDA(cudaMemsetAsync(w.cnt + C_PENDING, 0, 8, s));
        k_ao_first<<<gt, kBlock, 0, s>>>(verts, w.tri, w.parent, w.stt, w.lb, nt, w.gk);
        if (int rc = b2v_check_launch("k_ao_first")) return rc;
        k_ao_decide<<<gt, kBlock, 0, s>>>(verts, w.tri, w.lstart, w.links, w.parent, w.stt, w.gk, nt, w.res, w.fl);
        if (int rc = b2v_check_launch("k_ao_decide")) return rc;
        k_ao_apply<<<gt, kBlock, 0, s>>>(w.parent, w.res, w.gk, nt, w.stt, w.lb, w.cnt);
        if (int rc = b2v_check_launch("k_ao_apply")) return rc;
        unsigned long long pending = 0;
        B2V_CUDA(cudaMemcpyAsync(&pending, w.cnt + C_PENDING, 8, cudaMemcpyDeviceToHost, s));
        B2V_CUDA(cudaStreamSynchronize(s));
        if (!pending) break;
      }
    }
    k_nm_seed_flags<<<gt, kBlock, 0, s>>>(w.parent, w.stt, auto_orient, nt, w.tflag);
    if (int rc = b2v_check_launch("k_nm_seed_flags")) return rc;
    if (int rc = scan(w.tflag, nt, w.scratch, w.cnt + C_NEXT, s)) return rc;
    k_nm_seeds<<<gt, kBlock, 0, s>>>(w.parent, w.stt, auto_orient, w.tflag, nt, w.seq, w.best);
    if (int rc = b2v_check_launch("k_nm_seeds")) return rc;
    unsigned long long nseed = 0;
    B2V_CUDA(cudaMemcpyAsync(&nseed, w.cnt + C_NEXT, 8, cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    const long long st[6] = {(long long)nseed, 0, 1, nseed > 0, (long long)nseed, 0};
    B2V_CUDA(cudaMemcpyAsync(w.ctl, st, sizeof(st), cudaMemcpyHostToDevice, s));
    if (int rc = launch_waves(E, B, w.ctl, s, "normals")) return rc;
    B2V_CUDA(cudaMemcpyAsync(&waves, w.ctl + W_DEPTH, 8, cudaMemcpyDeviceToHost, s));
    regions = (long long)nseed;
  } else {
    // one region at a time, in the checker's order
    const long long st[W_CTL] = {0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0};
    B2V_CUDA(cudaMemcpyAsync(w.ctl, st, sizeof(st), cudaMemcpyHostToDevice, s));
    unsigned long long after = 0;
    for (;;) {
      B2V_CUDA(cudaMemsetAsync(w.cnt + C_NEXT, 0xff, 8, s));
      k_nm_next<<<gt, kBlock, 0, s>>>(verts, w.tri, w.best, auto_orient, after, nt, w.cnt);
      if (int rc = b2v_check_launch("k_nm_next")) return rc;
      k_nm_seed_one<<<1, 1, 0, s>>>(verts, w.tri, w.lstart, w.links, auto_orient, w.ctl, w.cnt, w.seq, w.best, w.fl);
      if (int rc = b2v_check_launch("k_nm_seed_one")) return rc;
      if (int rc = launch_waves(E, B, w.ctl, s, "normals")) return rc;
      unsigned long long next[2];
      long long depth = 0;
      B2V_CUDA(cudaMemcpyAsync(next, w.cnt + C_NEXT, 16, cudaMemcpyDeviceToHost, s));
      B2V_CUDA(cudaMemcpyAsync(&depth, w.ctl + W_DEPTH, 8, cudaMemcpyDeviceToHost, s));
      B2V_CUDA(cudaStreamSynchronize(s));
      if (!next[1]) break;
      ++regions;
      if (depth > waves) waves = depth;
      after = next[0] + 1;                             // auto-orient: that point is popped
    }
  }

  // cell normals, flips, splitting
  k_nm_cell_normals<<<gt, kBlock, 0, s>>>(verts, w.tri, w.fl, nt, w.cn, w.cnt);
  if (int rc = b2v_check_launch("k_nm_cell_normals")) return rc;
  k_nm_split<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(w.tri, w.lstart, w.links, w.cn, cos_angle, nv, w.grp,
                                                         w.ngrp, w.noff);
  if (int rc = b2v_check_launch("k_nm_split")) return rc;
  if (int rc = scan(w.noff, nv, w.scratch, w.cnt + C_NEW, s)) return rc;
  unsigned long long c[2];
  B2V_CUDA(cudaMemcpyAsync(c, w.cnt + C_FLIPS, 16, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  counts_host[0] = regions;
  counts_host[1] = (int64_t)c[0];
  counts_host[2] = (int64_t)c[1];
  counts_host[3] = waves;
  return B2V_OK;
}

extern "C" int b2v_normals_emit(const float* verts, int64_t nv, int64_t nt, int face_cols, int faces_i64,
                                const int64_t* counts_host, void* workspace, float* points_out, void* faces_out,
                                float* point_normals, float* cell_normals, void* stream) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL && nt >= 0 && nt <= 0x7fffffffLL / 3 && counts_host && workspace,
              B2V_ERR_ARG, "normals_emit: bad arguments");
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "normals_emit: faces must be [T,3] or [T,4]");
  const int64_t nnew = counts_host[2];
  B2V_REQUIRE(nnew >= 0 && nnew <= 3 * nt, B2V_ERR_ARG, "normals_emit: counts do not come from normals_count");
  B2V_REQUIRE((nv == 0 || (verts && points_out && point_normals)) && (nt == 0 || (faces_out && cell_normals)),
              B2V_ERR_ARG, "normals_emit: null output");
  cudaStream_t s = (cudaStream_t)stream;
  const NmWs w = carve(workspace, nv, nt);
  if (nv > 0) {
    k_nm_points<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(verts, w.lstart, w.links, w.grp, w.ngrp, w.noff, w.cn,
                                                            nv, points_out, point_normals);
    if (int rc = b2v_check_launch("k_nm_points")) return rc;
  }
  if (nt == 0) return B2V_OK;
  k_nm_faces<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(w.tri, w.fl, w.lstart, w.links, w.grp, w.noff, w.cn, nv,
                                                         nt, face_cols, faces_i64, faces_out, cell_normals);
  return b2v_check_launch("k_nm_faces");
}

extern "C" int b2v_mass_properties(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                                   int faces_i64, void* workspace, void* stream, double* out_host) {
  if (int rc = check_args(verts, nv, faces, nt, face_cols, faces_i64, "mass_properties")) return rc;
  B2V_REQUIRE(workspace && out_host, B2V_ERR_ARG, "mass_properties: null argument");
  out_host[0] = out_host[1] = 0.0;
  if (nt == 0) return B2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  NmWs w = carve(workspace, nv, nt);
  B2V_CUDA(cudaMemsetAsync(w.status, 0, 16, s));
  B2V_CUDA(cudaMemsetAsync(w.ccount, 0, 8 * 8, s));
  const Faces F{faces, nt, face_cols, faces_i64, nv};
  k_mp_terms<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(verts, F, w.terms, w.cls, w.ccount, w.status);
  if (int rc = b2v_check_launch("k_mp_terms")) return rc;
  k_mp_sum<<<1, kBlock, 0, s>>>(w.terms, nt, w.part);
  if (int rc = b2v_check_launch("k_mp_sum")) return rc;
  double sum[4];
  unsigned long long cc[8];
  uint32_t status = 0;
  B2V_CUDA(cudaMemcpyAsync(sum, w.part, sizeof(sum), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(cc, w.ccount, sizeof(cc), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(&status, w.status, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!(status & ST_BAD_FACE), B2V_ERR_ARG,
              "mass_properties: a face has an index outside [0, V) (or a leading entry other than 3)");
  const double munc[3] = {(double)cc[0], (double)cc[1], (double)cc[2]};
  const double wxyz = (double)cc[3], wxy = (double)cc[4], wxz = (double)cc[5], wyz = (double)cc[6];
  const double n = (double)nt;
  const double kx = (munc[0] + (wxyz / 3.0) + ((wxy + wxz) / 2.0)) / n;
  const double ky = (munc[1] + (wxyz / 3.0) + ((wxy + wyz) / 2.0)) / n;
  const double kz = (munc[2] + (wxyz / 3.0) + ((wxz + wyz) / 2.0)) / n;
  out_host[0] = fabs(kx * sum[1] + ky * sum[2] + kz * sum[3]);
  out_host[1] = sum[0];
  return B2V_OK;
}
