// The geodesic surface measurement on the device: the closest points of the picks (vtkPointLocator::
// FindClosestPoint) and vtkDijkstraGraphGeodesicPath's distances, path and length, behind the curved measurement
// of the 3-D viewer (measures.py:1202-1273, GeodesicMeasure._draw_line). The contract is restated once, in the C
// checker's header (DESIGN.md §3 "Geodesic measurement").
//
//   build_links        faces -> int32 [T][3] and the point -> cell links (mesh_links.cuh). A point's neighbours
//                      are the other corners of its cells: an edge shared by two cells, or a corner repeated in a
//                      degenerate cell, comes up more than once with the same weight, which changes nothing.
//   k_geo_edge_sum / k_geo_delta  the bucket width: kDeltaEdges mean edge lengths, summed in a fixed order.
//   k_geo_closest_d2 / k_geo_closest_id  the smallest (distance^2, id) per pick, in two grid-stride passes.
//   k_geo_relax        single-source relaxation in one persistent cooperative launch: near-far delta-stepping.
//                      Distances are float64 whose bit patterns take atomicMin (every value is >= 0, so the
//                      bit order is the numeric order). A round relaxes the near list; a point lowered below the
//                      threshold theta joins the next near list once (a per-round stamp), a point lowered to
//                      theta or above joins the far list once (a flag). When the near list is empty the far
//                      list's smallest live distance m sets the next theta = m + delta, and the far list is
//                      split into the new near list and what stays far. Rounds of at most kSmall near points
//                      (and far lists of at most kSmallFar) run in block 0 alone with block barriers. The result
//                      is the least fixpoint of d[v] = min_u fl(d[u] + w_uv), which Dijkstra's result equals bit
//                      for bit. With an end point the launch stops once the near list is empty and d[end] <
//                      theta: every point below theta is then final, and that covers every point the trace reads
//                      (DESIGN.md gives the argument).
//   k_geo_trace        one warp walks from the end to the start: at v, the neighbour u with fl(d[u] + w) == d[v]
//                      and the smallest (d[u], id); a step is ambiguous when two distinct neighbours share that
//                      smallest d[u]. It writes the ids, the float32 points and the length, summed in path order.
#include <math.h>

#include <cooperative_groups.h>

#include "b2v_common.cuh"
#include "mesh_links.cuh"

namespace {

namespace gcg = cooperative_groups;

constexpr int64_t kSmall = 2048;          // near lists this small run in block 0 alone
constexpr int64_t kSmallFar = 8192;       // ... as long as the far list is no longer than this
constexpr double kDeltaEdges = 8.0;       // bucket width in mean edge lengths
constexpr unsigned long long kInfBits = 0x7ff0000000000000ull;
constexpr int kSumBlocks = 1024;          // blocks of k_geo_edge_sum: a fixed sum order

// ctl words
enum { G_CNT = 0, G_FCNT = 4, G_MIN = 6, G_ROUNDS = 8, G_BUCKETS = 9, G_STATE = 16, G_CTL = 32 };

struct GeoWs {
  unsigned long long* ctl;         // [G_CTL]
  uint32_t* status;
  int32_t* tri;                    // [T][3]
  unsigned long long* lstart;      // [V + 1]
  int32_t* links;                  // [3T]
  uint32_t *ka, *va, *kb, *vb;     // [3T] sort ping-pong
  unsigned long long* hist;
  unsigned long long* scratch;
  double* part;                    // [kSumBlocks] edge-length partial sums
  double* delta;                   // [1]
  unsigned long long* dist;        // [V] float64 bits
  int32_t* stamp;                  // [V] the round whose near list holds the point
  int32_t* infar;                  // [V] 1 while the point is on a far list
  int32_t *near0, *near1;          // [V]
  int32_t *far0, *far1;            // [V]
  int64_t* tout;                   // [4] trace: points, ambiguous steps, unreached, error
  double* tlen;                    // [2] trace: segment length, running total
  size_t bytes;
};

GeoWs carve(void* base, int64_t nv, int64_t nt) {
  GeoWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const size_t V = (size_t)nv, T = (size_t)nt, C3 = 3 * T;
  const int64_t nb3 = ceil_div64((int64_t)(C3 > 0 ? C3 : 1), kBlock);
  const int64_t hist_n = 256 * nb3 + 1;
  const int64_t longest = hist_n > (int64_t)V + 1 ? hist_n : (int64_t)V + 1;
  w.ctl = (unsigned long long*)take(G_CTL * 8);
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
  w.part = (double*)take(kSumBlocks * 8);
  w.delta = (double*)take(8);
  w.dist = (unsigned long long*)take(V * 8);
  w.stamp = (int32_t*)take(V * 4);
  w.infar = (int32_t*)take(V * 4);
  w.near0 = (int32_t*)take(V * 4);
  w.near1 = (int32_t*)take(V * 4);
  w.far0 = (int32_t*)take(V * 4);
  w.far1 = (int32_t*)take(V * 4);
  w.tout = (int64_t*)take(4 * 8);
  w.tlen = (double*)take(2 * 8);
  w.bytes = o;
  return w;
}

template <typename T>
__device__ __forceinline__ void point(const T* __restrict__ v, int64_t i, double p[3]) {
  p[0] = (double)v[3 * i];
  p[1] = (double)v[3 * i + 1];
  p[2] = (double)v[3 * i + 2];
}

// vtkMath::Distance2BetweenPoints in double, summed in that order (the library builds with -fmad=false)
__device__ __forceinline__ double dist2(const double a[3], const double b[3]) {
  const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return dx * dx + dy * dy + dz * dz;
}

__device__ __forceinline__ double ld_dist(const unsigned long long* d, int64_t i) {
  return __longlong_as_double((long long)__ldcg(d + i));
}

// ---- bucket width ----------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kBlock) k_geo_edge_sum(const T* __restrict__ verts, const int32_t* __restrict__ tri,
                                                         int64_t nt, double* part) {
  __shared__ double s_w[kBlock / 32];
  double s = 0.0;
  for (int64_t t = gtid(); t < nt; t += gstride()) {
    double p[3][3];
    for (int j = 0; j < 3; ++j) point(verts, tri[3 * t + j], p[j]);
    for (int j = 0; j < 3; ++j) s += sqrt(dist2(p[j], p[(j + 1) % 3]));
  }
  const double tot = block_sum(s, s_w);
  if (threadIdx.x == 0) part[blockIdx.x] = tot;
}

__global__ void k_geo_delta(const double* part, int nb, int64_t nt, double* delta) {
  double s = 0.0;
  for (int b = 0; b < nb; ++b) s += part[b];
  const double d = kDeltaEdges * s / (3.0 * (double)nt);
  *delta = d > 0.0 && d < INFINITY ? d : INFINITY;   // no positive finite width: one bucket (Bellman-Ford)
}

// ---- closest points --------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kBlock) k_geo_closest_d2(const T* __restrict__ verts, int64_t nv,
                                                           const double* __restrict__ picks, int64_t np,
                                                           unsigned long long* best) {
  for (int64_t i = gtid(); i < nv; i += gstride()) {
    double p[3];
    point(verts, i, p);
    for (int64_t k = 0; k < np; ++k) {
      const double q[3] = {picks[3 * k], picks[3 * k + 1], picks[3 * k + 2]};
      const unsigned long long b = (unsigned long long)__double_as_longlong(dist2(q, p));
      if (b < __ldcg(best + k)) atomicMin(best + k, b);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kBlock) k_geo_closest_id(const T* __restrict__ verts, int64_t nv,
                                                           const double* __restrict__ picks, int64_t np,
                                                           const unsigned long long* __restrict__ best,
                                                           long long* ids) {
  for (int64_t i = gtid(); i < nv; i += gstride()) {
    double p[3];
    point(verts, i, p);
    for (int64_t k = 0; k < np; ++k) {
      const double q[3] = {picks[3 * k], picks[3 * k + 1], picks[3 * k + 2]};
      if ((unsigned long long)__double_as_longlong(dist2(q, p)) == best[k] && i < __ldcg(ids + k))
        atomicMin(ids + k, (long long)i);
    }
  }
}

// ---- relaxation ------------------------------------------------------------------------------------------
struct Relax {
  const int32_t* tri;
  const unsigned long long* lstart;
  const int32_t* links;
  unsigned long long* dist;
  int32_t* stamp;
  int32_t* infar;
  int32_t *near0, *near1;
  int32_t *far0, *far1;
  unsigned long long* ctl;
  const double* delta;             // [1] the bucket width
  int64_t end;                     // -1: the whole field
};

__device__ __forceinline__ int32_t* near_list(const Relax& R, long long k) { return k & 1 ? R.near1 : R.near0; }
__device__ __forceinline__ int32_t* far_list(const Relax& R, long long k) { return k & 1 ? R.far1 : R.far0; }

// the state every block keeps a copy of; block 0 hands it over after a single-block stretch
struct GeoState {
  long long r;        // the round whose near list is next: near[r & 1], counted in ctl[G_CNT + r % 3]
  long long n;        // its length
  long long fp;       // the current far list: far[fp], counted in ctl[G_FCNT + fp]
  long long nf;       // its length
  long long phase;    // buckets opened
  double theta;       // every point below theta that is not on the near list is final
  long long done;
};

__device__ __forceinline__ unsigned long long rd(const unsigned long long* p) {
  return *(const volatile unsigned long long*)p;
}

template <bool kGrid>
__device__ __forceinline__ void geo_sync() {
  if (kGrid) gcg::this_grid().sync(); else __syncthreads();
}

// One round over the near list, or, when it is empty, the opening of the next bucket (or the end).
template <bool kGrid, typename T>
__device__ void geo_step(const Relax& R, const T* __restrict__ verts, GeoState& st, int b, int nb) {
  const bool lead = b == 0 && threadIdx.x == 0;
  const int64_t tid = (int64_t)b * kBlock + threadIdx.x, stride = (int64_t)nb * kBlock;
  if (st.n > 0) {
    const int32_t* cur = near_list(R, st.r);
    int32_t* nxt = near_list(R, st.r + 1);
    unsigned long long* ncnt = R.ctl + G_CNT + (st.r + 1) % 3;
    const int32_t tag = (int32_t)(st.r + 1);
    for (int64_t i = tid; i < st.n; i += stride) {
      const int32_t u = __ldcg(cur + i);
      const double du = ld_dist(R.dist, u);
      double pu[3];
      point(verts, u, pu);
      for (unsigned long long k = R.lstart[u]; k < R.lstart[u + 1]; ++k) {
        const int64_t c = R.links[k];
        for (int j = 0; j < 3; ++j) {
          const int32_t x = R.tri[3 * c + j];
          if (x == u) continue;
          double px[3];
          point(verts, x, px);
          const double nd = du + sqrt(dist2(px, pu));
          if (!(nd < ld_dist(R.dist, x))) continue;
          const unsigned long long bits = (unsigned long long)__double_as_longlong(nd);
          if (atomicMin(R.dist + x, bits) <= bits) continue;
          if (nd < st.theta) {
            if (atomicExch(R.stamp + x, tag) != tag) nxt[atomicAdd(ncnt, 1ull)] = x;
          } else if (atomicExch(R.infar + x, 1) == 0) {
            far_list(R, st.fp)[atomicAdd(R.ctl + G_FCNT + st.fp, 1ull)] = x;
          }
        }
      }
    }
    if (lead) R.ctl[G_CNT + (st.r + 2) % 3] = 0;   // read last after the sync before this round's
    geo_sync<kGrid>();
    st.r += 1;
    st.n = (long long)rd(R.ctl + G_CNT + st.r % 3);
    st.nf = (long long)rd(R.ctl + G_FCNT + st.fp);
    if (lead) R.ctl[G_ROUNDS] += 1;
    return;
  }
  // the near list is empty: every point below theta is final
  if ((R.end >= 0 && ld_dist(R.dist, R.end) < st.theta) || st.nf == 0) { st.done = 1; return; }
  const int32_t* far = far_list(R, st.fp);
  unsigned long long* gmin = R.ctl + G_MIN + (st.phase & 1);
  for (int64_t i = tid; i < st.nf; i += stride) {
    const int32_t x = __ldcg(far + i);
    const double dx = ld_dist(R.dist, x);
    if (dx >= st.theta) atomicMin(gmin, (unsigned long long)__double_as_longlong(dx));
  }
  if (lead) R.ctl[G_FCNT + (st.fp ^ 1)] = 0;
  geo_sync<kGrid>();
  const unsigned long long mb = rd(gmin);
  if (mb >= kInfBits) { st.done = 1; return; }    // only points final already are left
  const double m = __longlong_as_double((long long)mb);
  double nt_ = m + *R.delta;
  if (!(nt_ > m)) nt_ = __longlong_as_double((long long)mb + 1);   // the next double above m
  int32_t* out = far_list(R, st.fp ^ 1);
  int32_t* nxt = near_list(R, st.r);                // empty: count ctl[G_CNT + r % 3] is 0
  for (int64_t i = tid; i < st.nf; i += stride) {
    const int32_t x = __ldcg(far + i);
    const double dx = ld_dist(R.dist, x);
    if (dx < st.theta) {
      R.infar[x] = 0;                             // lowered below theta since: it went through a near list
    } else if (dx < nt_) {
      R.infar[x] = 0;
      nxt[atomicAdd(R.ctl + G_CNT + st.r % 3, 1ull)] = x;
    } else {
      out[atomicAdd(R.ctl + G_FCNT + (st.fp ^ 1), 1ull)] = x;
    }
  }
  if (lead) {
    R.ctl[G_MIN + ((st.phase + 1) & 1)] = kInfBits;
    R.ctl[G_BUCKETS] += 1;
  }
  geo_sync<kGrid>();
  st.theta = nt_;
  st.phase += 1;
  st.fp ^= 1;
  st.n = (long long)rd(R.ctl + G_CNT + st.r % 3);
  st.nf = (long long)rd(R.ctl + G_FCNT + st.fp);
}

__device__ __forceinline__ bool geo_small(const GeoState& st) {
  return st.n <= kSmall && st.nf <= kSmallFar;
}

__device__ __forceinline__ void store_st(unsigned long long* ctl, const GeoState& st) {
  long long* c = (long long*)ctl;
  c[0] = st.r; c[1] = st.n; c[2] = st.fp; c[3] = st.nf; c[4] = st.phase; c[5] = __double_as_longlong(st.theta);
  c[6] = st.done;
}

__device__ __forceinline__ void load_st(const unsigned long long* ctl, GeoState& st) {
  const volatile long long* c = (const volatile long long*)ctl;
  st.r = c[0]; st.n = c[1]; st.fp = c[2]; st.nf = c[3]; st.phase = c[4]; st.theta = __longlong_as_double(c[5]);
  st.done = c[6];
}

template <typename T>
__global__ void __launch_bounds__(kBlock, 2) k_geo_relax(Relax R, const T* __restrict__ verts) {
  gcg::grid_group g = gcg::this_grid();
  GeoState st{0, 1, 0, 0, 0, *R.delta, 0};
  int flip = 0;
  while (!st.done) {
    if (geo_small(st)) {
      if (blockIdx.x == 0) {
        do geo_step<false>(R, verts, st, 0, 1); while (!st.done && geo_small(st));
        if (threadIdx.x == 0) store_st(R.ctl + G_STATE + 8 * flip, st);
      }
      g.sync();
      load_st(R.ctl + G_STATE + 8 * flip, st);
      flip ^= 1;
      continue;
    }
    geo_step<true>(R, verts, st, blockIdx.x, gridDim.x);
  }
}

__global__ void k_geo_start(unsigned long long* dist, int32_t* near0, unsigned long long* ctl, int64_t start) {
  dist[start] = 0ull;
  near0[0] = (int32_t)start;
  for (int k = 0; k < G_CTL; ++k) ctl[k] = 0;
  ctl[G_CNT] = 1;
  ctl[G_MIN] = ctl[G_MIN + 1] = kInfBits;
}

// ---- trace -----------------------------------------------------------------------------------------------
// (d[u] bits, u, another distinct u shares d[u]) ordered by (d, id)
__device__ __forceinline__ void pick_min(unsigned long long& bd, int32_t& bu, int& tie, unsigned long long od,
                                         int32_t ou, int otie) {
  if (od < bd) { bd = od; bu = ou; tie = otie; }
  else if (od == bd && od != ~0ull) {
    tie = tie | otie | (ou != bu);
    if (ou < bu) bu = ou;
  }
}

template <typename T>
__global__ void __launch_bounds__(32) k_geo_trace(const T* __restrict__ verts, int64_t nv, const int32_t* __restrict__ tri,
                                                  const unsigned long long* __restrict__ lstart,
                                                  const int32_t* __restrict__ links,
                                                  const unsigned long long* __restrict__ dist, int64_t start,
                                                  int64_t end, double total_in, long long* ids, float* pts,
                                                  int64_t* tout, double* tlen) {
  const int lane = threadIdx.x;
  int64_t v = end, n = 0, amb = 0;
  double seg = 0.0, tot = total_in;
  double pv[3];
  point(verts, v, pv);
  const bool unreached = dist[end] >= kInfBits;
  int err = 0;
  for (;;) {
    const float f[3] = {(float)pv[0], (float)pv[1], (float)pv[2]};
    if (lane == 0) {
      ids[n] = v;
      pts[3 * n] = f[0]; pts[3 * n + 1] = f[1]; pts[3 * n + 2] = f[2];
      if (n > 0) {   // the length over the float32 points, as measures.py sums it
        const double a[3] = {(double)pts[3 * n - 3], (double)pts[3 * n - 2], (double)pts[3 * n - 1]};
        const double bq[3] = {(double)f[0], (double)f[1], (double)f[2]};
        const double s = sqrt(dist2(a, bq));
        seg += s;
        tot += s;
      }
    }
    ++n;
    if (v == start || unreached) break;
    if (n >= nv) { err = 1; break; }
    const double dv = __longlong_as_double((long long)dist[v]);
    unsigned long long bd = ~0ull;
    int32_t bu = -1;
    int tie = 0;
    for (unsigned long long k = lstart[v] + lane; k < lstart[v + 1]; k += 32) {
      const int64_t c = links[k];
      for (int j = 0; j < 3; ++j) {
        const int32_t u = tri[3 * c + j];
        if (u == v) continue;
        const double du = __longlong_as_double((long long)dist[u]);
        double pu[3];
        point(verts, u, pu);
        if (du + sqrt(dist2(pu, pv)) == dv) pick_min(bd, bu, tie, dist[u], u, 0);
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long od = __shfl_xor_sync(0xffffffffu, bd, o);
      const int32_t ou = __shfl_xor_sync(0xffffffffu, bu, o);
      const int ot = __shfl_xor_sync(0xffffffffu, tie, o);
      pick_min(bd, bu, tie, od, ou, ot);
    }
    if (bu < 0) { err = 1; break; }
    amb += tie;
    v = bu;
    point(verts, v, pv);
  }
  if (lane == 0) {
    tout[0] = n; tout[1] = amb; tout[2] = unreached; tout[3] = err;
    tlen[0] = seg; tlen[1] = tot;
  }
}

int check_verts(const void* verts, int64_t nv, int verts_f64, const char* what) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL, B2V_ERR_ARG, "%s: bad vertex count", what);
  B2V_REQUIRE(verts_f64 == 0 || verts_f64 == 1, B2V_ERR_ARG, "%s: verts_f64 must be 0 or 1", what);
  B2V_REQUIRE(nv == 0 || verts, B2V_ERR_ARG, "%s: null device pointer", what);
  return B2V_OK;
}

int check_surface(const void* verts, int64_t nv, int verts_f64, int64_t nt, void* ws, const char* what) {
  if (int rc = check_verts(verts, nv, verts_f64, what)) return rc;
  B2V_REQUIRE(nt > 0 && nt <= 0x7fffffffLL / 3 && nv > 0 && ws, B2V_ERR_ARG,
              "%s: needs a surface with cells and its workspace", what);
  return B2V_OK;
}

}  // namespace

extern "C" int64_t b2v_geodesic_workspace_bytes(int64_t nv, int64_t nt) {
  if (nv < 0 || nt < 0) return -1;
  return (int64_t)carve(nullptr, nv, nt).bytes;
}

extern "C" int b2v_geodesic_links(const void* verts, int64_t nv, int verts_f64, const void* faces, int64_t nt,
                                  int face_cols, int faces_i64, void* workspace, void* stream) {
  if (int rc = check_surface(verts, nv, verts_f64, nt, workspace, "geodesic_links")) return rc;
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "geodesic_links: faces must be [T,3] or [T,4]");
  B2V_REQUIRE(faces, B2V_ERR_ARG, "geodesic_links: null device pointer");
  cudaStream_t s = (cudaStream_t)stream;
  GeoWs w = carve(workspace, nv, nt);
  const Faces F{faces, nt, face_cols, faces_i64 ? 1 : 0, nv};
  if (int rc = build_links(w, F, "geodesic", s)) return rc;
  if (verts_f64)
    k_geo_edge_sum<double><<<kSumBlocks, kBlock, 0, s>>>((const double*)verts, w.tri, nt, w.part);
  else
    k_geo_edge_sum<float><<<kSumBlocks, kBlock, 0, s>>>((const float*)verts, w.tri, nt, w.part);
  if (int rc = b2v_check_launch("k_geo_edge_sum")) return rc;
  k_geo_delta<<<1, 1, 0, s>>>(w.part, kSumBlocks, nt, w.delta);
  return b2v_check_launch("k_geo_delta");
}

extern "C" int b2v_closest_points(const void* verts, int64_t nv, int verts_f64, const double* picks, int64_t np,
                                  double* scratch, int64_t* ids_out, void* stream) {
  if (int rc = check_verts(verts, nv, verts_f64, "closest_points")) return rc;
  B2V_REQUIRE(nv > 0 && np >= 0, B2V_ERR_ARG, "closest_points: needs points");
  if (np == 0) return B2V_OK;
  B2V_REQUIRE(picks && scratch && ids_out, B2V_ERR_ARG, "closest_points: null device pointer");
  cudaStream_t s = (cudaStream_t)stream;
  unsigned long long* best = (unsigned long long*)scratch;
  const unsigned g = b2v_grid(nv, kBlock, 8);
  k_fill<unsigned long long><<<b2v_grid(np, kBlock, 1), kBlock, 0, s>>>(best, np, ~0ull);
  if (int rc = b2v_check_launch("k_fill")) return rc;
  k_fill<long long><<<b2v_grid(np, kBlock, 1), kBlock, 0, s>>>((long long*)ids_out, np, (long long)nv);
  if (int rc = b2v_check_launch("k_fill")) return rc;
  if (verts_f64) {
    k_geo_closest_d2<double><<<g, kBlock, 0, s>>>((const double*)verts, nv, picks, np, best);
    if (int rc = b2v_check_launch("k_geo_closest_d2")) return rc;
    k_geo_closest_id<double><<<g, kBlock, 0, s>>>((const double*)verts, nv, picks, np, best, (long long*)ids_out);
  } else {
    k_geo_closest_d2<float><<<g, kBlock, 0, s>>>((const float*)verts, nv, picks, np, best);
    if (int rc = b2v_check_launch("k_geo_closest_d2")) return rc;
    k_geo_closest_id<float><<<g, kBlock, 0, s>>>((const float*)verts, nv, picks, np, best, (long long*)ids_out);
  }
  return b2v_check_launch("k_geo_closest_id");
}

extern "C" int b2v_geodesic_distances(const void* verts, int64_t nv, int verts_f64, int64_t nt, void* workspace,
                                      int64_t start, int64_t end, double* dist_out, void* stream,
                                      int64_t* stats_host) {
  if (int rc = check_surface(verts, nv, verts_f64, nt, workspace, "geodesic_distances")) return rc;
  B2V_REQUIRE(start >= 0 && start < nv && end >= -1 && end < nv && stats_host, B2V_ERR_ARG,
              "geodesic_distances: start / end outside [0, V)");
  cudaStream_t s = (cudaStream_t)stream;
  GeoWs w = carve(workspace, nv, nt);
  const unsigned gv = b2v_grid(nv, kBlock, 16);
  k_fill<unsigned long long><<<gv, kBlock, 0, s>>>(w.dist, nv, kInfBits);
  if (int rc = b2v_check_launch("k_fill")) return rc;
  k_fill<int32_t><<<gv, kBlock, 0, s>>>(w.stamp, nv, -1);
  if (int rc = b2v_check_launch("k_fill")) return rc;
  B2V_CUDA(cudaMemsetAsync(w.infar, 0, (size_t)nv * 4, s));
  k_geo_start<<<1, 1, 0, s>>>(w.dist, w.near0, w.ctl, start);
  if (int rc = b2v_check_launch("k_geo_start")) return rc;
  Relax R{w.tri, w.lstart, w.links, w.dist, w.stamp, w.infar, w.near0, w.near1, w.far0, w.far1, w.ctl, w.delta,
          end};
  const void* vp = verts;
  void* args[] = {&R, &vp};
  const void* fn = verts_f64 ? (const void*)k_geo_relax<double> : (const void*)k_geo_relax<float>;
  if (int rc = launch_coop(fn, args, s, "geodesic_distances", "k_geo_relax")) return rc;
  if (dist_out) B2V_CUDA(cudaMemcpyAsync(dist_out, w.dist, (size_t)nv * 8, cudaMemcpyDeviceToDevice, s));
  unsigned long long c[2];
  B2V_CUDA(cudaMemcpyAsync(c, w.ctl + G_ROUNDS, 16, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  stats_host[0] = (int64_t)c[0];
  stats_host[1] = (int64_t)c[1];
  return B2V_OK;
}

extern "C" int b2v_geodesic_trace(const void* verts, int64_t nv, int verts_f64, int64_t nt, void* workspace,
                                  int64_t start, int64_t end, double total_in, int64_t* ids_out, float* points_out,
                                  void* stream, int64_t* counts_host, double* lengths_host) {
  if (int rc = check_surface(verts, nv, verts_f64, nt, workspace, "geodesic_trace")) return rc;
  B2V_REQUIRE(start >= 0 && start < nv && end >= 0 && end < nv, B2V_ERR_ARG,
              "geodesic_trace: start / end outside [0, V)");
  B2V_REQUIRE(ids_out && points_out && counts_host && lengths_host, B2V_ERR_ARG, "geodesic_trace: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  GeoWs w = carve(workspace, nv, nt);
  if (verts_f64)
    k_geo_trace<double><<<1, 32, 0, s>>>((const double*)verts, nv, w.tri, w.lstart, w.links, w.dist, start, end,
                                         total_in, (long long*)ids_out, points_out, w.tout, w.tlen);
  else
    k_geo_trace<float><<<1, 32, 0, s>>>((const float*)verts, nv, w.tri, w.lstart, w.links, w.dist, start, end,
                                        total_in, (long long*)ids_out, points_out, w.tout, w.tlen);
  if (int rc = b2v_check_launch("k_geo_trace")) return rc;
  int64_t t[4];
  B2V_CUDA(cudaMemcpyAsync(t, w.tout, sizeof(t), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(lengths_host, w.tlen, 16, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!t[3], B2V_ERR_RANGE, "geodesic_trace: no predecessor chain from the end to the start (distances "
              "not computed from this start?)");
  counts_host[0] = t[0];
  counts_host[1] = t[1];
  counts_host[2] = t[2];
  return B2V_OK;
}
