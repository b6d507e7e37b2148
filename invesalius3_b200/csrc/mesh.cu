// Context-aware mesh smoothing (SURVEY 8f-2): invesalius_rs.context_aware_smoothing / Mesh.ca_smoothing
// (invesalius_rs/src/mesh.rs:27-395, called by invesalius/data/surface_process.py:312-320 on the merged
// surface). float32 vertices [V][3] (smoothed in place), int64 faces [M][4] with the leading 3, float32 face
// normals [M][3]. The reference's stages, each a kernel over the vertices:
//   vertex -> faces   (build_map_vface :89-101): CSR from the caller's stable ordering of the 4 M face
//                     entries — EVERY column is taken as a vertex id, the leading 3 included, as the
//                     reference does (vertex 3 collects every face). The reference only looks the map up
//                     for ids in [0, V), so a leading entry outside that range is ignored (a mesh of at
//                     most 3 vertices is valid); an entry of columns 1..3 outside it is an error;
//   adjacency         (build_vertex_connectivity :103-123): neighbours in first-appearance order over the
//                     faces — the order fixes the float64 summation order of the smoother;
//   staircase seeds   (find_staircase_artifacts :125-189): the reference's max / min tracking with its
//                     `else if`, kept as it is. After a vertex's first face min is still f64::MAX, so
//                     every vertex that has a face becomes a seed for any finite T (none for T = NaN);
//                     for T = +inf a vertex is a seed exactly when its first face has a NaN normal
//                     (|f64::MIN - f64::MAX| overflows to inf);
//   weights           (propagate_weights :202-295): frontier rounds; a round is resolved by atomic minimum
//                     on the squared distance, then the seed of the winner (smallest seed on ties) — the
//                     reference resolves a round by compare-and-swap in whatever order its threads run.
//                     With every seed at distance 0 the first round claims nothing: the later rounds
//                     run only for T = +inf with NaN normals;
//   Taubin            (taubin_smooth :345-395): lambda 0.5, mu -0.53; D in float64 in adjacency order,
//                     updates cast to float32 and added in float32.
// Bit-exact against the sequential CPU checker whenever no vertex receives offers from two seeds, and against
// the round-by-round schedule of the NumPy restatement in tests/ca_smoothing_model.py.
#include "b2v_common.cuh"
#include "scan.cuh"

namespace {

struct MeshWs {
  long long* first;     // [V] start of the vertex's entries in `order` (-1: none)
  long long* last;      // [V]
  uint32_t* deg;        // [V + 1] adjacency degrees, then exclusive offsets
  uint32_t* adj;        // [6 M] neighbour ids (a triangle contributes at most two per vertex)
  uint32_t* bsum;       // [scan_blocks(V + 1) + 1] scan scratch
  unsigned long long* dist;   // [V] squared distance bits
  int* seed;            // [V]
  int* frontier[2];     // [adjacency size] each
  int* fcount;          // [4]
  double* w;            // [V]
  double* d;            // [3 V]
  int* status;
  long long bytes;
};

MeshWs carve(void* base, long long nv, long long nf) {
  MeshWs w;
  char* p = (char*)base;
  long long off = 0;
  w.first = (long long*)(p + off); off += align256(nv * 8);
  w.last = (long long*)(p + off); off += align256(nv * 8);
  w.deg = (uint32_t*)(p + off); off += align256((nv + 1) * 4);
  w.adj = (uint32_t*)(p + off); off += align256(6 * nf * 4 + 4);
  w.bsum = (uint32_t*)(p + off); off += align256((scan_blocks(nv + 1) + 1) * 4);
  w.dist = (unsigned long long*)(p + off); off += align256(nv * 8);
  w.seed = (int*)(p + off); off += align256(nv * 4);
  w.frontier[0] = (int*)(p + off); off += align256(6 * nf * 4 + nv * 4 + 4);
  w.frontier[1] = (int*)(p + off); off += align256(6 * nf * 4 + nv * 4 + 4);
  w.fcount = (int*)(p + off); off += 256;
  w.w = (double*)(p + off); off += align256(nv * 8);
  w.d = (double*)(p + off); off += align256(nv * 24);
  w.status = (int*)(p + off); off += 256;
  w.bytes = off;
  return w;
}

// entries sorted by vertex id (stable): segment bounds per vertex. A leading-column entry outside [0, V) is
// skipped (the reference never looks it up); an entry of columns 1..3 outside [0, V) is an error
__global__ void __launch_bounds__(256) k_mesh_segments(const long long* __restrict__ faces, const long long* __restrict__ order,
                                                       long long ne, long long nv, long long* first, long long* last, int* status) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < ne; e += stride) {
    const long long ent = order[e], key = faces[ent];
    if (key < 0 || key >= nv) { if (ent & 3) *status = 1; continue; }
    if (e == 0 || faces[order[e - 1]] != key) first[key] = e;
    if (e == ne - 1 || faces[order[e + 1]] != key) last[key] = e + 1;
  }
}

// neighbours of v in the reference's order: faces that hold v in columns 1..3, by face id; per face its
// other vertices in column order; first appearance only. Calls f(vj, k) for the k-th neighbour.
// The faces around v are gathered first (one pass over the segment: vertex 3's segment also holds the
// leading 3 of EVERY face row), then deduplicated among themselves.
constexpr int kMaxRing = 96;
template <typename F>
__device__ __forceinline__ int for_each_neighbour(const long long* __restrict__ faces, const long long* __restrict__ order,
                                                  long long e0, long long e1, long long v, F f) {
  long long ring[kMaxRing];
  int nr = 0;
  long long prev_fb = -1;
  for (long long e = e0; e < e1; ++e) {
    const long long ent = order[e];
    if ((ent & 3) == 0) continue;                 // the leading 3 of a face row is not a vertex of the face
    const long long fb = ent & ~3ll;
    if (fb == prev_fb) continue;                  // v twice in one face: handled at its first column
    prev_fb = fb;
    if (nr < kMaxRing) ring[nr] = fb;
    ++nr;
  }
  if (nr > kMaxRing) nr = kMaxRing;               // (a vertex with more than 96 faces keeps its first 96: reported by the host)
  int k = 0;
  for (int a = 0; a < nr; ++a) {
    const long long fb = ring[a];
    for (int c = 1; c < 4; ++c) {
      const long long vj = faces[fb + c];
      if (vj == v) continue;
      bool seen = false;
      for (int a2 = 0; a2 <= a && !seen; ++a2) {
        const int cend = a2 == a ? c : 4;
        for (int c2 = 1; c2 < cend; ++c2) seen |= faces[ring[a2] + c2] == vj;
      }
      if (!seen) f(vj, k++);
    }
  }
  return k;
}

// distinct faces around a vertex (columns 1..3 only), counted as for_each_neighbour counts them: the host
// refuses meshes with more than kMaxRing
__global__ void __launch_bounds__(256) k_mesh_ring_check(const long long* __restrict__ order, long long nv,
                                                         const long long* __restrict__ first, const long long* __restrict__ last,
                                                         int* status) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv || first[v] < 0) return;
  if (last[v] - first[v] <= kMaxRing) return;     // cannot exceed it
  long long n = 0, prev_fb = -1;
  for (long long e = first[v]; e < last[v]; ++e) {
    const long long ent = order[e];
    if ((ent & 3) == 0 || (ent & ~3ll) == prev_fb) continue;    // v twice in one face: one face
    prev_fb = ent & ~3ll;
    ++n;
  }
  if (n > kMaxRing) *status = 2;
}

__global__ void __launch_bounds__(128) k_mesh_degree(const long long* __restrict__ faces, const long long* __restrict__ order,
                                                     long long nv, const long long* __restrict__ first,
                                                     const long long* __restrict__ last, uint32_t* __restrict__ deg) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v > nv) return;
  uint32_t n = 0;
  if (v < nv && first[v] >= 0) n = (uint32_t)for_each_neighbour(faces, order, first[v], last[v], v, [](long long, int) {});
  deg[v] = n;       // deg[nv] = 0: the scan turns it into the total
}

__global__ void __launch_bounds__(128) k_mesh_adjacency(const long long* __restrict__ faces, const long long* __restrict__ order,
                                                        long long nv, const long long* __restrict__ first,
                                                        const long long* __restrict__ last, const uint32_t* __restrict__ off,
                                                        uint32_t* __restrict__ adj) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv || first[v] < 0) return;
  uint32_t* out = adj + off[v];
  for_each_neighbour(faces, order, first[v], last[v], v, [&](long long vj, int k) { out[k] = (uint32_t)vj; });
}

// find_staircase_artifacts + the initial state of propagate_weights
__global__ void __launch_bounds__(128) k_mesh_seeds(const long long* __restrict__ order, const float* __restrict__ normals,
                                                    long long nv, const long long* __restrict__ first,
                                                    const long long* __restrict__ last, double t, unsigned long long* dist,
                                                    int* seed, int* frontier, int* fcount) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  const double DMIN = -1.7976931348623157e308, DMAX = 1.7976931348623157e308;
  bool hit = false;
  if (first[v] >= 0) {
    double max_z = DMIN, min_z = DMAX, max_y = DMIN, min_y = DMAX, max_x = DMIN, min_x = DMAX;
    for (long long e = first[v]; e < last[v] && !hit; ++e) {
      const float* nr = normals + 3 * (order[e] >> 2);
      const double nx = nr[0], ny = nr[1], nz = nr[2];
      const double of_z = 1.0 - fabs(nx * 0.0 + ny * 0.0 + nz * 1.0);
      const double of_y = 1.0 - fabs(nx * 0.0 + ny * 1.0 + nz * 0.0);
      const double of_x = 1.0 - fabs(nx * 1.0 + ny * 0.0 + nz * 0.0);
      if (of_z > max_z) max_z = of_z; else if (of_z < min_z) min_z = of_z;
      if (of_y > max_y) max_y = of_y; else if (of_y < min_y) min_y = of_y;
      if (of_x > max_x) max_x = of_x; else if (of_x < min_x) min_x = of_x;
      hit = fabs(max_z - min_z) >= t || fabs(max_y - min_y) >= t || fabs(max_x - min_x) >= t;
    }
  }
  dist[v] = hit ? 0ull : 0x7ff0000000000000ull;     // 0.0 / +inf (non-negative doubles order like their bit patterns)
  seed[v] = hit ? (int)v : -1;
  if (hit) frontier[atomicAdd(fcount, 1)] = (int)v;
}

__device__ __forceinline__ double sqdist(const float* __restrict__ p, long long a, long long b) {
  const double dx = (double)p[3 * a] - (double)p[3 * b], dy = (double)p[3 * a + 1] - (double)p[3 * b + 1],
               dz = (double)p[3 * a + 2] - (double)p[3 * b + 2];
  return dx * dx + dy * dy + dz * dz;
}

// one round, pass 1: offers lower the distances
__global__ void __launch_bounds__(256) k_mesh_offer(const float* __restrict__ pos, const uint32_t* __restrict__ off,
                                                    const uint32_t* __restrict__ adj, const int* __restrict__ seed,
                                                    const int* __restrict__ frontier, int nfr, double tmax_sq, unsigned long long* dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nfr) return;
  const int v = frontier[i], s = seed[v];
  for (uint32_t e = off[v]; e < off[v + 1]; ++e) {
    const uint32_t vj = adj[e];
    const double d_sq = sqdist(pos, vj, s);
    if (d_sq > tmax_sq) continue;
    const unsigned long long bits = (unsigned long long)__double_as_longlong(d_sq);
    if (bits < dist[vj]) atomicMin(&dist[vj], bits);
  }
}
// pass 2: the offers that won take the seed (smallest seed on equal distances) and enter the next frontier
__global__ void __launch_bounds__(256) k_mesh_claim(const float* __restrict__ pos, const uint32_t* __restrict__ off,
                                                    const uint32_t* __restrict__ adj, const int* __restrict__ seed_in,
                                                    int* seed_new, const int* __restrict__ frontier, int nfr, double tmax_sq,
                                                    const unsigned long long* __restrict__ dist,
                                                    const unsigned long long* __restrict__ dist_before, int* next, int* ncount) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nfr) return;
  const int v = frontier[i], s = seed_in[v];
  for (uint32_t e = off[v]; e < off[v + 1]; ++e) {
    const uint32_t vj = adj[e];
    const double d_sq = sqdist(pos, vj, s);
    if (d_sq > tmax_sq) continue;
    const unsigned long long bits = (unsigned long long)__double_as_longlong(d_sq);
    if (bits == dist[vj] && bits < dist_before[vj]) {
      const int old = atomicMin(&seed_new[vj], s);
      if (old == 0x7fffffff) next[atomicAdd(ncount, 1)] = (int)vj;      // first claim of this round
    }
  }
}

__global__ void __launch_bounds__(256) k_mesh_weights(const unsigned long long* __restrict__ dist, long long nv, double tmax,
                                                      double bmin, double* __restrict__ w) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  const double d = __longlong_as_double((long long)dist[i]);
  w[i] = isinf(d) ? bmin : (1.0 - sqrt(d) / tmax) * (1.0 - bmin) + bmin;
}

__global__ void __launch_bounds__(256) k_mesh_calc_d(const float* __restrict__ pos, const uint32_t* __restrict__ off,
                                                     const uint32_t* __restrict__ adj, long long nv, double* __restrict__ d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  const double px = pos[3 * i], py = pos[3 * i + 1], pz = pos[3 * i + 2];
  double dx = 0.0, dy = 0.0, dz = 0.0;
  const uint32_t e0 = off[i], e1 = off[i + 1];
  for (uint32_t e = e0; e < e1; ++e) {
    const uint32_t j = adj[e];
    dx += px - (double)pos[3ll * j];
    dy += py - (double)pos[3ll * j + 1];
    dz += pz - (double)pos[3ll * j + 2];
  }
  if (e1 > e0) { const double n = (double)(e1 - e0); dx /= n; dy /= n; dz /= n; }
  d[3 * i] = dx; d[3 * i + 1] = dy; d[3 * i + 2] = dz;
}

__global__ void __launch_bounds__(256) k_mesh_step(float* pos, const double* __restrict__ d, const double* __restrict__ w,
                                                   long long nv, double factor) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  const double wf = w[i] * factor;                 // (weights[i] * l) * d[k]
  pos[3 * i] += (float)(wf * d[3 * i]);
  pos[3 * i + 1] += (float)(wf * d[3 * i + 1]);
  pos[3 * i + 2] += (float)(wf * d[3 * i + 2]);
}

// after a round: vertices claimed this round take their new seed; the marker array is reset
__global__ void k_mesh_commit(int* seed, int* seed_new, const int* __restrict__ next, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = next[i];
  seed[v] = seed_new[v];
  seed_new[v] = 0x7fffffff;
}

}  // namespace

extern "C" int64_t b2v_ca_smoothing_workspace_bytes(int64_t nverts, int64_t nfaces) {
  if (nverts <= 0 || nfaces <= 0) return 0;
  return carve(nullptr, nverts, nfaces).bytes + (nverts * 8 + 256) + (nverts * 4 + 256);
}

extern "C" int b2v_ca_smoothing(float* vertices, int64_t nverts, const int64_t* faces4, int64_t nfaces, const float* normals,
                                const int64_t* order, double t, double tmax, double bmin, uint32_t n_iters, void* workspace,
                                void* stream) {
  B2V_REQUIRE(vertices && faces4 && normals && order && workspace, B2V_ERR_ARG, "ca_smoothing: null pointer");
  B2V_REQUIRE(nverts > 0 && nfaces > 0 && nverts < (1ll << 31) && nfaces < (1ll << 28), B2V_ERR_ARG, "ca_smoothing: bad mesh size");
  cudaStream_t s = (cudaStream_t)stream;
  MeshWs w = carve(workspace, nverts, nfaces);
  unsigned long long* dist_before = (unsigned long long*)((char*)workspace + w.bytes);
  int* seed_new = (int*)((char*)dist_before + align256(nverts * 8));
  const long long ne = 4 * nfaces, nv = nverts;
  int rc;
  B2V_CUDA(cudaMemsetAsync(w.status, 0, 4, s));
  B2V_CUDA(cudaMemsetAsync(w.fcount, 0, 16, s));
  k_fill<long long><<<(unsigned)ceil_div64(nv, 256), 256, 0, s>>>(w.first, nv, -1);
  k_fill<int><<<(unsigned)ceil_div64(nv, 256), 256, 0, s>>>(seed_new, nv, 0x7fffffff);
  k_mesh_segments<<<b2v_grid(ne, 256, 32), 256, 0, s>>>((const long long*)faces4, (const long long*)order, ne, nv,
                                                        w.first, w.last, w.status);
  if ((rc = b2v_check_launch("k_mesh_segments"))) return rc;
  int st = 0;
  B2V_CUDA(cudaMemcpyAsync(&st, w.status, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(st == 0, B2V_ERR_RANGE, "ca_smoothing: a face entry (columns 1..3) lies outside the vertex array (the reference panics here)");
  k_mesh_ring_check<<<(unsigned)ceil_div64(nv, 256), 256, 0, s>>>((const long long*)order, nv, w.first, w.last, w.status);
  if ((rc = b2v_check_launch("k_mesh_ring_check"))) return rc;
  B2V_CUDA(cudaMemcpyAsync(&st, w.status, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(st == 0, B2V_ERR_ARG, "ca_smoothing: a vertex belongs to more than 96 faces (not supported)");
  // adjacency: degrees, exclusive scan, fill
  k_mesh_degree<<<(unsigned)ceil_div64(nv + 1, 128), 128, 0, s>>>((const long long*)faces4, (const long long*)order, nv, w.first, w.last, w.deg);
  if ((rc = b2v_check_launch("k_mesh_degree"))) return rc;
  if ((rc = scan(w.deg, nv + 1, w.bsum, nullptr, s))) return rc;
  k_mesh_adjacency<<<(unsigned)ceil_div64(nv, 128), 128, 0, s>>>((const long long*)faces4, (const long long*)order, nv, w.first, w.last, w.deg, w.adj);
  if ((rc = b2v_check_launch("k_mesh_adjacency"))) return rc;
  // seeds, then the frontier rounds of propagate_weights
  k_mesh_seeds<<<(unsigned)ceil_div64(nv, 128), 128, 0, s>>>((const long long*)order, normals, nv, w.first, w.last, t, w.dist, w.seed, w.frontier[0], w.fcount);
  if ((rc = b2v_check_launch("k_mesh_seeds"))) return rc;
  const double tmax_sq = tmax * tmax;
  int cur = 0, nfr = 0;
  B2V_CUDA(cudaMemcpyAsync(&nfr, w.fcount, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  for (int round = 0; nfr > 0; ++round) {
    B2V_REQUIRE(round < (1 << 20), B2V_ERR_NOCONV, "ca_smoothing: weight propagation does not terminate");
    B2V_CUDA(cudaMemcpyAsync(dist_before, w.dist, (size_t)nv * 8, cudaMemcpyDeviceToDevice, s));
    B2V_CUDA(cudaMemsetAsync(w.fcount + 1, 0, 4, s));
    k_mesh_offer<<<(unsigned)ceil_div64(nfr, 256), 256, 0, s>>>(vertices, w.deg, w.adj, w.seed, w.frontier[cur], nfr, tmax_sq, w.dist);
    k_mesh_claim<<<(unsigned)ceil_div64(nfr, 256), 256, 0, s>>>(vertices, w.deg, w.adj, w.seed, seed_new, w.frontier[cur], nfr, tmax_sq,
                                                              w.dist, dist_before, w.frontier[cur ^ 1], w.fcount + 1);
    if ((rc = b2v_check_launch("k_mesh_claim"))) return rc;
    int nn = 0;
    B2V_CUDA(cudaMemcpyAsync(&nn, w.fcount + 1, 4, cudaMemcpyDeviceToHost, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    if (nn > 0) {
      k_mesh_commit<<<(unsigned)ceil_div64(nn, 256), 256, 0, s>>>(w.seed, seed_new, w.frontier[cur ^ 1], nn);
      if ((rc = b2v_check_launch("k_mesh_commit"))) return rc;
    }
    cur ^= 1;
    nfr = nn;
  }
  k_mesh_weights<<<(unsigned)ceil_div64(nv, 256), 256, 0, s>>>(w.dist, nv, tmax, bmin, w.w);
  if ((rc = b2v_check_launch("k_mesh_weights"))) return rc;
  const double lm[2] = {0.5, -0.53};
  for (uint32_t it = 0; it < n_iters; ++it)
    for (int half = 0; half < 2; ++half) {
      k_mesh_calc_d<<<(unsigned)ceil_div64(nv, 256), 256, 0, s>>>(vertices, w.deg, w.adj, nv, w.d);
      k_mesh_step<<<(unsigned)ceil_div64(nv, 256), 256, 0, s>>>(vertices, w.d, w.w, nv, lm[half]);
    }
  return b2v_check_launch("k_mesh_step");
}
