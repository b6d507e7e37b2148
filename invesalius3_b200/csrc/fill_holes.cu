// Surface hole filling on the device: vtkFillHolesFilter on triangles, as InVesalius's "Smooth surface"
// (polydata_utils.py:85-107, HoleSize 1000), the surface dialog's "Fill holes" (surface_process.py:396-411,
// 300), FillSurfaceHole (500) and the marker surface geometry use it. The contract is restated once, in the
// C checker's header (fill_holes.c, DESIGN.md §3 "Surface hole filling"); every step below reproduces its
// sequential result exactly.
//
//   build_links    faces -> int32 [T][3] and the point -> cell links (mesh_links.cuh).
//   k_fh_edges     one thread per (cell, edge): an edge without GetCellEdgeNeighbors is a boundary line; a
//                  scan of the flags numbers the lines in VTK's order and k_fh_lines writes them, with each
//                  point's line count and (for the first two) its lines.
//   darts          every non-degenerate line l is two darts, 2l running p0 -> p1 and 2l + 1 running back.
//                  A dart's successor leaves its head on the head's other line when the head has exactly two
//                  line incidences; otherwise the dart ends a path. So the darts form paths (the chains
//                  between points with != 2 lines, once each way) and cycles (pure loops, once each way).
//   k_fh_jump      pointer jumping in one cooperative launch: per dart, the end of its path and the darts
//                  left to it, or, on a cycle, the lowest dart of the cycle and the distance to it.
//   k_fh_loops     which traversals of the sequential loop close (see below), and their point counts.
//   k_fh_points    a scan over the lines numbers the loops in the order of their first line; every dart of
//                  a loop writes its tail at its rank.
//   k_fh_sphere    one thread per loop: the bounding sphere, in loop order.
//   k_fh_tri       one block per loop to fill: the greedy ear clipping, an argmin over the kept ear keys
//                  per step (only the two ears next to a clipped point are recomputed).
//
// Which traversals close. A traversal starting on line L walks from L.p0 through points with two lines and
// stops at the first other point (invalid) or back at L.p0 (valid). It never passes a point with != 2
// lines except at its start, so chains and cycles are independent, and it marks the lines it walks.
//  - A cycle's lowest line is its first start: the loop is the cycle from that line's p0, in its direction.
//  - On a chain l_1 .. l_m from point A to point B (positions along the chain), a start on a line running
//    with the chain marks the suffix from it, one running against it the prefix up to it. A loop closes
//    only when A == B and l_1 (running with the chain) or l_m (running against it) starts. l_1 starts iff
//    every prefix minimum of the line ids, in position order, runs with the chain; l_m iff every suffix
//    minimum runs against it. (A prefix minimum is exactly a line that starts while no line running
//    against the chain has started yet.) One thread per closed chain walks it both ways to test this.
//  - A degenerate line (x, x) is a loop of one point on its own.
//
// A call synchronises the host twice: the face check in build_links, and the counts of b2v_holes_count
// (lines, loops, new triangles) that size the output. b2v_holes_emit does not synchronise.
#include <cooperative_groups.h>
#include <float.h>
#include <math.h>

#include "b2v_common.cuh"
#include "mesh_links.cuh"

namespace cg = cooperative_groups;

namespace {

enum : int8_t { FILLED = 0, FAILED = 1, TOO_LARGE = 2 };

struct FhWs {
  unsigned long long* ctl;         // [32]: counters
  uint32_t* status;
  int32_t* tri;                    // [T][3]
  unsigned long long* lstart;      // [V + 1] link offsets
  int32_t* links;                  // [3T]
  uint32_t *ka, *va, *kb, *vb;     // [3T] sort ping-pong
  unsigned long long* hist;        // [256 * nb3 + 1]
  unsigned long long* scratch;     // scan block sums
  unsigned long long* lpos;        // [3T + 1] boundary flags, then line ids
  int32_t* lines;                  // [L][2], L = 3T: room for every edge
  int32_t* deg;                    // [V] line incidences per point
  int32_t* slot;                   // [V][2] a point's first two lines
  int32_t* succ;                   // [2L] dart successor (-1: the dart ends a path)
  int32_t* nx[2];                  // [2L] pointer jumping: the dart 2^k ahead (-1: past the path's end)
  uint32_t* dd[2];                 // [2L] darts covered: to the path's end, inclusive, once nx is -1
  unsigned long long* mn[2];       // [2L] (lowest dart << 32) | its distance, over the covered darts
  int32_t* last[2];                // [2L] the path's last dart (-1: not reached yet)
  unsigned long long* lkey;        // [L + 1] per line: (starts a loop << 32) | loop points; scanned
  int32_t* lsd;                    // [L] the start dart of the loop starting on a line
  int32_t* lterm;                  // [L] the last dart of that loop when it is a chain
  int32_t* dloop;                  // [2L] loop of a cycle's start dart or of a chain loop's last dart
  int32_t* poly;                   // [L] the loops' points, loop after loop
  int32_t* first;                  // [L] per loop: first line
  int32_t* npts;                   //              points
  unsigned long long* off;         //              offset in poly (and of its triangle slots)
  double* radius;                  //              bounding-sphere radius
  int8_t* state;                   //              filled / failed / too large
  unsigned long long* toff;        // [L + 1] new triangles per loop, scanned by the emit
  int32_t* prv;                    // [L] ear clipping: remaining neighbours and ear keys, per loop slot
  int32_t* nxt;                    // [L]
  double* key;                     // [L]
  int32_t* otri;                   // [L][3] new triangles at their loop's slots
  size_t bytes;
};

FhWs carve(void* base, int64_t nv, int64_t nt) {
  FhWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const size_t V = (size_t)nv, T = (size_t)nt, L = 3 * T, D = 2 * L;
  const int64_t nb3 = ceil_div64((int64_t)(L > 0 ? L : 1), kBlock);
  const int64_t hist_n = 256 * nb3 + 1;
  int64_t longest = hist_n > (int64_t)V + 1 ? hist_n : (int64_t)V + 1;
  if ((int64_t)L + 1 > longest) longest = (int64_t)L + 1;
  w.ctl = (unsigned long long*)take(32 * 8);
  w.status = (uint32_t*)take(16);
  w.tri = (int32_t*)take(L * 4);
  w.lstart = (unsigned long long*)take((V + 1) * 8);
  w.links = (int32_t*)take(L * 4);
  w.ka = (uint32_t*)take(L * 4);
  w.va = (uint32_t*)take(L * 4);
  w.kb = (uint32_t*)take(L * 4);
  w.vb = (uint32_t*)take(L * 4);
  w.hist = (unsigned long long*)take((size_t)hist_n * 8);
  w.scratch = (unsigned long long*)take((size_t)(scan_blocks(longest) + 1) * 8);
  w.lpos = (unsigned long long*)take((L + 1) * 8);
  w.lines = (int32_t*)take(D * 4);
  w.deg = (int32_t*)take(V * 4);
  w.slot = (int32_t*)take(2 * V * 4);
  w.succ = (int32_t*)take(D * 4);
  for (int b = 0; b < 2; ++b) {
    w.nx[b] = (int32_t*)take(D * 4);
    w.dd[b] = (uint32_t*)take(D * 4);
    w.mn[b] = (unsigned long long*)take(D * 8);
    w.last[b] = (int32_t*)take(D * 4);
  }
  w.lkey = (unsigned long long*)take((L + 1) * 8);
  w.lsd = (int32_t*)take(L * 4);
  w.lterm = (int32_t*)take(L * 4);
  w.dloop = (int32_t*)take(D * 4);
  w.poly = (int32_t*)take(L * 4);
  w.first = (int32_t*)take(L * 4);
  w.npts = (int32_t*)take(L * 4);
  w.off = (unsigned long long*)take(L * 8);
  w.radius = (double*)take(L * 8);
  w.state = (int8_t*)take(L);
  w.toff = (unsigned long long*)take((L + 1) * 8);
  w.prv = (int32_t*)take(L * 4);
  w.nxt = (int32_t*)take(L * 4);
  w.key = (double*)take(L * 8);
  w.otri = (int32_t*)take(L * 12);
  w.bytes = o;
  return w;
}

// ctl words
enum { C_LINES = 0,     // boundary lines
       C_PACK = 1,      // (loops << 32) | points in loops
       C_TRIS = 2,      // new triangles
       C_BUF = 3 };     // the pointer-jumping buffer holding the result

// darts when there are at least three lines; none otherwise (the output is the input)
__device__ __forceinline__ int64_t ndarts(const unsigned long long* ctl) {
  const int64_t n = (int64_t)ctl[C_LINES];
  return n >= 3 ? 2 * n : 0;
}

__device__ __forceinline__ int64_t nloops(const unsigned long long* ctl) { return (int64_t)(ctl[C_PACK] >> 32); }

// ---- boundary lines ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_fh_edges(const int32_t* __restrict__ tri,
                                                     const unsigned long long* __restrict__ lstart,
                                                     const int32_t* __restrict__ links, int64_t nt,
                                                     unsigned long long* flag) {
  for (int64_t q = gtid(); q < 3 * nt; q += gstride()) {
    const int64_t c = q / 3;
    const int i = (int)(q - 3 * c);
    int64_t first = -1, lowest = INT64_MAX;
    flag[q] = edge_neighbors(tri, lstart, links, c, tri[q], tri[3 * c + (i + 1) % 3], &first, &lowest) == 0;
  }
}

__global__ void __launch_bounds__(kBlock) k_fh_lines(const int32_t* __restrict__ tri,
                                                     const unsigned long long* __restrict__ lpos, int64_t nt,
                                                     int32_t* lines, int32_t* deg, int32_t* slot) {
  for (int64_t q = gtid(); q < 3 * nt; q += gstride()) {
    if (lpos[q + 1] == lpos[q]) continue;
    const int64_t l = (int64_t)lpos[q], c = q / 3;
    const int i = (int)(q - 3 * c);
    const int32_t e[2] = {tri[q], tri[3 * c + (i + 1) % 3]};
    for (int k = 0; k < 2; ++k) {
      lines[2 * l + k] = e[k];
      const int s = atomicAdd(&deg[e[k]], 1);
      if (s < 2) slot[2 * (int64_t)e[k] + s] = (int32_t)l;
    }
  }
}

// ---- darts --------------------------------------------------------------------------------------------------
__device__ __forceinline__ int32_t tail_of(const int32_t* lines, int64_t x) { return lines[x]; }
__device__ __forceinline__ int32_t head_of(const int32_t* lines, int64_t x) { return lines[x ^ 1]; }
__device__ __forceinline__ bool degenerate(const int32_t* lines, int64_t x) {
  return lines[x & ~1ll] == lines[x | 1];
}

// dart 2l runs line l from p0 to p1, dart 2l + 1 from p1 to p0: a dart's tail is lines[x], its head
// lines[x ^ 1]
__global__ void __launch_bounds__(kBlock) k_fh_darts(const int32_t* __restrict__ lines,
                                                     const int32_t* __restrict__ deg,
                                                     const int32_t* __restrict__ slot,
                                                     const unsigned long long* __restrict__ ctl, int32_t* succ,
                                                     int32_t* nx, uint32_t* dd, unsigned long long* mn,
                                                     int32_t* last) {
  const int64_t nd = ndarts(ctl);
  for (int64_t x = gtid(); x < nd; x += gstride()) {
    int32_t s = -1;
    const int32_t h = head_of(lines, x);
    if (!degenerate(lines, x) && deg[h] == 2) {
      const int32_t l = (int32_t)(x >> 1), a = slot[2 * (int64_t)h], b = slot[2 * (int64_t)h + 1];
      const int32_t n = a == l ? b : a;
      s = 2 * n + (lines[2 * (int64_t)n] == h ? 0 : 1);   // the dart of n whose tail is h
    }
    succ[x] = s;
    nx[x] = s;
    dd[x] = 1;
    mn[x] = (unsigned long long)x << 32;
    last[x] = s < 0 ? (int32_t)x : -1;
  }
}

struct Pj {
  int32_t* nx[2];
  uint32_t* dd[2];
  unsigned long long* mn[2];
  int32_t* last[2];
  unsigned long long* ctl;
};

// Round r doubles the window of every dart: after it, a dart covers the 2^(r+1) darts ahead of it (fewer at
// a path's end). With 2^R >= lines no path or cycle is longer than the window.
__global__ void __launch_bounds__(kBlock) k_fh_jump(Pj J) {
  cg::grid_group g = cg::this_grid();
  const int64_t nd = ndarts(J.ctl);
  int rounds = 0;
  while ((1ll << rounds) < nd / 2) ++rounds;
  for (int r = 0; r < rounds; ++r) {
    const int a = r & 1, b = a ^ 1;
    for (int64_t x = gtid(); x < nd; x += gstride()) {
      const int32_t y = J.nx[a][x];
      if (y < 0) {
        J.nx[b][x] = -1; J.dd[b][x] = J.dd[a][x]; J.mn[b][x] = J.mn[a][x]; J.last[b][x] = J.last[a][x];
      } else {
        const uint32_t d = J.dd[a][x];
        const unsigned long long m2 = J.mn[a][y] + d;
        J.nx[b][x] = J.nx[a][y];
        J.dd[b][x] = d + J.dd[a][y];
        J.mn[b][x] = m2 < J.mn[a][x] ? m2 : J.mn[a][x];
        J.last[b][x] = J.last[a][y];
      }
    }
    g.sync();
  }
  if (gtid() == 0) J.ctl[C_BUF] = (unsigned long long)(rounds & 1);
}

// true when, walking the path from dart x, every prefix minimum of the line ids runs with the path
__device__ bool prefix_minima_forward(const int32_t* succ, int32_t x) {
  int32_t lo = INT32_MAX;
  for (int32_t y = x; y >= 0; y = succ[y]) {
    const int32_t l = y >> 1;
    if (l < lo) {
      if (y & 1) return false;
      lo = l;
    }
  }
  return true;
}

// the loops: lkey[l] gets (1 << 32) | points for the line l a loop starts on, lsd[l] its start dart and
// lterm[l] the last dart of a chain loop
__global__ void __launch_bounds__(kBlock) k_fh_loops(const int32_t* __restrict__ lines,
                                                     const int32_t* __restrict__ deg,
                                                     const int32_t* __restrict__ succ, Pj J,
                                                     unsigned long long* lkey, int32_t* lsd, int32_t* lterm) {
  const int64_t nd = ndarts(J.ctl);
  const int b = (int)J.ctl[C_BUF];
  const int32_t* nx = J.nx[b];
  const uint32_t* dd = J.dd[b];
  const unsigned long long* mn = J.mn[b];
  const int32_t* last = J.last[b];
  for (int64_t x = gtid(); x < nd; x += gstride()) {
    const int64_t l = x >> 1;
    if (degenerate(lines, x)) {
      if (!(x & 1)) { lkey[l] = (1ull << 32) | 1ull; lsd[l] = (int32_t)x; }
      continue;
    }
    if (nx[x] >= 0) {                                    // on a cycle
      const int64_t rep = (int64_t)(mn[x] >> 32);
      if (rep & 1) continue;                             // the cycle run against its lowest line
      atomicAdd(&lkey[rep >> 1], (x == rep ? (1ull << 32) : 0ull) + 1ull);
      if (x == rep) lsd[l] = (int32_t)x;
      continue;
    }
    if (deg[tail_of(lines, x)] == 2) continue;           // not the first dart of a path
    const int32_t t = last[x], back = t ^ 1;             // back: the first dart of the reverse path
    if (x > back || tail_of(lines, x) != head_of(lines, t)) continue;   // each closed chain once
    int32_t s = -1, e = -1;
    if (prefix_minima_forward(succ, (int32_t)x)) { s = (int32_t)x; e = t; }
    else if (prefix_minima_forward(succ, back)) { s = back; e = (int32_t)(x ^ 1); }
    if (s < 0) continue;
    lkey[s >> 1] = (1ull << 32) | dd[x];
    lsd[s >> 1] = s;
    lterm[s >> 1] = e;
  }
}

__global__ void __launch_bounds__(kBlock) k_fh_records(const int32_t* __restrict__ lines,
                                                       const unsigned long long* __restrict__ lkey,
                                                       const int32_t* __restrict__ lsd,
                                                       const int32_t* __restrict__ lterm,
                                                       Pj J, int32_t* dloop, int32_t* poly, int32_t* first,
                                                       int32_t* npts, unsigned long long* off) {
  const int64_t nl = ndarts(J.ctl) / 2;
  const int32_t* nx = J.nx[J.ctl[C_BUF]];
  const unsigned long long lo = 0xffffffffull;
  for (int64_t l = gtid(); l < nl; l += gstride()) {
    const unsigned long long k0 = lkey[l], k1 = lkey[l + 1];
    if ((k1 >> 32) == (k0 >> 32)) continue;
    const int32_t li = (int32_t)(k0 >> 32), s = lsd[l];
    first[li] = (int32_t)l;
    npts[li] = (int32_t)((k1 & lo) - (k0 & lo));
    off[li] = k0 & lo;
    if (degenerate(lines, s)) poly[k0 & lo] = lines[s];
    else dloop[nx[s] >= 0 ? s : lterm[l]] = li;
  }
}

// every dart of a loop writes its tail at its rank in the loop
__global__ void __launch_bounds__(kBlock) k_fh_points(const int32_t* __restrict__ lines, Pj J,
                                                      const int32_t* __restrict__ dloop,
                                                      const int32_t* __restrict__ npts,
                                                      const unsigned long long* __restrict__ off, int32_t* poly) {
  const int64_t nd = ndarts(J.ctl);
  const int b = (int)J.ctl[C_BUF];
  const int32_t* nx = J.nx[b];
  for (int64_t x = gtid(); x < nd; x += gstride()) {
    if (degenerate(lines, x)) continue;
    int64_t rank;
    int32_t li;
    if (nx[x] >= 0) {
      const unsigned long long m = J.mn[b][x];
      li = dloop[m >> 32];
      if (li < 0) continue;
      const int64_t n = npts[li], dist = (int64_t)(m & 0xffffffffull);
      rank = (n - dist) % n;
    } else {
      li = dloop[J.last[b][x]];
      if (li < 0) continue;
      rank = (int64_t)npts[li] - (int64_t)J.dd[b][x];
    }
    poly[off[li] + rank] = tail_of(lines, x);
  }
}

// ---- size test and triangulation --------------------------------------------------------------------------
__device__ __forceinline__ void pt(const float* P, int32_t p, double x[3]) {
  x[0] = (double)P[3 * (int64_t)p]; x[1] = (double)P[3 * (int64_t)p + 1]; x[2] = (double)P[3 * (int64_t)p + 2];
}

__global__ void __launch_bounds__(kBlock) k_fh_sphere(const float* __restrict__ P, const int32_t* __restrict__ poly,
                                                      const int32_t* __restrict__ npts,
                                                      const unsigned long long* __restrict__ off,
                                                      const unsigned long long* ctl, double hole_size,
                                                      double* radius, int8_t* state) {
  const int64_t nl = nloops(ctl);
  for (int64_t li = gtid(); li < nl; li += gstride()) {
    const int32_t* q = poly + off[li];
    double c[3], r = 0.0;
    pt(P, q[0], c);
    for (int32_t k = 0; k < npts[li]; ++k) {
      double p[3];
      pt(P, q[k], p);
      const double v0 = p[0] - c[0], v1 = p[1] - c[1], v2 = p[2] - c[2];
      const double d2 = (v0 * v0 + v1 * v1) + v2 * v2;
      if (d2 > r * r) {
        const double d = sqrt(d2);
        r = (r + d) / 2.0;
        const double delta = d - r;
        for (int a = 0; a < 3; ++a) c[a] = (r * c[a] + delta * p[a]) / d;
      }
    }
    radius[li] = r;
    state[li] = r <= hole_size ? FILLED : TOO_LARGE;
  }
}

__device__ __forceinline__ double len3(double v0, double v1, double v2) { return sqrt((v0 * v0 + v1 * v1) + v2 * v2); }

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double n[3]) {
  n[0] = a[1] * b[2] - a[2] * b[1];
  n[1] = a[2] * b[0] - a[0] * b[2];
  n[2] = a[0] * b[1] - a[1] * b[0];
}

// the ear (prev, i, next): its perimeter when its normal agrees with N, +inf otherwise
__device__ double ear_key(const float* P, const int32_t* q, int32_t prev, int32_t i, int32_t next,
                          const double N[3]) {
  double a[3], b[3], c[3], u[3], v[3], e[3];
  pt(P, q[prev], a); pt(P, q[i], b); pt(P, q[next], c);
  for (int k = 0; k < 3; ++k) { u[k] = c[k] - b[k]; v[k] = a[k] - b[k]; }
  cross3(u, v, e);
  const double el = len3(e[0], e[1], e[2]);
  if (el != 0.0) { e[0] /= el; e[1] /= el; e[2] /= el; }
  if (!((e[0] * N[0] + e[1] * N[1]) + e[2] * N[2] > 0.0)) return INFINITY;
  return (len3(b[0] - a[0], b[1] - a[1], b[2] - a[2]) + len3(c[0] - b[0], c[1] - b[1], c[2] - b[2])) +
         len3(a[0] - c[0], a[1] - c[1], a[2] - c[2]);
}

// (key, position) order: the smaller key, then the lower position
__device__ __forceinline__ void better(double& k, int32_t& i, double ok, int32_t oi) {
  if (ok < k || (ok == k && oi < i)) { k = ok; i = oi; }
}

struct Tr {
  const float* P;
  const int32_t* poly;
  const int32_t* npts;
  const unsigned long long* off;
  const unsigned long long* ctl;
  int8_t* state;
  int32_t* prv;
  int32_t* nxt;
  double* key;
  int32_t* otri;
  unsigned long long* toff;
  unsigned long long* tris;
};

__global__ void __launch_bounds__(kBlock) k_fh_tri(Tr K) {
  __shared__ double s_k[kBlock / 32];
  __shared__ int32_t s_i[kBlock / 32];
  __shared__ double s_n[3];
  __shared__ int32_t s_best, s_head;
  const int64_t nl = nloops(K.ctl);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int64_t li = blockIdx.x; li < nl; li += gridDim.x) {
    const int32_t n = K.npts[li];
    if (K.state[li] == TOO_LARGE || n < 3) {
      if (threadIdx.x == 0) {
        if (K.state[li] != TOO_LARGE) K.state[li] = FAILED;
        K.toff[li] = 0;
      }
      continue;
    }
    const unsigned long long o = K.off[li];
    const int32_t* q = K.poly + o;
    int32_t *prv = K.prv + o, *nxt = K.nxt + o, *tri = K.otri + 3 * o;
    double* key = K.key + o;
    if (threadIdx.x == 0) {                              // the fan sum, in order
      double N[3] = {0.0, 0.0, 0.0}, p0[3];
      pt(K.P, q[0], p0);
      for (int32_t i = 1; i + 1 < n; ++i) {
        double a[3], b[3], x[3];
        pt(K.P, q[i], a); pt(K.P, q[i + 1], b);
        for (int k = 0; k < 3; ++k) { a[k] -= p0[k]; b[k] -= p0[k]; }
        cross3(a, b, x);
        for (int k = 0; k < 3; ++k) N[k] += x[k];
      }
      const double nl2 = len3(N[0], N[1], N[2]);
      if (nl2 != 0.0) { N[0] /= nl2; N[1] /= nl2; N[2] /= nl2; }
      s_n[0] = N[0]; s_n[1] = N[1]; s_n[2] = N[2];
      s_head = 0;
    }
    __syncthreads();
    const double N[3] = {s_n[0], s_n[1], s_n[2]};
    for (int32_t i = threadIdx.x; i < n; i += blockDim.x) {
      prv[i] = (i + n - 1) % n;
      nxt[i] = (i + 1) % n;
      key[i] = n > 3 ? ear_key(K.P, q, (i + n - 1) % n, i, (i + 1) % n, N) : INFINITY;
    }
    __syncthreads();
    int32_t rem = n, made = 0;
    bool failed = false;
    while (rem > 3) {
      double bk = INFINITY;
      int32_t bi = INT32_MAX;
      for (int32_t i = threadIdx.x; i < n; i += blockDim.x) better(bk, bi, key[i], i);
      for (int s = 16; s > 0; s >>= 1)
        better(bk, bi, __shfl_down_sync(0xffffffffu, bk, s), __shfl_down_sync(0xffffffffu, bi, s));
      if (lane == 0) { s_k[wid] = bk; s_i[wid] = bi; }
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) better(bk, bi, s_k[w], s_i[w]);
        if (!(bk < INFINITY)) {
          s_best = -1;
        } else {
          const int32_t p = prv[bi], x = nxt[bi];
          tri[3 * made] = q[p]; tri[3 * made + 1] = q[bi]; tri[3 * made + 2] = q[x];
          key[bi] = INFINITY;
          nxt[p] = x; prv[x] = p;
          if (bi == s_head) s_head = x;
          if (rem - 1 > 3) {
            key[p] = ear_key(K.P, q, prv[p], p, x, N);
            key[x] = ear_key(K.P, q, p, x, nxt[x], N);
          }
          s_best = bi;
        }
      }
      __syncthreads();
      if (s_best < 0) { failed = true; break; }
      ++made;
      --rem;
    }
    if (threadIdx.x == 0) {
      if (!failed) {
        const int32_t h = s_head;
        tri[3 * made] = q[h]; tri[3 * made + 1] = q[nxt[h]]; tri[3 * made + 2] = q[nxt[nxt[h]]];
        ++made;
      }
      K.state[li] = failed ? FAILED : FILLED;
      K.toff[li] = failed ? 0ull : (unsigned long long)made;
      if (!failed) atomicAdd(K.tris, (unsigned long long)made);
    }
    __syncthreads();
  }
}

// ---- output -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_fh_emit(const int32_t* __restrict__ otri,
                                                    const unsigned long long* __restrict__ off,
                                                    const unsigned long long* __restrict__ toff, int64_t nloop,
                                                    int64_t nt, int cols, int i64, void* out) {
  for (int64_t li = blockIdx.x; li < nloop; li += gridDim.x) {
    const unsigned long long b = toff[li], e = toff[li + 1];
    const int32_t* src = otri + 3 * off[li];
    for (unsigned long long k = threadIdx.x; k < e - b; k += blockDim.x) {
      const int64_t row = (nt + (int64_t)(b + k)) * cols;
      const int c0 = cols == 4 ? 1 : 0;
      if (i64) {
        int64_t* f = (int64_t*)out + row;
        if (c0) f[0] = 3;
        for (int j = 0; j < 3; ++j) f[c0 + j] = src[3 * k + j];
      } else {
        int32_t* f = (int32_t*)out + row;
        if (c0) f[0] = 3;
        for (int j = 0; j < 3; ++j) f[c0 + j] = src[3 * k + j];
      }
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_fh_out(const int32_t* __restrict__ first,
                                                   const int32_t* __restrict__ npts,
                                                   const double* __restrict__ radius,
                                                   const int8_t* __restrict__ state, int64_t nloop,
                                                   int64_t* first_out, int64_t* npts_out, double* radius_out,
                                                   int8_t* state_out) {
  for (int64_t li = gtid(); li < nloop; li += gstride()) {
    first_out[li] = first[li];
    npts_out[li] = npts[li];
    radius_out[li] = radius[li];
    state_out[li] = state[li];
  }
}

int check_sizes(int64_t nv, int64_t nt, const char* what) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL && nt >= 0 && nt <= 0x7fffffffLL / 6, B2V_ERR_ARG,
              "%s: need V < 2^31 and 6T < 2^31", what);
  return B2V_OK;
}

}  // namespace

extern "C" int64_t b2v_holes_workspace_bytes(int64_t nv, int64_t nt) {
  if (nv < 0 || nt < 0) return -1;
  return (int64_t)carve(nullptr, nv, nt).bytes;
}

extern "C" int b2v_holes_layout(int64_t nv, int64_t nt, int64_t* layout_out) {
  B2V_REQUIRE(nv >= 0 && nt >= 0 && layout_out, B2V_ERR_ARG, "holes_layout: bad arguments");
  const FhWs w = carve(nullptr, nv, nt);
  layout_out[0] = (int64_t)((char*)w.lines - (char*)nullptr);     // int32 [lines][2]: the boundary lines
  layout_out[1] = (int64_t)((char*)w.poly - (char*)nullptr);      // int32 [points]: the loops' points
  layout_out[2] = (int64_t)((char*)w.off - (char*)nullptr);       // uint64 [loops]: where each loop starts
  layout_out[3] = (int64_t)((char*)w.npts - (char*)nullptr);      // int32 [loops]: its points
  return B2V_OK;
}

extern "C" int b2v_holes_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                               int faces_i64, double hole_size, void* workspace, void* stream,
                               int64_t* counts_host) {
  if (int rc = check_sizes(nv, nt, "holes_count")) return rc;
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "holes_count: faces must be [T,3] or [T,4]");
  B2V_REQUIRE(faces_i64 == 0 || faces_i64 == 1, B2V_ERR_ARG, "holes_count: faces_i64 must be 0 or 1");
  B2V_REQUIRE(nt == 0 || nv > 0, B2V_ERR_ARG, "holes_count: faces without vertices");
  B2V_REQUIRE(!(hole_size != hole_size), B2V_ERR_ARG, "holes_count: the hole size is NaN");
  B2V_REQUIRE((nv == 0 || verts) && (nt == 0 || faces) && workspace && counts_host, B2V_ERR_ARG,
              "holes_count: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  counts_host[0] = counts_host[1] = counts_host[2] = 0;
  if (nt == 0) return B2V_OK;
  hole_size = hole_size < 0.0 ? 0.0 : (hole_size > (double)FLT_MAX ? (double)FLT_MAX : hole_size);
  FhWs w = carve(workspace, nv, nt);
  const int64_t L = 3 * nt, D = 2 * L;
  B2V_CUDA(cudaMemsetAsync(w.ctl, 0, 32 * 8, s));
  const Faces F{faces, nt, face_cols, faces_i64, nv};
  if (int rc = build_links(w, F, "fill_holes", s)) return rc;

  // boundary lines in VTK's order
  const unsigned g3 = b2v_grid(L, kBlock, 16);
  k_fh_edges<<<g3, kBlock, 0, s>>>(w.tri, w.lstart, w.links, nt, w.lpos);
  if (int rc = b2v_check_launch("k_fh_edges")) return rc;
  B2V_CUDA(cudaMemsetAsync(w.lpos + L, 0, 8, s));
  if (int rc = scan(w.lpos, L + 1, w.scratch, w.ctl + C_LINES, s)) return rc;
  B2V_CUDA(cudaMemsetAsync(w.deg, 0, (size_t)nv * 4, s));
  k_fh_lines<<<g3, kBlock, 0, s>>>(w.tri, w.lpos, nt, w.lines, w.deg, w.slot);
  if (int rc = b2v_check_launch("k_fh_lines")) return rc;

  // darts, pointer jumping, loops
  const unsigned gd = b2v_grid(D, kBlock, 16);
  k_fh_darts<<<gd, kBlock, 0, s>>>(w.lines, w.deg, w.slot, w.ctl, w.succ, w.nx[0], w.dd[0], w.mn[0], w.last[0]);
  if (int rc = b2v_check_launch("k_fh_darts")) return rc;
  Pj J{{w.nx[0], w.nx[1]}, {w.dd[0], w.dd[1]}, {w.mn[0], w.mn[1]}, {w.last[0], w.last[1]}, w.ctl};
  void* args[] = {&J};
  if (int rc = launch_coop((const void*)k_fh_jump, args, s, "fill_holes", "k_fh_jump")) return rc;
  B2V_CUDA(cudaMemsetAsync(w.lkey, 0, (size_t)(L + 1) * 8, s));
  k_fh_loops<<<gd, kBlock, 0, s>>>(w.lines, w.deg, w.succ, J, w.lkey, w.lsd, w.lterm);
  if (int rc = b2v_check_launch("k_fh_loops")) return rc;
  if (int rc = scan(w.lkey, L + 1, w.scratch, w.ctl + C_PACK, s)) return rc;
  B2V_CUDA(cudaMemsetAsync(w.dloop, 0xff, (size_t)D * 4, s));
  k_fh_records<<<g3, kBlock, 0, s>>>(w.lines, w.lkey, w.lsd, w.lterm, J, w.dloop, w.poly, w.first, w.npts,
                                     w.off);
  if (int rc = b2v_check_launch("k_fh_records")) return rc;
  k_fh_points<<<gd, kBlock, 0, s>>>(w.lines, J, w.dloop, w.npts, w.off, w.poly);
  if (int rc = b2v_check_launch("k_fh_points")) return rc;

  // size test and triangulation
  k_fh_sphere<<<g3, kBlock, 0, s>>>(verts, w.poly, w.npts, w.off, w.ctl, hole_size, w.radius, w.state);
  if (int rc = b2v_check_launch("k_fh_sphere")) return rc;
  Tr K{verts, w.poly, w.npts, w.off, w.ctl, w.state, w.prv, w.nxt, w.key, w.otri, w.toff, w.ctl + C_TRIS};
  k_fh_tri<<<b2v_grid(L, 1, 4), kBlock, 0, s>>>(K);
  if (int rc = b2v_check_launch("k_fh_tri")) return rc;

  unsigned long long ctl[3];
  B2V_CUDA(cudaMemcpyAsync(ctl, w.ctl, sizeof(ctl), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  counts_host[0] = (int64_t)ctl[C_LINES];
  counts_host[1] = (int64_t)(ctl[C_PACK] >> 32);
  counts_host[2] = (int64_t)ctl[C_TRIS];
  return B2V_OK;
}

extern "C" int b2v_holes_emit(const void* faces, int64_t nv, int64_t nt, int face_cols, int faces_i64,
                              const int64_t* counts_host, void* workspace, void* faces_out, int64_t* first_line,
                              int64_t* npts, double* radius, int8_t* status, void* stream) {
  if (int rc = check_sizes(nv, nt, "holes_emit")) return rc;
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "holes_emit: faces must be [T,3] or [T,4]");
  B2V_REQUIRE(faces_i64 == 0 || faces_i64 == 1, B2V_ERR_ARG, "holes_emit: faces_i64 must be 0 or 1");
  B2V_REQUIRE(counts_host && (nt == 0 || (faces && workspace && faces_out)), B2V_ERR_ARG,
              "holes_emit: null argument");
  const int64_t nloop = counts_host[1];
  B2V_REQUIRE(nloop >= 0 && nloop <= 3 * nt && counts_host[2] >= 0 && counts_host[2] <= 3 * nt, B2V_ERR_ARG,
              "holes_emit: counts do not come from holes_count");
  B2V_REQUIRE(nloop == 0 || (first_line && npts && radius && status), B2V_ERR_ARG, "holes_emit: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  if (nt == 0) return B2V_OK;
  const size_t row = (size_t)face_cols * (faces_i64 ? 8 : 4);
  B2V_CUDA(cudaMemcpyAsync(faces_out, faces, (size_t)nt * row, cudaMemcpyDeviceToDevice, s));
  if (nloop == 0) return B2V_OK;
  FhWs w = carve(workspace, nv, nt);
  B2V_CUDA(cudaMemsetAsync(w.toff + nloop, 0, 8, s));
  if (int rc = scan(w.toff, nloop + 1, w.scratch, nullptr, s)) return rc;
  k_fh_emit<<<b2v_grid(nloop, 1, 8), kBlock, 0, s>>>(w.otri, w.off, w.toff, nloop, nt, face_cols, faces_i64,
                                                     faces_out);
  if (int rc = b2v_check_launch("k_fh_emit")) return rc;
  k_fh_out<<<b2v_grid(nloop, kBlock, 16), kBlock, 0, s>>>(w.first, w.npts, w.radius, w.state, nloop, first_line,
                                                          npts, radius, status);
  return b2v_check_launch("k_fh_out");
}
