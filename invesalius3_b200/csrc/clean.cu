// vtkCleanPolyData (point merging at tolerance 0, unused points removed, polys -> lines -> verts and strips ->
// polys -> lines -> verts) and vtkTriangleFilter on the polys and strips of a surface, on the device. The
// rules are those stated in the header of the C checker (clean.c), which reproduces every output array.
//
// Cells come in two families, polys then strips, each as offsets + connectivity (VTK 9's cell arrays) or as
// faces [n,3] / [n,4] with a leading 3. Corners are numbered over both families in traversal order (the polys'
// connectivity, then the strips'), cells likewise (polys, then strips).
//
// Clean:
//   k_cl_check_*      malformed offsets (not starting at 0, decreasing, not ending at the connectivity's
//                     length) and ids outside [0, V) set status bits; the count call reports them first.
//   k_merge_insert    mesh_merge.cuh: exactly coincident points share one hash slot.
//   k_cl_first_use    note_first_use over every corner.
//   k_cl_mark / k_cl_corner_flags   per corner: whether it is the first use of its slot (it numbers an
//                     output point) and whether it survives the removal of consecutive repeats (the first
//                     corner of a cell, or a slot other than the previous corner's).
//   k_cl_cells        per cell: kept corners = a difference of the corner scan; a poly whose last kept slot is
//                     its first drops the last; the category (vert, line, poly, strip) and its counts.
//   scans             the corner flags, then per category the cell and corner counts (six scans).
//   k_cl_emit_*       points and point_ids per first-use corner, offsets and cell_ids per cell, connectivity
//                     per kept corner (the cell of a corner: k / 3 for faces, a binary search of the offsets).
//
// Triangle filter:
//   k_tf_count        per cell: 1 for a triangle, n - 2 for a strip of n points, 0 below that.
//   k_tf_polygons     vtkPolygon's ear cut of each poly of more than 3 points: one warp per polygon of at most
//                     kPolyWarpMax points, one block per longer one (as k_fh_tri). The group's leader keeps the
//                     ring and the queue; the argmin over the queued measures and the split-plane test of a
//                     non-convex ear are spread over the group. The triangles go to a scratch area at the
//                     polygon's corner offset, their number to the cell's count.
//   k_tf_emit         per corner at position j >= 2 of a triangle or strip: triangle j - 2, with
//                     vtkTriangleStrip's alternating winding; per corner j of a clipped polygon: its triangle j
//                     from the scratch area; and the cell ids.
//
// Every pass is a stream over the corners or the cells plus the random 4-byte gathers of the hash slots; the
// scans are scan.cuh's device-wide scan.
#include <float.h>

#include "b2v_common.cuh"
#include "mesh_merge.cuh"
#include "scan.cuh"

namespace {

constexpr int kBlock = 256;

enum : uint32_t { ST_BAD_OFFSETS = 2u };   // beside ST_BAD_FACE (1)
constexpr int kPolyWarpMax = 256;   // longer polygons are clipped by a whole block
enum : uint8_t { CAT_NONE = 0, CAT_VERT = 1, CAT_LINE = 2, CAT_POLY = 3, CAT_STRIP = 4 };
enum { K_VERT = 0, K_LINE = 1, K_POLY = 2, K_STRIP = 3, K_PCONN = 4, K_SCONN = 5, K_ROWS = 6 };

struct Cells {
  const void* conn;
  const int64_t* offs;   // [n + 1] with form 0, else null
  int64_t n;             // cells
  int64_t nconn;         // corners
  int form;              // 0: offsets + connectivity; 3: [n,3]; 4: [n,4] with a leading 3
  int i64;
};

__device__ __forceinline__ int64_t cell_start(const Cells& C, int64_t c) { return C.form ? 3 * c : C.offs[c]; }

__device__ __forceinline__ int64_t corner_pt(const Cells& C, int64_t k) {
  const int64_t at = C.form == 4 ? (k / 3) * 4 + 1 + k % 3 : k;
  return C.i64 ? ((const int64_t*)C.conn)[at] : (int64_t)((const int32_t*)C.conn)[at];
}

// the cell holding corner k: the last c with offs[c] <= k
__device__ __forceinline__ int64_t cell_of(const Cells& C, int64_t k) {
  if (C.form) return k / 3;
  int64_t lo = 0, hi = C.n - 1;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo + 1) / 2;
    if (C.offs[mid] <= k) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// polys, then strips: global cell g and corner k
struct Mesh {
  Cells p, s;
  int64_t nv;
  __device__ __forceinline__ int64_t cells() const { return p.n + s.n; }
  __device__ __forceinline__ int64_t corners() const { return p.nconn + s.nconn; }
  __device__ __forceinline__ int64_t pt(int64_t k) const { return k < p.nconn ? corner_pt(p, k) : corner_pt(s, k - p.nconn); }
  __device__ __forceinline__ int64_t start(int64_t g) const {
    return g < p.n ? cell_start(p, g) : p.nconn + cell_start(s, g - p.n);
  }
  __device__ __forceinline__ int64_t cell(int64_t k) const {
    return k < p.nconn ? cell_of(p, k) : p.n + cell_of(s, k - p.nconn);
  }
};

// ---- input checks ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_cl_check_cells(Cells C, uint32_t* status) {
  for (int64_t c = gtid(); c < C.n; c += gstride()) {
    bool bad = false;
    if (C.form == 0) {
      const int64_t a = C.offs[c], b = C.offs[c + 1];
      bad = a > b || (c == 0 && a != 0) || (c == C.n - 1 && b != C.nconn);
    } else if (C.form == 4) {
      const int64_t lead = C.i64 ? ((const int64_t*)C.conn)[4 * c] : ((const int32_t*)C.conn)[4 * c];
      if (lead != 3) atomicOr(status, (uint32_t)ST_BAD_FACE);
    }
    if (bad) atomicOr(status, (uint32_t)ST_BAD_OFFSETS);
  }
}

__global__ void __launch_bounds__(kBlock) k_cl_check_corners(Cells C, int64_t nv, uint32_t* status) {
  bool bad = false;
  for (int64_t k = gtid(); k < C.nconn; k += gstride()) {
    const int64_t p = corner_pt(C, k);
    bad |= p < 0 || p >= nv;
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(status, (uint32_t)ST_BAD_FACE);
}

// ---- workspace ------------------------------------------------------------------------------------------------
struct ClWs {
  uint32_t* status;
  unsigned long long* totals;   // [0] points, [1] kept corners, [2 + K_*] category totals
  int32_t* slots;               // [H]
  uint32_t* rep;                // [V]
  unsigned long long* first;    // [H]
  int32_t* newid;               // [H]
  unsigned long long* fscan;    // [C + 1] first-use flags, then their exclusive scan
  unsigned long long* kscan;    // [C + 1] kept-corner flags, then their exclusive scan
  unsigned long long* cnt;      // [K_ROWS][G + 1]
  int64_t* ncell;               // [G] kept corners of the cell
  uint8_t* cat;                 // [G]
  unsigned long long* scratch;  // scan_blocks(max(C, G) + 1) + 1
  uint64_t hmask;
  size_t bytes;
};

ClWs carve_clean(void* base, int64_t nv, int64_t G, int64_t C) {
  ClWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const uint64_t H = merge_slots(nv);
  w.hmask = H - 1;
  w.status = (uint32_t*)take(16);
  w.totals = (unsigned long long*)take(8 * 8);
  w.slots = (int32_t*)take(H * 4);
  w.rep = (uint32_t*)take((size_t)nv * 4);
  w.first = (unsigned long long*)take(H * 8);
  w.newid = (int32_t*)take(H * 4);
  w.fscan = (unsigned long long*)take((size_t)(C + 1) * 8);
  w.kscan = (unsigned long long*)take((size_t)(C + 1) * 8);
  w.cnt = (unsigned long long*)take((size_t)K_ROWS * (G + 1) * 8);
  w.ncell = (int64_t*)take((size_t)G * 8);
  w.cat = (uint8_t*)take((size_t)G);
  w.scratch = (unsigned long long*)take((size_t)(scan_blocks((C > G ? C : G) + 1) + 1) * 8);
  w.bytes = o;
  return w;
}

struct TfWs {
  uint32_t* status;
  unsigned long long* totals;   // [0] triangles
  unsigned long long* tcnt;     // [G + 1] triangles per cell, then their exclusive scan
  unsigned long long* scratch;
  int32_t* prv;                 // [poly corners] the ring of each clipped polygon, by position
  int32_t* nxt;
  double* key;                  // [poly corners] measures
  uint8_t* inq;                 // [poly corners] in the queue
  uint8_t* alive;               // [poly corners] still in the ring
  int64_t* tri;                 // [poly corners][3] the triangles of a polygon at its corner offset
  size_t bytes;
};

TfWs carve_tri(void* base, int64_t G, int64_t PC) {
  TfWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  w.status = (uint32_t*)take(16);
  w.totals = (unsigned long long*)take(8);
  w.tcnt = (unsigned long long*)take((size_t)(G + 1) * 8);
  w.scratch = (unsigned long long*)take((size_t)(scan_blocks(G + 1) + 1) * 8);
  w.prv = (int32_t*)take((size_t)PC * 4);
  w.nxt = (int32_t*)take((size_t)PC * 4);
  w.key = (double*)take((size_t)PC * 8);
  w.inq = (uint8_t*)take((size_t)PC);
  w.alive = (uint8_t*)take((size_t)PC);
  w.tri = (int64_t*)take((size_t)PC * 24);
  w.bytes = o;
  return w;
}

// ---- clean ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_cl_first_use(Mesh M, const uint32_t* __restrict__ rep,
                                                         unsigned long long* first) {
  const int64_t C = M.corners();
  for (int64_t k = gtid(); k < C; k += gstride()) note_first_use(first, rep[M.pt(k)], (unsigned long long)k);
}

__global__ void __launch_bounds__(kBlock) k_cl_mark(Mesh M, unsigned long long* __restrict__ kscan) {
  const int64_t G = M.cells();
  for (int64_t g = gtid(); g < G; g += gstride()) {
    const int64_t s = M.start(g), e = g + 1 < G ? M.start(g + 1) : M.corners();
    if (s < e) kscan[s] = 1;   // the first corner of a non-empty cell
  }
}

__global__ void __launch_bounds__(kBlock) k_cl_corner_flags(Mesh M, const uint32_t* __restrict__ rep,
                                                            const unsigned long long* __restrict__ first,
                                                            unsigned long long* __restrict__ fscan,
                                                            unsigned long long* __restrict__ kscan) {
  const int64_t C = M.corners();
  for (int64_t k = gtid(); k < C; k += gstride()) {
    const uint32_t r = rep[M.pt(k)];
    fscan[k] = is_first_use(first, r, (unsigned long long)k) ? 1ull : 0ull;
    if (kscan[k] == 0) kscan[k] = r != rep[M.pt(k - 1)] ? 1ull : 0ull;   // not a cell's first corner: k >= 1
  }
}

__global__ void __launch_bounds__(kBlock) k_cl_cells(Mesh M, const uint32_t* __restrict__ rep,
                                                     const unsigned long long* __restrict__ kscan, int64_t rowlen,
                                                     unsigned long long* __restrict__ cnt, int64_t* __restrict__ ncell,
                                                     uint8_t* __restrict__ cat) {
  const int64_t G = M.cells(), Cn = M.corners();
  for (int64_t g = gtid(); g < G; g += gstride()) {
    const int64_t s = M.start(g), e = g + 1 < G ? M.start(g + 1) : Cn;
    const bool poly = g < M.p.n;
    int64_t n = s < e ? (int64_t)(kscan[e] - kscan[s]) : 0;
    if (poly && n > 2 && rep[M.pt(s)] == rep[M.pt(e - 1)]) --n;   // the last point repeats the first
    uint8_t c = CAT_NONE;
    if (n >= (poly ? 3 : 4)) c = poly ? CAT_POLY : CAT_STRIP;
    else if (n == 3) c = CAT_POLY;
    else if (n == 2) c = CAT_LINE;
    else if (n == 1) c = CAT_VERT;
    ncell[g] = n;
    cat[g] = c;
    cnt[K_VERT * rowlen + g] = c == CAT_VERT;
    cnt[K_LINE * rowlen + g] = c == CAT_LINE;
    cnt[K_POLY * rowlen + g] = c == CAT_POLY;
    cnt[K_STRIP * rowlen + g] = c == CAT_STRIP;
    cnt[K_PCONN * rowlen + g] = c == CAT_POLY ? (unsigned long long)n : 0ull;
    cnt[K_SCONN * rowlen + g] = c == CAT_STRIP ? (unsigned long long)n : 0ull;
  }
}

__global__ void __launch_bounds__(kBlock) k_cl_emit_points(Mesh M, const float* __restrict__ P,
                                                           const uint32_t* __restrict__ rep,
                                                           const unsigned long long* __restrict__ fscan,
                                                           int32_t* __restrict__ newid, float* __restrict__ pts,
                                                           int64_t* __restrict__ point_ids) {
  const int64_t C = M.corners();
  for (int64_t k = gtid(); k < C; k += gstride()) {
    const unsigned long long id = fscan[k];
    if (fscan[k + 1] == id) continue;   // not a first use
    const int64_t p = M.pt(k);
    newid[rep[p]] = (int32_t)id;
    pts[3 * id] = P[3 * p];
    pts[3 * id + 1] = P[3 * p + 1];
    pts[3 * id + 2] = P[3 * p + 2];
    point_ids[id] = p;
  }
}

struct ClOut {
  int64_t* vconn;
  int64_t* lconn;
  int64_t* poffs;
  int64_t* pconn;
  int64_t* soffs;
  int64_t* sconn;
  int64_t* cell_ids;   // verts, lines, polys, strips
};

__global__ void __launch_bounds__(kBlock) k_cl_emit_cells(Mesh M, const unsigned long long* __restrict__ cnt,
                                                          int64_t rowlen, const uint8_t* __restrict__ cat,
                                                          const unsigned long long* __restrict__ totals, ClOut O) {
  const int64_t G = M.cells();
  const unsigned long long nvc = totals[2 + K_VERT], nlc = totals[2 + K_LINE], npc = totals[2 + K_POLY];
  if (gtid() == 0) {
    O.poffs[npc] = (int64_t)totals[2 + K_PCONN];
    O.soffs[totals[2 + K_STRIP]] = (int64_t)totals[2 + K_SCONN];
  }
  for (int64_t g = gtid(); g < G; g += gstride()) {
    switch (cat[g]) {
      case CAT_VERT: O.cell_ids[cnt[K_VERT * rowlen + g]] = g; break;
      case CAT_LINE: O.cell_ids[nvc + cnt[K_LINE * rowlen + g]] = g; break;
      case CAT_POLY: {
        const unsigned long long i = cnt[K_POLY * rowlen + g];
        O.cell_ids[nvc + nlc + i] = g;
        O.poffs[i] = (int64_t)cnt[K_PCONN * rowlen + g];
        break;
      }
      case CAT_STRIP: {
        const unsigned long long i = cnt[K_STRIP * rowlen + g];
        O.cell_ids[nvc + nlc + npc + i] = g;
        O.soffs[i] = (int64_t)cnt[K_SCONN * rowlen + g];
        break;
      }
      default: break;
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_cl_emit_corners(Mesh M, const uint32_t* __restrict__ rep,
                                                            const unsigned long long* __restrict__ kscan,
                                                            const unsigned long long* __restrict__ cnt, int64_t rowlen,
                                                            const int64_t* __restrict__ ncell,
                                                            const uint8_t* __restrict__ cat,
                                                            const int32_t* __restrict__ newid, ClOut O) {
  const int64_t C = M.corners();
  for (int64_t k = gtid(); k < C; k += gstride()) {
    if (kscan[k + 1] == kscan[k]) continue;   // a repeat of the previous corner
    const int64_t g = M.cell(k);
    const int64_t pos = (int64_t)(kscan[k] - kscan[M.start(g)]);
    if (pos >= ncell[g]) continue;            // a poly's last point that repeats its first
    const int64_t id = newid[rep[M.pt(k)]];
    switch (cat[g]) {
      case CAT_VERT: O.vconn[cnt[K_VERT * rowlen + g]] = id; break;
      case CAT_LINE: O.lconn[2 * cnt[K_LINE * rowlen + g] + pos] = id; break;
      case CAT_POLY: O.pconn[cnt[K_PCONN * rowlen + g] + pos] = id; break;
      case CAT_STRIP: O.sconn[cnt[K_SCONN * rowlen + g] + pos] = id; break;
      default: break;
    }
  }
}

// ---- triangle filter ------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t cell_end(const Mesh& M, int64_t g) {
  return g + 1 < M.cells() ? M.start(g + 1) : M.corners();
}

__global__ void __launch_bounds__(kBlock) k_tf_count(Mesh M, unsigned long long* __restrict__ tcnt) {
  const int64_t G = M.cells();
  for (int64_t g = gtid(); g < G; g += gstride()) {
    const int64_t n = cell_end(M, g) - M.start(g);
    int64_t t = 0;
    if (g < M.p.n) t = n == 3 ? 1 : 0;   // longer polygons: k_tf_polygons
    else t = n > 2 ? n - 2 : 0;
    tcnt[g] = (unsigned long long)t;
  }
}

// ---- vtkPolygon::EarCutTriangulation (rule 10 of the checker's header), in double ------------------------
struct Ring {
  const float* P;
  const Cells* C;   // the polys
  int64_t s;        // the polygon's first corner
  __device__ __forceinline__ void x(int32_t i, double r[3]) const {
    const int64_t p = corner_pt(*C, s + i);
    r[0] = (double)P[3 * p]; r[1] = (double)P[3 * p + 1]; r[2] = (double)P[3 * p + 2];
  }
};

__device__ __forceinline__ void sub3(const double* a, const double* b, double* r) {
  r[0] = a[0] - b[0]; r[1] = a[1] - b[1]; r[2] = a[2] - b[2];
}
__device__ __forceinline__ double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
__device__ __forceinline__ double len3(const double* a) { return sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]); }
__device__ __forceinline__ void cross3(const double* a, const double* b, double* n) {
  n[0] = a[1] * b[2] - a[2] * b[1];
  n[1] = a[2] * b[0] - a[0] * b[2];
  n[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double normalize3(double* a) {
  const double d = len3(a);
  if (d != 0.0) { a[0] /= d; a[1] /= d; a[2] /= d; }
  return d;
}

__device__ double ear_measure(const Ring& R, int32_t prev, int32_t v, int32_t next, const double* N) {
  double a[3], b[3], c[3], v1[3], v2[3], v3[3], cr[3];
  R.x(prev, a); R.x(v, b); R.x(next, c);
  sub3(b, a, v1); sub3(c, b, v2); sub3(a, c, v3);
  cross3(v1, v2, cr);
  const double area = dot3(cr, N);
  if (area < 0.0) return -1.0;
  if (area == 0.0) return -DBL_MAX;
  const double p = (len3(v1) + len3(v2)) + len3(v3);
  return p * p / area;
}

__device__ bool segments_meet(const double* a1, const double* a2, const double* b1, const double* b2) {
  double a[3], b[3], c[3];
  sub3(a2, a1, a); sub3(b2, b1, b); sub3(b1, a1, c);
  const double r00 = dot3(a, a), r01 = -dot3(a, b), r11 = dot3(b, b), c0 = dot3(a, c), c1 = -dot3(b, c);
  const double det = r00 * r11 - r01 * r01;
  if (det == 0.0) return true;
  const double u = (r11 * c0 - r01 * c1) / det, w = (-r01 * c0 + r00 * c1) / det;
  return 0.0 <= u && u <= 1.0 && 0.0 <= w && w <= 1.0;
}

__device__ __forceinline__ int side(const double* sN, const double* o, const double* x, double tol) {
  const double e = (sN[0] * (x[0] - o[0]) + sN[1] * (x[1] - o[1])) + sN[2] * (x[2] - o[2]);
  return e > tol ? 1 : (e < -tol ? -1 : 0);
}

// (key, position) order: the smaller key, then the lower position; +inf keys stand for "not queued"
__device__ __forceinline__ void better(double& k, int32_t& i, double ok, int32_t oi) {
  if (ok < k || (ok == k && oi < i)) { k = ok; i = oi; }
}

struct PolyState {
  int32_t head, m, nq, made, best, removable;
  double N[3], tol;
};

// A group of NW warps clips one polygon at a time; NW == 1: 8 groups a block, NW == 8: the whole block.
template <int NW>
__global__ void __launch_bounds__(kBlock) k_tf_polygons(Mesh M, const float* __restrict__ P, TfWs w) {
  constexpr int GN = 32 * NW, GPB = kBlock / GN;
  __shared__ PolyState s_st[GPB];
  __shared__ double s_k[kBlock / 32];
  __shared__ int32_t s_i[kBlock / 32];
  const int lane = threadIdx.x % GN, gid = threadIdx.x / GN, wid = threadIdx.x >> 5;
  PolyState& S = s_st[gid];
  auto sync = [] { if (NW == 1) __syncwarp(); else __syncthreads(); };
  const int64_t np = M.p.n;
  for (int64_t c = (int64_t)blockIdx.x * GPB + gid; c < np; c += (int64_t)gridDim.x * GPB) {
    const int64_t s = cell_start(M.p, c), e = c + 1 < np ? cell_start(M.p, c + 1) : M.p.nconn;
    const int32_t n = (int32_t)(e - s);
    if (n <= 3 || (NW == 1) != (n <= kPolyWarpMax)) continue;   // uniform over the group
    const Ring R{P, &M.p, s};
    int32_t *prv = w.prv + s, *nxt = w.nxt + s;
    double* key = w.key + s;
    uint8_t *inq = w.inq + s, *alive = w.alive + s;
    int64_t* tri = w.tri + 3 * s;
    if (lane == 0) {   // bounds, the ring without near-coincident points, the normal, the first queue
      double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
      for (int32_t i = 0; i < n; ++i) {
        double x[3];
        R.x(i, x);
        for (int k = 0; k < 3; ++k) { lo[k] = x[k] < lo[k] ? x[k] : lo[k]; hi[k] = x[k] > hi[k] ? x[k] : hi[k]; }
        nxt[i] = i + 1 < n ? i + 1 : 0;
        prv[i] = i > 0 ? i - 1 : n - 1;
        inq[i] = 0;
        alive[i] = 0;
      }
      const double ext[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
      const double tol = 1e-6 * len3(ext), tol2 = tol * tol;
      int32_t head = 0, m = n, v = 0;
      for (int32_t i = 0; i < n; ++i) {
        const int32_t u = nxt[v];
        double a[3], b[3], d[3];
        R.x(v, a); R.x(u, b);
        sub3(a, b, d);
        if ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] < tol2) {
          prv[nxt[u]] = v;
          nxt[v] = nxt[u];
          if (u == head) head = v;
          --m;
        } else {
          v = u;
        }
      }
      double N[3] = {0.0, 0.0, 0.0}, h[3];
      R.x(head, h);
      for (v = nxt[head]; nxt[v] != head; v = nxt[v]) {
        double a[3], b[3], v1[3], v2[3], cr[3];
        R.x(v, a); R.x(nxt[v], b);
        sub3(a, h, v1); sub3(b, h, v2);
        cross3(v1, v2, cr);
        for (int k = 0; k < 3; ++k) N[k] += cr[k];
      }
      int32_t nq = 0;
      if (normalize3(N) == 0.0) {
        m = 0;   // no triangle
      } else {
        v = head;
        for (int32_t i = 0; i < m; ++i, v = nxt[v]) {
          alive[v] = 1;
          key[v] = ear_measure(R, prv[v], v, nxt[v], N);
          if (key[v] > 0.0) { inq[v] = 1; ++nq; }
        }
      }
      S.head = head; S.m = m; S.nq = nq; S.made = 0; S.tol = tol;
      S.N[0] = N[0]; S.N[1] = N[1]; S.N[2] = N[2];
    }
    sync();
    const double N[3] = {S.N[0], S.N[1], S.N[2]}, tol = S.tol;
    while (S.m > 2 && S.nq > 0) {
      const int32_t m = S.m;
      const bool convex = S.nq == m;
      // the queued vertex of the smallest measure, the lowest position on a tie
      double bk = INFINITY;
      int32_t bi = INT32_MAX;
      for (int32_t i = lane; i < n; i += GN)
        if (inq[i]) better(bk, bi, key[i], i);
      for (int o = 16; o > 0; o >>= 1)
        better(bk, bi, __shfl_xor_sync(0xffffffffu, bk, o), __shfl_xor_sync(0xffffffffu, bi, o));
      if (NW > 1) {
        if ((threadIdx.x & 31) == 0) { s_k[wid] = bk; s_i[wid] = bi; }
        __syncthreads();
        bk = INFINITY; bi = INT32_MAX;
        for (int k = 0; k < NW; ++k) better(bk, bi, s_k[k], s_i[k]);
      }
      // queued measures may be +inf; an empty slot has bi == INT32_MAX, and the queue is not empty
      bool ok = convex || m <= 3;
      if (!ok) {   // the split-plane test over the rest of the ring, spread over the group
        const int32_t pv = prv[bi], nx = nxt[bi], nn = nxt[nx];
        double a[3], b[3], d[3], sN[3];
        R.x(pv, a); R.x(nx, b);
        sub3(b, a, d);
        cross3(d, N, sN);
        const bool split = normalize3(sN) != 0.0;
        bool neg = false, hit = false;
        if (split)
          for (int32_t u = lane; u < n; u += GN) {
            if (!alive[u] || u == bi || u == pv || u == nx) continue;
            double x[3];
            R.x(u, x);
            const int sg = side(sN, a, x, tol);
            neg |= sg < 0;
            if (u == nn) continue;
            double y[3];
            R.x(prv[u], y);
            if (sg != side(sN, a, y, tol) && segments_meet(a, b, x, y)) hit = true;
          }
        if (NW == 1) {
          neg = __any_sync(0xffffffffu, neg);
          hit = __any_sync(0xffffffffu, hit);
        } else {
          neg = __syncthreads_or(neg);
          hit = __syncthreads_or(hit);
        }
        ok = split && neg && !hit;
      }
      sync();
      if (lane == 0) {
        inq[bi] = 0;
        --S.nq;
        if (ok) {
          const int32_t pv = prv[bi], nx = nxt[bi];
          const int32_t t = S.made++;
          tri[3 * t] = corner_pt(M.p, s + bi);
          tri[3 * t + 1] = corner_pt(M.p, s + nx);
          tri[3 * t + 2] = corner_pt(M.p, s + pv);
          if (--S.m >= 3) {
            if (bi == S.head) S.head = nx;
            nxt[pv] = nx;
            prv[nx] = pv;
            alive[bi] = 0;
            const int32_t nb[2] = {pv, nx};
            for (int j = 0; j < 2; ++j) {
              const int32_t u = nb[j];
              if (inq[u]) { inq[u] = 0; --S.nq; }
              key[u] = ear_measure(R, prv[u], u, nxt[u], N);
              if (key[u] > 0.0) { inq[u] = 1; ++S.nq; }
            }
          }
        }
      }
      sync();
    }
    if (lane == 0) w.tcnt[c] = (unsigned long long)S.made;
    sync();
  }
}

__global__ void __launch_bounds__(kBlock) k_tf_emit(Mesh M, const unsigned long long* __restrict__ tcnt,
                                                    const int64_t* __restrict__ ptri, int64_t* __restrict__ tris,
                                                    int64_t* __restrict__ cell_ids) {
  const int64_t C = M.corners();
  for (int64_t k = gtid(); k < C; k += gstride()) {
    const int64_t g = M.cell(k), s = M.start(g), j = k - s;
    const unsigned long long t0 = tcnt[g], nt = tcnt[g + 1] - t0;
    if (g < M.p.n && cell_end(M, g) - s > 3) {   // a clipped polygon: its triangle j, if any
      if ((unsigned long long)j >= nt) continue;
      for (int c = 0; c < 3; ++c) tris[3 * (t0 + j) + c] = ptri[3 * k + c];
      cell_ids[t0 + j] = g;
      continue;
    }
    if (j < 2 || nt == 0) continue;   // not a triangle's last corner, or a cell with none
    const int64_t i = j - 2;
    const unsigned long long t = t0 + (unsigned long long)i;
    const int64_t a = M.pt(k - 2), b = M.pt(k - 1), c = M.pt(k);
    const bool odd = g >= M.p.n && (i & 1);   // vtkTriangleStrip::DecomposeStrip flips every other one
    tris[3 * t] = odd ? b : a;
    tris[3 * t + 1] = odd ? a : b;
    tris[3 * t + 2] = c;
    cell_ids[t] = g;
  }
}

// ---- host -----------------------------------------------------------------------------------------------------
Cells make_cells(const void* conn, const int64_t* offs, int64_t n, int64_t nconn, int form, int i64) {
  Cells c;
  c.conn = conn; c.offs = offs; c.n = n; c.nconn = nconn; c.form = form; c.i64 = i64;
  return c;
}

int check_cells_args(const Cells& C, const char* what, const char* fam) {
  B2V_REQUIRE(C.form == 0 || C.form == 3 || C.form == 4, B2V_ERR_ARG, "%s: %s form must be 0, 3 or 4", what, fam);
  B2V_REQUIRE(C.i64 == 0 || C.i64 == 1, B2V_ERR_ARG, "%s: %s i64 must be 0 or 1", what, fam);
  B2V_REQUIRE(C.n >= 0 && C.nconn >= 0, B2V_ERR_ARG, "%s: negative %s sizes", what, fam);
  if (C.form) B2V_REQUIRE(C.nconn == 3 * C.n, B2V_ERR_ARG, "%s: %s faces give 3 corners a cell", what, fam);
  B2V_REQUIRE(C.nconn == 0 || C.conn, B2V_ERR_ARG, "%s: null %s connectivity", what, fam);
  B2V_REQUIRE(C.form || C.n == 0 || C.offs, B2V_ERR_ARG, "%s: null %s offsets", what, fam);
  B2V_REQUIRE(C.form || C.n > 0 || C.nconn == 0, B2V_ERR_ARG, "%s: %s connectivity without cells", what, fam);
  return B2V_OK;
}

// the checks every call runs; status and the stream sync at the end report malformed input
int validate(const Mesh& M, uint32_t* status, const char* what, cudaStream_t s) {
  B2V_CUDA(cudaMemsetAsync(status, 0, 4, s));
  for (const Cells* C : {&M.p, &M.s}) {
    if (C->n > 0) {
      k_cl_check_cells<<<b2v_grid(C->n, kBlock, 8), kBlock, 0, s>>>(*C, status);
      if (int rc = b2v_check_launch("k_cl_check_cells")) return rc;
    }
    if (C->nconn > 0) {
      k_cl_check_corners<<<b2v_grid(C->nconn, kBlock, 8), kBlock, 0, s>>>(*C, M.nv, status);
      if (int rc = b2v_check_launch("k_cl_check_corners")) return rc;
    }
  }
  uint32_t st = 0;
  B2V_CUDA(cudaMemcpyAsync(&st, status, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!(st & ST_BAD_OFFSETS), B2V_ERR_ARG,
              "%s: malformed offsets (they must start at 0, never decrease and end at the connectivity's length)",
              what);
  B2V_REQUIRE(!(st & ST_BAD_FACE), B2V_ERR_ARG,
              "%s: a cell has a point id outside [0, V) (or a face a leading entry other than 3)", what);
  return B2V_OK;
}

int setup(const float* verts, int64_t nv, const Cells& p, const Cells& s, const char* what, Mesh* M) {
  B2V_REQUIRE(nv >= 0 && nv <= 0x7fffffffLL, B2V_ERR_ARG, "%s: need 0 <= V < 2^31", what);
  B2V_REQUIRE(nv == 0 || verts, B2V_ERR_ARG, "%s: null points", what);
  if (int rc = check_cells_args(p, what, "polys")) return rc;
  if (int rc = check_cells_args(s, what, "strips")) return rc;
  M->p = p; M->s = s; M->nv = nv;
  return B2V_OK;
}

}  // namespace

extern "C" int64_t b2v_clean_workspace_bytes(int64_t nv, int64_t ncells, int64_t ncorners) {
  if (nv < 0 || ncells < 0 || ncorners < 0) return -1;
  return (int64_t)carve_clean(nullptr, nv, ncells, ncorners).bytes;
}

extern "C" int b2v_clean_count(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs, int64_t np,
                               int64_t npconn, int pform, int pi64, const void* sconn, const int64_t* soffs, int64_t ns,
                               int64_t nsconn, int sform, int si64, void* workspace, void* stream,
                               int64_t* counts_host) {
  Mesh M;
  if (int rc = setup(verts, nv, make_cells(pconn, poffs, np, npconn, pform, pi64),
                     make_cells(sconn, soffs, ns, nsconn, sform, si64), "clean_polydata", &M))
    return rc;
  B2V_REQUIRE(workspace && counts_host, B2V_ERR_ARG, "clean_polydata: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t G = np + ns, C = npconn + nsconn;
  const ClWs w = carve_clean(workspace, nv, G, C);
  if (int rc = validate(M, w.status, "clean_polydata", s)) return rc;
  B2V_CUDA(cudaMemsetAsync(w.totals, 0, 8 * 8, s));
  if (C > 0) {
    if (int rc = merge_reset(w.slots, w.first, w.hmask + 1, s)) return rc;
    if (int rc = merge_points(verts, nv, w.hmask, w.slots, w.rep, s)) return rc;
    B2V_CUDA(cudaMemsetAsync(w.kscan, 0, (size_t)(C + 1) * 8, s));
    B2V_CUDA(cudaMemsetAsync(w.fscan + C, 0, 8, s));
    k_cl_first_use<<<b2v_grid(C, kBlock, 16), kBlock, 0, s>>>(M, w.rep, w.first);
    if (int rc = b2v_check_launch("k_cl_first_use")) return rc;
    k_cl_mark<<<b2v_grid(G, kBlock, 16), kBlock, 0, s>>>(M, w.kscan);
    if (int rc = b2v_check_launch("k_cl_mark")) return rc;
    k_cl_corner_flags<<<b2v_grid(C, kBlock, 16), kBlock, 0, s>>>(M, w.rep, w.first, w.fscan, w.kscan);
    if (int rc = b2v_check_launch("k_cl_corner_flags")) return rc;
    if (int rc = scan(w.fscan, C + 1, w.scratch, w.totals + 0, s)) return rc;
    if (int rc = scan(w.kscan, C + 1, w.scratch, w.totals + 1, s)) return rc;
  }
  if (G > 0) {
    B2V_CUDA(cudaMemsetAsync(w.cnt, 0, (size_t)K_ROWS * (G + 1) * 8, s));
    k_cl_cells<<<b2v_grid(G, kBlock, 16), kBlock, 0, s>>>(M, w.rep, w.kscan, G + 1, w.cnt, w.ncell, w.cat);
    if (int rc = b2v_check_launch("k_cl_cells")) return rc;
    for (int r = 0; r < K_ROWS; ++r)
      if (int rc = scan(w.cnt + (int64_t)r * (G + 1), G + 1, w.scratch, w.totals + 2 + r, s)) return rc;
  }
  unsigned long long tot[8];
  B2V_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  const int order[K_ROWS] = {K_VERT, K_LINE, K_POLY, K_PCONN, K_STRIP, K_SCONN};   // the ABI's order
  counts_host[0] = (int64_t)tot[0];   // points
  for (int r = 0; r < K_ROWS; ++r) counts_host[1 + r] = (int64_t)tot[2 + order[r]];
  return B2V_OK;
}

extern "C" int b2v_clean_emit(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs, int64_t np,
                              int64_t npconn, int pform, int pi64, const void* sconn, const int64_t* soffs, int64_t ns,
                              int64_t nsconn, int sform, int si64, void* workspace, float* points_out,
                              int64_t* point_ids_out, int64_t* vconn_out, int64_t* lconn_out, int64_t* poffs_out,
                              int64_t* pconn_out, int64_t* soffs_out, int64_t* sconn_out, int64_t* cell_ids_out,
                              void* stream) {
  Mesh M;
  if (int rc = setup(verts, nv, make_cells(pconn, poffs, np, npconn, pform, pi64),
                     make_cells(sconn, soffs, ns, nsconn, sform, si64), "clean_polydata", &M))
    return rc;
  B2V_REQUIRE(workspace && poffs_out && soffs_out, B2V_ERR_ARG, "clean_polydata: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t G = np + ns, C = npconn + nsconn;
  const ClWs w = carve_clean(workspace, nv, G, C);
  if (C == 0 || G == 0) {   // no cell, or only empty ones: two offsets arrays of a single 0
    const int64_t zero = 0;
    B2V_CUDA(cudaMemcpyAsync(poffs_out, &zero, 8, cudaMemcpyHostToDevice, s));
    B2V_CUDA(cudaMemcpyAsync(soffs_out, &zero, 8, cudaMemcpyHostToDevice, s));
    B2V_CUDA(cudaStreamSynchronize(s));
    return B2V_OK;
  }
  const ClOut O{vconn_out, lconn_out, poffs_out, pconn_out, soffs_out, sconn_out, cell_ids_out};
  k_cl_emit_points<<<b2v_grid(C, kBlock, 16), kBlock, 0, s>>>(M, verts, w.rep, w.fscan, w.newid, points_out,
                                                               point_ids_out);
  if (int rc = b2v_check_launch("k_cl_emit_points")) return rc;
  k_cl_emit_cells<<<b2v_grid(G, kBlock, 16), kBlock, 0, s>>>(M, w.cnt, G + 1, w.cat, w.totals, O);
  if (int rc = b2v_check_launch("k_cl_emit_cells")) return rc;
  k_cl_emit_corners<<<b2v_grid(C, kBlock, 16), kBlock, 0, s>>>(M, w.rep, w.kscan, w.cnt, G + 1, w.ncell, w.cat,
                                                                w.newid, O);
  return b2v_check_launch("k_cl_emit_corners");
}

extern "C" int64_t b2v_triangle_filter_workspace_bytes(int64_t ncells, int64_t npoly_corners) {
  if (ncells < 0 || npoly_corners < 0) return -1;
  return (int64_t)carve_tri(nullptr, ncells, npoly_corners).bytes;
}

extern "C" int b2v_triangle_filter_count(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs,
                                         int64_t np, int64_t npconn, int pform, int pi64, const void* sconn,
                                         const int64_t* soffs, int64_t ns, int64_t nsconn, int sform, int si64,
                                         void* workspace, void* stream, int64_t* counts_host) {
  Mesh M;
  if (int rc = setup(verts, nv, make_cells(pconn, poffs, np, npconn, pform, pi64),
                     make_cells(sconn, soffs, ns, nsconn, sform, si64), "triangle_filter", &M))
    return rc;
  B2V_REQUIRE(workspace && counts_host, B2V_ERR_ARG, "triangle_filter: null argument");
  B2V_REQUIRE(npconn < 0x7fffffffLL, B2V_ERR_ARG, "triangle_filter: a polygon needs fewer than 2^31 points");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t G = np + ns;
  const TfWs w = carve_tri(workspace, G, npconn);
  if (int rc = validate(M, w.status, "triangle_filter", s)) return rc;
  B2V_CUDA(cudaMemsetAsync(w.totals, 0, 8, s));
  if (G > 0) {
    B2V_CUDA(cudaMemsetAsync(w.tcnt + G, 0, 8, s));
    k_tf_count<<<b2v_grid(G, kBlock, 16), kBlock, 0, s>>>(M, w.tcnt);
    if (int rc = b2v_check_launch("k_tf_count")) return rc;
    if (np > 0 && pform == 0) {   // faces hold triangles only
      k_tf_polygons<1><<<b2v_grid(np, kBlock / 32, 8), kBlock, 0, s>>>(M, verts, w);
      if (int rc = b2v_check_launch("k_tf_polygons<1>")) return rc;
      k_tf_polygons<kBlock / 32><<<b2v_grid(np, 1, 4), kBlock, 0, s>>>(M, verts, w);
      if (int rc = b2v_check_launch("k_tf_polygons<8>")) return rc;
    }
    if (int rc = scan(w.tcnt, G + 1, w.scratch, w.totals, s)) return rc;
  }
  unsigned long long tot = 0;
  B2V_CUDA(cudaMemcpyAsync(&tot, w.totals, 8, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  counts_host[0] = (int64_t)tot;
  return B2V_OK;
}

extern "C" int b2v_triangle_filter_emit(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs,
                                        int64_t np, int64_t npconn, int pform, int pi64, const void* sconn,
                                        const int64_t* soffs, int64_t ns, int64_t nsconn, int sform, int si64,
                                        void* workspace, int64_t* tris_out, int64_t* cell_ids_out, void* stream) {
  Mesh M;
  if (int rc = setup(verts, nv, make_cells(pconn, poffs, np, npconn, pform, pi64),
                     make_cells(sconn, soffs, ns, nsconn, sform, si64), "triangle_filter", &M))
    return rc;
  B2V_REQUIRE(workspace, B2V_ERR_ARG, "triangle_filter: null workspace");
  const int64_t C = npconn + nsconn;
  if (C == 0) return B2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const TfWs w = carve_tri(workspace, np + ns, npconn);
  k_tf_emit<<<b2v_grid(C, kBlock, 16), kBlock, 0, s>>>(M, w.tcnt, w.tri, tris_out, cell_ids_out);
  return b2v_check_launch("k_tf_emit");
}
