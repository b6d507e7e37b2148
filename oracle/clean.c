/* CPU checker of the surface clean and triangle filter — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * Sequential restatements of vtkCleanPolyData and vtkTriangleFilter (VTK 9.3) on polys and strips, at the
 * settings InVesalius uses (surface_process.py, surface.py decimate_polydata, markers/surface_geometry.py,
 * measures.py). The rules below are restated from the upstream VTK source as remembered and are UNVERIFIED
 * (VTK cannot be built here); the device (csrc/clean.cu) follows this text, and parity with VTK itself is
 * unpinned.
 *
 * vtkCleanPolyData: PointMerging on, tolerance 0 (vtkMergePoints), RemoveUnusedPoints, ConvertPolysToLines,
 * ConvertLinesToPoints and ConvertStripsToPolys on.
 *  1. Cells are walked in the order polys, then strips; the input cell ids are numbered the same way (polys
 *     0 .. P-1, strips P .. P+S-1). Each corner's point is inserted as it is met.
 *  2. Merge. Two points merge when their float coordinates compare ==, so -0 equals +0 and a point with a NaN
 *     coordinate merges with no other point (the same input id met twice is still one point).
 *  3. Output points are numbered in order of first use; a point used only by a cell that later degenerates
 *     still counts, unused points are dropped. point_ids[k] is the input point of output point k's first use
 *     (the one whose data VTK copies).
 *  4. Each cell loses consecutive repeated points (after the merge). A poly with more than 2 points left whose
 *     last point is its first loses the last.
 *  5. A poly with 3 or more points stays a poly, with 2 it becomes a line, with 1 a vert, with 0 it goes.
 *     A strip with 4 or more points stays a strip, with 3 it becomes a poly, with 2 a line, with 1 a vert.
 *  6. Within each output category the cells keep traversal order; cell_ids lists the input cell of every
 *     output cell in the order verts, lines, polys, strips.
 *
 * vtkTriangleFilter on polys and strips:
 *  7. A poly of 3 points is copied; a poly of fewer points gives no triangle.
 *  8. A strip of n points gives n - 2 triangles (vtkTriangleStrip::DecomposeStrip): triangle i is
 *     (p[i], p[i+1], p[i+2]) for even i and (p[i+1], p[i], p[i+2]) for odd i. Degenerate triangles are kept.
 *  9. Polys come out first, then strips, each in input order; cell_ids maps each triangle to its input cell.
 * 10. A poly of n > 3 points is clipped by vtkPolygon::EarCutTriangulation (reached through
 *     vtkPolygon::Triangulate). This is not the NonDegenerateTriangulate rule that fill_holes.c step 7 restates
 *     for vtkFillHolesFilter: the ear cut ranks ears by perimeter^2 / area, not by perimeter; it admits a
 *     non-convex vertex only after a split-plane and segment-crossing test; it drops near-coincident points
 *     first; and it emits (i, next, prev), not (prev, i, next). So that code cannot stand for it. In double,
 *     with positions 0 .. n-1 of the polygon's points:
 *     a. tol = 1e-6 d, d the diagonal sqrt((dx dx + dy dy) + dz dz) of the points' bounding box.
 *     b. The points form a ring (next / prev), head = 0, m = n. For i = 0 .. n-1, with v starting at head:
 *        w = next(v); when |v - w|^2 < tol^2 (|a|^2 = (a0 a0 + a1 a1) + a2 a2) w is unlinked, head = v if
 *        w was head, m -= 1; otherwise v = w.
 *     c. The normal N: the sum, for v from next(head) while next(v) != head, of (v - head) x (next(v) - head),
 *        normalised by its length sqrt((N0 N0 + N1 N1) + N2 N2); a zero length ends the polygon with no
 *        triangle. a x b = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0).
 *     d. The measure of v: v1 = v - prev, v2 = next - v, v3 = prev - next, area = (c0 N0 + c1 N1) + c2 N2 with
 *        c = v1 x v2; -1 when area < 0, -DBL_MAX when area == 0, else p p / area with
 *        p = (|v1| + |v2|) + |v3|. A vertex is in the queue when its measure is > 0.
 *     e. While m > 2 and the queue is not empty: pop the vertex of the smallest measure (the lowest position
 *        on a tie: vtkPriorityQueue's heap order among equal measures is not reproduced). When the queue held
 *        m vertices before the pop it is removed; otherwise only if it can be removed (f).
 *        Removing v emits (v, next, prev), m -= 1; if m < 3 this ends the polygon, else head = next if v was
 *        head, v is unlinked, prev and next leave the queue and re-enter with their new measures if > 0.
 *     f. v can be removed when m <= 3; otherwise with sN = (next - prev) x N normalised (length 0: not
 *        removable), sign(x) = +1 / -1 / 0 for e = (sN0 (x0 - prev0) + sN1 (x1 - prev1)) + sN2 (x2 - prev2)
 *        > tol / < -tol / otherwise, over the ring from next(next) up to, not including, prev: a vertex w
 *        (after the first) whose sign differs from its predecessor's crosses the split line, and v is not
 *        removable when the segment (prev, next) meets (w, prev(w)) (g); and v is removable only when some
 *        vertex of that range has sign -1.
 *     g. Segments (a1, a2) and (b1, b2) meet (vtkLine::Intersection) when, with a = a2 - a1, b = b2 - b1,
 *        c = b1 - a1, r00 = a.a, r01 = -(a.b), r11 = b.b, c0 = a.c, c1 = -(b.c) (dot products summed left to
 *        right), det = r00 r11 - r01 r01 is 0 (colinear), or u = (r11 c0 - r01 c1) / det and
 *        w = (-r01 c0 + r00 c1) / det both lie in [0, 1].
 *     The triangles emitted before the clipping stops are kept; a polygon that cannot be finished gives fewer
 *     than n - 2.
 *
 * Cells are given as VTK 9 cell arrays: offsets int64 [n + 1] starting at 0, non-decreasing, ending at the
 * connectivity's length, and connectivity int64. Returns 0, 1 on an id outside [0, V), 3 when out of memory,
 * 4 on malformed offsets.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int check_cells(const int64_t* off, int64_t n, const int64_t* conn, int64_t nv) {
  if (off[0] != 0) return 4;
  for (int64_t c = 0; c < n; ++c)
    if (off[c + 1] < off[c]) return 4;
  for (int64_t k = 0; k < off[n]; ++k)
    if (conn[k] < 0 || conn[k] >= nv) return 1;
  return 0;
}

static uint32_t canon(float f) {
  uint32_t u;
  if (f == 0.0f) f = 0.0f;
  memcpy(&u, &f, 4);
  return u;
}

/* the locator: an open-addressing table of output point ids, keyed by the canonical coordinate bits */
typedef struct {
  const float* P;
  int64_t* slot;      /* output id or -1 */
  int64_t* first;     /* output id -> its input point */
  uint64_t mask;
} Locator;

static int64_t lookup_or_insert(Locator* L, int64_t p, int64_t* nout) {
  const float x = L->P[3 * p], y = L->P[3 * p + 1], z = L->P[3 * p + 2];
  uint64_t h = ((uint64_t)canon(x) * 0x9E3779B97F4A7C15ull) ^ ((uint64_t)canon(y) * 0xC2B2AE3D27D4EB4Full) ^
               ((uint64_t)canon(z) * 0x165667B19E3779F9ull);
  h ^= h >> 29;
  h &= L->mask;
  for (;;) {
    const int64_t o = L->slot[h];
    if (o < 0) break;
    const int64_t q = L->first[o];
    if (L->P[3 * q] == x && L->P[3 * q + 1] == y && L->P[3 * q + 2] == z) return o;
    h = (h + 1) & L->mask;
  }
  L->slot[h] = *nout;
  L->first[*nout] = p;
  return (*nout)++;
}

/* counts[7] = {points, verts, lines, polys, poly corners, strips, strip corners}. Capacities: points and
 * corners of every kind up to the input corners, cells up to the input cells (+ 1 for offsets). */
int orc_clean(const float* P, int64_t nv, const int64_t* poff, const int64_t* pconn, int64_t np,
              const int64_t* soff, const int64_t* sconn, int64_t ns, float* pts_out, int64_t* point_ids,
              int64_t* vconn, int64_t* lconn, int64_t* poffs_out, int64_t* pconn_out, int64_t* soffs_out,
              int64_t* sconn_out, int64_t* cell_ids, int64_t* counts) {
  for (int k = 0; k < 7; ++k) counts[k] = 0;
  int rc = check_cells(poff, np, pconn, nv);
  if (!rc) rc = check_cells(soff, ns, sconn, nv);
  if (rc) return rc;
  const int64_t C = poff[np] + soff[ns], G = np + ns;
  uint64_t H = 1024;
  while (H < 2 * (uint64_t)(C > 0 ? C : 1)) H <<= 1;
  Locator L;
  L.P = P;
  L.mask = H - 1;
  L.slot = malloc(H * 8);
  L.first = malloc((size_t)(C + 1) * 8);
  int64_t* of_input = malloc((size_t)(nv + 1) * 8);   /* output id of an input point already met */
  /* per output cell: its category, input cell, and where its points sit in `kept` */
  int8_t* cat = malloc((size_t)(G + 1));
  int64_t *cstart = malloc((size_t)(G + 1) * 8), *clen = malloc((size_t)(G + 1) * 8);
  int64_t* kept = malloc((size_t)(C + 1) * 8);
  rc = 3;
  if (!L.slot || !L.first || !of_input || !cat || !cstart || !clen || !kept) goto done;
  rc = 0;
  memset(L.slot, 0xff, H * 8);
  for (int64_t p = 0; p < nv; ++p) of_input[p] = -1;
  int64_t nout = 0, nk = 0;
  for (int64_t g = 0; g < G; ++g) {
    const int strip = g >= np;
    const int64_t* off = strip ? soff : poff;
    const int64_t* conn = strip ? sconn : pconn;
    const int64_t c = strip ? g - np : g;
    int64_t n = 0;
    cstart[g] = nk;
    for (int64_t k = off[c]; k < off[c + 1]; ++k) {
      const int64_t p = conn[k];
      if (of_input[p] < 0) of_input[p] = lookup_or_insert(&L, p, &nout);
      const int64_t id = of_input[p];
      if (n == 0 || kept[nk + n - 1] != id) kept[nk + n++] = id;
    }
    if (!strip && n > 2 && kept[nk] == kept[nk + n - 1]) --n;
    nk += n;
    clen[g] = n;
    if (!strip) cat[g] = n >= 3 ? 3 : (int8_t)n;
    else cat[g] = n >= 4 ? 4 : (int8_t)n;
  }
  for (int64_t k = 0; k < nout; ++k) {
    const int64_t p = L.first[k];
    point_ids[k] = p;
    for (int a = 0; a < 3; ++a) pts_out[3 * k + a] = P[3 * p + a];
  }
  int64_t nvc = 0, nlc = 0, npc = 0, nsc = 0, npk = 0, nsk = 0, ci = 0;
  for (int want = 1; want <= 4; ++want)
    for (int64_t g = 0; g < G; ++g) {
      if (cat[g] != want) continue;
      const int64_t* src = kept + cstart[g];
      cell_ids[ci++] = g;
      if (want == 1) vconn[nvc++] = src[0];
      else if (want == 2) { lconn[2 * nlc] = src[0]; lconn[2 * nlc + 1] = src[1]; ++nlc; }
      else if (want == 3) { poffs_out[npc++] = npk; for (int64_t j = 0; j < clen[g]; ++j) pconn_out[npk++] = src[j]; }
      else { soffs_out[nsc++] = nsk; for (int64_t j = 0; j < clen[g]; ++j) sconn_out[nsk++] = src[j]; }
    }
  poffs_out[npc] = npk;
  soffs_out[nsc] = nsk;
  counts[0] = nout; counts[1] = nvc; counts[2] = nlc; counts[3] = npc; counts[4] = npk; counts[5] = nsc;
  counts[6] = nsk;
done:
  free(L.slot); free(L.first); free(of_input); free(cat); free(cstart); free(clen); free(kept);
  return rc;
}

/* ---- rule 10: vtkPolygon::EarCutTriangulation --------------------------------------------------------- */
typedef struct { double x[3]; int64_t next, prev; } Vtx;

static void sub3(const double* a, const double* b, double* r) { for (int k = 0; k < 3; ++k) r[k] = a[k] - b[k]; }
static double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static double len3(const double* a) { return sqrt((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]); }
static void cross3(const double* a, const double* b, double* n) {
  n[0] = a[1] * b[2] - a[2] * b[1];
  n[1] = a[2] * b[0] - a[0] * b[2];
  n[2] = a[0] * b[1] - a[1] * b[0];
}
static double normalize3(double* a) {
  const double d = len3(a);
  if (d != 0.0) { a[0] /= d; a[1] /= d; a[2] /= d; }
  return d;
}

static double ear_measure(const Vtx* a, int64_t v, const double* N) {
  double v1[3], v2[3], v3[3], c[3];
  sub3(a[v].x, a[a[v].prev].x, v1);
  sub3(a[a[v].next].x, a[v].x, v2);
  sub3(a[a[v].prev].x, a[a[v].next].x, v3);
  cross3(v1, v2, c);
  const double area = dot3(c, N);
  if (area < 0.0) return -1.0;
  if (area == 0.0) return -DBL_MAX;
  const double p = (len3(v1) + len3(v2)) + len3(v3);
  return p * p / area;
}

static int segments_meet(const double* a1, const double* a2, const double* b1, const double* b2) {
  double a[3], b[3], c[3];
  sub3(a2, a1, a); sub3(b2, b1, b); sub3(b1, a1, c);
  const double r00 = dot3(a, a), r01 = -dot3(a, b), r11 = dot3(b, b), c0 = dot3(a, c), c1 = -dot3(b, c);
  const double det = r00 * r11 - r01 * r01;
  if (det == 0.0) return 1;
  const double u = (r11 * c0 - r01 * c1) / det, w = (-r01 * c0 + r00 * c1) / det;
  return 0.0 <= u && u <= 1.0 && 0.0 <= w && w <= 1.0;
}

static int side(const double* sN, const double* o, const double* x, double tol) {
  const double e = (sN[0] * (x[0] - o[0]) + sN[1] * (x[1] - o[1])) + sN[2] * (x[2] - o[2]);
  return e > tol ? 1 : (e < -tol ? -1 : 0);
}

static int can_remove(const Vtx* a, int64_t v, int64_t m, const double* N, double tol) {
  if (m <= 3) return 1;
  const int64_t prev = a[v].prev, next = a[v].next;
  double d[3], sN[3];
  sub3(a[next].x, a[prev].x, d);
  cross3(d, N, sN);
  if (normalize3(sN) == 0.0) return 0;
  int cur = side(sN, a[prev].x, a[a[next].next].x, tol), neg = cur < 0;
  for (int64_t w = a[a[next].next].next; w != prev; w = a[w].next) {
    const int sg = side(sN, a[prev].x, a[w].x, tol);
    if (sg < 0) neg = 1;
    if (sg != cur && segments_meet(a[prev].x, a[next].x, a[w].x, a[a[w].prev].x)) return 0;
    cur = sg;
  }
  return neg;
}

/* the polygon ids[n] (n > 3) into out [n - 2][3]; returns the triangles emitted */
static int64_t ear_cut(const float* P, const int64_t* ids, int64_t n, Vtx* a, double* key, char* inq, int64_t* out) {
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t i = 0; i < n; ++i) {
    for (int k = 0; k < 3; ++k) {
      a[i].x[k] = (double)P[3 * ids[i] + k];
      lo[k] = a[i].x[k] < lo[k] ? a[i].x[k] : lo[k];
      hi[k] = a[i].x[k] > hi[k] ? a[i].x[k] : hi[k];
    }
    a[i].next = (i + 1) % n;
    a[i].prev = (i + n - 1) % n;
    inq[i] = 0;
  }
  const double ext[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
  const double tol = 1e-6 * len3(ext), tol2 = tol * tol;
  int64_t head = 0, m = n, v = head;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t w = a[v].next;
    double d[3];
    sub3(a[v].x, a[w].x, d);
    if ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] < tol2) {
      a[a[w].next].prev = v;
      a[v].next = a[w].next;
      if (w == head) head = v;
      --m;
    } else {
      v = w;
    }
  }
  double N[3] = {0.0, 0.0, 0.0};
  for (v = a[head].next; a[v].next != head; v = a[v].next) {
    double v1[3], v2[3], c[3];
    sub3(a[v].x, a[head].x, v1);
    sub3(a[a[v].next].x, a[head].x, v2);
    cross3(v1, v2, c);
    for (int k = 0; k < 3; ++k) N[k] += c[k];
  }
  if (normalize3(N) == 0.0) return 0;
  int64_t nq = 0, nt = 0;
  v = head;
  for (int64_t i = 0; i < m; ++i, v = a[v].next) {
    key[v] = ear_measure(a, v, N);
    if (key[v] > 0.0) { inq[v] = 1; ++nq; }
  }
  while (m > 2 && nq > 0) {
    int64_t best = -1;
    for (int64_t i = 0; i < n; ++i)
      if (inq[i] && (best < 0 || key[i] < key[best])) best = i;
    const int convex = nq == m;
    inq[best] = 0;
    --nq;
    if (!convex && !can_remove(a, best, m, N, tol)) continue;
    const int64_t prev = a[best].prev, next = a[best].next;
    out[3 * nt] = ids[best]; out[3 * nt + 1] = ids[next]; out[3 * nt + 2] = ids[prev];
    ++nt;
    if (--m < 3) break;
    if (best == head) head = next;
    a[prev].next = next;
    a[next].prev = prev;
    const int64_t nb[2] = {prev, next};
    for (int j = 0; j < 2; ++j) {
      if (inq[nb[j]]) { inq[nb[j]] = 0; --nq; }
      key[nb[j]] = ear_measure(a, nb[j], N);
      if (key[nb[j]] > 0.0) { inq[nb[j]] = 1; ++nq; }
    }
  }
  return nt;
}

/* tris [<= corners][3], cell_ids [<= corners]; *ntris = the triangles written */
int orc_triangle_filter(const float* P, int64_t nv, const int64_t* poff, const int64_t* pconn, int64_t np,
                        const int64_t* soff, const int64_t* sconn, int64_t ns, int64_t* tris, int64_t* cell_ids,
                        int64_t* ntris) {
  *ntris = 0;
  int rc = check_cells(poff, np, pconn, nv);
  if (!rc) rc = check_cells(soff, ns, sconn, nv);
  if (rc) return rc;
  int64_t nmax = 1;
  for (int64_t c = 0; c < np; ++c)
    if (poff[c + 1] - poff[c] > nmax) nmax = poff[c + 1] - poff[c];
  Vtx* a = malloc((size_t)nmax * sizeof(Vtx));
  double* key = malloc((size_t)nmax * 8);
  char* inq = malloc((size_t)nmax);
  if (!a || !key || !inq) { free(a); free(key); free(inq); return 3; }
  int64_t t = 0;
  for (int64_t c = 0; c < np; ++c) {
    const int64_t n = poff[c + 1] - poff[c];
    if (n == 3) {
      for (int j = 0; j < 3; ++j) tris[3 * t + j] = pconn[poff[c] + j];
      cell_ids[t++] = c;
    } else if (n > 3) {
      const int64_t k = ear_cut(P, pconn + poff[c], n, a, key, inq, tris + 3 * t);
      for (int64_t j = 0; j < k; ++j) cell_ids[t + j] = c;
      t += k;
    }
  }
  free(a); free(key); free(inq);
  for (int64_t c = 0; c < ns; ++c) {
    const int64_t* p = sconn + soff[c];
    const int64_t n = soff[c + 1] - soff[c];
    for (int64_t i = 0; i + 2 < n; ++i) {
      tris[3 * t] = i % 2 ? p[i + 1] : p[i];
      tris[3 * t + 1] = i % 2 ? p[i] : p[i + 1];
      tris[3 * t + 2] = p[i + 2];
      cell_ids[t++] = np + c;
    }
  }
  *ntris = t;
  return 0;
}
