/* CPU checker of the surface hole filler — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of vtkFillHolesFilter (VTK 9.3) on triangles, as InVesalius's
 * polydata_utils.ApplySmoothFilter (HoleSize 1000), surface_process.join_process_surface (300),
 * FillSurfaceHole (500) and markers/surface_geometry use it. The contract below is restated from the upstream
 * VTK source as remembered and is UNVERIFIED (VTK cannot be installed here): the bounding-sphere hints and
 * the triangulation rule (step 7) in particular are this project's statement, not a transcription. The
 * device (csrc/fill_holes.cu) follows this text, and parity with VTK itself is unpinned.
 *
 *  1. Links. Each point's cells in ascending id; a degenerate triangle appears once per corner it occupies.
 *  2. Boundary lines. Cells c in id order, edges i = 0, 1, 2 with p1 = t[i], p2 = t[(i + 1) % 3]: when no
 *     cell d != c in p1's links contains p2 (GetCellEdgeNeighbors finds none), the line (p1, p2) is
 *     appended. Line ids follow this order.
 *  3. Too few lines. With fewer than 3 lines the output is the input and no loop is reported.
 *  4. Line links. Each point's lines in ascending id, a line (x, x) twice at x.
 *  5. Tracing. visited[] = 0. For each line L in id order with !visited[L]: visited[L] = 1, start = L.p0,
 *     poly = [start], end = L.p1, cur = L; while end != start and the loop is valid: append end; the lines
 *     in end's links other than cur, counted with multiplicity, must be exactly one line n (otherwise the
 *     loop is invalid); visited[n] = 1, end = n's other endpoint (n.p0 if end == n.p1, else n.p1), cur = n.
 *     A traversal does not test visited[n]. Only valid loops are reported, in the order of their first line.
 *  6. Size test. vtkSphere::ComputeBoundingSphere over poly's points in order, in double, with the hints
 *     {0, 0}: the sphere starts at poly[0] with r = 0; for each point p in order, with v = p - c and
 *     d2 = (v0 v0 + v1 v1) + v2 v2, when d2 > r r: d = sqrt(d2), r = (r + d) / 2, delta = d - r and
 *     c[k] = (r c[k] + delta p[k]) / d. The loop is filled when r <= hole_size (the hole size is clamped to
 *     [0, FLT_MAX] by the caller, as SetHoleSize does); otherwise it is reported as too large.
 *  7. Triangulation (vtkPolygon::NonDegenerateTriangulate as this project states it). Points in double.
 *     - Fewer than 3 points: nothing is emitted and the loop is reported as failed.
 *     - The polygon normal N is the fan sum over i = 1 .. n-2, in order, of (p[i] - p[0]) x (p[i+1] - p[0]),
 *       divided by its length sqrt((N0 N0 + N1 N1) + N2 N2) unless that is 0. A cross product a x b is
 *       (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0).
 *     - The remaining points keep their loop order (positions 0 .. n-1). While more than 3 remain, every
 *       remaining position i, with prev and next its remaining neighbours (cyclically), offers the ear
 *       (prev, i, next). Its normal is vtkTriangle::ComputeNormal(prev, i, next): (next - i) x (prev - i),
 *       divided by its length unless that is 0. The ear qualifies when (e0 N0 + e1 N1) + e2 N2 > 0. Its
 *       perimeter is (|i - prev| + |next - i|) + |prev - next|, |v| = sqrt((v0 v0 + v1 v1) + v2 v2). The
 *       qualifying ear with the smallest perimeter wins, the lowest position on a tie; the triangle
 *       (prev, i, next) is emitted and i is removed.
 *     - When three remain, they are emitted in position order.
 *     - When no ear qualifies, none of the loop's triangles are emitted and it is reported as failed.
 *  8. Output. The points are unchanged; the faces are the input triangles in order, then the new triangles:
 *     loops in the order of their first line, each loop's triangles in the order they were emitted.
 *
 * orc_fill_holes writes new_tris [<= lines][3] (point ids), and per valid loop first_line, npts, radius
 * and status (0 filled, 1 failed, 2 too large) into arrays with room for `lines` loops; counts = {lines,
 * loops, new triangles}. Returns 0, 1 on a bad face index, 3 when out of memory.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { FILLED = 0, FAILED = 1, TOO_LARGE = 2 };

static void point(const float* P, int64_t p, double x[3]) {
  for (int k = 0; k < 3; ++k) x[k] = (double)P[3 * p + k];
}

static double dist(const double a[3], const double b[3]) {
  const double v0 = a[0] - b[0], v1 = a[1] - b[1], v2 = a[2] - b[2];
  return sqrt((v0 * v0 + v1 * v1) + v2 * v2);
}

static void cross(const double a[3], const double b[3], double n[3]) {
  n[0] = a[1] * b[2] - a[2] * b[1];
  n[1] = a[2] * b[0] - a[0] * b[2];
  n[2] = a[0] * b[1] - a[1] * b[0];
}

static void unit(double n[3]) {
  const double len = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  if (len != 0.0) { n[0] /= len; n[1] /= len; n[2] /= len; }
}

static double sphere_radius(const float* P, const int64_t* poly, int64_t n) {
  double c[3], r = 0.0;
  point(P, poly[0], c);
  for (int64_t k = 0; k < n; ++k) {
    double p[3];
    point(P, poly[k], p);
    const double v0 = p[0] - c[0], v1 = p[1] - c[1], v2 = p[2] - c[2];
    const double d2 = (v0 * v0 + v1 * v1) + v2 * v2;
    if (d2 > r * r) {
      const double d = sqrt(d2);
      r = (r + d) / 2.0;
      const double delta = d - r;
      for (int a = 0; a < 3; ++a) c[a] = (r * c[a] + delta * p[a]) / d;
    }
  }
  return r;
}

/* key of the ear at position i: its perimeter when it qualifies, +inf otherwise */
static double ear_key(const float* P, const int64_t* poly, int64_t prev, int64_t i, int64_t next,
                      const double N[3]) {
  double a[3], b[3], c[3], u[3], w[3], e[3];
  point(P, poly[prev], a); point(P, poly[i], b); point(P, poly[next], c);
  for (int k = 0; k < 3; ++k) { u[k] = c[k] - b[k]; w[k] = a[k] - b[k]; }
  cross(u, w, e);
  unit(e);
  if (!((e[0] * N[0] + e[1] * N[1]) + e[2] * N[2] > 0.0)) return INFINITY;
  return (dist(b, a) + dist(c, b)) + dist(a, c);
}

/* triangulates poly[n] into out (n - 2 triangles); returns the number emitted, 0 when the loop fails. An
 * ear's key depends only on (prev, i, next), so the keys are kept and only the two ears next to a clipped
 * point are recomputed; the argmin over the remaining positions is taken afresh at every step. */
static int64_t triangulate(const float* P, const int64_t* poly, int64_t n, int64_t* prv, int64_t* nxt,
                           double* key, int64_t* out) {
  if (n < 3) return 0;
  double N[3] = {0.0, 0.0, 0.0}, p0[3];
  point(P, poly[0], p0);
  for (int64_t i = 1; i + 1 < n; ++i) {
    double a[3], b[3], x[3];
    point(P, poly[i], a); point(P, poly[i + 1], b);
    for (int k = 0; k < 3; ++k) { a[k] -= p0[k]; b[k] -= p0[k]; }
    cross(a, b, x);
    for (int k = 0; k < 3; ++k) N[k] += x[k];
  }
  unit(N);
  for (int64_t i = 0; i < n; ++i) { prv[i] = (i + n - 1) % n; nxt[i] = (i + 1) % n; }
  for (int64_t i = 0; i < n; ++i) key[i] = n > 3 ? ear_key(P, poly, prv[i], i, nxt[i], N) : INFINITY;
  int64_t rem = n, nt = 0, head = 0;
  while (rem > 3) {
    int64_t best = -1;
    double bk = INFINITY;
    for (int64_t i = 0; i < n; ++i)     /* a clipped position keeps the key +inf */
      if (key[i] < bk) { bk = key[i]; best = i; }
    if (best < 0) return 0;
    const int64_t p = prv[best], q = nxt[best];
    out[3 * nt] = poly[p]; out[3 * nt + 1] = poly[best]; out[3 * nt + 2] = poly[q];
    ++nt;
    key[best] = INFINITY;
    nxt[p] = q; prv[q] = p;
    if (best == head) head = q;
    if (--rem > 3) {
      key[p] = ear_key(P, poly, prv[p], p, q, N);
      key[q] = ear_key(P, poly, p, q, nxt[q], N);
    }
  }
  out[3 * nt] = poly[head]; out[3 * nt + 1] = poly[nxt[head]]; out[3 * nt + 2] = poly[nxt[nxt[head]]];
  return nt + 1;
}

int orc_fill_holes(const float* P, int64_t nv, const int64_t* tri, int64_t nt, double hole_size,
                   int64_t* new_tris, int64_t* first_line, int64_t* npts, double* radius, int8_t* status,
                   int64_t* counts) {
  counts[0] = counts[1] = counts[2] = 0;
  for (int64_t k = 0; k < 3 * nt; ++k)
    if (tri[k] < 0 || tri[k] >= nv) return 1;
  int rc = 3;
  int64_t *lstart = calloc((size_t)nv + 1, 8), *links = malloc((size_t)(3 * nt + 1) * 8);
  int64_t *lines = malloc((size_t)(6 * nt + 1) * 8), *mstart = calloc((size_t)nv + 1, 8);
  int64_t *mlinks = malloc((size_t)(6 * nt + 1) * 8), *fill = calloc((size_t)nv + 1, 8);
  int64_t *poly = malloc((size_t)(3 * nt + 1) * 8), *prv = malloc((size_t)(3 * nt + 1) * 8);
  int64_t* nxt = malloc((size_t)(3 * nt + 1) * 8);
  char* visited = calloc((size_t)(3 * nt + 1), 1);
  double* key = malloc((size_t)(3 * nt + 1) * 8);
  if (!lstart || !links || !lines || !mstart || !mlinks || !fill || !poly || !prv || !nxt || !visited || !key)
    goto done;
  rc = 0;
  /* 1. links */
  for (int64_t k = 0; k < 3 * nt; ++k) lstart[tri[k] + 1]++;
  for (int64_t p = 0; p < nv; ++p) lstart[p + 1] += lstart[p];
  for (int64_t k = 0; k < 3 * nt; ++k) links[lstart[tri[k]] + fill[tri[k]]++] = k / 3;
  /* 2. boundary lines */
  int64_t nl = 0;
  for (int64_t c = 0; c < nt; ++c)
    for (int i = 0; i < 3; ++i) {
      const int64_t p1 = tri[3 * c + i], p2 = tri[3 * c + (i + 1) % 3];
      int nei = 0;
      for (int64_t k = lstart[p1]; k < lstart[p1 + 1] && !nei; ++k) {
        const int64_t d = links[k];
        if (d != c && (tri[3 * d] == p2 || tri[3 * d + 1] == p2 || tri[3 * d + 2] == p2)) nei = 1;
      }
      if (!nei) { lines[2 * nl] = p1; lines[2 * nl + 1] = p2; ++nl; }
    }
  counts[0] = nl;
  /* 3. too few lines */
  if (nl < 3) goto done;
  /* 4. line links */
  memset(fill, 0, (size_t)(nv + 1) * 8);
  for (int64_t k = 0; k < 2 * nl; ++k) mstart[lines[k] + 1]++;
  for (int64_t p = 0; p < nv; ++p) mstart[p + 1] += mstart[p];
  for (int64_t k = 0; k < 2 * nl; ++k) mlinks[mstart[lines[k]] + fill[lines[k]]++] = k / 2;
  /* 5 - 7 */
  int64_t nloops = 0, ntris = 0;
  for (int64_t L = 0; L < nl; ++L) {
    if (visited[L]) continue;
    visited[L] = 1;
    const int64_t start = lines[2 * L];
    int64_t end = lines[2 * L + 1], cur = L, n = 0;
    int valid = 1;
    poly[n++] = start;
    while (end != start && valid) {
      poly[n++] = end;
      int64_t count = 0, other = -1;
      for (int64_t k = mstart[end]; k < mstart[end + 1]; ++k)
        if (mlinks[k] != cur) { ++count; other = mlinks[k]; }
      if (count != 1) {
        valid = 0;
      } else {
        visited[other] = 1;
        end = lines[2 * other] == end ? lines[2 * other + 1] : lines[2 * other];
        cur = other;
      }
    }
    if (!valid) continue;
    const double r = sphere_radius(P, poly, n);
    first_line[nloops] = L;
    npts[nloops] = n;
    radius[nloops] = r;
    if (r <= hole_size) {
      const int64_t k = triangulate(P, poly, n, prv, nxt, key, new_tris + 3 * ntris);
      status[nloops] = k ? FILLED : FAILED;
      ntris += k;
    } else {
      status[nloops] = TOO_LARGE;
    }
    ++nloops;
  }
  counts[1] = nloops;
  counts[2] = ntris;
done:
  free(lstart); free(links); free(lines); free(mstart); free(mlinks); free(fill); free(poly); free(prv);
  free(nxt); free(visited); free(key);
  return rc;
}
