/* CPU checker of the Laplacian surface smoothing — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of vtkSmoothPolyDataFilter (VTK 9.3) on triangles, as InVesalius's
 * polydata_utils.ApplySmoothFilter, surface.decimate_polydata and markers/surface_geometry use it. The
 * contract below is restated from the upstream VTK source as remembered and is UNVERIFIED (VTK cannot be
 * installed here); the device (csrc/smoothing.cu) follows this text, and parity with VTK itself is unpinned.
 *
 *  - Input. Points float32 [V][3]; cells the triangles in input order. Vertex codes are VTK's: simple 0,
 *    fixed 1, feature-edge 2, boundary-edge 3. Every point starts simple with no edge list.
 *  - Nothing to do. With no cells, 0 iterations or a relaxation factor of exactly 0 the points are passed
 *    through unchanged and 0 iterations are reported. (VTK returns early in all three cases.)
 *  - Links. Each point's cells in ascending id (vtkCellLinks::BuildLinks); a degenerate triangle appears once
 *    per corner it occupies. GetCellEdgeNeighbors(c, p1, p2) lists the cells of p1's link list, other than
 *    c, that contain p2, in link order, duplicates included.
 *  - Edge analysis. Cells c in id order, edges i = 0, 1, 2 with p1 = pts[i], p2 = pts[(i + 1) % 3]; every
 *    point of the cell gets an (empty) edge list. With numNei neighbours:
 *      numNei == 0                          boundary edge;
 *      numNei >= 2                          feature edge, unless some neighbour id is < c: then simple;
 *      numNei == 1, neighbour n > c         simple, or feature when feature-edge smoothing is on and
 *                                           dot(normal(c), normal(n)) <= cos(feature angle);
 *      numNei == 1, neighbour n < c         skipped (already visited).
 *    Normals are vtkTriangle::ComputeNormal of the input points in double: (v3 - v2) x (v1 - v2),
 *    divided by its length unless that is 0. A non-skipped edge of type e then updates p1 (other end p2)
 *    and then p2 (other end p1):
 *      simple vertex, e non-simple          the list becomes {other}, the vertex takes type e;
 *      boundary/feature vertex, e non-simple,
 *      or simple vertex, e simple           other is appended; a boundary/feature vertex whose list grows
 *                                           past 2 entries becomes fixed;
 *      otherwise (fixed vertex, or a boundary/feature vertex hit by a simple edge)   nothing.
 *  - Post-pass, per point. A boundary vertex becomes fixed when boundary smoothing is off. A boundary or
 *    feature vertex whose list does not hold exactly 2 entries becomes fixed. Otherwise, with list {a, b}
 *    and input points in double, l1 = x - a and l2 = b - x are normalised (vtkMath::Normalize: divided by
 *    sqrt(l.l) unless that is 0) and the vertex becomes fixed when dot(l1, l2) < cos(edge angle).
 *  - Sweep. for (maxDist = DBL_MAX, it = 0; maxDist > conv && it < iterations; ++it): maxDist = 0; for
 *    every point i in ascending id that is not fixed and has a non-empty list of n entries: x = the current
 *    (float32) point in double; d = 0; for each entry j in list order d += (y_j - x) / n, y_j the current
 *    point j (already moved in this iteration when j < i); x' = x + relax * d; maxDist = max(maxDist,
 *    |x - x'|^2) with |v|^2 = (v0 v0 + v1 v1) + v2 v2, compared with >; the point is stored back as
 *    float32 (round to nearest) before the next point reads it. After the points, maxDist = sqrt(maxDist).
 *    The number of iterations done is `it` at exit.
 *  - Early stop. VTK measures, per iteration, the largest Euclidean distance between a moved point's
 *    position before the move and its double-precision new position (before the float32 store), and stops
 *    when that is <= conv = Convergence * GetLength(). GetLength() is the diagonal of the bounding box,
 *    sqrt((dx dx + dy dy) + dz dz) in double, of the points the cells use (vtkPolyData's bounds count only
 *    points that cells reference). With Convergence = 0 the sweep stops after the first iteration that
 *    moves no point at all.
 *  - Angles. The caller passes cos(feature angle) and cos(edge angle) as doubles (VTK: cos(angle * pi/180)
 *    with both angles clamped to [0, 180]); Convergence is clamped to [0, 1] by the caller.
 *
 * orc_smooth_run moves points[V][3] in place and fills types[V] (int8), nlist[V], lists (the edge lists,
 * concatenated in point order; room for 6T entries) and counts = {iterations done, total list entries}.
 * Returns 0, 1 on a bad argument (face index outside [0, V), negative iterations), 3 when out of memory.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { SIMPLE = 0, FIXED = 1, FEATURE = 2, BOUNDARY = 3 };

static void normal(const float* P, const int64_t* t, double n[3]) {
  double v1[3], v2[3], v3[3];
  for (int k = 0; k < 3; ++k) {
    v1[k] = P[3 * t[0] + k];
    v2[k] = P[3 * t[1] + k];
    v3[k] = P[3 * t[2] + k];
  }
  const double ax = v3[0] - v2[0], ay = v3[1] - v2[1], az = v3[2] - v2[2];
  const double bx = v1[0] - v2[0], by = v1[1] - v2[1], bz = v1[2] - v2[2];
  n[0] = ay * bz - az * by;
  n[1] = az * bx - ax * bz;
  n[2] = ax * by - ay * bx;
  const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  if (len != 0.0) {
    n[0] /= len; n[1] /= len; n[2] /= len;
  }
}

static double normalize(double v[3]) {
  const double den = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (den != 0.0)
    for (int k = 0; k < 3; ++k) v[k] /= den;
  return den;
}

typedef struct {
  int type;
  int64_t n, cap;
  int64_t* ids;   /* NULL: the point is in no cell */
} Vert;

static int push(Vert* v, int64_t id) {
  if (v->n == v->cap) {
    const int64_t cap = v->cap ? 2 * v->cap : 8;
    int64_t* ids = (int64_t*)realloc(v->ids, (size_t)cap * sizeof(int64_t));
    if (!ids) return 3;
    v->ids = ids;
    v->cap = cap;
  }
  v->ids[v->n++] = id;
  return 0;
}

/* VTK's per-vertex state machine: point v hit by an edge of type e whose other end is other */
static int hit(Vert* v, int e, int64_t other) {
  if (e != SIMPLE && v->type == SIMPLE) {
    v->n = 0;
    v->type = e;
    return push(v, other);
  }
  if ((e != SIMPLE && (v->type == BOUNDARY || v->type == FEATURE)) || (e == SIMPLE && v->type == SIMPLE)) {
    if (push(v, other)) return 3;
    if (v->type != SIMPLE && v->n > 2) v->type = FIXED;
  }
  return 0;
}

int orc_smooth_run(float* points, int64_t nv, const int64_t* faces, int64_t nt, int64_t iterations,
                   double relax, double cos_feature, double cos_edge, int feature_edge_smoothing,
                   int boundary_smoothing, double convergence, int8_t* types, int32_t* nlist, int32_t* lists,
                   int64_t* counts) {
  if (nv < 0 || nt < 0 || iterations < 0) return 1;
  for (int64_t i = 0; i < 3 * nt; ++i)
    if (faces[i] < 0 || faces[i] >= nv) return 1;
  counts[0] = counts[1] = 0;
  for (int64_t p = 0; p < nv; ++p) { types[p] = SIMPLE; nlist[p] = 0; }
  if (nt == 0) return 0;

  /* vtkCellLinks */
  int64_t* lstart = (int64_t*)calloc((size_t)nv + 1, sizeof(int64_t));
  int64_t* links = (int64_t*)malloc((size_t)3 * nt * sizeof(int64_t));
  int64_t* fill = (int64_t*)malloc(((size_t)nv + 1) * sizeof(int64_t));
  Vert* V = (Vert*)calloc((size_t)nv, sizeof(Vert));
  int rc = 0;
  if (!lstart || !links || !fill || !V) { rc = 3; goto done; }
  for (int64_t i = 0; i < 3 * nt; ++i) ++lstart[faces[i] + 1];
  for (int64_t p = 0; p < nv; ++p) lstart[p + 1] += lstart[p];
  for (int64_t p = 0; p <= nv; ++p) fill[p] = lstart[p];
  for (int64_t t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) links[fill[faces[3 * t + j]]++] = t;

  /* edge analysis, cell by cell */
  for (int64_t c = 0; c < nt; ++c) {
    const int64_t* pts = faces + 3 * c;
    for (int i = 0; i < 3; ++i) {
      const int64_t p1 = pts[i], p2 = pts[(i + 1) % 3];
      int64_t num = 0, nei = -1, lower = 0;
      for (int64_t k = lstart[p1]; k < lstart[p1 + 1]; ++k) {
        const int64_t d = links[k];
        if (d == c) continue;
        if (faces[3 * d] == p2 || faces[3 * d + 1] == p2 || faces[3 * d + 2] == p2) {
          if (num == 0) nei = d;
          ++num;
          if (d < c) lower = 1;
        }
      }
      int e = SIMPLE;
      if (num == 0) {
        e = BOUNDARY;
      } else if (num >= 2) {
        if (!lower) e = FEATURE;
      } else if (nei > c) {
        if (feature_edge_smoothing) {
          double n[3], m[3];
          normal(points, pts, n);
          normal(points, faces + 3 * nei, m);
          if (n[0] * m[0] + n[1] * m[1] + n[2] * m[2] <= cos_feature) e = FEATURE;
        }
      } else {
        continue;
      }
      if (hit(&V[p1], e, p2) || hit(&V[p2], e, p1)) { rc = 3; goto done; }
    }
  }

  /* post-pass */
  for (int64_t p = 0; p < nv; ++p) {
    Vert* v = &V[p];
    if (v->type != FEATURE && v->type != BOUNDARY) continue;
    if (!boundary_smoothing && v->type == BOUNDARY) {
      v->type = FIXED;
    } else if (v->n != 2) {
      v->type = FIXED;
    } else {
      double l1[3], l2[3];
      for (int k = 0; k < 3; ++k) {
        const double x1 = points[3 * v->ids[0] + k], x2 = points[3 * p + k], x3 = points[3 * v->ids[1] + k];
        l1[k] = x2 - x1;
        l2[k] = x3 - x2;
      }
      if (normalize(l1) >= 0.0 && normalize(l2) >= 0.0 && l1[0] * l2[0] + l1[1] * l2[1] + l1[2] * l2[2] < cos_edge)
        v->type = FIXED;
    }
  }
  int64_t total = 0;
  for (int64_t p = 0; p < nv; ++p) {
    types[p] = (int8_t)V[p].type;
    nlist[p] = (int32_t)V[p].n;
    for (int64_t k = 0; k < V[p].n; ++k) lists[total++] = (int32_t)V[p].ids[k];
  }
  counts[1] = total;

  /* the bounding-box diagonal of the points the cells use */
  double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  int any = 0;
  for (int64_t p = 0; p < nv; ++p) {
    if (lstart[p + 1] == lstart[p]) continue;
    for (int k = 0; k < 3; ++k) {
      const double x = points[3 * p + k];
      if (!any || x < lo[k]) lo[k] = x;
      if (!any || x > hi[k]) hi[k] = x;
    }
    any = 1;
  }
  const double dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
  const double conv = convergence * sqrt(dx * dx + dy * dy + dz * dz);

  if (iterations == 0 || relax == 0.0) goto done;
  int64_t it = 0;
  for (double maxDist = 1.79769313486231570815e+308; maxDist > conv && it < iterations; ++it) {
    maxDist = 0.0;
    for (int64_t p = 0; p < nv; ++p) {
      const Vert* v = &V[p];
      if (v->type == FIXED || v->ids == NULL || v->n == 0) continue;
      double x[3], d[3] = {0.0, 0.0, 0.0}, y[3];
      for (int k = 0; k < 3; ++k) x[k] = points[3 * p + k];
      for (int64_t j = 0; j < v->n; ++j)
        for (int k = 0; k < 3; ++k) d[k] += ((double)points[3 * v->ids[j] + k] - x[k]) / (double)v->n;
      for (int k = 0; k < 3; ++k) y[k] = x[k] + relax * d[k];
      const double dist = (x[0] - y[0]) * (x[0] - y[0]) + (x[1] - y[1]) * (x[1] - y[1]) + (x[2] - y[2]) * (x[2] - y[2]);
      if (dist > maxDist) maxDist = dist;
      for (int k = 0; k < 3; ++k) points[3 * p + k] = (float)y[k];
    }
    maxDist = sqrt(maxDist);
  }
  counts[0] = it;

done:
  if (V)
    for (int64_t p = 0; p < nv; ++p) free(V[p].ids);
  free(V); free(lstart); free(links); free(fill);
  return rc;
}
