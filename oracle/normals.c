/* CPU checker of surface normals and mass properties — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of vtkPolyDataNormals (VTK 9.3) on triangles, with Consistency, Splitting and
 * NonManifoldTraversal on (every InVesalius caller sets them), FeatureAngle and AutoOrientNormals as
 * parameters, ComputeCellNormals on; and of vtkMassProperties' Volume and SurfaceArea. Every step that
 * restates VTK is [upstream, from memory — unverified here]: VTK cannot be installed here, so parity with
 * VTK itself is unpinned. The device (csrc/normals.cu) follows this text bit for bit.
 *
 *  0. Links. Cells are the triangles in input order. A point's links are its cells in ascending id, a cell
 *     once per corner at that point (vtkCellLinks::BuildLinks). GetCellEdgeNeighbors(c, p1, p2) is the list
 *     of cells d != c in p1's links that contain p2, in link order, duplicates included.
 *  1. Consistent ordering (TraverseAndOrder) [upstream, from memory — unverified here]. A wave is a list of
 *     cells. For each cell c of the wave in order, for each edge j = 0, 1, 2 of c's CURRENT corner order
 *     (p1 = pts[j], p2 = pts[(j + 1) % 3]), for each d of GetCellEdgeNeighbors(c, p1, p2) in order (every
 *     count is crossed: non-manifold traversal): if d is not visited, let l be the first corner of d equal
 *     to p2; when d's corner l + 1 is not p1, d is reversed, (a, b, c) -> (c, b, a), and counted as a flip;
 *     d is marked visited and appended to the next wave. A cell is marked when it is appended. The waves
 *     run until one is empty; every wave processed counts, the seed wave included, and `waves` is the most
 *     waves one region needed.
 *     - Without auto_orient, cells are scanned in ascending id; each unvisited one seeds a region.
 *     - With auto_orient, the points are popped in ascending x (the float coordinate; -0 equals +0, NaN
 *       after everything), ties by ascending id (VTK's vtkPriorityQueue leaves ties to its heap; here they
 *       are fixed). For each popped point, its unvisited link cells are scanned in link order and the one
 *       whose normal (step 2's double normal of its INPUT order) has the largest |x| is kept, a later cell
 *       only when strictly larger, and none when every |x| is 0. When one is kept, it is reversed (and
 *       counted as a flip) if that x is positive, marked visited and traversed as a region. A region none of
 *       whose cells is ever kept is never traversed: its cells keep their input order.
 *     Because a cell with a repeated point has an edge (a, a) whose neighbours are every cell at a, the
 *     cells one traversal reaches depend on where it starts; the regions are the traversals, not a fixed
 *     partition.
 *  2. Cell normals [upstream, from memory — unverified here]. vtkTriangle::ComputeNormal in double of the
 *     float coordinates of the final corner order v1, v2, v3: a = v3 - v2, b = v1 - v2,
 *     n = (ay bz - az by, az bx - ax bz, ax by - ay bx), len = sqrt((n0 n0 + n1 n1) + n2 n2), n / len when
 *     len != 0 (else n stays 0). The cell normal is n rounded to float32.
 *  3. Splitting (MarkAndSplit) [upstream, from memory — unverified here]. cos_angle = cos(angle *
 *     0.017453292519943295), the angle clamped to [0, 180]. Every point p in ascending id with more than
 *     one link entry groups its link cells: in link order, an ungrouped cell c starts group g; from c the
 *     walk goes both ways around p, first across the edge (p, nA) then (p, nB), where, with s the first
 *     corner of c equal to p (INPUT order), (nA, nB) = (pts[1], pts[2]) for s = 0, (pts[2], pts[0]) for
 *     s = 1, (pts[1], pts[0]) for s = 2. A step from cell x across (p, nei) moves to d when
 *     GetCellEdgeNeighbors(x, p, nei) holds exactly one cell d, d is ungrouped, and the double dot product
 *     (x0 d0 + x1 d1) + x2 d2 of the float32 cell normals is GREATER than cos_angle (VTK's test is strict;
 *     a boundary, a non-manifold edge, a grouped cell or a feature edge ends the walk). From d the walk goes
 *     on across d's other edge at p: with s d's first corner at p, the candidate pts[1] (s = 0 or 2) or
 *     pts[2] (s = 1) unless it equals the edge just crossed, else pts[2] (s = 0) or pts[0] (s = 1, 2). The
 *     first group keeps p; group g >= 1 gets the new point V + (new points made so far) + g - 1, a copy of
 *     p's coordinates, and every corner of its cells equal to p is rewritten to it.
 *  4. Point normals [upstream, from memory — unverified here]. Float32 sums: for each cell in ascending id,
 *     for each corner, the corner's output point adds the cell normal, component by component. Each sum s
 *     is then scaled by 1 / den with den = sqrtf((s0 s0 + s1 s1) + s2 s2) in float32, when den != 0
 *     (vtkMath::Normalize on floats). A point used by no cell keeps (0, 0, 0).
 *  5. Mass properties (vtkMassProperties) [upstream, from memory — unverified here]. Per triangle, in
 *     double of the float coordinates: i, j, k as VTK forms them, the unit normal u (0 when its length is
 *     0), its class (the strict largest |u| component, or the ties xyz, xy, xz, yz), the side lengths a, b,
 *     c, area = sqrt(|s (s - a) (s - b) (s - c)|) with s = 0.5 (a + b + c), and the projected-volume terms
 *     area u[k] avg[k] with avg the corner mean ((c0 + c1) + c2) / 3. The area and the three terms are
 *     summed in cell order; kxyz weighs the classes as VTK does; volume = |kx Vx + ky Vy + kz Vz|. No
 *     triangles: volume and area 0. A NaN normal has no class (VTK stops with an error there).
 *
 * orc_normals writes pts_out [V + new][3], faces_out [T][3] (final order, split ids), pnormals [V + new][3],
 * cnormals [T][3] and counts = {regions, flips, new points, waves}; both output point arrays need room for
 * V + 3T points. orc_mass_properties writes out = {volume, area} and, when terms is not NULL, terms [T][4]
 * = {area, Vx, Vy, Vz terms} and cls [T] (0, 1, 2: x, y, z; 3: xyz; 4: xy; 5: xz; 6: yz; -1: none). Both
 * return 0, 1 on a bad argument (face index outside [0, V), NaN angle), 3 when out of memory.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  const float* v;
  int64_t nv, nt;
  const int64_t* tri;    /* input order */
  int64_t* cur;          /* current order */
  int64_t *lstart, *links;
} Mesh;

static void tri_normal(const float* v, const int64_t* t, double n[3]) {
  double v1[3], v2[3], v3[3];
  for (int k = 0; k < 3; ++k) {
    v1[k] = (double)v[3 * t[0] + k];
    v2[k] = (double)v[3 * t[1] + k];
    v3[k] = (double)v[3 * t[2] + k];
  }
  const double ax = v3[0] - v2[0], ay = v3[1] - v2[1], az = v3[2] - v2[2];
  const double bx = v1[0] - v2[0], by = v1[1] - v2[1], bz = v1[2] - v2[2];
  n[0] = ay * bz - az * by;
  n[1] = az * bx - ax * bz;
  n[2] = ax * by - ay * bx;
  const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  if (len != 0.0) { n[0] /= len; n[1] /= len; n[2] /= len; }
}

static int contains(const int64_t* t, int64_t p) { return t[0] == p || t[1] == p || t[2] == p; }

/* GetCellEdgeNeighbors(c, p1, p2): the count, and the first of them */
static int64_t edge_neighbors(const Mesh* m, int64_t c, int64_t p1, int64_t p2, int64_t* first, int64_t* out) {
  int64_t n = 0;
  for (int64_t k = m->lstart[p1]; k < m->lstart[p1 + 1]; ++k) {
    const int64_t d = m->links[k];
    if (d != c && contains(m->tri + 3 * d, p2)) {
      if (n == 0 && first) *first = d;
      if (out) out[n] = d;
      ++n;
    }
  }
  return n;
}

static void reverse(int64_t* t) { const int64_t a = t[0]; t[0] = t[2]; t[2] = a; }

/* TraverseAndOrder from wave[0, n); returns the waves processed */
static int64_t traverse(Mesh* m, char* visited, int64_t* wave, int64_t n, int64_t* wave2, int64_t* nbr,
                        int64_t* flips) {
  int64_t waves = 0;
  while (n > 0) {
    ++waves;
    int64_t n2 = 0;
    for (int64_t i = 0; i < n; ++i) {
      const int64_t c = wave[i];
      for (int j = 0; j < 3; ++j) {
        const int64_t p1 = m->cur[3 * c + j], p2 = m->cur[3 * c + (j + 1) % 3];
        const int64_t cnt = edge_neighbors(m, c, p1, p2, 0, nbr);
        for (int64_t k = 0; k < cnt; ++k) {
          const int64_t d = nbr[k];
          if (visited[d]) continue;
          int64_t* t = m->cur + 3 * d;
          int l = 0;
          while (t[l] != p2) ++l;
          if (t[(l + 1) % 3] != p1) { reverse(t); ++*flips; }
          visited[d] = 1;
          wave2[n2++] = d;
        }
      }
    }
    int64_t* x = wave; wave = wave2; wave2 = x;
    n = n2;
  }
  return waves;
}

static const float* g_x;
static int by_x(const void* a, const void* b) {
  const int64_t i = *(const int64_t*)a, j = *(const int64_t*)b;
  const float xi = g_x[3 * i], xj = g_x[3 * j];
  const int ni = xi != xi, nj = xj != xj;
  if (ni != nj) return ni - nj;                /* NaN after everything */
  if (!ni && xi < xj) return -1;
  if (!ni && xi > xj) return 1;
  return (i > j) - (i < j);
}

int orc_normals(const float* verts, int64_t nv, const int64_t* faces, int64_t nt, double feature_angle,
                int auto_orient, float* pts_out, int64_t* faces_out, float* pnormals, float* cnormals,
                int64_t* counts) {
  if (nv < 0 || nt < 0 || feature_angle != feature_angle) return 1;
  for (int64_t i = 0; i < 3 * nt; ++i)
    if (faces[i] < 0 || faces[i] >= nv) return 1;
  counts[0] = counts[1] = counts[2] = counts[3] = 0;
  Mesh m = {verts, nv, nt, faces, faces_out, 0, 0};
  memcpy(faces_out, faces, (size_t)(3 * nt) * sizeof(int64_t));
  m.lstart = (int64_t*)calloc((size_t)nv + 1, sizeof(int64_t));
  m.links = (int64_t*)malloc(((size_t)3 * nt + 1) * sizeof(int64_t));
  int64_t* fill = (int64_t*)malloc(((size_t)nv + 1) * sizeof(int64_t));
  char* visited = (char*)calloc((size_t)nt + 1, 1);
  int64_t* wave = (int64_t*)malloc(((size_t)nt + 1) * sizeof(int64_t));
  int64_t* wave2 = (int64_t*)malloc(((size_t)nt + 1) * sizeof(int64_t));
  int64_t* nbr = (int64_t*)malloc(((size_t)3 * nt + 1) * sizeof(int64_t));
  int64_t* order = (int64_t*)malloc(((size_t)nv + 1) * sizeof(int64_t));
  int64_t* grp = (int64_t*)malloc(((size_t)nt + 1) * sizeof(int64_t));
  int64_t* map = (int64_t*)malloc(((size_t)nv + 3 * (size_t)nt + 1) * sizeof(int64_t));
  if (!m.lstart || !m.links || !fill || !visited || !wave || !wave2 || !nbr || !order || !grp || !map) {
    free(m.lstart); free(m.links); free(fill); free(visited); free(wave); free(wave2); free(nbr); free(order);
    free(grp); free(map);
    return 3;
  }
  for (int64_t i = 0; i < 3 * nt; ++i) ++m.lstart[faces[i] + 1];
  for (int64_t p = 0; p < nv; ++p) m.lstart[p + 1] += m.lstart[p];
  for (int64_t p = 0; p <= nv; ++p) fill[p] = m.lstart[p];
  for (int64_t t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) m.links[fill[faces[3 * t + j]]++] = t;

  /* 1. consistent ordering */
  int64_t regions = 0, flips = 0, waves = 0;
  if (!auto_orient) {
    for (int64_t t = 0; t < nt; ++t) {
      if (visited[t]) continue;
      visited[t] = 1;
      wave[0] = t;
      const int64_t w = traverse(&m, visited, wave, 1, wave2, nbr, &flips);
      if (w > waves) waves = w;
      ++regions;
    }
  } else {
    for (int64_t p = 0; p < nv; ++p) order[p] = p;
    g_x = verts;
    qsort(order, (size_t)nv, sizeof(int64_t), by_x);
    for (int64_t q = 0; q < nv; ++q) {
      const int64_t p = order[q];
      double best = 0.0;
      int64_t cell = -1;
      int rev = 0;
      for (int64_t k = m.lstart[p]; k < m.lstart[p + 1]; ++k) {
        const int64_t d = m.links[k];
        if (visited[d]) continue;
        double n[3];
        tri_normal(verts, faces + 3 * d, n);
        if (fabs(n[0]) > best) { best = fabs(n[0]); cell = d; rev = n[0] > 0; }
      }
      if (cell < 0) continue;
      if (rev) { reverse(faces_out + 3 * cell); ++flips; }
      visited[cell] = 1;
      wave[0] = cell;
      const int64_t w = traverse(&m, visited, wave, 1, wave2, nbr, &flips);
      if (w > waves) waves = w;
      ++regions;
    }
  }

  /* 2. cell normals of the final order */
  for (int64_t t = 0; t < nt; ++t) {
    double n[3];
    tri_normal(verts, faces_out + 3 * t, n);
    for (int k = 0; k < 3; ++k) cnormals[3 * t + k] = (float)n[k];
  }

  /* 3. splitting: grp[c] is the group of cell c at the current point (-1: none yet) */
  double a = feature_angle < 0.0 ? 0.0 : (feature_angle > 180.0 ? 180.0 : feature_angle);
  const double cos_angle = cos(a * 0.017453292519943295);
  for (int64_t p = 0; p < nv; ++p) map[p] = p;
  int64_t nout = nv;
  for (int64_t p = 0; p < nv; ++p) {
    const int64_t lo = m.lstart[p], hi = m.lstart[p + 1];
    if (hi - lo <= 1) continue;
    for (int64_t k = lo; k < hi; ++k) grp[m.links[k]] = -1;
    int64_t ng = 0;
    for (int64_t k = lo; k < hi; ++k) {
      const int64_t c0 = m.links[k];
      if (grp[c0] >= 0) continue;
      grp[c0] = ng;
      const int64_t* t = faces + 3 * c0;
      const int s = t[0] == p ? 0 : (t[1] == p ? 1 : 2);
      const int64_t nei0[2] = {s == 1 ? t[2] : t[1], s == 0 ? t[2] : t[0]};
      for (int i = 0; i < 2; ++i) {
        int64_t c = c0, nei = nei0[i];
        while (c >= 0) {
          int64_t d = -1;
          if (edge_neighbors(&m, c, p, nei, &d, 0) == 1 && grp[d] < 0) {
            const float *x = cnormals + 3 * c, *y = cnormals + 3 * d;
            const double dot = (double)x[0] * (double)y[0] + (double)x[1] * (double)y[1] + (double)x[2] * (double)y[2];
            if (dot > cos_angle) {
              grp[d] = ng;
              c = d;
              const int64_t* u = faces + 3 * c;
              const int su = u[0] == p ? 0 : (u[1] == p ? 1 : 2);
              if (su == 0) nei = u[1] != nei ? u[1] : u[2];
              else if (su == 2) nei = u[1] != nei ? u[1] : u[0];
              else nei = u[2] != nei ? u[2] : u[0];
            } else {
              c = -1;
            }
          } else {
            c = -1;
          }
        }
      }
      ++ng;
    }
    if (ng <= 1) continue;
    for (int64_t k = lo; k < hi; ++k) {
      const int64_t c = m.links[k];
      if (grp[c] <= 0) continue;
      const int64_t q = nout + grp[c] - 1;
      map[q] = p;
      for (int j = 0; j < 3; ++j)
        if (faces_out[3 * c + j] == p) { faces_out[3 * c + j] = q; break; }   /* ReplaceCellPoint: the first */
    }
    nout += ng - 1;
  }
  for (int64_t q = 0; q < nout; ++q)
    for (int k = 0; k < 3; ++k) pts_out[3 * q + k] = verts[3 * map[q] + k];

  /* 4. point normals */
  memset(pnormals, 0, (size_t)(3 * nout) * sizeof(float));
  for (int64_t t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) {
      float* s = pnormals + 3 * faces_out[3 * t + j];
      for (int k = 0; k < 3; ++k) s[k] += cnormals[3 * t + k];
    }
  for (int64_t q = 0; q < nout; ++q) {
    float* s = pnormals + 3 * q;
    const float den = sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
    if (den != 0.0f) { s[0] /= den; s[1] /= den; s[2] /= den; }
  }

  counts[0] = regions;
  counts[1] = flips;
  counts[2] = nout - nv;
  counts[3] = waves;
  free(m.lstart); free(m.links); free(fill); free(visited); free(wave); free(wave2); free(nbr); free(order);
  free(grp); free(map);
  return 0;
}

int orc_mass_properties(const float* verts, int64_t nv, const int64_t* faces, int64_t nt, double* terms,
                        int8_t* cls, double* out) {
  if (nv < 0 || nt < 0) return 1;
  for (int64_t i = 0; i < 3 * nt; ++i)
    if (faces[i] < 0 || faces[i] >= nv) return 1;
  double munc[3] = {0.0, 0.0, 0.0}, wxyz = 0.0, wxy = 0.0, wxz = 0.0, wyz = 0.0;
  double vol[3] = {0.0, 0.0, 0.0}, area_sum = 0.0;
  for (int64_t t = 0; t < nt; ++t) {
    double x[3], y[3], z[3];
    for (int c = 0; c < 3; ++c) {
      const float* p = verts + 3 * faces[3 * t + c];
      x[c] = (double)p[0]; y[c] = (double)p[1]; z[c] = (double)p[2];
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
    if (a0 > a1 && a0 > a2) { munc[0]++; c = 0; }
    else if (a1 > a0 && a1 > a2) { munc[1]++; c = 1; }
    else if (a2 > a0 && a2 > a1) { munc[2]++; c = 2; }
    else if (a0 == a1 && a0 == a2) { wxyz++; c = 3; }
    else if (a0 == a1 && a0 > a2) { wxy++; c = 4; }
    else if (a0 == a2 && a0 > a1) { wxz++; c = 5; }
    else if (a1 == a2 && a0 < a2) { wyz++; c = 6; }
    const double ii[3] = {i[0] * i[0], i[1] * i[1], i[2] * i[2]};
    const double jj[3] = {j[0] * j[0], j[1] * j[1], j[2] * j[2]};
    const double kk[3] = {k[0] * k[0], k[1] * k[1], k[2] * k[2]};
    const double a = sqrt(ii[1] + jj[1] + kk[1]);
    const double b = sqrt(ii[0] + jj[0] + kk[0]);
    const double cc = sqrt(ii[2] + jj[2] + kk[2]);
    const double s = 0.5 * (a + b + cc);
    const double area = sqrt(fabs(s * (s - a) * (s - b) * (s - cc)));
    const double zavg = (z[0] + z[1] + z[2]) / 3.0;
    const double yavg = (y[0] + y[1] + y[2]) / 3.0;
    const double xavg = (x[0] + x[1] + x[2]) / 3.0;
    const double t2 = area * u[2] * zavg, t1 = area * u[1] * yavg, t0 = area * u[0] * xavg;
    area_sum += area;
    vol[2] += t2;
    vol[1] += t1;
    vol[0] += t0;
    if (terms) { terms[4 * t] = area; terms[4 * t + 1] = t0; terms[4 * t + 2] = t1; terms[4 * t + 3] = t2; }
    if (cls) cls[t] = c;
  }
  if (nt == 0) { out[0] = out[1] = 0.0; return 0; }
  const double n = (double)nt;
  const double kx = (munc[0] + (wxyz / 3.0) + ((wxy + wxz) / 2.0)) / n;
  const double ky = (munc[1] + (wxyz / 3.0) + ((wxy + wyz) / 2.0)) / n;
  const double kz = (munc[2] + (wxyz / 3.0) + ((wxz + wyz) / 2.0)) / n;
  out[0] = fabs(kx * vol[0] + ky * vol[1] + kz * vol[2]);
  out[1] = area_sum;
  return 0;
}
