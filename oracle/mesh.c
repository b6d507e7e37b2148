/* CPU checker — TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * context_aware_smoothing: invesalius_rs/src/mesh.rs:27-395 (float32 vertices, int64 faces [M][4] with
 * the leading 3, float32 face normals), restated sequentially in the reference's iteration order:
 *   build_map_vface          :89-101  every column of a face row is taken as a vertex id, the leading 3
 *                                      included (so vertex 3 collects every face) — kept as it is; the
 *                                      map is only looked up for ids in [0, nv), so a leading entry
 *                                      outside that range is ignored
 *   build_vertex_connectivity:103-123 neighbours in first-appearance order over the faces
 *   find_staircase_artifacts :125-189 the max / min tracking with its `else if` (after the first face min
 *                                      is still f64::MAX, so |max - min| >= t: for finite t every vertex
 *                                      that has a face is returned; for t = inf, those whose first face
 *                                      has a NaN normal) — kept as it is
 *   propagate_weights        :202-295 frontier by frontier; the reference runs a frontier in parallel
 *                                      with compare-and-swap (its result can depend on thread timing);
 *                                      here the frontier is walked in order, one valid execution
 *   taubin_smooth            :345-395 lambda 0.5, mu -0.53, float64 sums in adjacency order, float32 updates
 * The reference has no test for this function: PARITY UNPINNED. tests/ca_smoothing_model.py, written from
 * mesh.rs independently of this file, pins it bit for bit. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { int64_t* off; int64_t* idx; } Csr;

static void calc_d(const float* v, const Csr* adj, int64_t i, double d[3]) {
  const double px = v[3 * i], py = v[3 * i + 1], pz = v[3 * i + 2];
  d[0] = d[1] = d[2] = 0.0;
  int64_t n = 0;
  for (int64_t e = adj->off[i]; e < adj->off[i + 1]; ++e) {
    const int64_t j = adj->idx[e];
    d[0] += px - (double)v[3 * j];
    d[1] += py - (double)v[3 * j + 1];
    d[2] += pz - (double)v[3 * j + 2];
    ++n;
  }
  if (n > 0) { d[0] /= (double)n; d[1] /= (double)n; d[2] /= (double)n; }
}

/* weights_out (optional): float64 [nv]. Returns 0, or 1 on an entry of columns 1..3 outside [0, nv). */
int orc_ca_smoothing(float* vertices, int64_t nv, const int64_t* faces, int64_t nf, const float* normals, double t,
                     double tmax, double bmin, uint32_t n_iters, double* weights_out) {
  /* map_vface as CSR, entries in (face, column) order */
  int64_t* cnt = (int64_t*)calloc((size_t)nv + 1, 8);
  for (int64_t e = 0; e < 4 * nf; ++e) {
    if (faces[e] >= 0 && faces[e] < nv) ++cnt[faces[e] + 1];
    else if (e % 4 != 0) { free(cnt); return 1; }
  }
  for (int64_t i = 0; i < nv; ++i) cnt[i + 1] += cnt[i];
  int64_t* vf = (int64_t*)malloc((size_t)(4 * nf + 1) * 8);
  int64_t* fill = (int64_t*)malloc((size_t)nv * 8);
  memcpy(fill, cnt, (size_t)nv * 8);
  for (int64_t f = 0; f < nf; ++f)
    for (int c = 0; c < 4; ++c)
      if (faces[4 * f + c] >= 0 && faces[4 * f + c] < nv) vf[fill[faces[4 * f + c]]++] = f;
  /* vertex connectivity */
  Csr adj;
  int64_t cap = 16 * nv + 16, used = 0;
  int64_t** lists = (int64_t**)calloc((size_t)nv, sizeof(int64_t*));
  int* len = (int*)calloc((size_t)nv, sizeof(int));
  int* capv = (int*)calloc((size_t)nv, sizeof(int));
  (void)cap; (void)used;
  for (int64_t f = 0; f < nf; ++f)
    for (int a = 1; a < 4; ++a)
      for (int b = 1; b < 4; ++b) {
        const int64_t vi = faces[4 * f + a], vj = faces[4 * f + b];
        if (vi == vj) continue;
        int found = 0;
        for (int k = 0; k < len[vi]; ++k) if (lists[vi][k] == vj) { found = 1; break; }
        if (found) continue;
        if (len[vi] == capv[vi]) { capv[vi] = capv[vi] ? 2 * capv[vi] : 8; lists[vi] = (int64_t*)realloc(lists[vi], (size_t)capv[vi] * 8); }
        lists[vi][len[vi]++] = vj;
      }
  adj.off = (int64_t*)malloc((size_t)(nv + 1) * 8);
  adj.off[0] = 0;
  for (int64_t i = 0; i < nv; ++i) adj.off[i + 1] = adj.off[i] + len[i];
  adj.idx = (int64_t*)malloc((size_t)(adj.off[nv] + 1) * 8);
  for (int64_t i = 0; i < nv; ++i) { memcpy(adj.idx + adj.off[i], lists[i], (size_t)len[i] * 8); free(lists[i]); }
  free(lists); free(len); free(capv);
  /* find_staircase_artifacts */
  const double DMIN = -1.7976931348623157e308, DMAX = 1.7976931348623157e308;
  int64_t* seeds = (int64_t*)malloc((size_t)nv * 8 + 8);
  int64_t nseeds = 0;
  for (int64_t v = 0; v < nv; ++v) {
    double max_z = DMIN, min_z = DMAX, max_y = DMIN, min_y = DMAX, max_x = DMIN, min_x = DMAX;
    for (int64_t e = cnt[v]; e < cnt[v + 1]; ++e) {
      const float* nr = normals + 3 * vf[e];
      const double nx = nr[0], ny = nr[1], nz = nr[2];
      const double of_z = 1.0 - fabs(nx * 0.0 + ny * 0.0 + nz * 1.0);
      const double of_y = 1.0 - fabs(nx * 0.0 + ny * 1.0 + nz * 0.0);
      const double of_x = 1.0 - fabs(nx * 1.0 + ny * 0.0 + nz * 0.0);
      if (of_z > max_z) max_z = of_z; else if (of_z < min_z) min_z = of_z;
      if (of_y > max_y) max_y = of_y; else if (of_y < min_y) min_y = of_y;
      if (of_x > max_x) max_x = of_x; else if (of_x < min_x) min_x = of_x;
      if (fabs(max_z - min_z) >= t || fabs(max_y - min_y) >= t || fabs(max_x - min_x) >= t) { seeds[nseeds++] = v; break; }
    }
  }
  /* propagate_weights */
  double* dist = (double*)malloc((size_t)nv * 8 + 8);
  int64_t* seed_map = (int64_t*)malloc((size_t)nv * 8 + 8);
  for (int64_t i = 0; i < nv; ++i) { dist[i] = INFINITY; seed_map[i] = -1; }
  int64_t* frontier = (int64_t*)malloc((size_t)nv * 8 + 8);
  int64_t nfr = nseeds;
  memcpy(frontier, seeds, (size_t)nseeds * 8);
  for (int64_t k = 0; k < nseeds; ++k) { dist[seeds[k]] = 0.0; seed_map[seeds[k]] = seeds[k]; }
  const double tmax_sq = tmax * tmax;
  int64_t* next = (int64_t*)malloc((size_t)(adj.off[nv] + 8) * 8);
  while (nfr > 0) {
    int64_t nn = 0;
    for (int64_t k = 0; k < nfr; ++k) {
      const int64_t v = frontier[k], s = seed_map[v];
      for (int64_t e = adj.off[v]; e < adj.off[v + 1]; ++e) {
        const int64_t vj = adj.idx[e];
        const double dx = (double)vertices[3 * vj] - (double)vertices[3 * s], dy = (double)vertices[3 * vj + 1] - (double)vertices[3 * s + 1],
                     dz = (double)vertices[3 * vj + 2] - (double)vertices[3 * s + 2];
        const double d_sq = dx * dx + dy * dy + dz * dz;
        if (d_sq > tmax_sq) continue;
        const double old = dist[vj];
        if (d_sq >= old && isfinite(old)) continue;
        dist[vj] = d_sq;
        seed_map[vj] = s;
        next[nn++] = vj;
      }
    }
    if (nn > nv) { /* duplicates can make the list longer than nv: keep it, as the reference does */ frontier = (int64_t*)realloc(frontier, (size_t)nn * 8 + 8); }
    memcpy(frontier, next, (size_t)nn * 8);
    nfr = nn;
  }
  double* w = (double*)malloc((size_t)nv * 8 + 8);
  for (int64_t i = 0; i < nv; ++i) {
    const double d = dist[i];
    w[i] = !isfinite(d) ? bmin : (1.0 - sqrt(d) / tmax) * (1.0 - bmin) + bmin;
  }
  if (weights_out) memcpy(weights_out, w, (size_t)nv * 8);
  /* taubin_smooth */
  double* dv = (double*)malloc((size_t)nv * 24 + 8);
  const double lm[2] = {0.5, -0.53};
  for (uint32_t it = 0; it < n_iters; ++it)
    for (int half = 0; half < 2; ++half) {
      for (int64_t i = 0; i < nv; ++i) calc_d(vertices, &adj, i, dv + 3 * i);
      for (int64_t i = 0; i < nv; ++i)
        for (int k = 0; k < 3; ++k) vertices[3 * i + k] += (float)(w[i] * lm[half] * dv[3 * i + k]);
    }
  free(cnt); free(vf); free(fill); free(adj.off); free(adj.idx); free(seeds); free(dist); free(seed_map); free(frontier);
  free(next); free(w); free(dv);
  return 0;
}
