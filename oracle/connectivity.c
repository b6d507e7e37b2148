/* CPU checker of the surface connectivity tools — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of vtkPolyDataConnectivityFilter (VTK 9.3) on triangles, as InVesalius's
 * polydata_utils.SelectLargestPart / SplitDisconectedParts / JoinSeedsParts use it. The contract below is
 * restated from the upstream VTK source as remembered and is UNVERIFIED (VTK cannot be installed here);
 * the device (csrc/connectivity.cu) follows this text, and parity with VTK itself is unpinned.
 *
 *  - Cells and links. Cells are the triangles in input order. The point -> cell links list each point's
 *    cells in ascending cell id (vtkCellLinks::BuildLinks); a degenerate triangle with a repeated point
 *    appears once per corner in that point's list.
 *  - Regions (all-regions, largest, specified). Cells are scanned in ascending id; an unvisited cell starts
 *    a new region, numbered 0, 1, ... in that order.
 *  - TraverseAndMark. The wave is a list that may hold duplicates. A cell is marked when it is taken from
 *    the wave, not when it is pushed; a marked cell taken again is skipped. For each newly marked cell its
 *    points j = 0, 1, 2 are visited: a point without a number gets PointMap[p] = PointNumber++, then every
 *    cell of that point's link list is appended to the next wave, marked or not. PointNumber carries on
 *    across regions.
 *  - RegionSizes[r] is the number of cells of region r.
 *  - Seeded mode: one region, 0. The first wave is built seed by seed, in the order given, from each seed's
 *    link list; negative seed ids are skipped (VTK's `if (pt >= 0)`). Only the cells reached are visited.
 *
 * orc_conn_run fills region[T] (-1 where not visited), pointmap[V] (-1 where not numbered), sizes[R] and
 * counts = {R, points numbered, cells visited, depth}. depth is the largest number of waves of one region
 * that marked at least one cell. Returns 0, 1 on a bad argument (face index outside [0, V), seed >= V),
 * 3 when out of memory.
 */
#include <stdint.h>
#include <stdlib.h>

static int64_t traverse(const int64_t* faces, const int64_t* lstart, const int64_t* links, int64_t* wave,
                        int64_t nwave, int64_t* wave2, int32_t region_number, int32_t* region, int32_t* pointmap,
                        int64_t* point_number, int64_t* ncells, int64_t* depth) {
  int64_t waves = 0;
  while (nwave > 0) {
    int64_t n2 = 0, marked = 0;
    for (int64_t w = 0; w < nwave; ++w) {
      const int64_t cell = wave[w];
      if (region[cell] >= 0) continue;
      region[cell] = region_number;
      ++*ncells;
      ++marked;
      for (int j = 0; j < 3; ++j) {
        const int64_t p = faces[3 * cell + j];
        if (pointmap[p] < 0) pointmap[p] = (int32_t)(*point_number)++;
        for (int64_t k = lstart[p]; k < lstart[p + 1]; ++k) wave2[n2++] = links[k];
      }
    }
    if (marked) ++waves;
    int64_t* t = wave; wave = wave2; wave2 = t;
    nwave = n2;
  }
  if (waves > *depth) *depth = waves;
  return waves;
}

int orc_conn_run(const int64_t* faces, int64_t nv, int64_t nt, const int64_t* seeds, int64_t nseeds, int seeded,
                 int32_t* region, int32_t* pointmap, int64_t* sizes, int64_t* counts) {
  if (nv < 0 || nt < 0 || nseeds < 0) return 1;
  for (int64_t i = 0; i < 3 * nt; ++i)
    if (faces[i] < 0 || faces[i] >= nv) return 1;
  for (int64_t i = 0; i < nseeds; ++i)
    if (seeds[i] >= nv) return 1;
  for (int64_t t = 0; t < nt; ++t) region[t] = -1;
  for (int64_t p = 0; p < nv; ++p) pointmap[p] = -1;
  counts[0] = counts[1] = counts[2] = counts[3] = 0;

  /* vtkCellLinks: counts, offsets, then the cells in ascending id, once per corner */
  int64_t* lstart = (int64_t*)calloc((size_t)nv + 1, sizeof(int64_t));
  int64_t* links = (int64_t*)malloc(((size_t)3 * nt + 1) * sizeof(int64_t));
  int64_t* fill = (int64_t*)malloc(((size_t)nv + 1) * sizeof(int64_t));
  if (!lstart || !links || !fill) { free(lstart); free(links); free(fill); return 3; }
  for (int64_t i = 0; i < 3 * nt; ++i) ++lstart[faces[i] + 1];
  for (int64_t p = 0; p < nv; ++p) lstart[p + 1] += lstart[p];
  for (int64_t p = 0; p <= nv; ++p) fill[p] = lstart[p];
  for (int64_t t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) links[fill[faces[3 * t + j]]++] = t;
  free(fill);

  /* a wave never holds more entries than the sum over its cells' points of the link lengths; the whole
     run appends at most sum_p deg(p)^2 entries, and one wave at most that */
  int64_t cap = 1;
  for (int64_t p = 0; p < nv; ++p) {
    const int64_t d = lstart[p + 1] - lstart[p];
    cap += d * d;
  }
  for (int64_t i = 0; i < nseeds; ++i)
    if (seeds[i] >= 0) cap += lstart[seeds[i] + 1] - lstart[seeds[i]];
  int64_t* wave = (int64_t*)malloc((size_t)cap * sizeof(int64_t));
  int64_t* wave2 = (int64_t*)malloc((size_t)cap * sizeof(int64_t));
  if (!wave || !wave2) { free(wave); free(wave2); free(lstart); free(links); return 3; }

  int64_t point_number = 0, ncells = 0, depth = 0, nregions = 0;
  if (seeded) {
    int64_t n = 0;
    for (int64_t i = 0; i < nseeds; ++i) {
      const int64_t pt = seeds[i];
      if (pt >= 0)
        for (int64_t k = lstart[pt]; k < lstart[pt + 1]; ++k) wave[n++] = links[k];
    }
    traverse(faces, lstart, links, wave, n, wave2, 0, region, pointmap, &point_number, &ncells, &depth);
    sizes[0] = ncells;
    nregions = 1;
  } else {
    for (int64_t t = 0; t < nt; ++t) {
      if (region[t] >= 0) continue;
      const int64_t before = ncells;
      wave[0] = t;
      traverse(faces, lstart, links, wave, 1, wave2, (int32_t)nregions, region, pointmap, &point_number, &ncells,
               &depth);
      sizes[nregions++] = ncells - before;
    }
  }
  counts[0] = nregions;
  counts[1] = point_number;
  counts[2] = ncells;
  counts[3] = depth;
  free(wave); free(wave2); free(lstart); free(links);
  return 0;
}
