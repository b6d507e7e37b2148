/* CPU checker of the geodesic surface measurement — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of what GeodesicMeasure._draw_line (invesalius/data/measures.py:1202-1273) runs for
 * each pair of consecutive picks: vtkPointLocator::FindClosestPoint for both picks, then
 * vtkDijkstraGraphGeodesicPath from the start point to the end point, then the length of the returned polyline.
 * Every step that restates VTK is [upstream, from memory — unverified here]: VTK cannot be installed here, so
 * parity with VTK itself is unpinned. The device (csrc/geodesic.cu) follows this text; where VTK's heap order
 * decides (an ambiguous step, below) the device's rule is stated and reported instead.
 *
 *  1. Graph [upstream, unverified]. Triangle cells only. Each triangle (a, b, c) adds the undirected edges
 *     a-b, b-c and c-a; duplicate edges collapse (VTK keeps one std::map per point keyed by neighbour id, so
 *     a point's neighbours are visited in ascending id); an edge (a, a) of a degenerate triangle is ignored.
 *     Points are never merged by coordinate. The weight of u-v (CalculateStaticEdgeCost) is
 *     sqrt((dx dx + dy dy) + dz dz) in double of the points converted to double (vtkMath::Distance2-
 *     BetweenPoints, then an IEEE sqrt); it is symmetric.
 *  2. Distances [upstream, unverified]. d[start] = 0, every other point starts open at +inf (VTK stores
 *     VTK_DOUBLE_MAX; +inf is reported). A binary min-heap on d (1-based array; insert appends and sifts up
 *     while the parent's key is strictly larger; extract-min moves the last entry to the root and sifts down to
 *     the strictly smaller child, the left one on a tie; decrease-key sifts up). Each extracted point u is
 *     closed; for each neighbour v not closed, in ascending id: du = d[u] + w in double; v not yet in the heap:
 *     d[v] = du, pre[v] = u, insert; else when du < d[v] (strictly): d[v] = du, pre[v] = u, decrease-key. The
 *     whole component of start is settled (StopWhenEndReached off). Rounding is monotone and w >= 0, so d is
 *     the least fixpoint of d[v] = min_u fl(d[u] + w_uv): any relaxation order gives the same bits.
 *  3. Predecessors. pre[v] is the earliest-settled neighbour u with fl(d[u] + w_uv) == d[v]; settling is in
 *     non-decreasing d, so it has the smallest d[u] of those neighbours. A point is AMBIGUOUS when two distinct
 *     neighbours attain d[v] with that same smallest d[u]: only the heap order picks between them. amb[v] says
 *     so, computed from d alone; rule[v] is the neighbour the device picks, the smallest (d[u], id) among the
 *     attaining neighbours (-1 for the start and for unreached points).
 *  4. Trace (TraceShortestPath) [upstream, unverified]. From the end: append v; stop at the start; else
 *     v = pre[v], and stop when that is -1. So start == end gives one point, and an unreached end gives the end
 *     point alone. The path's points are float32 (the vtkPoints default).
 *  5. Closest point (vtkPointLocator::FindClosestPoint). The smallest (dx dx + dy dy) + dz dz in double from
 *     the pick to each point, ties to the smallest id (VTK's bucket order on exact ties is unverified).
 *  6. Length (measures.py:1246-1249). total += sqrt(Distance2BetweenPoints(p_j, p_j+1)) over the float32 path
 *     points in output order, segment after segment, in double.
 *
 * orc_geodesic: dist [nv] (+inf unreached), pre [nv] (-1 start and unreached), rule [nv], amb [nv] (0/1).
 * orc_geodesic_trace: ids_out [nv] from the end; returns the number of points.
 * orc_closest_points: ids_out [np].
 * orc_path_length: lengths {segment sum from 0, total_in continued}.
 * Points are float64 [nv][3] (float32 input converts exactly); faces int64 [nt][3]. Return 0, 1 on a bad
 * argument, 3 when out of memory.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static int cmp_i64(const void* a, const void* b) {
  const int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;
  return (x > y) - (x < y);
}

static double weight(const double* v, int64_t a, int64_t b) {
  const double dx = v[3 * a] - v[3 * b], dy = v[3 * a + 1] - v[3 * b + 1], dz = v[3 * a + 2] - v[3 * b + 2];
  return sqrt(dx * dx + dy * dy + dz * dz);
}

/* ---- the heap ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t* h;    /* [1..n] point ids */
  int64_t* at;   /* heap index of each point, 0 when not in the heap */
  const double* key;
  int64_t n;
} Heap;

static void heap_swap(Heap* q, int64_t i, int64_t j) {
  const int64_t t = q->h[i];
  q->h[i] = q->h[j];
  q->h[j] = t;
  q->at[q->h[i]] = i;
  q->at[q->h[j]] = j;
}

static void heap_up(Heap* q, int64_t i) {
  while (i > 1 && q->key[q->h[i / 2]] > q->key[q->h[i]]) {
    heap_swap(q, i, i / 2);
    i /= 2;
  }
}

static void heap_insert(Heap* q, int64_t v) {
  q->h[++q->n] = v;
  q->at[v] = q->n;
  heap_up(q, q->n);
}

static int64_t heap_pop(Heap* q) {
  if (q->n == 0) return -1;
  const int64_t top = q->h[1];
  q->h[1] = q->h[q->n--];
  q->at[q->h[1]] = 1;
  q->at[top] = 0;
  int64_t i = 1;
  for (;;) {
    const int64_t l = 2 * i, r = l + 1;
    int64_t s = i;
    if (l <= q->n && q->key[q->h[l]] < q->key[q->h[s]]) s = l;
    if (r <= q->n && q->key[q->h[r]] < q->key[q->h[s]]) s = r;
    if (s == i) break;
    heap_swap(q, i, s);
    i = s;
  }
  return top;
}

/* ---- the graph: per point, its neighbours in ascending id, each once --------------------------------- */
static int adjacency(int64_t nv, const int64_t* tri, int64_t nt, int64_t** start_out, int64_t** nb_out) {
  int64_t* cnt = calloc((size_t)nv + 1, sizeof(int64_t));
  int64_t* nb = malloc((size_t)(6 * nt + 1) * sizeof(int64_t));
  if (!cnt || !nb) { free(cnt); free(nb); return 3; }
  for (int64_t t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) {
      const int64_t a = tri[3 * t + j], b = tri[3 * t + (j + 1) % 3];
      if (a < 0 || a >= nv || b < 0 || b >= nv) { free(cnt); free(nb); return 1; }
      if (a != b) { ++cnt[a + 1]; ++cnt[b + 1]; }
    }
  for (int64_t p = 0; p < nv; ++p) cnt[p + 1] += cnt[p];
  int64_t* fill = malloc((size_t)(nv + 1) * sizeof(int64_t));
  if (!fill) { free(cnt); free(nb); return 3; }
  for (int64_t p = 0; p <= nv; ++p) fill[p] = cnt[p];
  for (int64_t t = 0; t < nt; ++t)
    for (int j = 0; j < 3; ++j) {
      const int64_t a = tri[3 * t + j], b = tri[3 * t + (j + 1) % 3];
      if (a != b) { nb[fill[a]++] = b; nb[fill[b]++] = a; }
    }
  /* sort and drop duplicates in place; cnt becomes the compacted starts */
  int64_t o = 0;
  for (int64_t p = 0; p < nv; ++p) {
    const int64_t lo = cnt[p], hi = cnt[p + 1];
    qsort(nb + lo, (size_t)(hi - lo), sizeof(int64_t), cmp_i64);
    cnt[p] = o;
    for (int64_t k = lo; k < hi; ++k)
      if (k == lo || nb[k] != nb[k - 1]) nb[o++] = nb[k];
  }
  cnt[nv] = o;
  free(fill);
  *start_out = cnt;
  *nb_out = nb;
  return 0;
}

int orc_geodesic(const double* v, int64_t nv, const int64_t* tri, int64_t nt, int64_t start, double* dist,
                 int64_t* pre, int64_t* rule, uint8_t* amb) {
  if (nv <= 0 || start < 0 || start >= nv || nt < 0) return 1;
  int64_t *st = NULL, *nb = NULL;
  int rc = adjacency(nv, tri, nt, &st, &nb);
  if (rc) return rc;
  Heap q = {malloc((size_t)(nv + 1) * sizeof(int64_t)), calloc((size_t)nv, sizeof(int64_t)), dist, 0};
  uint8_t* closed = calloc((size_t)nv, 1);
  uint8_t* open = calloc((size_t)nv, 1);
  if (!q.h || !q.at || !closed || !open) { rc = 3; goto out; }
  for (int64_t p = 0; p < nv; ++p) { dist[p] = INFINITY; pre[p] = -1; }
  dist[start] = 0.0;
  heap_insert(&q, start);
  open[start] = 1;
  for (int64_t u; (u = heap_pop(&q)) >= 0;) {
    closed[u] = 1;
    open[u] = 0;
    for (int64_t k = st[u]; k < st[u + 1]; ++k) {
      const int64_t w = nb[k];
      if (closed[w]) continue;
      const double du = dist[u] + weight(v, u, w);
      if (!open[w]) {
        open[w] = 1;
        dist[w] = du;
        pre[w] = u;
        heap_insert(&q, w);
      } else if (du < dist[w]) {
        dist[w] = du;
        pre[w] = u;
        heap_up(&q, q.at[w]);
      }
    }
  }
  /* the device's rule and the ambiguity, from d alone */
  for (int64_t p = 0; p < nv; ++p) {
    rule[p] = -1;
    amb[p] = 0;
    if (p == start || isinf(dist[p])) continue;
    double best = INFINITY;
    int64_t n_best = 0;
    for (int64_t k = st[p]; k < st[p + 1]; ++k) {
      const int64_t u = nb[k];
      if (!(dist[u] + weight(v, u, p) == dist[p])) continue;
      if (dist[u] < best) { best = dist[u]; rule[p] = u; n_best = 1; }
      else if (dist[u] == best) ++n_best;    /* neighbours ascend, so rule keeps the smallest id */
    }
    amb[p] = n_best > 1;
  }
out:
  free(q.h); free(q.at); free(closed); free(open); free(st); free(nb);
  return rc;
}

int64_t orc_geodesic_trace(const int64_t* pre, int64_t nv, int64_t start, int64_t end, int64_t* ids_out) {
  int64_t n = 0, x = end;
  for (;;) {
    if (n >= nv) return -1;
    ids_out[n++] = x;
    if (x == start) break;
    x = pre[x];
    if (x < 0) break;
  }
  return n;
}

void orc_closest_points(const double* v, int64_t nv, const double* picks, int64_t np, int64_t* ids_out) {
  for (int64_t i = 0; i < np; ++i) {
    double best = INFINITY;
    int64_t id = -1;
    for (int64_t p = 0; p < nv; ++p) {
      const double dx = picks[3 * i] - v[3 * p], dy = picks[3 * i + 1] - v[3 * p + 1],
                   dz = picks[3 * i + 2] - v[3 * p + 2];
      const double d2 = dx * dx + dy * dy + dz * dz;
      if (d2 < best || id < 0) { best = d2; id = p; }
    }
    ids_out[i] = id;
  }
}

void orc_path_length(const float* pts, int64_t n, double total_in, double* lengths) {
  double seg = 0.0, tot = total_in;
  for (int64_t j = 0; j + 1 < n; ++j) {
    const double dx = (double)pts[3 * j] - (double)pts[3 * j + 3], dy = (double)pts[3 * j + 1] - (double)pts[3 * j + 4],
                 dz = (double)pts[3 * j + 2] - (double)pts[3 * j + 5];
    const double s = sqrt(dx * dx + dy * dy + dz * dz);
    seg += s;
    tot += s;
  }
  lengths[0] = seg;
  lengths[1] = tot;
}
