/* watershed.c — CPU restatement of skimage.segmentation.watershed as the reference uses it
 * (invesalius/data/watershed_process.py:39,52: watershed(gradient, markers.astype(int16),
 * bstruct), no mask, no compactness, no watershed line).
 *
 * TEST INFRASTRUCTURE ONLY (see oracle.c).
 *
 * scikit-image 0.24.0 is a third-party dependency of the reference (pyproject.toml:35) that
 * is not vendored with it, so this follows its published algorithm
 * (skimage/segmentation/_watershed_cy.pyx::watershed_raveled + heap_general.pxi) from
 * memory — PARITY UNPINNED:
 *   - every marker voxel is pushed (raveled order) with key (value = image, age = 0);
 *   - the heap is a plain array binary heap ordered by (value, age);
 *   - pop the smallest; for each neighbour in the order of _offsets_to_raveled_neighbors
 *     (footprint entries sorted by squared distance from the centre, stable, centre
 *     dropped): skip if out of the image or already labelled; otherwise label it with the
 *     popped voxel's label AT PUSH TIME and push it with (image[neighbour], ++age).
 * The SciPy callees (watershed_ift, morphological_gradient) are present in this image and
 * are called directly by oracle/__init__.py, so they need no restatement.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  double value;
  int64_t age;
  int64_t index;
} elem_t;

typedef struct {
  elem_t* a;
  int64_t n, cap;
} heap_t;

static int smaller(const elem_t* x, const elem_t* y) {
  if (x->value != y->value) return x->value < y->value;
  return x->age < y->age;
}
static void heap_push(heap_t* h, elem_t e) {
  if (h->n == h->cap) {
    h->cap *= 2;
    h->a = (elem_t*)realloc(h->a, sizeof(elem_t) * (size_t)h->cap);
  }
  int64_t child = h->n++;
  h->a[child] = e;
  while (child > 0) {
    int64_t parent = (child + 1) / 2 - 1;
    if (smaller(&h->a[child], &h->a[parent])) {
      elem_t t = h->a[child]; h->a[child] = h->a[parent]; h->a[parent] = t;
      child = parent;
    } else break;
  }
}
static elem_t heap_pop(heap_t* h) {
  elem_t top = h->a[0];
  if (h->n <= 1) { h->n = 0; return top; }
  h->n -= 1;
  h->a[0] = h->a[h->n];
  int64_t parent = 0, child = 1;
  while (child < h->n) {
    if (child + 1 < h->n && smaller(&h->a[child + 1], &h->a[child])) child += 1;
    if (smaller(&h->a[child], &h->a[parent])) {
      elem_t t = h->a[child]; h->a[child] = h->a[parent]; h->a[parent] = t;
      parent = child;
      child = 2 * child + 1;
    } else break;
  }
  return top;
}

/* image uint16 [nz][ny][nx]; markers int16; strct uint8 [sz][sy][sx] (odd dims); out int16 */
int orc_watershed_skimage(const uint16_t* image, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                          const uint8_t* strct, int64_t sz, int64_t sy, int64_t sx, int16_t* out) {
  int64_t n = nz * ny * nx;
  /* neighbour list sorted by squared distance (stable), centre removed */
  int64_t cz = sz / 2, cy = sy / 2, cx = sx / 2;
  int64_t cnt = 0;
  int64_t(*nb)[4] = (int64_t(*)[4])malloc(sizeof(int64_t) * 4 * (size_t)(sz * sy * sx));
  for (int64_t k = 0; k < sz; ++k)
    for (int64_t j = 0; j < sy; ++j)
      for (int64_t i = 0; i < sx; ++i)
        if (strct[(k * sy + j) * sx + i]) {
          int64_t dz = k - cz, dy = j - cy, dx = i - cx;
          if (dz == 0 && dy == 0 && dx == 0) continue;
          nb[cnt][0] = dz; nb[cnt][1] = dy; nb[cnt][2] = dx; nb[cnt][3] = dz * dz + dy * dy + dx * dx;
          ++cnt;
        }
  for (int64_t a = 1; a < cnt; ++a) { /* stable insertion sort by distance */
    int64_t t[4];
    memcpy(t, nb[a], sizeof(t));
    int64_t b = a - 1;
    while (b >= 0 && nb[b][3] > t[3]) { memcpy(nb[b + 1], nb[b], sizeof(t)); --b; }
    memcpy(nb[b + 1], t, sizeof(t));
  }
  memcpy(out, markers, sizeof(int16_t) * (size_t)n);
  heap_t h;
  h.cap = 1 << 16;
  h.n = 0;
  h.a = (elem_t*)malloc(sizeof(elem_t) * (size_t)h.cap);
  for (int64_t p = 0; p < n; ++p)
    if (out[p]) {
      elem_t e = {(double)image[p], 0, p};
      heap_push(&h, e);
    }
  int64_t age = 1;
  while (h.n > 0) {
    elem_t e = heap_pop(&h);
    int64_t z = e.index / (ny * nx), r = e.index % (ny * nx), y = r / nx, x = r % nx;
    for (int64_t k = 0; k < cnt; ++k) {
      int64_t zz = z + nb[k][0], yy = y + nb[k][1], xx = x + nb[k][2];
      if (zz < 0 || zz >= nz || yy < 0 || yy >= ny || xx < 0 || xx >= nx) continue; /* padded border: mask False */
      int64_t q = (zz * ny + yy) * nx + xx;
      if (out[q]) continue;
      age += 1;
      out[q] = out[e.index];
      elem_t ne = {(double)image[q], age, q};
      heap_push(&h, ne);
    }
  }
  free(h.a);
  free(nb);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * Order-independence model of the two sequential floods (TEST INFRASTRUCTURE).
 *
 * Both references label a voxel p from the neighbour that reaches it first in queue order.
 * Whatever that order is, the parent of p is one of its ADMISSIBLE predecessors:
 *   mode 0 (scipy.ndimage.watershed_ift): v -> p with max(C(v), |I(v) - I(p)|) == C(p), where C
 *          is the exact minimax path cost (SciPy relabels only on a strictly smaller cost and
 *          pops in non-decreasing cost order, so the final parent offered exactly C(p));
 *          neighbourhood = flat index + structure offset inside [0, N) as SciPy walks it;
 *   mode 1 (skimage.segmentation.watershed): p is labelled when its FIRST neighbour is popped;
 *          pops are ordered by flood level, so that neighbour has the smallest C among p's
 *          neighbours (C(marker) = I(marker), C(p) = max(I(p), min over neighbours C)).
 * set_out[p] = the label if every chain of admissible predecessors back to the markers
 * carries the same label (the reference's answer CANNOT depend on its queue order there),
 * INT32_MIN if two different labels can reach p (order dependent), 0 if unreachable.
 * cost_out = C. Costs by a bucket-queue Dijkstra (uint16 weights), sets by a worklist to the
 * least fixed point of  S(p) = join over admissible v of S(v).
 * ------------------------------------------------------------------------------------------ */
#define WS_MULTI INT32_MIN

int orc_ws_model(const uint16_t* image, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                 const uint8_t* strct, int64_t sz, int64_t sy, int64_t sx, int mode, uint32_t* cost_out,
                 int32_t* set_out) {
  const int64_t n = nz * ny * nx;
  int64_t noff = 0, off[27][3];
  for (int64_t k = 0; k < sz; ++k)
    for (int64_t j = 0; j < sy; ++j)
      for (int64_t i = 0; i < sx; ++i)
        if (strct[(k * sy + j) * sx + i]) {
          int64_t dz = k - sz / 2, dy = j - sy / 2, dx = i - sx / 2;
          if (dz == 0 && dy == 0 && dx == 0) continue;
          off[noff][0] = dz; off[noff][1] = dy; off[noff][2] = dx;
          ++noff;
        }
  const uint32_t INF = 0xffffffffu;
  /* neighbour of p by offset o (the voxel p + o), or -1 */
#define WS_NB(p, o, sign, q)                                                                          \
  do {                                                                                                \
    if (mode == 0) {                                                                                  \
      int64_t qq = (p) + (sign) * ((off[o][0] * ny + off[o][1]) * nx + off[o][2]);                    \
      (q) = (qq >= 0 && qq < n) ? qq : -1;                                                            \
    } else {                                                                                          \
      int64_t z = (p) / (ny * nx), r = (p) % (ny * nx), y = r / nx, x = r % nx;                       \
      int64_t zz = z + (sign)*off[o][0], yy = y + (sign)*off[o][1], xx = x + (sign)*off[o][2];        \
      (q) = (zz >= 0 && zz < nz && yy >= 0 && yy < ny && xx >= 0 && xx < nx) ? (zz * ny + yy) * nx + xx : -1; \
    }                                                                                                 \
  } while (0)
  /* ---- costs: label-correcting with a FIFO worklist (small test volumes) */
  int64_t* queue = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
  uint8_t* inq = (uint8_t*)calloc((size_t)n, 1);
  int64_t qh = 0, qt = 0, qn = 0;
  for (int64_t p = 0; p < n; ++p) {
    if (markers[p]) {
      cost_out[p] = mode == 0 ? 0u : (uint32_t)image[p];
      queue[qt] = p; qt = (qt + 1) % n; ++qn; inq[p] = 1;
    } else cost_out[p] = INF;
    set_out[p] = markers[p];
  }
  while (qn) {
    int64_t v = queue[qh]; qh = (qh + 1) % n; --qn; inq[v] = 0;
    for (int64_t o = 0; o < noff; ++o) {
      int64_t p;
      WS_NB(v, o, 1, p);
      if (p < 0 || markers[p]) continue;
      uint32_t w = mode == 0 ? (uint32_t)abs((int)image[v] - (int)image[p]) : (uint32_t)image[p];
      uint32_t cand = cost_out[v] > w ? cost_out[v] : w;
      if (cand < cost_out[p]) {
        cost_out[p] = cand;
        if (!inq[p]) { queue[qt] = p; qt = (qt + 1) % n; ++qn; inq[p] = 1; }
      }
    }
  }
  /* ---- label sets */
  qh = qt = qn = 0;
  for (int64_t p = 0; p < n; ++p)
    if (markers[p]) { queue[qt] = p; qt = (qt + 1) % n; ++qn; inq[p] = 1; }
  while (qn) {
    int64_t v = queue[qh]; qh = (qh + 1) % n; --qn; inq[v] = 0;
    const int32_t sv = set_out[v];
    if (sv == 0) continue;
    for (int64_t o = 0; o < noff; ++o) {
      int64_t p;
      WS_NB(v, o, 1, p);
      if (p < 0 || markers[p] || cost_out[p] == INF) continue;
      int admissible;
      if (mode == 0) {
        uint32_t w = (uint32_t)abs((int)image[v] - (int)image[p]);
        uint32_t via = cost_out[v] > w ? cost_out[v] : w;
        admissible = via == cost_out[p];
      } else {
        uint32_t cmin = INF;
        for (int64_t o2 = 0; o2 < noff; ++o2) {
          int64_t u;
          WS_NB(p, o2, -1, u);      /* the voxels that reach p */
          if (u >= 0 && cost_out[u] < cmin) cmin = cost_out[u];
        }
        admissible = cost_out[v] == cmin;
      }
      if (!admissible) continue;
      int32_t sp = set_out[p], ns = sp == 0 ? sv : (sp == sv ? sp : WS_MULTI);
      if (sv == WS_MULTI) ns = WS_MULTI;
      if (ns != sp) {
        set_out[p] = ns;
        if (!inq[p]) { queue[qt] = p; qt = (qt + 1) % n; ++qn; inq[p] = 1; }
      }
    }
  }
  free(queue);
  free(inq);
#undef WS_NB
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * Pointer-faithful restatement of scipy.ndimage.watershed_ift (scipy/ndimage/src/ni_measure.c,
 * NI_WatershedIFT; SciPy 1.14.0 pinned by the reference, 1.18.1 in this image) — TEST
 * INFRASTRUCTURE. SciPy itself is the reference's callee and is present, so it stays the
 * oracle; this restatement exists to EXPLAIN it (tests/test_oracle_watershed.py checks that it
 * reproduces SciPy bit for bit on hundreds of random volumes):
 *   - one doubly linked list per cost value; positive labels are pushed at the HEAD (so a
 *     bucket is a stack: depth-first, the marker with the highest raveled index first),
 *     negative labels at the tail;
 *   - a neighbour is  flat index + structure offset  inside [0, N): rows and planes wrap;
 *   - a voxel is relabelled only on a STRICTLY smaller cost max(cost(v), |I(v) - I(p)|);
 *   - quirk: before re-inserting an improved voxel SciPy unlinks it from its old list only
 *     `if (p->next || p->prev)`, so a voxel that is ALONE in its bucket stays linked there
 *     (first[old] keeps pointing at it) while it also enters the new bucket; later pushes into
 *     the old bucket then overwrite its `prev`, and a subsequent unlink splices the two lists:
 *     elements can be processed in the wrong bucket or never, and the final costs are then NOT
 *     the minimax costs. quirk = 0 runs the algorithm as intended (unlink whenever queued).
 * out: labels. *n_nonminimax (optional): voxels whose final cost differs from the exact minimax
 * cost can be found by comparing with orc_ws_model; here we only count sole-element events.
 * ------------------------------------------------------------------------------------------ */
int orc_ift_scipy(const uint16_t* image, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                  const uint8_t* strct, int64_t sz, int64_t sy, int64_t sx, int quirk, int16_t* out,
                  int64_t* sole_events) {
  const int64_t n = nz * ny * nx;
  int64_t noff = 0, offs[27];
  for (int64_t k = 0; k < sz; ++k)
    for (int64_t j = 0; j < sy; ++j)
      for (int64_t i = 0; i < sx; ++i)
        if (strct[(k * sy + j) * sx + i]) {
          int64_t o = ((k - sz / 2) * ny + (j - sy / 2)) * nx + (i - sx / 2);
          if (o != 0) offs[noff++] = o;
        }
  int maxval = 0;
  for (int64_t p = 0; p < n; ++p) if (image[p] > maxval) maxval = image[p];
  const int64_t NIL = -1;
  int64_t* nxt = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
  int64_t* prv = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
  int32_t* cost = (int32_t*)malloc(sizeof(int32_t) * (size_t)n);
  uint8_t* done = (uint8_t*)calloc((size_t)n, 1);
  uint8_t* queued = (uint8_t*)calloc((size_t)n, 1);   /* quirk = 0 only: is the voxel in a list? */
  int64_t* first = (int64_t*)malloc(sizeof(int64_t) * (size_t)(maxval + 2));
  int64_t* last = (int64_t*)malloc(sizeof(int64_t) * (size_t)(maxval + 2));
  for (int b = 0; b <= maxval + 1; ++b) first[b] = last[b] = NIL;
  int64_t sole = 0;
  for (int64_t j = 0; j < n; ++j) {
    out[j] = markers[j];
    nxt[j] = prv[j] = NIL;
    if (markers[j]) {
      cost[j] = 0;
      queued[j] = 1;
      if (first[0] == NIL) { first[0] = j; last[0] = j; }
      else if (markers[j] > 0) { nxt[j] = first[0]; prv[first[0]] = j; first[0] = j; }
      else { prv[j] = last[0]; nxt[last[0]] = j; last[0] = j; }
    } else cost[j] = maxval + 1;
  }
  for (int b = 0; b <= maxval; ++b)
    while (first[b] != NIL) {
      const int64_t v = first[b];
      first[b] = nxt[v];
      if (first[b] != NIL) prv[first[b]] = NIL;
      prv[v] = nxt[v] = NIL;
      done[v] = 1;
      queued[v] = 0;
      for (int64_t h = 0; h < noff; ++h) {
        const int64_t p = v + offs[h];
        if (p < 0 || p >= n || done[p]) continue;
        int w = (int)image[p] - (int)image[v];
        if (w < 0) w = -w;
        const int pc = cost[p], mx = cost[v] > w ? cost[v] : w;
        if (mx >= pc) continue;
        cost[p] = mx;
        out[p] = out[v];
        const int linked = quirk ? (nxt[p] != NIL || prv[p] != NIL) : queued[p];
        if (linked) {
          const int64_t pr = prv[p], nx_ = nxt[p];
          if (first[pc] == p) first[pc] = nx_;
          if (last[pc] == p) last[pc] = pr;
          if (pr != NIL) nxt[pr] = nx_;
          if (nx_ != NIL) prv[nx_] = pr;
        } else if (quirk && pc <= maxval && first[pc] == p) ++sole;
        queued[p] = 1;
        if (out[v] < 0) {
          prv[p] = last[mx]; nxt[p] = NIL;
          if (last[mx] != NIL) nxt[last[mx]] = p;
          last[mx] = p;
          if (first[mx] == NIL) first[mx] = p;
        } else {
          nxt[p] = first[mx]; prv[p] = NIL;
          if (first[mx] != NIL) prv[first[mx]] = p;
          first[mx] = p;
          if (last[mx] == NIL) last[mx] = p;
        }
      }
    }
  if (sole_events) *sole_events = sole;
  free(nxt); free(prv); free(cost); free(done); free(queued); free(first); free(last);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * orc_ws_labels — the device engines' complete labelling rule (b2v_ws_flood, DESIGN.md §6) in
 * O(N), so that every voxel of large volumes can be checked, ambiguous ones included (TEST
 * INFRASTRUCTURE). Same cost model and admissibility as orc_ws_model / tests/ws_model.py:
 *   1. C = exact minimax cost, by a bucket-queue Dijkstra (Dial: costs are uint16 values and a
 *      path's cost never decreases along it, so buckets are popped in increasing order);
 *   2. v -> p admissible: p is no marker, C(p) and C(v) finite and
 *        mode 0: max(C(v), |I(v) - I(p)|) == C(p);   mode 1: C(v) == min over p's neighbours of C;
 *   3. key (hops, code), code = label + 32768: breadth-first over admissible edges from the
 *      markers (hops 0, own code), in hop order; a voxel first seen at hop h + 1 takes the smallest
 *      code among its admissible predecessors at hop h (the minimum of hops << 32 | code);
 *   4. ambiguous: two different labels reach p along admissible edges (least fixed point of the
 *      label-set join, by a worklist: a set changes at most twice, empty -> one label -> several).
 * labels_out int16 (0 where no marker reaches); amb_out uint8; hops_out uint32 (optional, may be
 * NULL; 0xffffffff where unreached). Returns 0, or -1 if memory runs out.
 * ------------------------------------------------------------------------------------------ */
int orc_ws_labels(const uint16_t* image, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                  const uint8_t* strct, int64_t sz, int64_t sy, int64_t sx, int mode, int16_t* labels_out,
                  uint8_t* amb_out, uint32_t* hops_out) {
  const int64_t n = nz * ny * nx;
  const uint32_t INF = 0xffffffffu;
  int64_t noff = 0, off[27][3];
  for (int64_t k = 0; k < sz; ++k)
    for (int64_t j = 0; j < sy; ++j)
      for (int64_t i = 0; i < sx; ++i)
        if (strct[(k * sy + j) * sx + i]) {
          int64_t dz = k - sz / 2, dy = j - sy / 2, dx = i - sx / 2;
          if (dz == 0 && dy == 0 && dx == 0) continue;
          off[noff][0] = dz; off[noff][1] = dy; off[noff][2] = dx;
          ++noff;
        }
#define WL_NB(p, o, sign, q)                                                                          \
  do {                                                                                                \
    if (mode == 0) {                                                                                  \
      int64_t qq = (p) + (sign) * ((off[o][0] * ny + off[o][1]) * nx + off[o][2]);                    \
      (q) = (qq >= 0 && qq < n) ? qq : -1;                                                            \
    } else {                                                                                          \
      int64_t z_ = (p) / (ny * nx), r_ = (p) % (ny * nx), y_ = r_ / nx, x_ = r_ % nx;                 \
      int64_t zz = z_ + (sign)*off[o][0], yy = y_ + (sign)*off[o][1], xx = x_ + (sign)*off[o][2];     \
      (q) = (zz >= 0 && zz < nz && yy >= 0 && yy < ny && xx >= 0 && xx < nx) ? (zz * ny + yy) * nx + xx : -1; \
    }                                                                                                 \
  } while (0)
  uint32_t* cost = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)n);
  int64_t* nxt = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
  int64_t* prv = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
  int64_t* head = (int64_t*)malloc(sizeof(int64_t) * 65536);
  if (!cost || !nxt || !prv || !head) { free(cost); free(nxt); free(prv); free(head); return -1; }
  /* ---- 1. costs: one doubly linked list per cost value; a voxel is in at most one list */
  for (int b = 0; b < 65536; ++b) head[b] = -1;
#define WL_PUSH(p, b) do { prv[p] = -1; nxt[p] = head[b]; if (head[b] >= 0) prv[head[b]] = (p); head[b] = (p); } while (0)
#define WL_UNLINK(p, b) do { if (prv[p] >= 0) nxt[prv[p]] = nxt[p]; else head[b] = nxt[p]; if (nxt[p] >= 0) prv[nxt[p]] = prv[p]; } while (0)
  for (int64_t p = 0; p < n; ++p) {
    if (markers[p]) {
      cost[p] = mode == 0 ? 0u : (uint32_t)image[p];
      WL_PUSH(p, cost[p]);
    } else cost[p] = INF;
  }
  for (int64_t b = 0; b < 65536; ++b)
    while (head[b] >= 0) {
      const int64_t v = head[b];
      head[b] = nxt[v];
      if (head[b] >= 0) prv[head[b]] = -1;
      for (int64_t o = 0; o < noff; ++o) {
        int64_t p;
        WL_NB(v, o, 1, p);
        if (p < 0 || markers[p]) continue;
        const uint32_t w = mode == 0 ? (uint32_t)abs((int)image[v] - (int)image[p]) : (uint32_t)image[p];
        const uint32_t cand = (uint32_t)b > w ? (uint32_t)b : w;
        if (cand < cost[p]) {      /* cand >= b: p is in a bucket not yet popped, or in none */
          if (cost[p] != INF) WL_UNLINK(p, cost[p]);
          cost[p] = cand;
          WL_PUSH(p, cand);
        }
      }
    }
#undef WL_PUSH
#undef WL_UNLINK
  free(nxt); free(prv); free(head);
  /* the cost an admissible predecessor offers: mode 0 C(p) itself, mode 1 the smallest C among p's
   * neighbours (the voxels u with p = u + offset) */
  uint32_t* want = cost;
  if (mode == 1) {
    want = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)n);
    if (!want) { free(cost); return -1; }
    for (int64_t p = 0; p < n; ++p) {
      uint32_t cmin = INF;
      for (int64_t o = 0; o < noff; ++o) {
        int64_t u;
        WL_NB(p, o, -1, u);
        if (u >= 0 && cost[u] < cmin) cmin = cost[u];
      }
      want[p] = cmin;
    }
  }
#define WL_ADM(v, p)                                                                                  \
  (!markers[p] && cost[p] != INF && cost[v] != INF &&                                                 \
   (mode == 0 ? ((cost[v] > (uint32_t)abs((int)image[v] - (int)image[p]) ? cost[v]                    \
                                                                          : (uint32_t)abs((int)image[v] - (int)image[p])) == cost[p]) \
              : cost[v] == want[p]))
  /* ---- 3. keys: breadth-first in hop order */
  uint32_t* hops = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)n);
  uint16_t* code = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)n);
  int64_t* queue = (int64_t*)malloc(sizeof(int64_t) * (size_t)n);
  if (!hops || !code || !queue) {
    free(hops); free(code); free(queue); if (want != cost) free(want); free(cost);
    return -1;
  }
  int64_t qh = 0, qt = 0;
  for (int64_t p = 0; p < n; ++p) {
    if (markers[p]) { hops[p] = 0; code[p] = (uint16_t)(markers[p] + 32768); queue[qt++] = p; }
    else { hops[p] = INF; code[p] = 0; }
  }
  while (qh < qt) {
    const int64_t v = queue[qh++];
    for (int64_t o = 0; o < noff; ++o) {
      int64_t p;
      WL_NB(v, o, 1, p);
      if (p < 0 || !WL_ADM(v, p)) continue;
      if (hops[p] == INF) { hops[p] = hops[v] + 1; code[p] = code[v]; queue[qt++] = p; }
      else if (hops[p] == hops[v] + 1 && code[v] < code[p]) code[p] = code[v];
    }
  }
  for (int64_t p = 0; p < n; ++p) labels_out[p] = hops[p] == INF ? 0 : (int16_t)((int)code[p] - 32768);
  if (hops_out) memcpy(hops_out, hops, sizeof(uint32_t) * (size_t)n);
  free(hops); free(code);
  /* ---- 4. label sets: -1 empty, -2 two different labels, else the one label's code */
  int32_t* set = (int32_t*)malloc(sizeof(int32_t) * (size_t)n);
  uint8_t* inq = (uint8_t*)calloc((size_t)n, 1);
  if (!set || !inq) { free(set); free(inq); free(queue); if (want != cost) free(want); free(cost); return -1; }
  int64_t qn = 0;
  qh = qt = 0;
  for (int64_t p = 0; p < n; ++p) {
    set[p] = markers[p] ? (int32_t)markers[p] + 32768 : -1;
    if (markers[p]) { queue[qt] = p; qt = (qt + 1) % n; ++qn; inq[p] = 1; }
  }
  while (qn) {
    const int64_t v = queue[qh]; qh = (qh + 1) % n; --qn; inq[v] = 0;
    const int32_t sv = set[v];
    for (int64_t o = 0; o < noff; ++o) {
      int64_t p;
      WL_NB(v, o, 1, p);
      if (p < 0 || !WL_ADM(v, p)) continue;
      const int32_t sp = set[p], ns = sp == -1 ? sv : (sp == sv ? sp : -2);
      if (ns != sp) {
        set[p] = ns;
        if (!inq[p]) { queue[qt] = p; qt = (qt + 1) % n; ++qn; inq[p] = 1; }
      }
    }
  }
  for (int64_t p = 0; p < n; ++p) amb_out[p] = set[p] == -2;
#undef WL_ADM
#undef WL_NB
  free(set); free(inq); free(queue);
  if (want != cost) free(want);
  free(cost);
  return 0;
}
