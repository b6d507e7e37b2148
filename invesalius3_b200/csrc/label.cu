// Connected-component labelling: scipy.ndimage.label as InVesalius calls it before
// fill_holes_automatically (invesalius/data/mask.py:526-530, :549-552), in
// get_largest_connected_component (imagedata_utils.py:717-721), and count_regions
// (invesalius_rs/src/count_regions.rs:5-18). SURVEY 8f-3.
//
// Union-find over the voxels (parents only ever decrease, the root of a component is its smallest
// flat index): every foreground voxel unites with its foreground neighbours in the BACKWARD half of
// the structuring element (the forward half is the neighbour's backward half); a union along y / z
// is skipped where the previous voxel of the row already made it (both rows continue their runs).
// Labels are then numbered in the order of the components' first voxel in raster order, which is
// SciPy's numbering: roots are flagged, an exclusive scan over the flags ranks them.
#include "b2v_common.cuh"
#include "scan.cuh"

#include <type_traits>

namespace {

__device__ __forceinline__ int uf_find(int* p, int i) {
  int c = i;
  while (true) {
    const int n = ((volatile int*)p)[c];
    if (n == c) return c;
    const int nn = ((volatile int*)p)[n];
    if (nn != n) p[c] = nn;      // path halving: nn is an ancestor of c
    c = n;
  }
}

__device__ __forceinline__ void uf_unite(int* p, int a, int b) {
  while (true) {
    a = uf_find(p, a);
    b = uf_find(p, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&p[a], b);      // hang the larger root under the smaller
    if (old == a) return;
    a = old;                                  // somebody re-parented a meanwhile: go on from there
  }
}

struct LDims { int nz, ny, nx; long long n; };

__global__ void __launch_bounds__(256) k_label_init(const uint8_t* __restrict__ fg, LDims d, int* __restrict__ parent) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < d.n; i += stride) parent[i] = fg[i] ? (int)i : -1;
}

// sb: bit (oz+1)*9 + (oy+1)*3 + (ox+1) of the 3x3x3 structuring element
__global__ void __launch_bounds__(256) k_label_merge(const uint8_t* __restrict__ fg, LDims d, uint32_t sb, int* parent) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < d.n; i += stride) {
    if (!fg[i]) continue;
    const int x = (int)(i % d.nx);
    const long long r = i / d.nx;
    const int y = (int)(r % d.ny), z = (int)(r / d.ny);
    const bool prev = x > 0 && fg[i - 1] && ((sb >> 12) & 1u);   // (0, 0, -1) set and foreground
#pragma unroll
    for (int o = 0; o < 13; ++o) {               // backward half: offsets with a negative flat index
      if (!((sb >> o) & 1u)) continue;
      const int oz = o / 9 - 1, oy = (o / 3) % 3 - 1, ox = o % 3 - 1;
      const int zz = z + oz, yy = y + oy, xx = x + ox;
      if (zz < 0 || yy < 0 || yy >= d.ny || xx < 0 || xx >= d.nx) continue;
      const long long j = ((long long)zz * d.ny + yy) * d.nx + xx;
      if (!fg[j]) continue;
      // straight neighbours across rows / planes: the previous voxel of my row made the same union if
      // it is foreground and so is its own neighbour across (the two runs continue side by side)
      if (ox == 0 && (oy != 0 || oz != 0) && prev && fg[j - 1]) continue;
      uf_unite(parent, (int)i, (int)j);
    }
  }
}

// flatten + root flags per block -> block sums
constexpr int kScanBlock = 2048;   // elements per block (256 threads x 8)

// read-only find: the flatten pass must not race with path-halving stores of other threads (a
// late store of a stale grandparent would leave an entry pointing at a non-root)
__device__ __forceinline__ int uf_find_ro(const int* p, int i) {
  int c = i;
  while (true) {
    const int n = p[c];
    if (n == c) return c;
    c = n;
  }
}

// labels[i] = root of i (0xffffffff: background); roots counted per block
__global__ void __launch_bounds__(256) k_label_flatten_count(const int* __restrict__ parent, LDims d,
                                                             uint32_t* __restrict__ labels, uint32_t* __restrict__ bsum) {
  __shared__ uint32_t s[8];
  const long long base = (long long)blockIdx.x * kScanBlock;
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long long i = base + threadIdx.x * 8 + k;
    if (i < d.n) {
      uint32_t r = 0xffffffffu;
      if (parent[i] >= 0) {
        r = (uint32_t)uf_find_ro(parent, (int)i);
        c += (r == (uint32_t)i);
      }
      labels[i] = r;
    }
  }
  const uint32_t t = block_sum(c, s);
  if (threadIdx.x == 0) bsum[blockIdx.x] = t;
}

// roots get their number (rank in raster order + 1), stored in parent[] (no longer needed as a forest)
__global__ void __launch_bounds__(256) k_label_number_roots(int* parent, LDims d, const uint32_t* __restrict__ bsum,
                                                            const uint32_t* __restrict__ labels) {
  __shared__ uint32_t s_w[8];
  __shared__ uint32_t s_tot;
  const long long base = (long long)blockIdx.x * kScanBlock;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long long i = base + threadIdx.x * 8 + k;
    if (i < d.n && labels[i] == (uint32_t)i) { flags |= 1u << k; ++c; }
  }
  uint32_t before = bsum[blockIdx.x] + block_exscan(c, s_w, &s_tot);
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if ((flags >> k) & 1u) parent[base + threadIdx.x * 8 + k] = (int)(++before);
}

// labels[i]: root index -> the root's number (read from parent[root]); background -> 0
__global__ void __launch_bounds__(256) k_label_assign(const int* __restrict__ parent, LDims d, uint32_t* labels) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < d.n; i += stride) {
    const uint32_t r = labels[i];
    labels[i] = r == 0xffffffffu ? 0u : (uint32_t)parent[r];
  }
}

// count_regions (count_regions.rs:5-18): out[p] = number of voxels that carry image[p]'s value.
// The size table is a histogram whose background bin usually holds most of the volume, so one atomic per
// voxel would serialise on it. Each lane keeps the run of equal values it is reading (value, length) and
// only adds a run to the table where its value changes; the lanes of a warp that end runs of one value at
// the same step add them with one atomic. A volume of one label costs one atomic per warp.
// All lanes of a warp call this together (f: this lane ends the run v of length c). The lanes that end runs
// of one value at one step are neighbours (they crossed the same edge); where no two neighbours do, as in
// noise, the grouping would buy nothing and each lane adds its own run.
__device__ __forceinline__ void add_runs(bool f, uint32_t v, uint32_t c, uint32_t* counts) {
  const unsigned any = __ballot_sync(0xffffffffu, f);
  if (!any) return;
  const uint32_t next = __shfl_down_sync(0xffffffffu, v, 1);
  const unsigned pairs = __ballot_sync(0xffffffffu, f && v == next) & (any >> 1);
  if (!f) return;
  if (!pairs) {
    atomicAdd(&counts[v], c);
    return;
  }
  const unsigned g = __match_any_sync(any, v);
  const unsigned s = __reduce_add_sync(g, c);
  if ((threadIdx.x & 31) == (unsigned)(__ffs(g) - 1)) atomicAdd(&counts[v], s);
}

// counts[v] += voxels holding v, v in [0, nbins); any other value sets *status. The trip count depends on
// the warp only, so every warp stays converged for add_runs (block size: a multiple of 32).
template <typename T>
__global__ void __launch_bounds__(256) k_region_sizes(const T* __restrict__ img, int64_t n, uint32_t nbins,
                                                      uint32_t* counts, int* status) {
  constexpr int U = 8;                       // loads in flight per lane
  const unsigned lane = threadIdx.x & 31;
  const int64_t step = gstride() * U;
  uint32_t cv = 0, cc = 0;                   // this lane's run: value, length (0: none yet)
  for (int64_t base = (gtid() - lane) * U; base < n; base += step) {
    T v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t i = base + k * 32 + lane;
      v[k] = i < n ? img[i] : T(0);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t x = (int64_t)v[k];
      const bool in = base + k * 32 + lane < n;
      const bool ok = in && x >= 0 && x < (int64_t)nbins;
      if (in && !ok) *status = 1;
      add_runs(ok && cc && (uint32_t)x != cv, cv, cc, counts);
      if (ok) {
        cc = (cc && (uint32_t)x == cv) ? cc + 1 : 1;
        cv = (uint32_t)x;
      }
    }
  }
  add_runs(cc != 0, cv, cc, counts);
}
template <typename T>
__global__ void __launch_bounds__(256) k_count_gather(const T* __restrict__ img, long long n, uint32_t nbins,
                                                      const uint32_t* __restrict__ counts, uint32_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long v = (long long)img[i];
    out[i] = (v >= 0 && v < (long long)nbins) ? counts[v] : 0u;
  }
}

// ---- the remove-tiny-objects plugin (plugins/remove_tiny_objects/gui.py) over a resident label image ----
// A voxel is tiny where its region holds at most min_size voxels (labels outside the size table never are).
struct TinyRegion {
  const uint32_t* __restrict__ labels;
  const uint32_t* __restrict__ sizes;
  int64_t nsizes;
  int64_t min_size;
  __device__ __forceinline__ bool of(uint32_t l) const { return l < nsizes && (int64_t)__ldg(sizes + l) <= min_size; }
  __device__ __forceinline__ bool operator()(int64_t i) const { return of(labels[i]); }
};

// The plugin's OnRemove selection: preview > 127.
struct PreviewSet {
  const uint8_t* __restrict__ preview;
  __device__ __forceinline__ bool operator()(int64_t i) const { return preview[i] > 127; }
};

// out[i] = 255 where tiny, else 0; vec: labels 16-byte and out 4-byte aligned, four voxels a lane
__global__ void __launch_bounds__(256) k_tiny_preview(TinyRegion t, int64_t n, uint8_t* __restrict__ out, bool vec) {
  const int64_t nv = vec ? n / 4 : 0;
  for (int64_t j = gtid(); j < nv; j += gstride()) {
    const uint4 l = reinterpret_cast<const uint4*>(t.labels)[j];
    reinterpret_cast<uint32_t*>(out)[j] = (t.of(l.x) ? 0xffu : 0u) | (t.of(l.y) ? 0xff00u : 0u) |
                                          (t.of(l.z) ? 0xff0000u : 0u) | (t.of(l.w) ? 0xff000000u : 0u);
  }
  for (int64_t i = nv * 4 + gtid(); i < n; i += gstride()) out[i] = t(i) ? 255 : 0;
}

// mask[1 + z][1 + y][1 + x] = 1 where sel(body index), on the padded [dz + 1][dy + 1][dx + 1] layout; the
// flag planes z = 0, y = 0 and x = 0 are never written. One block a body row.
template <class Sel>
__global__ void __launch_bounds__(256) k_mark_body(Sel sel, int64_t dy, int64_t dx, int64_t nrows, uint8_t* mask) {
  for (int64_t r = blockIdx.x; r < nrows; r += gridDim.x) {
    const int64_t z = r / dy, y = r - z * dy;
    uint8_t* row = mask + ((z + 1) * (dy + 1) + y + 1) * (dx + 1) + 1;
    for (int64_t x = threadIdx.x; x < dx; x += blockDim.x)
      if (sel(r * dx + x)) row[x] = 1;
  }
}

// ---- Z-sharded labelling (dist.label): boundary forest, resolve, relabel ------------------------------
// The two planes around a shard boundary: the lower shard's last plane of local labels (`lo`, ids
// 1..n_lo) and the upper shard's first plane (`hi`, ids 1..n_hi). Node of a label: l for the lower
// plane, n_lo + l for the upper one, so node order is provisional-id order (P = base_lo + node, since
// the upper shard's base is base_lo + n_lo). Only the labels present on the two planes are ever
// touched in the node-indexed arrays, so the work is O(plane) whatever the label counts.
struct BDims { int ny, nx; int a; uint32_t n_lo; };      // a = ny * nx voxels per plane

__device__ __forceinline__ int lb_node(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, const BDims& d,
                                       int v) {
  if (v < d.a) return (int)lo[v];
  const uint32_t l = hi[v - d.a];
  return l ? (int)(d.n_lo + l) : 0;
}

// parent[node] = node, rep[node] = INT_MAX for every label on the two planes (racing writers store equal values)
__global__ void __launch_bounds__(256) k_lb_init(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, BDims d,
                                                 int* __restrict__ parent, int* __restrict__ rep) {
  for (int64_t v = gtid(); v < 2ll * d.a; v += gstride()) {
    const int a = lb_node(lo, hi, d, (int)v);
    if (a) { parent[a] = a; rep[a] = 0x7fffffff; }
  }
}

// rep[node] = first plane voxel carrying it (lower plane first, raster order); every lower voxel unites
// with the upper voxels at the structure's z = +1 offsets (zb: bit (oy+1)*3 + (ox+1)). A union is skipped
// where the previous voxel of the row made the same one (same label below, same label at the shifted offset).
__global__ void __launch_bounds__(256) k_lb_unite(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, BDims d,
                                                  uint32_t zb, int* parent, int* __restrict__ rep) {
  for (int64_t vv = gtid(); vv < 2ll * d.a; vv += gstride()) {
    const int v = (int)vv;
    const int a = lb_node(lo, hi, d, v);
    if (!a) continue;
    atomicMin(&rep[a], v);
    if (v >= d.a) continue;
    const int y = v / d.nx, x = v % d.nx;
    const bool prev = x > 0 && lo[v - 1] == (uint32_t)a;
#pragma unroll
    for (int o = 0; o < 9; ++o) {
      if (!((zb >> o) & 1u)) continue;
      const int yy = y + o / 3 - 1, xx = x + o % 3 - 1;
      if (yy < 0 || yy >= d.ny || xx < 0 || xx >= d.nx) continue;
      const int j = yy * d.nx + xx;
      const uint32_t b = hi[j];
      if (!b) continue;
      if (prev && xx > 0 && hi[j - 1] == b) continue;
      uf_unite(parent, a, (int)(d.n_lo + b));
    }
  }
}

// plane voxel v emits its label's pair iff it is the label's representative and the label is not a root
__device__ __forceinline__ bool lb_emits(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, const BDims& d,
                                         const int* parent, const int* __restrict__ rep, int64_t v, int* a_out, int* r_out) {
  if (v >= 2ll * d.a) return false;
  const int a = lb_node(lo, hi, d, (int)v);
  if (!a || rep[a] != (int)v) return false;
  const int r = uf_find_ro(parent, a);
  *a_out = a;
  *r_out = r;
  return r != a;
}

__global__ void __launch_bounds__(256) k_lb_count(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, BDims d,
                                                  const int* parent, const int* __restrict__ rep, uint32_t* __restrict__ bsum) {
  __shared__ uint32_t s[8];
  const int64_t base = (int64_t)blockIdx.x * kScanBlock;
  uint32_t c = 0;
  int a, r;
#pragma unroll
  for (int k = 0; k < 8; ++k) c += lb_emits(lo, hi, d, parent, rep, base + threadIdx.x * 8 + k, &a, &r);
  const uint32_t t = block_sum(c, s);
  if (threadIdx.x == 0) bsum[blockIdx.x] = t;
}

// pairs[k] = (P(node), P(root of node)) in the order of the representatives (bsum: scanned block counts)
__global__ void __launch_bounds__(256) k_lb_emit(const uint32_t* __restrict__ lo, const uint32_t* __restrict__ hi, BDims d,
                                                 const int* parent, const int* __restrict__ rep,
                                                 const uint32_t* __restrict__ bsum, int64_t base_lo, int64_t* __restrict__ pairs) {
  __shared__ uint32_t s_w[8];
  __shared__ uint32_t s_tot;
  const int64_t base = (int64_t)blockIdx.x * kScanBlock;
  int a[8], r[8];
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if (lb_emits(lo, hi, d, parent, rep, base + threadIdx.x * 8 + k, &a[k], &r[k])) { flags |= 1u << k; ++c; }
  int64_t at = bsum[blockIdx.x] + block_exscan(c, s_w, &s_tot);
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if ((flags >> k) & 1u) {
      pairs[2 * at] = base_lo + a[k];
      pairs[2 * at + 1] = base_lo + r[k];
      ++at;
    }
}

// first index of the sorted ends[0, n) that is >= key
__device__ __forceinline__ int64_t lower_bound64(const int64_t* __restrict__ ends, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (ends[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(256) k_lr_init(int64_t n, int* __restrict__ parent) {
  for (int64_t i = gtid(); i < n; i += gstride()) parent[i] = (int)i;
}

// union-find over the positions of the pair endpoints in `ends` (position order = id order, so the root of
// every set is its smallest id); an endpoint missing from `ends` sets *status
__global__ void __launch_bounds__(256) k_lr_unite(const int64_t* __restrict__ pairs, int64_t npairs,
                                                  const int64_t* __restrict__ ends, int64_t n, int* parent, int* status) {
  for (int64_t j = gtid(); j < npairs; j += gstride()) {
    const int64_t p = pairs[2 * j], q = pairs[2 * j + 1];
    const int64_t a = lower_bound64(ends, n, p), b = lower_bound64(ends, n, q);
    if (a >= n || b >= n || ends[a] != p || ends[b] != q) { *status = 1; continue; }
    uf_unite(parent, (int)a, (int)b);
  }
}

// root[i] = root position of i; non-roots (the set M) counted per block
__global__ void __launch_bounds__(256) k_lr_flatten_count(const int* parent, int64_t n, int* __restrict__ root,
                                                          uint32_t* __restrict__ bsum) {
  __shared__ uint32_t s[8];
  const int64_t base = (int64_t)blockIdx.x * kScanBlock;
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int64_t i = base + threadIdx.x * 8 + k;
    if (i < n) {
      const int r = uf_find_ro(parent, (int)i);
      root[i] = r;
      c += (r != (int)i);
    }
  }
  const uint32_t t = block_sum(c, s);
  if (threadIdx.x == 0) bsum[blockIdx.x] = t;
}

// before[i] = |{non-roots at positions < i}| (bsum: scanned block counts)
__global__ void __launch_bounds__(256) k_lr_rank(const int* __restrict__ root, int64_t n, const uint32_t* __restrict__ bsum,
                                                 uint32_t* __restrict__ before) {
  __shared__ uint32_t s_w[8];
  __shared__ uint32_t s_tot;
  const int64_t base = (int64_t)blockIdx.x * kScanBlock;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int64_t i = base + threadIdx.x * 8 + k;
    if (i < n && root[i] != (int)i) { flags |= 1u << k; ++c; }
  }
  uint32_t at = bsum[blockIdx.x] + block_exscan(c, s_w, &s_tot);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int64_t i = base + threadIdx.x * 8 + k;
    if (i < n) before[i] = at;
    at += (flags >> k) & 1u;
  }
}

// lut[l] = Final(base + l) = R - |{Q in M : Q < R}|, R = root(base + l) (itself when it is no endpoint);
// lut[0] = 0. nmerged = |M|.
__global__ void __launch_bounds__(256) k_lr_lut(const int64_t* __restrict__ ends, int64_t n, const int* __restrict__ root,
                                                const uint32_t* __restrict__ before, const uint32_t* __restrict__ nmerged,
                                                int64_t base, int64_t nlocal, uint32_t* __restrict__ lut) {
  for (int64_t l = gtid(); l <= nlocal; l += gstride()) {
    if (l == 0) { lut[0] = 0; continue; }
    const int64_t p = base + l;
    const int64_t k = lower_bound64(ends, n, p);
    int64_t r = p, c;
    if (k < n && ends[k] == p) {
      const int ri = root[k];
      r = ends[ri];
      c = before[ri];
    } else {
      c = k < n ? before[k] : *nmerged;
    }
    lut[l] = (uint32_t)(r - c);
  }
}

// labels[i] = lut[labels[i]] (values outside the table are left as they are)
__global__ void __launch_bounds__(256) k_label_relabel(uint32_t* labels, int64_t n, const uint32_t* __restrict__ lut,
                                                       int64_t nlut, bool vec) {
  const auto map = [&](uint32_t v) { return v < (uint64_t)nlut ? __ldg(lut + v) : v; };
  const int64_t nv = vec ? n / 4 : 0;
  uint4* l4 = reinterpret_cast<uint4*>(labels);
  for (int64_t i = gtid(); i < nv; i += gstride()) {
    uint4 v = l4[i];
    v.x = map(v.x); v.y = map(v.y); v.z = map(v.z); v.w = map(v.w);
    l4[i] = v;
  }
  for (int64_t i = nv * 4 + gtid(); i < n; i += gstride()) labels[i] = map(labels[i]);
}

// sb: the strct_mask of a 1- or 3-wide structuring element; B2V_ERR_ARG (with SciPy's message
// where it has one) for any other shape or an asymmetric element
int structure_bits(const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, uint32_t* sb_out) {
  B2V_REQUIRE(odz >= 1 && ody >= 1 && odx >= 1 && odz <= 3 && ody <= 3 && odx <= 3 && (odz & 1) && (ody & 1) && (odx & 1),
              B2V_ERR_ARG, "label: the structuring element must be 1 or 3 wide on every axis");
  const uint32_t sb = strct_mask(strct_host, odz, ody, odx);
  for (int o = 0; o < 13; ++o)     // SciPy: "structuring element is not symmetric"
    B2V_REQUIRE(((sb >> o) & 1u) == ((sb >> (26 - o)) & 1u), B2V_ERR_ARG, "label: structuring element is not symmetric");
  *sb_out = sb;
  return B2V_OK;
}

struct LbLayout { int* parent; int* rep; uint32_t* bsum; int64_t nb; };

LbLayout lb_layout(void* ws, int64_t ny, int64_t nx, int64_t n_lo, int64_t n_hi) {
  const int64_t nodes = n_lo + n_hi + 1;
  char* p = (char*)ws;
  LbLayout L;
  L.parent = (int*)p;
  L.rep = (int*)(p + align256(nodes * 4));
  L.bsum = (uint32_t*)(p + 2 * align256(nodes * 4));
  L.nb = ceil_div64(2 * ny * nx, kScanBlock);
  return L;
}

}  // namespace

extern "C" int64_t b2v_label_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return align256(n * 4) + align256((ceil_div64(n, kScanBlock) + 1) * 4) + 256;
}

extern "C" int b2v_label(const uint8_t* input, int64_t nz, int64_t ny, int64_t nx, const uint8_t* strct_host, int64_t odz,
                         int64_t ody, int64_t odx, uint32_t* labels, void* workspace, void* stream, int64_t* nlabels_host) {
  B2V_REQUIRE(input && labels && workspace && nlabels_host && strct_host, B2V_ERR_ARG, "label: null pointer");
  B2V_REQUIRE(nz > 0 && ny > 0 && nx > 0 && nz * ny * nx < (1ll << 31), B2V_ERR_ARG, "label: empty volume or more than 2^31 voxels");
  uint32_t sb = 0;
  int rc;
  if ((rc = structure_bits(strct_host, odz, ody, odx, &sb))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  LDims d = {(int)nz, (int)ny, (int)nx, nz * ny * nx};
  int* parent = (int*)workspace;
  uint32_t* bsum = (uint32_t*)((char*)workspace + align256(d.n * 4));
  const long long nb = ceil_div64(d.n, kScanBlock);
  k_label_init<<<b2v_grid(d.n, 256 * 4, 16), 256, 0, s>>>(input, d, parent);
  if ((rc = b2v_check_launch("k_label_init"))) return rc;
  k_label_merge<<<b2v_grid(d.n, 256 * 4, 16), 256, 0, s>>>(input, d, sb, parent);
  if ((rc = b2v_check_launch("k_label_merge"))) return rc;
  k_label_flatten_count<<<(unsigned)nb, 256, 0, s>>>(parent, d, labels, bsum);
  if ((rc = b2v_check_launch("k_label_flatten_count"))) return rc;
  k_scan_sums<uint32_t><<<1, 1024, 0, s>>>(bsum, nb, bsum + nb);
  if ((rc = b2v_check_launch("k_scan_sums"))) return rc;
  k_label_number_roots<<<(unsigned)nb, 256, 0, s>>>(parent, d, bsum, labels);
  if ((rc = b2v_check_launch("k_label_number_roots"))) return rc;
  k_label_assign<<<b2v_grid(d.n, 256 * 4, 16), 256, 0, s>>>(parent, d, labels);
  if ((rc = b2v_check_launch("k_label_assign"))) return rc;
  uint32_t total = 0;
  B2V_CUDA(cudaMemcpyAsync(&total, bsum + nb, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  *nlabels_host = (int64_t)total;
  return B2V_OK;
}

extern "C" int64_t b2v_label_boundary_workspace_bytes(int64_t ny, int64_t nx, int64_t n_lo, int64_t n_hi) {
  if (ny <= 0 || nx <= 0 || n_lo < 0 || n_hi < 0) return 0;
  return 2 * align256((n_lo + n_hi + 1) * 4) + align256((ceil_div64(2 * ny * nx, kScanBlock) + 1) * 4);
}

static int lb_check(const uint32_t* lo, const uint32_t* hi, int64_t ny, int64_t nx, int64_t n_lo, int64_t n_hi, void* ws) {
  B2V_REQUIRE(lo && hi && ws, B2V_ERR_ARG, "label_boundary: null pointer");
  B2V_REQUIRE(ny > 0 && nx > 0 && 2 * ny * nx < (1ll << 31), B2V_ERR_ARG, "label_boundary: empty plane or more than 2^30 voxels");
  B2V_REQUIRE(n_lo >= 0 && n_hi >= 0 && n_lo + n_hi < (1ll << 31) - 1, B2V_ERR_ARG,
              "label_boundary: the two shards hold 2^31 - 1 labels or more");
  return B2V_OK;
}

extern "C" int b2v_label_boundary_count(const uint32_t* lo_plane, const uint32_t* hi_plane, int64_t ny, int64_t nx,
                                        const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, int64_t n_lo,
                                        int64_t n_hi, void* workspace, void* stream, int64_t* npairs_host) {
  int rc;
  if ((rc = lb_check(lo_plane, hi_plane, ny, nx, n_lo, n_hi, workspace))) return rc;
  B2V_REQUIRE(strct_host && npairs_host, B2V_ERR_ARG, "label_boundary: null pointer");
  uint32_t sb = 0;
  if ((rc = structure_bits(strct_host, odz, ody, odx, &sb))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const LbLayout L = lb_layout(workspace, ny, nx, n_lo, n_hi);
  const BDims d = {(int)ny, (int)nx, (int)(ny * nx), (uint32_t)n_lo};
  const uint32_t zb = (sb >> 18) & 0x1ffu;      // the structure's z = +1 plane
  if (!zb) {                                    // 1 wide along z: the shards do not touch
    B2V_CUDA(cudaMemsetAsync(L.bsum, 0, (L.nb + 1) * 4, s));
    *npairs_host = 0;
    return B2V_OK;
  }
  k_lb_init<<<b2v_grid(2ll * d.a, 256 * 4, 16), 256, 0, s>>>(lo_plane, hi_plane, d, L.parent, L.rep);
  if ((rc = b2v_check_launch("k_lb_init"))) return rc;
  k_lb_unite<<<b2v_grid(2ll * d.a, 256 * 4, 16), 256, 0, s>>>(lo_plane, hi_plane, d, zb, L.parent, L.rep);
  if ((rc = b2v_check_launch("k_lb_unite"))) return rc;
  k_lb_count<<<(unsigned)L.nb, 256, 0, s>>>(lo_plane, hi_plane, d, L.parent, L.rep, L.bsum);
  if ((rc = b2v_check_launch("k_lb_count"))) return rc;
  k_scan_sums<uint32_t><<<1, 1024, 0, s>>>(L.bsum, L.nb, L.bsum + L.nb);
  if ((rc = b2v_check_launch("k_scan_sums"))) return rc;
  uint32_t total = 0;
  B2V_CUDA(cudaMemcpyAsync(&total, L.bsum + L.nb, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  *npairs_host = (int64_t)total;
  return B2V_OK;
}

extern "C" int b2v_label_boundary_emit(const uint32_t* lo_plane, const uint32_t* hi_plane, int64_t ny, int64_t nx,
                                       int64_t n_lo, int64_t n_hi, int64_t base_lo, int64_t npairs, int64_t* pairs,
                                       void* workspace, void* stream) {
  int rc;
  if ((rc = lb_check(lo_plane, hi_plane, ny, nx, n_lo, n_hi, workspace))) return rc;
  if (!npairs) return B2V_OK;         // also where the count never built the forest (structure 1 wide along z)
  B2V_REQUIRE(pairs && base_lo >= 0, B2V_ERR_ARG, "label_boundary: null pointer or negative base");
  cudaStream_t s = (cudaStream_t)stream;
  const LbLayout L = lb_layout(workspace, ny, nx, n_lo, n_hi);
  const BDims d = {(int)ny, (int)nx, (int)(ny * nx), (uint32_t)n_lo};
  k_lb_emit<<<(unsigned)L.nb, 256, 0, s>>>(lo_plane, hi_plane, d, L.parent, L.rep, L.bsum, base_lo, pairs);
  return b2v_check_launch("k_lb_emit");
}

extern "C" int64_t b2v_label_resolve_workspace_bytes(int64_t nends) {
  if (nends < 0) return 0;
  return 3 * align256(nends * 4) + align256((ceil_div64(nends, kScanBlock) + 1) * 4) + 256;
}

extern "C" int b2v_label_resolve(const int64_t* pairs, int64_t npairs, const int64_t* ends, int64_t nends, int64_t base,
                                 int64_t nlocal, uint32_t* lut, void* workspace, void* stream, int64_t* nmerged_host) {
  B2V_REQUIRE(lut && workspace && nmerged_host && (pairs || !npairs) && (ends || !nends), B2V_ERR_ARG,
              "label_resolve: null pointer");
  B2V_REQUIRE(npairs >= 0 && nends >= 0 && nends < (1ll << 31) && base >= 0 && nlocal >= 0, B2V_ERR_ARG,
              "label_resolve: bad sizes");
  B2V_REQUIRE(base + nlocal < (1ll << 32), B2V_ERR_RANGE, "label_resolve: provisional ids beyond uint32");
  cudaStream_t s = (cudaStream_t)stream;
  char* p = (char*)workspace;
  int* parent = (int*)p;
  int* root = (int*)(p + align256(nends * 4));
  uint32_t* before = (uint32_t*)(p + 2 * align256(nends * 4));
  uint32_t* bsum = (uint32_t*)(p + 3 * align256(nends * 4));
  const int64_t nb = ceil_div64(nends, kScanBlock);
  int* status = (int*)(p + 3 * align256(nends * 4) + align256((nb + 1) * 4));
  int rc;
  B2V_CUDA(cudaMemsetAsync(status, 0, 4, s));
  if (nends) {
    k_lr_init<<<b2v_grid(nends, 256 * 4, 16), 256, 0, s>>>(nends, parent);
    if ((rc = b2v_check_launch("k_lr_init"))) return rc;
    if (npairs) {
      k_lr_unite<<<b2v_grid(npairs, 256, 16), 256, 0, s>>>(pairs, npairs, ends, nends, parent, status);
      if ((rc = b2v_check_launch("k_lr_unite"))) return rc;
    }
    k_lr_flatten_count<<<(unsigned)nb, 256, 0, s>>>(parent, nends, root, bsum);
    if ((rc = b2v_check_launch("k_lr_flatten_count"))) return rc;
    k_scan_sums<uint32_t><<<1, 1024, 0, s>>>(bsum, nb, bsum + nb);
    if ((rc = b2v_check_launch("k_scan_sums"))) return rc;
    k_lr_rank<<<(unsigned)nb, 256, 0, s>>>(root, nends, bsum, before);
    if ((rc = b2v_check_launch("k_lr_rank"))) return rc;
  } else {
    B2V_CUDA(cudaMemsetAsync(bsum, 0, 4, s));
  }
  k_lr_lut<<<b2v_grid(nlocal + 1, 256 * 4, 16), 256, 0, s>>>(ends, nends, root, before, bsum + nb, base, nlocal, lut);
  if ((rc = b2v_check_launch("k_lr_lut"))) return rc;
  uint32_t host[2] = {0, 0};
  B2V_CUDA(cudaMemcpyAsync(&host[0], bsum + nb, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(&host[1], status, 4, cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(host[1] == 0, B2V_ERR_ARG, "label_resolve: a pair endpoint is missing from ends");
  *nmerged_host = (int64_t)host[0];
  return B2V_OK;
}

extern "C" int b2v_label_relabel(uint32_t* labels, int64_t n, const uint32_t* lut, int64_t nlut, void* stream) {
  B2V_REQUIRE(labels && lut && n >= 0 && nlut > 0, B2V_ERR_ARG, "label_relabel: bad arguments");
  if (!n) return B2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  k_label_relabel<<<b2v_grid(n, 256 * 16, 16), 256, 0, s>>>(labels, n, lut, nlut, b2v_aligned16(labels));
  return b2v_check_launch("k_label_relabel");
}

// f((const T*)image) for the label dtypes of count_regions; B2V_ERR_ARG for any other
template <class F>
static int with_label_type(const void* image, int dtype, F&& f) {
  switch (dtype) {
    case B2V_I16: return f((const int16_t*)image);
    case B2V_U8: return f((const uint8_t*)image);
    case B2V_I32: return f((const int32_t*)image);
    case B2V_I64: return f((const int64_t*)image);
  }
  B2V_REQUIRE(false, B2V_ERR_ARG, "count_regions: image must be int16, int32, int64 or uint8");
}

// sizes[0, nbins) = the histogram of image; status (device int) set where a value lies outside it. Enqueues only.
static int region_sizes(const void* image, int dtype, int64_t n, uint32_t nbins, uint32_t* sizes, int* status,
                        cudaStream_t s) {
  B2V_CUDA(cudaMemsetAsync(status, 0, sizeof(int), s));
  B2V_CUDA(cudaMemsetAsync(sizes, 0, (size_t)nbins * 4, s));
  const int rc = with_label_type(image, dtype, [&](auto img) {
    using T = std::remove_const_t<std::remove_pointer_t<decltype(img)>>;
    k_region_sizes<T><<<b2v_grid(n, 256 * 8, 16), 256, 0, s>>>(img, n, nbins, sizes, status);
    return b2v_check_launch("k_region_sizes");
  });
  return rc;
}

static int range_status(const int* status, cudaStream_t s) {
  int st = 0;
  B2V_CUDA(cudaMemcpyAsync(&st, status, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(st == 0, B2V_ERR_RANGE, "count_regions: a value lies outside [0, number_regions] (the reference panics here)");
  return B2V_OK;
}

extern "C" int b2v_region_sizes(const void* image, int dtype, int64_t n, uint32_t number_regions, uint32_t* sizes,
                                void* workspace, void* stream) {
  B2V_REQUIRE(image && sizes && workspace && n > 0, B2V_ERR_ARG, "region_sizes: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if ((rc = region_sizes(image, dtype, n, number_regions + 1, sizes, (int*)workspace, s))) return rc;
  return range_status((const int*)workspace, s);
}

extern "C" int b2v_count_regions(const void* image, int dtype, int64_t n, uint32_t number_regions, uint32_t* out,
                                 void* workspace, void* stream) {
  B2V_REQUIRE(image && out && workspace && n > 0, B2V_ERR_ARG, "count_regions: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const uint32_t nbins = number_regions + 1;
  int* status = (int*)workspace;
  uint32_t* counts = (uint32_t*)((char*)workspace + 256);
  int rc;
  if ((rc = region_sizes(image, dtype, n, nbins, counts, status, s))) return rc;
  rc = with_label_type(image, dtype, [&](auto img) {
    using T = std::remove_const_t<std::remove_pointer_t<decltype(img)>>;
    k_count_gather<T><<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>(img, n, nbins, counts, out);
    return b2v_check_launch("k_count_gather");
  });
  if (rc) return rc;
  return range_status(status, s);
}

static int tiny_check(const void* in, const uint32_t* sizes, int64_t nsizes, const void* out) {
  B2V_REQUIRE(in && out && (sizes || !nsizes), B2V_ERR_ARG, "tiny_objects: null pointer");
  B2V_REQUIRE(nsizes >= 0 && nsizes <= (1ll << 32), B2V_ERR_ARG, "tiny_objects: the size table holds 0 .. 2^32 entries");
  return B2V_OK;
}

extern "C" int b2v_tiny_objects_preview(const uint32_t* labels, int64_t n, const uint32_t* sizes, int64_t nsizes,
                                        int64_t min_size, uint8_t* out, void* stream) {
  int rc;
  if ((rc = tiny_check(labels, sizes, nsizes, out))) return rc;
  B2V_REQUIRE(n >= 0, B2V_ERR_ARG, "tiny_objects_preview: negative voxel count");
  if (!n) return B2V_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const bool vec = b2v_aligned16(labels) && ((uintptr_t)out & 3u) == 0;
  k_tiny_preview<<<b2v_grid(n, 256 * 16, 16), 256, 0, s>>>(TinyRegion{labels, sizes, nsizes, min_size}, n, out, vec);
  return b2v_check_launch("k_tiny_preview");
}

template <class Sel>
static int mark_body(Sel sel, int64_t dz, int64_t dy, int64_t dx, uint8_t* mask, cudaStream_t s) {
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0, B2V_ERR_ARG, "tiny_objects: negative body shape");
  const int64_t nrows = dz * dy;
  if (!nrows || !dx) return B2V_OK;
  k_mark_body<<<b2v_grid(nrows, 1, 16), 256, 0, s>>>(sel, dy, dx, nrows, mask);
  return b2v_check_launch("k_mark_body");
}

extern "C" int b2v_tiny_objects_remove(const uint32_t* labels, int64_t dz, int64_t dy, int64_t dx, const uint32_t* sizes,
                                       int64_t nsizes, int64_t min_size, uint8_t* mask, void* stream) {
  int rc;
  if ((rc = tiny_check(labels, sizes, nsizes, mask))) return rc;
  return mark_body(TinyRegion{labels, sizes, nsizes, min_size}, dz, dy, dx, mask, (cudaStream_t)stream);
}

extern "C" int b2v_tiny_objects_apply_preview(const uint8_t* preview, int64_t dz, int64_t dy, int64_t dx, uint8_t* mask,
                                              void* stream) {
  int rc;
  if ((rc = tiny_check(preview, nullptr, 0, mask))) return rc;
  return mark_body(PreviewSet{preview}, dz, dy, dx, mask, (cudaStream_t)stream);
}
