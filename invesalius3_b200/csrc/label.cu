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
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int k = 0; k < 8; ++k) t += s[k];
    bsum[blockIdx.x] = t;
  }
}

// exclusive scan of the block sums by one block; total -> bsum[nb]
__global__ void __launch_bounds__(1024) k_label_scan_bsums(uint32_t* bsum, long long nb) {
  __shared__ uint32_t s_w[32];
  __shared__ uint32_t s_carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (long long b0 = 0; b0 < nb; b0 += 1024) {
    const long long i = b0 + tid;
    const uint32_t v = i < nb ? bsum[i] : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_w[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += u;
      }
      s_w[lane] = w;
    }
    __syncthreads();
    const uint32_t before = s_carry + (warp ? s_w[warp - 1] : 0u) + incl - v;
    if (i < nb) bsum[i] = before;
    __syncthreads();
    if (tid == 1023) s_carry = before + v;
    __syncthreads();
  }
  if (tid == 0) bsum[nb] = s_carry;
}

// roots get their number (rank in raster order + 1), stored in parent[] (no longer needed as a forest)
__global__ void __launch_bounds__(256) k_label_number_roots(int* parent, LDims d, const uint32_t* __restrict__ bsum,
                                                            const uint32_t* __restrict__ labels) {
  __shared__ uint32_t s[8];
  const long long base = (long long)blockIdx.x * kScanBlock;
  uint32_t flags = 0, c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long long i = base + threadIdx.x * 8 + k;
    if (i < d.n && labels[i] == (uint32_t)i) { flags |= 1u << k; ++c; }
  }
  uint32_t incl = c;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s[warp] = incl;
  __syncthreads();
  uint32_t before = bsum[blockIdx.x] + incl - c;
  for (int k = 0; k < warp; ++k) before += s[k];
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

// count_regions (count_regions.rs:5-18): out[p] = number of voxels that carry image[p]'s value
template <typename T>
__global__ void __launch_bounds__(256) k_count_hist(const T* __restrict__ img, long long n, uint32_t nbins, uint32_t* counts,
                                                    int* status) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long v = (long long)img[i];
    if (v < 0 || v >= (long long)nbins) { *status = 1; continue; }
    atomicAdd(&counts[v], 1u);
  }
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

}  // namespace

extern "C" int64_t b2v_label_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return align256(n * 4) + align256((ceil_div64(n, kScanBlock) + 1) * 4) + 256;
}

extern "C" int b2v_label(const uint8_t* input, int64_t nz, int64_t ny, int64_t nx, const uint8_t* strct_host, int64_t odz,
                         int64_t ody, int64_t odx, uint32_t* labels, void* workspace, void* stream, int64_t* nlabels_host) {
  B2V_REQUIRE(input && labels && workspace && nlabels_host && strct_host, B2V_ERR_ARG, "label: null pointer");
  B2V_REQUIRE(nz > 0 && ny > 0 && nx > 0 && nz * ny * nx < (1ll << 31), B2V_ERR_ARG, "label: empty volume or more than 2^31 voxels");
  B2V_REQUIRE(odz >= 1 && ody >= 1 && odx >= 1 && odz <= 3 && ody <= 3 && odx <= 3 && (odz & 1) && (ody & 1) && (odx & 1),
              B2V_ERR_ARG, "label: the structuring element must be 1 or 3 wide on every axis");
  uint32_t sb = 0;
  for (int64_t kk = 0; kk < odz; ++kk)
    for (int64_t jj = 0; jj < ody; ++jj)
      for (int64_t ii = 0; ii < odx; ++ii)
        if (strct_host[(kk * ody + jj) * odx + ii]) {
          const int oz = (int)(kk - odz / 2), oy = (int)(jj - ody / 2), ox = (int)(ii - odx / 2);
          sb |= 1u << ((oz + 1) * 9 + (oy + 1) * 3 + (ox + 1));
        }
  for (int o = 0; o < 13; ++o)     // SciPy: "structuring element is not symmetric"
    B2V_REQUIRE(((sb >> o) & 1u) == ((sb >> (26 - o)) & 1u), B2V_ERR_ARG, "label: structuring element is not symmetric");
  cudaStream_t s = (cudaStream_t)stream;
  LDims d = {(int)nz, (int)ny, (int)nx, nz * ny * nx};
  int* parent = (int*)workspace;
  uint32_t* bsum = (uint32_t*)((char*)workspace + align256(d.n * 4));
  const long long nb = ceil_div64(d.n, kScanBlock);
  int rc;
  k_label_init<<<b2v_grid(d.n, 256 * 4, 16), 256, 0, s>>>(input, d, parent);
  if ((rc = b2v_check_launch("k_label_init"))) return rc;
  k_label_merge<<<b2v_grid(d.n, 256 * 4, 16), 256, 0, s>>>(input, d, sb, parent);
  if ((rc = b2v_check_launch("k_label_merge"))) return rc;
  k_label_flatten_count<<<(unsigned)nb, 256, 0, s>>>(parent, d, labels, bsum);
  if ((rc = b2v_check_launch("k_label_flatten_count"))) return rc;
  k_label_scan_bsums<<<1, 1024, 0, s>>>(bsum, nb);
  if ((rc = b2v_check_launch("k_label_scan_bsums"))) return rc;
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

extern "C" int b2v_count_regions(const void* image, int dtype, int64_t n, uint32_t number_regions, uint32_t* out,
                                 void* workspace, void* stream) {
  B2V_REQUIRE(image && out && workspace && n > 0, B2V_ERR_ARG, "count_regions: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const uint32_t nbins = number_regions + 1;
  int* status = (int*)workspace;
  uint32_t* counts = (uint32_t*)((char*)workspace + 256);
  B2V_CUDA(cudaMemsetAsync(workspace, 0, 256 + (size_t)nbins * 4, s));
  int rc;
  if (dtype == B2V_I16) {
    k_count_hist<int16_t><<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>((const int16_t*)image, n, nbins, counts, status);
    if ((rc = b2v_check_launch("k_count_hist"))) return rc;
    k_count_gather<int16_t><<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>((const int16_t*)image, n, nbins, counts, out);
  } else if (dtype == B2V_U8) {
    k_count_hist<uint8_t><<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>((const uint8_t*)image, n, nbins, counts, status);
    if ((rc = b2v_check_launch("k_count_hist"))) return rc;
    k_count_gather<uint8_t><<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>((const uint8_t*)image, n, nbins, counts, out);
  } else {
    B2V_REQUIRE(false, B2V_ERR_ARG, "count_regions: image must be int16 or uint8");
  }
  if ((rc = b2v_check_launch("k_count_gather"))) return rc;
  int st = 0;
  B2V_CUDA(cudaMemcpyAsync(&st, status, sizeof(int), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(st == 0, B2V_ERR_RANGE, "count_regions: a value lies outside [0, number_regions] (the reference panics here)");
  return B2V_OK;
}
