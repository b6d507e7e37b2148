// The porous-scaffold "Voronoi" generator (plugins/porous_creation/schwarzp.py:37-84):
//   b2v_jump_flooding            invesalius_rs.jump_flooding (floodfill_py.rs:262-276 -> floodfill.rs:298-507)
//   b2v_voronoi_borders          mag > 0 of np.gradient(map_owners) (schwarzp.py:43-49, 75-81)
//   b2v_image_normalize_f32_i16  imagedata_utils.image_normalize(float32 image, min_, max_) into int16
//                                (imagedata_utils.py:580-587; porous_creation/gui.py:28, 237)
// The float32 gaussian_filter between the last two is b2v_correlate1d (filters.cu).
//
// Jump flooding, bit-exact against the crate:
//   seeding        k_sites_mark / k_sites_claim / k_sites_write: the last site naming a voxel wins (an atomicMax of
//                  the site index in a scratch word per named voxel), whatever the voxel held before.
//   k_jfa_step     one Jacobi step: every voxel visits its 26 neighbours at the per-axis offsets in the crate's
//                  (zi, yi, xi) order, reading only their owners; distances are float32
//                  sqrt((dz dz + dy dy) + dx dx) from the owner's site, no FMA (the library builds with
//                  -fmad=false), correctly rounded sqrtf. An axis whose offset is 0 visits the voxel itself, as the
//                  crate does. A block is 32 x 8 voxels, so a warp is 32 consecutive x of one row and every gather
//                  of a warp reads one contiguous 128-byte span.
//   normalize      k_norm_sums: per-site voxel count and integer coordinate sums (exact in any order);
//                  k_norm_centroids: truncating int64 quotients; k_norm_max: per-site maximum distance to the
//                  centroid (atomicMax on the float bits, exact: distances are >= 0); k_norm_apply: d / max.
//                  The per-site atomics are aggregated per warp over the lanes that share an owner.
#include <math.h>

#include "b2v_common.cuh"

namespace {

constexpr int kBx = 32, kBy = 8;

struct Dims {
  int nz, ny, nx;
};

__device__ __forceinline__ int64_t vox(const Dims& d, int z, int y, int x) {
  return ((int64_t)z * d.ny + y) * d.nx + x;
}

// site i of the int32 [n][3] (z, y, x) table -> its voxel, or -1 when a coordinate is negative or out of range
__device__ __forceinline__ int64_t site_voxel(const int32_t* sites, int64_t i, const Dims& d) {
  const int z = sites[3 * i], y = sites[3 * i + 1], x = sites[3 * i + 2];
  if (z < 0 || y < 0 || x < 0 || z >= d.nz || y >= d.ny || x >= d.nx) return -1;
  return vox(d, z, y, x);
}

// float (z, y, x) of every site for the steps; a named voxel's scratch word starts below every site index
__global__ void __launch_bounds__(256) k_sites_mark(const int32_t* __restrict__ sites, int64_t n, Dims d,
                                                    float4* __restrict__ site_f, int32_t* scratch) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  site_f[i] = make_float4((float)sites[3 * i], (float)sites[3 * i + 1], (float)sites[3 * i + 2], 0.f);
  const int64_t v = site_voxel(sites, i, d);
  if (v >= 0) scratch[v] = -1;
}

__global__ void __launch_bounds__(256) k_sites_claim(const int32_t* __restrict__ sites, int64_t n, Dims d,
                                                     int32_t* scratch) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t v = site_voxel(sites, i, d);
  if (v >= 0) atomicMax(&scratch[v], (int32_t)i);
}

__global__ void __launch_bounds__(256) k_sites_write(const int32_t* __restrict__ sites, int64_t n, Dims d,
                                                     const int32_t* __restrict__ scratch, int32_t* owners,
                                                     float* dist) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t v = site_voxel(sites, i, d);
  if (v >= 0 && scratch[v] == (int32_t)i) {
    owners[v] = (int32_t)i + 1;
    dist[v] = 0.f;
  }
}

__device__ __forceinline__ float site_dist(float fz, float fy, float fx, float4 s) {
  const float dz = fz - s.x, dy = fy - s.y, dx = fx - s.z;
  return sqrtf(dz * dz + dy * dy + dx * dx);
}

__global__ void __launch_bounds__(kBx* kBy) k_jfa_step(const int32_t* __restrict__ own_in,
                                                       const float* __restrict__ dist_in, int32_t* __restrict__ own_out,
                                                       float* __restrict__ dist_out, Dims d, int oz, int oy, int ox,
                                                       const float4* __restrict__ site_f, int n_sites) {
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= d.nx || y >= d.ny) return;
  const float fy = (float)y, fx = (float)x;
  for (int z = blockIdx.z; z < d.nz; z += gridDim.z) {
    const int64_t v = vox(d, z, y, x);
    const float fz = (float)z;
    int idx0 = own_in[v];
    float best = dist_in[v];
    int last = 0;        // neighbours mostly share an owner: reuse the distance computed for the previous one
    float last_d = 0.f;
    for (int zi = -1; zi <= 1; ++zi) {
      const int sz = z + zi * oz;
      if (sz < 0 || sz >= d.nz) continue;
      for (int yi = -1; yi <= 1; ++yi) {
        const int sy = y + yi * oy;
        if (sy < 0 || sy >= d.ny) continue;
        const int64_t row = ((int64_t)sz * d.ny + sy) * d.nx;
        for (int xi = -1; xi <= 1; ++xi) {
          if (xi == 0 && yi == 0 && zi == 0) continue;
          const int sx = x + xi * ox;
          if (sx < 0 || sx >= d.nx) continue;
          const int idx1 = own_in[row + sx];
          if (idx1 <= 0 || idx1 > n_sites) continue;
          if (idx1 != last) {
            last = idx1;
            last_d = site_dist(fz, fy, fx, site_f[idx1 - 1]);
          }
          if (idx0 <= 0 || last_d < best) {   // an unowned voxel takes the first valid neighbour
            idx0 = idx1;
            best = last_d;
          }
        }
      }
    }
    own_out[v] = idx0;
    dist_out[v] = best;
  }
}

// ---- normalize: warp-aggregated per-site reductions ---------------------------------------------------------------
// A warp is one row segment (fixed z and y, x = x0 .. x0 + 31), so lanes that share an owner differ only in x.
struct NormWs {
  uint32_t* count;
  unsigned long long* sum;   // [3][n]: z, y, x
  uint32_t* max_bits;
  float4* centroid;
};

__device__ __forceinline__ int owner_key(const int32_t* own, int64_t v, bool in, int n_sites) {
  if (!in) return 0;
  const int o = own[v];
  return (o > 0 && o <= n_sites) ? o : 0;
}

__global__ void __launch_bounds__(kBx* kBy) k_norm_sums(const int32_t* __restrict__ own, Dims d, int n_sites,
                                                        NormWs w) {
  const int x0 = blockIdx.x * kBx, x = x0 + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (y >= d.ny) return;   // whole warps
  const bool in = x < d.nx;
  for (int z = blockIdx.z; z < d.nz; z += gridDim.z) {
    const int key = owner_key(own, in ? vox(d, z, y, x) : 0, in, n_sites);
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key == 0) continue;
    const unsigned cnt = __popc(peers);
    const unsigned rx = __reduce_add_sync(peers, (unsigned)(x - x0));
    if ((int)threadIdx.x == __ffs(peers) - 1) {
      const int i = key - 1;
      atomicAdd(&w.count[i], cnt);
      atomicAdd(&w.sum[i], (unsigned long long)cnt * (unsigned)z);
      atomicAdd(&w.sum[n_sites + i], (unsigned long long)cnt * (unsigned)y);
      atomicAdd(&w.sum[2 * n_sites + i], (unsigned long long)cnt * (unsigned)x0 + rx);
    }
  }
}

__global__ void __launch_bounds__(256) k_norm_centroids(int n_sites, NormWs w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_sites) return;
  const unsigned long long c = w.count[i];
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c > 0)   // the sums are >= 0: unsigned division truncates like the crate's i64 quotient
    s = make_float4((float)(int32_t)(w.sum[i] / c), (float)(int32_t)(w.sum[n_sites + i] / c),
                    (float)(int32_t)(w.sum[2 * n_sites + i] / c), 0.f);
  w.centroid[i] = s;
}

__global__ void __launch_bounds__(kBx* kBy) k_norm_max(const int32_t* __restrict__ own, Dims d, int n_sites, NormWs w) {
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (y >= d.ny) return;
  const bool in = x < d.nx;
  for (int z = blockIdx.z; z < d.nz; z += gridDim.z) {
    const int key = owner_key(own, in ? vox(d, z, y, x) : 0, in, n_sites);
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key == 0) continue;
    const float dd = site_dist((float)z, (float)y, (float)x, w.centroid[key - 1]);
    const unsigned m = __reduce_max_sync(peers, __float_as_uint(dd));   // >= 0: the bits order like the values
    if ((int)threadIdx.x == __ffs(peers) - 1) atomicMax(&w.max_bits[key - 1], m);
  }
}

__global__ void __launch_bounds__(kBx* kBy) k_norm_apply(const int32_t* __restrict__ own, float* __restrict__ dist,
                                                         Dims d, int n_sites, NormWs w) {
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= d.nx || y >= d.ny) return;
  for (int z = blockIdx.z; z < d.nz; z += gridDim.z) {
    const int64_t v = vox(d, z, y, x);
    const int key = owner_key(own, v, true, n_sites);
    if (key == 0) continue;   // unowned, or owned beyond the site table: the distance stays
    float dd = site_dist((float)z, (float)y, (float)x, w.centroid[key - 1]);
    const float m = __uint_as_float(w.max_bits[key - 1]);
    if (m > 0.f) dd = dd / m;
    dist[v] = dd;
  }
}

// ---- scaffold borders ---------------------------------------------------------------------------------------------
// np.gradient along one axis is non-zero exactly where the integer difference is: central in the interior,
// one-sided at the two ends (n >= 2).
__device__ __forceinline__ bool grad_nonzero(const int32_t* __restrict__ own, int64_t v, int i, int n, int64_t step) {
  if (i == 0) return own[v + step] != own[v];
  if (i == n - 1) return own[v] != own[v - step];
  return own[v + step] != own[v - step];
}

__global__ void __launch_bounds__(kBx* kBy) k_voronoi_borders(const int32_t* __restrict__ own, Dims d, int planar,
                                                              float* __restrict__ out) {
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= d.nx || y >= d.ny) return;
  const int64_t plane = (int64_t)d.ny * d.nx;
  for (int z = blockIdx.z; z < d.nz; z += gridDim.z) {
    const int64_t v = vox(d, z, y, x);
    const bool b = (!planar && grad_nonzero(own, v, z, d.nz, plane)) || grad_nonzero(own, v, y, d.ny, d.nx) ||
                   grad_nonzero(own, v, x, d.nx, 1);
    out[v] = b ? 1.f : 0.f;
  }
}

// ---- image_normalize ----------------------------------------------------------------------------------------------
// float32 throughout, as NumPy evaluates (image - imin) * (span / (imax - imin)) + min_ on a float32 image with
// Python-scalar bounds (normalize_i16; the float64 form is in porous.cu).
__global__ void __launch_bounds__(256) k_image_normalize(const float* __restrict__ in, int64_t n, float imin, float imax,
                                                         float span, float min_f, int16_t fill,
                                                         int16_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const bool flat = imin == imax;
  const float scale = span / (imax - imin);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = flat ? fill : normalize_i16<float>(in[i], imin, scale, min_f);
}

struct Layout {
  int64_t own_b, dist_b, site_f, count, sum, max_bits, centroid, total;
};

Layout layout(int64_t nvox, int64_t n) {
  Layout L;
  L.own_b = 0;
  L.dist_b = L.own_b + align256(4 * nvox);
  L.site_f = L.dist_b + align256(4 * nvox);
  L.count = L.site_f + align256(16 * n);
  L.sum = L.count + align256(4 * n);
  L.max_bits = L.sum + align256(24 * n);
  L.centroid = L.max_bits + align256(4 * n);
  L.total = L.centroid + align256(16 * n);
  return L;
}

dim3 vol_grid(const Dims& d) {
  return dim3((unsigned)ceil_div64(d.nx, kBx), (unsigned)ceil_div64(d.ny, kBy), (unsigned)(d.nz < 65535 ? d.nz : 65535));
}

bool dims_ok(int64_t dz, int64_t dy, int64_t dx) {
  return dz > 0 && dy > 0 && dx > 0 && dz < (1ll << 31) && dx < (1ll << 31) && ceil_div64(dy, kBy) <= 65535 &&
         ceil_div64(dx, kBx) < (1ll << 31);
}

}  // namespace

extern "C" int64_t b2v_jump_flooding_workspace_bytes(int64_t dz, int64_t dy, int64_t dx, int64_t n_sites) {
  if (dz <= 0 || dy <= 0 || dx <= 0 || n_sites <= 0) return 0;
  return layout(dz * dy * dx, n_sites).total;
}

extern "C" int b2v_jump_flooding(float* distance_map, int32_t* map_owners, int64_t dz, int64_t dy, int64_t dx,
                                 const int32_t* sites, int64_t n_sites, int normalize, void* workspace, void* stream) {
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0 && n_sites >= 0, B2V_ERR_ARG, "jump_flooding: negative size");
  if (n_sites == 0 || dz == 0 || dy == 0 || dx == 0) return B2V_OK;   // the crate returns untouched
  B2V_REQUIRE(distance_map && map_owners && sites && workspace, B2V_ERR_ARG, "jump_flooding: null pointer");
  B2V_REQUIRE(dims_ok(dz, dy, dx), B2V_ERR_ARG, "jump_flooding: shape (%lld, %lld, %lld) too large", (long long)dz,
              (long long)dy, (long long)dx);
  B2V_REQUIRE(n_sites < INT32_MAX, B2V_ERR_ARG, "jump_flooding: %lld sites overflow the int32 owners",
              (long long)n_sites);
  const int64_t nvox = dz * dy * dx;
  B2V_REQUIRE(!normalize || nvox <= (int64_t)UINT32_MAX, B2V_ERR_ARG,
              "jump_flooding: %lld voxels could wrap the u32 per-site counts of normalize", (long long)nvox);
  cudaStream_t s = (cudaStream_t)stream;
  const Dims d{(int)dz, (int)dy, (int)dx};
  const Layout L = layout(nvox, n_sites);
  char* ws = (char*)workspace;
  int32_t* own_b = (int32_t*)(ws + L.own_b);
  float* dist_b = (float*)(ws + L.dist_b);
  float4* site_f = (float4*)(ws + L.site_f);
  const int n = (int)n_sites;
  const unsigned sblocks = (unsigned)ceil_div64(n_sites, 256);
  int rc;

  // seeding into the caller's arrays; own_b is scratch until the first step overwrites all of it
  k_sites_mark<<<sblocks, 256, 0, s>>>(sites, n_sites, d, site_f, own_b);
  if ((rc = b2v_check_launch("k_sites_mark"))) return rc;
  k_sites_claim<<<sblocks, 256, 0, s>>>(sites, n_sites, d, own_b);
  if ((rc = b2v_check_launch("k_sites_claim"))) return rc;
  k_sites_write<<<sblocks, 256, 0, s>>>(sites, n_sites, d, own_b, map_owners, distance_map);
  if ((rc = b2v_check_launch("k_sites_write"))) return rc;

  const int64_t max_dim = dz > dy ? (dz > dx ? dz : dx) : (dy > dx ? dy : dx);
  int n_steps = 0;
  while ((max_dim >> (n_steps + 1)) > 0) ++n_steps;   // floor(log2(max_dim)); 0 when max_dim <= 1
  int oz = d.nz / 2, oy = d.ny / 2, ox = d.nx / 2;
  int32_t *own_cur = map_owners, *own_nxt = own_b;
  float *dist_cur = distance_map, *dist_nxt = dist_b;
  const dim3 grid = vol_grid(d), block(kBx, kBy);
  for (int step = 0; step < n_steps; ++step) {
    k_jfa_step<<<grid, block, 0, s>>>(own_cur, dist_cur, own_nxt, dist_nxt, d, oz, oy, ox, site_f, n);
    if ((rc = b2v_check_launch("k_jfa_step"))) return rc;
    int32_t* to = own_cur; own_cur = own_nxt; own_nxt = to;
    float* td = dist_cur; dist_cur = dist_nxt; dist_nxt = td;
    oz /= 2; oy /= 2; ox /= 2;
  }
  if (own_cur != map_owners) {   // an odd number of steps ends in the workspace
    B2V_CUDA(cudaMemcpyAsync(map_owners, own_cur, 4 * nvox, cudaMemcpyDeviceToDevice, s));
    B2V_CUDA(cudaMemcpyAsync(distance_map, dist_cur, 4 * nvox, cudaMemcpyDeviceToDevice, s));
  }
  if (!normalize) return B2V_OK;

  NormWs w;
  w.count = (uint32_t*)(ws + L.count);
  w.sum = (unsigned long long*)(ws + L.sum);
  w.max_bits = (uint32_t*)(ws + L.max_bits);
  w.centroid = (float4*)(ws + L.centroid);
  B2V_CUDA(cudaMemsetAsync(ws + L.count, 0, L.centroid - L.count, s));   // count, sum and max_bits
  k_norm_sums<<<grid, block, 0, s>>>(map_owners, d, n, w);
  if ((rc = b2v_check_launch("k_norm_sums"))) return rc;
  k_norm_centroids<<<sblocks, 256, 0, s>>>(n, w);
  if ((rc = b2v_check_launch("k_norm_centroids"))) return rc;
  k_norm_max<<<grid, block, 0, s>>>(map_owners, d, n, w);
  if ((rc = b2v_check_launch("k_norm_max"))) return rc;
  k_norm_apply<<<grid, block, 0, s>>>(map_owners, distance_map, d, n, w);
  return b2v_check_launch("k_norm_apply");
}

extern "C" int b2v_voronoi_borders(const int32_t* owners, int64_t dz, int64_t dy, int64_t dx, int planar, float* out,
                                   void* stream) {
  B2V_REQUIRE(owners && out, B2V_ERR_ARG, "voronoi_borders: null pointer");
  B2V_REQUIRE(dims_ok(dz, dy, dx), B2V_ERR_ARG, "voronoi_borders: bad shape");
  B2V_REQUIRE(planar ? dz == 1 && dy >= 2 && dx >= 2 : dz >= 2 && dy >= 2 && dx >= 2, B2V_ERR_ARG,
              "voronoi_borders: every differentiated axis needs at least 2 voxels (planar: dz == 1)");
  const Dims d{(int)dz, (int)dy, (int)dx};
  k_voronoi_borders<<<vol_grid(d), dim3(kBx, kBy), 0, (cudaStream_t)stream>>>(owners, d, planar, out);
  return b2v_check_launch("k_voronoi_borders");
}

extern "C" int b2v_image_normalize_f32_i16(const float* in, int64_t n, float imin, float imax, float span, float min_f,
                                           int16_t fill, int16_t* out, void* stream) {
  B2V_REQUIRE(n >= 0, B2V_ERR_ARG, "image_normalize: negative size");
  if (n == 0) return B2V_OK;
  B2V_REQUIRE(in && out, B2V_ERR_ARG, "image_normalize: null pointer");
  k_image_normalize<<<b2v_grid(n, 256, 16), 256, 0, (cudaStream_t)stream>>>(in, n, imin, imax, span, min_f, fill, out);
  return b2v_check_launch("k_image_normalize");
}
