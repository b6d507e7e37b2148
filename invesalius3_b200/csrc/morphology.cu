// Binary erosion and dilation with Euclidean disk / ball footprints (plugins/mask_morphology/gui.py:98-175:
// skimage.morphology.binary_erosion / binary_dilation with disk(r) per axial slice or ball(r), which are
// scipy.ndimage.binary_erosion(border_value=True) / binary_dilation(border_value=False)).
//   b2v_binary_morphology   one op, radius 0..15, planar (disk per z-slice) or volumetric (ball)
//
// Both footprints are {d : |d|^2 <= r^2}. A voxel of the dilation is set when some in-volume SOURCE voxel lies
// within the ball, the sources being the set voxels; erosion is the complement of the same test with the unset
// in-volume voxels as sources (outside the volume never counts as unset). The bounded squared distance to the
// nearest source is separable and exact in integers:
//   k_morph_xy   per z-plane tile of 64 x 64 voxels with an r halo in shared memory. The sources of a row are
//                ballot bits, so the x pass is O(1) per voxel: the nearest source within r to the left and to the
//                right of a voxel is a find-first-set on a (2r + 1)-bit window. The y pass is min over |s| <= r of
//                g1[y + s] + s^2 in byte SIMD (__vaddus4 / __vminu4), four voxels per instruction.
//   k_morph_z    the same min-plus along z on the planes k_morph_xy wrote into the workspace; each thread owns a
//                column of four voxels and stages kZC + 2r of its words in shared memory.
// Intermediates are clamped at r^2 + 1 <= 226, so they fit a byte; a saturated add only raises values that are
// already > r^2. The last pass writes set_value / 0 and counts the set voxels (warp sums, one 64-bit atomic per
// warp: the counts are exact and order-free).
#include "b2v_common.cuh"

namespace {

constexpr int kMaxR = 15;
constexpr int kTX = 64, kTY = 64;                 // k_morph_xy output tile
constexpr int kRowsMax = kTY + 2 * kMaxR;         // tile rows with the y halo
constexpr int kXyThreads = 256;
constexpr int kZThreads = 128, kZC = 32;          // k_morph_z: words per block, z outputs per block

struct Dims {
  int64_t nz;
  int ny, nx;
};

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void add_count(unsigned long long* c, unsigned long long v) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(c, v);
}

// four squared distances -> output bytes (set_value / 0) and the number of set voxels among the first n_valid
__device__ __forceinline__ uint32_t finish4(uint32_t g, uint32_t r2x4, int erode, uint32_t set4, int n_valid,
                                            unsigned long long& cnt) {
  uint32_t m = __vcmpleu4(g, r2x4);   // 0xff where a source lies within the ball
  if (erode) m = ~m;
  const uint32_t valid = n_valid >= 4 ? 0xffffffffu : (1u << (8 * n_valid)) - 1u;
  cnt += __popc(m & valid & 0x01010101u);
  return m & set4;
}

__device__ __forceinline__ void store4(uint8_t* p, uint32_t w, int n_valid, int vec) {
  if (vec && n_valid == 4) {
    *reinterpret_cast<uint32_t*>(p) = w;
  } else {
    for (int j = 0; j < n_valid; ++j) p[j] = (uint8_t)(w >> (8 * j));
  }
}

// planar: the final bytes go to out ([nz][ny][nx]); otherwise the y pass's squared distances go to the
// workspace ([nz][ny][nxp] words, nxp = nx rounded up to 4).
__global__ void __launch_bounds__(kXyThreads) k_morph_xy(const uint8_t* __restrict__ in, Dims d, uint8_t thr, int erode,
                                                         int r, int planar, uint8_t set_value, uint8_t* __restrict__ out,
                                                         int out_vec, uint8_t* __restrict__ ws, int64_t nxp,
                                                         unsigned long long* counts) {
  __shared__ uint32_t bits[kRowsMax][3];
  __shared__ __align__(16) uint8_t g1[kRowsMax][kTX];
  const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = kTY + 2 * r, width = kTX + 2 * r;
  const uint32_t sent = (uint32_t)(r * r + 1), sent4 = sent * 0x01010101u, r2x4 = (uint32_t)(r * r) * 0x01010101u;
  const uint32_t set4 = set_value * 0x01010101u;
  unsigned long long cnt_in = 0, cnt_out = 0;
  for (int64_t z = blockIdx.z; z < d.nz; z += gridDim.z) {
    const uint8_t* plane = in + z * d.ny * d.nx;
    // sources of the tile and its halo as bits: word k of a row holds columns x0 - r + 32 k .. + 31
    for (int row = warp; row < rows; row += kXyThreads / 32) {
      const int y = y0 - r + row;
      const bool yin = y >= 0 && y < d.ny;
      const bool centre_row = row >= r && row < r + kTY;
      for (int k = 0; k < 3; ++k) {
        const int c = 32 * k + lane, x = x0 - r + c;
        bool src = false;
        if (yin && c < width && x >= 0 && x < d.nx) {
          const bool set = plane[(int64_t)y * d.nx + x] > thr;
          if (centre_row && c >= r && c < r + kTX) cnt_in += set;
          src = set != (bool)erode;
        }
        const uint32_t b = __ballot_sync(0xffffffffu, src);
        if (lane == 0) bits[row][k] = b;
      }
    }
    __syncthreads();
    // x pass: g1 = t^2 of the nearest source in the row with |t| <= r, else r^2 + 1
    for (int i = threadIdx.x; i < rows * kTX; i += kXyThreads) {
      const int row = i / kTX, x = i % kTX, w = x >> 5;
      const uint64_t pair = ((uint64_t)bits[row][w + 1] << 32) | bits[row][w];
      const uint32_t win = (uint32_t)(pair >> (x & 31)) & ((2u << (2 * r)) - 1u);   // columns x - r .. x + r
      const uint32_t right = win >> r, left = win & ((2u << r) - 1u);              // bit 0 / bit r: the voxel
      int dist = r + 1;
      if (right) dist = __ffs(right) - 1;
      if (left) dist = min(dist, r - (31 - __clz(left)));
      g1[row][x] = (uint8_t)(dist <= r ? dist * dist : sent);
    }
    __syncthreads();
    // y pass, four voxels per thread and step
    for (int i = threadIdx.x; i < kTY * (kTX / 4); i += kXyThreads) {
      const int yy = i / (kTX / 4), xw = i % (kTX / 4);
      const int y = y0 + yy, x = x0 + 4 * xw;
      if (y >= d.ny || x >= d.nx) continue;
      uint32_t acc = sent4;
      for (int s = -r; s <= r; ++s) {
        const uint32_t v = *reinterpret_cast<const uint32_t*>(&g1[yy + r + s][4 * xw]);
        acc = __vminu4(acc, __vaddus4(v, (uint32_t)(s * s) * 0x01010101u));
      }
      acc = __vminu4(acc, sent4);
      if (planar) {
        const int n_valid = min(4, d.nx - x);
        store4(out + (z * d.ny + y) * d.nx + x, finish4(acc, r2x4, erode, set4, n_valid, cnt_out), n_valid, out_vec);
      } else {
        *reinterpret_cast<uint32_t*>(ws + (z * d.ny + y) * nxp + x) = acc;
      }
    }
    __syncthreads();   // the next plane reuses the shared tile
  }
  add_count(&counts[0], cnt_in);
  if (planar) add_count(&counts[1], cnt_out);
}

// z pass over the workspace words: thread i of the plane owns word i (row y, columns 4 xw .. 4 xw + 3)
__global__ void __launch_bounds__(kZThreads) k_morph_z(const uint32_t* __restrict__ ws, Dims d, int64_t qrow, int r,
                                                       int erode, uint8_t set_value, uint8_t* __restrict__ out,
                                                       int out_vec, unsigned long long* counts) {
  extern __shared__ uint32_t col[];   // [kZC + 2r][kZThreads], each thread reads only its own column
  const int64_t q = (int64_t)d.ny * qrow;
  const int64_t i = (int64_t)blockIdx.x * kZThreads + threadIdx.x;
  const bool active = i < q;
  const int y = active ? (int)(i / qrow) : 0;
  const int x = active ? (int)(i % qrow) * 4 : 0;
  const int n_valid = active ? min(4, d.nx - x) : 0;   // padding words (x >= nx) write and count nothing
  const uint32_t sent4 = (uint32_t)(r * r + 1) * 0x01010101u, r2x4 = (uint32_t)(r * r) * 0x01010101u;
  const uint32_t set4 = set_value * 0x01010101u;
  uint32_t* mine = col + threadIdx.x;
  unsigned long long cnt = 0;
  for (int64_t z0 = (int64_t)blockIdx.y * kZC; z0 < d.nz; z0 += (int64_t)gridDim.y * kZC) {
    for (int k = 0; k < kZC + 2 * r; ++k) {
      const int64_t z = z0 - r + k;
      mine[k * kZThreads] = (active && z >= 0 && z < d.nz) ? ws[z * q + i] : sent4;
    }
    if (n_valid > 0) {
      for (int zz = 0; zz < kZC && z0 + zz < d.nz; ++zz) {
        uint32_t acc = sent4;
        for (int u = -r; u <= r; ++u)
          acc = __vminu4(acc, __vaddus4(mine[(zz + r + u) * kZThreads], (uint32_t)(u * u) * 0x01010101u));
        const uint32_t w = finish4(acc, r2x4, erode, set4, n_valid, cnt);
        store4(out + ((z0 + zz) * d.ny + y) * d.nx + x, w, n_valid, out_vec);
      }
    }
  }
  add_count(&counts[1], cnt);
}

int64_t padded_row(int64_t dx) { return (dx + 3) & ~(int64_t)3; }

bool dims_ok(int64_t dz, int64_t dy, int64_t dx) {
  return dz > 0 && dy > 0 && dx > 0 && dy < (1ll << 31) - 3 && dx < (1ll << 31) - 3 &&
         ceil_div64(dy, kTY) <= 65535 && ceil_div64(dy * padded_row(dx) / 4, kZThreads) < (1ll << 31);
}

}  // namespace

extern "C" int64_t b2v_binary_morphology_workspace_bytes(int64_t dz, int64_t dy, int64_t dx, int planar) {
  if (planar || dz <= 0 || dy <= 0 || dx <= 0) return 0;
  return dz * dy * padded_row(dx);
}

extern "C" int b2v_binary_morphology(const uint8_t* in, int64_t dz, int64_t dy, int64_t dx, uint8_t threshold, int op,
                                     int radius, int planar, uint8_t set_value, uint8_t* out, int64_t* counts,
                                     void* workspace, void* stream) {
  B2V_REQUIRE(op == B2V_MORPH_ERODE || op == B2V_MORPH_DILATE, B2V_ERR_ARG, "binary_morphology: bad op %d", op);
  B2V_REQUIRE(radius >= 0 && radius <= kMaxR, B2V_ERR_ARG, "binary_morphology: radius %d outside 0..%d", radius,
              kMaxR);
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0, B2V_ERR_ARG, "binary_morphology: negative size");
  B2V_REQUIRE(counts, B2V_ERR_ARG, "binary_morphology: null counts");
  cudaStream_t s = (cudaStream_t)stream;
  B2V_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), s));
  if (dz == 0 || dy == 0 || dx == 0) return B2V_OK;
  B2V_REQUIRE(in && out && (planar || workspace), B2V_ERR_ARG, "binary_morphology: null pointer");
  B2V_REQUIRE(dims_ok(dz, dy, dx), B2V_ERR_ARG, "binary_morphology: shape (%lld, %lld, %lld) too large",
              (long long)dz, (long long)dy, (long long)dx);
  const Dims d{dz, (int)dy, (int)dx};
  const int erode = op == B2V_MORPH_ERODE;
  const int out_vec = (dx % 4 == 0) && (reinterpret_cast<uintptr_t>(out) % 4 == 0);
  const int64_t nxp = padded_row(dx);
  unsigned long long* c = reinterpret_cast<unsigned long long*>(counts);
  const dim3 grid((unsigned)ceil_div64(dx, kTX), (unsigned)ceil_div64(dy, kTY), (unsigned)(dz < 65535 ? dz : 65535));
  k_morph_xy<<<grid, kXyThreads, 0, s>>>(in, d, threshold, erode, radius, planar, set_value, out, out_vec,
                                         (uint8_t*)workspace, nxp, c);
  int rc;
  if ((rc = b2v_check_launch("k_morph_xy"))) return rc;
  if (planar) return B2V_OK;
  const int64_t words = dy * nxp / 4;
  const int64_t zblocks = ceil_div64(dz, kZC);
  const dim3 zgrid((unsigned)ceil_div64(words, kZThreads), (unsigned)(zblocks < 65535 ? zblocks : 65535));
  const size_t smem = (size_t)(kZC + 2 * radius) * kZThreads * sizeof(uint32_t);
  k_morph_z<<<zgrid, kZThreads, smem, s>>>((const uint32_t*)workspace, d, nxp / 4, radius, erode, set_value, out,
                                           out_vec, c);
  return b2v_check_launch("k_morph_z");
}
