// Region growing (invesalius/data/styles.py:2991-3251) and Slice.calc_image_density (slice_.py:2284-2297).
//
//   k_lut255<T>     get_LUT_value_255(data, window, level) (imagedata_utils.py:540-552): the np.piecewise of
//                   k_ws_lut (watershed.cu) with 255 in place of `window`, in the input's dtype. Where the two
//                   conditions overlap (window <= 1) the later one (255) wins, as in np.piecewise.
//   masked moments  count, min, max, np.mean and np.std of image[selection], bit-identical to NumPy. The
//                   selection is `sel == value` or `sel > 127`, OR a clipped voxel box. Steps:
//                     k_sel_count   per-tile selected counts (a tile is 4096 voxels, 16 per thread)
//                     k_scan_sums   exclusive scan of the tile counts in place -> tile offsets; the total goes
//                                   to the host
//                     k_compact<T>  the selected voxels in raveled order, in the image's dtype
//                     k_pairwise    NumPy's pairwise summation (loops_utils.h.src) over subtrees of at most
//                                   kSub elements, one block each; min and max ride along in the first pass
//                   The host expands the recursion down to those subtrees and adds their sums up the same tree,
//                   so the order of every addition is NumPy's: pass 1 gives mean = S1 / n, pass 2 sums
//                   (v - mean)^2 and std = sqrt(S2 / n). No floating-point atomics: the result is deterministic.
#include <math.h>

#include <vector>

#include "b2v_common.cuh"
#include "scan.cuh"

namespace {

// ---- get_LUT_value_255 ----------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T lut_cast(double v) { return (T)(long long)v; }   // C cast: truncation
template <>
__device__ __forceinline__ double lut_cast<double>(double v) { return v; }

template <typename T>
__global__ void __launch_bounds__(256) k_lut255(const T* __restrict__ img, int64_t n, double lo, double hi, double c,
                                                double wm1, T* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double v = (double)img[i];
    T r;
    if (v > hi) r = (T)255;                          // condition 2, assigned after condition 1
    else if (v <= lo) r = (T)0;
    else r = lut_cast<T>(((v - c) / wm1 + 0.5) * 255.0);   // neither: the default branch
    out[i] = r;
  }
}

// ---- selection ------------------------------------------------------------------------------
constexpr int kPer = 16;                  // voxels per thread
constexpr int kThreads = 256;
constexpr int64_t kTile = kPer * kThreads;

struct SelParams {
  int64_t n, dy, dx;
  int mode, value, has_box, sel_aligned;
  int64_t z0, y0, x0, z1, y1, x1;         // inclusive, clipped
};

// bit k: voxel i0 + k is selected
__device__ __forceinline__ uint32_t sel_bits(const uint8_t* __restrict__ sel, const SelParams& P, int64_t i0) {
  if (i0 >= P.n) return 0u;
  const int cnt = P.n - i0 < kPer ? (int)(P.n - i0) : kPer;
  uint32_t bits = 0u;
  if (sel) {
    if (cnt == kPer && P.sel_aligned) {
      const uint4 v = ld_stream(reinterpret_cast<const uint4*>(sel + i0));
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < kPer; ++k) {
        const uint32_t b = (w[k >> 2] >> (8 * (k & 3))) & 0xffu;
        if (P.mode == B2V_SEL_EQ ? b == (uint32_t)P.value : b > 127u) bits |= 1u << k;
      }
    } else {
      for (int k = 0; k < cnt; ++k) {
        const uint32_t b = sel[i0 + k];
        if (P.mode == B2V_SEL_EQ ? b == (uint32_t)P.value : b > 127u) bits |= 1u << k;
      }
    }
  }
  if (P.has_box) {
    int64_t x = i0 % P.dx, r = i0 / P.dx, y = r % P.dy, z = r / P.dy;
    for (int k = 0; k < cnt; ++k) {
      if (z >= P.z0 && z <= P.z1 && y >= P.y0 && y <= P.y1 && x >= P.x0 && x <= P.x1) bits |= 1u << k;
      if (++x == P.dx) {
        x = 0;
        if (++y == P.dy) { y = 0; ++z; }
      }
    }
  }
  return bits;
}

__global__ void __launch_bounds__(kThreads) k_sel_count(const uint8_t* __restrict__ sel, const SelParams P,
                                                        long long* __restrict__ counts) {
  __shared__ int s_warp[kThreads / 32];
  const uint32_t bits = sel_bits(sel, P, (int64_t)blockIdx.x * kTile + (int64_t)threadIdx.x * kPer);
  const int total = block_sum(__popc(bits), s_warp);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_compact(const T* __restrict__ img, const uint8_t* __restrict__ sel,
                                                      const SelParams P, const int64_t* __restrict__ offsets,
                                                      T* __restrict__ vals) {
  __shared__ int s_warp[kThreads / 32];
  const int64_t i0 = (int64_t)blockIdx.x * kTile + (int64_t)threadIdx.x * kPer;
  uint32_t bits = sel_bits(sel, P, i0);
  int total;
  int64_t dst = offsets[blockIdx.x] + block_exscan<int, kThreads / 32>(__popc(bits), s_warp, &total);
  while (bits) {
    const int k = __ffs(bits) - 1;
    bits &= bits - 1;
    vals[dst++] = img[i0 + k];
  }
}

// ---- NumPy's pairwise summation -------------------------------------------------------------
// pairwise_sum(a, n): n < 8: sequential from -0.0; n <= 128: eight strided accumulators combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail in order; else split at n2 = n/2 - (n/2) % 8.
constexpr int64_t kSub = 16384;           // elements per block-evaluated subtree
constexpr int kMaxNodes = 256;            // a split never leaves fewer than 64 elements in a leaf
constexpr int kMaxDepth = 12;             // a subtree of kSub elements is at most 9 levels deep

__host__ __device__ __forceinline__ int64_t pw_split(int64_t n) {
  int64_t n2 = n / 2;
  return n2 - n2 % 8;
}
// NaN-propagating, as np.min / np.max
__host__ __device__ __forceinline__ double nan_min(double a, double b) { return (a < b || a != a) ? a : b; }
__host__ __device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

// SQ = false: the sum of the values, with min and max; SQ = true: the sum of (v - mean)^2.
template <typename T, bool SQ>
__global__ void __launch_bounds__(kThreads) k_pairwise(const T* __restrict__ vals, const int64_t* __restrict__ subs,
                                                       double mean, double* __restrict__ part) {
  __shared__ int s_len[kMaxDepth][kMaxNodes];
  __shared__ int s_first[kMaxDepth][kMaxNodes];   // index of the node's first child one level down
  __shared__ int s_off[2][kMaxNodes];
  __shared__ int s_cnt[kMaxDepth];
  __shared__ double s_val[2][kMaxNodes];
  __shared__ double s_mm[2][kThreads / 32];
  __shared__ int s_warp[kThreads / 32];
  const int tid = threadIdx.x;
  const int64_t base = subs[2 * blockIdx.x];
  const int len = (int)subs[2 * blockIdx.x + 1];
  if (tid == 0) { s_len[0][0] = len; s_off[0][0] = 0; s_cnt[0] = 1; }
  __syncthreads();
  // expand the recursion level by level; a leaf (<= 128) is carried down unchanged
  int d = 0;
  for (;;) {
    const int cnt = s_cnt[d];
    const int L = tid < cnt ? s_len[d][tid] : 0;
    const int k = tid < cnt ? (L > 128 ? 2 : 1) : 0;
    int total;
    const int first = block_exscan<int, kThreads / 32>(k, s_warp, &total);
    if (total == cnt) break;                       // uniform: nothing split, level d holds the leaves
    if (tid < cnt) {
      const int off = s_off[d & 1][tid];
      s_first[d][tid] = first;
      if (k == 2) {
        const int n2 = (int)pw_split(L);
        s_len[d + 1][first] = n2;       s_off[(d + 1) & 1][first] = off;
        s_len[d + 1][first + 1] = L - n2; s_off[(d + 1) & 1][first + 1] = off + n2;
      } else {
        s_len[d + 1][first] = L;        s_off[(d + 1) & 1][first] = off;
      }
    }
    if (tid == 0) s_cnt[d + 1] = total;
    __syncthreads();
    ++d;
  }
  // the leaves, one per thread
  const int nleaf = s_cnt[d];
  double mn = __longlong_as_double(0x7ff0000000000000LL), mx = -mn;   // +inf, -inf
  if (tid < nleaf) {
    const T* a = vals + base + s_off[d & 1][tid];
    const int L = s_len[d][tid];
    auto term = [&](int i) -> double {
      const double v = (double)a[i];
      if (!SQ) { mn = nan_min(mn, v); mx = nan_max(mx, v); }
      if (SQ) { const double e = v - mean; return e * e; }
      return v;
    };
    double res;
    if (L < 8) {
      res = -0.0;
      for (int i = 0; i < L; ++i) res += term(i);
    } else {
      double r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = term(j);
      int i = 8;
      for (; i < L - (L % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += term(i + j);
      }
      res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
      for (; i < L; ++i) res += term(i);
    }
    s_val[d & 1][tid] = res;
  }
  // and back up the tree
  for (int l = d - 1; l >= 0; --l) {
    __syncthreads();
    if (tid < s_cnt[l]) {
      const int f = s_first[l][tid];
      const double* below = s_val[(l + 1) & 1];
      s_val[l & 1][tid] = s_len[l][tid] > 128 ? below[f] + below[f + 1] : below[f];
    }
  }
  if (!SQ) {
    const int lane = tid & 31, w = tid >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = nan_min(mn, __shfl_down_sync(0xffffffffu, mn, o));
      mx = nan_max(mx, __shfl_down_sync(0xffffffffu, mx, o));
    }
    if (lane == 0) { s_mm[0][w] = mn; s_mm[1][w] = mx; }
  }
  __syncthreads();
  if (tid == 0) {
    part[blockIdx.x] = s_val[0][0];
    if (!SQ) {
      for (int w = 1; w < kThreads / 32; ++w) { mn = nan_min(mn, s_mm[0][w]); mx = nan_max(mx, s_mm[1][w]); }
      part[gridDim.x + blockIdx.x] = mn;
      part[2 * gridDim.x + blockIdx.x] = mx;
    }
  }
}

// The subtrees of the recursion over [off, off + n), left to right, and their sums added up the same tree.
void pw_plan(int64_t off, int64_t n, std::vector<int64_t>& subs) {
  if (n <= kSub) { subs.push_back(off); subs.push_back(n); return; }
  const int64_t n2 = pw_split(n);
  pw_plan(off, n2, subs);
  pw_plan(off + n2, n - n2, subs);
}
double pw_combine(int64_t n, const double* part, size_t* idx) {
  if (n <= kSub) return part[(*idx)++];
  const int64_t n2 = pw_split(n);
  const double a = pw_combine(n2, part, idx);
  const double b = pw_combine(n - n2, part, idx);
  return a + b;
}

int64_t max_subtrees(int64_t n) { return n / (kSub / 4) + 2; }   // every subtree of a split holds > kSub/2 - 8

struct MomentsLayout { int64_t offsets, vals, subs, part, total; };
MomentsLayout moments_layout(int64_t n) {
  const int64_t nt = ceil_div64(n, kTile), ms = max_subtrees(n);
  MomentsLayout L;
  L.offsets = 0;
  L.vals = align256(L.offsets + (nt + 1) * 8);
  L.subs = align256(L.vals + n * 8);
  L.part = align256(L.subs + ms * 16);
  L.total = align256(L.part + ms * 24);
  return L;
}

template <typename T>
int lut_launch(const void* img, int64_t n, double window, double level, void* out, cudaStream_t s) {
  const double c = level - 0.5, lo = level - 0.5 - (window - 1.0) / 2.0, hi = level - 0.5 + (window - 1.0) / 2.0;
  k_lut255<T><<<b2v_grid(n, 256 * 4, 16), 256, 0, s>>>((const T*)img, n, lo, hi, c, window - 1.0, (T*)out);
  return b2v_check_launch("k_lut255");
}

template <typename T>
int moments_typed(const void* img, const uint8_t* sel, const SelParams& P, int64_t count, char* ws,
                  const MomentsLayout& L, b2v_moments* st, cudaStream_t s) {
  const int64_t nt = ceil_div64(P.n, kTile);
  T* vals = (T*)(ws + L.vals);
  k_compact<T><<<(unsigned)nt, kThreads, 0, s>>>((const T*)img, sel, P, (const int64_t*)(ws + L.offsets), vals);
  int rc = b2v_check_launch("k_compact");
  if (rc) return rc;
  std::vector<int64_t> subs;
  pw_plan(0, count, subs);
  const int64_t nsub = (int64_t)subs.size() / 2;
  B2V_REQUIRE(nsub <= max_subtrees(P.n), B2V_ERR_ARG, "masked_moments: subtree bound exceeded");
  int64_t* d_subs = (int64_t*)(ws + L.subs);
  double* d_part = (double*)(ws + L.part);
  B2V_CUDA(cudaMemcpyAsync(d_subs, subs.data(), subs.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  std::vector<double> part(3 * nsub);
  k_pairwise<T, false><<<(unsigned)nsub, kThreads, 0, s>>>(vals, d_subs, 0.0, d_part);
  if ((rc = b2v_check_launch("k_pairwise"))) return rc;
  B2V_CUDA(cudaMemcpyAsync(part.data(), d_part, part.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  size_t idx = 0;
  const double mean = pw_combine(count, part.data(), &idx) / (double)count;
  double mn = part[nsub], mx = part[2 * nsub];
  for (int64_t j = 1; j < nsub; ++j) {
    mn = nan_min(mn, part[nsub + j]);
    mx = nan_max(mx, part[2 * nsub + j]);
  }
  k_pairwise<T, true><<<(unsigned)nsub, kThreads, 0, s>>>(vals, d_subs, mean, d_part);
  if ((rc = b2v_check_launch("k_pairwise"))) return rc;
  B2V_CUDA(cudaMemcpyAsync(part.data(), d_part, nsub * sizeof(double), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  idx = 0;
  const double s2 = pw_combine(count, part.data(), &idx);
  st->count = count;
  st->min = mn;
  st->max = mx;
  st->mean = mean;
  st->std = sqrt(s2 / (double)count);
  return B2V_OK;
}

}  // namespace

extern "C" int b2v_lut255(const void* img, int dtype, int64_t n, double window, double level, void* out,
                          void* stream) {
  B2V_REQUIRE(n >= 0, B2V_ERR_ARG, "lut255: negative size");
  if (n == 0) return B2V_OK;
  B2V_REQUIRE(img && out, B2V_ERR_ARG, "lut255: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  switch (dtype) {
    case B2V_I16: return lut_launch<int16_t>(img, n, window, level, out, s);
    case B2V_U8: return lut_launch<uint8_t>(img, n, window, level, out, s);
    case B2V_F64: return lut_launch<double>(img, n, window, level, out, s);
    default: break;
  }
  B2V_REQUIRE(false, B2V_ERR_ARG, "lut255: bad dtype code %d", dtype);
  return B2V_ERR_ARG;
}

extern "C" int64_t b2v_masked_moments_workspace_bytes(int64_t dz, int64_t dy, int64_t dx) {
  if (dz < 0 || dy < 0 || dx < 0) return 0;
  return moments_layout(dz * dy * dx).total;
}

extern "C" int b2v_masked_moments(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, const uint8_t* sel,
                                  int sel_mode, int sel_value, const int64_t* box_host, b2v_moments* stats_host,
                                  void* workspace, void* stream) {
  B2V_REQUIRE(stats_host, B2V_ERR_ARG, "masked_moments: null stats");
  B2V_REQUIRE(dz >= 0 && dy >= 0 && dx >= 0, B2V_ERR_ARG, "masked_moments: negative size");
  B2V_REQUIRE(dtype == B2V_I16 || dtype == B2V_U8 || dtype == B2V_F64, B2V_ERR_ARG, "masked_moments: bad dtype code %d",
              dtype);
  B2V_REQUIRE(sel_mode == B2V_SEL_EQ || sel_mode == B2V_SEL_GT127, B2V_ERR_ARG, "masked_moments: bad selection mode %d",
              sel_mode);
  stats_host->count = 0;
  stats_host->min = stats_host->max = stats_host->mean = stats_host->std = NAN;
  SelParams P;
  P.n = dz * dy * dx; P.dy = dy; P.dx = dx;
  P.mode = sel_mode; P.value = sel_value; P.has_box = 0;
  P.sel_aligned = sel && b2v_aligned16(sel);
  P.z0 = P.y0 = P.x0 = 0; P.z1 = P.y1 = P.x1 = -1;
  if (box_host) {
    P.z0 = box_host[0] > 0 ? box_host[0] : 0; P.z1 = box_host[3] < dz - 1 ? box_host[3] : dz - 1;
    P.y0 = box_host[1] > 0 ? box_host[1] : 0; P.y1 = box_host[4] < dy - 1 ? box_host[4] : dy - 1;
    P.x0 = box_host[2] > 0 ? box_host[2] : 0; P.x1 = box_host[5] < dx - 1 ? box_host[5] : dx - 1;
    P.has_box = P.z0 <= P.z1 && P.y0 <= P.y1 && P.x0 <= P.x1;
  }
  if (P.n == 0 || (!sel && !P.has_box)) return B2V_OK;
  B2V_REQUIRE(img && workspace, B2V_ERR_ARG, "masked_moments: null device pointer");
  const int64_t nt = ceil_div64(P.n, kTile);
  B2V_REQUIRE(nt <= 0x7fffffffLL, B2V_ERR_ARG, "masked_moments: volume too large");
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const MomentsLayout L = moments_layout(P.n);
  long long* offsets = (long long*)(ws + L.offsets);
  k_sel_count<<<(unsigned)nt, kThreads, 0, s>>>(sel, P, offsets);
  int rc = b2v_check_launch("k_sel_count");
  if (rc) return rc;
  k_scan_sums<long long><<<1, 1024, 0, s>>>(offsets, nt, offsets + nt);
  if ((rc = b2v_check_launch("k_scan_sums"))) return rc;
  int64_t count = 0;
  B2V_CUDA(cudaMemcpyAsync(&count, ws + L.offsets + nt * 8, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  if (count == 0) return B2V_OK;
  switch (dtype) {
    case B2V_I16: return moments_typed<int16_t>(img, sel, P, count, ws, L, stats_host, s);
    case B2V_U8: return moments_typed<uint8_t>(img, sel, P, count, ws, L, stats_host, s);
    default: return moments_typed<double>(img, sel, P, count, ws, L, stats_host, s);
  }
}
