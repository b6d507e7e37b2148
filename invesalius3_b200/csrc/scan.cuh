// Exclusive scans of integer arrays in device memory. Every name is in an anonymous namespace and every
// kernel is a template, so a translation unit that includes this header compiles only the instantiations it
// launches.
//
//   scan<T>         the device-wide exclusive scan in place: tiles of kScanTile, the tile sums, an add pass.
//   k_scan_sums<T>  one block of 1024 threads scans a row of block sums in place and writes its total.
#pragma once
#include "b2v_common.cuh"

namespace {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 4;                      // items per thread of the device-wide scan
constexpr int kScanTile = kScanThreads * kScanItems;

inline int64_t scan_blocks(int64_t n) { return ceil_div64(n > 0 ? n : 1, kScanTile); }

template <typename T>
__global__ void __launch_bounds__(kScanThreads) k_scan_tiles(T* a, int64_t n, T* sums) {
  __shared__ T s_w[kScanThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  T v[kScanItems], s = 0;
  for (int k = 0; k < kScanItems; ++k) {
    v[k] = base + k < n ? a[base + k] : (T)0;
    s += v[k];
  }
  T tot;
  T ex = block_exscan<T>(s, s_w, &tot);
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) a[base + k] = ex;
    ex += v[k];
  }
  if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

// Block b scans a[b n, (b + 1) n) in place and writes the row's total to total[b] (total may be null).
template <typename T>
__global__ void __launch_bounds__(1024) k_scan_sums(T* a, int64_t n, T* total) {
  __shared__ T s_w[32];
  a += (int64_t)blockIdx.x * n;
  T carry = 0;
  for (int64_t base = 0; base < n; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    const T x = i < n ? a[i] : (T)0;
    T tot;
    const T ex = block_exscan<T>(x, s_w, &tot);
    if (i < n) a[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0 && total) total[blockIdx.x] = carry;
}

template <typename T>
__global__ void __launch_bounds__(kScanThreads) k_scan_add(T* a, int64_t n, const T* __restrict__ sums) {
  const T add = sums[blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  for (int k = threadIdx.x; k < kScanTile; k += kScanThreads)
    if (base + k < n) a[base + k] += add;
}

// scratch: scan_blocks(n) + 1 words; total (may be null): the sum of a[0, n), written on the device. T is
// deduced from a alone (decltype makes total a non-deduced parameter), so total may be nullptr.
template <typename T>
int scan(T* a, int64_t n, T* scratch, decltype(a) total, cudaStream_t s) {
  const int64_t nb = scan_blocks(n);
  B2V_REQUIRE(nb <= 0x7fffffffLL, B2V_ERR_ARG, "scan too long");
  k_scan_tiles<T><<<(unsigned)nb, kScanThreads, 0, s>>>(a, n, scratch);
  if (int rc = b2v_check_launch("k_scan_tiles")) return rc;
  k_scan_sums<T><<<1, 1024, 0, s>>>(scratch, nb, total);
  if (int rc = b2v_check_launch("k_scan_sums")) return rc;
  k_scan_add<T><<<(unsigned)nb, kScanThreads, 0, s>>>(a, n, scratch);
  return b2v_check_launch("k_scan_add");
}

}  // namespace
