// The wave traversal of a triangle mesh in VTK's processing order, shared by the surface tools that walk
// cells wave by wave (connectivity.cu: TraverseAndMark; normals.cu: TraverseAndOrder). Every name is in an
// anonymous namespace, so each translation unit has its own copy.
//
// One persistent cooperative launch (k_waves) runs every wave of every region. The appended list of wave
// L + 1 is laid out by a scan over wave L (item order, then the enumeration's own order), each unclaimed
// candidate takes the atomicMin of its positions, and a second scan compacts the winners in position order.
// That is the sequential processing order, in linear work and without a sort. A wave of at most kSmall
// items runs in block 0 alone, with block barriers, until the waves grow again.
//
// The caller supplies the neighbour enumeration E, with
//   unsigned long long count(const State&, int64_t i)   entries item i of the current wave appends
//   void each(const State&, int64_t i, F f)             calls f(d, j) for those entries in order: cell d, and
//                                                       a tag j the enumeration hands back to win
//   void win(const State&, int64_t i, int j, int32_t d) d is claimed by item i's entry tagged j
// and the buffers of WaveBufs: best [T] is kInf for every cell still to claim (a claimed cell holds a
// position below the current base), seq the cells in wave order.
#pragma once
#include <cooperative_groups.h>

#include "b2v_common.cuh"

namespace {

namespace wcg = cooperative_groups;

constexpr int kWaveBlock = 256;
constexpr int kMaxGrid = 1024;                     // blocks of the persistent launch (btot capacity)
constexpr int64_t kSmall = 2048;                   // waves this small run in one block
constexpr unsigned long long kInf = ~0ull;

struct WaveBufs {
  int32_t* seq;                // cells in wave order
  unsigned long long* best;    // [T] lowest position a cell was reached at; kInf: unclaimed
  unsigned long long* loc1;    // [items] per item: its first entry, then its first winner, within the block
  unsigned long long* loc2;
  unsigned long long* btot;    // [2 kMaxGrid]: entries per block, then winners per block
};

// one wave; every block of a team computes the same record from the per-block totals
struct State {
  long long n;        // items of the current wave
  long long cur;      // its offset in seq (a seed wave outside seq: none)
  long long base;     // first position of the wave's appended list; every earlier position is smaller
  long long depth;    // waves that marked a cell
  long long total;    // cells marked so far
  long long seed;     // 1 while the current wave is a list the enumeration reads from elsewhere
};

// ctl words: [0, 6) the starting state, [6, 12) the second hand-over record, then the results
enum { W_DEPTH = 12, W_TOTAL = 13, W_BASE = 14, W_CTL = 16 };

// sum over blocks [0, b) and [0, nb) of btot[off + .], with the block's threads; s_r: 2 shared words
__device__ __forceinline__ void block_prefix(const unsigned long long* btot, int b, int nb,
                                             unsigned long long* s_r) {
  if (threadIdx.x < 32) {
    unsigned long long pre = 0, all = 0;
    for (int k = threadIdx.x; k < nb; k += 32) {
      const unsigned long long x = ((const volatile unsigned long long*)btot)[k];
      all += x;
      if (k < b) pre += x;
    }
    for (int o = 16; o > 0; o >>= 1) {
      pre += __shfl_xor_sync(0xffffffffu, pre, o);
      all += __shfl_xor_sync(0xffffffffu, all, o);
    }
    if (threadIdx.x == 0) { s_r[0] = pre; s_r[1] = all; }
  }
  __syncthreads();
}

template <bool kGrid>
__device__ __forceinline__ void team_sync() {
  if (kGrid) wcg::this_grid().sync(); else __syncthreads();
}

template <bool kGrid, class E>
__device__ void run_wave(const E& e, const WaveBufs& B, State& st, int b, int nb) {
  __shared__ unsigned long long s_w[kWaveBlock / 32];
  __shared__ unsigned long long s_r[4];
  const int64_t chunk = ceil_div64(st.n, nb);
  const int64_t lo = (int64_t)b * chunk, hi = lo + chunk < st.n ? lo + chunk : st.n;
  // 1. entries each item appends
  unsigned long long carry = 0;
  for (int64_t t0 = lo; t0 < hi; t0 += kWaveBlock) {
    const int64_t i = t0 + threadIdx.x;
    const unsigned long long c = i < hi ? e.count(st, i) : 0ull;
    unsigned long long tot;
    const unsigned long long ex = block_exscan<unsigned long long>(c, s_w, &tot);
    if (i < hi) B.loc1[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) B.btot[b] = carry;
  team_sync<kGrid>();
  // 2. every unclaimed candidate takes the lowest of its positions
  block_prefix(B.btot, b, nb, s_r);
  const unsigned long long pre1 = s_r[0] + (unsigned long long)st.base, all1 = s_r[1];
  const unsigned long long base = (unsigned long long)st.base;
  for (int64_t i = lo + threadIdx.x; i < hi; i += kWaveBlock) {
    unsigned long long q = pre1 + B.loc1[i];
    e.each(st, i, [&](int32_t d, int) {
      if (((volatile unsigned long long*)B.best)[d] >= base) atomicMin(&B.best[d], q);
      ++q;
    });
  }
  team_sync<kGrid>();
  // 3. winners per item: the entries at their cell's lowest position
  carry = 0;
  for (int64_t t0 = lo; t0 < hi; t0 += kWaveBlock) {
    const int64_t i = t0 + threadIdx.x;
    unsigned long long c = 0;
    if (i < hi) {
      unsigned long long q = pre1 + B.loc1[i];
      e.each(st, i, [&](int32_t d, int) { c += B.best[d] == q; ++q; });
    }
    unsigned long long tot;
    const unsigned long long ex = block_exscan<unsigned long long>(c, s_w, &tot);
    if (i < hi) B.loc2[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) B.btot[kMaxGrid + b] = carry;
  team_sync<kGrid>();
  // 4. the winners, in position order, are the next wave
  block_prefix(B.btot + kMaxGrid, b, nb, s_r + 2);
  const unsigned long long pre2 = s_r[2], all2 = s_r[3];
  const long long out = st.seed ? 0 : st.cur + st.n;
  for (int64_t i = lo + threadIdx.x; i < hi; i += kWaveBlock) {
    unsigned long long q = pre1 + B.loc1[i];
    long long pos = out + (long long)(pre2 + B.loc2[i]);
    e.each(st, i, [&](int32_t d, int j) {
      if (B.best[d] == q) { B.seq[pos++] = d; e.win(st, i, j, d); }
      ++q;
    });
  }
  team_sync<kGrid>();
  st.cur = out;
  st.n = (long long)all2;
  st.base += (long long)all1 + 1;
  st.depth += all2 > 0;
  st.total += (long long)all2;
  st.seed = 0;
}

__device__ __forceinline__ void load_state(const long long* ctl, State& st) {
  const volatile long long* c = ctl;
  st.n = c[0]; st.cur = c[1]; st.base = c[2]; st.depth = c[3]; st.total = c[4]; st.seed = c[5];
}

__device__ __forceinline__ void store_state(long long* ctl, const State& st) {
  ctl[0] = st.n; ctl[1] = st.cur; ctl[2] = st.base; ctl[3] = st.depth; ctl[4] = st.total; ctl[5] = st.seed;
}

// ctl[0..5]: the starting state; ctl[6..11] and ctl[0..5] alternate as the hand-over record of each
// single-block stretch (a block may still read one record while block 0 writes the other). At the end,
// ctl[W_DEPTH], ctl[W_TOTAL] and ctl[W_BASE] hold the final depth, total and base.
template <class E>
__global__ void __launch_bounds__(kWaveBlock, 2) k_waves(E e, WaveBufs B, long long* ctl) {
  wcg::grid_group g = wcg::this_grid();
  State st;
  load_state(ctl, st);
  int flip = 1;
  while (st.n > 0) {
    if (st.n <= kSmall) {
      if (blockIdx.x == 0) {
        do run_wave<false>(e, B, st, 0, 1); while (st.n > 0 && st.n <= kSmall);
        if (threadIdx.x == 0) store_state(ctl + 6 * flip, st);
      }
      g.sync();
      load_state(ctl + 6 * flip, st);
      flip ^= 1;
      continue;
    }
    run_wave<true>(e, B, st, blockIdx.x, gridDim.x);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { ctl[W_DEPTH] = st.depth; ctl[W_TOTAL] = st.total; ctl[W_BASE] = st.base; }
}

// Runs k_waves<E> from the state in ctl[0..5] (device memory) on stream s: as many blocks as fit at once, at
// most two per SM and kMaxGrid in all. `what` names the caller in errors.
template <class E>
int launch_waves(const E& e, const WaveBufs& B, long long* ctl, cudaStream_t s, const char* what) {
  int per_sm = 0;
  B2V_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)k_waves<E>, kWaveBlock, 0));
  B2V_REQUIRE(per_sm >= 1, B2V_ERR_CUDA, "%s: the wave kernel does not fit on an SM", what);
  if (per_sm > 2) per_sm = 2;
  int grid = per_sm * b2v_sm_count();
  if (grid > kMaxGrid) grid = kMaxGrid;
  E ea = e;
  WaveBufs Ba = B;
  void* args[] = {&ea, &Ba, &ctl};
  B2V_CUDA(cudaLaunchCooperativeKernel((const void*)k_waves<E>, dim3(grid), dim3(kWaveBlock), args, 0, s));
  return b2v_check_launch("k_waves");
}

}  // namespace
