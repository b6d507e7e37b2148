// MaxIP / MinIP / MeanIP along axis 0, 1 or 2 of a dense [dz][dy][dx] volume.
// Reference semantics: NumPy tmp_array.max/min/mean(axis) in
// invesalius/data/slice_.py:881-886, 970-975, 1057-1062.
//   max/min keep the input dtype; mean is float64 = exact integer sum / count
//   (NumPy accumulates int16 in float64, which is exact below 2^53, so any summation
//   order gives the same bits).
// HBM-bound: 2 B/voxel read for int16, output plane is negligible.
//
// Two kernel shapes:
//   keep-x  (axis 0 and 1): the reduced axis is strided, x stays contiguous. A block is
//           32 x-vectors (128-bit, 8 voxels each) wide and 8 reduction lanes deep;
//           axis 0 treats the whole [dy*dx] plane as one flat row.
//   along-x (axis 2): one warp folds one contiguous row with packed min/max and a
//           shuffle tree.
#include "b2v_common.cuh"

namespace {

enum { KMAX = B2V_MIP_MAX, KMIN = B2V_MIP_MIN, KMEAN = B2V_MIP_MEAN };

struct Acc8 {  // eight int32 accumulators for one 128-bit vector of int16
  int v[8];
};

template <int KIND>
__device__ __forceinline__ void fold_packed(uint4& acc, const int4& a) {
  if (KIND == KMAX) {
    acc.x = max_s16x2(acc.x, a.x); acc.y = max_s16x2(acc.y, a.y);
    acc.z = max_s16x2(acc.z, a.z); acc.w = max_s16x2(acc.w, a.w);
  } else {
    acc.x = min_s16x2(acc.x, a.x); acc.y = min_s16x2(acc.y, a.y);
    acc.z = min_s16x2(acc.z, a.z); acc.w = min_s16x2(acc.w, a.w);
  }
}
__device__ __forceinline__ void add_packed(Acc8& s, const int4& a) {
  s.v[0] += (int)(int16_t)(a.x & 0xffff); s.v[1] += (int)a.x >> 16;
  s.v[2] += (int)(int16_t)(a.y & 0xffff); s.v[3] += (int)a.y >> 16;
  s.v[4] += (int)(int16_t)(a.z & 0xffff); s.v[5] += (int)a.z >> 16;
  s.v[6] += (int)(int16_t)(a.w & 0xffff); s.v[7] += (int)a.w >> 16;
}

// ---------------- keep-x, int16, vectorised -----------------------------------
// grid = (ceil(nxv/32), no, S); block = (32, 8)
// in : img[o*so + r*sr + x]  (element strides, multiples of 8)
// out: S == 1 -> final result (T or f64) at out[o*nx + x]
//      S  > 1 -> partial[s][o*nx + x] as int16 (max/min) or int64 (sum)
template <int KIND>
__global__ void __launch_bounds__(256) k_keepx_i16_vec(const int16_t* __restrict__ img, int64_t nx, int64_t nxv,
                                                       int64_t nr, int64_t so, int64_t sr, void* __restrict__ out,
                                                       void* __restrict__ partial, int64_t plane) {
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t xv = (int64_t)blockIdx.x * 32 + tx;
  const int64_t o = blockIdx.y;
  const int S = gridDim.z, s = blockIdx.z;
  const int64_t rchunk = ceil_div64(nr, S);
  const int64_t r0 = (int64_t)s * rchunk;
  const int64_t r1 = (r0 + rchunk < nr) ? r0 + rchunk : nr;
  const bool live = xv < nxv;

  uint4 acc;
  Acc8 sum;
  if (KIND == KMAX) acc = make_uint4(0x80008000u, 0x80008000u, 0x80008000u, 0x80008000u);
  if (KIND == KMIN) acc = make_uint4(0x7fff7fffu, 0x7fff7fffu, 0x7fff7fffu, 0x7fff7fffu);
  if (KIND == KMEAN) {
#pragma unroll
    for (int i = 0; i < 8; ++i) sum.v[i] = 0;
  }
  if (live) {
    const int16_t* p = img + o * so + xv * 8;
    int64_t r = r0 + ty;
    for (; r + 24 < r1; r += 32) {
      int4 a = ld_stream((const int4*)(p + r * sr));
      int4 b = ld_stream((const int4*)(p + (r + 8) * sr));
      int4 c = ld_stream((const int4*)(p + (r + 16) * sr));
      int4 d = ld_stream((const int4*)(p + (r + 24) * sr));
      if (KIND == KMEAN) {
        add_packed(sum, a); add_packed(sum, b); add_packed(sum, c); add_packed(sum, d);
      } else {
        fold_packed<KIND>(acc, a); fold_packed<KIND>(acc, b); fold_packed<KIND>(acc, c); fold_packed<KIND>(acc, d);
      }
    }
    for (; r < r1; r += 8) {
      int4 a = ld_stream((const int4*)(p + r * sr));
      if (KIND == KMEAN) add_packed(sum, a); else fold_packed<KIND>(acc, a);
    }
  }
  // fold the 8 reduction lanes through shared memory
  if (KIND == KMEAN) {
    __shared__ int ssum[8][32][9];
#pragma unroll
    for (int i = 0; i < 8; ++i) ssum[ty][tx][i] = sum.v[i];
    __syncthreads();
    if (ty == 0 && live) {
      long long tot[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        long long t = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += ssum[j][tx][i];
        tot[i] = t;
      }
      int64_t base = o * nx + xv * 8;
      if (S == 1) {
        double* dst = (double*)out + base;
        double cnt = (double)nr;
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[i] = (double)tot[i] / cnt;
      } else {
        long long* dst = (long long*)partial + (int64_t)s * plane + base;
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[i] = tot[i];
      }
    }
  } else {
    __shared__ uint4 sacc[8][33];
    sacc[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && live) {
#pragma unroll
      for (int j = 1; j < 8; ++j) {
        uint4 t = sacc[j][tx];
        fold_packed<KIND>(acc, *reinterpret_cast<int4*>(&t));
      }
      int64_t base = o * nx + xv * 8;
      int16_t* dst = (S == 1) ? (int16_t*)out + base : (int16_t*)partial + (int64_t)s * plane + base;
      *reinterpret_cast<uint4*>(dst) = acc;
    }
  }
}

// ---------------- keep-x, generic scalar (uint8, unaligned int16, tail columns) ----
// one thread per output element (o, x) with x in [x0, nx); reduction chunk s of S
template <typename T, int KIND>
__global__ void __launch_bounds__(256) k_keepx_scalar(const T* __restrict__ img, int64_t nx, int64_t x0,
                                                      int64_t nr, int64_t so, int64_t sr, void* __restrict__ out,
                                                      void* __restrict__ partial, int64_t plane) {
  const int64_t x = x0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t o = blockIdx.y;
  const int S = gridDim.z, s = blockIdx.z;
  if (x >= nx) return;
  const int64_t rchunk = ceil_div64(nr, S);
  const int64_t r0 = (int64_t)s * rchunk;
  const int64_t r1 = (r0 + rchunk < nr) ? r0 + rchunk : nr;
  const T* p = img + o * so + x;
  int64_t base = o * nx + x;
  if (KIND == KMEAN) {
    long long t = 0;
#pragma unroll 4
    for (int64_t r = r0; r < r1; ++r) t += (long long)p[r * sr];
    if (S == 1) ((double*)out)[base] = (double)t / (double)nr;
    else ((long long*)partial)[(int64_t)s * plane + base] = t;
  } else {
    // an empty chunk (r0 >= r1) can only happen for s > 0; seed with the identity
    int m = (KIND == KMAX) ? -2147483647 - 1 : 2147483647;
#pragma unroll 4
    for (int64_t r = r0; r < r1; ++r) {
      int v = (int)p[r * sr];
      m = (KIND == KMAX) ? max(m, v) : min(m, v);
    }
    // clamp the identity into T's range so a partial never overflows the cast
    if (r0 >= r1) m = (KIND == KMAX) ? (sizeof(T) == 1 ? 0 : -32768) : (sizeof(T) == 1 ? 255 : 32767);
    T* dst = (S == 1) ? (T*)out : (T*)partial + (int64_t)s * plane;
    dst[base] = (T)m;
  }
}

// folds partial[S][plane] into out[plane] for elements [i0, i1) per row of length nx
template <typename T, int KIND>
__global__ void __launch_bounds__(256) k_keepx_finish(const void* __restrict__ partial, int S, int64_t plane,
                                                      int64_t nr, void* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= plane) return;
  if (KIND == KMEAN) {
    const long long* p = (const long long*)partial;
    long long t = 0;
    for (int s = 0; s < S; ++s) t += p[(int64_t)s * plane + i];
    ((double*)out)[i] = (double)t / (double)nr;
  } else {
    const T* p = (const T*)partial;
    int m = (int)p[i];
    for (int s = 1; s < S; ++s) {
      int v = (int)p[(int64_t)s * plane + i];
      m = (KIND == KMAX) ? max(m, v) : min(m, v);
    }
    ((T*)out)[i] = (T)m;
  }
}

// ---------------- along-x: one warp per row --------------------------------------
template <int KIND>
__global__ void __launch_bounds__(256) k_alongx_i16_vec(const int16_t* __restrict__ img, int64_t nrows, int64_t nx,
                                                        void* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t nxv = nx >> 3;  // nx % 8 == 0 on this path
  for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < nrows; row += nwarps) {
    const int4* p = (const int4*)(img + row * nx);
    uint4 acc;
    long long tot = 0;
    if (KIND == KMAX) acc = make_uint4(0x80008000u, 0x80008000u, 0x80008000u, 0x80008000u);
    if (KIND == KMIN) acc = make_uint4(0x7fff7fffu, 0x7fff7fffu, 0x7fff7fffu, 0x7fff7fffu);
    int64_t i = lane;
    for (; i + 96 < nxv; i += 128) {
      int4 a = ld_stream(p + i), b = ld_stream(p + i + 32), c = ld_stream(p + i + 64), d = ld_stream(p + i + 96);
      if (KIND == KMEAN) {
        Acc8 s;
#pragma unroll
        for (int k = 0; k < 8; ++k) s.v[k] = 0;
        add_packed(s, a); add_packed(s, b); add_packed(s, c); add_packed(s, d);
        tot += (long long)(s.v[0] + s.v[1] + s.v[2] + s.v[3] + s.v[4] + s.v[5] + s.v[6] + s.v[7]);
      } else {
        fold_packed<KIND>(acc, a); fold_packed<KIND>(acc, b); fold_packed<KIND>(acc, c); fold_packed<KIND>(acc, d);
      }
    }
    for (; i < nxv; i += 32) {
      int4 a = ld_stream(p + i);
      if (KIND == KMEAN) {
        Acc8 s;
#pragma unroll
        for (int k = 0; k < 8; ++k) s.v[k] = 0;
        add_packed(s, a);
        tot += (long long)(s.v[0] + s.v[1] + s.v[2] + s.v[3] + s.v[4] + s.v[5] + s.v[6] + s.v[7]);
      } else {
        fold_packed<KIND>(acc, a);
      }
    }
    if (KIND == KMEAN) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      if (lane == 0) ((double*)out)[row] = (double)tot / (double)nx;
    } else {
      uint32_t m = (KIND == KMAX) ? max_s16x2(max_s16x2(acc.x, acc.y), max_s16x2(acc.z, acc.w))
                                  : min_s16x2(min_s16x2(acc.x, acc.y), min_s16x2(acc.z, acc.w));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        uint32_t t = __shfl_xor_sync(0xffffffffu, m, o);
        m = (KIND == KMAX) ? max_s16x2(m, t) : min_s16x2(m, t);
      }
      if (lane == 0) {
        int a = (int)(int16_t)(m & 0xffff), b = (int)(int16_t)(m >> 16);
        ((int16_t*)out)[row] = (int16_t)((KIND == KMAX) ? max(a, b) : min(a, b));
      }
    }
  }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(256) k_alongx_scalar(const T* __restrict__ img, int64_t nrows, int64_t nx,
                                                       void* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < nrows; row += nwarps) {
    const T* p = img + row * nx;
    long long tot = 0;
    int m = (KIND == KMAX) ? -2147483647 - 1 : 2147483647;
    for (int64_t i = lane; i < nx; i += 32) {
      int v = (int)p[i];
      if (KIND == KMEAN) tot += v; else m = (KIND == KMAX) ? max(m, v) : min(m, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      if (KIND == KMEAN) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      else {
        int t = __shfl_xor_sync(0xffffffffu, m, o);
        m = (KIND == KMAX) ? max(m, t) : min(m, t);
      }
    }
    if (lane == 0) {
      if (KIND == KMEAN) ((double*)out)[row] = (double)tot / (double)nx;
      else ((T*)out)[row] = (T)m;
    }
  }
}

struct KeepX {
  int64_t no, nx, nr, so, sr;
};
KeepX keepx_geom(int64_t dz, int64_t dy, int64_t dx, int axis) {
  KeepX g;
  if (axis == 0) { g.no = 1; g.nx = dy * dx; g.nr = dz; g.so = 0; g.sr = dy * dx; }
  else           { g.no = dz; g.nx = dx; g.nr = dy; g.so = dy * dx; g.sr = dx; }
  return g;
}
// number of reduction splits so that the grid covers the machine a few times over
int keepx_splits(const KeepX& g) {
  int64_t blocks = ceil_div64(ceil_div64(g.nx, 8), 32) * g.no;
  int64_t want = (int64_t)b2v_sm_count() * 4;
  int64_t S = 1;
  while (blocks * S < want && S < 16 && g.nr / (S * 2) >= 32) S *= 2;
  return (int)S;
}

template <typename T, int KIND>
int run_keepx(const T* img, const KeepX& g, void* out, void* ws, cudaStream_t st) {
  const int S = keepx_splits(g);
  const int64_t plane = g.no * g.nx;
  B2V_REQUIRE(g.no <= 65535, B2V_ERR_ARG, "mip: more than 65535 slices along the kept axis");
  B2V_REQUIRE(S == 1 || ws, B2V_ERR_ARG, "mip: workspace required");
  int rc;
  int64_t x0 = 0;
  if (sizeof(T) == 2) {
    bool vec = b2v_aligned16(img) && (g.sr % 8 == 0) && (g.so % 8 == 0) && g.nx >= 8 &&
               (KIND != KMEAN || g.nr <= 8 * 32768) &&
               (S == 1 ? (KIND == KMEAN || (b2v_aligned16(out) && (g.no == 1 || g.nx % 8 == 0)))
                       : (b2v_aligned16(ws) && plane % 8 == 0 && (g.no == 1 || g.nx % 8 == 0)));
    if (vec) {
      int64_t nxv = g.nx / 8;
      dim3 grid((unsigned)ceil_div64(nxv, 32), (unsigned)g.no, (unsigned)S), block(32, 8);
      k_keepx_i16_vec<KIND><<<grid, block, 0, st>>>((const int16_t*)img, g.nx, nxv, g.nr, g.so, g.sr, out, ws, plane);
      if ((rc = b2v_check_launch("k_keepx_i16_vec"))) return rc;
      x0 = nxv * 8;
    }
  }
  if (x0 < g.nx) {
    dim3 grid((unsigned)ceil_div64(g.nx - x0, 256), (unsigned)g.no, (unsigned)S);
    k_keepx_scalar<T, KIND><<<grid, 256, 0, st>>>(img, g.nx, x0, g.nr, g.so, g.sr, out, ws, plane);
    if ((rc = b2v_check_launch("k_keepx_scalar"))) return rc;
  }
  if (S > 1) {
    k_keepx_finish<T, KIND><<<(unsigned)ceil_div64(plane, 256), 256, 0, st>>>(ws, S, plane, g.nr, out);
    if ((rc = b2v_check_launch("k_keepx_finish"))) return rc;
  }
  return B2V_OK;
}

template <typename T, int KIND>
int run_alongx(const T* img, int64_t nrows, int64_t nx, void* out, cudaStream_t st) {
  const int blocks = b2v_grid(nrows, 8, 16);
  if (sizeof(T) == 2 && b2v_aligned16(img) && nx % 8 == 0)
    k_alongx_i16_vec<KIND><<<blocks, 256, 0, st>>>((const int16_t*)img, nrows, nx, out);
  else
    k_alongx_scalar<T, KIND><<<blocks, 256, 0, st>>>(img, nrows, nx, out);
  return b2v_check_launch("k_alongx");
}

template <typename T>
int run_mip(const T* img, int64_t dz, int64_t dy, int64_t dx, int axis, int kind, void* out, void* ws,
            cudaStream_t st) {
  if (axis == 2) {
    switch (kind) {
      case KMAX: return run_alongx<T, KMAX>(img, dz * dy, dx, out, st);
      case KMIN: return run_alongx<T, KMIN>(img, dz * dy, dx, out, st);
      default: return run_alongx<T, KMEAN>(img, dz * dy, dx, out, st);
    }
  }
  KeepX g = keepx_geom(dz, dy, dx, axis);
  switch (kind) {
    case KMAX: return run_keepx<T, KMAX>(img, g, out, ws, st);
    case KMIN: return run_keepx<T, KMIN>(img, g, out, ws, st);
    default: return run_keepx<T, KMEAN>(img, g, out, ws, st);
  }
}

// ---- float64 volumes (the third dtype invesalius_rs dispatches, types.rs:5-70): MaxIP / MinIP
// with NumPy's NaN propagation. 8 B/voxel; one thread per output pixel (rays along z / y: coalesced
// over x) or one warp per row (rays along x).
__device__ __forceinline__ double pick_f64(double a, double b, bool want_max) {
  if (a != a) return a;
  if (b != b) return b;
  return want_max ? (a > b ? a : b) : (a < b ? a : b);
}

__global__ void __launch_bounds__(256) k_mip_f64_keepx(const double* __restrict__ img, KeepX g, int want_max,
                                                       double* __restrict__ out) {
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t o = blockIdx.y;
  if (x >= g.nx) return;
  const double* p = img + o * g.so + x;
  double acc = p[0];
  for (int64_t r = 1; r < g.nr; ++r) acc = pick_f64(acc, p[r * g.sr], want_max != 0);
  out[o * g.nx + x] = acc;
}

__global__ void __launch_bounds__(256) k_mip_f64_alongx(const double* __restrict__ img, int64_t nrows, int64_t nx,
                                                        int want_max, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < nrows; row += nwarps) {
    const double* p = img + row * nx;
    double acc = p[lane < nx ? lane : 0];
    for (int64_t x = lane + 32; x < nx; x += 32) acc = pick_f64(acc, p[x], want_max != 0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = pick_f64(acc, __shfl_xor_sync(0xffffffffu, acc, o), want_max != 0);
    if (lane == 0) out[row] = acc;
  }
}

int run_mip_f64(const double* img, int64_t dz, int64_t dy, int64_t dx, int axis, int kind, double* out, cudaStream_t st) {
  B2V_REQUIRE(kind == KMAX || kind == KMIN, B2V_ERR_ARG, "mip: MeanIP of a float64 volume is not built (NumPy sums pairwise)");
  if (axis == 2) {
    k_mip_f64_alongx<<<b2v_grid(dz * dy, 8, 16), 256, 0, st>>>(img, dz * dy, dx, kind == KMAX, out);
    return b2v_check_launch("k_mip_f64_alongx");
  }
  KeepX g = keepx_geom(dz, dy, dx, axis);
  B2V_REQUIRE(g.no <= 65535, B2V_ERR_ARG, "mip: more than 65535 slices along the kept axis");
  k_mip_f64_keepx<<<dim3((unsigned)ceil_div64(g.nx, 256), (unsigned)g.no), 256, 0, st>>>(img, g, kind == KMAX, out);
  return b2v_check_launch("k_mip_f64_keepx");
}

}  // namespace

extern "C" int64_t b2v_mip_workspace_bytes(int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, int kind) {
  if (axis == 2 || axis < 0 || dz <= 0 || dy <= 0 || dx <= 0 || dtype == B2V_F64) return 0;
  KeepX g = keepx_geom(dz, dy, dx, axis);
  int S = keepx_splits(g);
  if (S == 1) return 0;
  int64_t elem = (kind == KMEAN) ? 8 : (dtype == B2V_U8 ? 1 : 2);
  return (int64_t)S * g.no * g.nx * elem;
}

extern "C" int b2v_mip(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, int kind, void* out,
                       void* workspace, void* stream) {
  B2V_REQUIRE(img && out, B2V_ERR_ARG, "mip: null pointer");
  B2V_REQUIRE(dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG, "mip: empty volume");
  B2V_REQUIRE(axis >= 0 && axis <= 2, B2V_ERR_ARG, "mip: axis must be 0, 1 or 2");
  B2V_REQUIRE(kind >= 0 && kind <= 2, B2V_ERR_ARG, "mip: kind must be MAX, MIN or MEAN");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == B2V_I16) return run_mip<int16_t>((const int16_t*)img, dz, dy, dx, axis, kind, out, workspace, st);
  if (dtype == B2V_U8) return run_mip<uint8_t>((const uint8_t*)img, dz, dy, dx, axis, kind, out, workspace, st);
  if (dtype == B2V_F64) return run_mip_f64((const double*)img, dz, dy, dx, axis, kind, (double*)out, st);
  B2V_REQUIRE(false, B2V_ERR_ARG, "mip: dtype code %d not supported (int16, uint8, float64)", dtype);
}
