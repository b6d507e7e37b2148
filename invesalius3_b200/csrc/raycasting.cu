// Data preparation of the 3-D volume rendering (invesalius/data/volume.py): the arrays VTK's ray caster is
// handed, not the rendering itself.
//   b2v_raycast_flip_shift_i16   vtkImageFlip (axis 1, about the origin) + vtkImageShiftScale to unsigned
//                                short with shift abs(min)                         volume.py:575-634
//   b2v_vtk_convolve5x5_u16      vtkImageConvolve with SetKernel5x5, one preset filter  volume.py:538-563
// The contract (VTK's boundary rule, restated from memory and unverified) is written once, in the header of
// the C checker, raycasting.c; every result here equals it bit for bit. float64, no FMA (-fmad=false).
#include <math.h>

#include <algorithm>

#include "b2v_common.cuh"

namespace {

// ---- flip and shift -----------------------------------------------------------------------------------
// u[z][y][x] = m[z][dy-1-y][x] + |min|. The values are integers below 2^16, so the int sum equals the
// contract's float64 sum. VEC: rows of a multiple of 8 voxels on 16-byte aligned buffers, 8 voxels a lane.
template <bool VEC>
__global__ void __launch_bounds__(256) k_flip_shift(const int16_t* __restrict__ in, int64_t rows, int dy, int row_items,
                                                    const float* __restrict__ mm, uint16_t* __restrict__ out) {
  const int s = (int)fabsf(mm[0]);
  for (int64_t r = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; r < rows; r += (int64_t)gridDim.x * blockDim.y) {
    const int64_t z = r / dy;
    const int64_t src = (z * dy + (dy - 1 - (r - z * dy))) * row_items, dst = r * row_items;
    for (int i = threadIdx.x; i < row_items; i += blockDim.x) {
      if constexpr (VEC) {
        const uint4 a = ld_stream(reinterpret_cast<const uint4*>(in) + src + i);
        uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t lo = (uint32_t)((int)(int16_t)(w[k] & 0xffffu) + s) & 0xffffu;
          const uint32_t hi = (uint32_t)((int)(int16_t)(w[k] >> 16) + s) & 0xffffu;
          w[k] = lo | (hi << 16);
        }
        st_stream(reinterpret_cast<uint4*>(out) + dst + i, make_uint4(w[0], w[1], w[2], w[3]));
      } else {
        out[dst + i] = (uint16_t)(in[src + i] + s);
      }
    }
  }
}

// ---- the 5x5 convolution ------------------------------------------------------------------------------
struct Weights {
  double w[25];
};

constexpr int TX = 32;        // outputs per tile along x: one per lane
constexpr int TR = 8;         // outputs per thread along y: eight independent float64 chains
constexpr int TW = 8;         // warps per block
constexpr int TY = TW * TR;   // outputs per tile along y
constexpr int SX = TX + 4, SY = TY + 4;
constexpr int RING_THREADS = TX * TW;

// Voxels of one slice whose 5x5 window leaves the slice: all of them when a side is shorter than 5, else the
// two outer rows and columns. Interior voxels are (y, x) with 2 <= y < ny - 2 and 2 <= x < nx - 2.
__host__ __device__ __forceinline__ int64_t ring_count(int ny, int nx) {
  return (ny < 5 || nx < 5) ? (int64_t)ny * nx : 4 * (int64_t)nx + 4 * (int64_t)(ny - 4);
}

// The truncation of a sum in [0, 65536); a sum that rounding carries to 65536 gives 65535, as in the checker.
__device__ __forceinline__ uint16_t to_u16(double sum) { return (uint16_t)min(__double2uint_rz(sum), 65535u); }

// One border voxel as the contract states it: the kernel index advances only on in-bounds taps.
__device__ __forceinline__ uint16_t ring_voxel(const uint16_t* __restrict__ sl, int ny, int nx, int y, int x,
                                               const Weights& w) {
  double sum = 0.0;
  int k = 0;
  for (int b = 0; b < 5; ++b) {
    const int yy = y + b - 2;
    if (yy < 0 || yy >= ny) continue;
    for (int a = 0; a < 5; ++a) {
      const int xx = x + a - 2;
      if (xx < 0 || xx >= nx) continue;
      sum += (double)sl[(int64_t)yy * nx + xx] * w.w[k];
      ++k;
    }
  }
  return to_u16(sum);
}

// blockIdx.x < tiles: one TY x TX tile of interior outputs, staged with its 2-voxel halo as float64 in shared
// memory. Each thread walks the 4 + TR input rows of its column once and adds every row to the outputs whose
// window holds it: for each output the rows arrive in order b = 0..4 and the taps of a row in order a = 0..4,
// the contract's order, and the weights are compile-time operands from the parameter bank.
// blockIdx.x >= tiles: the ring voxels of the slice, one per thread, read from global memory.
__global__ void __launch_bounds__(TX * TW) k_convolve5x5(const uint16_t* __restrict__ in, int64_t nz, int ny, int nx,
                                                         int tiles_x, int tiles, const __grid_constant__ Weights w,
                                                         uint16_t* __restrict__ out) {
  __shared__ double tile[SY][SX];
  const int64_t plane = (int64_t)ny * nx;
  for (int64_t z = blockIdx.y; z < nz; z += gridDim.y) {
    const uint16_t* sl = in + z * plane;
    uint16_t* ol = out + z * plane;
    if ((int)blockIdx.x >= tiles) {
      const int64_t i = (int64_t)((int)blockIdx.x - tiles) * RING_THREADS + threadIdx.y * TX + threadIdx.x;
      if (i >= ring_count(ny, nx)) continue;
      int y, x;
      if (ny < 5 || nx < 5) {
        y = (int)(i / nx);
        x = (int)(i - (int64_t)y * nx);
      } else if (i < 4 * (int64_t)nx) {
        const int r = (int)(i / nx);
        y = r < 2 ? r : ny - 4 + r;
        x = (int)(i - (int64_t)r * nx);
      } else {
        const int j = (int)(i - 4 * (int64_t)nx), c = j & 3;
        y = 2 + (j >> 2);
        x = c < 2 ? c : nx - 4 + c;
      }
      ol[(int64_t)y * nx + x] = ring_voxel(sl, ny, nx, y, x, w);
      continue;
    }
    // tile origin in output coordinates (interior: +2 on both axes); the halo starts 2 before it
    const int ox = 2 + ((int)blockIdx.x % tiles_x) * TX, oy = 2 + ((int)blockIdx.x / tiles_x) * TY;
    __syncthreads();   // the previous slice's reads of the tile are done
    for (int t = threadIdx.y * TX + threadIdx.x; t < SY * SX; t += TX * TW) {
      const int ty = t / SX, tx = t - ty * SX;
      const int gy = oy - 2 + ty, gx = ox - 2 + tx;
      tile[ty][tx] = (gy < ny && gx < nx) ? (double)sl[(int64_t)gy * nx + gx] : 0.0;
    }
    __syncthreads();
    const int x = ox + threadIdx.x, y0 = oy + threadIdx.y * TR;
    if (x >= nx - 2 || y0 >= ny - 2) continue;
    double acc[TR];
#pragma unroll
    for (int j = 0; j < TR; ++j) acc[j] = 0.0;
    const double* col = &tile[threadIdx.y * TR][threadIdx.x];
#pragma unroll
    for (int r = 0; r < TR + 4; ++r) {       // input row y0 - 2 + r
      double v[5];
#pragma unroll
      for (int a = 0; a < 5; ++a) v[a] = col[r * SX + a];
#pragma unroll
      for (int j = 0; j < TR; ++j) {         // output row y0 + j reads this row as its row b = r - j
        const int b = r - j;
        if (b >= 0 && b < 5) {
#pragma unroll
          for (int a = 0; a < 5; ++a) acc[j] += v[a] * w.w[b * 5 + a];
        }
      }
    }
#pragma unroll
    for (int j = 0; j < TR; ++j)
      if (y0 + j < ny - 2) ol[(int64_t)(y0 + j) * nx + x] = to_u16(acc[j]);
  }
}

}  // namespace

extern "C" int b2v_raycast_flip_shift_i16(const int16_t* in, int64_t dz, int64_t dy, int64_t dx, const float* minmax_dev,
                                          uint16_t* out, void* stream) {
  B2V_REQUIRE(in && minmax_dev && out && (const void*)in != (const void*)out && dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG,
              "raycast_flip_shift: bad arguments");
  B2V_REQUIRE(dy < (1ll << 31) && dx < (1ll << 31), B2V_ERR_ARG, "raycast_flip_shift: rows or columns too many");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t rows = dz * dy;
  const bool vec = dx % 8 == 0 && b2v_aligned16(in) && b2v_aligned16(out);
  const int items = (int)(vec ? dx / 8 : dx);
  const dim3 block(32, 8);
  const int grid = b2v_grid(rows, 8, 8);
  if (vec) k_flip_shift<true><<<grid, block, 0, s>>>(in, rows, (int)dy, items, minmax_dev, out);
  else k_flip_shift<false><<<grid, block, 0, s>>>(in, rows, (int)dy, items, minmax_dev, out);
  return b2v_check_launch("k_flip_shift");
}

extern "C" int b2v_vtk_convolve5x5_u16(const uint16_t* in, int64_t dz, int64_t dy, int64_t dx, const double* weights_host,
                                       uint16_t* out, void* stream) {
  B2V_REQUIRE(in && weights_host && out && in != out && dz > 0 && dy > 0 && dx > 0, B2V_ERR_ARG,
              "vtk_convolve5x5: bad arguments");
  B2V_REQUIRE(dy < (1ll << 30) && dx < (1ll << 30), B2V_ERR_ARG, "vtk_convolve5x5: slice too large");
  Weights w;
  double sum = 0.0;
  for (int k = 0; k < 25; ++k) {
    w.w[k] = weights_host[k];
    B2V_REQUIRE(isfinite(w.w[k]) && w.w[k] >= 0.0, B2V_ERR_ARG,
                "vtk_convolve5x5: weight %d is negative or not finite", k);
    sum += w.w[k];
  }
  B2V_REQUIRE(65535.0 * sum < 65536.0, B2V_ERR_ARG,
              "vtk_convolve5x5: the weights sum to %.17g; 65535 times that must stay below 65536", sum);
  const int ny = (int)dy, nx = (int)dx;
  const bool interior = ny >= 5 && nx >= 5;
  const int tiles_x = interior ? (int)ceil_div64(nx - 4, TX) : 0;
  const int64_t tiles = interior ? (int64_t)tiles_x * ceil_div64(ny - 4, TY) : 0;
  const int64_t blocks = tiles + ceil_div64(ring_count(ny, nx), RING_THREADS);
  B2V_REQUIRE(blocks < (1ll << 31), B2V_ERR_ARG, "vtk_convolve5x5: slice too large");
  const dim3 grid((unsigned)blocks, (unsigned)std::min<int64_t>(dz, 65535)), block(TX, TW);
  k_convolve5x5<<<grid, block, 0, (cudaStream_t)stream>>>(in, dz, ny, nx, tiles_x, (int)tiles, w, out);
  return b2v_check_launch("k_convolve5x5");
}
