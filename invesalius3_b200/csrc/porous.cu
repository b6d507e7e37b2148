// The porous-creation plugin's TPMS and Blobs scaffolds (plugins/porous_creation/schwarzp.py:11-34) and the
// float64 image_normalize of its OK step (gui.py:237):
//   b2v_tpms_f64                 create_schwarzp's float64 field
//   b2v_tpms_i16                 image_normalize(create_schwarzp(...), min_, max_): two launches that both evaluate
//                                the field, one reducing it to its min / max, one storing the int16 result
//   b2v_image_normalize_f64_i16  image_normalize of a float64 device array (the Blobs field), the same two passes
//
// create_schwarzp takes cos and sin of 1-D np.ogrid axes only and then broadcasts float64 *, + and - over the
// volume. The caller computes the six 1-D tables [cos_x | sin_x | cos_y | sin_y | cos_z | sin_z] with NumPy, and
// tpms_value combines them per voxel in NumPy's evaluation order; the library builds with -fmad=false, so every
// product and sum is rounded on its own and the field equals NumPy's bit for bit.
//
// Voxels are walked as rows: blocks grid-stride over the (z, y) rows, the threads of a block stride over x, so the
// y and z table entries are read once per row. A float64 array is walked as rows of kArrayRow elements.
#include <math.h>

#include "b2v_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kArraySrc = -1;          // "surface" code of a float64 array source
constexpr int64_t kArrayRow = 4096;
constexpr int kMaxBlocks = 2048;       // per-block (min, max) partials in the workspace

// One TPMS value from the table entries of its voxel (B2V_TPMS_* codes), in NumPy's order of operations.
template <int S>
__device__ __forceinline__ double tpms_value(double cx, double snx, double cy, double sny, double cz, double snz) {
  if (S == B2V_TPMS_SCHWARZ_P) return (cx + cy) + cz;
  if (S == B2V_TPMS_SCHWARZ_D)
    return (((snx * sny) * snz + (snx * cy) * cz) + (cx * sny) * cz) + (cx * cy) * snz;
  if (S == B2V_TPMS_GYROID) return (cx * sny + cy * snz) + cz * snx;
  if (S == B2V_TPMS_NEOVIUS) return 3.0 * ((cx + cy) + cz) + ((4.0 * cx) * cy) * cz;
  if (S == B2V_TPMS_IWP) return ((cx * cy + cy * cz) + cz * cx) - (cx * cy) * cz;
  return (4.0 * ((cx * cy + cy * cz) + cz * cx) - ((3.0 * cx) * cy) * cz) + 2.4;   // B2V_TPMS_P_W_HYBRID
}

// A field to walk: a TPMS surface from its tables, or a dense float64 array (S == kArraySrc).
struct Field {
  const double* tab;   // TPMS tables, or the array
  int64_t nz, ny, nx;  // TPMS shape; an array is (1, rows, kArrayRow) with n voxels
  int64_t rows, row_len, n;
};

struct Row {
  int64_t base;        // flat index of the row's first voxel
  int64_t len;         // voxels in the row
  double cy, sny, cz, snz;
};

template <int S>
__device__ __forceinline__ Row row_of(const Field& f, int64_t r) {
  Row w;
  w.base = r * f.row_len;
  if (S == kArraySrc) {
    w.len = f.n - w.base < f.row_len ? f.n - w.base : f.row_len;
    w.cy = w.sny = w.cz = w.snz = 0.0;
  } else {
    const int64_t z = r / f.ny, y = r - z * f.ny;
    w.len = f.nx;
    w.cy = f.tab[2 * f.nx + y];
    w.sny = f.tab[2 * f.nx + f.ny + y];
    w.cz = f.tab[2 * (f.nx + f.ny) + z];
    w.snz = f.tab[2 * (f.nx + f.ny) + f.nz + z];
  }
  return w;
}

template <int S>
__device__ __forceinline__ double value_at(const Field& f, const Row& w, int64_t x) {
  if (S == kArraySrc) return f.tab[w.base + x];
  return tpms_value<S>(f.tab[x], f.tab[f.nx + x], w.cy, w.sny, w.cz, w.snz);
}

// NumPy's min / max: a NaN anywhere is the result
__device__ __forceinline__ double nan_min(double a, double b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

// (min, max) over the block, returned to every thread; s holds 2 x 8 doubles
__device__ __forceinline__ double2 block_minmax(double lo, double hi, double* s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    s[threadIdx.x >> 5] = lo;
    s[8 + (threadIdx.x >> 5)] = hi;
  }
  __syncthreads();
  lo = s[0];
  hi = s[8];
  for (int k = 1; k < kThreads / 32; ++k) {
    lo = nan_min(lo, s[k]);
    hi = nan_max(hi, s[8 + k]);
  }
  __syncthreads();
  return make_double2(lo, hi);
}

template <int S>
__global__ void __launch_bounds__(kThreads) k_field_store(Field f, double* __restrict__ out) {
  for (int64_t r = blockIdx.x; r < f.rows; r += gridDim.x) {
    const Row w = row_of<S>(f, r);
    for (int64_t x = threadIdx.x; x < w.len; x += kThreads) out[w.base + x] = value_at<S>(f, w, x);
  }
}

// pass 1: part[blockIdx.x] = (min, max) of the block's voxels
template <int S>
__global__ void __launch_bounds__(kThreads) k_field_minmax(Field f, double2* __restrict__ part) {
  __shared__ double s[16];
  double lo = INFINITY, hi = -INFINITY;
  for (int64_t r = blockIdx.x; r < f.rows; r += gridDim.x) {
    const Row w = row_of<S>(f, r);
    for (int64_t x = threadIdx.x; x < w.len; x += kThreads) {
      const double v = value_at<S>(f, w, x);
      lo = nan_min(lo, v);
      hi = nan_max(hi, v);
    }
  }
  const double2 m = block_minmax(lo, hi, s);
  if (threadIdx.x == 0) part[blockIdx.x] = m;
}

// pass 2: every block reduces the nparts partials to (imin, imax), then evaluates its voxels again and stores
// image_normalize's int16; block 0 leaves (imin, imax) in mm for the caller
template <int S>
__global__ void __launch_bounds__(kThreads) k_field_normalize(Field f, const double2* __restrict__ part, int nparts,
                                                              double span, double min_f, int16_t fill,
                                                              int16_t* __restrict__ out, double2* mm) {
  __shared__ double s[16];
  double lo = INFINITY, hi = -INFINITY;
  for (int k = threadIdx.x; k < nparts; k += kThreads) {
    const double2 p = part[k];
    lo = nan_min(lo, p.x);
    hi = nan_max(hi, p.y);
  }
  const double2 m = block_minmax(lo, hi, s);
  if (blockIdx.x == 0 && threadIdx.x == 0) *mm = m;
  const bool flat = m.x == m.y;
  const double scale = span / (m.y - m.x);
  for (int64_t r = blockIdx.x; r < f.rows; r += gridDim.x) {
    const Row w = row_of<S>(f, r);
    for (int64_t x = threadIdx.x; x < w.len; x += kThreads)
      out[w.base + x] = flat ? fill : normalize_i16<double>(value_at<S>(f, w, x), m.x, scale, min_f);
  }
}

Field tpms_field(const double* tables, int64_t nz, int64_t ny, int64_t nx) {
  return Field{tables, nz, ny, nx, nz * ny, nx, nz * ny * nx};
}

Field array_field(const double* in, int64_t n) {
  const int64_t rows = ceil_div64(n, kArrayRow);
  return Field{in, 1, rows, kArrayRow, rows, kArrayRow, n};
}

int blocks_for(const Field& f) {
  int64_t b = b2v_grid(f.n, 4 * kThreads, 8);
  if (b > f.rows) b = f.rows;
  return (int)(b < kMaxBlocks ? b : kMaxBlocks);
}

// Layout of the normalise workspace: (imin, imax) of the last call, then kMaxBlocks partials.
constexpr int64_t kWsBytes = 256 + 16 * (int64_t)kMaxBlocks;

template <int S>
int store_f64(const Field& f, double* out, cudaStream_t s) {
  k_field_store<S><<<blocks_for(f), kThreads, 0, s>>>(f, out);
  return b2v_check_launch("k_field_store");
}

template <int S>
int normalize_i16_passes(const Field& f, double span, double min_f, int16_t fill, void* workspace, int16_t* out,
                         cudaStream_t s) {
  double2* mm = (double2*)workspace;
  double2* part = (double2*)((char*)workspace + 256);
  const int nb = blocks_for(f);
  k_field_minmax<S><<<nb, kThreads, 0, s>>>(f, part);
  int rc = b2v_check_launch("k_field_minmax");
  if (rc) return rc;
  k_field_normalize<S><<<nb, kThreads, 0, s>>>(f, part, nb, span, min_f, fill, out, mm);
  return b2v_check_launch("k_field_normalize");
}

bool tpms_args_ok(const double* tables, int64_t nz, int64_t ny, int64_t nx, int surface) {
  return tables && nz > 0 && ny > 0 && nx > 0 && surface >= B2V_TPMS_SCHWARZ_P && surface <= B2V_TPMS_P_W_HYBRID &&
         nz <= INT64_MAX / ny / nx;
}

}  // namespace

extern "C" int b2v_tpms_f64(const double* tables, int64_t nz, int64_t ny, int64_t nx, int surface, double* out,
                            void* stream) {
  B2V_REQUIRE(nz >= 0 && ny >= 0 && nx >= 0, B2V_ERR_ARG, "tpms: negative size");
  if (nz == 0 || ny == 0 || nx == 0) return B2V_OK;
  B2V_REQUIRE(tpms_args_ok(tables, nz, ny, nx, surface) && out, B2V_ERR_ARG,
              "tpms: null pointer, bad shape or unknown surface %d", surface);
  const Field f = tpms_field(tables, nz, ny, nx);
  cudaStream_t s = (cudaStream_t)stream;
  switch (surface) {
    case B2V_TPMS_SCHWARZ_P: return store_f64<B2V_TPMS_SCHWARZ_P>(f, out, s);
    case B2V_TPMS_SCHWARZ_D: return store_f64<B2V_TPMS_SCHWARZ_D>(f, out, s);
    case B2V_TPMS_GYROID: return store_f64<B2V_TPMS_GYROID>(f, out, s);
    case B2V_TPMS_NEOVIUS: return store_f64<B2V_TPMS_NEOVIUS>(f, out, s);
    case B2V_TPMS_IWP: return store_f64<B2V_TPMS_IWP>(f, out, s);
    default: return store_f64<B2V_TPMS_P_W_HYBRID>(f, out, s);
  }
}

extern "C" int64_t b2v_tpms_i16_workspace_bytes(int64_t nz, int64_t ny, int64_t nx) {
  return (nz > 0 && ny > 0 && nx > 0) ? kWsBytes : 0;
}

extern "C" int b2v_tpms_i16(const double* tables, int64_t nz, int64_t ny, int64_t nx, int surface, double span,
                            double min_f, int16_t fill, void* workspace, int16_t* out, void* stream) {
  B2V_REQUIRE(nz >= 0 && ny >= 0 && nx >= 0, B2V_ERR_ARG, "tpms: negative size");
  if (nz == 0 || ny == 0 || nx == 0) return B2V_OK;
  B2V_REQUIRE(tpms_args_ok(tables, nz, ny, nx, surface) && out && workspace, B2V_ERR_ARG,
              "tpms: null pointer, bad shape or unknown surface %d", surface);
  const Field f = tpms_field(tables, nz, ny, nx);
  cudaStream_t s = (cudaStream_t)stream;
  switch (surface) {
    case B2V_TPMS_SCHWARZ_P: return normalize_i16_passes<B2V_TPMS_SCHWARZ_P>(f, span, min_f, fill, workspace, out, s);
    case B2V_TPMS_SCHWARZ_D: return normalize_i16_passes<B2V_TPMS_SCHWARZ_D>(f, span, min_f, fill, workspace, out, s);
    case B2V_TPMS_GYROID: return normalize_i16_passes<B2V_TPMS_GYROID>(f, span, min_f, fill, workspace, out, s);
    case B2V_TPMS_NEOVIUS: return normalize_i16_passes<B2V_TPMS_NEOVIUS>(f, span, min_f, fill, workspace, out, s);
    case B2V_TPMS_IWP: return normalize_i16_passes<B2V_TPMS_IWP>(f, span, min_f, fill, workspace, out, s);
    default: return normalize_i16_passes<B2V_TPMS_P_W_HYBRID>(f, span, min_f, fill, workspace, out, s);
  }
}

extern "C" int64_t b2v_image_normalize_f64_workspace_bytes(int64_t n) { return n > 0 ? kWsBytes : 0; }

extern "C" int b2v_image_normalize_f64_i16(const double* in, int64_t n, double span, double min_f, int16_t fill,
                                           void* workspace, int16_t* out, void* stream) {
  B2V_REQUIRE(n >= 0, B2V_ERR_ARG, "image_normalize: negative size");
  if (n == 0) return B2V_OK;
  B2V_REQUIRE(in && out && workspace, B2V_ERR_ARG, "image_normalize: null pointer");
  return normalize_i16_passes<kArraySrc>(array_field(in, n), span, min_f, fill, workspace, out,
                                         (cudaStream_t)stream);
}
