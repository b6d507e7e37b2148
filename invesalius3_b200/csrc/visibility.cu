// Remove non-visible faces (plugins/remove_non_visible_faces/remove_non_visible_faces.py:19-119) on the
// device: six (or any number of) off-screen depth buffers of the surface, vtkSelectVisiblePoints on each,
// the faces of the selected points, and vtkCleanPolyData's point merge and renumbering.
//
// The cameras are computed on the host (b2v_visibility_cameras) from the vertex bounds, in float64, as
// VTK's vtkRenderer::ResetCamera / ResetCameraClippingRange and vtkCamera's view and projection
// transforms compute them. Every device step is float64 as well, without FMA contraction (-fmad=false),
// so the sequential C checker reproduces each depth and flag bit for bit.
//
//   k_vis_bounds       vertex bounds through order-preserving uint32 keys (and a non-finite flag).
//   k_vis_project      one thread per (view, vertex): display x, y and window depth z_w, 24 B written.
//   k_vis_raster       one thread per (view, triangle): a triangle whose pixel box holds at most
//                      kSmallBox pixels is rasterised by its thread, with 64-bit atomicMin on the
//                      depth's bits (non-negative doubles order like unsigned integers); a larger one is
//                      queued for k_vis_raster_big, so a coarse mesh never serialises a warp.
//   k_vis_raster_big   a persistent grid; one block per queued triangle, its threads stride the box.
//   k_vis_points       one thread per vertex: z_w < zbuf + tolerance in any view.
//   k_merge_insert     exactly coincident vertices share one slot of an open-addressing hash table
//                      (mesh_merge.cuh, shared with the clean of clean.cu).
//   k_vis_first_use    note_first_use: atomicMin of the corner index over the kept faces, per slot.
//   k_vis_block_counts / k_scan_sums / k_vis_emit_*   the O(T) compaction: a corner is the first
//                      use of its (merged) vertex when its index is that minimum; scans of those flags
//                      number the output vertices, scans of the kept, non-degenerate faces order them.
//
// The passes are bound by the random 24-byte gathers of the projected vertices and by the atomics on the
// depth buffers (6 x 800 x 800 x 8 B = 30.7 MB, L2-resident in part), not by HBM bandwidth.
#include <math.h>
#include <string.h>

#include "b2v_common.cuh"
#include "mesh_merge.cuh"
#include "scan.cuh"

namespace {

// ---- VTK 9.3 constants: restated from the upstream sources, UNVERIFIED (VTK cannot be built here). ----
// The same table is in the C checker; parity with VTK itself is unpinned.
constexpr int kRes = 800;                             // render_window.SetSize(800, 800) (the plugin)
constexpr double kViewAngleDeg = 30.0;                // vtkCamera: ViewAngle default
constexpr double kRadPerDeg = 0.017453292519943295;   // vtkMath::RadiansFromDegrees
constexpr double kViewUpDot = 0.999;                  // vtkRenderer::ResetCamera: |vup . vn| > 0.999
constexpr double kClipExpansion = 0.5;                // vtkRenderer: ClippingRangeExpansion default
constexpr double kMinGap = 0.2;                       // ResetCameraClippingRange: far - near >= 0.2 tan(a/2) far
constexpr double kFarInit = 1e-18;                    // ResetCameraClippingRange: initial far
constexpr double kNearShrink = 0.99, kFarGrow = 1.01; // ResetCameraClippingRange: breathing room
constexpr double kNearIfInverted = 0.01;              // near >= far -> near = 0.01 far
constexpr double kNearTolerance = 0.001;              // NearClippingPlaneTolerance, depth buffer > 16 bits
constexpr double kPointTolerance = 0.01;              // vtkSelectVisiblePoints: Tolerance default
// --------------------------------------------------------------------------------------------------------

constexpr int64_t kPix = (int64_t)kRes * kRes;
constexpr int kMaxViews = 64;
constexpr int kSmallBox = 64;           // pixel-box area one thread rasterises alone
constexpr int kBlock = 256;
constexpr int kCamDoubles = B2V_VIS_CAMERA_DOUBLES;
constexpr unsigned long long kDepthOne = 0x3FF0000000000000ull;   // bits of 1.0

enum : uint32_t { ST_NONFINITE = 2u };   // a status bit beside ST_BAD_FACE (1)

struct P3 { double x, y, z; };

// ---- host: the camera of each view ---------------------------------------------------------------------
struct Cam { double pos[3], fp[3], vup[3], vn[3], clip[2], dist, radius; };

void cam_compute_distance(Cam& c) {   // vtkCamera::ComputeDistance + ComputeViewPlaneNormal
  const double d0 = c.fp[0] - c.pos[0], d1 = c.fp[1] - c.pos[1], d2 = c.fp[2] - c.pos[2];
  const double dist = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  c.vn[0] = -(d0 / dist); c.vn[1] = -(d1 / dist); c.vn[2] = -(d2 / dist);
}

void cam_set_view_up(Cam& c, double x, double y, double z) {   // vtkCamera::SetViewUp normalises
  const double n = sqrt(x * x + y * y + z * z);
  if (n != 0.0) { x /= n; y /= n; z /= n; } else { x = 0.0; y = 1.0; z = 0.0; }
  c.vup[0] = x; c.vup[1] = y; c.vup[2] = z;
}

void reset_clipping_range(Cam& c, const double* b) {   // vtkRenderer::ResetCameraClippingRange(bounds)
  const double a = -c.vn[0], bb = -c.vn[1], cc = -c.vn[2];
  const double d = -(a * c.pos[0] + bb * c.pos[1] + cc * c.pos[2]);
  double r0 = a * b[0] + bb * b[2] + cc * b[4] + d, r1 = kFarInit;
  for (int k = 0; k < 2; ++k)
    for (int j = 0; j < 2; ++j)
      for (int i = 0; i < 2; ++i) {
        const double dist = a * b[i] + bb * b[2 + j] + cc * b[4 + k] + d;
        r0 = dist < r0 ? dist : r0;
        r1 = dist > r1 ? dist : r1;
      }
  double gap = kMinGap * tan(kViewAngleDeg * kRadPerDeg / 2.0) * r1;
  if (r1 - r0 < gap) {
    gap = gap - r1 + r0;
    r1 += gap / 2.0;
    r0 -= gap / 2.0;
  }
  if (r0 < 0.0) r0 = 0.0;
  r0 = kNearShrink * r0 - (r1 - r0) * kClipExpansion;
  r1 = kFarGrow * r1 + (r1 - r0) * kClipExpansion;
  r0 = r0 >= r1 ? kNearIfInverted * r1 : r0;
  if (r0 < kNearTolerance * r1) r0 = kNearTolerance * r1;
  c.clip[0] = r0; c.clip[1] = r1;
}

void reset_camera(Cam& c, const double* b) {   // vtkRenderer::ResetCamera(bounds), aspect 1
  double center[3];
  for (int i = 0; i < 3; ++i) center[i] = (b[2 * i] + b[2 * i + 1]) / 2.0;
  double w1 = b[1] - b[0], w2 = b[3] - b[2], w3 = b[5] - b[4];
  w1 *= w1; w2 *= w2; w3 *= w3;
  double radius = w1 + w2 + w3;
  radius = radius == 0.0 ? 1.0 : radius;
  radius = sqrt(radius) * 0.5;
  const double angle = kViewAngleDeg * kRadPerDeg;
  const double distance = radius / sin(angle * 0.5);
  const double vn[3] = {c.vn[0], c.vn[1], c.vn[2]};
  const double dot = c.vup[0] * vn[0] + c.vup[1] * vn[1] + c.vup[2] * vn[2];
  if (fabs(dot) > kViewUpDot) cam_set_view_up(c, -c.vup[2], c.vup[0], c.vup[1]);
  for (int i = 0; i < 3; ++i) c.fp[i] = center[i];
  cam_compute_distance(c);
  for (int i = 0; i < 3; ++i) c.pos[i] = center[i] + distance * vn[i];
  cam_compute_distance(c);
  reset_clipping_range(c, b);
  c.dist = distance;
  c.radius = radius;
}

void mat_mul(const double* A, const double* B, double* C) {   // vtkMatrix4x4::Multiply4x4 order
  for (int i = 0; i < 4; ++i)
    for (int k = 0; k < 4; ++k)
      C[4 * i + k] = A[4 * i] * B[k] + A[4 * i + 1] * B[4 + k] + A[4 * i + 2] * B[8 + k] + A[4 * i + 3] * B[12 + k];
}

void normalize3(double* v) {   // vtkMath::Normalize
  const double den = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (den != 0.0) for (int i = 0; i < 3; ++i) v[i] /= den;
}

void cross3(const double* a, const double* b, double* c) {   // vtkMath::Cross
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// GetCompositeProjectionTransformMatrix(aspect 1, 0, 1) = (AdjustZBuffer(-1, 1, 0, 1) . Frustum) . View
void composite_matrix(const Cam& c, double* M) {
  double V[16] = {0}, n[3], s[3], u[3];
  for (int i = 0; i < 3; ++i) n[i] = c.pos[i] - c.fp[i];   // vtkPerspectiveTransform::SetupCamera
  normalize3(n);
  cross3(c.vup, n, s);
  normalize3(s);
  cross3(n, s, u);
  for (int j = 0; j < 3; ++j) { V[j] = s[j]; V[4 + j] = u[j]; V[8 + j] = n[j]; }
  const double delta[4] = {-c.pos[0], -c.pos[1], -c.pos[2], 0.0};
  for (int i = 0; i < 3; ++i)
    V[4 * i + 3] = V[4 * i] * delta[0] + V[4 * i + 1] * delta[1] + V[4 * i + 2] * delta[2] + V[4 * i + 3] * delta[3];
  V[15] = 1.0;
  const double zn = c.clip[0], zf = c.clip[1];
  const double tmp = tan(kViewAngleDeg * kRadPerDeg / 2.0);
  const double width = zn * tmp * 1.0, height = zn * tmp;
  const double xmin = (0.0 - 1.0) * width, xmax = (0.0 + 1.0) * width;
  const double ymin = (0.0 - 1.0) * height, ymax = (0.0 + 1.0) * height;
  double F[16] = {0};
  F[0] = 2 * zn / (xmax - xmin);
  F[5] = 2 * zn / (ymax - ymin);
  F[2] = (xmin + xmax) / (xmax - xmin);
  F[6] = (ymin + ymax) / (ymax - ymin);
  F[10] = -(zn + zf) / (zf - zn);
  F[14] = -1;
  F[11] = -2 * zn * zf / (zf - zn);
  double A[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  A[10] = (1.0 - 0.0) / (1.0 - -1.0);
  A[11] = (0.0 * 1.0 - 1.0 * -1.0) / (1.0 - -1.0);
  double P[16];
  mat_mul(A, F, P);
  mat_mul(P, V, M);
}

// ---- workspace --------------------------------------------------------------------------------------------
struct VisWs {
  uint32_t* misc;               // [0..5] bound keys, [6] status
  unsigned long long* totals;   // [0] output vertices, [1] output faces
  double* cams;                 // [views][16] composite matrices
  P3* proj;                     // [views][nv]
  unsigned long long* zbuf;     // [views][800][800] depth bits
  unsigned long long* qcount;   // queued large triangles
  unsigned long long* queue;    // [views * nt] (view * nt + t)
  uint8_t* vis;                 // [nv]
  int32_t* slots;               // [H] vertex index or -1
  uint32_t* rep;                // [nv] slot of the vertex's coincident group
  unsigned long long* first;    // [H] first kept corner of the group
  int32_t* newid;               // [H] output vertex id of the group
  unsigned long long* bcount;   // [2][nb] per-block corner / face counts, then their exclusive scan
  uint64_t hmask;
  int64_t nb;
  size_t bytes;
};

VisWs carve(void* base, int64_t nv, int64_t nt, int nviews) {
  VisWs w;
  char* p = (char*)base;
  size_t o = 0;
  auto take = [&](size_t n) { char* r = p + o; o += align256(n); return r; };
  const uint64_t H = merge_slots(nv);
  w.hmask = H - 1;
  w.nb = ceil_div64(nt, kBlock);
  w.misc = (uint32_t*)take(64);
  w.totals = (unsigned long long*)take(16);
  w.qcount = (unsigned long long*)take(8);
  w.cams = (double*)take((size_t)nviews * 16 * sizeof(double));
  w.zbuf = (unsigned long long*)take((size_t)nviews * kPix * 8);
  w.vis = (uint8_t*)take((size_t)nv);
  w.proj = (P3*)take((size_t)nviews * nv * sizeof(P3));
  w.queue = (unsigned long long*)take((size_t)nviews * nt * 8);
  w.slots = (int32_t*)take(H * 4);
  w.rep = (uint32_t*)take((size_t)nv * 4);
  w.first = (unsigned long long*)take(H * 8);
  w.newid = (int32_t*)take(H * 4);
  w.bcount = (unsigned long long*)take((size_t)w.nb * 2 * 8);
  w.bytes = o;
  return w;
}

// ---- device helpers ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t u = canon_bits(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __forceinline__ float key_to_float(uint32_t k) {
  uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// ---- bounds -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_vis_bounds(const float* __restrict__ v, int64_t nv, uint32_t* misc) {
  uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0, 0, 0};
  bool bad = false;
  for (int64_t i = gtid(); i < nv; i += gstride()) {
    for (int a = 0; a < 3; ++a) {
      const float f = v[3 * i + a];
      if (!isfinite(f)) { bad = true; continue; }
      const uint32_t k = order_key(f);
      lo[a] = min(lo[a], k);
      hi[a] = max(hi[a], k);
    }
  }
  for (int a = 0; a < 3; ++a)
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
  bad = __any_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    for (int a = 0; a < 3; ++a) { atomicMin(&misc[2 * a], lo[a]); atomicMax(&misc[2 * a + 1], hi[a]); }
    if (bad) atomicOr(&misc[6], (uint32_t)ST_NONFINITE);
  }
}

// ---- projection -------------------------------------------------------------------------------------------
// vtkSelectVisiblePoints::IsPointOccluded: view = M [x y z 1] (vtkMatrix4x4::MultiplyPoint), then
// vtkViewport::ViewToDisplay: ((x/w + 1) * 800) / 2; the depth is z/w. w == 0 marks the point invisible.
__global__ void __launch_bounds__(kBlock) k_vis_project(const float* __restrict__ v, int64_t nv, int nviews,
                                                        const double* __restrict__ cams, P3* __restrict__ proj) {
  const int64_t n = (int64_t)nviews * nv;
  for (int64_t i = gtid(); i < n; i += gstride()) {
    const int view = (int)(i / nv);
    const int64_t k = i - (int64_t)view * nv;
    const double* M = cams + 16 * view;
    const double x = v[3 * k], y = v[3 * k + 1], z = v[3 * k + 2];
    const double o0 = x * M[0] + y * M[1] + z * M[2] + 1.0 * M[3];
    const double o1 = x * M[4] + y * M[5] + z * M[6] + 1.0 * M[7];
    const double o2 = x * M[8] + y * M[9] + z * M[10] + 1.0 * M[11];
    const double o3 = x * M[12] + y * M[13] + z * M[14] + 1.0 * M[15];
    P3 p;
    if (o3 == 0.0) {
      p.x = p.y = p.z = __longlong_as_double(0x7ff8000000000000ll);
    } else {
      p.x = (o0 / o3 + 1.0) * (double)kRes / 2.0;
      p.y = (o1 / o3 + 1.0) * (double)kRes / 2.0;
      p.z = o2 / o3;
    }
    proj[i] = p;
  }
}

// ---- rasterisation ----------------------------------------------------------------------------------------
struct Tri {
  P3 a, b, c;
  double area;
  int x0, x1, y0, y1;
};

// Orients the triangle counter-clockwise in display space (y up); false when it covers no pixel centre.
__device__ __forceinline__ bool tri_setup(P3 a, P3 b, P3 c, Tri& T) {
  double area = (b.x - a.x) * (c.y - a.y) - (b.y - a.y) * (c.x - a.x);
  if (!(area > 0.0) && !(area < 0.0)) return false;   // zero area (or a point with w == 0)
  if (area < 0.0) { const P3 t = b; b = c; c = t; area = -area; }
  const double lx = fmin(fmin(a.x, b.x), c.x), hx = fmax(fmax(a.x, b.x), c.x);
  const double ly = fmin(fmin(a.y, b.y), c.y), hy = fmax(fmax(a.y, b.y), c.y);
  double fx0 = floor(lx - 0.5), fx1 = ceil(hx - 0.5), fy0 = floor(ly - 0.5), fy1 = ceil(hy - 0.5);
  fx0 = fmax(fx0, 0.0); fy0 = fmax(fy0, 0.0);
  fx1 = fmin(fx1, (double)(kRes - 1)); fy1 = fmin(fy1, (double)(kRes - 1));
  if (!(fx0 <= fx1) || !(fy0 <= fy1)) return false;
  T.a = a; T.b = b; T.c = c; T.area = area;
  T.x0 = (int)fx0; T.x1 = (int)fx1; T.y0 = (int)fy0; T.y1 = (int)fy1;
  return true;
}

__device__ __forceinline__ double edge_fn(const P3& p, const P3& q, double px, double py) {
  return (q.x - p.x) * (py - p.y) - (q.y - p.y) * (px - p.x);
}
// top-left rule for a counter-clockwise triangle in a y-up frame: left edges run down, top edges run -x
__device__ __forceinline__ bool top_left(const P3& p, const P3& q) {
  const double dy = q.y - p.y, dx = q.x - p.x;
  return dy < 0.0 || (dy == 0.0 && dx < 0.0);
}
__device__ __forceinline__ bool inside(double w, const P3& p, const P3& q) { return w > 0.0 || (w == 0.0 && top_left(p, q)); }

// depth of pixel (i, j) if its centre is covered: screen-space affine interpolation of z_w, >= 0
__device__ __forceinline__ void raster_pixel(const Tri& T, int i, int j, unsigned long long* __restrict__ zb) {
  const double px = i + 0.5, py = j + 0.5;
  const double w0 = edge_fn(T.b, T.c, px, py), w1 = edge_fn(T.c, T.a, px, py), w2 = edge_fn(T.a, T.b, px, py);
  if (!inside(w0, T.b, T.c) || !inside(w1, T.c, T.a) || !inside(w2, T.a, T.b)) return;
  double z = (w0 * T.a.z + w1 * T.b.z + w2 * T.c.z) / T.area;
  if (!(z > 0.0)) z = 0.0;
  const unsigned long long bits = (unsigned long long)__double_as_longlong(z);
  unsigned long long* cell = zb + (int64_t)j * kRes + i;
  if (bits < *cell) atomicMin(cell, bits);
}

__device__ __forceinline__ bool tri_of(const Faces& F, const P3* __restrict__ proj, int64_t nv, int view, int64_t t,
                                       Tri& T) {
  int64_t v[3];
  if (!load_face(F, t, v)) return false;
  const P3* pv = proj + (int64_t)view * nv;
  return tri_setup(pv[v[0]], pv[v[1]], pv[v[2]], T);
}

__global__ void __launch_bounds__(kBlock) k_vis_raster(Faces F, int nviews, const P3* __restrict__ proj,
                                                       unsigned long long* __restrict__ zbuf,
                                                       unsigned long long* __restrict__ queue,
                                                       unsigned long long* qcount, uint32_t* misc) {
  const int64_t n = (int64_t)nviews * F.nt;
  for (int64_t i = gtid(); i < n; i += gstride()) {
    const int view = (int)(i / F.nt);
    const int64_t t = i - (int64_t)view * F.nt;
    if (view == 0) {
      int64_t v[3];
      if (!load_face(F, t, v)) atomicOr(&misc[6], (uint32_t)ST_BAD_FACE);
    }
    Tri T;
    if (!tri_of(F, proj, F.nv, view, t, T)) continue;
    const int64_t box = (int64_t)(T.x1 - T.x0 + 1) * (T.y1 - T.y0 + 1);
    if (box > kSmallBox) {
      queue[atomicAdd(qcount, 1ull)] = (unsigned long long)i;
      continue;
    }
    unsigned long long* zb = zbuf + (int64_t)view * kPix;
    for (int j = T.y0; j <= T.y1; ++j)
      for (int x = T.x0; x <= T.x1; ++x) raster_pixel(T, x, j, zb);
  }
}

__global__ void __launch_bounds__(kBlock) k_vis_raster_big(Faces F, const P3* __restrict__ proj,
                                                           unsigned long long* __restrict__ zbuf,
                                                           const unsigned long long* __restrict__ queue,
                                                           const unsigned long long* qcount) {
  const unsigned long long nq = *qcount;
  for (unsigned long long q = blockIdx.x; q < nq; q += gridDim.x) {
    const int64_t i = (int64_t)queue[q];
    const int view = (int)(i / F.nt);
    const int64_t t = i - (int64_t)view * F.nt;
    Tri T;
    if (!tri_of(F, proj, F.nv, view, t, T)) continue;   // uniform over the block
    const int bw = T.x1 - T.x0 + 1;
    const int64_t box = (int64_t)bw * (T.y1 - T.y0 + 1);
    unsigned long long* zb = zbuf + (int64_t)view * kPix;
    for (int64_t p = threadIdx.x; p < box; p += blockDim.x)
      raster_pixel(T, T.x0 + (int)(p % bw), T.y0 + (int)(p / bw), zb);
  }
}

// ---- point visibility -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_vis_points(int64_t nv, int nviews, const P3* __restrict__ proj,
                                                       const unsigned long long* __restrict__ zbuf,
                                                       uint8_t* __restrict__ vis) {
  for (int64_t k = gtid(); k < nv; k += gstride()) {
    uint8_t seen = 0;
    for (int view = 0; view < nviews && !seen; ++view) {
      const P3 p = proj[(int64_t)view * nv + k];
      if (p.x >= 0.0 && p.x <= (double)(kRes - 1) && p.y >= 0.0 && p.y <= (double)(kRes - 1)) {
        const double z = __longlong_as_double(
            (long long)zbuf[(int64_t)view * kPix + (int64_t)(int)p.y * kRes + (int)p.x]);
        if (p.z < z + kPointTolerance) seen = 1;
      }
    }
    vis[k] = seen;
  }
}

// ---- face selection and compaction ------------------------------------------------------------------------
__device__ __forceinline__ bool face_kept(const Faces& F, int64_t t, const uint8_t* __restrict__ vis, uint8_t flip,
                                          int64_t v[3]) {
  if (!load_face(F, t, v)) return false;
  return ((vis[v[0]] ^ flip) | (vis[v[1]] ^ flip) | (vis[v[2]] ^ flip)) != 0;
}

__global__ void __launch_bounds__(kBlock) k_vis_first_use(Faces F, const uint8_t* __restrict__ vis, uint8_t flip,
                                                          const uint32_t* __restrict__ rep,
                                                          unsigned long long* first) {
  for (int64_t t = gtid(); t < F.nt; t += gstride()) {
    int64_t v[3];
    if (!face_kept(F, t, vis, flip, v)) continue;
    for (int c = 0; c < 3; ++c) note_first_use(first, rep[v[c]], (unsigned long long)(3 * t + c));
  }
}

struct FaceFlags {
  uint32_t corners;     // bit c: corner c is the first use of its merged vertex
  bool emit;            // kept and not degenerate after the merge
  uint32_t r[3];
  int64_t v[3];
};

__device__ __forceinline__ FaceFlags face_flags(const Faces& F, int64_t t, const uint8_t* __restrict__ vis, uint8_t flip,
                                                const uint32_t* __restrict__ rep,
                                                const unsigned long long* __restrict__ first) {
  FaceFlags o;
  o.corners = 0;
  o.emit = false;
  if (t >= F.nt || !face_kept(F, t, vis, flip, o.v)) return o;
  for (int c = 0; c < 3; ++c) {
    o.r[c] = rep[o.v[c]];
    if (is_first_use(first, o.r[c], (unsigned long long)(3 * t + c))) o.corners |= 1u << c;
  }
  o.emit = o.r[0] != o.r[1] && o.r[1] != o.r[2] && o.r[0] != o.r[2];
  return o;
}

__global__ void __launch_bounds__(kBlock) k_vis_block_counts(Faces F, const uint8_t* __restrict__ vis, uint8_t flip,
                                                             const uint32_t* __restrict__ rep,
                                                             const unsigned long long* __restrict__ first,
                                                             unsigned long long* __restrict__ bcount, int64_t nb) {
  __shared__ uint32_t s_w[kBlock / 32];
  const int64_t t = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const FaceFlags f = face_flags(F, t, vis, flip, rep, first);
  const uint32_t packed = (uint32_t)__popc(f.corners) | ((uint32_t)f.emit << 16);
  uint32_t tot;
  block_exscan<uint32_t>(packed, s_w, &tot);
  if (threadIdx.x == 0) {
    bcount[blockIdx.x] = tot & 0xffffu;
    bcount[nb + blockIdx.x] = tot >> 16;
  }
}

__global__ void __launch_bounds__(kBlock) k_vis_emit_verts(Faces F, const float* __restrict__ verts,
                                                           const uint8_t* __restrict__ vis, uint8_t flip,
                                                           const uint32_t* __restrict__ rep,
                                                           const unsigned long long* __restrict__ first,
                                                           const unsigned long long* __restrict__ boff,
                                                           int32_t* __restrict__ newid, float* __restrict__ out) {
  __shared__ uint32_t s_w[kBlock / 32];
  const int64_t t = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const FaceFlags f = face_flags(F, t, vis, flip, rep, first);
  uint32_t tot;
  uint64_t id = boff[blockIdx.x] + block_exscan<uint32_t>((uint32_t)__popc(f.corners), s_w, &tot);
  for (int c = 0; c < 3; ++c) {
    if (!(f.corners >> c & 1u)) continue;
    newid[f.r[c]] = (int32_t)id;
    const int64_t k = f.v[c];
    out[3 * id] = verts[3 * k];
    out[3 * id + 1] = verts[3 * k + 1];
    out[3 * id + 2] = verts[3 * k + 2];
    ++id;
  }
}

__global__ void __launch_bounds__(kBlock) k_vis_emit_faces(Faces F, const uint8_t* __restrict__ vis, uint8_t flip,
                                                           const uint32_t* __restrict__ rep,
                                                           const unsigned long long* __restrict__ first,
                                                           const unsigned long long* __restrict__ boff,
                                                           const int32_t* __restrict__ newid,
                                                           int32_t* __restrict__ out) {
  __shared__ uint32_t s_w[kBlock / 32];
  const int64_t t = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  const FaceFlags f = face_flags(F, t, vis, flip, rep, first);
  uint32_t tot;
  const uint64_t id = boff[blockIdx.x] + block_exscan<uint32_t>((uint32_t)f.emit, s_w, &tot);
  if (!f.emit) return;
  for (int c = 0; c < 3; ++c) out[3 * id + c] = newid[f.r[c]];
}

int check_mesh(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
               int nviews, const char* what) {
  B2V_REQUIRE(nv > 0 && nv <= 0x7fffffffLL && nt >= 0, B2V_ERR_ARG, "%s: need 1 <= V < 2^31 and T >= 0", what);
  B2V_REQUIRE(face_cols == 3 || face_cols == 4, B2V_ERR_ARG, "%s: faces must be [T,3] or [T,4]", what);
  B2V_REQUIRE(faces_i64 == 0 || faces_i64 == 1, B2V_ERR_ARG, "%s: faces_i64 must be 0 or 1", what);
  B2V_REQUIRE(nviews >= 1 && nviews <= kMaxViews, B2V_ERR_ARG, "%s: 1..%d views", what, kMaxViews);
  B2V_REQUIRE(verts && (nt == 0 || faces), B2V_ERR_ARG, "%s: null device pointer", what);
  return B2V_OK;
}

}  // namespace

extern "C" int b2v_visibility_cameras(const double* bounds_host, const double* positions_host, int nviews,
                                      double* cameras_host) {
  B2V_REQUIRE(bounds_host && positions_host && cameras_host, B2V_ERR_ARG, "visibility_cameras: null argument");
  B2V_REQUIRE(nviews >= 1 && nviews <= kMaxViews, B2V_ERR_ARG, "visibility_cameras: 1..%d views", kMaxViews);
  for (int i = 0; i < 6; ++i)
    B2V_REQUIRE(isfinite(bounds_host[i]), B2V_ERR_ARG, "visibility_cameras: bounds must be finite");
  for (int k = 0; k < nviews; ++k) {
    const double* d = positions_host + 3 * k;
    B2V_REQUIRE(isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2]), B2V_ERR_ARG,
                "visibility_cameras: position %d is not finite", k);
    B2V_REQUIRE(d[0] != 0.0 || d[1] != 0.0 || d[2] != 0.0, B2V_ERR_ARG,
                "visibility_cameras: position %d is the zero vector (it gives no view direction)", k);
  }
  // the default camera: position (0, 0, 1), focal point 0, view-up (0, 1, 0); renderer.ResetCamera()
  Cam c;
  memset(&c, 0, sizeof(c));
  c.pos[2] = 1.0;
  cam_set_view_up(c, 0.0, 1.0, 0.0);
  cam_compute_distance(c);
  reset_camera(c, bounds_host);
  const double v[3] = {c.pos[0] - c.fp[0], c.pos[1] - c.fp[1], c.pos[2] - c.fp[2]};
  const double mag = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const double fp[3] = {c.fp[0], c.fp[1], c.fp[2]};
  for (int k = 0; k < nviews; ++k) {
    const double* d = positions_host + 3 * k;
    for (int i = 0; i < 3; ++i) c.pos[i] = fp[i] + d[i] * mag;   // camera.SetPosition(fp + position * mag)
    const double e0 = c.fp[0] - c.pos[0], e1 = c.fp[1] - c.pos[1], e2 = c.fp[2] - c.pos[2];
    B2V_REQUIRE(sqrt(e0 * e0 + e1 * e1 + e2 * e2) > 0.0, B2V_ERR_ARG,
                "visibility_cameras: position %d puts the camera on the focal point", k);
    cam_compute_distance(c);
    reset_camera(c, bounds_host);
    double* out = cameras_host + (int64_t)kCamDoubles * k;
    composite_matrix(c, out);
    for (int i = 0; i < 3; ++i) { out[16 + i] = c.pos[i]; out[19 + i] = c.fp[i]; out[22 + i] = c.vup[i]; }
    out[25] = c.clip[0]; out[26] = c.clip[1];
    out[27] = c.dist; out[28] = c.radius;
    out[29] = out[30] = out[31] = 0.0;
  }
  return B2V_OK;
}

extern "C" int64_t b2v_visibility_workspace_bytes(int64_t nv, int64_t nt, int nviews) {
  if (nv < 0 || nt < 0 || nviews < 1 || nviews > kMaxViews) return -1;
  return (int64_t)carve(nullptr, nv, nt, nviews).bytes;
}

extern "C" int b2v_visibility_layout(int64_t nv, int64_t nt, int nviews, int64_t* layout_out) {
  B2V_REQUIRE(nv >= 0 && nt >= 0 && nviews >= 1 && nviews <= kMaxViews && layout_out, B2V_ERR_ARG,
              "visibility_layout: bad arguments");
  const VisWs w = carve(nullptr, nv, nt, nviews);
  layout_out[0] = (int64_t)((char*)w.zbuf - (char*)nullptr);   // float64 [views][800][800]
  layout_out[1] = (int64_t)((char*)w.vis - (char*)nullptr);    // uint8 [V]: seen by some view
  layout_out[2] = (int64_t)((char*)w.qcount - (char*)nullptr); // uint64: triangles the cooperative path drew
  return B2V_OK;
}

extern "C" int b2v_visibility_bounds(const float* verts, int64_t nv, void* workspace, void* stream,
                                     double* bounds_host) {
  B2V_REQUIRE(nv > 0 && verts && workspace && bounds_host, B2V_ERR_ARG, "visibility_bounds: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  uint32_t init[8] = {0xffffffffu, 0, 0xffffffffu, 0, 0xffffffffu, 0, 0, 0};
  uint32_t* misc = (uint32_t*)workspace;
  B2V_CUDA(cudaMemcpyAsync(misc, init, sizeof(init), cudaMemcpyHostToDevice, s));
  k_vis_bounds<<<b2v_grid(nv, kBlock, 8), kBlock, 0, s>>>(verts, nv, misc);
  if (int rc = b2v_check_launch("k_vis_bounds")) return rc;
  uint32_t got[8];
  B2V_CUDA(cudaMemcpyAsync(got, misc, sizeof(got), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!(got[6] & ST_NONFINITE), B2V_ERR_ARG, "remove_non_visible_faces: vertices must be finite");
  for (int i = 0; i < 6; ++i) bounds_host[i] = (double)key_to_float(got[i]);
  return B2V_OK;
}

extern "C" int b2v_visibility_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                                    int faces_i64, const double* cameras_host, int nviews, int remove_visible,
                                    void* workspace, void* stream, int64_t* nverts_host, int64_t* nfaces_host) {
  if (int rc = check_mesh(verts, nv, faces, nt, face_cols, faces_i64, nviews, "visibility_count")) return rc;
  B2V_REQUIRE(cameras_host && workspace && nverts_host && nfaces_host, B2V_ERR_ARG,
              "visibility_count: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const VisWs w = carve(workspace, nv, nt, nviews);
  const Faces F{faces, nt, face_cols, faces_i64, nv};
  const uint8_t flip = remove_visible ? 1 : 0;
  double mats[kMaxViews * 16];
  for (int k = 0; k < nviews; ++k) memcpy(mats + 16 * k, cameras_host + (int64_t)kCamDoubles * k, 16 * sizeof(double));
  B2V_CUDA(cudaMemcpyAsync(w.cams, mats, (size_t)nviews * 16 * sizeof(double), cudaMemcpyHostToDevice, s));
  B2V_CUDA(cudaMemsetAsync(w.misc, 0, 64, s));
  B2V_CUDA(cudaMemsetAsync(w.totals, 0, 16, s));
  B2V_CUDA(cudaMemsetAsync(w.qcount, 0, 8, s));
  if (int rc = merge_reset(w.slots, w.first, w.hmask + 1, s)) return rc;

  k_fill<unsigned long long><<<b2v_grid((int64_t)nviews * kPix, kBlock, 8), kBlock, 0, s>>>(
      w.zbuf, (int64_t)nviews * kPix, kDepthOne);
  if (int rc = b2v_check_launch("k_fill")) return rc;
  k_vis_project<<<b2v_grid((int64_t)nviews * nv, kBlock, 16), kBlock, 0, s>>>(verts, nv, nviews, w.cams, w.proj);
  if (int rc = b2v_check_launch("k_vis_project")) return rc;
  if (int rc = merge_points(verts, nv, w.hmask, w.slots, w.rep, s)) return rc;
  if (nt > 0) {
    k_vis_raster<<<b2v_grid((int64_t)nviews * nt, kBlock, 16), kBlock, 0, s>>>(F, nviews, w.proj, w.zbuf, w.queue,
                                                                               w.qcount, w.misc);
    if (int rc = b2v_check_launch("k_vis_raster")) return rc;
    k_vis_raster_big<<<(unsigned)b2v_sm_count() * 4, kBlock, 0, s>>>(F, w.proj, w.zbuf, w.queue, w.qcount);
    if (int rc = b2v_check_launch("k_vis_raster_big")) return rc;
  }
  k_vis_points<<<b2v_grid(nv, kBlock, 16), kBlock, 0, s>>>(nv, nviews, w.proj, w.zbuf, w.vis);
  if (int rc = b2v_check_launch("k_vis_points")) return rc;
  if (nt > 0) {
    k_vis_first_use<<<b2v_grid(nt, kBlock, 16), kBlock, 0, s>>>(F, w.vis, flip, w.rep, w.first);
    if (int rc = b2v_check_launch("k_vis_first_use")) return rc;
    B2V_REQUIRE(w.nb <= 0x7fffffffLL, B2V_ERR_ARG, "visibility_count: too many faces");
    k_vis_block_counts<<<(unsigned)w.nb, kBlock, 0, s>>>(F, w.vis, flip, w.rep, w.first, w.bcount, w.nb);
    if (int rc = b2v_check_launch("k_vis_block_counts")) return rc;
    k_scan_sums<unsigned long long><<<2, 1024, 0, s>>>(w.bcount, w.nb, w.totals);
    if (int rc = b2v_check_launch("k_scan_sums")) return rc;
  }
  unsigned long long tot[2];
  uint32_t status = 0;
  B2V_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaMemcpyAsync(&status, w.misc + 6, sizeof(status), cudaMemcpyDeviceToHost, s));
  B2V_CUDA(cudaStreamSynchronize(s));
  B2V_REQUIRE(!(status & ST_BAD_FACE), B2V_ERR_ARG,
              "remove_non_visible_faces: a face has an index outside [0, V) (or a leading entry other than 3)");
  *nverts_host = (int64_t)tot[0];
  *nfaces_host = (int64_t)tot[1];
  return B2V_OK;
}

extern "C" int b2v_visibility_emit(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols,
                                   int faces_i64, int nviews, int remove_visible, void* workspace, float* verts_out,
                                   int32_t* faces_out, void* stream) {
  if (int rc = check_mesh(verts, nv, faces, nt, face_cols, faces_i64, nviews, "visibility_emit")) return rc;
  B2V_REQUIRE(workspace, B2V_ERR_ARG, "visibility_emit: null workspace");
  if (nt == 0) return B2V_OK;   // (an empty output may be NULL: nothing is written to it)
  cudaStream_t s = (cudaStream_t)stream;
  const VisWs w = carve(workspace, nv, nt, nviews);
  const Faces F{faces, nt, face_cols, faces_i64, nv};
  const uint8_t flip = remove_visible ? 1 : 0;
  k_vis_emit_verts<<<(unsigned)w.nb, kBlock, 0, s>>>(F, verts, w.vis, flip, w.rep, w.first, w.bcount, w.newid,
                                                      verts_out);
  if (int rc = b2v_check_launch("k_vis_emit_verts")) return rc;
  k_vis_emit_faces<<<(unsigned)w.nb, kBlock, 0, s>>>(F, w.vis, flip, w.rep, w.first, w.bcount + w.nb, w.newid,
                                                      faces_out);
  return b2v_check_launch("k_vis_emit_faces");
}
