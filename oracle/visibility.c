/* CPU checker for "Remove non-visible faces" — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of plugins/remove_non_visible_faces/remove_non_visible_faces.py:19-119:
 *   1. the camera of each view: VTK's default camera, renderer.ResetCamera(), then per position
 *      camera.SetPosition(fp + position * mag) and ResetCamera() (vtkRenderer::ResetCamera,
 *      ResetCameraClippingRange, vtkCamera::ComputeDistance / SetViewUp, the view transform of
 *      vtkPerspectiveTransform::SetupCamera, Frustum and AdjustZBuffer composed as
 *      GetCompositeProjectionTransformMatrix(1, 0, 1));
 *   2. an 800x800 float64 depth buffer per view, cleared to 1.0: a triangle covers pixel (i, j) when the
 *      centre (i + 0.5, j + 0.5) is inside it or on a top / left edge, both faces drawn, its depth the
 *      screen-space affine interpolation of the vertices' window depths (clamped at 0), the minimum wins;
 *   3. vtkSelectVisiblePoints (tolerance 0.01): display point ((x/w + 1) 800) / 2, visible when inside
 *      [0, 799]^2 and z/w < zbuf[int(dy)][int(dx)] + 0.01 in any view;
 *   4. the faces with any selected vertex, in input order, cleaned as vtkCleanPolyData does: exactly
 *      coincident points merged (first use wins), vertices numbered in order of first use over the kept
 *      faces' corners, faces that degenerate after the merge dropped (VTK makes lines of them; the points
 *      they use stay, as in VTK's output).
 *
 * UNPINNED: VTK is neither vendored nor installable here, so the constants in the table below are restated
 * from the upstream VTK 9.3 sources and have not been checked against VTK; the depth buffer is this
 * restatement's own float64 rasteriser, not OpenGL's. The device code (invesalius3_b200/csrc/visibility.cu)
 * keeps its own copy of the table; the two must agree bit for bit, which the GPU tests check.
 * Arithmetic: float64 throughout, -ffp-contract=off.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- VTK 9.3 constants: restated from the upstream sources, UNVERIFIED ---------------------------------- */
#define RES 800                            /* render_window.SetSize(800, 800) */
#define VIEW_ANGLE_DEG 30.0                /* vtkCamera ViewAngle default */
#define RAD_PER_DEG 0.017453292519943295   /* vtkMath::RadiansFromDegrees */
#define VIEW_UP_DOT 0.999                  /* ResetCamera: |vup . vn| > 0.999 rotates the view-up */
#define CLIP_EXPANSION 0.5                 /* vtkRenderer ClippingRangeExpansion */
#define MIN_GAP 0.2                        /* far - near >= 0.2 tan(angle / 2) far */
#define FAR_INIT 1e-18                     /* initial far of ResetCameraClippingRange */
#define NEAR_SHRINK 0.99
#define FAR_GROW 1.01
#define NEAR_IF_INVERTED 0.01              /* near >= far -> near = 0.01 far */
#define NEAR_TOLERANCE 0.001               /* NearClippingPlaneTolerance for a depth buffer > 16 bits */
#define POINT_TOLERANCE 0.01               /* vtkSelectVisiblePoints Tolerance */
/* --------------------------------------------------------------------------------------------------------- */

#define CAM_DOUBLES 32

typedef struct { double pos[3], fp[3], vup[3], vn[3], clip[2], dist, radius; } Cam;
typedef struct { double x, y, z; } P3;

static void compute_distance(Cam* c) {
  double d0 = c->fp[0] - c->pos[0], d1 = c->fp[1] - c->pos[1], d2 = c->fp[2] - c->pos[2];
  double dist = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
  c->vn[0] = -(d0 / dist);
  c->vn[1] = -(d1 / dist);
  c->vn[2] = -(d2 / dist);
}

static void set_view_up(Cam* c, double x, double y, double z) {
  double n = sqrt(x * x + y * y + z * z);
  if (n != 0.0) {
    x /= n; y /= n; z /= n;
  } else {
    x = 0.0; y = 1.0; z = 0.0;
  }
  c->vup[0] = x; c->vup[1] = y; c->vup[2] = z;
}

static void clipping_range(Cam* c, const double* b) {
  double a = -c->vn[0], bb = -c->vn[1], cc = -c->vn[2];
  double d = -(a * c->pos[0] + bb * c->pos[1] + cc * c->pos[2]);
  double near = a * b[0] + bb * b[2] + cc * b[4] + d, far = FAR_INIT;
  for (int k = 0; k < 2; ++k)
    for (int j = 0; j < 2; ++j)
      for (int i = 0; i < 2; ++i) {
        double dist = a * b[i] + bb * b[2 + j] + cc * b[4 + k] + d;
        if (dist < near) near = dist;
        if (dist > far) far = dist;
      }
  double gap = MIN_GAP * tan(VIEW_ANGLE_DEG * RAD_PER_DEG / 2.0) * far;
  if (far - near < gap) {
    gap = gap - far + near;
    far += gap / 2.0;
    near -= gap / 2.0;
  }
  if (near < 0.0) near = 0.0;
  near = NEAR_SHRINK * near - (far - near) * CLIP_EXPANSION;
  far = FAR_GROW * far + (far - near) * CLIP_EXPANSION;
  if (near >= far) near = NEAR_IF_INVERTED * far;
  if (near < NEAR_TOLERANCE * far) near = NEAR_TOLERANCE * far;
  c->clip[0] = near;
  c->clip[1] = far;
}

static void reset_camera(Cam* c, const double* b) {
  double center[3], vn[3];
  for (int i = 0; i < 3; ++i) center[i] = (b[2 * i] + b[2 * i + 1]) / 2.0;
  double w1 = b[1] - b[0], w2 = b[3] - b[2], w3 = b[5] - b[4];
  w1 *= w1; w2 *= w2; w3 *= w3;
  double radius = w1 + w2 + w3;
  if (radius == 0.0) radius = 1.0;
  radius = sqrt(radius) * 0.5;
  double distance = radius / sin(VIEW_ANGLE_DEG * RAD_PER_DEG * 0.5);
  for (int i = 0; i < 3; ++i) vn[i] = c->vn[i];
  if (fabs(c->vup[0] * vn[0] + c->vup[1] * vn[1] + c->vup[2] * vn[2]) > VIEW_UP_DOT)
    set_view_up(c, -c->vup[2], c->vup[0], c->vup[1]);
  for (int i = 0; i < 3; ++i) c->fp[i] = center[i];
  compute_distance(c);
  for (int i = 0; i < 3; ++i) c->pos[i] = center[i] + distance * vn[i];
  compute_distance(c);
  clipping_range(c, b);
  c->dist = distance;
  c->radius = radius;
}

static void mul4(const double* A, const double* B, double* C) {
  for (int i = 0; i < 4; ++i)
    for (int k = 0; k < 4; ++k)
      C[4 * i + k] = A[4 * i] * B[k] + A[4 * i + 1] * B[4 + k] + A[4 * i + 2] * B[8 + k] + A[4 * i + 3] * B[12 + k];
}

static void unit(double* v) {
  double den = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (den != 0.0)
    for (int i = 0; i < 3; ++i) v[i] /= den;
}

static void cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

static void composite(const Cam* c, double* M) {
  double V[16] = {0}, n[3], s[3], u[3];
  for (int i = 0; i < 3; ++i) n[i] = c->pos[i] - c->fp[i];
  unit(n);
  cross(c->vup, n, s);
  unit(s);
  cross(n, s, u);
  for (int j = 0; j < 3; ++j) {
    V[j] = s[j];
    V[4 + j] = u[j];
    V[8 + j] = n[j];
  }
  double delta[4] = {-c->pos[0], -c->pos[1], -c->pos[2], 0.0};
  for (int i = 0; i < 3; ++i)
    V[4 * i + 3] = V[4 * i] * delta[0] + V[4 * i + 1] * delta[1] + V[4 * i + 2] * delta[2] + V[4 * i + 3] * delta[3];
  V[15] = 1.0;
  double zn = c->clip[0], zf = c->clip[1];
  double t = tan(VIEW_ANGLE_DEG * RAD_PER_DEG / 2.0);
  double width = zn * t * 1.0, height = zn * t;
  double xmin = (0.0 - 1.0) * width, xmax = (0.0 + 1.0) * width;
  double ymin = (0.0 - 1.0) * height, ymax = (0.0 + 1.0) * height;
  double F[16] = {0};
  F[0] = 2 * zn / (xmax - xmin);
  F[5] = 2 * zn / (ymax - ymin);
  F[2] = (xmin + xmax) / (xmax - xmin);
  F[6] = (ymin + ymax) / (ymax - ymin);
  F[10] = -(zn + zf) / (zf - zn);
  F[14] = -1;
  F[11] = -2 * zn * zf / (zf - zn);
  double A[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  A[10] = (1.0 - 0.0) / (1.0 - -1.0);               /* AdjustZBuffer(-1, 1, 0, 1) */
  A[11] = (0.0 * 1.0 - 1.0 * -1.0) / (1.0 - -1.0);
  double P[16];
  mul4(A, F, P);
  mul4(P, V, M);
}

/* 0 ok, 1 a zero or non-finite direction, 2 non-finite bounds */
int orc_vis_cameras(const double* bounds, const double* positions, int nviews, double* out) {
  for (int i = 0; i < 6; ++i)
    if (!isfinite(bounds[i])) return 2;
  for (int k = 0; k < nviews; ++k) {
    const double* d = positions + 3 * k;
    if (!isfinite(d[0]) || !isfinite(d[1]) || !isfinite(d[2])) return 1;
    if (d[0] == 0.0 && d[1] == 0.0 && d[2] == 0.0) return 1;
  }
  Cam c;
  memset(&c, 0, sizeof(c));
  c.pos[2] = 1.0;
  set_view_up(&c, 0.0, 1.0, 0.0);
  compute_distance(&c);
  reset_camera(&c, bounds);
  double v[3] = {c.pos[0] - c.fp[0], c.pos[1] - c.fp[1], c.pos[2] - c.fp[2]};
  double mag = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  double fp[3] = {c.fp[0], c.fp[1], c.fp[2]};
  for (int k = 0; k < nviews; ++k) {
    const double* d = positions + 3 * k;
    for (int i = 0; i < 3; ++i) c.pos[i] = fp[i] + d[i] * mag;
    double e0 = c.fp[0] - c.pos[0], e1 = c.fp[1] - c.pos[1], e2 = c.fp[2] - c.pos[2];
    if (!(sqrt(e0 * e0 + e1 * e1 + e2 * e2) > 0.0)) return 1;
    compute_distance(&c);
    reset_camera(&c, bounds);
    double* o = out + (int64_t)CAM_DOUBLES * k;
    composite(&c, o);
    for (int i = 0; i < 3; ++i) {
      o[16 + i] = c.pos[i];
      o[19 + i] = c.fp[i];
      o[22 + i] = c.vup[i];
    }
    o[25] = c.clip[0];
    o[26] = c.clip[1];
    o[27] = c.dist;
    o[28] = c.radius;
    o[29] = o[30] = o[31] = 0.0;
  }
  return 0;
}

/* vertex bounds (xmin, xmax, ymin, ymax, zmin, zmax); a zero bound is +0 */
void orc_vis_bounds(const float* v, int64_t nv, double* b) {
  for (int a = 0; a < 3; ++a) {
    float lo = v[a], hi = v[a];
    for (int64_t i = 1; i < nv; ++i) {
      float f = v[3 * i + a];
      if (f < lo) lo = f;
      if (f > hi) hi = f;
    }
    b[2 * a] = lo == 0.0f ? 0.0 : (double)lo;
    b[2 * a + 1] = hi == 0.0f ? 0.0 : (double)hi;
  }
}

static P3 project(const double* M, const float* v) {
  double x = v[0], y = v[1], z = v[2];
  double o0 = x * M[0] + y * M[1] + z * M[2] + 1.0 * M[3];
  double o1 = x * M[4] + y * M[5] + z * M[6] + 1.0 * M[7];
  double o2 = x * M[8] + y * M[9] + z * M[10] + 1.0 * M[11];
  double o3 = x * M[12] + y * M[13] + z * M[14] + 1.0 * M[15];
  P3 p;
  if (o3 == 0.0) {
    p.x = p.y = p.z = NAN;
  } else {
    p.x = (o0 / o3 + 1.0) * (double)RES / 2.0;
    p.y = (o1 / o3 + 1.0) * (double)RES / 2.0;
    p.z = o2 / o3;
  }
  return p;
}

static double edge(P3 p, P3 q, double px, double py) { return (q.x - p.x) * (py - p.y) - (q.y - p.y) * (px - p.x); }
static int top_left(P3 p, P3 q) {
  double dy = q.y - p.y, dx = q.x - p.x;
  return dy < 0.0 || (dy == 0.0 && dx < 0.0);
}
static int in_edge(double w, P3 p, P3 q) { return w > 0.0 || (w == 0.0 && top_left(p, q)); }

/* draws one triangle; returns its pixel-box area (0 when nothing was drawn) */
static int64_t draw(P3 a, P3 b, P3 c, double* zb) {
  double area = (b.x - a.x) * (c.y - a.y) - (b.y - a.y) * (c.x - a.x);
  if (!(area > 0.0) && !(area < 0.0)) return 0;
  if (area < 0.0) {
    P3 t = b; b = c; c = t;
    area = -area;
  }
  double lx = fmin(fmin(a.x, b.x), c.x), hx = fmax(fmax(a.x, b.x), c.x);
  double ly = fmin(fmin(a.y, b.y), c.y), hy = fmax(fmax(a.y, b.y), c.y);
  double fx0 = fmax(floor(lx - 0.5), 0.0), fx1 = fmin(ceil(hx - 0.5), RES - 1.0);
  double fy0 = fmax(floor(ly - 0.5), 0.0), fy1 = fmin(ceil(hy - 0.5), RES - 1.0);
  if (!(fx0 <= fx1) || !(fy0 <= fy1)) return 0;
  int x0 = (int)fx0, x1 = (int)fx1, y0 = (int)fy0, y1 = (int)fy1;
  for (int j = y0; j <= y1; ++j)
    for (int i = x0; i <= x1; ++i) {
      double px = i + 0.5, py = j + 0.5;
      double w0 = edge(b, c, px, py), w1 = edge(c, a, px, py), w2 = edge(a, b, px, py);
      if (!in_edge(w0, b, c) || !in_edge(w1, c, a) || !in_edge(w2, a, b)) continue;
      double z = (w0 * a.z + w1 * b.z + w2 * c.z) / area;
      if (!(z > 0.0)) z = 0.0;
      double* cell = zb + (int64_t)j * RES + i;
      if (z < *cell) *cell = z;
    }
  return (int64_t)(x1 - x0 + 1) * (y1 - y0 + 1);
}

static const float* g_sort_v;
static int cmp_vertex(const void* pa, const void* pb) {
  int64_t ia = *(const int64_t*)pa, ib = *(const int64_t*)pb;
  const float *a = g_sort_v + 3 * ia, *b = g_sort_v + 3 * ib;
  for (int k = 0; k < 3; ++k) {
    if (a[k] < b[k]) return -1;
    if (a[k] > b[k]) return 1;
  }
  return ia < ib ? -1 : (ia > ib);
}

/* The whole operation. faces: int64 [nt][3], every index in [0, nv). zbuf (nullable): float64
 * [nviews][800][800]; vis: uint8 [nv]; verts_out: float32 [nv][3] capacity; faces_out: int32 [nt][3]
 * capacity; counts[0..2] = output vertices, output faces, triangles whose pixel box exceeds 64 pixels.
 * Returns orc_vis_cameras' code, or 3 when out of memory. */
int orc_vis_run(const float* v, int64_t nv, const int64_t* faces, int64_t nt, const double* positions, int nviews,
                int remove_visible, double* cams, double* zbuf, uint8_t* vis, float* verts_out, int32_t* faces_out,
                int64_t* counts) {
  double bounds[6];
  counts[0] = counts[1] = counts[2] = 0;
  orc_vis_bounds(v, nv, bounds);
  int rc = orc_vis_cameras(bounds, positions, nviews, cams);
  if (rc) return rc;
  P3* proj = malloc((size_t)nv * sizeof(P3));
  double* zb = malloc((size_t)RES * RES * sizeof(double));
  int64_t* order = malloc((size_t)nv * sizeof(int64_t));
  int64_t* group = malloc((size_t)nv * sizeof(int64_t));
  int64_t* gnew = malloc((size_t)nv * sizeof(int64_t));
  uint8_t* keep = malloc((size_t)(nt > 0 ? nt : 1));
  if (!proj || !zb || !order || !group || !gnew || !keep) {
    free(proj); free(zb); free(order); free(group); free(gnew); free(keep);
    return 3;
  }
  memset(vis, 0, (size_t)nv);
  for (int k = 0; k < nviews; ++k) {
    const double* M = cams + (int64_t)CAM_DOUBLES * k;
    for (int64_t i = 0; i < nv; ++i) proj[i] = project(M, v + 3 * i);
    for (int64_t i = 0; i < (int64_t)RES * RES; ++i) zb[i] = 1.0;
    for (int64_t t = 0; t < nt; ++t) {
      const int64_t* f = faces + 3 * t;
      if (draw(proj[f[0]], proj[f[1]], proj[f[2]], zb) > 64) counts[2]++;
    }
    for (int64_t i = 0; i < nv; ++i) {
      P3 p = proj[i];
      if (p.x >= 0.0 && p.x <= RES - 1.0 && p.y >= 0.0 && p.y <= RES - 1.0 &&
          p.z < zb[(int64_t)(int)p.y * RES + (int)p.x] + POINT_TOLERANCE)
        vis[i] = 1;
    }
    if (zbuf) memcpy(zbuf + (int64_t)k * RES * RES, zb, (size_t)RES * RES * sizeof(double));
  }
  /* coincident groups: sort by (x, y, z) with float comparison (-0 == +0), the smallest index labels a run */
  for (int64_t i = 0; i < nv; ++i) order[i] = i;
  g_sort_v = v;
  qsort(order, (size_t)nv, sizeof(int64_t), cmp_vertex);
  for (int64_t r = 0; r < nv; ++r) {
    int64_t i = order[r];
    if (r > 0) {
      int64_t p = order[r - 1];
      if (v[3 * p] == v[3 * i] && v[3 * p + 1] == v[3 * i + 1] && v[3 * p + 2] == v[3 * i + 2]) {
        group[i] = group[p];
        continue;
      }
    }
    group[i] = i;
  }
  uint8_t flip = remove_visible ? 1 : 0;
  for (int64_t i = 0; i < nv; ++i) gnew[i] = -1;
  int64_t nvo = 0, nto = 0;
  for (int64_t t = 0; t < nt; ++t) {   /* the corner walk of vtkCleanPolyData */
    const int64_t* f = faces + 3 * t;
    keep[t] = (uint8_t)(((vis[f[0]] ^ flip) | (vis[f[1]] ^ flip) | (vis[f[2]] ^ flip)) != 0);
    if (!keep[t]) continue;
    for (int c = 0; c < 3; ++c) {
      int64_t g = group[f[c]];
      if (gnew[g] < 0) {
        gnew[g] = nvo;
        memcpy(verts_out + 3 * nvo, v + 3 * f[c], 3 * sizeof(float));
        nvo++;
      }
    }
  }
  for (int64_t t = 0; t < nt; ++t) {
    if (!keep[t]) continue;
    const int64_t* f = faces + 3 * t;
    int64_t a = gnew[group[f[0]]], b = gnew[group[f[1]]], c = gnew[group[f[2]]];
    if (a == b || b == c || a == c) continue;
    faces_out[3 * nto] = (int32_t)a;
    faces_out[3 * nto + 1] = (int32_t)b;
    faces_out[3 * nto + 2] = (int32_t)c;
    nto++;
  }
  counts[0] = nvo;
  counts[1] = nto;
  free(proj); free(zb); free(order); free(group); free(gnew); free(keep);
  return 0;
}
