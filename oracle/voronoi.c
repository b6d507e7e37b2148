/* CPU checker — TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * invesalius_rs.jump_flooding (floodfill_py.rs:262-276 -> floodfill.rs:298-507), restated line for line in
 * C: float32 arithmetic in the crate's operation order, -ffp-contract=off (Rust never fuses multiply-add),
 * sqrtf correctly rounded. The Jacobi steps are threaded over z with pthreads; every voxel's result
 * depends on the previous step's buffers only, so the thread count cannot change it. normalize runs
 * serially, as the crate does.
 * The reference holds no test or golden vector for jump_flooding, and the crate cannot be built without
 * rustc: PARITY UNPINNED against the crate itself. tests/test_oracle_voronoi.py pins this file on cases with
 * known answers and against an independent pure-Python restatement. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  const int32_t* own_in;
  const float* dist_in;
  int32_t* own_out;
  float* dist_out;
  const int32_t* sites;
  int64_t n_sites, nz, ny, nx, oz, oy, ox, z0, z1;
} step_args;

static float site_dist(int64_t z, int64_t y, int64_t x, float z1, float y1, float x1) {
  float dz = (float)z - z1;
  float dy = (float)y - y1;
  float dx = (float)x - x1;
  return sqrtf(dz * dz + dy * dy + dx * dx);
}

static void* step_range(void* p) {
  const step_args* a = (const step_args*)p;
  for (int64_t z = a->z0; z < a->z1; ++z)
    for (int64_t y = 0; y < a->ny; ++y)
      for (int64_t x = 0; x < a->nx; ++x) {
        const int64_t v = (z * a->ny + y) * a->nx + x;
        int32_t idx0 = a->own_in[v];
        float best = a->dist_in[v];
        for (int zi = -1; zi <= 1; ++zi)
          for (int yi = -1; yi <= 1; ++yi)
            for (int xi = -1; xi <= 1; ++xi) {
              if (xi == 0 && yi == 0 && zi == 0) continue;
              const int64_t sz = z + zi * a->oz, sy = y + yi * a->oy, sx = x + xi * a->ox;
              if (sz < 0 || sy < 0 || sx < 0 || sz >= a->nz || sy >= a->ny || sx >= a->nx) continue;
              const int32_t idx1 = a->own_in[(sz * a->ny + sy) * a->nx + sx];
              if (idx1 <= 0) continue;
              const int64_t site_i = (int64_t)idx1 - 1;
              if (site_i >= a->n_sites) continue;
              const int32_t* s = a->sites + 3 * site_i;
              const float dist1 = site_dist(z, y, x, (float)s[0], (float)s[1], (float)s[2]);
              if (idx0 > 0) {
                if (dist1 < best) {
                  idx0 = idx1;
                  best = dist1;
                }
              } else {
                idx0 = idx1;
                best = dist1;
              }
            }
        a->own_out[v] = idx0;
        a->dist_out[v] = best;
      }
  return NULL;
}

/* dist float32 / owners int32: dense [nz][ny][nx], in place. sites: dense int32 [n_sites][3] (z, y, x). */
void orc_jump_flooding(float* dist, int32_t* owners, int64_t nz, int64_t ny, int64_t nx, const int32_t* sites,
                       int64_t n_sites, int normalize, int nthreads) {
  if (n_sites == 0 || nx == 0 || ny == 0 || nz == 0) return;
  const int64_t n = nz * ny * nx;
  int32_t* own_cur = malloc(4 * n);
  float* dist_cur = malloc(4 * n);
  memcpy(own_cur, owners, 4 * n);
  memcpy(dist_cur, dist, 4 * n);

  for (int64_t i = 0; i < n_sites; ++i) {
    const int32_t z = sites[3 * i], y = sites[3 * i + 1], x = sites[3 * i + 2];
    if (z < 0 || y < 0 || x < 0) continue;
    if (z >= nz || y >= ny || x >= nx) continue;
    own_cur[((int64_t)z * ny + y) * nx + x] = (int32_t)i + 1;
    dist_cur[((int64_t)z * ny + y) * nx + x] = 0.0f;
  }

  const int64_t max_dim = nx > ny ? (nx > nz ? nx : nz) : (ny > nz ? ny : nz);
  int64_t n_steps = 0;
  if (max_dim > 1)
    while ((max_dim >> (n_steps + 1)) != 0) ++n_steps;
  int64_t ox = nx / 2, oy = ny / 2, oz = nz / 2;

  int32_t* own_next = malloc(4 * n);
  float* dist_next = malloc(4 * n);
  memcpy(own_next, own_cur, 4 * n);
  memcpy(dist_next, dist_cur, 4 * n);

  if (nthreads < 1) nthreads = 1;
  if (nthreads > nz) nthreads = (int)nz;
  pthread_t* th = malloc(sizeof(pthread_t) * nthreads);
  step_args* args = malloc(sizeof(step_args) * nthreads);
  for (int64_t step = 0; step < n_steps; ++step) {
    for (int t = 0; t < nthreads; ++t) {
      step_args a = {own_cur, dist_cur, own_next, dist_next, sites, n_sites, nz, ny, nx, oz, oy, ox,
                     nz * t / nthreads, nz * (t + 1) / nthreads};
      args[t] = a;
      if (t > 0) pthread_create(&th[t], NULL, step_range, &args[t]);
    }
    step_range(&args[0]);
    for (int t = 1; t < nthreads; ++t) pthread_join(th[t], NULL);
    int32_t* to = own_cur; own_cur = own_next; own_next = to;
    float* td = dist_cur; dist_cur = dist_next; dist_next = td;
    ox /= 2;
    oy /= 2;
    oz /= 2;
  }
  free(th);
  free(args);

  if (normalize) {
    uint32_t* counts = calloc(n_sites, sizeof(uint32_t));
    int64_t* sums = calloc(3 * n_sites, sizeof(int64_t));
    for (int64_t z = 0; z < nz; ++z)
      for (int64_t y = 0; y < ny; ++y)
        for (int64_t x = 0; x < nx; ++x) {
          const int32_t owner = own_cur[(z * ny + y) * nx + x];
          if (owner <= 0) continue;
          const int64_t idx = (int64_t)owner - 1;
          if (idx >= n_sites) continue;
          counts[idx] += 1;
          sums[3 * idx] += z;
          sums[3 * idx + 1] += y;
          sums[3 * idx + 2] += x;
        }
    int32_t* new_sites = calloc(3 * n_sites, sizeof(int32_t));
    for (int64_t i = 0; i < n_sites; ++i) {
      const int64_t c = (int64_t)counts[i];
      if (c > 0) {
        new_sites[3 * i] = (int32_t)(sums[3 * i] / c);
        new_sites[3 * i + 1] = (int32_t)(sums[3 * i + 1] / c);
        new_sites[3 * i + 2] = (int32_t)(sums[3 * i + 2] / c);
      }
    }
    float* max_dists = calloc(n_sites, sizeof(float));
    for (int64_t z = 0; z < nz; ++z)
      for (int64_t y = 0; y < ny; ++y)
        for (int64_t x = 0; x < nx; ++x) {
          const int64_t v = (z * ny + y) * nx + x;
          const int32_t owner = own_cur[v];
          if (owner <= 0) continue;
          const int64_t idx = (int64_t)owner - 1;
          if (idx >= n_sites) continue;
          const int32_t* c = new_sites + 3 * idx;
          const float d = site_dist(z, y, x, (float)c[0], (float)c[1], (float)c[2]);
          dist_cur[v] = d;
          if (d > max_dists[idx]) max_dists[idx] = d;
        }
    for (int64_t z = 0; z < nz; ++z)
      for (int64_t y = 0; y < ny; ++y)
        for (int64_t x = 0; x < nx; ++x) {
          const int64_t v = (z * ny + y) * nx + x;
          const int32_t owner = own_cur[v];
          if (owner <= 0) continue;
          const int64_t idx = (int64_t)owner - 1;
          if (idx >= n_sites) continue;
          const float max_d = max_dists[idx];
          if (max_d > 0.0f) dist_cur[v] /= max_d;
        }
    free(counts);
    free(sums);
    free(new_sites);
    free(max_dists);
  }

  memcpy(owners, own_cur, 4 * n);
  memcpy(dist, dist_cur, 4 * n);
  free(own_cur);
  free(dist_cur);
  free(own_next);
  free(dist_next);
}
