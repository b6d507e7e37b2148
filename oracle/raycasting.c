/* CPU checker of the volume rendering's data preparation — TEST INFRASTRUCTURE ONLY, never linked into the product.
 *
 * A sequential restatement of what Volume.LoadVolume (invesalius/data/volume.py:575-634), ApplyConvolution
 * (:538-563) and CalculateHistogram (:723-735) compute with VTK before the ray caster sees the volume. The
 * rendering itself (mappers, colour and opacity tables, shading, the cut plane) is not part of it. Steps marked
 * [upstream, from memory — unverified] restate VTK, whose source is not at hand: parity with VTK itself is
 * unpinned. The device (invesalius3_b200/csrc/raycasting.cu) follows this text bit for bit.
 *
 * Input: Slice.matrix, int16 m[dz][dy][dx], wrapped by to_vtk(matrix, spacing, 0, "AXIAL"): extent
 * (0, dx-1, 0, dy-1, 0, dz-1), origin 0, spacing (sx, sy, sz).
 *
 *  1. Flip (vtkImageFlip, SetFilteredAxis(1), FlipAboutOriginOn): f[z][y][x] = m[z][dy-1-y][x].
 *     [upstream, unverified] The output keeps the extent and the spacing; its origin becomes (0, -(dy-1) sy, 0).
 *  2. Range (GetScalarRange): (min, max) of the image as doubles; Volume.scale, read by the colour tables.
 *  3. Shift (vtkImageShiftScale, shift abs(min), scale 1, unsigned short output, no clamping):
 *     u = (uint16)((double)f + fabs(min)). When min > 0 the shift adds min (the reference's abs); every value
 *     lies in [0, 65534], so nothing overflows for int16. u is Volume.imagedata.GetOutput(), which __load_preset
 *     (:295-306) convolves again on every preset change.
 *  4. Convolution (vtkImageConvolve, SetKernel5x5(w), a 5x5x1 kernel), one pass per entry of the preset's
 *     convolutionFilters, in list order, each reading the previous pass's output (none: the result is u).
 *     Each slice z on its own, output unsigned short, the taps taken in kernel order (a correlation):
 *         sum = 0.0; k = 0;
 *         for b in 0..4, and within it a in 0..4: tap (y + b - 2, x + a - 2);
 *             if the tap lies inside the slice: sum += (double)u[z][y+b-2][x+a-2] * w[k]; k += 1;
 *         out = (uint16)sum, truncated.
 *     [upstream, unverified] VTK advances the kernel index only on in-bounds taps, so a voxel with n in-bounds
 *     taps (those within two voxels of the slice's edge) uses w[0..n-1], not the weights at those taps'
 *     positions. Only the two-voxel border of each slice depends on this rule.
 *     float64, no fused multiply-add. The weights: exactly 25, finite, none negative, and 65535 * sum(w) < 65536
 *     with sum(w) added in double in order; anything else is rejected. Every sum then lies in [0, 65536) up to
 *     the rounding of 25 non-negative terms, and the cast truncates it. A sum that this rounding carries to
 *     65536 or above gives 65535 here and on the device, where VTK's cast is undefined.
 *  5. Histogram (vtkImageAccumulate over the int16 image, component extent (0, r-1), origin min, spacing 1),
 *     r = int(max - min): counts[k] = #(m == min + k) for k < r. [upstream, unverified] Voxels equal to max fall
 *     outside the extent and are not counted; r == 0 (a constant image) gives no bins.
 *
 * orc_rc_flip_shift: u [dz][dy][dx], range {min, max}.
 * orc_rc_convolve: out [dz][dy][dx] (out != in); returns 0, or 1 on rejected weights.
 * orc_rc_range / orc_rc_histogram: range {min, max}; counts [r] for the given lo and r.
 */
#include <math.h>
#include <stdint.h>

void orc_rc_range(const int16_t* m, int64_t n, double* range) {
  int lo = 32767, hi = -32768;
  for (int64_t i = 0; i < n; ++i) {
    if (m[i] < lo) lo = m[i];
    if (m[i] > hi) hi = m[i];
  }
  range[0] = lo;
  range[1] = hi;
}

void orc_rc_flip_shift(const int16_t* m, int64_t dz, int64_t dy, int64_t dx, uint16_t* u, double* range) {
  orc_rc_range(m, dz * dy * dx, range);
  const double shift = fabs(range[0]);
  for (int64_t z = 0; z < dz; ++z)
    for (int64_t y = 0; y < dy; ++y)
      for (int64_t x = 0; x < dx; ++x)
        u[(z * dy + y) * dx + x] = (uint16_t)((double)m[(z * dy + (dy - 1 - y)) * dx + x] + shift);
}

int orc_rc_convolve(const uint16_t* in, int64_t dz, int64_t dy, int64_t dx, const double* w, uint16_t* out) {
  double total = 0.0;
  for (int k = 0; k < 25; ++k) {
    if (!isfinite(w[k]) || w[k] < 0.0) return 1;
    total += w[k];
  }
  if (!(65535.0 * total < 65536.0)) return 1;
  for (int64_t z = 0; z < dz; ++z) {
    const uint16_t* sl = in + z * dy * dx;
    for (int64_t y = 0; y < dy; ++y)
      for (int64_t x = 0; x < dx; ++x) {
        double sum = 0.0;
        int k = 0;
        for (int b = 0; b < 5; ++b)
          for (int a = 0; a < 5; ++a) {
            const int64_t yy = y + b - 2, xx = x + a - 2;
            if (yy >= 0 && yy < dy && xx >= 0 && xx < dx) {
              sum += (double)sl[yy * dx + xx] * w[k];
              k += 1;
            }
          }
        out[(z * dy + y) * dx + x] = sum < 65535.0 ? (uint16_t)sum : 65535;
      }
  }
  return 0;
}

void orc_rc_histogram(const int16_t* m, int64_t n, int lo, int64_t r, int64_t* counts) {
  for (int64_t k = 0; k < r; ++k) counts[k] = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t k = (int64_t)m[i] - lo;
    if (k >= 0 && k < r) counts[k] += 1;
  }
}
