/* b2v.h — C ABI of libb2v.so, the H100 (sm_90a) replacement for the
 * per-voxel hot path of InVesalius 3.
 *
 * Conventions (all entry points):
 *   - every pointer is a DEVICE pointer unless the parameter name ends in `_host`;
 *   - volumes are dense C-order [dz][dy][dx] (x fastest); strided / file-backed host
 *     views are packed by b2v_copy3d_* before the call;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - return value is a B2V_* status; b2v_last_error() gives the message of the
 *     last failure on the calling thread;
 *   - nothing is retained after return; scratch memory is supplied by the caller
 *     (query the size with the matching *_workspace_bytes function);
 *   - no entry point synchronises the stream unless documented.
 *
 * Each function cites the reference interface it replaces (paths relative to the
 * invesalius3 checkout).
 */
#ifndef B2V_H
#define B2V_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2V_OK 0
#define B2V_ERR_ARG 1      /* bad argument (shape, dtype code, axis, alignment) */
#define B2V_ERR_CUDA 2     /* CUDA runtime failure */
#define B2V_ERR_RANGE 3    /* value not representable (mirrors a Rust NumCast panic) */
#define B2V_ERR_NOCONV 4   /* iterative kernel hit its round cap */

/* element type codes (reference: invesalius_rs/src/types.rs:5-70) */
#define B2V_I16 0
#define B2V_U8 1
#define B2V_F64 2
/* B2V_F32 (3) is defined with b2v_zoom below; label images of count_regions also come as int32 / int64 */
#define B2V_I32 4
#define B2V_I64 5

/* projection kinds for b2v_mip */
#define B2V_MIP_MAX 0
#define B2V_MIP_MIN 1
#define B2V_MIP_MEAN 2

const char* b2v_last_error(void);
int b2v_version(void);
/* number of kernels launched by this library on the calling thread since the last reset */
int64_t b2v_launch_count(void);
void b2v_launch_count_reset(void);

/* ---- host<->device packing of strided views --------------------------------
 * Replaces the implicit stride handling of rust-numpy `as_array()` for callers that
 * pass `mask.matrix[1:,1:,1:]` (invesalius/data/styles.py:2493,2917,3157).
 * Copies a [dz][dy][dx] box of `elem` byte elements between a host view with byte
 * pitches (row_pitch, plane_pitch; x contiguous) and a dense device buffer. */
int b2v_copy3d_h2d(void* dst_dev, const void* src_host, int64_t dz, int64_t dy, int64_t dx, int64_t elem,
                   int64_t src_row_pitch, int64_t src_plane_pitch, void* stream);
int b2v_copy3d_d2h(void* dst_host, const void* src_dev, int64_t dz, int64_t dy, int64_t dx, int64_t elem,
                   int64_t dst_row_pitch, int64_t dst_plane_pitch, void* stream);

/* ---- threshold ---------------------------------------------------------------
 * Slice.SetMaskThreshold (whole-volume branch) invesalius/data/slice_.py:1238-1246:
 *     mask[v] = 255 if lo <= img[v] <= hi else 0               (preserve_markers = 0)
 * Slice.do_threshold_to_a_slice / do_threshold_to_all_slices slice_.py:1722-1769:
 *     same, except voxels whose OLD mask value is 1, 2, 253 or 254 keep it
 *                                                              (preserve_markers = 1)
 * img: int16 [n]; mask: uint8 [n] (read only when preserve_markers). Elementwise over
 * n voxels of a dense buffer. Algorithmic bytes: 3 B/voxel (4 with preservation). */
int b2v_threshold_i16(const int16_t* img, int64_t n, int32_t lo, int32_t hi, uint8_t* mask,
                      int preserve_markers, void* stream);
/* same on the padded Mask layout of invesalius/data/mask.py:422-431: mask has shape
 * [dz+1][dy+1][dx+1], voxel (z,y,x) at [z+1][y+1][x+1]; also sets the axial flag
 * mask[z+1][0][0] = 1 (slice_.py:1246,1767). When only_dirty != 0, slices whose flag is
 * already non-zero are skipped (slice_.py:1762-1763). */
int b2v_threshold_i16_masklayout(const int16_t* img, int64_t dz, int64_t dy, int64_t dx, int32_t lo, int32_t hi,
                                 uint8_t* mask_padded, int preserve_markers, int only_dirty, void* stream);

/* ---- intensity projections ---------------------------------------------------
 * NumPy reductions in Slice.get_image_slice, invesalius/data/slice_.py:881-886 /
 * 970-975 / 1057-1062: tmp_array.max(axis) / .min(axis) / .mean(axis).
 * img dense [dz][dy][dx] of dtype code `dtype` (int16 or uint8); axis 0/1/2.
 * out: same dtype for MAX/MIN, float64 for MEAN; shape [dy][dx] / [dz][dx] / [dz][dy].
 * workspace: b2v_mip_workspace_bytes() bytes (may be 0). 2 B/voxel for int16. */
int64_t b2v_mip_workspace_bytes(int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, int kind);
int b2v_mip(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, int kind, void* out,
            void* workspace, void* stream);

/* global min/max of a dense buffer as float32 (first step of MIDA,
 * invesalius_rs/src/mips.rs:113-122). minmax_out: float[2] on the device. */
int64_t b2v_minmax_workspace_bytes(int64_t n);
int b2v_minmax_f32(const void* img, int dtype, int64_t n, float* minmax_out, void* workspace, void* stream);

/* ---- seeded flood fill / region grow -------------------------------------------
 * invesalius_rs.floodfill_threshold(data, seeds, t0, t1, fill, strct, out)
 *   invesalius_rs/__init__.py:21-40 -> src/floodfill_py.rs:137-185 -> src/floodfill.rs:96-166
 * data: dense [dz][dy][dx] of dtype code `dtype`; out: uint8, same shape, read-write.
 * seeds_host: HOST array of nseeds (x, y, z) triples (int64). A seed is used only if
 * t0 <= data[seed] <= t1. Voxels of `out` already equal to `fill` are walls. Result: every
 * voxel reachable from the valid seeds gets out = fill; everything else is untouched.
 * strct_host: HOST uint8 [odz][ody][odx], each dim <= 3; offset of entry (kk,jj,ii) is
 * (kk - odz/2, jj - ody/2, ii - odx/2) as in floodfill.rs:110-112.
 * A seed outside the volume returns B2V_ERR_RANGE (the reference panics).
 * SYNCHRONISES the stream (round control reads one flag per batch of rounds).
 * rounds_out (optional, host): number of flood rounds launched.
 * Algorithmic bytes: 4 B/voxel (int16 data 2 + out read 1 + out write 1). */
int64_t b2v_floodfill_workspace_bytes(int64_t dz, int64_t dy, int64_t dx, int64_t nseeds);
/* Convergence engine of the flood-fill family: 1 (default) = every round inside ONE
 * persistent cooperative launch (rotating bitmaps of active tiles, grid-wide barrier per
 * round), 0 = one launch per round driven from the host. Same result either way.
 * Environment knob read once per process (tuning only, results identical): B2V_FF_GRID=n
 * (blocks of the persistent grid). */
void b2v_floodfill_set_engine(int persistent);
int b2v_floodfill_threshold(const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                            const int64_t* seeds_host, int64_t nseeds, double t0, double t1, uint8_t fill,
                            const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, uint8_t* out,
                            void* workspace, void* stream, int* rounds_out);
/* invesalius_rs.floodfill_threshold_inplace(data, seeds, t0, t1, fill, strct)
 *   __init__.py:43-54 -> floodfill_py.rs:187-231 -> floodfill.rs:168-237
 * Same walk, but `data` is both the tested and the written array (visited <=> data == fill). */
int b2v_floodfill_threshold_inplace(void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                    const int64_t* seeds_host, int64_t nseeds, double t0, double t1, double fill,
                                    const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx,
                                    void* workspace, void* stream, int* rounds_out);
/* invesalius_rs.floodfill(data, i, j, k, v, fill, out): floodfill_py.rs:87-135 -> floodfill.rs:5-49.
 * 6-connected walk over data == v starting at (x=i, y=j, z=k); the seed is marked
 * unconditionally. */
int b2v_floodfill_equal(const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx, int64_t i, int64_t j,
                        int64_t k, double v, uint8_t fill, uint8_t* out, void* workspace, void* stream,
                        int* rounds_out);
/* invesalius_rs.fill_holes_automatically(mask, labels, nlabels, max_size) -> bool
 *   floodfill_py.rs:233-249 -> floodfill.rs:51-94. mask uint8 [n] rw, labels uint32 [n].
 * modified_out (host) receives the bool. SYNCHRONISES the stream. 6 B/voxel. */
int64_t b2v_fill_holes_workspace_bytes(uint32_t nlabels);
/* In two stages for Z-sharded masks (labels of the WHOLE mask, mask.py:526-530): 1 = histogram
 * of this shard's labels into the workspace (uint32 [nlabels + 1] at byte offset 256; the shards
 * sum them with one all_reduce), 2 = qualify + apply + report. stages = 3 is b2v_fill_holes. */
int b2v_fill_holes_staged(int stages, uint8_t* mask, const uint32_t* labels, int64_t n, uint32_t nlabels,
                          uint32_t max_size, void* workspace, void* stream, int* modified_out);
int b2v_fill_holes(uint8_t* mask, const uint32_t* labels, int64_t n, uint32_t nlabels, uint32_t max_size,
                   void* workspace, void* stream, int* modified_out);

/* ---- ray-sequential projections -----------------------------------------------------
 * workspace for the three functions below: b2v_proj_workspace_bytes(dz*dy*dx) bytes.
 * All three SYNCHRONISE the stream (they report B2V_ERR_RANGE where the reference's
 * NumCast panics: NaN / out-of-range MIDA result, contour intensity overflowing T).
 * out shape: axis 0 -> [dy][dx], axis 1 -> [dz][dx], axis 2 -> [dz][dy].
 *
 * invesalius_rs.mida(image, axis, wl, ww, out): __init__.py:91-95 -> mips_py.rs:161-202 ->
 * mips.rs:102-168. dtype pairs (int16,int16), (uint8,uint8), (float64,uint8); anything else
 * is B2V_ERR_ARG ("Invalid image or output type"). wl / ww are taken AS THE IMAGE TYPE
 * (mips_py.rs:174-175). 4 B/voxel for int16 (min/max pass + ray pass). */
int64_t b2v_proj_workspace_bytes(int64_t n);
int b2v_mida(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double wl, double ww,
             void* out, int out_dtype, void* workspace, void* stream);
/* same, with the (min, max) pair of mips.rs:113-122 supplied by the caller as float[2] on
 * the device: a Z shard passes the all-reduced global pair (invesalius3_b200/dist.py). */
int b2v_mida_minmax(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double wl, double ww,
                    const float* minmax_dev, void* out, int out_dtype, void* workspace, void* stream);
/* lmip(image, axis, tmin, tmax, out): mips.rs:7-86 (called as mips.lmip by slice_.py:892,
 * 980,1063 although the crate forgets to export it). out has the image dtype. */
int b2v_lmip(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, double tmin, double tmax,
             void* out, void* workspace, void* stream);
/* invesalius_rs.fast_countour_mip(image, n, axis, wl, ww, tmip, out): __init__.py:98-101 ->
 * mips_py.rs:204-253 -> mips.rs:215-279. int16, uint8 or float64, out of the same dtype. tmip 0:
 * max, 1: lmip(700, 3033) (uint8: B2V_ERR_RANGE, the reference panics), 2: mida (float64:
 * B2V_ERR_ARG, not built). As in the reference the contour volume tmp[z, y, x] =
 * T(calc_fcm_intensity) (mips.rs:197-242) is materialised — b2v_fcm_volume, one stencil pass,
 * sizeof(T) read + sizeof(T) written per voxel — and then projected by the same kernels as the
 * plain projections. workspace: b2v_fcm_workspace_bytes (holds the contour volume).
 * b2v_fcm_volume alone (workspace: b2v_proj_workspace_bytes) serves the Z-sharded projections:
 * computed on an extended slab, its own planes are exact. */
int64_t b2v_fcm_workspace_bytes(int dtype, int64_t dz, int64_t dy, int64_t dx, int axis, int tmip);
int b2v_fcm_volume(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, float n, int axis, void* tmp,
                   void* workspace, void* stream);
int b2v_fast_countour_mip(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, float n, int axis,
                          double wl, double ww, int tmip, void* out, void* workspace, void* stream);

/* ---- context-aware mesh smoothing (SURVEY 8f-2) ------------------------------------------------
 * invesalius_rs.context_aware_smoothing(vertices, faces, normals, T, tmax, bmin, n_iters)
 * (mesh_py.rs -> mesh.rs:27-395; Mesh.ca_smoothing, invesalius_rs/__init__.py:220-249; caller
 * invesalius/data/surface_process.py:312-320). vertices float32 [V][3], smoothed in place; faces4
 * int64 [M][4] with the leading 3; normals float32 [M][3] (per face). order: int64 [4 M], the STABLE
 * ascending argsort of the 4 M face entries (any stable sort; the host wrapper uses torch.sort).
 * The reference's quirks are kept (every column of a face row counts as a vertex id in the
 * vertex->face map; the staircase test flags every vertex that has a face). workspace:
 * b2v_ca_smoothing_workspace_bytes. SYNCHRONISES. */
int64_t b2v_ca_smoothing_workspace_bytes(int64_t nverts, int64_t nfaces);
int b2v_ca_smoothing(float* vertices, int64_t nverts, const int64_t* faces4, int64_t nfaces, const float* normals,
                     const int64_t* order, double t, double tmax, double bmin, uint32_t n_iters, void* workspace,
                     void* stream);

/* ---- pre-filters and mask algebra (SURVEY 8f-4) -------------------------------------------------
 * b2v_boolean_op: Slice.do_boolean_op (invesalius/data/slice_.py:1906-1916) on two mask bodies:
 *   op 0 union, 1 difference, 2 intersection, 3 xor; selected <=> value > 2; out = 0 / 255.
 * b2v_convolve_non_zero: invesalius_rs.convolve_non_zero (transforms_py.rs:52-93; Slice.calc_mask_area,
 *   slice_.py:2299-2322): float64 volume and kernel (device), out[p] = sum over the kernel window
 *   (cval outside the volume) where volume[p] != 0, else 0; summed in the reference's loop order.
 * b2v_median_filter_i16: scipy.ndimage.median_filter(matrix, size) with size 3, 4 or 5, mode 'reflect'
 *   (filters.py:9-12). in != out.
 * b2v_uniform_filter_i16: scipy.ndimage.uniform_filter(matrix, size) on int16 (filters.py:15-18):
 *   three separable passes, each storing trunc(window sum / size) in int16 as SciPy does when the
 *   output array is int16. tmp: a third int16 volume. All bit-exact against SciPy. */
int b2v_boolean_op(const uint8_t* m1, const uint8_t* m2, int64_t n, int op, uint8_t* out, void* stream);
int b2v_convolve_non_zero(const double* volume, int64_t sz, int64_t sy, int64_t sx, const double* kernel_dev, int64_t skz,
                          int64_t sky, int64_t skx, double cval, double* out, void* stream);
int b2v_median_filter_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int16_t* out, void* stream);
int b2v_uniform_filter_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int16_t* out, int16_t* tmp,
                           void* stream);
/* The Gaussian-based filters of filters.py (gaussian_blur :5-6, sharpening :21-29, despeckle :32-36,
 * border detection :39-66) are built from scipy.ndimage.correlate1d evaluated exactly as SciPy's
 * NI_Correlate1D does for symmetric (symmetry = +1) and antisymmetric (-1) odd kernels: tmp = x[c] w[0];
 * for jj = -radius .. -1: tmp += (x[c + jj] +/- x[c - jj]) w[jj]; float64; 'reflect'; an int16 output
 * takes the C cast. weights_dev: 2 radius + 1 centred float64 weights on the device (for a Gaussian:
 * scipy.ndimage._filters._gaussian_kernel1d, reversed). dtype pairs (int16,int16), (int16,float64),
 * (float64,float64), (float32,float32) (the sum stays float64 and is rounded to float, as SciPy's line
 * buffer does). b2v_sharpen_i16, b2v_sobel_magnitude, b2v_rescale_cast_i16: the elementwise
 * float64 statements around them, in NumPy's order. Bit-exact against SciPy. */
int b2v_correlate1d(const void* in, int in_dtype, int64_t nz, int64_t ny, int64_t nx, int axis, const double* weights_dev,
                    int radius, int symmetry, void* out, int out_dtype, void* stream);
int b2v_sharpen_i16(const int16_t* img, const double* blurred, int64_t n, double value, double lo, double hi, int16_t* out,
                    void* stream);
int b2v_sobel_magnitude(double* sx_inout, const double* sy, const double* sz, int64_t n, void* stream);
int b2v_rescale_cast_i16(const double* m, int64_t n, int rescale, double mag_min, double mag_range, double span,
                         double min_val, int16_t* out, void* stream);
/* The 2-D filters of every slice along `axis` (0, 1 or 2) of a [nz][ny][nx] volume in one launch sequence, as
 * Slice.__apply_image_filter's "2D" branch (slice_.py:2363-2422) applies filters.py to each slice:
 * b2v_median_filter_slices_i16: median_filter of each slice with a size x size window (window 1 along
 *   `axis`, otherwise as b2v_median_filter_i16). in != out.
 * b2v_uniform_filter_slices_i16: uniform_filter of each slice: two int16 passes along the in-slice axes in
 *   ascending order, in -> tmp -> out. Three distinct volumes.
 * b2v_sobel_magnitude with sz == NULL: the two-term magnitude sqrt(sx**2 + sy**2) of a 2-D sobel.
 * b2v_slice_minmax: [min, max] of every slice as float64 pairs, minmax_out[2 s], minmax_out[2 s + 1] (device,
 *   2 * n_slices doubles); dtype B2V_I16 or B2V_F64 (no NaN). One reduction over the volume, no host sync.
 * b2v_sharpen_slices_i16, b2v_rescale_cast_slices_i16: b2v_sharpen_i16 / b2v_rescale_cast_i16 with each
 *   slice's own constants read from b2v_slice_minmax pairs on the device: the slice's image [min, max] as
 *   clip bounds; mag_min and mag_range = max - mag_min of the slice's magnitude, span and min_val from the
 *   slice's image pair, and a plain cast where the slice's mag_range is not > 0 (filters.py:60-66).
 * b2v_histogram_i16: np.histogram(a, bins, (lo, lo + bins))[0] for int16 a, 1 <= bins <= 65535: counts[k] =
 *   #(a == lo + k), the last bin also counting lo + bins, values outside [lo, lo + bins] not counted (the image
 *   histogram of Slice.matrix, slice_.py:190-192, 2490-2493, has lo = min, bins = max - min). counts: bins
 *   int64 on the device, overwritten. */
int b2v_median_filter_slices_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int axis, int16_t* out,
                                 void* stream);
int b2v_uniform_filter_slices_i16(const int16_t* in, int64_t nz, int64_t ny, int64_t nx, int size, int axis, int16_t* out,
                                  int16_t* tmp, void* stream);
int b2v_slice_minmax(const void* in, int dtype, int64_t nz, int64_t ny, int64_t nx, int axis, double* minmax_out,
                     void* stream);
int b2v_sharpen_slices_i16(const int16_t* img, const double* blurred, int64_t nz, int64_t ny, int64_t nx, int axis,
                           double value, const double* minmax_dev, int16_t* out, void* stream);
int b2v_rescale_cast_slices_i16(const double* m, int64_t nz, int64_t ny, int64_t nx, int axis, const double* mag_minmax_dev,
                                const double* img_minmax_dev, int16_t* out, void* stream);
int b2v_histogram_i16(const int16_t* a, int64_t n, int lo, int bins, int64_t* counts, void* stream);

/* ---- connected components (SURVEY 8f-3) ------------------------------------------------------
 * b2v_label: scipy.ndimage.label(input, structure, output=uint32) as InVesalius calls it
 * (invesalius/data/mask.py:526-530, 549-552; imagedata_utils.py:717-721): input uint8, non-zero =
 * feature; strct_host uint8, 1 or 3 wide per axis, centrosymmetric (else B2V_ERR_ARG, SciPy raises
 * too); labels uint32, numbered in raster order of each component's first voxel like SciPy.
 * *nlabels_host receives the count. SYNCHRONISES. workspace: b2v_label_workspace_bytes(n voxels).
 * b2v_count_regions: invesalius_rs.count_regions (count_regions.rs:5-18): out[p] = number of voxels
 * holding image[p]'s value; image dtype B2V_I16, B2V_U8, B2V_I32 or B2V_I64 (else B2V_ERR_ARG); values
 * outside [0, number_regions] are B2V_ERR_RANGE (the reference panics). SYNCHRONISES. workspace:
 * 256 + 4 * (number_regions + 1) bytes.
 * b2v_region_sizes: the size table of count_regions alone: sizes[v] = number of voxels holding v, for v in
 * [0, number_regions] (device uint32 [number_regions + 1]); same dtypes and errors. SYNCHRONISES.
 * workspace: 256 bytes.
 * Both add each run of equal values a warp reads with one atomic, so a dominant label (the background)
 * does not serialise the count. 64-bit indexing: n may exceed 2^31. */
int64_t b2v_label_workspace_bytes(int64_t n);
int b2v_label(const uint8_t* input, int64_t nz, int64_t ny, int64_t nx, const uint8_t* strct_host, int64_t odz, int64_t ody,
              int64_t odx, uint32_t* labels, void* workspace, void* stream, int64_t* nlabels_host);
int b2v_count_regions(const void* image, int dtype, int64_t n, uint32_t number_regions, uint32_t* out, void* workspace,
                      void* stream);
int b2v_region_sizes(const void* image, int dtype, int64_t n, uint32_t number_regions, uint32_t* sizes, void* workspace,
                     void* stream);

/* The "Remove tiny objects" plugin (plugins/remove_tiny_objects/gui.py:36-62, 134-144) over a resident label
 * image: labels uint32 [dz][dy][dx] (b2v_label's output) and its size table sizes uint32 [nsizes]
 * (b2v_region_sizes). A voxel is tiny where sizes[labels[p]] <= min_size, compared exactly as int64 (a
 * negative min_size selects nothing); a label >= nsizes is never tiny. nsizes: 0 .. 2^32. None of the three
 * synchronises; all index in 64 bits.
 *   b2v_tiny_objects_preview        out[p] = tiny ? 255 : 0, out dense uint8 [n] (the plugin's preview,
 *                                   `(counts <= min_size) * 255`). 4 B read + 1 B written per voxel.
 *   b2v_tiny_objects_remove         mask[1 + z][1 + y][1 + x] = 1 where (z, y, x) is tiny, on the padded
 *                                   uint8 [dz + 1][dy + 1][dx + 1] mask layout, in place; the flag planes
 *                                   (z = 0, y = 0, x = 0) and the other body voxels are not written.
 *   b2v_tiny_objects_apply_preview  the same write where preview[p] > 127, preview dense uint8 [dz][dy][dx]
 *                                   (OnRemove's `m[preview > 127] = 1`). */
int b2v_tiny_objects_preview(const uint32_t* labels, int64_t n, const uint32_t* sizes, int64_t nsizes, int64_t min_size,
                             uint8_t* out, void* stream);
int b2v_tiny_objects_remove(const uint32_t* labels, int64_t dz, int64_t dy, int64_t dx, const uint32_t* sizes,
                            int64_t nsizes, int64_t min_size, uint8_t* mask, void* stream);
int b2v_tiny_objects_apply_preview(const uint8_t* preview, int64_t dz, int64_t dy, int64_t dx, uint8_t* mask,
                                   void* stream);

/* Labelling of a Z-sharded volume (dist.label): every shard labels its own planes with b2v_label
 * (local labels 1..n_r); the provisional id of local label l on shard r is P = base_r + l, base_r the
 * sum of the lower shards' counts. These three stages turn provisional ids into SciPy's numbering of
 * the whole volume. Ids are int64, labels uint32.
 * b2v_label_boundary_count / _emit: the boundary between a shard and the next one. lo_plane = the
 *   lower shard's last plane of local labels (ids 1..n_lo), hi_plane = the upper shard's first plane
 *   (ids 1..n_hi), both [ny][nx]. Every foreground voxel below is paired with the foreground voxels
 *   above at the structure's z = +1 offsets (strct_host as for b2v_label); the pairs are reduced to a
 *   spanning forest in which the root of a set is its smallest id, and one pair (P, P(root)) is made for
 *   every label on the two planes that is not a root: at most one per distinct label. _count builds the
 *   forest and reports the pair count (SYNCHRONISES; 0 without building anything when the structure is 1
 *   wide along z); _emit writes the npairs pairs, int64 [npairs][2], in the order of each label's first
 *   voxel (lower plane first, raster order), with base_lo = the lower shard's base. Both calls share one
 *   workspace of b2v_label_boundary_workspace_bytes(ny, nx, n_lo, n_hi) bytes; only the labels on the
 *   two planes are touched in it. 2 ny nx < 2^31 and n_lo + n_hi < 2^31 - 1.
 * b2v_label_resolve: the pairs of every boundary, int64 [npairs][2], and ends = their distinct
 *   endpoints, sorted (int64 [nends]). Union-find over the endpoints, the larger root under the
 *   smaller; M = the endpoints that are not their set's root. Writes lut[l] = Final(base + l) for
 *   l in [0, nlocal] (lut[0] = 0), Final(P) = R - |{Q in M : Q < R}| with R = the root of P's set (P
 *   itself when it is no endpoint): the rank of the component's smallest provisional id among all
 *   components. *nmerged_host = |M|, so the volume holds sum(n_r) - |M| labels. SYNCHRONISES; an endpoint
 *   missing from ends is B2V_ERR_ARG. workspace: b2v_label_resolve_workspace_bytes(nends).
 * b2v_label_relabel: labels[i] = lut[labels[i]] over n labels (values >= nlut are left as they are). */
int64_t b2v_label_boundary_workspace_bytes(int64_t ny, int64_t nx, int64_t n_lo, int64_t n_hi);
int b2v_label_boundary_count(const uint32_t* lo_plane, const uint32_t* hi_plane, int64_t ny, int64_t nx,
                             const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, int64_t n_lo, int64_t n_hi,
                             void* workspace, void* stream, int64_t* npairs_host);
int b2v_label_boundary_emit(const uint32_t* lo_plane, const uint32_t* hi_plane, int64_t ny, int64_t nx, int64_t n_lo,
                            int64_t n_hi, int64_t base_lo, int64_t npairs, int64_t* pairs, void* workspace, void* stream);
int64_t b2v_label_resolve_workspace_bytes(int64_t nends);
int b2v_label_resolve(const int64_t* pairs, int64_t npairs, const int64_t* ends, int64_t nends, int64_t base,
                      int64_t nlocal, uint32_t* lut, void* workspace, void* stream, int64_t* nmerged_host);
int b2v_label_relabel(uint32_t* labels, int64_t n, const uint32_t* lut, int64_t nlut, void* stream);

/* ---- view-matrix resampling (SURVEY 8f-1) --------------------------------------------
 * invesalius_rs.apply_view_matrix_transform(volume, spacing, M, n, orientation, minterpol, cval,
 * out): __init__.py:84 -> transforms_py.rs:96-148 -> transforms.rs:9-55 -> interpolation.rs.
 * out[cz, cy, cx] samples `volume` at M * (z sz, y sy, x sx, 1) with (z, y, x) = the output
 * index shifted by n along the slab axis (orientation 0 AXIAL: z, 1 CORONAL: y, 2 SAGITAL: x,
 * anything else: no shift); minterpol 0 nearest, 1 trilinear, 2 tricubic, else Lanczos-4; outside
 * [0, d - 1) on any axis: cval. float64 arithmetic in the reference's order. spacing_host =
 * (sx, sy, sz), m_host = 16 doubles row-major, both on the HOST. volume / out: dense device
 * arrays of the same dtype (int16, uint8, float64). workspace: >= 256 bytes. SYNCHRONISES (a value
 * that does not fit the output type is B2V_ERR_RANGE: the reference panics; so is a Lanczos-4 sample
 * in range on an axis of 2 voxels, whose tap floor(f) - 3 stays outside after the one-step wrap,
 * where the reference's index panics: nothing is read outside the volume). */
int b2v_apply_view_matrix_transform(const void* volume, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                    const double* spacing_host, const double* m_host, int64_t n, int orientation,
                                    int minterpol, double cval, void* out, int64_t odz, int64_t ody, int64_t odx,
                                    void* workspace, void* stream);

/* ---- 3-D mask editor --------------------------------------------------------------------------
 * The three crate functions behind invesalius/data/mask3d_editor_state.py:14. float64 in the
 * reference's order; integer conversions as the crate's release build performs them.
 * b2v_polygon2mask: invesalius_rs.polygon2mask_rs((w, h), polygon) (polygon_mask_py.rs:7-27 ->
 *   polygon_mask.rs:4-79). polygon_host: n (x, y) float64 pairs on the HOST; out: dense [w][h] uint8,
 *   1 inside and 0 outside (cell [r][c] is the screen point (r, c)); only the polygon's bounding box,
 *   widened by one cell, is tested by the even-odd ray cast, every other cell is 0. A non-finite
 *   vertex is B2V_ERR_ARG. workspace: >= 16 n bytes on the device.
 * b2v_mask_cut: invesalius_rs.mask_cut(image, sx, sy, sz, max_depth, mask, M, MV, out, edit_mode)
 *   (mask_cut_py.rs:8-69 -> mask_cut.rs:7-62). out: dense [dz][dy][dx] uint8, 16-byte aligned, edited in
 *   place: a voxel > 127 at p = (x sx, y sy, z sz, 1) becomes 0 when M p has w > 0, |MV p / (MV p)_w|
 *   <= max_depth, and either it projects onto the viewport where filter is non-zero or it projects
 *   off the viewport and edit_mode == 0. filter: dense [h][w] uint8 (device). spacing_host = (sx, sy,
 *   sz), m_host / mv_host = 16 doubles row-major, all on the HOST. The image is not needed.
 * b2v_brush_mask_box: the brush's voxel box (brush_mask.rs:24-31) on the HOST: box_host = (z0, y0,
 *   x0, z1, y1, x1), inclusive; (0, 0, 0, -1, -1, -1) when empty. b2v_brush_mask computes the same box.
 * b2v_brush_mask: invesalius_rs.brush_mask_rs(out, orig, spacing, center, radius, edit_mode)
 *   (brush_mask_py.rs:7-28 -> brush_mask.rs:5-71) on a [dz][dy][dx] volume with center_host = (cx, cy,
 *   cz) in millimetres. out (and orig, or NULL) hold volume voxel (oz, oy, ox) at their first byte and
 *   voxel (z, y, x) at (z - oz) plane_pitch + (y - oy) row_pitch + (x - ox); they must cover the box.
 *   So the buffers may be the whole volume (origin 0) or a dense copy of just the box (origin z0, y0,
 *   x0). Mode 1 zeroes voxels > 0 inside the sphere; mode 0 copies orig > 0 into it (255 without
 *   orig); any other mode does nothing. */
int b2v_polygon2mask(const double* polygon_host, int64_t n, int64_t w, int64_t h, uint8_t* out, void* workspace,
                     void* stream);
int b2v_mask_cut(uint8_t* out, int64_t dz, int64_t dy, int64_t dx, const double* spacing_host, double max_depth,
                 const uint8_t* filter, int64_t h, int64_t w, const double* m_host, const double* mv_host, int edit_mode,
                 void* stream);
int b2v_brush_mask_box(int64_t dz, int64_t dy, int64_t dx, const double* spacing_host, const double* center_host,
                       double radius, int64_t* box_host);
int b2v_brush_mask(uint8_t* out, const uint8_t* orig, int64_t dz, int64_t dy, int64_t dx, int64_t oz, int64_t oy,
                   int64_t ox, int64_t row_pitch, int64_t plane_pitch, const double* spacing_host,
                   const double* center_host, double radius, int edit_mode, void* stream);

/* ---- region growing -----------------------------------------------------------------------------
 * The "Region growing" tool (invesalius/data/styles.py:2991-3251) and Slice.calc_image_density
 * (slice_.py:2284-2297).
 * b2v_lut255: get_LUT_value_255(data, window, level) (imagedata_utils.py:540-552) over n voxels of
 *   dtype B2V_I16 / B2V_U8 / B2V_F64; out has the input's dtype (integers truncate, as a C cast does).
 *   float64 arithmetic in NumPy's order; where the two conditions overlap (window <= 1) 255 wins.
 * b2v_masked_moments: count, min, max, np.mean and np.std (bit-identical: NumPy's pairwise summation
 *   order) of the image's voxels in the selection: sel[i] == sel_value (B2V_SEL_EQ) or sel[i] > 127
 *   (B2V_SEL_GT127) on a dense uint8 [dz][dy][dx] sel (or NULL: none), OR the voxel box box_host =
 *   (z0, y0, x0, z1, y1, x1) on the HOST, inclusive, clipped to the volume (or NULL: none). stats_host
 *   is written on the host; count 0 leaves min, max, mean and std NaN. Synchronises the stream.
 *   workspace: b2v_masked_moments_workspace_bytes(dz, dy, dx) bytes on the device. */
#define B2V_SEL_EQ 0
#define B2V_SEL_GT127 1
typedef struct b2v_moments {
  int64_t count;
  double min, max, mean, std;
} b2v_moments;
int b2v_lut255(const void* img, int dtype, int64_t n, double window, double level, void* out, void* stream);
int64_t b2v_masked_moments_workspace_bytes(int64_t dz, int64_t dy, int64_t dx);
int b2v_masked_moments(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, const uint8_t* sel, int sel_mode,
                       int sel_value, const int64_t* box_host, b2v_moments* stats_host, void* workspace, void* stream);

/* ---- spline resampling ------------------------------------------------------------------------------
 * b2v_zoom: scipy.ndimage.zoom(input, zoom, output, order, mode, cval) with prefilter=True and
 * grid_mode=False, as imagedata_utils.resize_image_array / resize_slice call it (order 2,
 * imagedata_utils.py:109-129; surface.py:1352-1353) and as the DICOM preview and the thumbnails do (order
 * 3, :132-139, :271-284). in: dense [nz][ny][nx] of in_dtype (B2V_I16, B2V_U8, B2V_F32, B2V_F64); ndim 2
 * for a 2-D image (passed with nz = out_nz = 1), 3 for a volume (SciPy's 3-D sum differs from the 2-D one
 * even where nz is 1). out: dense [out_nz][out_ny][out_nx] of out_dtype. order 0-3; orders 2 and 3 first
 * run SciPy's spline prefilter into the float64 workspace (b2v_zoom_workspace_bytes: 8 B per input voxel,
 * 0 for orders 0 and 1). Output index o samples o * (n_in - 1) / (n_out - 1) (1 when n_out is 1); taps past
 * an edge fold by mirror. mode B2V_ZOOM_CONSTANT: a coordinate that rounds past n_in - 1 writes cval
 * (SciPy's test is strict); B2V_ZOOM_MIRROR: it is interpolated. Integer outputs round half away from zero
 * and clip to their range; float outputs take the float64 value's cast. float64, SciPy's evaluation order:
 * bit-exact. Algorithmic bytes, orders 2 and 3: 3 reads + 2 writes of 8 B per voxel and axis (the z pass
 * reads the input dtype), then the gather (its taps mostly hit cache: ~8 B per input voxel read, out
 * written once). */
#define B2V_F32 3
#define B2V_ZOOM_CONSTANT 0
#define B2V_ZOOM_MIRROR 1
int64_t b2v_zoom_workspace_bytes(int64_t nz, int64_t ny, int64_t nx, int order);
int b2v_zoom(const void* in, int in_dtype, int ndim, int64_t nz, int64_t ny, int64_t nx, int64_t out_nz, int64_t out_ny,
             int64_t out_nx, int order, int mode, double cval, void* out, int out_dtype, void* workspace, void* stream);

/* b2v_shift: scipy.ndimage.shift(input, shift, output, order, mode, cval) with prefilter=True, the call behind
 * imagedata_utils.FixGantryTilt (imagedata_utils.py:28, :143-154). Arguments as b2v_zoom's, with the output of the
 * input's shape (out != in) and shift: host array of ndim float64 values in axis order. Output index o samples
 * input coordinate o - shift per axis. mode B2V_ZOOM_CONSTANT writes cval where a coordinate is below 0 or above
 * n - 1 (strict on both sides); B2V_ZOOM_MIRROR folds it as SciPy does. Workspace and algorithmic bytes as
 * b2v_zoom's at a factor of 1 (b2v_shift_workspace_bytes: 8 B per voxel for orders 2 and 3, else 0). Bit-exact. */
int64_t b2v_shift_workspace_bytes(int64_t nz, int64_t ny, int64_t nx, int order);
int b2v_shift(const void* in, int in_dtype, int ndim, int64_t nz, int64_t ny, int64_t nx, const double* shift,
              int order, int mode, double cval, void* out, int out_dtype, void* workspace, void* stream);

/* b2v_gantry_tilt: imagedata_utils.FixGantryTilt in place on a dense int16 [nz][ny][nx] device volume: slice n is
 * replaced by scipy.ndimage.shift(slice n, shifts[2n : 2n + 2], order=3, mode='constant', cval=matrix.min()), the
 * minimum taken over the volume as the sequential loop leaves it (shifted slices 0..n-1, original slices n..).
 * shifts: host array of nz (y, x) pairs, computed by the caller in the reference's float64 order. The slices are
 * interpolated together; the cvals come from a scan over per-slice minima (see zoom.cu). cvals: optional device
 * array of nz int16 that receives each slice's cval (NULL: not written). slab: slices per prefilter pass (0: as
 * many as fit 1 GiB of float64), so b2v_gantry_tilt_workspace_bytes is 8 B per voxel of one slab plus 32 B per
 * slice, not of the volume. Algorithmic bytes: 2 B per voxel read for the original slice minima; then per slab
 * 2 B + 3 x 8 B read and 2 x 8 B written by the y pass, 3 x 8 B read and 2 x 8 B written by the x pass, and the
 * gather's ~8 B read and 2 B written per voxel; the fill writes 2 B per out-of-range voxel. Bit-exact. */
int64_t b2v_gantry_tilt_workspace_bytes(int64_t nz, int64_t ny, int64_t nx, int64_t slab);
int b2v_gantry_tilt(int16_t* vol, int64_t nz, int64_t ny, int64_t nx, const double* shifts, int64_t slab,
                    void* workspace, int16_t* cvals, void* stream);

/* ---- porous scaffolds: Voronoi ---------------------------------------------------------------------
 * The "Voronoi" scaffolds of the porous-creation plugin (plugins/porous_creation/schwarzp.py:37-84).
 * b2v_jump_flooding: invesalius_rs.jump_flooding(distance_map, map_owners, sites, normalize)
 *   (floodfill_py.rs:262-276 -> floodfill.rs:298-507), in place on dense [dz][dy][dx] float32 distances and
 *   int32 owners. sites: dense int32 [n_sites][3] (z, y, x) on the device. Site i seeds owner i + 1 and
 *   distance 0 at its voxel (the last site naming a voxel wins; a negative or out-of-range site seeds
 *   nothing). Then floor(log2(max(dz, dy, dx))) Jacobi steps with per-axis offsets size / 2, halved after
 *   every step: each voxel takes the neighbour owner (1 .. n_sites) whose site is strictly nearer, in float32
 *   sqrt((dz dz + dy dy) + dx dx), or the first one when it has no owner (owner <= 0). normalize != 0 then
 *   replaces every distance of a voxel owned by 1 .. n_sites by its distance to the owner's truncated
 *   centroid over that site's largest such distance (when > 0). n_sites == 0 or an empty volume returns
 *   untouched. Shapes of more than 2^32 - 1 voxels with normalize (the crate's u32 per-site counts could
 *   wrap), more than 2^31 - 2 sites or dims beyond the grid are B2V_ERR_ARG. workspace:
 *   b2v_jump_flooding_workspace_bytes (a second owner and distance volume, 8 B per voxel, and 64 B per site).
 *   Algorithmic bytes per step: 16 B per voxel compulsory (owner and distance read and written) and 104 B
 *   gathered (26 neighbour owners); normalize adds 12 B per voxel.
 * b2v_voronoi_borders: mag > 0 of the owners' np.gradient (schwarzp.py:43-49): out[v] = 1.0f where the
 *   integer owner difference along any differentiated axis is non-zero (central in the interior, one-sided
 *   at the ends), else 0.0f. planar != 0: y and x only, dz must be 1 (the 2-D preview); planar == 0: all
 *   three axes. Every differentiated axis needs >= 2 voxels (NumPy raises otherwise): B2V_ERR_ARG.
 *   4 B read + 4 B written per voxel (the neighbours hit cache).
 * b2v_image_normalize_f32_i16: imagedata_utils.image_normalize(image, min_, max_) for a float32 image and an
 *   int16 output (imagedata_utils.py:580-587, plugins/porous_creation/gui.py:237): out = C cast of
 *   (in - imin) * (span / (imax - imin)) + min_f, all float32 (span = float32(max_ - min_), min_f =
 *   float32(min_), as NumPy promotes Python scalars against float32); `fill` everywhere when imin == imax.
 *   imin / imax: the image's minimum and maximum. 4 B read + 2 B written per voxel. */
int64_t b2v_jump_flooding_workspace_bytes(int64_t dz, int64_t dy, int64_t dx, int64_t n_sites);
int b2v_jump_flooding(float* distance_map, int32_t* map_owners, int64_t dz, int64_t dy, int64_t dx, const int32_t* sites,
                      int64_t n_sites, int normalize, void* workspace, void* stream);
int b2v_voronoi_borders(const int32_t* owners, int64_t dz, int64_t dy, int64_t dx, int planar, float* out, void* stream);
int b2v_image_normalize_f32_i16(const float* in, int64_t n, float imin, float imax, float span, float min_f,
                                int16_t fill, int16_t* out, void* stream);

/* ---- porous scaffolds: TPMS and Blobs ---------------------------------------------------------------
 * The other scaffolds of the porous-creation plugin (plugins/porous_creation/schwarzp.py:11-34, gui.py:117-245).
 * surface: the triply periodic minimal surfaces in the plugin's combo order (B2V_TPMS_*). tables: dense float64
 *   [cos_x (nx) | sin_x (nx) | cos_y (ny) | sin_y (ny) | cos_z (nz) | sin_z (nz)] on the device, NumPy's cos / sin
 *   of the np.ogrid axes. Per voxel (z, y, x), with cx = cos_x[x], snx = sin_x[x] and so on, each product and sum
 *   rounded on its own in this order (NumPy's broadcast evaluation of create_schwarzp, bit for bit):
 *     P           (cx + cy) + cz
 *     D           (((snx sny) snz + (snx cy) cz) + (cx sny) cz) + (cx cy) snz
 *     Gyroid      (cx sny + cy snz) + cz snx
 *     Neovius     3 ((cx + cy) + cz) + ((4 cx) cy) cz
 *     iWP         ((cx cy + cy cz) + cz cx) - (cx cy) cz
 *     P_W_Hybrid  (4 ((cx cy + cy cz) + cz cx) - ((3 cx) cy) cz) + 2.4
 * b2v_tpms_f64: the float64 field into dense out [nz][ny][nx]. 8 B written per voxel.
 * b2v_tpms_i16: image_normalize(field, min_, max_) into dense int16 out, without storing the field: one launch
 *   evaluates it and reduces it to (imin, imax) (NaN-propagating, as NumPy's min / max), a second evaluates it
 *   again and stores the C cast of (v - imin) * (span / (imax - imin)) + min_f in float64, or `fill` everywhere
 *   when imin == imax. span = float64(max_ - min_), min_f = float64(min_). workspace:
 *   b2v_tpms_i16_workspace_bytes; after the call its first 16 bytes hold (imin, imax) as float64. 2 B written per
 *   voxel.
 * b2v_image_normalize_f64_i16: the same two passes over a dense float64 device array of n elements
 *   (imagedata_utils.py:580-587 for a float64 image): 2 x 8 B read + 2 B written per element. workspace:
 *   b2v_image_normalize_f64_workspace_bytes, (imin, imax) in its first 16 bytes after the call.
 * Empty shapes return B2V_OK untouched; negative sizes, null pointers and unknown surfaces are B2V_ERR_ARG. */
#define B2V_TPMS_SCHWARZ_P 0
#define B2V_TPMS_SCHWARZ_D 1
#define B2V_TPMS_GYROID 2
#define B2V_TPMS_NEOVIUS 3
#define B2V_TPMS_IWP 4
#define B2V_TPMS_P_W_HYBRID 5
int b2v_tpms_f64(const double* tables, int64_t nz, int64_t ny, int64_t nx, int surface, double* out, void* stream);
int64_t b2v_tpms_i16_workspace_bytes(int64_t nz, int64_t ny, int64_t nx);
int b2v_tpms_i16(const double* tables, int64_t nz, int64_t ny, int64_t nx, int surface, double span, double min_f,
                 int16_t fill, void* workspace, int16_t* out, void* stream);
int64_t b2v_image_normalize_f64_workspace_bytes(int64_t n);
int b2v_image_normalize_f64_i16(const double* in, int64_t n, double span, double min_f, int16_t fill, void* workspace,
                                int16_t* out, void* stream);

/* ---- binary morphology ---------------------------------------------------------------------------
 * b2v_binary_morphology: scipy.ndimage.binary_erosion(border_value=True) / binary_dilation(border_value=False)
 *   with the Euclidean footprint {d : |d|^2 <= radius^2}: skimage's disk(radius) on every z-slice alone
 *   (planar != 0) or ball(radius) on the volume (planar == 0), as the mask-morphology plugin applies them
 *   (plugins/mask_morphology/gui.py:98-175). in: dense uint8 [dz][dy][dx]; a voxel is set where in > threshold.
 *   out: dense uint8 [dz][dy][dx] (not aliasing in), set_value where the result is set, else 0. counts: device
 *   int64[2], overwritten with the set voxels of the input and of the result. radius 0 (the identity) .. 15;
 *   anything else, or an op other than B2V_MORPH_ERODE / B2V_MORPH_DILATE, is B2V_ERR_ARG. workspace:
 *   b2v_binary_morphology_workspace_bytes (planar: 0; volumetric: one byte per voxel with rows padded to a
 *   multiple of 4). Exact integer arithmetic: the bounded squared distance to the nearest source voxel is
 *   taken one axis at a time. Algorithmic bytes: planar 2 B per voxel (in read, out written); volumetric 4 B
 *   (in, the workspace written and read, out). */
#define B2V_MORPH_ERODE 0
#define B2V_MORPH_DILATE 1
int64_t b2v_binary_morphology_workspace_bytes(int64_t dz, int64_t dy, int64_t dx, int planar);
int b2v_binary_morphology(const uint8_t* in, int64_t dz, int64_t dy, int64_t dx, uint8_t threshold, int op, int radius,
                          int planar, uint8_t set_value, uint8_t* out, int64_t* counts, void* workspace, void* stream);

/* ---- remove non-visible faces --------------------------------------------------------------------
 * plugins/remove_non_visible_faces/remove_non_visible_faces.py:19-119 on arrays, without OpenGL: the
 * surface is depth-rendered at 800x800 from each camera, a vertex is visible when some view sees it
 * (vtkSelectVisiblePoints, tolerance 0.01), a face is kept when any vertex is selected (the visible ones,
 * or the invisible ones with remove_visible != 0), and the kept faces are cleaned as vtkCleanPolyData
 * does (exactly coincident points merged, the first use wins; vertices numbered in order of first use
 * over the kept faces' corners; faces degenerate after the merge dropped). VTK's camera and clipping
 * constants are restated, not verified against VTK; all arithmetic is float64 without FMA.
 *   verts: float32 [nv][3] (1 <= nv < 2^31, finite); faces: int32 (faces_i64 = 0) or int64 [nt][face_cols],
 *   face_cols 3, or 4 with a leading 3 in every row; views: 1..64.
 *   b2v_visibility_bounds   vertex bounds (xmin, xmax, ymin, ymax, zmin, zmax) to bounds_host, -0 read
 *                           as +0; B2V_ERR_ARG on a non-finite vertex. Synchronises the stream.
 *   b2v_visibility_cameras  host only: for each direction of positions_host [nviews][3] (zero: ERR_ARG),
 *                           B2V_VIS_CAMERA_DOUBLES doubles: [0..15] the composite projection (row-major,
 *                           depth in [0, 1]), [16..18] position, [19..21] focal point, [22..24] view-up,
 *                           [25..26] clipping range, [27] camera distance, [28] bounding radius.
 *   b2v_visibility_count    renders, selects and counts the output (V', T'); ERR_ARG on a bad face.
 *                           Synchronises the stream. The workspace then holds what b2v_visibility_layout
 *                           locates: [0] byte offset of the float64 depth buffers [views][800 (y)][800 (x)],
 *                           [1] of the uint8 per-vertex visibility, [2] of the uint64 count of triangles
 *                           drawn by the cooperative (large-triangle) path.
 *   b2v_visibility_emit     writes verts_out float32 [V'][3] and faces_out int32 [T'][3]; same arguments
 *                           and workspace as the count. */
#define B2V_VIS_CAMERA_DOUBLES 32
int64_t b2v_visibility_workspace_bytes(int64_t nv, int64_t nt, int nviews);
int b2v_visibility_layout(int64_t nv, int64_t nt, int nviews, int64_t* layout_out);
int b2v_visibility_bounds(const float* verts, int64_t nv, void* workspace, void* stream, double* bounds_host);
int b2v_visibility_cameras(const double* bounds_host, const double* positions_host, int nviews, double* cameras_host);
int b2v_visibility_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                         const double* cameras_host, int nviews, int remove_visible, void* workspace, void* stream,
                         int64_t* nverts_host, int64_t* nfaces_host);
int b2v_visibility_emit(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                        int nviews, int remove_visible, void* workspace, float* verts_out, int32_t* faces_out,
                        void* stream);

/* ---- clean and triangulate surfaces ---------------------------------------------------------------
 * vtkCleanPolyData at InVesalius's settings (tolerance 0, unused points removed, polys -> lines -> verts,
 * strips -> polys -> lines -> verts) and vtkTriangleFilter, on the polys and strips of a surface. The rules
 * (restated from VTK 9.3, unverified) are in the header of the C checker, clean.c.
 *   Each cell family (polys, strips) is conn, offs, n cells, nconn corners, form, i64: form 0 is VTK 9's
 *   offsets int64 [n + 1] + connectivity [nconn]; form 3 is faces [n][3] and form 4 faces [n][4] with a
 *   leading 3 (offs NULL, nconn = 3 n). Ids are int32 (i64 = 0) or int64. verts: float32 [nv][3], nv < 2^31.
 *   Malformed offsets and ids outside [0, nv) are B2V_ERR_ARG.
 *   b2v_clean_count    counts_host[7] = {points, verts, lines, polys, poly corners, strips, strip corners}.
 *                      Synchronises the stream.
 *   b2v_clean_emit     from the same workspace: points_out float32 [points][3] in order of first use,
 *                      point_ids_out int64 (their input points); vconn_out, lconn_out int64 (one and two
 *                      points a cell); poffs_out / soffs_out int64 [cells + 1] and pconn_out / sconn_out;
 *                      cell_ids_out int64: the input cell (polys numbered first, then strips) of every
 *                      output cell, in the order verts, lines, polys, strips.
 *   b2v_triangle_filter_count  counts_host[1] = {triangles}; polys of more than 3 points are clipped by
 *                      vtkPolygon's ear cut (a polygon it cannot finish gives fewer than n - 2). The workspace
 *                      query takes the cells and the polys' corners. Synchronises the stream.
 *   b2v_triangle_filter_emit   tris_out int64 [triangles][3]: the polys' triangles, then each strip's n - 2
 *                      in vtkTriangleStrip's alternating winding; cell_ids_out int64 [triangles]. */
int64_t b2v_clean_workspace_bytes(int64_t nv, int64_t ncells, int64_t ncorners);
int b2v_clean_count(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs, int64_t np, int64_t npconn,
                    int pform, int pi64, const void* sconn, const int64_t* soffs, int64_t ns, int64_t nsconn, int sform,
                    int si64, void* workspace, void* stream, int64_t* counts_host);
int b2v_clean_emit(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs, int64_t np, int64_t npconn,
                   int pform, int pi64, const void* sconn, const int64_t* soffs, int64_t ns, int64_t nsconn, int sform,
                   int si64, void* workspace, float* points_out, int64_t* point_ids_out, int64_t* vconn_out,
                   int64_t* lconn_out, int64_t* poffs_out, int64_t* pconn_out, int64_t* soffs_out, int64_t* sconn_out,
                   int64_t* cell_ids_out, void* stream);
int64_t b2v_triangle_filter_workspace_bytes(int64_t ncells, int64_t npoly_corners);
int b2v_triangle_filter_count(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs, int64_t np,
                              int64_t npconn, int pform, int pi64, const void* sconn, const int64_t* soffs, int64_t ns,
                              int64_t nsconn, int sform, int si64, void* workspace, void* stream, int64_t* counts_host);
int b2v_triangle_filter_emit(const float* verts, int64_t nv, const void* pconn, const int64_t* poffs, int64_t np,
                             int64_t npconn, int pform, int pi64, const void* sconn, const int64_t* soffs, int64_t ns,
                             int64_t nsconn, int sform, int si64, void* workspace, int64_t* tris_out,
                             int64_t* cell_ids_out, void* stream);

/* ---- surface connectivity ------------------------------------------------------------------------
 * vtkPolyDataConnectivityFilter on triangles, behind polydata_utils.SelectLargestPart, SplitDisconectedParts
 * and JoinSeedsParts (invesalius/data/polydata_utils.py:206-278; surface.py:319-411). The contract (VTK's
 * region numbering, wave order and PointMap, restated and unverified) is in DESIGN.md §3 and the header of
 * the C checker, connectivity.c.
 *   verts: float32 [nv][3]; faces: int32 (faces_i64 = 0) or int64 [nt][face_cols], face_cols 3, or 4 with a
 *   leading 3 in every row; nv, nt < 2^31. seeded = 0: every region (all-regions mode; seeds ignored);
 *   seeded = 1: one region grown from the point ids seeds_host[nseeds] (negative ids skipped, an id >= nv is
 *   B2V_ERR_ARG). A bad face is B2V_ERR_ARG.
 *   b2v_conn_count   runs the filter; counts_host[5] = {regions R, points numbered N, cells visited C,
 *                    the deepest region's wave count, the largest region (ties: the lowest number; -1 if
 *                    none)}. Synchronises the stream.
 *   b2v_conn_emit    from the same workspace: verts_out float32 [N][3] in PointMap order and point_ids
 *                    int32 [N] (their input ids); faces_out int32 [C][3] (corners through PointMap) and
 *                    cell_ids int32 [C]: the visited cells grouped by region, ascending id inside each;
 *                    point_offsets / cell_offsets int64 [R + 1]: region r owns the points
 *                    [point_offsets[r], point_offsets[r + 1]) and the faces [cell_offsets[r], cell_offsets[r+1]).
 *   b2v_conn_layout  byte offsets in the workspace, valid after the count: [0] int32 [nt] region of each cell
 *                    (-1: not visited), [1] int32 [nv] PointMap (-1: not numbered), [2] int32 [C] the visited
 *                    cells in wave order, [3] int32 [C] region-major, [4] int32 [3 nt] the point -> cell
 *                    links, [5] uint64 [nv + 1] their offsets. */
int64_t b2v_conn_workspace_bytes(int64_t nv, int64_t nt, int64_t nseeds);
int b2v_conn_layout(int64_t nv, int64_t nt, int64_t nseeds, int64_t* layout_out);
int b2v_conn_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                   int seeded, const int64_t* seeds_host, int64_t nseeds, void* workspace, void* stream,
                   int64_t* counts_host);
int b2v_conn_emit(const float* verts, int64_t nv, int64_t nt, int64_t nseeds, const int64_t* counts_host,
                  void* workspace, float* verts_out, int32_t* point_ids, int32_t* faces_out, int32_t* cell_ids,
                  int64_t* point_offsets, int64_t* cell_offsets, void* stream);

/* ---- surface smoothing ---------------------------------------------------------------------------
 * vtkSmoothPolyDataFilter (Laplacian, in place in ascending point id) on triangles, behind
 * polydata_utils.ApplySmoothFilter, surface.decimate_polydata and markers/surface_geometry. The contract
 * (VTK's edge analysis, vertex types, sweep order and early stop, restated and unverified) is in DESIGN.md §3
 * and the header of the C checker, smoothing.c. The result equals the sequential sweep bit for bit.
 *   verts: float32 [nv][3]; faces: int32 (faces_i64 = 0) or int64 [nt][face_cols], face_cols 3, or 4 with a
 *   leading 3 in every row; nv < 2^31, 6 nt < 2^32. A bad face is B2V_ERR_ARG.
 *   b2v_smooth_analyse  edge analysis, vertex types and edge lists, and the dependency levels of the sweep.
 *                       cos_feature / cos_edge: the cosines of the feature and edge angles.
 *                       bounds_host[6] = {xmin, xmax, ymin, ymax, zmin, zmax} of the points the faces use
 *                       (0 without faces); counts_host[3] = {movable points, levels, grid barriers}.
 *                       Synchronises the stream.
 *   b2v_smooth_run      from the same workspace: verts_out float32 [nv][3] = the smoothed points (verts is
 *                       not modified). The sweep stops after `iterations` iterations, or after the first
 *                       whose largest move is <= conv (an absolute distance). counts_host[3] = {iterations
 *                       done, steps (levels x iterations done), grid barriers}. Synchronises the stream.
 *   b2v_smooth_layout   byte offsets in the workspace, valid after the analysis: [0] int8 [nv] vertex types
 *                       (VTK's codes: 0 simple, 1 fixed, 2 feature edge, 3 boundary edge), [1] int32 [nv]
 *                       edge-list lengths, [2] uint64 [nv + 1] where each point's list starts in [3] int32
 *                       [6 nt], [4] int32 [movable] the movable points level by level, [5] uint64
 *                       [levels + 1] the level offsets. */
int64_t b2v_smooth_workspace_bytes(int64_t nv, int64_t nt);
int b2v_smooth_layout(int64_t nv, int64_t nt, int64_t* layout_out);
int b2v_smooth_analyse(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                       double cos_feature, double cos_edge, int feature_edge_smoothing, int boundary_smoothing,
                       void* workspace, void* stream, double* bounds_host, int64_t* counts_host);
int b2v_smooth_run(const float* verts, int64_t nv, int64_t nt, int64_t iterations, double relaxation, double conv,
                   void* workspace, float* verts_out, void* stream, int64_t* counts_host);

/* ---- surface hole filling -------------------------------------------------------------------------
 * vtkFillHolesFilter on triangles, behind polydata_utils.ApplySmoothFilter, surface_process's "Fill holes",
 * FillSurfaceHole and markers/surface_geometry. The contract (boundary lines, the loop tracing, the bounding-
 * sphere test and the ear-clipping rule, restated and unverified) is in DESIGN.md §3 and the header of the C
 * checker, fill_holes.c. The result equals the sequential filter bit for bit.
 *   verts: float32 [nv][3]; faces: int32 (faces_i64 = 0) or int64 [nt][face_cols], face_cols 3, or 4 with a
 *   leading 3 in every row; nv < 2^31, 6 nt < 2^31. A bad face is B2V_ERR_ARG.
 *   b2v_holes_count   finds, traces, sizes and triangulates the holes. hole_size: NaN is B2V_ERR_ARG, other
 *                     values are clamped to [0, FLT_MAX]. counts_host[3] = {boundary lines, loops, new
 *                     triangles}. Synchronises the stream.
 *   b2v_holes_emit    from the same workspace: faces_out [nt + new triangles][face_cols] in the input's dtype
 *                     and form, the input faces first; per loop, in the order of its first line: first_line
 *                     and npts (int64), radius (double) and status (int8: 0 filled, 1 failed, 2 too large).
 *                     Does not synchronise.
 *   b2v_holes_layout  byte offsets in the workspace, valid after the count: [0] int32 [lines][2] the boundary
 *                     lines, [1] int32 [points] the loops' points, loop after loop, [2] uint64 [loops] where
 *                     each loop starts in [1], [3] int32 [loops] its points. */
int64_t b2v_holes_workspace_bytes(int64_t nv, int64_t nt);
int b2v_holes_layout(int64_t nv, int64_t nt, int64_t* layout_out);
int b2v_holes_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                    double hole_size, void* workspace, void* stream, int64_t* counts_host);
int b2v_holes_emit(const void* faces, int64_t nv, int64_t nt, int face_cols, int faces_i64,
                   const int64_t* counts_host, void* workspace, void* faces_out, int64_t* first_line,
                   int64_t* npts, double* radius, int8_t* status, void* stream);

/* ---- surface normals, volume and area --------------------------------------------------------------------
 * vtkPolyDataNormals on triangles with consistency, splitting and non-manifold traversal on, and
 * vtkMassProperties' volume and area, behind every InVesalius surface (surface_process, surface.py,
 * viewer_volume, brainmesh_handler). The contract is restated in the C checker, normals.c; the result equals
 * the sequential filter bit for bit. verts float32 [nv][3]; faces int32 / int64 (faces_i64) [nt][face_cols],
 * face_cols 3, or 4 with a leading 3. A bad face or a NaN feature angle is B2V_ERR_ARG; the angle (degrees)
 * is clamped to [0, 180]. The workspace (b2v_normals_workspace_bytes) serves all three calls.
 *   b2v_normals_count   orders, orients (auto_orient != 0: VTK's leftmost-point seeds), computes the cell
 *                       normals and splits; synchronises. counts_host[4] = {regions, flips, new points,
 *                       waves}.
 *   b2v_normals_emit    from the same workspace: points_out float32 [nv + new][3], faces_out [nt][face_cols]
 *                       in the input's dtype and form, point_normals float32 [nv + new][3], cell_normals
 *                       float32 [nt][3]. Does not synchronise.
 *   b2v_mass_properties out_host[2] = {volume, area} (doubles, on the host); synchronises.
 *   b2v_normals_layout  byte offsets in the workspace: [0] uint8 [nt] 1 where a cell was reversed, [1] int32
 *                       cells in wave order, [2] float64 [nt][4] the mass terms of each triangle (area, then
 *                       the x, y, z projected-volume terms), [3] int8 [nt] its normal class. */
int64_t b2v_normals_workspace_bytes(int64_t nv, int64_t nt);
int b2v_normals_layout(int64_t nv, int64_t nt, int64_t* layout_out);
int b2v_normals_count(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                      double feature_angle, int auto_orient, void* workspace, void* stream, int64_t* counts_host);
int b2v_normals_emit(const float* verts, int64_t nv, int64_t nt, int face_cols, int faces_i64,
                     const int64_t* counts_host, void* workspace, float* points_out, void* faces_out,
                     float* point_normals, float* cell_normals, void* stream);
int b2v_mass_properties(const float* verts, int64_t nv, const void* faces, int64_t nt, int face_cols, int faces_i64,
                        void* workspace, void* stream, double* out_host);

/* ---- geodesic surface measurement -------------------------------------------------------------------------
 * The curved measurement of the 3-D viewer (measures.py:1202-1273): vtkPointLocator::FindClosestPoint and
 * vtkDijkstraGraphGeodesicPath on triangle cells. The contract is restated in the C checker, geodesic.c; the
 * distances equal the sequential Dijkstra bit for bit. verts float32 or float64 (verts_f64) [nv][3]; faces int32 /
 * int64 (faces_i64) [nt][face_cols], face_cols 3, or 4 with a leading 3. The workspace
 * (b2v_geodesic_workspace_bytes) holds the links and one distance field.
 *   b2v_geodesic_links      builds the point -> cell links and the bucket width; a bad face is B2V_ERR_ARG;
 *                           synchronises. Needs nt > 0.
 *   b2v_closest_points      picks float64 [np][3] (device) -> ids_out int64 [np] (device): the smallest
 *                           (distance^2, id); scratch: device float64 [np]. Does not synchronise.
 *   b2v_geodesic_distances  from start; end >= 0 stops once every point with d <= d[end] is final, end = -1
 *                           settles the whole component (GetCumulativeWeights). dist_out float64 [nv] (device,
 *                           may be NULL; +inf where unreached). stats_host[2] = {rounds, buckets}; synchronises.
 *   b2v_geodesic_trace      the path of the last distances from end back to start: ids_out int64 [<= nv] and
 *                           points_out float32 [<= nv][3] (device); counts_host[3] = {points, ambiguous steps,
 *                           unreached (0/1)}, lengths_host[2] = {the path's length, total_in plus it, summed
 *                           step by step}; synchronises. */
int64_t b2v_geodesic_workspace_bytes(int64_t nv, int64_t nt);
int b2v_geodesic_links(const void* verts, int64_t nv, int verts_f64, const void* faces, int64_t nt, int face_cols,
                       int faces_i64, void* workspace, void* stream);
int b2v_closest_points(const void* verts, int64_t nv, int verts_f64, const double* picks, int64_t np,
                       double* scratch, int64_t* ids_out, void* stream);
int b2v_geodesic_distances(const void* verts, int64_t nv, int verts_f64, int64_t nt, void* workspace, int64_t start,
                           int64_t end, double* dist_out, void* stream, int64_t* stats_host);
int b2v_geodesic_trace(const void* verts, int64_t nv, int verts_f64, int64_t nt, void* workspace, int64_t start,
                       int64_t end, double total_in, int64_t* ids_out, float* points_out, void* stream,
                       int64_t* counts_host, double* lengths_host);

/* ---- volume rendering: data preparation ---------------------------------------------------------------------
 * The arrays the 3-D volume rendering hands to VTK (Volume.LoadVolume, ApplyConvolution, volume.py:538-634).
 * The contract (vtkImageFlip, vtkImageShiftScale, vtkImageConvolve's boundary rule, restated and unverified) is
 * in the header of the C checker, raycasting.c; both results equal it bit for bit. Volumes dense [dz][dy][dx].
 *   b2v_raycast_flip_shift_i16  out[z][y][x] = (uint16)(in[z][dy-1-y][x] + |min|), min = minmax_dev[0], the
 *                               float pair b2v_minmax_f32 leaves on the device (no host round trip). in != out.
 *                               Algorithmic bytes: 4 B per voxel.
 *   b2v_vtk_convolve5x5_u16     one vtkImageConvolve pass with SetKernel5x5(weights_host): each slice on its own,
 *                               float64 sums in the kernel's order, truncated to uint16. weights_host: 25 doubles
 *                               on the HOST, passed to the kernel by value; a weight that is negative or not
 *                               finite, or 65535 * sum >= 65536, is B2V_ERR_ARG. in != out. Algorithmic bytes:
 *                               4 B per voxel; 25 float64 multiplies and 25 adds per voxel. */
int b2v_raycast_flip_shift_i16(const int16_t* in, int64_t dz, int64_t dy, int64_t dx, const float* minmax_dev,
                               uint16_t* out, void* stream);
int b2v_vtk_convolve5x5_u16(const uint16_t* in, int64_t dz, int64_t dy, int64_t dx, const double* weights_host,
                            uint16_t* out, void* stream);

/* ---- marching cubes ---------------------------------------------------------------
 * Replaces the contour step of create_surface_piece, invesalius/data/surface_process.py:
 * 156-186 (vtkImageFlip about the origin + vtkContourFilter at iso 127 on the uint8 mask,
 * or at tmin / tmax on the int16 image); geometry as converters.to_vtk, converters.py:34-101.
 * vol: dense [nz][ny][nx] uint8 or int16. inside(p) <=> vol[p] >= iso.
 * Two calls sharing one caller-owned workspace:
 *   b2v_mc_count  classifies, scans and returns the vertex / triangle counts (host);
 *                 SYNCHRONISES the stream.
 *   b2v_mc_emit   writes verts float32 [V][3] and tris int32 [T][3] (shared vertices).
 * Vertex (i + ox [+t], j + oy [+t], k + oz [+t]) * (sx, sy, sz), y negated when flip_y
 * (and the winding reversed, so normals keep pointing from inside to outside);
 * t = (iso - s0) / (s1 - s0) in float32. Canonical ordering: see DESIGN.md.
 * Algorithmic bytes: 1 B/voxel (uint8) or 2 B/voxel (int16) + 12 B per vertex + 12 B per
 * triangle. */
int64_t b2v_mc_workspace_bytes(int64_t nz, int64_t ny, int64_t nx);
int b2v_mc_count(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso, void* workspace,
                 void* stream, int64_t* nverts_host, int64_t* ntris_host);
int b2v_mc_emit(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso, const void* workspace,
                float sx, float sy, float sz, int32_t ox, int32_t oy, int32_t oz, int flip_y, float* verts,
                int32_t* tris, void* stream);

/* ---- watershed -------------------------------------------------------------------------
 * do_watershed, invesalius/data/watershed_process.py:19-60.
 * b2v_ws_lut_i16: get_LUT_value(image, ww, wl).astype('uint16'), invesalius/data/
 *   imagedata_utils.py:555-564 (float64 piecewise, truncated into int16, reinterpreted).
 * b2v_ws_shift_i16: (image - image.min()).astype('uint16') (watershed_process.py:50,55);
 *   workspace: b2v_ws_workspace_bytes.
 * b2v_ws_morph_gradient_u16: scipy.ndimage.morphological_gradient(pre, size=(sz,sy,sx)),
 *   mode 'reflect' (watershed_process.py:36,49). Bit-exact against SciPy.
 * b2v_ws_flood: mode 0 = scipy.ndimage.watershed_ift cost model (max |dI| along the path),
 *   mode 1 = skimage.segmentation.watershed cost model (max I along the path). markers
 *   int16 (0 = unlabeled); labels int16 out. Exact minimax costs; labels follow cost-optimal
 *   edges, ties resolved by hop count then smaller label (the reference's ties follow its
 *   queue order: see DESIGN.md section 6). ambiguous (uint8, optional, may be NULL): 1 where two
 *   different labels can reach the voxel along cost-optimal edges, i.e. where the reference's
 *   answer is an artefact of its queue order; everywhere else (0) the labelling IS the
 *   reference's, whatever its order. SYNCHRONISES the stream. strct_host: uint8, dims
 *   1 or 3. 14 B/voxel for the whole do_watershed as the reference defines it. */
int b2v_ws_lut_i16(const int16_t* img, int64_t n, double window, double level, uint16_t* out, void* stream);
int b2v_ws_shift_i16(const int16_t* img, int64_t n, uint16_t* out, void* workspace, void* stream);
int b2v_ws_morph_gradient_u16(const uint16_t* in, int64_t nz, int64_t ny, int64_t nx, int sz, int sy, int sx,
                              uint16_t* out, void* stream);
int64_t b2v_ws_workspace_bytes(int64_t nz, int64_t ny, int64_t nx);
int b2v_ws_flood(const uint16_t* img, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                 const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, int mode, int16_t* labels,
                 uint8_t* ambiguous, void* workspace, void* stream, int* rounds_out);

/* The flood in stages, for Z-sharded volumes (6-connected only; dist.watershed drives it). The slab
 * passed in is an extended slab: with frozen_lo / frozen_hi its first / last plane is a halo plane
 * that is never relaxed locally; b2v_ws_plane reads a plane (merge = 0) or merges a neighbour's
 * values into one (merge = 1: minimum of the costs / of the keys, join of the label sets; tiles
 * next to a voxel that changed are queued for the next *_CONVERGE; *changed_host = 1 if any did).
 * what = 0: uint32 costs (phase 1); what = 1: uint64 keys followed by uint32 label sets (phase 2);
 * plane buffers are device memory of b2v_ws_plane_bytes(ny, nx, what) bytes.
 * stages (bit mask, executed in this order): 1 INIT, 2 COST_CONVERGE, 4 LABEL_BEGIN (admissible
 * predecessors from the final costs), 8 LABEL_CONVERGE, 16 FINISH (labels + ambiguous mask out).
 * *rounds_io accumulates the rounds. Every *_CONVERGE synchronises the stream.
 * b2v_ws_shift_i16_with: (image - min).astype('uint16') with the minimum supplied on the device
 * (minmax_dev[0], float32: the global minimum of a sharded volume after its all_reduce). */
int b2v_ws_flood_staged(int stages, const uint16_t* img, const int16_t* markers, int64_t nz, int64_t ny, int64_t nx,
                        int mode, int frozen_lo, int frozen_hi, int16_t* labels, uint8_t* ambiguous, void* workspace,
                        void* stream, int* rounds_io);
int64_t b2v_ws_plane_bytes(int64_t ny, int64_t nx, int what);
int b2v_ws_plane(int merge, int what, int64_t nz, int64_t ny, int64_t nx, int mode, int frozen_lo, int frozen_hi,
                 int64_t z, void* plane, void* workspace, void* stream, int* changed_host);
int b2v_ws_shift_i16_with(const int16_t* img, int64_t n, const float* minmax_dev, uint16_t* out, void* stream);
/* diagnostics of the persistent engine: [0..2] phase-1 tile visits / sweep sets / visits that
 * changed something, [4..6] the same for phase 2, [3] visits that re-queued their own tile (not
 * settled within the sweep-set cap, either phase), [7] phase-2 runs on 32-bit keys stopped by the
 * 24-bit hop limit (and re-run on 64-bit keys); reset != 0 clears them */
int b2v_ws_stats(int* out8, int reset);

/* ---- Z-sharded volumes (one shard per GPU; invesalius3_b200/dist.py drives these) ---------
 * The reference's only decomposition is the Z-piece split of the surface step
 * (invesalius/data/surface.py:1360-1381: pieces of 20 slices + 1 overlap, stitched by
 * vtkAppendPolyData + vtkCleanPolyData, surface_process.py:229-268). Here every shard holds
 * a slab plus one halo plane per inner side.
 *
 * Flood fill in stages (bit 0 BEGIN: build + seeds, bit 1 CONVERGE: rounds from *round_io,
 * bit 2 FINISH: write). Between CONVERGE calls the caller exchanges the reached bits of the
 * shared planes with its neighbours (byte offsets from b2v_floodfill_layout: [0] passable
 * bits, [1] reached bits, [2] round flags (int32 each), [3] bytes per z-plane, [4] tiles,
 * [5] round capacity) and ORs them in with b2v_floodfill_merge_plane, which re-activates
 * the touched tiles for round `round` and raises flags[round]. */
int b2v_floodfill_threshold_staged(int stages, const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                   const int64_t* seeds_host, int64_t nseeds, double t0, double t1, uint8_t fill,
                                   const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, uint8_t* out,
                                   void* workspace, void* stream, int* round_io);
int b2v_floodfill_layout(int64_t dz, int64_t dy, int64_t dx, int64_t nseeds, int64_t* layout_out);
int b2v_floodfill_merge_plane(int64_t dz, int64_t dy, int64_t dx, int64_t nseeds, void* workspace, int64_t z,
                              const uint32_t* plane_bits, int round, void* stream);
/* Marching cubes on a slab whose last plane is shared with the next shard: that plane's
 * vertices are owned (numbered, emitted) by the next shard. b2v_mc_layout (layout_out[4]): [0]
 * byte offset of the dense plane-0 records {cx, cy, cz, vertex offset} in the workspace (filled
 * by b2v_mc_count_shard), [1] their size in bytes, [2] byte offset of the uint64 totals (V, T).
 * The emitting shard receives the next shard's plane-0 records and global
 * vertex base; concatenating the shards' outputs in rank order reproduces the single-GPU
 * output bit for bit (the boundary stitch). */
int b2v_mc_count_shard(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                       int skip_last_plane, void* workspace, void* stream, int64_t* nverts_host,
                       int64_t* ntris_host);
int b2v_mc_emit_shard(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                      const void* workspace, float sx, float sy, float sz, int32_t ox, int32_t oy, int32_t oz,
                      int flip_y, int skip_last_plane, int32_t vertex_base, const void* next_shard_plane0_records,
                      int32_t next_shard_vertex_base, float* verts, int32_t* tris, void* stream);
int b2v_mc_layout(int64_t nz, int64_t ny, int64_t nx, int64_t* layout_out);

/* ---- peer mailboxes: the NVLink exchange layer of the Z-sharded ops ------------------------------
 * Replaces the temp-file exchange between the reference's worker processes
 * (invesalius/data/surface.py:1360-1430 pieces -> surface_process.py:229-268 stitch;
 * invesalius/data/styles.py:2083-2108 watershed child). One process per GPU; every rank owns one
 * MAILBOX in its HBM (b2v_peer_alloc: cudaMalloc + cudaIpc export), maps every other rank's
 * (b2v_peer_open) and hands the array of the `world` base pointers (its own included, index =
 * rank) to the *_peer entry points. Ranks only WRITE into peers (stores over NVLink + a release
 * store of a signal word) and poll their own mailbox, with a time-out (B2V_ERR_NOCONV), so a
 * mismatched call sequence cannot hang a GPU. `epoch` is a job-wide counter >= 1 that every rank
 * advances identically: b2v_floodfill_threshold_peer reports how many epochs it consumed, the
 * other calls consume one. Layout and protocol: invesalius3_b200/csrc/peer.cuh.
 * b2v_peer_mailbox_bytes(dy, dx): size for shards whose planes are dy x dx voxels; the
 * `mailbox_plane_bytes` argument of the calls below is dy * ceil(dx / 32) * 4 of that link. */
int64_t b2v_peer_mailbox_bytes(int64_t dy, int64_t dx);
int b2v_peer_alloc(int64_t bytes, void** dev_ptr_out, uint8_t* handle_out /* [64] */);
int b2v_peer_open(const uint8_t* handle /* [64] */, void** dev_ptr_out);
int b2v_peer_close(void* mapped_ptr);
int b2v_peer_free(void* dev_ptr);
/* all ranks meet (consumes one epoch); the self-check of a new link. Synchronises the stream. */
int b2v_peer_barrier(int rank, int world, const void* const* mailboxes_host, int64_t mailbox_plane_bytes,
                     uint32_t epoch, void* stream);
/* invesalius_rs.floodfill_threshold over one Z shard with the boundary exchange FUSED into the
 * persistent flood kernel: data / out are the extended slab (own planes + one halo plane per
 * inner side, halo planes of data valid), seeds are local to it (a shard without seeds passes
 * nseeds = 0 and still takes part). After local convergence the kernel pushes the reached bits
 * of the two planes around each inner boundary into the neighbours' mailboxes, merges what they
 * pushed, all ranks agree whether anyone gained a bit, and the rounds resume — ONE launch per
 * GPU for the whole sharded flood, no host round trip. Synchronises the stream (verdict). */
int b2v_floodfill_threshold_peer(const void* data, int dtype, int64_t dz, int64_t dy, int64_t dx,
                                 const int64_t* seeds_host, int64_t nseeds, double t0, double t1, uint8_t fill,
                                 const uint8_t* strct_host, int64_t odz, int64_t ody, int64_t odx, uint8_t* out,
                                 void* workspace, void* stream, int rank, int world,
                                 const void* const* mailboxes_host, int64_t mailbox_plane_bytes, uint32_t epoch,
                                 int* rounds_out, int* epochs_used_out);
/* b2v_mc_count_shard + the exchange the stitch needs, in one stream-ordered sequence: every
 * rank's (V, T) lands in counts_host [world][2], and the upper neighbour's plane-0 records land
 * in this rank's mailbox at byte offset b2v_peer_mc_inbox_offset(plane_bytes, epoch) — pass that
 * device address as next_shard_plane0_records to b2v_mc_emit_shard. Synchronises the stream. */
int b2v_mc_count_shard_peer(const void* vol, int dtype, int64_t nz, int64_t ny, int64_t nx, double iso,
                            int skip_last_plane, void* workspace, void* stream, int rank, int world,
                            const void* const* mailboxes_host, int64_t mailbox_plane_bytes, uint32_t epoch,
                            int64_t* counts_host);
int64_t b2v_peer_mc_inbox_offset(int64_t mailbox_plane_bytes, uint32_t epoch);
/* MIDA (mips.rs:102-168) / LMIP (mips.rs:7-86) with rays along z over ONE Z shard: the rays
 * cross the shards, so each shard continues from the per-ray state its predecessor left and
 * hands its own on (the per-ray operation order is that of the whole-volume walk: bit-exact).
 * state: device uint32 [3][dy][dx] — MIDA: (fmax, alpha, colour) as float bits; LMIP: running
 * maximum (two words), then bit 0 "inside [tmin, tmax] seen", bit 1 "ray finished".
 * first != 0: this slab starts the rays (state is written, not read); last != 0: it ends
 * them and writes out [dy][dx] (otherwise out may be NULL). minmax_dev: device float[2], the
 * GLOBAL (min, max) of the volume. b2v_mida_z_partial synchronises the stream (range check). */
int b2v_mida_z_partial(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, double wl, double ww,
                       const float* minmax_dev, uint32_t* state, int first, int last, void* out, int out_dtype,
                       void* workspace, void* stream);
int b2v_lmip_z_partial(const void* img, int dtype, int64_t dz, int64_t dy, int64_t dx, double tmin, double tmax,
                       uint32_t* state, int first, int last, void* out, void* workspace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2V_H */
