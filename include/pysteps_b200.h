/*
 * pysteps_b200.h -- C ABI of libpysteps_b200.so (hand-written sm_90a CUDA).
 *
 * Drop-in boundary for the advection hot path of pySTEPS/pysteps (reference
 * v1.21.3).  pysteps is pure Python; the callables it exposes through
 *   pysteps/extrapolation/interface.py:107-145  (_extrapolation_methods / get_method)
 *   pysteps/motion/interface.py:36-111          (_methods / get_method)
 * are mirrored in Python by pysteps_b200.{extrapolation,motion}; every array
 * operation behind them is one of the entry points below, reached through
 * ctypes.  All functions return 0 on success or a non-zero code (a cudaError_t,
 * or a B200_E* code); b200_last_error() returns the message of the last
 * failure on the calling thread.
 *
 * Conventions
 *   - "device" pointers are CUDA device pointers on the current device,
 *     "host" pointers are ordinary host memory.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *     Device-pointer entry points only ENQUEUE work; they never synchronise.
 *   - images are row-major (m rows, n columns); vector fields are planar
 *     (2, m, n) with [0] = x / column component, [1] = y / row component, as in
 *     pysteps/motion/interface.py:11-19.
 *   - field dtype codes: B200_F32 / B200_F64 (storage of precip, velocity and
 *     outputs).  Trajectories (displacement) are always float64.
 */
#ifndef PYSTEPS_B200_H
#define PYSTEPS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Field dtype codes.  An entry point refuses any other code with B200_EINVAL, and names it in
 * b200_last_error(), before it does any device work (allocation, memset, copy or launch) and
 * before it returns early on empty input. */
#define B200_F32 0
#define B200_F64 1

#define B200_MODE_CONSTANT 0 /* scipy map_coordinates mode="constant" */
#define B200_MODE_NEAREST 1  /* scipy map_coordinates mode="nearest"  */

#define B200_LAYOUT_PLANAR 0      /* velocity (2,m,n) as in pysteps */
#define B200_LAYOUT_INTERLEAVED 1 /* velocity (m,n,2): what the kernels read */

#define B200_EINVAL 100001  /* bad argument */
#define B200_ENOTSUP 100002 /* unsupported option */

int b200_version(void);
const char *b200_last_error(void);
/* number of kernels this library has launched in this process (all threads) */
long long b200_launch_count(void);
/* number of SMs / device name of the current device (diagnostics) */
int b200_device_info(int *sm_count, int *cc_major, int *cc_minor, char *name, int name_len);

/* ------------------------------------------------------------------------
 * Semi-Lagrangian extrapolation
 * replaces pysteps/extrapolation/semilagrangian.py:181-232 (the leadtime loop:
 * interpolate_motion + map_coordinates warp), interp_order == 1.
 *
 *   precip      device (m,n) of precip_dtype, or NULL (displacement only)
 *   velocity    device (2,m,n) [B200_LAYOUT_PLANAR] or (m,n,2)
 *               [B200_LAYOUT_INTERLEAVED] of velocity_dtype
 *   xy_coords   device (2,m,n) float64, or NULL for the default pixel grid
 *               (semilagrangian.py:174-179)
 *   disp_prev   device (2,m,n) float64 or NULL (semilagrangian.py:200-207)
 *   tdiff       HOST array of T timestep differences (semilagrangian.py:165)
 *   vel_timestep, n_iter, outval, mode: as in the reference
 *   out         device (T,m,n) of precip_dtype, or NULL when precip is NULL
 *   disp_out    device (2,m,n) float64 or NULL
 * All arithmetic is float64 in the reference's operation order, whatever the
 * storage dtypes (scipy converts each tap to double too), so results are
 * bit-identical to the reference run on arrays of the same dtypes: trajectory,
 * integer tap indices and values; float32 outputs are the float64 value
 * rounded once, as scipy does.
 * ---------------------------------------------------------------------- */
int b200_sl_extrapolate(const void *precip, const void *velocity,
                        const double *xy_coords, const double *disp_prev,
                        const double *tdiff, int T, double vel_timestep,
                        int n_iter, double outval, int mode, int velocity_dtype,
                        int velocity_layout, int precip_dtype, int m, int n, void *out,
                        double *disp_out, void *stream);

/* Same for the output rows [row_begin, row_begin + row_count) only: precip, velocity and
 * xy_coords are full (m,n) frames, while disp_prev / out / disp_out are band shaped
 * ((2,row_count,n), (T,row_count,n), (2,row_count,n)).  A pixel's trajectory reads the fields
 * anywhere but writes only its own pixel, so a frame is partitioned over GPUs by output
 * bands with replicated inputs and no halo exchange (SURVEY.md section 8e, config[4]). */
int b200_sl_extrapolate_rows(const void *precip, const void *velocity,
                             const double *xy_coords, const double *disp_prev,
                             const double *tdiff, int T, double vel_timestep,
                             int n_iter, double outval, int mode, int velocity_dtype,
                             int velocity_layout, int precip_dtype, int m, int n,
                             int row_begin, int row_count, void *out, double *disp_out,
                             void *stream);

/* OPT-IN float32-tap variant of b200_sl_extrapolate_rows (no counterpart in the reference, whose
 * arithmetic is float64 throughout; the north star allows "a stated float32 tolerance (bit-exact
 * for the integer displacement indices)"): the trajectory stays float64, the fields are sampled from
 * float32 copies.  A per-pixel error bound certifies that every sample floors to the same tap indices
 * as the exact kernel; pixels that cannot be certified (near a cell boundary, the border, outside,
 * non-finite) are recomputed by the exact code inside the same launch.  Values: within float32
 * rounding of b200_sl_extrapolate_rows.  Restrictions: n_iter = 1, pixel-grid coordinates, a
 * precipitation field, T <= 32.  fallback_count (device uint64, optional, accumulated not reset):
 * number of recomputed pixels. */
int b200_sl_extrapolate_rows_f32(const void *precip, const void *velocity, const double *disp_prev,
                                 const double *tdiff, int T, double vel_timestep, double outval, int mode,
                                 int velocity_dtype, int velocity_layout, int precip_dtype, int m, int n,
                                 int row_begin, int row_count, void *out, double *disp_out,
                                 unsigned long long *fallback_count, void *stream);

/* Displacement field after EVERY leadtime, disp_steps (T, 2, row_count, n) float64: the
 * trajectory part of b200_sl_extrapolate_rows alone (semilagrangian.py:201-219), for samplers
 * other than the built-in order-1 warp (interp_order 0 and 2..5 below).  Same arithmetic as the fused
 * loop: the kernel is resumed once per leadtime. */
int b200_sl_trajectories(const void *velocity, const double *xy_coords, const double *disp_prev,
                         const double *tdiff, int T, double vel_timestep, int n_iter,
                         int velocity_dtype, int velocity_layout, int m, int n, int row_begin,
                         int row_count, double *disp_steps, void *stream);

/* interp_order 0 and 2..5 (semilagrangian.py:144-157,224-253; scipy.ndimage.map_coordinates with
 * prefilter).  b200_spline_prepare: coeffs (m+2p, n+2p) float64, p = 12 for order >= 2 with
 * B200_MODE_NEAREST and 0 otherwise = the field (non-finite values zeroed when zero_fill) edge
 * padded and, for order >= 2, run through scipy's B-spline prefilter.  poles (HOST array, order/2
 * entries) are the filter poles -- the doubles nearest to the exact values, e.g. sqrt(3)-2 for
 * order 3 -- and zpow_axis0/1 (HOST arrays) pole^(L-1) for MODE_CONSTANT ("mirror" boundary) or
 * pole^L for MODE_NEAREST ("reflect"), L the padded length of the axis, evaluated by the caller
 * with the host's pow so that it is the libm value scipy uses.  For order >= 2 also mask_min =
 * (precip > nanmin) and mask_finite as float64 0/1 (m, n).  stats = b200_field_stats of precip.
 * b200_spline_sample: out (T, row_count, n) of out_dtype, pixel (y, x) of leadtime t sampled at
 * xy + disp_steps[t] -- (order+1)^2 taps (mirrored / clamped) or the nearest tap (order 0) -- then,
 * for order >= 2, reset to nanmin / NaN where the order-1 warps of the masks fall below 0.5. */
int b200_spline_prepare(const void *precip, int precip_dtype, int m, int n, int order, int mode,
                        const double *stats, int zero_fill, const double *poles,
                        const double *zpow_axis0, const double *zpow_axis1, double *coeffs,
                        double *mask_min, double *mask_finite, void *stream);
int b200_spline_sample(const double *coeffs, int m, int n, int order, int mode,
                       const double *xy_coords, const double *disp_steps, int T, int row_begin,
                       int row_count, double outval, const double *mask_min,
                       const double *mask_finite, const double *stats, int out_dtype, void *out,
                       void *stream);

/* planar (2,m,n) -> interleaved (m,n,2) copy of an advection field, so that a
 * caller reusing one field for many calls pays the re-layout once
 * (b200_sl_extrapolate does it internally for B200_LAYOUT_PLANAR). */
int b200_sl_interleave_velocity(const void *velocity, int velocity_dtype, int m, int n,
                                void *out, void *stream);

/* pysteps/noise/motion.py:129-180 (initialize_bps :129-141, generate_bps :172-180) fused with
 * the call site pysteps/nowcasts/utils.py:448-451 `velocity + velocity_pert_gen[i](t)`:
 *   p = (a_par * V/|V| + a_perp * perp(V/|V|)) / vsf     at every grid node,
 * a_par = g_par(t)*eps_par, a_perp = g_perp(t)*eps_perp (host scalars).  velocity is planar
 * (2,m,n) of velocity_dtype; `what` selects the float64 output:
 *   B200_BPS_FIELD_INTERLEAVED  V + p as (m,n,2) -- what b200_sl_extrapolate takes with
 *                               B200_LAYOUT_INTERLEAVED; replaces a 64 MB host array and its
 *                               upload per member and time step
 *   B200_BPS_FIELD_PLANAR       V + p as (2,m,n)
 *   B200_BPS_PERTURBATION       p as (2,m,n)       (the value of generate_bps)
 *   B200_BPS_UNIT               V/|V| as (2,m,n)   (perturbator["V_par"]; a, b, vsf unused)
 * n_nonfinite (device, may be NULL) receives the number of non-finite output elements -- the
 * np.isfinite(velocity) check of extrapolation/semilagrangian.py:116-123 on the field the
 * reference would have been given -- without another pass over it. */
#define B200_BPS_FIELD_INTERLEAVED 0
#define B200_BPS_FIELD_PLANAR 1
#define B200_BPS_PERTURBATION 2
#define B200_BPS_UNIT 3
int b200_bps_perturb_velocity(const void *velocity, int velocity_dtype, int m, int n,
                              double a_par, double a_perp, double vsf, int what, double *out,
                              double *n_nonfinite, void *stream);

/* One lead time of EVERY ensemble member of this GPU (nowcasts/utils.py:440-458: per member a
 * single-step extrapolator call with its own BPS-perturbed motion field, precipitation field and
 * carried displacement) in one perturbation launch and one trajectory launch per 8 members.
 *   velocity   (2,m,n) planar base field (device);  pert_coefs  HOST, members x 2: the (a, b) =
 *              (g_par(t) eps_par, g_perp(t) eps_perp) of noise/motion.py:177-180 per member
 *   precip     (members,m,n);  disp_prev (members,2,m,n) or NULL at the first lead time
 *   out        (members,m,n) precip dtype;  disp_out (members,2,m,n)
 *   n_nonfinite (device, members doubles, may be NULL): non-finite elements of each perturbed field
 * Each member's results are those of b200_bps_perturb_velocity + b200_sl_extrapolate with
 * T = 1, n_iter = 1, bit for bit. */
int b200_sl_step_batched(const void *velocity, int velocity_dtype, int m, int n, int members,
                         const double *pert_coefs, double vsf, const void *precip, int precip_dtype,
                         const double *disp_prev, double tdiff, double vel_timestep, double outval,
                         int mode, void *out, double *disp_out, double *n_nonfinite, void *stream);

/* Same operation on HOST buffers: allocates device scratch from the stream
 * ordered pool, copies in, runs, copies out and synchronises.  This is the
 * call a non-Python binding (cgo / JNI / plain C) would make. */
int b200_sl_extrapolate_host(const void *precip, const void *velocity,
                             const double *xy_coords, const double *disp_prev,
                             const double *tdiff, int T, double vel_timestep,
                             int n_iter, double outval, int mode, int velocity_dtype,
                             int precip_dtype, int m, int n, void *out, double *disp_out);

/* Field statistics used by the input validation of the reference
 * (semilagrangian.py:112-123, 171-172).  `stats` is a device array of 4
 * doubles: [0] number of non-finite elements, [1] np.nanmin, [2] np.nanmax
 * (NaN when every element is NaN), [3] number of NaN elements. */
int b200_field_stats(const void *a, int field_dtype, int64_t count, double *stats,
                     void *stream);

/* dst[0..count) = value (float64) */
int b200_fill_f64(double *dst, int64_t count, double value, void *stream);


/* ------------------------------------------------------------------------
 * Dense Lucas-Kanade motion estimation
 * replaces the array work of pysteps/motion/lucaskanade.py:38-279 and the helpers
 * it calls.  pysteps delegates most of it to opencv-python / scipy; each entry
 * point names the reference call it stands for.  All pointers are device
 * pointers; images are (m,n) row-major.  "n_dev" arguments are optional device
 * pointers to an element count produced by an earlier stage (NULL: use the
 * capacity argument), so the chain runs without host round trips.
 * ---------------------------------------------------------------------- */

/* np.ma.masked_invalid + MaskedArray.min()/max()  (motion/lucaskanade.py:213-219):
 * mask_out = user_mask | !isfinite(img); stats[0..2] = min, max, count of unmasked. */
int b200_mask_invalid(const double *img, const uint8_t *user_mask, int m, int n,
                      uint8_t *mask_out, double *stats, void *stream);

/* pysteps/utils/images.py:27-86 morph_opening (cv2.morphologyEx MORPH_OPEN with the
 * 3x3 cross): pixels > *thr_dev removed by the opening are set to *min_dev (device scalars,
 * e.g. the stats of b200_mask_invalid). size must be 3. */
int b200_morph_opening(const double *img, const uint8_t *mask, int m, int n, int size,
                       const double *thr_dev, const double *min_dev, double *out, void *stream);

/* stats (12 doubles): min / max / count over unmasked pixels of all rows [0..2], of rows
 * >= 1 [3..5], of rows >= 2 [6..8]; [11] = number of pixels whose dilate x dilate buffered
 * mask (cv2.dilate, feature/shitomasi.py:131-139) is clear.  The row sets reproduce the
 * integer-indexing quirk of shitomasi.py:139 (see csrc/lk_dense.cu).  stats0 (optional) is
 * the output of b200_mask_invalid: when it shows no masked pixel the dilation is skipped. */
int b200_masked_minmax(const double *img, const uint8_t *mask, int m, int n, int dilate,
                       const double *stats0, double *stats, void *stream);

/* "scale between 0 and 255" + astype(uint8).  mode 0: tracking/lucaskanade.py:144-160;
 * mode 1: feature/shitomasi.py:131-151 (buffer_mask = dilate) with valid = buffered mask
 * clear.  stats = output of b200_masked_minmax, masked pixels take *fill_dev.
 * mode | B200_QUANTISE_F32: the frames were float32 at the API (img holds them widened): scale in
 * float32 arithmetic as NumPy does for a float32 array. */
#define B200_QUANTISE_F32 2
int b200_quantise_u8(const double *img, const uint8_t *mask, int m, int n, int mode, int dilate,
                     const double *stats, const double *fill_dev, uint8_t *out, uint8_t *valid,
                     void *stream);
/* The four stages above for one frame in three passes (mask + raw min; opening + statistics;
 * opening + both uint8 images), the opened float64 image never written to HBM: the stencil
 * passes stage (64+4) x (16+4) float64 halo tiles in shared memory with TMA
 * (cp.async.bulk.tensor.2d, two-deep mbarrier ring, persistent CTAs; csrc/lk_frontend.cu).
 * Results are those of b200_mask_invalid -> b200_morph_opening -> b200_masked_minmax ->
 * b200_quantise_u8 (mode 0 into q_track; mode 1 into q_det / valid when q_det is not NULL).
 * Needs an even n (16-byte rows for the copy engine) and buffer_mask <= 5. */
int b200_lk_frontend(const double *img, const uint8_t *user_mask, int m, int n, int size_opening,
                     int buffer_mask, int flags, uint8_t *mask, double *stats0, double *stats,
                     uint8_t *q_track, uint8_t *q_det, uint8_t *valid, void *stream);

/* cv::pyrDown (uint8, BORDER_REFLECT_101) and the int16 Scharr pair image of
 * cv::calcOpticalFlowPyrLK's pyramid (dst holds (Ix, Iy) interleaved). */
int b200_pyr_down_u8(const uint8_t *src, int h, int w, uint8_t *dst, void *stream);
int b200_scharr_i16(const uint8_t *src, int h, int w, int16_t *dst, void *stream);

/* cv::cornerMinEigenVal(q, blockSize=5, ksize=3) -> float32 (m,n), bit-identical to
 * opencv-python 4.13.0 (AVX-512 build). */
int b200_min_eig(const uint8_t *q, int m, int n, float *eig, void *stream);

/* cv::goodFeaturesToTrack selection on a minimum-eigenvalue map
 * (feature/shitomasi.py:153-162): out_xy (max_corners,2) float32 (x,y), *out_count.
 * Synchronises the stream once (the sort network is sized by the candidate count). */
int b200_good_features(const float *eig, const uint8_t *valid, int m, int n, int max_corners,
                       double quality_level, double min_distance, float *out_xy,
                       int *out_count, void *stream);

/* Pyramid levels the LK entry points hold: every level cv::buildOpticalFlowPyramid keeps for
 * a frame below 2^32 pixels (a 16th halving needs both sides above 2^16). */
#define B200_LK_MAX_LEVELS 16
/* Pyramid geometry of cv::buildOpticalFlowPyramid (HOST pointers, B200_LK_MAX_LEVELS entries
 * each).  max_level is not capped: a geometry deeper than B200_LK_MAX_LEVELS levels is refused
 * with B200_EINVAL. */
int b200_lk_pyramid_layout(int h, int w, int win_w, int win_h, int max_level, int *levels_out,
                           int64_t *offsets, int *hs, int *ws, int64_t *total_pixels);
/* Gaussian pyramid (levels contiguous) and, if deriv != NULL, its Scharr pyramid. */
int b200_lk_build_pyramid(const uint8_t *img, int h, int w, int win_w, int win_h, int max_level,
                          uint8_t *pyr, int16_t *deriv, void *stream);
/* cv::calcOpticalFlowPyrLK (tracking/lucaskanade.py:171), flags = 0: next_pts (npts,2)
 * float32, status (npts) uint8; bit-identical to opencv-python 4.13.0 for EVERY point, lost
 * ones included (NaN coordinates fail the window bounds test as in its x86 build; NaN payloads
 * are not part of the contract).  Windows of 1 .. 4096 pixels (cv2 itself wants both sides
 * above 2); max_count and epsilon as cv::TermCriteria leaves them after calcOpticalFlowPyrLK's
 * clamps (the caller applies them). */
int b200_lk_track(const uint8_t *pyrI, const uint8_t *pyrJ, const int16_t *derivI, int h, int w,
                  int win_w, int win_h, int max_level, int max_count, double epsilon,
                  double min_eig_thr, const float *prev_pts, int npts, const int *npts_dev,
                  float *next_pts, uint8_t *status, void *stream);
/* keep status == 1 rows (tracking/lucaskanade.py:174-181) and append xy = p0,
 * uv = p1 - p0 (float32 arithmetic, widened) to a float64 pool at *pool_count. */
int b200_lk_compact_tracks(const float *p0, const float *p1, const uint8_t *status,
                           const int *npts_dev, int npts_cap, double *pool_xy, double *pool_uv,
                           int *pool_count, int pool_cap, void *stream);

/* pysteps/utils/cleansing.py:124-249 detect_outliers(uv, thr, xy, k), multivariate local
 * branch: out[i] = 1 where the Mahalanobis distance to the k nearest vectors exceeds thr.  The
 * k+1 nearest vectors are taken in scipy.spatial.cKDTree's own order (cleansing.py:219-221), ties
 * and coincident vectors included: the tree is built and queried on the device exactly as scipy
 * does (csrc/knn.cu, knn_body.cuh) -- with integer corner coordinates that order decides tests. */
int b200_detect_outliers(const double *uv, const double *xy, const int *n_dev, int n_cap,
                         double thr, int k, uint8_t *out, void *stream);
/* scipy.spatial.cKDTree(xy) (leafsize 16, median splits by std::nth_element) built on the device:
 * tree_indices[n_cap] = tree.indices (the tree order of the points), *node_count = number of
 * nodes; both device pointers.  Stage entry used by the parity tests of the build. */
int b200_kdtree_build(const double *xy, const int *n_dev, int n_cap, int *tree_indices,
                      int *node_count, void *stream);
/* cleansing.py:201-214, the global branch (k is None): Mahalanobis distance of every vector to the
 * mean of ALL vectors under their sample covariance; out[i] = MD > thr. */
int b200_detect_outliers_global(const double *uv, const int *n_dev, int n_cap, double thr,
                                uint8_t *out, void *stream);
/* rows with drop == 0, order preserved */
int b200_compact_rows(const double *xy, const double *uv, const uint8_t *drop, const int *n_dev,
                      int n_cap, double *out_xy, double *out_uv, int *out_count, void *stream);
/* pysteps/utils/cleansing.py:21-121 decluster(xy, uv, scale, min_samples): per-cell medians,
 * cells in np.unique(axis=0) order.  n_cap <= 16384.  As in the reference, a row with a NaN
 * coordinate belongs to no cell and +-inf coordinates form their own cells (first / last).  Cells
 * floor(xy / scale) outside [1 - 2^24, 2^24 - 2], and NaN coordinates with min_samples < 1 (the
 * reference appends a NaN median for each), are refused on the device: *out_count = -1 and nothing
 * else is written. */
int b200_decluster(const double *xy, const double *uv, const int *n_dev, int n_cap, double scale,
                   int min_samples, double *out_xy, double *out_uv, int *out_count, void *stream);

/* pysteps/utils/interpolate.py:26-114 idwinterp2d: k-nearest inverse-distance weighting of
 * (npts, nvar) values onto the (ny, nx) grid -> out (nvar, ny, nx). k <= 32.  Exhaustive
 * tile-culled search; grid points whose k-th and (k+1)-th neighbours are exactly equidistant are
 * recomputed from scipy.spatial.cKDTree's query order (tree built on a library-internal side
 * stream), so the neighbour SET is the reference's everywhere (interpolate.py:78-81).
 * coords_on_16th_grid != 0 is the caller's promise that every vector and grid coordinate is
 * a multiple of 1/16 with magnitude < 2^14 (true for dense_lucaskanade: pixel grids and
 * medians of integer corners); it enables a faster, result-identical key packing.  The value 2
 * promises more: vectors on multiples of 1/2 and INTEGER grid coordinates -- the search then runs
 * on exact 32-bit integer keys. */
int b200_idw_fill(const double *xy, const double *vals, const int *npts_dev, int npts_cap,
                  int nvar, int k, double power, double dist_offset, double mean_res,
                  const double *xgrid, int nx, const double *ygrid, int ny,
                  int coords_on_16th_grid, double *out, void *stream);

/* What dense_lucaskanade decides about its declustered vectors before the interpolation
 * (lucaskanade.py:245-269, decorators.py:190-208), computed on the device so that the fill is
 * enqueued without a read-back.  48 bytes: the host copies it to pinned memory. */
typedef struct {
    int n_pool, n_kept, n_dec;  /* counts[0..2] of the sparse stage */
    int nonfinite;              /* bit 0: a value (uv) is not finite, bit 1: a coordinate (xy) */
    int mode;                   /* B200_IDW_ZERO / _CONSTANT / _INTERPOLATE / _REFUSED (non-finite input) */
    int on_grid;                /* the coords_on_16th_grid level b200_idw_fill would be promised: 0, 1, 2 */
    int n_fill;                 /* n_dec when mode == B200_IDW_INTERPOLATE, else 0 */
    int pad;
    double c0, c1;              /* the constant field (ZERO: 0, 0) */
} B200IdwPlan;
enum { B200_IDW_ZERO = 0, B200_IDW_CONSTANT = 1, B200_IDW_INTERPOLATE = 2, B200_IDW_REFUSED = 3 };

/* counts = the sparse stage's (pool, kept, declustered) counts, xy/uv = the (cap, 2) declustered
 * vectors.  Zero when no vector was pooled or declustered; constant (uv[0, :]) for one vector,
 * (uv[0, 0], uv[0, 0]) when every value is equal; refused when a value or coordinate is not
 * finite.  grid_ok != 0: every grid coordinate is an integer below 2^14 (on_grid may then be set). */
int b200_idw_plan(const int *counts, const double *xy, const double *uv, int cap, int grid_ok,
                  B200IdwPlan *plan, void *stream);
/* b200_idw_fill for two variables with the plan on the device: vector count and path (zero or
 * constant fill, 32-bit keys, packed or unpacked 64-bit keys) are taken from `plan` by the
 * kernels, nothing is read back.  Grids and scratch are sized from npts_cap.  Fills out (2, ny, nx)
 * and, when twin is not null, twin (ny, nx, 2) with the same values.  A refused plan writes nothing. */
int b200_idw_fill_planned(const double *xy, const double *vals, const B200IdwPlan *plan, int npts_cap,
                          int k, double power, double dist_offset, const double *xgrid, int nx,
                          const double *ygrid, int ny, double *out, double *twin, void *stream);

/* idwinterp2d with the k nearest vectors of every grid point found, ordered and weighted exactly
 * as the reference does it (scipy.spatial.cKDTree's query order, numpy's pairwise sum of the
 * weights, values accumulated in neighbour order): equal to the reference at EVERY grid point to
 * the last bits (np.power vs pow), ties included; much slower than b200_idw_fill (a tree search
 * per grid point; b200_idw_fill runs it only where the neighbour set depends on it).  k <= 128. */
int b200_idw_fill_ckdtree(const double *xy, const double *vals, const int *npts_dev, int npts_cap,
                          int nvar, int k, double power, double dist_offset, double mean_res,
                          const double *xgrid, int nx, const double *ygrid, int ny, double *out,
                          void *stream);
/* idwinterp2d with k = None (interpolate.py:82-88): every vector contributes to every grid point.
 * nvar <= 8. */
int b200_idw_fill_all(const double *xy, const double *vals, const int *npts_dev, int npts_cap, int nvar,
                      double power, double dist_offset, double mean_res, const double *xgrid, int nx,
                      const double *ygrid, int ny, double *out, void *stream);

/* ------------------------------------------------------------------------
 * Variational Echo Tracking -- replaces the native extension of the reference,
 * pysteps/motion/_vet.pyx.  The CG optimiser (scipy.optimize.minimize, vet.py:593-600)
 * stays on the host; every point it visits costs one b200_vet_value_and_gradient call.
 * Note the reference's axis naming: axis 0 of the images is "x", axis 1 is "y"
 * (_vet.pyx:129-130); sector_disp is (2, xs, ys), images are (nx, ny), mask is int8.
 * ---------------------------------------------------------------------- */

/* _vet.pyx:238-621 _cost_function.  gradient == 0: out[0] = residuals, out[1] =
 * smoothness penalty.  gradient != 0: out (2, xs, ys) = grad_residuals + grad_smooth.
 * smooth_gain is a C float in the reference (:242) and is one here. */
int b200_vet_cost(const double *sector_disp, const double *templ, const double *input,
                  const int8_t *mask, int xs, int ys, int nx, int ny, float smooth_gain,
                  int gradient, double *out, void *stream);
/* vet_cost_function AND vet_cost_function_gradient (vet.py:165-299) at the same point from one
 * pass over the images -- what a line search asks for.  x_host: sector displacements (2, xs, ys)
 * on the HOST; images (nframes, nx, ny) and mask (nx, ny) int8 on the device (2 or 3 frames: the
 * pairs of vet.py:257-268, summed in its order); work: device scratch of 6 * xs * ys + 4 doubles.
 * Returns value_host[0] = residuals, [1] = smoothness penalty (the cost is their sum) and
 * gradient_host (2, xs, ys).  Synchronises the stream (the optimiser needs the numbers). */
int b200_vet_value_and_gradient(const double *x_host, const double *images, int nframes,
                                const int8_t *mask, int xs, int ys, int nx, int ny,
                                float smooth_gain, double *work, double *value_host,
                                double *gradient_host, void *stream);
/* The image stack and mask of one minimisation level from the raw frames (vet.py:507-523 cleaning,
 * :510-517 the global `padding` frame, :548-561 the level's divisibility padding): images
 * (nframes, M, N) zero where a frame is invalid (user_mask set, or -- user_mask NULL -- not finite),
 * edge-replicated into the level padding; mask (M, N) int8 = any frame invalid | global padding
 * ring | level padding.  The level frame starts (pad_i_before, pad_j_before) before the globally
 * padded input. */
int b200_vet_level_images(const double *frames, const uint8_t *user_mask, int nframes, int m,
                          int n, int padding, int pad_i_before, int pad_j_before, int M, int N,
                          double *images, int8_t *mask, void *stream);
/* _vet.pyx:66-232 _warp (vet.morph, vet.py:93-153): out, out_mask (int8) and, if grad is
 * not NULL, the gradient (2, nx, ny). */
int b200_vet_warp(const double *image, const int8_t *mask, const double *displacement, int nx,
                  int ny, double *out, int8_t *out_mask, double *grad, void *stream);
/* scipy.ndimage.zoom(a (c,h,w), (1, oh/h, ow/w), order=1, mode="nearest") (vet.py:621-630) */
int b200_zoom_bilinear(const double *a, int c, int h, int w, int oh, int ow, double *out,
                       void *stream);

/* ------------------------------------------------------------------------
 * Proesmans et al. (1994) optical flow -- replaces the other native extension of the reference,
 * pysteps/motion/_proesmans.pyx (called from pysteps/motion/proesmans.py:88).
 * ---------------------------------------------------------------------- */

/* pysteps/motion/proesmans.py:79-83: out = (frames - im_min) / (im_max - im_min) * 255.0 when
 * do_scale, else a float64 copy. */
int b200_proesmans_scale(const void *frames, int dtype, int64_t count, double im_min, double im_max,
                         int do_scale, double *out, void *stream);
/* scipy.ndimage.gaussian_filter(in, sigma) of a float64 (h,w) image (proesmans.py:85-87): weights
 * (HOST array, 2*radius+1 entries) is scipy's normalised kernel exp(-0.5 x^2 / sigma^2), radius =
 * int(4 sigma + 0.5) <= 64; axis 0 then axis 1, "reflect" boundary, scipy's accumulation order. */
int b200_gaussian_filter(const double *in, int h, int w, const double *weights, int radius, double *out,
                         void *stream);
/* _proesmans.pyx:19-44 _compute_advection_field(R, lam, num_iter, n_levels): frames (2,m,n)
 * float64 -> advfield (2,2,m,n) (forward / backward flow, x / y component) and quality (2,m,n)
 * (the consistency maps).  The relaxation sweep keeps the reference's raster-order Gauss-Seidel
 * update order (wavefronts t = x + 2y inside one CTA per flow field). */
int b200_proesmans_field(const double *frames, int m, int n, double lam, int num_iter, int num_levels,
                         double *advfield, double *quality, void *stream);

/* ------------------------------------------------------------------------
 * Constant advection field (pysteps/motion/constant.py:41-49): the objective that
 * scipy.optimize.minimize (Nelder-Mead, on the host) evaluates at every point it visits,
 *   f(v) = -corrcoef(next[mask], warped[mask])[0, 1]
 *   warped = map_coordinates(prev, [Y + vy, X + vx], order=0, mode="constant", cval=nan)
 *   mask   = isfinite(next) & isfinite(warped)
 * ---------------------------------------------------------------------- */

/* bits of record[2]: the floating-point events of NumPy's corrcoef tail, in its order */
#define B200_CONST_EMPTY 1         /* N == 0: "Mean of empty slice." and 0/0 in the mean */
#define B200_CONST_DOF 2           /* N - 1 <= 0: "Degrees of freedom <= 0 for slice" and 1/0.0 */
#define B200_CONST_SCALE_INVALID 4 /* c *= 1/fact: 0 * inf */
#define B200_CONST_ROW_INVALID 8   /* c /= stddev[:, None]: invalid, divide by zero, overflow */
#define B200_CONST_ROW_DIVZERO 16
#define B200_CONST_ROW_OVERFLOW 32
#define B200_CONST_COL_INVALID 64  /* c /= stddev[None, :] */
#define B200_CONST_COL_DIVZERO 128
#define B200_CONST_COL_OVERFLOW 256
#define B200_CONST_SUM_BLOCKS 256  /* the centred sums: 256 CTAs x 256 threads, element i on lane i % 65536 */

/* Bytes of device scratch b200_constant_eval needs for an (m, n) frame (written to *bytes, a host
 * pointer).  The scratch must be zeroed before its first use; the evaluations leave it reusable. */
int b200_constant_scratch_bytes(int m, int n, int64_t *bytes);
/* One evaluation of f at (vx, vy) = (v[0], v[1]).  prev = R[-2], next = R[-1]: (m, n) device
 * frames of `dtype` (float32 frames are widened, never narrowed).  Only enqueues kernels; record
 * (device, 3 doubles) receives f, the number N of counted pixels and the B200_CONST_* bits.
 * The means are NumPy's pairwise sums of the counted values in raster order, bit for bit; the
 * centred sums are float64 in the fixed order of B200_CONST_SUM_BLOCKS. */
int b200_constant_eval(const void *prev, const void *next, int dtype, int m, int n, double vx, double vy,
                       void *scratch, double *record, void *stream);

/* ------------------------------------------------------------------------
 * DARTS (pysteps/motion/darts.py:22-220).  Complex arrays are interleaved float64 (re, im) pairs.
 * The 50 x 50 solve (at the defaults) runs on the host; the device computes the block of the
 * spectrum the reference reads, the normal equations MM = M^H M and M^H y, and the field.
 * ---------------------------------------------------------------------- */
#define B200_DARTS_MAX_COLS 242   /* n_c = 2 (2 M_x + 1)(2 M_y + 1): M_x, M_y <= 5 */
#define B200_DARTS_MAX_SIDE 121   /* 2 M + 1 of one axis of the field's coefficients */
#define B200_DARTS_NORMAL_ROWS 512 /* rows of M per partial of b200_darts_normal */

/* The (Kt, Ky, 2K+1) complex block X[kt, ky, kx] = sum_{t,y,x} frames[t, y, x] tw_t[kt, t] tw_y[ky, y]
 * tw_x(kx, x) of the (T, m, n) device frames of `dtype` (float32 is widened).  Host-built tables,
 * exp(-2 pi i ((k j) mod L) / L) of the wrapped numpy index k: tw_t (Kt, T), tw_y (Ky, m) one row per
 * block index, tw_x (fx, n) for the frequencies f = 0 .. fx-1 <= n / 2; block column kx = -K..K reads
 * f = w or conj at f = n - w, w = kx mod n, whichever is <= n / 2.  Passes: x (real rows against tw_x,
 * fixed order over x), t, y.  work: (T m fx + Kt m (2K+1)) complex.  The x pass reads the frames less
 * frames[0, 0, 0]: only the DC coefficient changes, which M and y only ever multiply by zero
 * (i_ = j_ = k_t = 0), and a constant stack gives an exactly zero block, as NumPy's FFT does. */
int b200_darts_spectrum(const void *frames, int dtype, int T, int m, int n, const double *tw_x, int fx,
                        const double *tw_y, int Ky, const double *tw_t, int Kt, int K, double *work,
                        double *spectrum, void *stream);
/* From the block of b200_darts_spectrum (Kt = 2 N_t + 1, Ky = 2 (N_y + M_y) + 1, Kx = 2 (N_x + M_x) + 1):
 * mm (n_c, n_c) = M^H M and mhy (n_c) = M^H y, M's rows i = (k_t, k_y, k_x) in the reference's
 * order, A scaled by sy * i_, B by sx * j_ (sy = c1 / T_y, sx = c1 / T_x), y = k_t X[k_y, k_x, k_t].
 * work: ceil(rows / B200_DARTS_NORMAL_ROWS) * (n_c (n_c + 1) / 2 + n_c) complex partials,
 * rows = (2 N_t + 1)(2 N_y + 1)(2 N_x + 1).  n_c <= B200_DARTS_MAX_COLS. */
int b200_darts_normal(const double *spectrum, int N_x, int N_y, int N_t, int M_x, int M_y, double sx, double sy,
                      double *work, double *mm, double *mhy, void *stream);
/* out (2, m, n) float64 planar: out[c, y, x] = Re(sum_{a,b} coef[c, a, b] ey[a, y] ex[b, x]) / (m n),
 * coef (2, h, w) complex, ey (h, m) and ex (w, n) the tables exp(+2 pi i ((k j) mod L) / L) of the
 * coefficients' wrapped indices.  w <= B200_DARTS_MAX_SIDE. */
int b200_darts_synthesize(const double *coef, int h, int w, const double *ey, const double *ex, int m, int n,
                          double *out, void *stream);

/* ------------------------------------------------------------------------
 * Local Lagrangian probability nowcast (pysteps/nowcasts/lagrangian_probability.py): the
 * exceedance probability of every lead time's extrapolated field in a disk neighbourhood whose
 * diameter grows with lead time.  The reference convolves with scipy's FFT; these counts are exact.
 * ---------------------------------------------------------------------- */
#define B200_PROBABILITY_MAX_SCALE (1 << 24) /* largest kernel diameter s */

/* field: T planes (m, n) of `dtype` on the device, plane t at field + t * plane_stride elements
 * (plane_stride 0: one field for every lead).  A NaN pixel is invalid and counts as an exceedance
 * when nan_exceeds != 0; any other pixel v is valid and exceeds when (double)v >= threshold.
 * scales (HOST, T entries): the kernel diameter s of each lead.  runs (device int32): for the leads
 * with s > 0 in order, s pairs (b0, b1) each -- kernel row a covers columns b0..b1 -- so that
 *   count(y, x) = sum_a sum_{b0(a) <= b <= b1(a)} A(y + c - a, x + c - b),  c = (s - 1) / 2,
 * pixels outside the frame counting zero (scipy.signal.convolve mode="same").  out (T, m, n) float64:
 * NaN at invalid pixels; else the exceedance (0 or 1) for s == 0 and min(count(exceeds) /
 * count(valid), 1) for s > 0, from exact 32-bit counts.  scratch: m (n + 1) 64-bit words on the
 * device, reused by every lead.  m n < 2^31 and max(m, n) + s < 2^31.  Only enqueues kernels. */
int b200_probability(const void *field, int dtype, int64_t plane_stride, int T, int m, int n,
                     double threshold, int nan_exceeds, const int *scales, const int *runs,
                     unsigned long long *scratch, double *out, void *stream);

/* ------------------------------------------------------------------------
 * Ensemble statistics (pysteps/postprocessing/ensemblestats.py): reductions over the member axis of
 * a (k, N) ensemble X of `dtype` on the device, member i at X + i * N elements, N < 2^31 pixels.
 * flags (device int, zeroed by the call): the warnings NumPy raises, as bits. */
#define B200_ENSEMBLE_OVERFLOW 1 /* a sum overflowed: "overflow encountered in reduce" */
#define B200_ENSEMBLE_INVALID 2  /* a sum met inf + -inf: "invalid value encountered in reduce" */
#define B200_ENSEMBLE_EMPTY 4    /* a pixel had no member to average: "Mean of empty slice" */

/* out (N) of `dtype`.  nan_mode 0: np.mean -- the sequential sum over members in `dtype`, divided
 * by k.  nan_mode 1: np.nanmean -- members that are NaN, or below thr when use_thr (compared in
 * double; thr is already rounded to NumPy's comparison dtype), add 0 and are not counted; out =
 * (dtype)((double)sum / count).  Only enqueues kernels. */
int b200_ensemble_mean(const void *X, int dtype, int k, int64_t N, int nan_mode, int use_thr, double thr,
                       void *out, int *flags, void *stream);

/* out (n_thr, N) float64: for every threshold thr[t] (HOST array) the exact count c of members with
 * finite X >= thr[t]; c / k, or NaN where a member is not finite (ignore_nan 0), or c / the number of
 * finite members (ignore_nan 1).  Only enqueues kernels. */
int b200_ensemble_excprob(const void *X, int dtype, int k, int64_t N, const double *thr, int n_thr,
                          int ignore_nan, double *out, int *flags, void *stream);

/* Band depth, step 1: the mask of the pixels whose members are all finite and some member >= thr,
 * col (N int32): the pixel's column among the masked pixels in C order, -1 elsewhere; *p (device
 * int64): the number of masked pixels.  Only enqueues kernels. */
int b200_ensemble_band_mask(const void *X, int dtype, int k, int64_t N, double thr, int *col, int64_t *p,
                            void *stream);

/* Band depth, step 2: b (k, p) float64 tie-breaks; at every masked pixel member i has the rank
 * r = 1 + #{j : X_j < X_i, or X_j == X_i and (b_j < b_i, or b_j == b_i and j < i)}; match (k
 * int64): the sum of (k - r) (r - 1) over the masked pixels.  Only enqueues kernels. */
int b200_ensemble_band_match(const void *X, int dtype, int k, int64_t N, const int *col, const double *b,
                             int64_t p, int64_t *match, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Linear and salient blending (pysteps/blending/linear_blending.py).  All arrays are device memory
 * unless stated otherwise; dtypes are B200_F32 / B200_F64. */
#define B200_BLEND_COPY 0   /* transform None */
#define B200_BLEND_SQUARE 1 /* "sqrt": x**2 */
#define B200_BLEND_DB 2     /* "dB": 10**(x/10) */
#define B200_BLEND_EXP 3    /* "BoxCox"/"log", lambda 0: exp(x) */
#define B200_BLEND_BOXCOX 4 /* "BoxCox"/"log": exp(log(lambda x + 1) / lambda) */
#define B200_BLEND_MM 1     /* unit "mm": x / a * b */
#define B200_BLEND_DBZ 2    /* unit "dBZ": (x / a) ** b */
#define B200_BLEND_NOWCAST 0 /* lead modes of b200_blend_linear */
#define B200_BLEND_NWP 1
#define B200_BLEND_LINEAR 2
#define B200_BLEND_SKIP 3

/* y (n) = the inverse transform `kind` of x (n) in the dtype, then y < thr -> zero for the
 * transcendental kinds.  A pixel whose value lies within the kernel's error bound of thr is left
 * unthresholded and appended to (fix_idx, fix_x) (its index and input value, in no fixed order, at
 * most cap of them); *nfix (device) is their number, which may exceed cap.  The exact kinds take
 * nfix = NULL. */
int b200_blend_transform(const void *x, void *y, int dtype, int64_t n, int kind, double lam, double thr,
                         double zero, long long *fix_idx, double *fix_x, int64_t cap, unsigned long long *nfix,
                         void *stream);

/* y (n) = x / a * b (B200_BLEND_MM) or (x / a) ** b (B200_BLEND_DBZ), a and b cast to the dtype; y may be x. */
int b200_blend_unit(const void *x, void *y, int dtype, int64_t n, int kind, double a, double b, void *stream);

/* y[idx[i]] = val[i] cast to the dtype, for i < n. */
int b200_blend_scatter(void *y, int dtype, const long long *idx, const double *val, int64_t n, void *stream);

/* out (n_out, T, P) of nwp_dtype.  Output member e reads nowcast member now_map[e] at
 * now + now_map[e] * now_member + lead * P and NWP member nwp_map[e] likewise; the NWP is
 * nan_to_num'd and a NaN of the nowcast becomes the NWP value (fill_nwp) or 0.  Per lead (device
 * arrays of T): mode (B200_BLEND_*), bits (1: w_nwp * nwp in float64, 2: w_now * now in float64,
 * 4: their sum in float64; otherwise in float32), w_nwp and w_now. */
int b200_blend_linear(const void *now, int now_dtype, const int *now_map, int64_t now_member, const void *nwp,
                      int nwp_dtype, const int *nwp_map, int64_t nwp_member, void *out, int n_out, int T, int64_t P,
                      const int *mode, const int *bits, const double *w_nwp, const double *w_now, int fill_nwp,
                      void *stream);

/* Device scratch of b200_blend_salient and b200_dense_rank for a slab of n < 2^31 values. */
int b200_blend_scratch_bytes(int64_t n, int64_t *bytes);

/* One lead of the salient blend, written to out[:, lead] (layout of b200_blend_linear): the dense
 * rank of diff over the (n_out, P) slab and _get_ws with w = weight, w1 = 1 - weight,
 * w2 = weight**2, w12 = (1 - weight)**2.  n_out * P < 2^31.  Reads nothing back. */
int b200_blend_salient(const void *now, int now_dtype, const int *now_map, int64_t now_member, const void *nwp,
                       int nwp_dtype, const int *nwp_map, int64_t nwp_member, void *out, int n_out, int T,
                       int64_t P, int lead, double w, double w1, double w2, double w12, int fill_nwp, void *scratch,
                       int64_t scratch_bytes, void *stream);

/* rank (n uint32): the dense rank (1-based) of every x, -0.0 equal to +0.0; *max_rank the largest;
 * *nan_flag 1 when some x is NaN (the ranks are then meaningless).  n < 2^31. */
int b200_dense_rank(const void *x, int dtype, int64_t n, unsigned *rank, unsigned *max_rank, int *nan_flag,
                    void *scratch, int64_t scratch_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Verification scores (pysteps/verification/probscores.py, ensscores.py): the accumulation steps of
 * CRPS, the rank histogram, the reliability diagram and the ROC curve.  X_f is a (k, N) ensemble
 * (member i at X_f + i * N elements), X_o, P the (N) observations and probabilities, each of dtype
 * B200_F32 or B200_F64; N < 2^31.  Thresholds are doubles already rounded to NumPy's comparison
 * dtype and compared in double.  Device memory unless stated otherwise. */
#define B200_VERIF_MAX_MEMBERS 512 /* k of b200_verif_crps and b200_verif_rankhist */
#define B200_VERIF_MAX_BINS 2048   /* n_bins of b200_verif_reldiag, n_thr of b200_verif_roc */

/* out[s] (nseg values of `dtype`) = np.sum(x[seg_off[s] : seg_off[s] + seg_len[s]]): NumPy's pairwise
 * summation in `dtype` (csrc/pairwise_body.cuh).  seg_off, seg_len: HOST arrays.  Only enqueues
 * kernels. */
int b200_pairwise_sum(const void *x, int dtype, const int64_t *seg_off, const int64_t *seg_len, int nseg,
                      void *out, void *stream);

/* CRPS: at every pixel whose members and observation are finite, in pixel order, res[j] = the
 * pixel's np.sum over its k + 1 columns of alpha p^2 + beta (1 - p)^2 (float64); *n (device int64)
 * the number of such pixels.  res: N doubles.  1 <= k <= B200_VERIF_MAX_MEMBERS.  Only enqueues
 * kernels. */
int b200_verif_crps(const void *Xf, int f_dtype, const void *Xo, int o_dtype, int k, int64_t N, double *res,
                    int64_t *n, void *stream);

/* Rank histogram, step 1.  The pixels whose members and observation are finite (and, with use_min,
 * some member >= thr_f or the observation >= thr_o); with use_min the values below their threshold
 * become sub_f / sub_o (already in the array's dtype).  b1 = #{members < obs}, b2 = k - #{members >
 * obs}.  hist (k + 1 int64, zeroed by the call) counts every untied pixel in bin b1; ties (N int32
 * pairs) receive (b1, b2) of the tied pixels in pixel order and *n_ties (device int64) their number.
 * 1 <= k <= B200_VERIF_MAX_MEMBERS.  Only enqueues kernels. */
int b200_verif_rankhist(const void *Xf, int f_dtype, const void *Xo, int o_dtype, int k, int64_t N, int use_min,
                        double thr_f, double sub_f, double thr_o, double sub_o, int64_t *hist, void *ties,
                        int64_t *n_ties, void *stream);

/* Rank histogram, step 2: hist[int(b1 + u[j] * (b2 + 1 - b1))] += 1 for the n_ties tied pixels of
 * step 1, u (n_ties float64) the uniform draws.  Only enqueues kernels. */
int b200_verif_rankhist_ties(const void *ties, int64_t n_ties, const double *u, int k, int64_t *hist,
                             void *stream);

/* Reliability diagram: the finite pairs, binned by np.digitize(P, edges, right=True) over the
 * n_edges increasing float64 edges (HOST array), n_edges - 1 <= B200_VERIF_MAX_BINS.  For the bins
 * 1 .. n_edges - 1: above[bin - 1] (int64) = #{obs >= thr_o}; sorted (N values of p_dtype) = P of
 * those pixels ordered by bin, in pixel order within a bin; seg (n_edges int64) = where every bin
 * starts in sorted, then their total.  Only enqueues kernels. */
int b200_verif_reldiag(const void *P, int p_dtype, const void *Xo, int o_dtype, int64_t N, const double *edges,
                       int n_edges, double thr_o, void *sorted, int64_t *seg, int64_t *above, void *stream);

/* ROC curve: counts (2 (n_thr + 1) int64): counts[c] the finite pairs with obs >= thr_o and exactly c
 * of the n_thr increasing float64 thresholds (HOST array) <= P, counts[n_thr + 1 + c] those with obs <
 * thr_o.  n_thr <= B200_VERIF_MAX_BINS.  Only enqueues kernels. */
int b200_verif_roc(const void *P, int p_dtype, const void *Xo, int o_dtype, int64_t N, const double *thr, int n_thr,
                   double thr_o, int64_t *counts, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Deterministic and spatial verification scores (pysteps/verification/detcatscores.py,
 * spatialscores.py, ensscores.py). */

/* Contingency table of det_cat_fct_accum: pred and obs are C-contiguous arrays of the same shape,
 * read at offset(kept index) + offset(reduced index), where each set of axes (at most 4, sizes and
 * element strides in HOST arrays, slowest first; none: one element) is walked in C order.  For every
 * output element m (M = the product of the kept sizes): counts[m], counts[M + m], counts[2M + m],
 * counts[3M + m] (int64) = the hits (pred > thr_p and obs > thr_o), false alarms, misses and correct
 * negatives over its reduced pairs.  NaN compares false.  M * R < 2^31.  Only enqueues kernels. */
int b200_verif_contab(const void *pred, int p_dtype, const void *obs, int o_dtype, double thr_p, double thr_o,
                      const int64_t *kept_size, const int64_t *kept_stride, int n_kept, const int64_t *red_size,
                      const int64_t *red_stride, int n_red, int64_t *counts, void *stream);

/* Moments of det_cont_fct_accum.  pred, obs: C-contiguous arrays of the same shape; NumPy's reduction
 * order as a plan: for every output element m (M = the product of the kept sizes) and every outer
 * index o (O = the product of the outer sizes, C order), a run of L contiguous elements starts at
 * offset(m) + offset(o) (axes as for b200_verif_contab).  conditioning: 0 every pair, 1 the pairs with
 * pred > thr_p or obs > thr_o, 2 both (the others become NaN).  For the nine summands k of the
 * reference's np.nanmean calls (0 obs, 1 pred, 2 res = pred - obs, 3 res^2, 4 (pred + obs)^2,
 * 5 |res|, 6 (obs - mobs)(pred - mpred), 7 |obs - mobs|^2, 8 |pred - mpred|^2, with the means mobs,
 * mpred of 0 and 1 broadcast): tot[k M + m] (double) = NumPy's np.sum of the summand with NaN as 0 in
 * its dtype (obs: obs's, pred: pred's, res-based: the result type); cnt[m] (int64) = the finite
 * residuals and cnt[(1 + k) M + m] the non-NaN summands; infs[m] bit 2k / 2k + 1: +inf / -inf was
 * summed; *flags the B200_MOM_* bits of the element-wise operations.  M O L < 2^31.  Only enqueues
 * kernels. */
#define B200_MOM_SUB_RES_OVER (1 << 0) /* pred - obs overflowed */
#define B200_MOM_SUB_RES_INV (1 << 1)  /* pred - obs made a NaN from non-NaN operands */
#define B200_MOM_ADD_SUM_OVER (1 << 2)
#define B200_MOM_ADD_SUM_INV (1 << 3)
#define B200_MOM_SQ_RES_OVER (1 << 4)
#define B200_MOM_SQ_SUM_OVER (1 << 5)
#define B200_MOM_SUB_OBS_OVER (1 << 6) /* obs - mobs */
#define B200_MOM_SUB_OBS_INV (1 << 7)
#define B200_MOM_SUB_PRED_OVER (1 << 8)
#define B200_MOM_SUB_PRED_INV (1 << 9)
#define B200_MOM_MUL_OVER (1 << 10) /* (obs - mobs) * (pred - mpred) */
#define B200_MOM_MUL_INV (1 << 11)
#define B200_MOM_SQ_VOBS_OVER (1 << 12)
#define B200_MOM_SQ_VPRED_OVER (1 << 13)
int b200_verif_cont_moments(const void *pred, int p_dtype, const void *obs, int o_dtype, int conditioning,
                            double thr_p, double thr_o, const int64_t *kept_size, const int64_t *kept_stride,
                            int n_kept, const int64_t *outer_size, const int64_t *outer_stride, int n_outer,
                            int64_t L, double *tot, int64_t *cnt, int *infs, int *flags, void *stream);

#define B200_FSS_GROUP 16 /* na, nb of b200_fss_sums */

/* Fractions of fss_accum for nf fields of m x n values of `dtype` (field f at X + f m n): the
 * indicator (x >= thr, a non-finite x taken as sub, both already rounded as NumPy rounds them),
 * smoothed with scipy.ndimage.uniform_filter(size=s, mode="constant") when s > 1, into S (nf m n
 * float64).  nf m n < 2^31.  Only enqueues kernels. */
int b200_fss_fractions(const void *X, int dtype, int nf, int m, int n, double thr, double sub, int s, double *S,
                       void *stream);

/* out[i nb + j] = np.sum(S[a0 + i] * S[b0 + j]) over the P values of each plane (NumPy's pairwise
 * summation, float64) for every i < na, j < nb with a0 + i <= b0 + j; the other entries are left as
 * they are.  S: planes of P float64, plane f at S + f P.  na, nb <= B200_FSS_GROUP, P < 2^31.  Only
 * enqueues kernels. */
int b200_fss_sums(const double *S, int64_t P, int a0, int na, int b0, int nb, double *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Probability matching (pysteps/postprocessing/probmatching.py).  Device memory unless stated
 * otherwise; dtypes B200_F32 / B200_F64; n < 2^31.  Ties are ranked in index order, as
 * argsort(kind="stable") ranks them.  Only enqueue kernels. */

/* Device scratch of b200_pm_match_stats, b200_pm_match and b200_pm_resample for n values. */
int b200_pm_scratch_bytes(int64_t n, int64_t *bytes);

/* stats (8 doubles) of nonparam_match_empirical_cdf's initial array x (n_x values, ignore: n_x bytes,
 * nonzero where ignored, or NULL) and target t (n_t values): [0] np.nanmin(x) (NaN when every x is
 * NaN), [1] the non-NaN x, [2] the non-finite x outside the mask, [3] the x inside it, [4] the x >
 * stats[0] outside it, [5] np.nanmin(t), [6] the non-NaN t, [7] the t > stats[5].  A zero minimum is
 * -0.0 when some minimal value is -0.0. */
int b200_pm_match_stats(const void *x, int x_dtype, const unsigned char *ignore, int64_t n_x, const void *t,
                        int t_dtype, int64_t n_t, double *stats, void *scratch, int64_t scratch_bytes, void *stream);

/* out (n float64) = nonparam_match_empirical_cdf(x, t, ignore) from the stats of b200_pm_match_stats
 * (stats[2] must be 0); n_xwet = stats[4] and n_twet = stats[7] as integers.  clip: the values of t
 * below p = _lerp(s[i0], s[i1], gamma) of the sorted t (NaN as stats[5]) become stats[5]. */
int b200_pm_match(const void *x, int x_dtype, const unsigned char *ignore, const void *t, int t_dtype, int64_t n,
                  const double *stats, int64_t n_xwet, int64_t n_twet, int clip, int64_t i0, int64_t i1,
                  double gamma, double *out, void *scratch, int64_t scratch_bytes, void *stream);

/* *n_nan (int64) = the indices i < n where a[i] or b[i] is NaN. */
int b200_pm_resample_nan(const void *a, int a_dtype, const void *b, int b_dtype, int64_t n, int64_t *n_nan,
                         void *stream);

/* out (n of out_dtype) = resample_distributions(a, b): n_nan (from b200_pm_resample_nan) NaNs, then
 * the values that are NaN in neither array, sorted in descending order, position n_nan + q taken
 * from a where draws[n_nan + q] (n bytes, 0 or 1) is nonzero and from b elsewhere, sorted again in
 * descending order. */
int b200_pm_resample(const void *a, int a_dtype, const void *b, int b_dtype, int64_t n, int64_t n_nan,
                     const unsigned char *draws, void *out, int out_dtype, void *scratch, int64_t scratch_bytes,
                     void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PYSTEPS_B200_H */
