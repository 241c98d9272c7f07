"""B200 dense Lucas-Kanade motion estimation -- drop-in for
``pysteps.motion.lucaskanade.dense_lucaskanade``
(pysteps/motion/lucaskanade.py:38-279).

The reference orchestrates OpenCV / SciPy calls from Python; here the same
orchestration (argument handling, early-outs, return shapes) stays in Python and
every array operation is a CUDA kernel of ``libpysteps_b200.so``:

  reference call                                   | kernel(s), csrc/
  -------------------------------------------------+---------------------------------
  np.ma.masked_invalid / .min() (:213-219)         | lk_dense.cu  mask_invalid
  utils.images.morph_opening (:222-224)            | lk_dense.cu  morph_open
  feature.shitomasi.detection (:227)               | lk_dense.cu  masked_minmax, quantise,
    cv2.dilate / goodFeaturesToTrack               |   cov_rowsum, box_eig; lk_features.cu
  tracking.lucaskanade.track_features (:234)       | lk_dense.cu  quantise, pyrdown, scharr;
    cv2.calcOpticalFlowPyrLK                       |   lk_track.cu lk_track, compact_tracks
  utils.cleansing.detect_outliers (:252)           | sparse.cu    outliers, compact_rows
  utils.cleansing.decluster (:265)                 | sparse.cu    decluster
  utils.interpolate.idwinterp2d (:274)             | idw.cu       idw

Sparse vectors stay on the device between stages; the host reads back only element
counts (to size the next launch / take the reference's early-outs).
"""
import ctypes
import os
import threading
import time

import numpy as np
import torch
from numpy.ma.core import MaskedArray

from .. import _device, _lib


def _call(name, *args):
    _lib.call(name, *args)


def _s():
    return _device.stream_ptr()


class _Frame:
    """Device state of one input frame after masking and morphological opening.  All buffers
    are allocated up front (on the caller's stream) so that the work itself can be enqueued on
    either stream without involving the caching allocator."""
    __slots__ = ("img", "user_mask", "mask", "stats0", "opened", "stats", "q_track",
                 "prepared", "have_stats", "have_q", "qflag", "q_det", "valid")

    def __init__(self, img_d, user_mask_d, m, n, size_opening, f32=False, fused=False, detect=False):
        # frames that were float32 at the API are scaled to uint8 in float32 arithmetic, as NumPy
        # does for a float32 array (tracking/lucaskanade.py:144-160, feature/shitomasi.py:141-151)
        self.qflag = 2 if f32 else 0
        self.img = img_d
        self.user_mask = user_mask_d
        self.mask = torch.empty((m, n), dtype=torch.uint8, device="cuda")
        self.stats0 = torch.empty(3, dtype=torch.float64, device="cuda")
        # fused front end (csrc/lk_frontend.cu): the opened float64 image is never materialised
        self.opened = None if fused else (torch.empty((m, n), dtype=torch.float64, device="cuda")
                                          if size_opening > 0 else img_d)
        self.stats = torch.empty(12, dtype=torch.float64, device="cuda")
        self.q_track = torch.empty((m, n), dtype=torch.uint8, device="cuda")
        self.q_det = torch.empty((m, n), dtype=torch.uint8, device="cuda") if (fused and detect) else None
        self.valid = torch.empty((m, n), dtype=torch.uint8, device="cuda") if (fused and detect) else None
        self.prepared = self.have_stats = self.have_q = False


def _front_end(f, m, n, size_opening, buffer_mask):
    """Everything dense_lucaskanade does to a frame before looking for features, three passes over
    it (csrc/lk_frontend.cu: TMA-staged halo tiles): mask, opening, the four min/max sets, the
    tracker's and -- for a frame that is the first of a pair -- the detector's uint8 image."""
    if f.prepared:
        return f
    _call("b200_lk_frontend", f.img.data_ptr(), _device.ptr(f.user_mask), m, n, int(size_opening),
          int(buffer_mask), f.qflag, f.mask.data_ptr(), f.stats0.data_ptr(), f.stats.data_ptr(),
          f.q_track.data_ptr(), _device.ptr(f.q_det), _device.ptr(f.valid), _s())
    f.prepared = f.have_stats = f.have_q = True
    return f


def _prepare_frame(f, m, n, size_opening):
    """masked_invalid + fill value + morph_opening (lucaskanade.py:213-224)."""
    if f.prepared:
        return f
    _call("b200_mask_invalid", f.img.data_ptr(), _device.ptr(f.user_mask), m, n, f.mask.data_ptr(),
          f.stats0.data_ptr(), _s())
    if size_opening > 0:
        # thr = prvs_img.min(); removed pixels take np.nanmin(prvs_img): both stats0[0]
        _call("b200_morph_opening", f.img.data_ptr(), f.mask.data_ptr(), m, n, int(size_opening),
              f.stats0.data_ptr(), f.stats0.data_ptr(), f.opened.data_ptr(), _s())
    f.prepared = True
    return f


def _frame_stats(f, m, n, buffer_mask):
    if not f.have_stats:
        _call("b200_masked_minmax", f.opened.data_ptr(), f.mask.data_ptr(), m, n, int(buffer_mask),
              f.stats0.data_ptr(), f.stats.data_ptr(), _s())
        f.have_stats = True
    return f.stats


def _track_image(f, m, n, buffer_mask):
    """the uint8 image track_features builds (tracking/lucaskanade.py:144-160)"""
    if not f.have_q:
        st = _frame_stats(f, m, n, buffer_mask)
        _call("b200_quantise_u8", f.opened.data_ptr(), f.mask.data_ptr(), m, n, 0 | f.qflag, 0, st.data_ptr(),
              st.data_ptr(), f.q_track.data_ptr(), None, _s())
        f.have_q = True
    return f.q_track


_DECLUSTER_MAX = 16384  # csrc/sparse.cu DC_MAX (vectors held in one CTA's shared memory)
_side_streams = {}
_grids = {}
_readback = threading.local()


def _readback_buffers(cap):
    """Pinned host buffers (counts, xy, uv) of the sparse stage's read-back, one set per host thread."""
    got = getattr(_readback, "bufs", None)
    if got is None or got[1].shape[0] < cap:
        got = _readback.bufs = (torch.empty(4, dtype=torch.int32, pin_memory=True),
                                torch.empty((cap, 2), dtype=torch.float64, pin_memory=True),
                                torch.empty((cap, 2), dtype=torch.float64, pin_memory=True))
    return got[0], got[1][:cap], got[2][:cap]


def _pixel_grid(a, b):
    """np.arange(a, b) as a float64 device vector (lucaskanade.py:271-272), built once."""
    key = (torch.cuda.current_device(), a, b)
    g = _grids.get(key)
    if g is None:
        if len(_grids) > 64:
            _grids.clear()
        g = _grids[key] = _device.to_device(np.arange(a, b, dtype=np.float64))
        torch.cuda.current_stream().synchronize()
    return g



def _side_stream():
    """One auxiliary stream per (device, host thread)."""
    key = (torch.cuda.current_device(), threading.get_ident())
    if key not in _side_streams:
        _side_streams[key] = torch.cuda.Stream()
    return _side_streams[key]


def _pyramid_layout(m, n, win, max_level):
    lv = ctypes.c_int(0)
    off = (ctypes.c_int64 * _lib.LK_MAX_LEVELS)()
    hs = (ctypes.c_int * _lib.LK_MAX_LEVELS)()
    ws = (ctypes.c_int * _lib.LK_MAX_LEVELS)()
    tot = ctypes.c_int64(0)
    _lib.check(_lib.load().b200_lk_pyramid_layout(m, n, int(win[0]), int(win[1]), int(max_level),
                                                  ctypes.byref(lv), off, hs, ws, ctypes.byref(tot)))
    return lv.value, int(tot.value)


_WINDOW_MAX = 64 * 64  # csrc/lk_track.cu: the window and its products live in one CTA's shared memory


def _tracker_args(winsize, nr_levels, criteria):
    """calcOpticalFlowPyrLK's argument check and TermCriteria clamps (tracking/lucaskanade.py:171), taken
    before anything is uploaded -> (win_w, win_h, nr_levels, max_count, epsilon).  cv2 raises its
    assertion as cv2.error, even without points to track; here it is a ValueError with the same text."""
    win_w, win_h = (int(v) for v in winsize)
    nr_levels = int(nr_levels)
    if not (nr_levels >= 0 and win_w > 2 and win_h > 2):
        raise ValueError("(-215:Assertion failed) maxLevel >= 0 && winSize.width > 2 && winSize.height > 2 "
                         "in function 'calc'")
    if win_w * win_h > _WINDOW_MAX:
        raise NotImplementedError(f"pysteps_b200 LK: tracking windows above {_WINDOW_MAX} pixels are not "
                                  f"implemented (winsize {win_w}x{win_h})")
    ctype, max_count, eps = criteria
    max_count = min(max(int(max_count), 0), 100) if (int(ctype) & 1) else 30
    eps = min(max(float(eps), 0.0), 10.0) if (int(ctype) & 2) else 0.01
    return win_w, win_h, nr_levels, max_count, eps


_KD_SHARED_MAX = 4096  # csrc/knn_device.cuh NMAX: the tree of the tie recomputation is built in one CTA
_plan_pin = threading.local()


def _fill_planned(interp_kwargs, counts, dec_xy, dec_uv, pool_cap, m, n, r0, r1, verbose):
    """The interpolation stage of a device-resident dense call without a read-back in front of it:
    b200_idw_plan derives the early-outs, checks and key level from the declustered vectors on the
    device, b200_idw_fill_planned is enqueued behind it at once and its kernels follow the plan, and the
    host reads the 48-byte plan while they run.  Raises and returns as the read-back path does;
    returns (out, twin, whether the vectors reached the interpolator), or None for the shapes that path keeps: k=None, k outside 1..32, more pooled
    vectors than the one-CTA tree build holds, fewer than two rows or columns, and interpolator
    arguments that are not numbers (the read-back path raises on those only once it interpolates)."""
    k = interp_kwargs.get("k", 20)
    try:
        power = float(interp_kwargs.get("power", 0.5))
        dist_offset = float(interp_kwargs.get("dist_offset", 0.5))
        k = None if k is None else int(k)
    except (TypeError, ValueError):
        return None
    if k is None or not 1 <= k <= 32 or pool_cap > min(_DECLUSTER_MAX, _KD_SHARED_MAX) or m < 2 or n < 2:
        return None
    mb = r1 - r0
    plan = torch.empty(12, dtype=torch.int32, device="cuda")  # B200IdwPlan, include/pysteps_b200.h
    _call("b200_idw_plan", counts.data_ptr(), dec_xy.data_ptr(), dec_uv.data_ptr(), pool_cap,
          int(max(m, n) < 16384), plan.data_ptr(), _s())
    pin = getattr(_plan_pin, "buf", None)
    if pin is None:
        pin = _plan_pin.buf = torch.empty(12, dtype=torch.int32, pin_memory=True)
    pin.copy_(plan, non_blocking=True)
    ready = torch.cuda.Event()
    ready.record()
    out = torch.empty((2, mb, n), dtype=torch.float64, device="cuda")
    twin = torch.empty((mb, n, 2), dtype=torch.float64, device="cuda")
    xgrid, ygrid = _pixel_grid(0, n), _pixel_grid(r0, r1)
    _call("b200_idw_fill_planned", dec_xy.data_ptr(), dec_uv.data_ptr(), plan.data_ptr(), pool_cap, k, power,
          dist_offset, xgrid.data_ptr(), n, ygrid.data_ptr(), mb, out.data_ptr(), twin.data_ptr(), _s())
    ready.synchronize()
    n_pool, n_kept, n_dec, nonfinite = pin[:4].tolist()
    # the read-back path's early-outs and errors, in its order (:245-269, decorators.py:190-208); a
    # zero field is written by the fill itself
    if n_pool == 0:
        return out, twin, False
    if verbose:
        print("--- LK found %i sparse vectors ---" % n_kept)
    if n_dec == 0:
        return out, twin, False
    if nonfinite & 1:
        raise ValueError("argument 'values' contains non-finite values")
    if nonfinite & 2:
        raise ValueError("argument 'xy_coord' contains non-finite values")
    return out, twin, True


def _attach_twin(out, twin, interp_kwargs):
    """The finiteness certificate (see the end of dense_lucaskanade) and the interleaved (m, n, 2) copy
    of the field the extrapolator reads: both hold for THIS version of the returned tensor only (torch
    bumps ._version on every in-place write, through views too)."""
    power = float(interp_kwargs.get("power", 0.5))
    dist_offset = float(interp_kwargs.get("dist_offset", 0.5))
    if dist_offset > 0.0 and 0.0 <= power <= 8.0:
        out._b200_finite_version = out._version
    out._b200_twin = twin
    out._b200_twin_version = out._version


# ---- the host-side tail of the interpolation, shared with stages.idwinterp2d -------------------------
def _idw_constant(out, v2):
    """decorators.py:200-208: the constant field of one vector, or of (n, nvar) values that are all equal,
    into the (nvar, ny, nx) device tensor `out`.  Returns whether the field was constant."""
    if v2.shape[0] == 1:
        for c in range(v2.shape[1]):
            _call("b200_fill_f64", out[c].data_ptr(), out[c].numel(), float(1.0 * v2[0, c]), _s())
        return True
    if v2.max() == v2.min():
        _call("b200_fill_f64", out.data_ptr(), out.numel(), float(1.0 * v2.ravel()[0]), _s())
        return True
    return False


def _key_level(xy_h, grid_level):
    """coords_on_16th_grid of b200_idw_fill: 1 when every coordinate is a multiple of 1/16 below 2^14 (squared
    distances are exact multiples of 1/256: packed 64-bit keys), 2 when moreover the vectors sit on the
    half-pixel grid (medians of integer corners) and the grid on integers (32-bit keys), else 0.  grid_level()
    is the grid's own level, asked only when the vectors qualify."""
    if not (np.all(xy_h * 16.0 == np.rint(xy_h * 16.0)) and np.abs(xy_h).max() < 16384.0):
        return 0
    g = grid_level()
    if not g:
        return 0
    return 2 if g == 2 and np.all(xy_h * 2.0 == np.rint(xy_h * 2.0)) else 1


def _idw_fill(dxy, dv, npts, nvar, k, power, dist_offset, mean_res, gx, nx, gy, ny, level, out):
    """Fills `out` (nvar, ny, nx) from npts device vectors: exhaustive tile search, grid points whose neighbour
    set depends on cKDTree's tie order recomputed from its query (csrc/idw.cu, knn.cu); k=None: every vector
    weighs in at every grid point (interpolate.py:82-88)."""
    if k is None:
        _call("b200_idw_fill_all", dxy.data_ptr(), dv.data_ptr(), None, npts, nvar, float(power),
              float(dist_offset), mean_res, gx.data_ptr(), nx, gy.data_ptr(), ny, out.data_ptr(), _s())
    else:
        _call("b200_idw_fill", dxy.data_ptr(), dv.data_ptr(), None, npts, nvar, int(min(int(k), npts)),
              float(power), float(dist_offset), mean_res, gx.data_ptr(), nx, gy.data_ptr(), ny, int(level),
              out.data_ptr(), _s())


def dense_lucaskanade(input_images, lk_kwargs=None, fd_method="shitomasi", fd_kwargs=None,
                      interp_method="idwinterp2d", interp_kwargs=None, dense=True,
                      nr_std_outlier=3, k_outlier=30, size_opening=3, decl_scale=20,
                      verbose=False):
    """Same contract as the reference (see its docstring, lucaskanade.py:54-180).

    input_images: ndarray / MaskedArray (T,m,n) -> NumPy results; CUDA torch tensor
    (NaN = no data) -> results stay on the device.  Only the default feature detector
    ("shitomasi") and interpolator ("idwinterp2d") are implemented; anything else raises
    NotImplementedError (there is no CPU fallback).
    """
    # decorators.check_input_frames(2): decorators.py:121-146
    if input_images.ndim != 3:
        raise ValueError(
            "input_images dimension mismatch.\n"
            f"input_images.shape: {str(tuple(input_images.shape))}\n"
            "(t, x, y ) dimensions expected"
        )
    if fd_method != "shitomasi":
        raise NotImplementedError(f"pysteps_b200 LK: fd_method={fd_method!r} is not implemented")
    if interp_method != "idwinterp2d":
        raise NotImplementedError(f"pysteps_b200 LK: interp_method={interp_method!r} is not implemented")
    if size_opening not in (0, 3):
        raise NotImplementedError("pysteps_b200 LK: size_opening must be 0 or 3")

    _device.require_cuda()
    on_device = _device.is_device_tensor(input_images)

    if verbose:
        print("Computing the motion field with the Lucas-Kanade method.")
        t0 = time.time()

    fd_kwargs = dict() if fd_kwargs is None else dict(fd_kwargs)
    lk_kwargs = dict() if lk_kwargs is None else dict(lk_kwargs)
    interp_kwargs = dict() if interp_kwargs is None else dict(interp_kwargs)

    # feature.shitomasi.detection defaults (shitomasi.py:26-38)
    max_corners = fd_kwargs.get("max_corners", 1000)
    if fd_kwargs.get("max_num_features", None) is not None:
        max_corners = fd_kwargs["max_num_features"]
    quality_level = fd_kwargs.get("quality_level", 0.01)
    min_distance = fd_kwargs.get("min_distance", 10)
    block_size = fd_kwargs.get("block_size", 5)
    buffer_mask = int(fd_kwargs.get("buffer_mask", 5))
    if block_size != 5 or fd_kwargs.get("use_harris", False):
        raise NotImplementedError("pysteps_b200 LK: only block_size=5, use_harris=False")
    if int(max_corners) <= 0:
        raise NotImplementedError("pysteps_b200 LK: max_corners must be positive")
    max_corners = int(max_corners)
    # tracking.lucaskanade.track_features defaults (tracking/lucaskanade.py:35-45)
    if lk_kwargs.get("flags", 0) != 0:
        raise NotImplementedError("pysteps_b200 LK: flags must be 0")
    win_w, win_h, nr_levels, max_count, eps = _tracker_args(lk_kwargs.get("winsize", (50, 50)),
                                                            lk_kwargs.get("nr_levels", 3),
                                                            tuple(lk_kwargs.get("criteria", (3, 10, 0))))
    min_eig_thr = float(lk_kwargs.get("min_eig_thr", 1e-4))

    nr_fields = int(input_images.shape[0])
    m, n = int(input_images.shape[1]), int(input_images.shape[2])

    # extension, see the interpolation stage below
    rows = interp_kwargs.get("b200_rows", None)
    r0, r1 = (0, m) if rows is None else (int(rows[0]), int(rows[1]))
    if not (0 <= r0 < r1 <= m):
        raise ValueError("b200_rows must satisfy 0 <= r0 < r1 <= m")
    mb = r1 - r0

    f32 = (input_images.dtype == torch.float32) if isinstance(input_images, torch.Tensor) \
        else (np.asarray(input_images).dtype == np.float32)

    # ---- upload (the reference copies its input, :182) ------------------------------------
    user_mask_d = None
    if isinstance(input_images, MaskedArray):
        user_mask_d = _device.to_device(np.ascontiguousarray(np.ma.getmaskarray(input_images),
                                                             dtype=np.uint8))
        frames_d = _device.to_device(np.ascontiguousarray(input_images.data), torch.float64)
        ensure = lambda t: None  # noqa: E731
    elif (isinstance(input_images, np.ndarray) and input_images.dtype == np.float64
          and input_images.flags.c_contiguous and input_images.flags.writeable):
        # NumPy float64 frames: frame t is uploaded on the stream that consumes it, right before its
        # front end is enqueued -- the upload of frame t+1 (32 MB at 2048^2, 0.7 ms of PCIe) then runs
        # under the detector kernels of frame t instead of in front of everything
        host = torch.from_numpy(input_images)
        frames_d = torch.empty((nr_fields, m, n), dtype=torch.float64, device="cuda")
        uploaded = [False] * nr_fields

        def ensure(t):
            if not uploaded[t]:
                frames_d[t].copy_(host[t], non_blocking=True)
                uploaded[t] = True
    else:
        frames_d = _device.to_device(input_images, torch.float64)
        ensure = lambda t: None  # noqa: E731

    # Two streams: the Shi-Tomasi chain of the previous frame (min-eigenvalue map, sort, ordered
    # selection -- latency-bound kernels that leave most SMs idle) runs on the caller's stream
    # while the side stream prepares the next frame and builds both pyramids.
    main = torch.cuda.current_stream()
    side = _side_stream()
    # fused, TMA-tiled front end whenever the copy engine can address the frame: 16-byte rows and a
    # 16-byte aligned first frame (then every frame is, m * n * 8 being a multiple of 16).  A view into
    # a larger tensor can start 8 bytes off; it takes the stage kernels.
    fused = n % 2 == 0 and 0 <= buffer_mask <= 5 and frames_d.data_ptr() % 16 == 0
    frames = [_Frame(frames_d[t], None if user_mask_d is None else user_mask_d[t], m, n, size_opening, f32,
                     fused, t < nr_fields - 1)
              for t in range(nr_fields)]

    def prepare(t):
        ensure(t)
        if fused:
            return _front_end(frames[t], m, n, size_opening, buffer_mask)
        return _prepare_frame(frames[t], m, n, size_opening)

    pool_cap = max_corners * max(nr_fields - 1, 1)
    pool_xy = torch.empty((pool_cap, 2), dtype=torch.float64, device="cuda")
    pool_uv = torch.empty((pool_cap, 2), dtype=torch.float64, device="cuda")
    counts = torch.zeros(4, dtype=torch.int32, device="cuda")  # pool, kept, declustered, corners
    lv, total = _pyramid_layout(m, n, (win_w, win_h), nr_levels)
    # pyramids: Gaussian levels of every frame, Scharr levels of every frame but the last
    pyr = [[torch.empty(total, dtype=torch.uint8, device="cuda"),
            torch.empty(2 * total, dtype=torch.int16, device="cuda") if t < nr_fields - 1 else None,
            False, False] for t in range(nr_fields)]

    def pyramid(t, with_deriv):
        """Gaussian pyramid of frame t's uint8 image (+ Scharr pyramid when it is the previous
        frame of a pair); a middle frame is built once and reused by both of its pairs."""
        args = (m, n, win_w, win_h, nr_levels)
        P, D, have_p, have_d = pyr[t]
        want_d = with_deriv and not have_d
        if not have_p:
            _call("b200_lk_build_pyramid", _track_image(frames[t], m, n, buffer_mask).data_ptr(), *args,
                  P.data_ptr(), D.data_ptr() if want_d else None, _s())
            pyr[t][2] = True
            pyr[t][3] = have_d or want_d
        elif want_d:
            _call("b200_lk_build_pyramid", None, *args, P.data_ptr(), D.data_ptr(), _s())
            pyr[t][3] = True
        return pyr[t]

    if nr_fields >= 1:
        prepare(0)
    for t in range(nr_fields - 1):
        f = frames[t]
        st = _frame_stats(f, m, n, buffer_mask)
        # ---- main stream: feature detection on the previous frame (:227) -------------------
        eig = torch.empty((m, n), dtype=torch.float32, device="cuda")
        ev_stats = torch.cuda.Event()
        ev_stats.record(main)
        if fused:
            q_det, valid = f.q_det, f.valid
        else:
            q_det = torch.empty((m, n), dtype=torch.uint8, device="cuda")
            valid = torch.empty((m, n), dtype=torch.uint8, device="cuda")
            _call("b200_quantise_u8", f.opened.data_ptr(), f.mask.data_ptr(), m, n, 1 | f.qflag, buffer_mask,
                  st.data_ptr(), st.data_ptr(), q_det.data_ptr(), valid.data_ptr(), _s())
        _call("b200_min_eig", q_det.data_ptr(), m, n, eig.data_ptr(), _s())
        # ---- side stream: next frame + both pyramids (needs this frame's stats only).  Enqueued
        # after the eigenvalue map so that it fills the SMs the sequential box-filter chains,
        # the sort and the single-warp selection leave idle ---------------------------------
        side.wait_event(ev_stats)
        with torch.cuda.stream(side):
            g = prepare(t + 1)
            _frame_stats(g, m, n, buffer_mask)
            pI = pyramid(t, True)
            pJ = pyramid(t + 1, False)
        corners = torch.empty((max_corners, 2), dtype=torch.float32, device="cuda")
        ncorner = counts[3:4]
        _call("b200_good_features", eig.data_ptr(), valid.data_ptr(), m, n, max_corners,
              float(quality_level), float(min_distance), corners.data_ptr(), ncorner.data_ptr(), _s())
        # ---- sparse tracking previous -> next (:234) --------------------------------------
        main.wait_stream(side)
        nxt = torch.empty((max_corners, 2), dtype=torch.float32, device="cuda")
        status = torch.empty(max_corners, dtype=torch.uint8, device="cuda")
        _call("b200_lk_track", pI[0].data_ptr(), pJ[0].data_ptr(), pI[1].data_ptr(), m, n,
              win_w, win_h, nr_levels, max_count, eps, min_eig_thr,
              corners.data_ptr(), max_corners, ncorner.data_ptr(), nxt.data_ptr(), status.data_ptr(),
              _s())
        _call("b200_lk_compact_tracks", corners.data_ptr(), nxt.data_ptr(), status.data_ptr(),
              ncorner.data_ptr(), max_corners, pool_xy.data_ptr(), pool_uv.data_ptr(),
              counts[0:1].data_ptr(), pool_cap, _s())

    def zeros_or_empty():
        if dense:
            z = torch.zeros((2, mb, n), dtype=torch.float64, device="cuda")
            return z if on_device else np.zeros((2, mb, n))
        e = np.empty(shape=(0, 2))
        return (torch.from_numpy(e).cuda(), torch.from_numpy(e).cuda()) if on_device else (e, e.copy())

    if nr_fields < 2:
        torch.cuda.current_stream().synchronize()  # the (asynchronous) upload reads the caller's array
        return zeros_or_empty()

    # ---- outliers (:252-254) on the pooled vectors --------------------------------------
    flags = torch.empty(pool_cap, dtype=torch.uint8, device="cuda")
    kept_xy = torch.empty((pool_cap, 2), dtype=torch.float64, device="cuda")
    kept_uv = torch.empty((pool_cap, 2), dtype=torch.float64, device="cuda")
    if k_outlier is None:
        # the global test (cleansing.py:201-214): every vector against the mean / covariance of all
        _call("b200_detect_outliers_global", pool_uv.data_ptr(), counts[0:1].data_ptr(), pool_cap,
              float(nr_std_outlier), flags.data_ptr(), _s())
    else:
        # equidistant / coincident neighbours in scipy.spatial.cKDTree's own order (csrc/knn.cu): with
        # integer corner coordinates that order decides outlier tests
        _call("b200_detect_outliers",
              pool_uv.data_ptr(), pool_xy.data_ptr(), counts[0:1].data_ptr(),
              pool_cap, float(nr_std_outlier), int(k_outlier), flags.data_ptr(), _s())
    _call("b200_compact_rows", pool_xy.data_ptr(), pool_uv.data_ptr(), flags.data_ptr(),
          counts[0:1].data_ptr(), pool_cap, kept_xy.data_ptr(), kept_uv.data_ptr(),
          counts[1:2].data_ptr(), _s())
    dec_xy, dec_uv = kept_xy, kept_uv
    if dense and decl_scale > 1:
        dec_xy = torch.empty((pool_cap, 2), dtype=torch.float64, device="cuda")
        dec_uv = torch.empty((pool_cap, 2), dtype=torch.float64, device="cuda")
        dc_cap = pool_cap
        if pool_cap > _DECLUSTER_MAX:
            # the kernel's capacity is about the vectors that exist, not the pool they could fill (many
            # frames x max_corners): one extra read-back on this rare shape instead of a refusal
            dc_cap = int(counts[1].item())
            if dc_cap > _DECLUSTER_MAX:
                raise NotImplementedError(
                    f"pysteps_b200 LK: declustering more than {_DECLUSTER_MAX} sparse vectors is not implemented "
                    f"({dc_cap} survived the outlier test)")
        _call("b200_decluster", kept_xy.data_ptr(), kept_uv.data_ptr(), counts[1:2].data_ptr(), max(dc_cap, 1),
              float(decl_scale), 1, dec_xy.data_ptr(), dec_uv.data_ptr(), counts[2:3].data_ptr(), _s())
    else:
        counts[2:3].copy_(counts[1:2])
    if on_device and dense:
        planned = _fill_planned(interp_kwargs, counts, dec_xy, dec_uv, pool_cap, m, n, r0, r1, verbose)
        if planned is not None:
            out, twin, filled = planned
            if verbose and filled:
                torch.cuda.current_stream().synchronize()
                print("--- total time: %.2f seconds ---" % (time.time() - t0))
            _attach_twin(out, twin, interp_kwargs)
            return out
    # the one host read-back of the sparse stage: the counts AND (dense case) the declustered vectors the
    # interpolator's host-side checks look at, in one round trip -- three separate .cpu() calls were three
    # waits with the GPU idle in between.  A device-resident dense call takes the planned fill above
    # instead; this path remains for sparse results (they are returned sized by the count), k=None (a
    # different kernel), pools beyond the one-CTA tree build, and NumPy results, whose 64 MB (2048^2)
    # download at the end waits for the whole fill anyway
    pin = _readback_buffers(pool_cap)
    pin[0].copy_(counts, non_blocking=True)
    if dense:
        pin[1].copy_(dec_xy, non_blocking=True)
        pin[2].copy_(dec_uv, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    n_pool, n_kept, n_dec, _ = pin[0].tolist()

    if n_pool == 0:  # :245-249
        return zeros_or_empty()
    if verbose:
        print("--- LK found %i sparse vectors ---" % n_kept)
    if not dense:  # :260-261
        xy, uv = kept_xy[:n_kept], kept_uv[:n_kept]
        return (xy, uv) if on_device else (xy.cpu().numpy(), uv.cpu().numpy())
    if n_dec == 0:  # :268-269
        return zeros_or_empty()

    # ---- interpolation (:272-274) behind decorators.prepare_interpolator ----------------
    power = float(interp_kwargs.get("power", 0.5))
    k = interp_kwargs.get("k", 20)
    dist_offset = float(interp_kwargs.get("dist_offset", 0.5))
    # extension (an unknown interpolator kwarg is ignored by the reference): fill only the grid
    # rows [r0, r1) -- the result is then band shaped (2, r1-r0, n).  The sparse stages are
    # deterministic, so ranks that each fill one band of the same frames agree bit for bit with
    # the rows of the full field (tile partitioning of one composite over GPUs).
    out = torch.empty((2, mb, n), dtype=torch.float64, device="cuda")
    xy_h = pin[1][:n_dec].numpy().copy()
    uv_h = pin[2][:n_dec].numpy().copy()
    if np.any(~np.isfinite(uv_h)):
        raise ValueError("argument 'values' contains non-finite values")
    if np.any(~np.isfinite(xy_h)):
        raise ValueError("argument 'xy_coord' contains non-finite values")
    if not _idw_constant(out, uv_h):
        if n < 2 or m < 2:
            raise ValueError("Shape of array too small to calculate a numerical gradient, "
                             "at least (edge_order + 1) elements are required.")
        xgrid, ygrid = _pixel_grid(0, n), _pixel_grid(r0, r1)
        # the integer pixel grid holds the key level while max(m, n) < 16384
        level = _key_level(xy_h, lambda: 2 if max(m, n) < 16384 else 0)
        _idw_fill(dec_xy, dec_uv, n_dec, 2, k, power, dist_offset, 1.0, xgrid, n, ygrid, mb, level, out)

    if verbose:
        torch.cuda.current_stream().synchronize()
        print("--- total time: %.2f seconds ---" % (time.time() - t0))
    # a weighted mean of finite vectors with weights (d + dist_offset)^-power, d >= 0: finite whenever
    # the offset is positive (the default 0.5); the consumer then skips its finiteness scan of the copy
    finite = bool(dense and dist_offset > 0.0 and 0.0 <= power <= 8.0)
    if on_device:
        if finite:
            # a device result the caller may edit: the certificate holds for THIS version of the tensor only
            # (torch bumps ._version on every in-place write, through views too)
            out._b200_finite_version = out._version
        return out
    return _device.remember_result(_device.to_host(out), out, finite=finite)
