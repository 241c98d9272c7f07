"""Stand-alone B200 mirrors of the helper functions dense_lucaskanade is built from
(SURVEY.md section 8a rows a5-a11).  Same names, arguments and return conventions as the
reference functions; NumPy in, NumPy out; every array operation is a kernel of
libpysteps_b200.so.

  morph_opening    pysteps/utils/images.py:27-86
  detection        pysteps/feature/shitomasi.py:26-171
  track_features   pysteps/tracking/lucaskanade.py:35-189
  detect_outliers  pysteps/utils/cleansing.py:124-249   (coord + k given, multivariate)
  decluster        pysteps/utils/cleansing.py:21-121
  idwinterp2d      pysteps/utils/interpolate.py:26-114  (behind decorators.prepare_interpolator)
"""
import numpy as np
import torch
from numpy.ma.core import MaskedArray

from . import _device, _lib
from .motion import lucaskanade as _lk


def _s():
    return _device.stream_ptr()


def _is_f32(image):
    return np.asarray(image).dtype == np.float32


def _frame(image):
    """(device image float64, device user mask or None) of an ndarray / MaskedArray."""
    if isinstance(image, MaskedArray):
        um = _device.to_device(np.ascontiguousarray(np.ma.getmaskarray(image), dtype=np.uint8))
        img = _device.to_device(np.ascontiguousarray(image.data), torch.float64)
        return img, um
    return _device.to_device(np.asarray(image), torch.float64), None


def morph_opening(input_image, thr, n):
    """Binary opening (3x3 cross) of ``input_image > thr``; removed pixels take the minimum."""
    _device.require_cuda()
    if n != 3:
        raise NotImplementedError("pysteps_b200 morph_opening: only n=3 is implemented")
    to_ndarray = not isinstance(input_image, MaskedArray)
    m, k = input_image.shape
    img, um = _frame(input_image)
    mask = torch.empty((m, k), dtype=torch.uint8, device="cuda")
    st0 = torch.empty(3, dtype=torch.float64, device="cuda")
    _lib.call("b200_mask_invalid", img.data_ptr(), _device.ptr(um), m, k, mask.data_ptr(), st0.data_ptr(), _s())
    thr_d = torch.tensor([float(thr)], dtype=torch.float64, device="cuda")
    out = torch.empty((m, k), dtype=torch.float64, device="cuda")
    _lib.call("b200_morph_opening", img.data_ptr(), mask.data_ptr(), m, k, 3, thr_d.data_ptr(),
              st0.data_ptr(), out.data_ptr(), _s())
    data = out.cpu().numpy()
    if to_ndarray:
        return data
    res = np.ma.MaskedArray(data, mask=mask.cpu().numpy().astype(bool))
    np.ma.set_fill_value(res, input_image.min())
    return res


def detection(input_image, max_corners=1000, max_num_features=None, quality_level=0.01,
              min_distance=10, block_size=5, buffer_mask=5, use_harris=False, k=0.04,
              verbose=False, **kwargs):
    """Shi-Tomasi corners (x, y) of an image, float32 (P, 2)."""
    _device.require_cuda()
    if input_image.ndim != 2:
        raise ValueError("input_image must be a two-dimensional array")
    if block_size != 5 or use_harris:
        raise NotImplementedError("pysteps_b200 detection: only block_size=5, use_harris=False")
    maxc = int(max_num_features if max_num_features is not None else max_corners)
    if maxc <= 0:
        raise NotImplementedError("pysteps_b200 detection: max_corners must be positive")
    m, n = input_image.shape
    img, um = _frame(input_image)
    f = _lk._Frame(img, um, m, n, 0, _is_f32(input_image))
    _lk._prepare_frame(f, m, n, 0)
    st = _lk._frame_stats(f, m, n, int(buffer_mask))
    q = torch.empty((m, n), dtype=torch.uint8, device="cuda")
    valid = torch.empty((m, n), dtype=torch.uint8, device="cuda")
    _lib.call("b200_quantise_u8", f.opened.data_ptr(), f.mask.data_ptr(), m, n, 1 | f.qflag, int(buffer_mask),
              st.data_ptr(), st.data_ptr(), q.data_ptr(), valid.data_ptr(), _s())
    eig = torch.empty((m, n), dtype=torch.float32, device="cuda")
    _lib.call("b200_min_eig", q.data_ptr(), m, n, eig.data_ptr(), _s())
    corners = torch.empty((maxc, 2), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.call("b200_good_features", eig.data_ptr(), valid.data_ptr(), m, n, maxc, float(quality_level),
              float(min_distance), corners.data_ptr(), cnt.data_ptr(), _s())
    c = int(cnt.item())
    if c == 0:
        return np.empty(shape=(0, 2))
    pts = corners[:c].cpu().numpy()
    if verbose:
        print(f"--- {pts.shape[0]} good features to track detected ---")
    return pts


def track_features(prvs_image, next_image, points, winsize=(50, 50), nr_levels=3,
                   criteria=(3, 10, 0), flags=0, min_eig_thr=1e-4, verbose=False):
    """Pyramidal Lucas-Kanade tracking of `points` from prvs_image to next_image -> (xy, uv)."""
    _device.require_cuda()
    if flags != 0:
        raise NotImplementedError("pysteps_b200 track_features: flags must be 0")
    m, n = prvs_image.shape
    win_w, win_h, nr_levels, max_count, eps = _lk._tracker_args(winsize, nr_levels, criteria)
    p0 = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 2)
    npts = p0.shape[0]
    if npts == 0:
        return np.empty(shape=(0, 2)), np.empty(shape=(0, 2))
    lv, total = _lk._pyramid_layout(m, n, (win_w, win_h), nr_levels)
    pyrs = []
    for image, deriv in ((prvs_image, True), (next_image, False)):
        img, um = _frame(image)
        f = _lk._Frame(img, um, m, n, 0, _is_f32(image))
        _lk._prepare_frame(f, m, n, 0)
        q = _lk._track_image(f, m, n, 0)
        P = torch.empty(total, dtype=torch.uint8, device="cuda")
        D = torch.empty(2 * total, dtype=torch.int16, device="cuda") if deriv else None
        _lib.call("b200_lk_build_pyramid", q.data_ptr(), m, n, win_w, win_h, nr_levels, P.data_ptr(),
                  _device.ptr(D), _s())
        pyrs.append((P, D, f))
    d0 = _device.to_device(p0)
    d1 = torch.empty((npts, 2), dtype=torch.float32, device="cuda")
    st = torch.empty(npts, dtype=torch.uint8, device="cuda")
    _lib.call("b200_lk_track", pyrs[0][0].data_ptr(), pyrs[1][0].data_ptr(), pyrs[0][1].data_ptr(), m, n,
              win_w, win_h, nr_levels, max_count, eps, float(min_eig_thr),
              d0.data_ptr(), npts, None, d1.data_ptr(), st.data_ptr(), _s())
    p1 = d1.cpu().numpy()
    keep = st.cpu().numpy() == 1
    if np.any(keep):
        xy = p0[keep, :]
        uv = p1[keep, :] - p0[keep, :]
    else:
        xy = uv = np.empty(shape=(0, 2))
    if verbose:
        print(f"--- {xy.shape[0]} sparse vectors found ---")
    return xy, uv


def detect_outliers(input_array, thr, coord=None, k=None, verbose=False):
    """Local multivariate (Mahalanobis) outlier flags of (n, 2) vectors at (n, 2) coordinates."""
    _device.require_cuda()
    input_array = np.copy(input_array)
    if np.any(~np.isfinite(input_array)):
        raise ValueError("input_array contains non-finite values")
    if input_array.ndim != 2 or input_array.shape[1] != 2:
        raise NotImplementedError("pysteps_b200 detect_outliers: (n, 2) vectors only")
    if coord is None or k is None:
        # global test (cleansing.py:201-214)
        nsamples = input_array.shape[0]
        if nsamples < 2:
            return np.zeros(nsamples, dtype=bool)
        duv = _device.to_device(np.ascontiguousarray(input_array, dtype=np.float64))
        flags = torch.empty(nsamples, dtype=torch.uint8, device="cuda")
        _lib.call("b200_detect_outliers_global", duv.data_ptr(), None, nsamples, float(thr), flags.data_ptr(), _s())
        out = flags.cpu().numpy().astype(bool)
        if verbose:
            print(f"--- {np.sum(out)} outliers detected ---")
        return out
    coord = np.copy(coord)
    if coord.ndim != 2 or coord.shape[1] != 2:
        raise NotImplementedError("pysteps_b200 detect_outliers: (n, 2) coordinates only")
    nsamples = input_array.shape[0]
    if coord.shape[0] != nsamples:
        raise ValueError("the number of samples in input_array does not match the "
                         f"number of coordinates {nsamples}!={coord.shape[0]}")
    if nsamples < 2:
        return np.zeros(nsamples, dtype=bool)
    duv = _device.to_device(np.ascontiguousarray(input_array, dtype=np.float64))
    dxy = _device.to_device(np.ascontiguousarray(coord, dtype=np.float64))
    flags = torch.empty(nsamples, dtype=torch.uint8, device="cuda")
    _lib.call("b200_detect_outliers",
              duv.data_ptr(), dxy.data_ptr(), None, nsamples, float(thr), int(k), flags.data_ptr(), _s())
    out = flags.cpu().numpy().astype(bool)
    if verbose:
        print(f"--- {np.sum(out)} outliers detected ---")
    return out


def decluster(coord, input_array, scale, min_samples=1, verbose=False):
    """Per-cell medians of (n, 2) vectors and coordinates -> (dcoord, dinput)."""
    _device.require_cuda()
    coord = np.copy(coord)
    input_array = np.copy(input_array)
    if np.any(~np.isfinite(input_array)):
        raise ValueError("input_array contains non-finite values")
    if input_array.ndim != 2 or input_array.shape[1] != 2 or coord.ndim != 2 or coord.shape[1] != 2:
        raise NotImplementedError("pysteps_b200 decluster: (n, 2) coordinates and (n, 2) values only")
    if coord.shape[0] != input_array.shape[0]:
        raise ValueError("the number of samples in the input_array does not match the "
                         + "number of coordinates %i!=%i" % (input_array.shape[0], coord.shape[0]))
    if not np.isscalar(scale):
        raise NotImplementedError("pysteps_b200 decluster: scalar scale only")
    n = coord.shape[0]
    if n == 0:
        return np.empty((0, 2)), np.empty((0, 2))
    dxy = _device.to_device(np.ascontiguousarray(coord, dtype=np.float64))
    duv = _device.to_device(np.ascontiguousarray(input_array, dtype=np.float64))
    oxy = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    ouv = torch.empty((n, 2), dtype=torch.float64, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.call("b200_decluster", dxy.data_ptr(), duv.data_ptr(), None, n, float(scale), int(min_samples),
              oxy.data_ptr(), ouv.data_ptr(), cnt.data_ptr(), _s())
    c = int(cnt.item())
    if c < 0:
        raise ValueError("pysteps_b200 decluster: a cell floor(coord / scale) lies outside [1 - 2**24, 2**24 - 2], "
                         "or coord has NaN values and min_samples < 1")
    if verbose:
        print("--- %i samples left after declustering ---" % c)
    return oxy[:c].cpu().numpy(), ouv[:c].cpu().numpy()


def idwinterp2d(xy_coord, values, xgrid, ygrid, power=0.5, k=20, dist_offset=0.5, **kwargs):
    """k-nearest inverse-distance weighting of (n, m) values at (n, 2) points onto the grid
    (ygrid.size, xgrid.size) -> (m, ny, nx) (squeezed).  A CUDA tensor for `values`/`xy_coord`
    is accepted and keeps the result on the device (used for band-partitioned fills)."""
    _device.require_cuda()
    on_device = _device.is_device_tensor(values)
    v_h = values.cpu().numpy() if on_device else np.array(values, dtype=np.float64)
    xy_h = xy_coord.cpu().numpy() if _device.is_device_tensor(xy_coord) else np.array(xy_coord, dtype=np.float64)
    input_ndims = v_h.ndim
    nvar = 1 if input_ndims == 1 else v_h.shape[1]
    ny, nx = int(np.size(ygrid)), int(np.size(xgrid))
    if np.any(~np.isfinite(v_h)):
        raise ValueError("argument 'values' contains non-finite values")
    if np.any(~np.isfinite(xy_h)):
        raise ValueError("argument 'xy_coord' contains non-finite values")
    if input_ndims > 2:
        raise ValueError("argument 'values' must have 1 (n) or 2 dimensions (n, m), "
                         f"but it has {input_ndims}")
    if xy_h.ndim != 2:
        raise ValueError("argument 'xy_coord' must have 2 dimensions (n, 2), "
                         f"but it has {xy_h.ndim}")
    if v_h.shape[0] != xy_h.shape[0]:
        raise ValueError("the number of samples in argument 'values' does not match the "
                         f"number of coordinates {v_h.shape[0]}!={xy_h.shape[0]}")
    out = torch.empty((nvar, ny, nx), dtype=torch.float64, device="cuda")
    v2 = v_h.reshape(v_h.shape[0], nvar)
    npts = v2.shape[0]
    if not _lk._idw_constant(out, v2):
        xg = np.ascontiguousarray(xgrid, dtype=np.float64)
        yg = np.ascontiguousarray(ygrid, dtype=np.float64)
        for g in (xg, yg):
            d = np.diff(g)
            if not (np.all(d >= 0) or np.all(d <= 0)):
                raise NotImplementedError("pysteps_b200 idwinterp2d: xgrid and ygrid must be monotonic")
        # decorators.py:210-236: the target grid is processed in nchunks sub-grids and the
        # pixel resolution (interpolate.py:96-99) is taken per sub-grid.  Results only depend on
        # the chunking through that resolution, so equal resolutions -> one launch.
        nchunks = int(kwargs.get("nchunks", 4) ** 0.5)
        subx = [x for x in np.array_split(xg, nchunks) if x.size > 0] if nchunks > 1 else [xg]
        suby = [y for y in np.array_split(yg, nchunks) if y.size > 0] if nchunks > 1 else [yg]
        res = [[float(np.mean(np.abs([np.gradient(sx).mean(), np.gradient(sy).mean()]))) for sy in suby]
               for sx in subx]

        def grid_level():  # the target grid's key level (motion.lucaskanade._key_level)
            if not (np.all(xg * 16.0 == np.rint(xg * 16.0)) and np.all(yg * 16.0 == np.rint(yg * 16.0))
                    and max(np.abs(xg).max(), np.abs(yg).max()) < 16384.0):
                return 0
            return 2 if np.all(xg == np.rint(xg)) and np.all(yg == np.rint(yg)) else 1

        level = _lk._key_level(xy_h, grid_level)
        dxy = _device.to_device(np.ascontiguousarray(xy_h))
        dv = _device.to_device(np.ascontiguousarray(v2))

        def fill(gx, gy, mean_res, dst):
            dgx, dgy = _device.to_device(gx), _device.to_device(gy)
            _lk._idw_fill(dxy, dv, npts, nvar, k, power, dist_offset, mean_res, dgx, gx.size, dgy, gy.size, level,
                          dst)

        if len({r for row in res for r in row}) == 1:
            fill(xg, yg, res[0][0], out)
        else:
            indx = 0
            for sx, rrow in zip(subx, res):
                indy = 0
                for sy, r in zip(suby, rrow):
                    part = torch.empty((nvar, sy.size, sx.size), dtype=torch.float64, device="cuda")
                    fill(np.ascontiguousarray(sx), np.ascontiguousarray(sy), r, part)
                    out[:, indy:indy + sy.size, indx:indx + sx.size] = part
                    indy += sy.size
                indx += sx.size
    if on_device:
        return out.squeeze()
    return out.cpu().numpy().squeeze()
