"""Oracle mirror of ``pysteps.motion.lucaskanade.dense_lucaskanade`` and the
helpers it calls -- TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

pysteps' own Python logic is restated in NumPy, each function citing the
reference lines it follows.  The OpenCV calls (third-party, unpinned:
requirements.txt:2; binary here: opencv-python 4.13.0) are restated from
OpenCV's published algorithms in ``lk_oracle.c`` / below and pinned against the
cv2 binary bit-for-bit (tests/test_oracle_lk.py).  The SciPy cKDTree queries
are restated as exhaustive searches.  Nothing here imports cv2 or scipy.
"""
import ctypes

import numpy as np
from numpy.ma.core import MaskedArray

from . import lib

_u8p = ctypes.POINTER(ctypes.c_uint8)
_i16p = ctypes.POINTER(ctypes.c_int16)
_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)


# ----------------------------------------------------------------------------- OpenCV pieces
def morph_open_cross3(b):
    """cv2.morphologyEx(b, MORPH_OPEN, getStructuringElement(MORPH_ELLIPSE,(3,3))) on a
    0/1 uint8 image: the 3x3 'ellipse' is the cross; erosion ignores out-of-image taps
    (border = max), dilation ignores them too (border = min)."""
    def nb(a, fill, op):
        p = np.pad(a, 1, constant_values=fill)
        r = p[1:-1, 1:-1].copy()
        for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
            r = op(r, p[1 + dy:p.shape[0] - 1 + dy, 1 + dx:p.shape[1] - 1 + dx])
        return r
    return nb(nb(b, 255, np.minimum), 0, np.maximum)


def dilate_rect(mask, k):
    """cv2.dilate(mask, np.ones((k,k))) (anchor at the centre, out-of-image ignored)."""
    r = k // 2
    p = np.pad(mask, ((r, k - 1 - r), (r, k - 1 - r)))
    out = np.zeros_like(mask)
    m, n = mask.shape
    for dy in range(k):
        for dx in range(k):
            out = np.maximum(out, p[dy:dy + m, dx:dx + n])
    return out


def corner_min_eigen_val(q):
    """cv2.cornerMinEigenVal(q, blockSize=5, ksize=3) -> float32 (m,n)."""
    q = np.ascontiguousarray(q, dtype=np.uint8)
    h, w = q.shape
    eig = np.empty((h, w), dtype=np.float32)
    L = lib()
    L.ora_min_eig_u8.restype = None
    L.ora_min_eig_u8.argtypes = [_u8p, ctypes.c_int, ctypes.c_int, _f32p]
    L.ora_min_eig_u8(q.ctypes.data_as(_u8p), h, w, eig.ctypes.data_as(_f32p))
    return eig


def good_features_to_track(q, mask, max_corners=1000, quality_level=0.01, min_distance=10,
                           eig=None):
    """cv2.goodFeaturesToTrack(q, maxCorners, qualityLevel, minDistance, mask, blockSize=5)
    -> (P,2) float32 (x, y): threshold at quality*max over the mask, 3x3 local maxima off
    the 1-px border, sort by value descending (ties: larger raster address first), greedy
    acceptance with squared distance >= minDistance^2 to every accepted corner.  Like cv2 the
    threshold minDistance^2 is formed in double and compared with the float sum
    dx*dx + dy*dy; that sum is the exact integer up to 2^24 and rounds above it."""
    if eig is None:
        eig = corner_min_eigen_val(q)
    H, W = eig.shape
    sel = eig if mask is None else eig[mask != 0]
    if sel.size == 0:
        return np.empty((0, 2), dtype=np.float32)
    mx = sel.max()
    thr = np.float32(np.float64(mx) * quality_level)
    e = np.where(eig > thr, eig, np.float32(0))
    p = np.pad(e, 1, constant_values=-np.inf)
    dil = e.copy()
    for dy in range(3):
        for dx in range(3):
            dil = np.maximum(dil, p[dy:dy + H, dx:dx + W])
    cand = (e != 0) & (e == dil)
    if mask is not None:
        cand &= mask != 0
    cand[0, :] = cand[-1, :] = False
    cand[:, 0] = cand[:, -1] = False
    ys, xs = np.nonzero(cand)
    vals = e[ys, xs]
    addr = ys.astype(np.int64) * W + xs
    order = np.lexsort((-addr, -vals.astype(np.float64)))
    ys, xs = ys[order], xs[order]
    out = []
    if min_distance >= 1:
        cell = int(round(min_distance))
        gw, gh = (W + cell - 1) // cell, (H + cell - 1) // cell
        grid = {}
        md2 = float(min_distance) * float(min_distance)
        for y, x in zip(ys.tolist(), xs.tolist()):
            xc, yc = x // cell, y // cell
            good = True
            for yy in range(max(0, yc - 1), min(gh - 1, yc + 1) + 1):
                for xx in range(max(0, xc - 1), min(gw - 1, xc + 1) + 1):
                    for (px, py) in grid.get((yy, xx), ()):
                        d2 = (x - px) ** 2 + (y - py) ** 2
                        if d2 > 1 << 24:  # float squares, float sum
                            d2 = float(np.float32((x - px) ** 2) + np.float32((y - py) ** 2))
                        if d2 < md2:
                            good = False
                            break
                    if not good:
                        break
                if not good:
                    break
            if good:
                grid.setdefault((yc, xc), []).append((x, y))
                out.append((x, y))
                if max_corners > 0 and len(out) == max_corners:
                    break
    else:
        for y, x in zip(ys.tolist(), xs.tolist()):
            out.append((x, y))
            if max_corners > 0 and len(out) == max_corners:
                break
    return np.array(out, dtype=np.float32).reshape(-1, 2)


def pyr_down(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    h, w = a.shape
    out = np.empty(((h + 1) // 2, (w + 1) // 2), np.uint8)
    L = lib()
    L.ora_pyrdown_u8.restype = None
    L.ora_pyrdown_u8.argtypes = [_u8p, ctypes.c_int, ctypes.c_int, _u8p]
    L.ora_pyrdown_u8(a.ctypes.data_as(_u8p), h, w, out.ctypes.data_as(_u8p))
    return out


def scharr_deriv(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    h, w = a.shape
    out = np.empty((h, w, 2), np.int16)
    L = lib()
    L.ora_scharr_i16.restype = None
    L.ora_scharr_i16.argtypes = [_u8p, ctypes.c_int, ctypes.c_int, _i16p]
    L.ora_scharr_i16(a.ctypes.data_as(_u8p), h, w, out.ctypes.data_as(_i16p))
    return out


def calc_optical_flow_pyr_lk(I0, J0, pts, win=(50, 50), max_level=3, criteria=(3, 10, 0),
                             min_eig_thr=1e-4):
    """cv2.calcOpticalFlowPyrLK(I0, J0, pts, None, winSize, maxLevel, criteria, flags=0,
    minEigThreshold) -> (next_pts (P,2) float32, status (P,) uint8)."""
    ctype, max_count, eps = criteria
    max_count = min(max(int(max_count), 0), 100) if (ctype & 1) else 30
    eps = min(max(float(eps), 0.0), 10.0) if (ctype & 2) else 0.01
    Is = [np.ascontiguousarray(I0, dtype=np.uint8)]
    Js = [np.ascontiguousarray(J0, dtype=np.uint8)]
    lv = 0
    for _ in range(max_level):
        h, w = Is[-1].shape
        nh, nw = (h + 1) // 2, (w + 1) // 2
        if nw <= win[0] or nh <= win[1]:
            break
        Is.append(pyr_down(Is[-1]))
        Js.append(pyr_down(Js[-1]))
        lv += 1
    n = len(pts)
    prev = np.ascontiguousarray(pts, dtype=np.float32).reshape(n, 2)
    nxt = np.zeros((n, 2), np.float32)
    st = np.ones(n, np.uint8)
    err = np.zeros(n, np.float32)
    L = lib()
    L.ora_lk_level.restype = None
    L.ora_lk_level.argtypes = [_u8p, _u8p, _i16p, ctypes.c_int, ctypes.c_int, _f32p, _f32p, _u8p,
                               _f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                               ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double]
    for level in range(lv, -1, -1):
        I, J = Is[level], Js[level]
        dI = scharr_deriv(I)
        h, w = I.shape
        L.ora_lk_level(I.ctypes.data_as(_u8p), J.ctypes.data_as(_u8p), dI.ctypes.data_as(_i16p),
                       h, w, prev.ctypes.data_as(_f32p), nxt.ctypes.data_as(_f32p),
                       st.ctypes.data_as(_u8p), err.ctypes.data_as(_f32p), n, win[0], win[1],
                       level, lv, max_count, eps * eps, float(min_eig_thr))
    return nxt, st


# ----------------------------------------------------------------------------- pysteps pieces
def _quantise_u8(img):
    """scale between 0 and 255 + astype('uint8') of a MaskedArray (shitomasi.py:143-151,
    tracking/lucaskanade.py:144-160).  The float->uint8 cast truncates toward zero and, as
    NumPy does on x86-64, wraps out-of-range values through int32."""
    im_min = img.min()
    im_max = img.max()
    if im_max - im_min > 1e-8:
        out = (img.filled() - im_min) / (im_max - im_min) * 255
    else:
        out = img.filled() - im_min
    with np.errstate(invalid="ignore"):
        return np.trunc(out).astype(np.int64).astype(np.uint8)


def morph_opening(input_image, thr, n):
    """pysteps/utils/images.py:27-86 (n == 3 only)."""
    if n != 3:
        raise NotImplementedError("oracle restates size_opening=3 only")
    input_image = input_image.copy()
    to_ndarray = False
    if not isinstance(input_image, MaskedArray):
        to_ndarray = True
        input_image = np.ma.masked_invalid(input_image)
    np.ma.set_fill_value(input_image, input_image.min())
    field_bin = np.ndarray.astype(input_image.filled() > thr, "uint8")
    field_bin_out = morph_open_cross3(field_bin)
    mask = (field_bin - field_bin_out) > 0
    input_image[mask] = input_image.min()  # np.nanmin of the masked array
    if to_ndarray:
        input_image = np.array(input_image)
    return input_image


def detection_image(input_image, buffer_mask=5):
    """The uint8 image and the validity mask that shitomasi.detection hands to
    cv2.goodFeaturesToTrack (pysteps/feature/shitomasi.py:119-152)."""
    input_image = input_image.copy()
    if input_image.ndim != 2:
        raise ValueError("input_image must be a two-dimensional array")
    if not isinstance(input_image, MaskedArray):
        input_image = np.ma.masked_invalid(input_image)
    np.ma.set_fill_value(input_image, input_image.min())
    mask = np.ma.getmaskarray(input_image).astype("uint8")
    if buffer_mask > 0:
        mask = dilate_rect(mask, int(buffer_mask))
        # NOTE (reference quirk, shitomasi.py:139): `mask` is uint8, so this is INTEGER
        # indexing -- it masks rows 0 and/or 1, not the buffered pixels.  Kept as is.
        input_image[mask] = np.ma.masked
    input_image = _quantise_u8(input_image)
    mask = ~mask & 1
    return input_image, mask


def detection(input_image, max_corners=1000, max_num_features=None, quality_level=0.01,
              min_distance=10, block_size=5, buffer_mask=5, use_harris=False, k=0.04,
              verbose=False, **kwargs):
    """pysteps/feature/shitomasi.py:26-171."""
    if use_harris or block_size != 5:
        raise NotImplementedError("oracle restates the default detector only")
    input_image, mask = detection_image(input_image, buffer_mask)
    points = good_features_to_track(
        input_image, mask, max_num_features if max_num_features is not None else max_corners,
        quality_level, min_distance)
    return points


def tracking_image(img):
    """The uint8 image track_features hands to cv2.calcOpticalFlowPyrLK
    (pysteps/tracking/lucaskanade.py:134-160)."""
    img = img.copy()
    if not isinstance(img, MaskedArray):
        img = np.ma.masked_invalid(img)
    np.ma.set_fill_value(img, img.min())
    return _quantise_u8(img)


def track_features(prvs_image, next_image, points, winsize=(50, 50), nr_levels=3,
                   criteria=(3, 10, 0), flags=0, min_eig_thr=1e-4, verbose=False):
    """pysteps/tracking/lucaskanade.py:35-189."""
    prvs_img = prvs_image.copy()
    next_img = next_image.copy()
    p0 = np.copy(points)
    if not isinstance(prvs_img, MaskedArray):
        prvs_img = np.ma.masked_invalid(prvs_img)
    np.ma.set_fill_value(prvs_img, prvs_img.min())
    if not isinstance(next_img, MaskedArray):
        next_img = np.ma.masked_invalid(next_img)
    np.ma.set_fill_value(next_img, next_img.min())
    prvs_img = _quantise_u8(prvs_img)
    next_img = _quantise_u8(next_img)
    p1, st = calc_optical_flow_pyr_lk(prvs_img, next_img, p0, winsize, nr_levels, criteria,
                                      min_eig_thr)
    st = np.atleast_1d(st.squeeze()) == 1
    if np.any(st):
        p1 = p1[st, :]
        p0 = p0[st, :]
        xy = p0
        uv = p1 - p0
    else:
        xy = uv = np.empty(shape=(0, 2))
    return xy, uv


# How equidistant / coincident neighbours are chosen and ordered by the two k-NN users
# (detect_outliers, idwinterp2d):
#   "ckdtree" (default) -- exactly as scipy.spatial.cKDTree returns them (oracle/ckdtree.py): with
#                          it the whole of dense_lucaskanade is bit-identical to the reference
#                          (tests/test_oracle_lk.py); the CUDA path follows the same order
#                          (csrc/knn.cu);
#   "lower_index"       -- ascending distance, ties by lower index (an exhaustive scan without a
#                          tree; OpenMP C for the grid fill, ~3x faster): a valid k-NN set that
#                          differs from the reference's only at exact distance ties.  Used as the
#                          CPU timing baseline of bench.py and by the tests that isolate the tie rule.
_KNN_MODE = ["ckdtree"]


class knn_mode:
    """with knn_mode("ckdtree"): ..."""

    def __init__(self, mode):
        assert mode in ("lower_index", "ckdtree")
        self.mode = mode

    def __enter__(self):
        self.prev = _KNN_MODE[0]
        _KNN_MODE[0] = self.mode

    def __exit__(self, *exc):
        _KNN_MODE[0] = self.prev


def _knn_bruteforce(coord, k):
    """scipy.spatial.cKDTree(coord).query(coord, k)[1]: exhaustive, ascending distance,
    ties by lower index."""
    d2 = ((coord[:, None, :] - coord[None, :, :]) ** 2).sum(axis=2)
    return np.argsort(d2, axis=1, kind="stable")[:, :k]


def detect_outliers(input_array, thr, coord=None, k=None, verbose=False):
    """pysteps/utils/cleansing.py:124-249 (multivariate local branch and the global
    branches used by dense_lucaskanade)."""
    input_array = np.copy(input_array)
    if np.any(~np.isfinite(input_array)):
        raise ValueError("input_array contains non-finite values")
    if input_array.ndim == 1:
        nvar = 1
    elif input_array.ndim == 2:
        nvar = input_array.shape[1]
    else:
        raise ValueError(f"input_array must have 1 (n) or 2 dimensions (n, m), but it has {coord.ndim}")
    if nvar < 2:
        input_array = input_array.reshape(-1, 1) if input_array.ndim == 2 else input_array
    nsamples = input_array.shape[0]
    if nsamples < 2:
        return np.zeros(nsamples, dtype=bool)
    if coord is not None and k is not None:
        coord = np.copy(coord)
        if coord.ndim == 1:
            coord = coord[:, None]
        k = np.min((nsamples, k + 1))
    if k is None or coord is None:
        zdata = input_array - np.mean(input_array, axis=0)
        V = np.cov(zdata.T)
        try:
            VI = np.linalg.inv(V)
            MD = np.sqrt(np.dot(np.dot(zdata, VI), zdata.T).diagonal())
        except np.linalg.LinAlgError:
            MD = np.zeros(nsamples)
        return MD > thr
    if _KNN_MODE[0] == "ckdtree":
        from .ckdtree import KDTree
        __, inds = KDTree(coord).query(coord, k=int(k))       # cleansing.py:219-220
        inds = inds.reshape(nsamples, -1)
    else:
        inds = _knn_bruteforce(coord.astype(np.float64), k)
    outliers = np.empty(nsamples, dtype=bool)
    for i in range(nsamples):
        thisdata = input_array[i, :]
        neighbours = input_array[inds[i, 1:], :].copy()
        thiszdata = thisdata - np.mean(neighbours, axis=0)
        neighbours = neighbours - np.mean(neighbours, axis=0)
        V = np.cov(neighbours.T)
        try:
            VI = np.linalg.inv(V)
            MD = np.sqrt(np.dot(np.dot(thiszdata, VI), thiszdata.T))
        except np.linalg.LinAlgError:
            MD = 0
        outliers[i] = MD > thr
    return outliers


def decluster(coord, input_array, scale, min_samples=1, verbose=False):
    """pysteps/utils/cleansing.py:21-121."""
    coord = np.copy(coord)
    input_array = np.copy(input_array)
    scale = float(scale)
    coord_ = np.floor(coord / scale)
    ucoord_ = np.unique(coord_, axis=0)
    nvar = input_array.shape[1]
    dinput = np.empty(shape=(0, nvar))
    dcoord = np.empty(shape=(0, coord.shape[1]))
    for i in range(ucoord_.shape[0]):
        idx = np.all(coord_ == ucoord_[i, :], axis=1)
        npoints = np.sum(idx)
        if npoints >= min_samples:
            dinput = np.append(dinput, np.median(input_array[idx, :], axis=0)[None, :], axis=0)
            dcoord = np.append(dcoord, np.median(coord[idx, :], axis=0)[None, :], axis=0)
    return dcoord, dinput


def idwinterp2d(xy_coord, values, xgrid, ygrid, power=0.5, k=20, dist_offset=0.5,
                return_ties=False, **kwargs):
    """pysteps/utils/interpolate.py:26-114 behind pysteps/decorators.py:153-250
    (the chunking of the target grid does not change results and is not restated).
    return_ties=True additionally returns the mask of grid points whose k-th and (k+1)-th
    neighbours are exactly equidistant: there scipy's cKDTree picks by traversal order, the
    restatement by lower index, and the two may legitimately differ."""
    values = np.array(values, dtype=np.float64)
    xy_coord = np.array(xy_coord, dtype=np.float64)
    input_ndims = values.ndim
    input_nvars = 1 if input_ndims == 1 else values.shape[1]
    grid_shape = (ygrid.size, xgrid.size)
    if np.any(~np.isfinite(values)):
        raise ValueError("argument 'values' contains non-finite values")
    if np.any(~np.isfinite(xy_coord)):
        raise ValueError("argument 'xy_coord' contains non-finite values")
    if values.shape[0] == 1:  # decorators.py:200-204
        output_array = np.ones((input_nvars,) + grid_shape)
        for n, v in enumerate(values[0, ...]):
            output_array[n, ...] *= v
        return output_array.squeeze()
    if values.max() == values.min():  # decorators.py:207-208
        return np.ones((input_nvars,) + grid_shape) * values.ravel()[0]
    if values.ndim == 1:
        values = values[:, None]
    npoints, nvar = values.shape
    if _KNN_MODE[0] == "ckdtree" and k is not None and not return_ties:
        # interpolate.py:67-114 verbatim, with the restated tree in place of scipy's
        from .ckdtree import KDTree
        xgridv, ygridv = np.meshgrid(xgrid, ygrid)
        gridv = np.column_stack((xgridv.ravel(), ygridv.ravel()))
        kk = int(np.min((k, npoints)))
        dist, inds = KDTree(xy_coord).query(gridv, k=kk)
        if dist.ndim == 1:
            dist = dist[..., None]
            inds = inds[..., None]
        mean_res = np.mean(np.abs([np.gradient(xgrid).mean(), np.gradient(ygrid).mean()]))
        dist /= mean_res
        dist += dist_offset
        weights = 1 / np.power(dist, power)
        weights = weights / np.sum(weights, axis=1, keepdims=True)
        output_array = np.sum(values[inds, :] * weights[..., None], axis=1)
        output_array = output_array.reshape(ygrid.size, xgrid.size, nvar)
        return np.moveaxis(output_array, -1, 0).squeeze()
    k = npoints if k is None else int(min(k, npoints))
    x_res = np.gradient(xgrid)
    y_res = np.gradient(ygrid)
    mean_res = np.mean(np.abs([x_res.mean(), y_res.mean()]))
    gx = np.ascontiguousarray(xgrid, dtype=np.float64)
    gy = np.ascontiguousarray(ygrid, dtype=np.float64)
    out = np.empty((nvar, gy.size, gx.size))
    L = lib()
    L.ora_idw.restype = None
    L.ora_idw.argtypes = [_f64p, _f64p, ctypes.c_int, ctypes.c_int, _f64p, ctypes.c_int, _f64p,
                          ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double,
                          ctypes.c_double, _f64p, _u8p]
    tie = np.zeros((gy.size, gx.size), dtype=np.uint8) if return_ties else None
    xyc = np.ascontiguousarray(xy_coord)
    vc = np.ascontiguousarray(values)
    L.ora_idw(xyc.ctypes.data_as(_f64p), vc.ctypes.data_as(_f64p), npoints, nvar,
              gx.ctypes.data_as(_f64p), gx.size, gy.ctypes.data_as(_f64p), gy.size, k,
              float(power), float(dist_offset), float(mean_res), out.ctypes.data_as(_f64p),
              None if tie is None else tie.ctypes.data_as(_u8p))
    if return_ties:
        return out.squeeze(), tie.astype(bool)
    return out.squeeze()


def dense_lucaskanade(input_images, lk_kwargs=None, fd_method="shitomasi", fd_kwargs=None,
                      interp_method="idwinterp2d", interp_kwargs=None, dense=True,
                      nr_std_outlier=3, k_outlier=30, size_opening=3, decl_scale=20,
                      verbose=False):
    """pysteps/motion/lucaskanade.py:38-279 (behind decorators.check_input_frames)."""
    if input_images.ndim != 3:
        raise ValueError("input_images dimension mismatch.\n"
                         f"input_images.shape: {str(input_images.shape)}\n"
                         "(t, x, y ) dimensions expected")
    if fd_method != "shitomasi" or interp_method != "idwinterp2d":
        raise NotImplementedError("oracle restates the default methods only")
    input_images = input_images.copy()
    nr_fields = input_images.shape[0]
    domain_size = (input_images.shape[1], input_images.shape[2])
    fd_kwargs = dict() if fd_kwargs is None else fd_kwargs
    lk_kwargs = dict() if lk_kwargs is None else lk_kwargs
    interp_kwargs = dict() if interp_kwargs is None else interp_kwargs
    xy = np.empty(shape=(0, 2))
    uv = np.empty(shape=(0, 2))
    for n in range(nr_fields - 1):
        prvs_img = input_images[n, :, :].copy()
        next_img = input_images[n + 1, :, :].copy()
        if not isinstance(prvs_img, MaskedArray):
            prvs_img = np.ma.masked_invalid(prvs_img)
        np.ma.set_fill_value(prvs_img, prvs_img.min())
        if not isinstance(next_img, MaskedArray):
            next_img = np.ma.masked_invalid(next_img)
        np.ma.set_fill_value(next_img, next_img.min())
        if size_opening > 0:
            prvs_img = morph_opening(prvs_img, prvs_img.min(), size_opening)
            next_img = morph_opening(next_img, next_img.min(), size_opening)
        points = detection(prvs_img, **fd_kwargs).astype(np.float32)
        if points.shape[0] == 0:
            continue
        xy_, uv_ = track_features(prvs_img, next_img, points, **lk_kwargs)
        if xy_.shape[0] == 0:
            continue
        xy = np.append(xy, xy_, axis=0)
        uv = np.append(uv, uv_, axis=0)
    if xy.shape[0] == 0:
        if dense:
            return np.zeros((2, domain_size[0], domain_size[1]))
        return xy, uv
    outliers = detect_outliers(uv, nr_std_outlier, xy, k_outlier, verbose)
    xy = xy[~outliers, :]
    uv = uv[~outliers, :]
    if not dense:
        return xy, uv
    if decl_scale > 1:
        xy, uv = decluster(xy, uv, decl_scale, 1, verbose)
    if xy.shape[0] == 0:
        return np.zeros((2, domain_size[0], domain_size[1]))
    xgrid = np.arange(domain_size[1])
    ygrid = np.arange(domain_size[0])
    return idwinterp2d(xy, uv, xgrid, ygrid, **interp_kwargs)
