"""B200 DARTS -- drop-in for ``pysteps.motion.darts.DARTS`` (pysteps/motion/darts.py:22-220).

The device computes what the reference's loops read: the (2N_t+1, 2(N_y+M_y)+1, 2(N_x+M_x)+1)
block of the frames' 3-D DFT (``b200_darts_spectrum``, a direct DFT at exactly those NumPy
indices), the normal equations ``MM = M^H M`` and ``M^H y`` without forming M
(``b200_darts_normal``), and the field (``b200_darts_synthesize``).  One pinned read-back brings MM
and M^H y to the host, where the reference's solve runs in NumPy with its thresholds and its
exceptions; the coefficients go back up for the field.

Deviation: ``fft_method`` "numpy", "scipy" and "pyfftw" name the same DFT and all take the device
path, so "pyfftw" works without pyfftw installed (DESIGN.md section 4).

Parity: tests/test_darts_gpu.py (device), tests/test_oracle_darts.py and
tests/test_host_logic_darts.py (oracle and host logic on the CPU).
"""
import functools
import time

import numpy as np
import torch
from numpy.linalg import lstsq, svd

from .. import _device, _lib

MAX_COLS = 242  # B200_DARTS_MAX_COLS
NORMAL_ROWS = 512  # B200_DARTS_NORMAL_ROWS

# pysteps.utils.get_method's names other than the FFTs, in the order of its error message
# (pysteps/utils/interface.py:182-237); every one of them is a plain function
UTILS_METHODS = (
    "none", "centred_coord", "decluster", "detect_outliers", "mm/h", "rainrate", "mm", "raindepth", "dbz",
    "reflectivity", "accumulate", "clip", "square", "upscale", "morph_opening", "rbfinterp2d", "idwinterp2d",
    "pca_transform", "pca_backtransform", "reproject_grids", "rapsd", "rm_rdisc", "compute_mask_window_function",
    "compute_window_function", "boxcox", "box-cox", "db", "decibel", "log", "nqt", "sqrt",
)


@functools.lru_cache(maxsize=32)
def twiddles(k, L, sign):
    """(len(k), L) complex128 table exp(sign 2 pi i ((k j) mod L) / L), k a tuple of NumPy indices
    (wrapped mod L), with the exactly reduced integer argument.  Cached; read-only."""
    r = (np.asarray(k, dtype=np.int64)[:, None] % L) * np.arange(L, dtype=np.int64)[None, :] % L
    ang = sign * 2.0 * np.pi * r / L
    out = np.empty(r.shape, dtype=np.complex128)
    out.real = np.cos(ang)
    out.imag = np.sin(ang)
    out.flags.writeable = False
    return out


def x_frequencies(K, n):
    """the frequencies f = 0 .. min(K, n // 2) of the x pass (b200_darts_spectrum)"""
    return tuple(range(min(K, n // 2) + 1))


def spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y):
    """(tw_x, tw_y, tw_t, K) of b200_darts_spectrum"""
    K, Ky = N_x + M_x, N_y + M_y
    return (twiddles(x_frequencies(K, n), n, -1), twiddles(tuple(range(-Ky, Ky + 1)), m, -1),
            twiddles(tuple(range(-N_t, N_t + 1)), T, -1), K)


def solve(MM, Mhy, lsq_method):
    """The reference's solve from the Gram matrix.  lsq_method != 1: _leastsq (darts.py:223-237) from
    its svd(MM) on.  lsq_method == 1: lstsq(M, y, rcond=0.01) keeps s(M) > 0.01 s0(M), which is
    s(MM) > 1e-4 s0(MM): lstsq(MM, M^H y, rcond=1e-4) is the pseudo-inverse on that subspace."""
    if lsq_method == 1:
        return lstsq(MM, Mhy, rcond=1e-4)[0]
    U, s, V = svd(MM, full_matrices=False)
    mask = s > 0.01 * s[0]
    s = 1.0 / s[mask]
    MM_inv = np.dot(np.dot(V[: len(s), :].conjugate().T, np.diag(s)), U[:, : len(s)].conjugate().T)
    return np.dot(MM_inv, Mhy)


def fill_tables(M_x, M_y, m, n):
    """_fill (darts.py:240-244) restated for separable synthesis: the distinct wrapped row and column
    indices the coefficients land on, and where each (h, w) coefficient goes (NumPy's fancy
    assignment decides aliased ones, the last write wins, as in the reference)."""
    k_x, k_y = np.meshgrid(np.arange(-M_x, M_x + 1), np.arange(-M_y, M_y + 1))
    rows, cols = np.unique(k_y % m), np.unique(k_x % n)
    return rows, cols, np.searchsorted(rows, k_y % m), np.searchsorted(cols, k_x % n)


def _out_of_bounds(k, L):
    return (k < -L) | (k >= L)


def _first_bad(bt, by, bx):
    """(a, b, c): the first (k_t, k_y, k_x) position of the reference's loops that fails, or None"""
    bad = bt[:, None, None] | by[None, :, None] | bx[None, None, :]
    if not bad.any():
        return None
    return np.unravel_index(int(np.argmax(bad.ravel())), bad.shape)


def index_errors(T, m, n, N_x, N_y, N_t, M_x, M_y):
    """The reference indexes the (m, n, T) spectrum with NumPy indices that wrap when negative and
    raise IndexError past the axis: -> (y_fail, h_fail), each None or a callable that raises the
    reference's IndexError by indexing a zero-stride view of that shape the same way."""
    view = np.broadcast_to(np.zeros((), dtype=complex), (m, n, T))
    kt, ky, kx = np.arange(-N_t, N_t + 1), np.arange(-N_y, N_y + 1), np.arange(-N_x, N_x + 1)
    y_bad = _first_bad(_out_of_bounds(kt, T), _out_of_bounds(ky, m), _out_of_bounds(kx, n))
    h_bad = _first_bad(np.zeros(kt.shape, bool), _out_of_bounds(ky + M_y, m) | _out_of_bounds(ky - M_y, m),
                       _out_of_bounds(kx + M_x, n) | _out_of_bounds(kx - M_x, n))

    def y_fail(a=y_bad):
        k_t_, k_y_, k_x_ = a[0] - N_t, a[1] - N_y, a[2] - N_x
        view[k_y_, k_x_, k_t_]

    def h_fail(a=h_bad):
        k_t_, k_y_, k_x_ = a[0] - N_t, a[1] - N_y, a[2] - N_x
        kp_y, kp_x = np.unravel_index(np.arange((2 * M_x + 1) * (2 * M_y + 1)), (2 * M_y + 1, 2 * M_x + 1))
        view[k_y_ - (kp_y[:] - M_y), k_x_ - (kp_x[:] - M_x), k_t_]

    return (None if y_bad is None else y_fail), (None if h_bad is None else h_fail)


def _check_fft_method(name):
    """utils.get_method(fft_method, ...) (pysteps/utils/interface.py:174-252) as DARTS uses it: the
    FFT names pass (-> None); another utils method is found, and the AttributeError returned here is
    raised where the reference calls its fftn; an unknown name raises get_method's ValueError."""
    if name is None:
        name = "none"
    name = name.lower()
    if name in ["numpy", "pyfftw", "scipy"]:
        return
    if name in UTILS_METHODS:
        return AttributeError("'function' object has no attribute 'fftn'")
    raise ValueError("Unknown method %s\n" % KeyError(name)
                     + "Supported methods:%s" % str({k: None for k in UTILS_METHODS}.keys()))


def _upload(table):
    return _device.to_device(np.ascontiguousarray(table))


def DARTS(input_images, **kwargs):
    """Same contract as the reference (darts.py:22-220): (T, m, n) frames, keyword arguments N_x,
    N_y, N_t, M_x, M_y, fft_method, output_type, lsq_method, verbose (others are ignored).  float32
    or float64 frames; NumPy input (a MaskedArray's data is what the reference's FFT sees) -> NumPy,
    CUDA tensor input -> a device tensor: (2, m, n) float64, or (2, 2M_y+1, 2M_x+1) complex128
    for output_type="spectral"."""
    if input_images.ndim != 3:  # check_input_frames(just_ndim=True)
        raise ValueError("input_images dimension mismatch.\n"
                         f"input_images.shape: {str(input_images.shape)}\n"
                         "(t, x, y ) dimensions expected")
    N_x = kwargs.get("N_x", 50)
    N_y = kwargs.get("N_y", 50)
    N_t = kwargs.get("N_t", 4)
    M_x = kwargs.get("M_x", 2)
    M_y = kwargs.get("M_y", 2)
    fft_method = kwargs.get("fft_method", "numpy")
    output_type = kwargs.get("output_type", "spatial")
    lsq_method = kwargs.get("lsq_method", 2)
    verbose = kwargs.get("verbose", True)

    T, m, n = (int(s) for s in input_images.shape)
    if N_t >= T - 1:
        raise ValueError("N_t = %d >= %d = T-1, but N_t < T-1 required" % (N_t, T - 1))
    if output_type not in ["spatial", "spectral"]:
        raise ValueError("invalid output_type=%s, must be 'spatial' or 'spectral'" % output_type)

    on_device = _device.is_device_tensor(input_images)
    masked = isinstance(input_images, np.ma.MaskedArray)
    data = np.ma.getdata(input_images) if masked else input_images
    lib = torch if isinstance(data, torch.Tensor) else np
    if data.dtype not in (lib.float32, lib.float64):
        raise NotImplementedError(f"pysteps_b200 DARTS: frames of dtype {data.dtype} are not supported "
                                  "(float32 or float64)")
    hw = (2 * M_x + 1) * (2 * M_y + 1)
    if 2 * hw > MAX_COLS:
        raise NotImplementedError(f"pysteps_b200 DARTS: 2 (2 M_x + 1)(2 M_y + 1) = {2 * hw} unknowns; at most "
                                  f"{MAX_COLS} (M_x, M_y <= 5) are supported")

    _device.require_cuda()
    stream = _device.stream_ptr()
    frames = _device.to_device(data)
    code = _device.dtype_code(frames.dtype)
    if masked:
        # masked non-finite values pass the reference's check; its FFT then sees them
        if np.any(~np.isfinite(input_images)):
            raise ValueError("the input images contain non-finite values")
    elif T * m * n:
        stats = torch.empty(4, dtype=torch.float64, device="cuda")
        _lib.call("b200_field_stats", frames.data_ptr(), code, T * m * n, stats.data_ptr(), stream)
        if float(_device.to_host(stats)[0]) > 0:
            raise ValueError("the input images contain non-finite values")

    if verbose:
        print("Computing the motion field with the DARTS method.")
        t0 = time.time()

    no_fftn = _check_fft_method(fft_method)

    if verbose:
        print("-----")
        print("DARTS")
        print("-----")
        print("  Computing the FFT of the reflectivity fields...", end="", flush=True)
        starttime = time.time()
    if no_fftn is not None:
        raise no_fftn

    y_fail, h_fail = index_errors(T, m, n, N_x, N_y, N_t, M_x, M_y)
    Kt, Ky, Kx = 2 * N_t + 1, 2 * (N_y + M_y) + 1, 2 * (N_x + M_x) + 1
    if y_fail is None and h_fail is None:
        tw_x, tw_y, tw_t, K = spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y)
        fx = tw_x.shape[0]
        d_tx, d_ty, d_tt = _upload(tw_x), _upload(tw_y), _upload(tw_t)
        work = torch.empty(T * m * fx + Kt * m * Kx, dtype=torch.complex128, device="cuda")
        spec = torch.empty((Kt, Ky, Kx), dtype=torch.complex128, device="cuda")
        _lib.call("b200_darts_spectrum", frames.data_ptr(), code, T, m, n, d_tx.data_ptr(), fx, d_ty.data_ptr(), Ky,
                  d_tt.data_ptr(), Kt, K, work.data_ptr(), spec.data_ptr(), stream)

    if verbose:
        print("Done in %.2f seconds." % (time.time() - starttime))
        print("  Constructing the y-vector...", end="", flush=True)
        starttime = time.time()
    if y_fail is not None:
        y_fail()
    if verbose:
        print("Done in %.2f seconds." % (time.time() - starttime))
        print("  Constructing the H-matrix...", end="", flush=True)
        starttime = time.time()
    if h_fail is not None:
        h_fail()

    T_x, T_y, T_t = n, m, T
    c1 = -1.0 * T_t / (T_x * T_y)
    nc = 2 * hw
    rows = Kt * (2 * N_y + 1) * (2 * N_x + 1)
    npairs = nc * (nc + 1) // 2 + nc
    part = torch.empty(-(-rows // NORMAL_ROWS) * npairs, dtype=torch.complex128, device="cuda")
    normal = torch.empty(nc * (nc + 1), dtype=torch.complex128, device="cuda")
    _lib.call("b200_darts_normal", spec.data_ptr(), N_x, N_y, N_t, M_x, M_y, c1 / T_x, c1 / T_y, part.data_ptr(),
              normal.data_ptr(), normal[nc * nc:].data_ptr(), stream)
    host = torch.empty(nc * (nc + 1), dtype=torch.complex128, pin_memory=True)
    host.copy_(normal, non_blocking=True)
    done = torch.cuda.Event()
    done.record()

    if verbose:
        print("Done in %.2f seconds." % (time.time() - starttime))
        print("  Solving the linear systems...", end="", flush=True)
        starttime = time.time()
    done.synchronize()
    h_np = host.numpy()
    x = solve(h_np[: nc * nc].reshape(nc, nc), h_np[nc * nc:], lsq_method)
    if verbose:
        print("Done in %.2f seconds." % (time.time() - starttime))

    h, w = 2 * M_y + 1, 2 * M_x + 1
    U = np.zeros((h, w), dtype=complex)
    V = np.zeros((h, w), dtype=complex)
    i, j = np.unravel_index(np.arange(h * w), (h, w))
    V[i, j] = x[0: h * w]
    U[i, j] = x[h * w: 2 * h * w]

    if output_type == "spatial":
        rows_, cols_, ri, ci = fill_tables(M_x, M_y, m, n)
        coef = np.zeros((2, len(rows_), len(cols_)), dtype=complex)
        coef[0][ri, ci] = U
        coef[1][ri, ci] = V
        d_coef = _upload(coef)
        d_ey, d_ex = _upload(twiddles(tuple(rows_), m, 1)), _upload(twiddles(tuple(cols_), n, 1))
        out = torch.empty((2, m, n), dtype=torch.float64, device="cuda")
        _lib.call("b200_darts_synthesize", d_coef.data_ptr(), len(rows_), len(cols_), d_ey.data_ptr(),
                  d_ex.data_ptr(), m, n, out.data_ptr(), stream)
        result = out if on_device else _device.to_host(out)
    else:
        result = np.stack([U, V])
        if on_device:
            result = _device.to_device(result)

    if verbose:
        print("--- %s seconds ---" % (time.time() - t0))
    return result
