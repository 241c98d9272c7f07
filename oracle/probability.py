"""Oracle of the local Lagrangian probability nowcast (pysteps/nowcasts/lagrangian_probability.py).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  The extrapolation is the oracle of
``oracle/semilagrangian.py``; the neighbourhood counts are exact int64 sums over the kernel's row
runs (row prefix sums), where the reference convolves with scipy's FFT in single precision.  The
argument flow restates the reference's: nowcasts/lagrangian_probability.py:69-107 and
nowcasts/extrapolation.py:69-117.
"""
import math

import numpy as np

from . import semilagrangian


def kernel_runs(s):
    """(s, 2) int64: the first and last column of every row of the reference's kernel of diameter
    s > 0 -- an s x s block of ones for s < 5, else the disk (a - mid)^2 + (b - mid)^2 <= mid^2
    on the s x s grid, mid = max(s // 2, 1).  Every row is one non-empty run."""
    if s < 5:
        return np.tile(np.array([0, s - 1], dtype=np.int64), (s, 1))
    mid = max(s // 2, 1)
    runs = np.empty((s, 2), dtype=np.int64)
    for a in range(s):
        r = math.isqrt(mid * mid - (a - mid) ** 2)
        runs[a] = max(mid - r, 0), min(mid + r, s - 1)
    return runs


def kernel(s):
    """The reference's kernel of diameter s as a 0/1 int64 array (for the checks against scipy)."""
    k = np.zeros((s, s), dtype=np.int64)
    for a, (b0, b1) in enumerate(kernel_runs(s)):
        k[a, b0:b1 + 1] = 1
    return k


def counts(A, s):
    """int64 count(y, x) = sum_{a, b} K_s[a, b] A[y + c - a, x + c - b], c = (s - 1) // 2, zero
    outside the frame: scipy.signal.convolve(A, K_s, mode="same") computed exactly."""
    A = np.asarray(A, dtype=np.int64)
    m, n = A.shape
    # row prefix sums P[:, j] = sum A[:, :j], edge-padded by s + 1 columns on both sides: a column
    # index clamped into [0, n] reads the padding, and a run that misses the frame reads the same
    # word twice and adds zero
    P = np.zeros((m, n + 1), dtype=np.int64)
    np.cumsum(A, axis=1, out=P[:, 1:])
    pad = s + 1
    P = np.pad(P, ((0, 0), (pad, pad)), mode="edge")
    c = (s - 1) // 2
    out = np.zeros((m, n), dtype=np.int64)
    for a, (b0, b1) in enumerate(kernel_runs(s)):
        ylo, yhi = max(0, a - c), min(m, m + a - c)  # output rows whose source row y + c - a is inside
        if ylo >= yhi:
            continue
        src = P[ylo + c - a:yhi + c - a]
        hi, lo = pad + c - b0 + 1, pad + c - b1  # columns x + c - b0 + 1 and x + c - b1 at x = 0
        out[ylo:yhi] += src[:, hi:hi + n]
        out[ylo:yhi] -= src[:, lo:lo + n]
    return out


def exceedances(F, threshold):
    """(B, valid) of the extrapolated field F, with the reference's rules: NaN pixels are invalid and
    take the value threshold - 1 (in F's dtype) before the comparison F >= threshold."""
    F = np.array(F)
    nanmask = np.isnan(F)
    F[nanmask] = threshold - 1
    return F >= threshold, ~nanmask


def neighbourhood(B, valid, s):
    """One lead's plane: B as 0/1 for s == 0, else count(B) / count(valid) clipped to [0, 1];
    NaN where the pixel is invalid."""
    if s == 0:
        out = B.astype(np.float64)
    else:
        with np.errstate(invalid="ignore", divide="ignore"):
            out = counts(B, s).astype(np.float64) / counts(valid, s).astype(np.float64)
    out = np.clip(out, 0, 1)
    out[~valid] = np.nan
    return out


def scales(timesteps, slope):
    """The kernel diameter of every lead, int(t * slope), with the reference's failure for a
    negative one."""
    out = []
    for t in timesteps:
        s = int(t * slope)
        if s < 0:
            raise ValueError("negative dimensions are not allowed")
        out.append(s)
    return out


def forecast(precip, velocity, timesteps, threshold, extrap_method="semilagrangian", extrap_kwargs=None, slope=5):
    if isinstance(timesteps, int) and timesteps > 0:
        timesteps = np.arange(1, timesteps + 1)
    elif not isinstance(timesteps, list):
        raise ValueError(f"invalid value for argument 'timesteps': {timesteps}")
    if precip.ndim != 2:
        raise ValueError("The input precipitation must be a two-dimensional array")
    if velocity.ndim != 3:
        raise ValueError("Input velocity must be a three-dimensional array")
    if precip.shape != velocity.shape[1:3]:
        raise ValueError("Dimension mismatch between input precipitation and velocity: "
                         + "shape(precip)=%s, shape(velocity)=%s" % (str(precip.shape), str(velocity.shape)))
    if isinstance(timesteps, list) and not sorted(timesteps) == timesteps:
        raise ValueError("timesteps is not in ascending order")
    kw = {} if extrap_kwargs is None else dict(extrap_kwargs)
    kw["allow_nonfinite_values"] = bool(np.any(~np.isfinite(precip)))
    if extrap_method == "eulerian":
        F = np.repeat(precip[np.newaxis], len(timesteps), axis=0)
    elif extrap_method == "semilagrangian":
        F = semilagrangian.extrapolate(precip, velocity, timesteps, **kw)
    else:
        raise ValueError(f"oracle: extrapolation method {extrap_method!r} is not restated")
    B, valid = exceedances(F, threshold)
    S = scales(timesteps, slope)
    return np.stack([neighbourhood(B[i], valid[i], s) for i, s in enumerate(S)])
