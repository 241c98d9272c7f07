"""Oracle of probability matching (pysteps/postprocessing/probmatching.py:55-140, 277-337).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Restates nonparam_match_empirical_cdf and
resample_distributions in the steps the device takes:
  * match: only the values above each array's minimum are sorted, with a stable order (ties in pixel
    order); rank r of the target is its minimum below the dry count and the sorted wet value after it;
    np.percentile's value is _lerp of two order statistics at the indices and gamma NumPy computes, and
    the target values below it become the minimum.  A zero minimum is -0.0 when some minimal value is.
  * resample: the values that are NaN in neither array, stably sorted and reversed, picked by the 0/1
    draws, stably sorted and reversed again, behind canonical NaNs.
The reference sorts with NumPy's default (unstable) argsort: where tied initial values meet different
target values the two differ in which tied pixel gets which value, never in the values of a tie group.
These functions return values only: the argument checks and warnings are the host's.
"""
import numpy as np


def signed_nanmin(a):
    """np.nanmin of a float64 array, -0.0 when some minimal value is -0.0; NaN when all are NaN"""
    v = a[~np.isnan(a)]
    if v.size == 0:
        return np.nan
    m = v.min()
    if m == 0:
        m = -0.0 if np.signbit(v[v == 0]).any() else 0.0
    return float(m)


def percentile_taps(n, x_wet):
    """(i0, i1, gamma) of np.percentile(target, 100 * (1 - x_wet / n)) over n sorted values (NumPy's
    "linear" method: virtual index (n - 1) q, its floor, and the last value past n - 1)"""
    war = np.int64(x_wet) / n
    q = np.true_divide(100 * (1 - war), np.float64(100))
    virtual = (n - 1) * q
    previous = -1 if virtual >= n - 1 else int(np.floor(virtual))
    gamma = float(virtual - np.intp(previous))
    return previous % n, (previous + 1 if previous >= 0 else -1) % n, gamma


def lerp(a, b, t):
    """numpy/lib/_function_base_impl.py:_lerp for scalars"""
    diff = b - a
    return b - diff * (1.0 - t) if t >= 0.5 else a + diff * t


def nonparam_match_empirical_cdf(initial_array, target_array, ignore_indices=None):
    """the float64 output of a valid call (no error raised by the reference)"""
    shape = np.shape(initial_array)
    x = np.array(initial_array, dtype=np.float64).reshape(-1)
    t = np.array(target_array, dtype=np.float64).reshape(-1)
    n = x.size
    mask = np.zeros(shape, dtype=bool)
    if ignore_indices is not None:
        mask[ignore_indices] = True
    mask = mask.reshape(-1)
    zx = signed_nanmin(x)
    zt = signed_nanmin(t)
    with np.errstate(invalid="ignore"):
        xi = np.flatnonzero(~mask & (x > zx))
        ti = np.flatnonzero(t > zt)
    xi = xi[np.argsort(x[xi], kind="stable")]
    ti = ti[np.argsort(t[ti], kind="stable")]
    dry = n - ti.size

    def ranked(r):
        r = np.asarray(r)
        return np.where(r < dry, zt, t[ti[np.clip(r - dry, 0, max(ti.size - 1, 0))]] if ti.size else zt)

    out = np.where(mask, x, zt)
    v = ranked(n - xi.size + np.arange(xi.size)).astype(np.float64)
    if ti.size > xi.size:
        i0, i1, gamma = percentile_taps(n, xi.size)
        with np.errstate(invalid="ignore"):
            p = lerp(float(ranked(i0)), float(ranked(i1)), gamma)
            v[v < p] = zt
    out[xi] = v
    return out.reshape(shape)


def resample_distributions(first_array, second_array, draws):
    """the output of a valid call, draws (n,) the 0/1 values of randgen.binomial(1, p, n)"""
    a = np.asarray(first_array).reshape(-1)
    b = np.asarray(second_array).reshape(-1)
    nan = np.isnan(a) | np.isnan(b)
    n_nan = int(nan.sum())
    dtype = np.float64 if n_nan else np.result_type(a, b)
    av, bv = a[~nan], b[~nan]
    ad = av[np.argsort(av, kind="stable")][::-1]
    bd = bv[np.argsort(bv, kind="stable")][::-1]
    picks = np.where(np.asarray(draws, dtype=bool)[n_nan:], ad, bd).astype(np.float64)
    picks = picks[np.argsort(picks, kind="stable")][::-1]
    return np.concatenate([np.full(n_nan, np.nan), picks]).astype(dtype)
