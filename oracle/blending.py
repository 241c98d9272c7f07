"""NumPy restatement of pysteps/blending/linear_blending.py for the canonical shapes (a (T, m, n) or
(n_ens, T, m, n) nowcast and NWP), written the way csrc/blending.cu computes it: member maps
instead of repeated arrays, the NaN fill per output member, and dense ranks from np.unique on
canonical keys (-0.0 as +0.0) instead of scipy's rankdata.

``blend(now, nwp, ...)`` takes fields already converted to rain rate; ``to_rainrate`` is the
reference's conversion for the transforms and units the package supports.
"""
import numpy as np


def to_rainrate(R, metadata):
    R = R.copy()
    md = dict(metadata)
    tr = md["transform"]
    if tr == "dB":
        thr = md.get("threshold", -10.0)
        R = 10.0 ** (R / 10.0)
        thr = 10.0 ** (thr / 10.0)
        R[R < thr] = 0.0
    elif tr in ("BoxCox", "log"):
        lam = md.pop("BoxCox_lambda", 0.0)
        thr = md.get("threshold", -10.0)
        if lam == 0.0:
            R = np.exp(R)
            thr = np.exp(thr)
        else:
            R = np.exp(np.log(lam * R + 1) / lam)
            thr = np.exp(np.log(lam * thr + 1) / lam)
        R[R < thr] = 0.0
    elif tr == "sqrt":
        R = R**2
    if md["unit"] == "mm":
        R = R / float(md["accutime"]) * 60.0
    elif md["unit"] == "dBZ":
        R = (R / md.get("zr_a", 200.0)) ** (1.0 / md.get("zr_b", 1.6))
    return R


def member_map(n_src, n_out):
    """output member -> source member of the reference's np.repeat (consecutive blocks)"""
    if n_src == n_out:
        return np.arange(n_out)
    if n_src == 1:
        return np.zeros(n_out, dtype=np.int64)
    return np.repeat(np.arange(n_src), [(n_out + i) // n_src for i in range(n_src)])


def dense_rank(x):
    """scipy.stats.rankdata(x, method="dense") as float64: all NaN when x has a NaN"""
    x = np.asarray(x, dtype=np.float64).ravel()
    if np.isnan(x).any():
        return np.full(x.shape, np.nan)
    _, inv = np.unique(np.where(x == 0, 0.0, x), return_inverse=True)
    return (inv + 1).astype(np.float64)


def _members(a):
    return a if a.ndim == 4 else a[None]


def blend(now, nwp, timesteps, timestep, start_blending=120, end_blending=240, fill_nwp=True, saliency=False):
    """now (T', m, n) or (E, T', m, n) and nwp (T, m, n) or (E', T, m, n), in rain rate."""
    N, W = _members(now), _members(nwp)[:, :timesteps]
    E = max(N.shape[0], W.shape[0])
    mn, mw = member_map(N.shape[0], E), member_map(W.shape[0], E)
    W = np.nan_to_num(W, nan=0.0)
    out = np.zeros((E,) + W.shape[1:], dtype=W.dtype)
    for i in range(timesteps):
        t = (i + 1) * timestep
        w_nwp = (t - start_blending) / (end_blending - start_blending)
        g = W[mw, i]
        if w_nwp >= 1.0:
            out[:, i] = g
            continue
        c = N[mn, i].copy()
        nan = np.isnan(c)
        c[nan] = g[nan] if fill_nwp else 0.0
        if w_nwp <= 0.0:
            out[:, i] = c
        else:
            w_now = 1.0 - w_nwp
            if saliency:
                nc = np.zeros_like(c) if np.max(c) == 0 else c / np.max(c)
                ng = np.zeros_like(g) if np.max(g) == 0 else g / np.max(g)
                r = dense_rank(nc - ng).reshape(c.shape)
                r /= r.max()
                ws = 0.5 * ((w_now * r) / (w_now * r + (1 - w_now) * (1 - r))
                            + np.sqrt(r**2 + w_now**2) / (np.sqrt(r**2 + w_now**2)
                                                           + np.sqrt((1 - r) ** 2 + (1 - w_now) ** 2)))
                out[:, i] = ws * c + (1 - ws) * g
            else:
                out[:, i] = w_nwp * g + w_now * c
    return out if E > 1 else out[0]
