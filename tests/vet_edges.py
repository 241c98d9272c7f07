"""The edge grid of the VET cost / gradient kernels (csrc/vet.cu), an independent NumPy restatement of one
evaluation of the reference's _cost_function (pysteps/motion/_vet.pyx:238-621), and the error bound of the
kernel's summation tree.

  restatement   per pixel, in float64 and in the reference's expression order: the sector centres, the four
                bilinear coefficients, the pixel displacement, the warp with its clamps and its truncated
                interpolated mask, the squared residual and the eight gradient terms g_a * c_k, the latter
                only on the rows the reference's gradient loops visit (each band stops one row short).
                NumPy's element-wise float64 operations round to nearest and are never contracted into
                FMAs, so every term is the kernel's and the C oracle's bit for bit.  Sums are exact
                (math.fsum), one per output, next to the sum of the terms' magnitudes.
  partition     vet_launch's strips per cell and the addition chains of the kernels, from which each
                output's bound |device - exact| <= gamma_D * sum |term| follows.
  cases         single-pixel probes (a mask set everywhere but at one pixel, which then alone contributes)
                and whole fields over the geometries, strip regimes, displacements, masks, gains and frame
                counts where the index logic turns.

tests/test_oracle_vet_edges.py pins the restatement to the oracle (CPU); tests/test_vet_edges_gpu.py holds the
kernels to both."""
import functools
import itertools
import math

import numpy as np

U = 2.0 ** -53                  # unit roundoff of float64
VET_THREADS = 256               # csrc/vet.cu: threads per CTA; block_reduce: 5 shuffle rounds, 8 warps
H100_SXM_SMS = 132              # the SM count the CPU tests assume (read at run time on the GPU)
GAINS = (0.0, 1e6, 0.1)         # smooth_gain; 0.1 is not a float32 and is rounded to one on the way in


# ---------------------------------------------------------------------------------------------- partition
def partition(nx, ny, xs, ys, sms):
    """vet_launch's launch geometry.  This restates csrc/vet.cu (strips per cell, rows per strip) and must
    follow it there: the strip regimes and the error bounds below are derived from it.
    -> dict with the per-band rows (bands along x: l, along y: m), strips, and the regimes reached."""
    xss, yss = nx // xs, ny // ys
    ncx, ncy = xs - 1, ys - 1
    ncells = ncx * ncy
    want = 8 * sms
    by_cells = -(-want // ncells)
    strips = max(1, min(by_cells, max(xss // 2, 1)))
    i_shift, j_shift = xss // 2, yss // 2
    rows = [(0 if l == 0 else i_shift + l * xss, nx if l == xs - 2 else i_shift + (l + 1) * xss)
            for l in range(ncx)]
    cols = [(0 if m == 0 else j_shift + m * yss, ny if m == ys - 2 else j_shift + (m + 1) * yss)
            for m in range(ncy)]
    rps = [-(-(e - b) // strips) for b, e in rows]
    used = [-(-(e - b) // r) for (b, e), r in zip(rows, rps)]        # non-empty strips per band
    regimes = set()
    if strips == 1 and by_cells == 1:
        regimes.add("strips=1")
    if strips == xss // 2 < by_cells and any(u < strips for u in used):
        regimes.add("strips=xss/2, empty trailing")
    if 1 < strips == by_cells < xss // 2:
        regimes.add("strips=8SMs/cells")
    pps = max(r for r in rps) * max(e - b for b, e in cols)            # most pixels one CTA reduces
    return dict(xss=xss, yss=yss, ncx=ncx, ncy=ncy, ncells=ncells, strips=strips, rows=rows, cols=cols,
                rps=rps, used=used, pps=pps, regimes=regimes)


REGIMES = {"strips=1", "strips=xss/2, empty trailing", "strips=8SMs/cells"}


def strip_rows(p, l):
    """(first, last) row of every non-empty strip of band l"""
    b, e = p["rows"][l]
    r = p["rps"][l]
    return [(s, min(s + r, e) - 1) for s in range(b, e, r)]


def chains(p, T=2):
    """Deepest addition chain D of each device output (a term passes through at most D roundings):
      per thread  ceil(pixels per CTA / 256), then 5 shuffle rounds and 7 warp additions (block_reduce);
      residual    the finaliser's ceil(cells x strips / 256) per thread, 5 + 7 again;
      gradient    vet_final_grad_kernel adds, per sector, the strips of each of its <= 4 cells one after
                  the other: (cells at the sector) x strips, and one addition of the smoothness part;
      smoothness  ceil(2 (xs-2)(ys-2) / 256) per thread, 5 + 7, and the product by the gain;
    three frames add one host addition of the two pairs (b200_vet_value_and_gradient)."""
    xs, ys = p["ncx"] + 1, p["ncy"] + 1
    blk = 5 + (VET_THREADS // 32 - 1)
    pix = -(-p["pps"] // VET_THREADS) + blk
    extra = 1 if T == 3 else 0
    ncell = np.zeros((xs, ys), np.int64)
    for dl, dm in ((0, 0), (0, 1), (1, 0), (1, 1)):
        ncell[dl:dl + p["ncx"], dm:dm + p["ncy"]] += 1
    ni = max(xs - 2, 0) * max(ys - 2, 0)
    return dict(res=pix + -(-p["ncells"] * p["strips"] // VET_THREADS) + blk + extra,
                grad=pix + ncell * p["strips"] + 1 + extra,
                smooth=-(-2 * ni // VET_THREADS) + blk + 1 + extra)


def gamma(D):
    return D * U / (1.0 - D * U)


# ------------------------------------------------------------------------------------------- restatement
def _centres(n, s):
    """sector centres: the mean of each sector's pixel indices, as the reference takes it"""
    return np.arange(n, dtype=np.float64).reshape(s, n // s).mean(axis=1)


def warp_terms(image, mask, x, y, dispx, dispy):
    """_vet._warp (_vet.pyx:160-228) at pixels (x, y): value, gradient, masked flag and where the source
    landed (clamped low / high, on an integer, on the last row or column)."""
    nx, ny = image.shape
    xmi, ymi = nx - 1, ny - 1
    out = {}
    src = []
    for name, p, d, mi in (("x", x, dispx, xmi), ("y", y, dispy, ymi)):
        f = p.astype(np.float64) - d
        low, high = f < 0, f > mi
        f = np.where(low, 0.0, np.where(high, float(mi), f))
        p0 = np.floor(f).astype(np.int64)
        p1 = np.where(low | high, p0, np.minimum(p0 + 1, mi))
        frac = f - p0
        inside = ~(low | high)
        out.update({f"{name}_low": low, f"{name}_high": high, f"{name}_integer": inside & (frac == 0.0),
                    f"{name}_on_last": inside & (f == float(mi)), f"{name}_frac": frac})
        src.append((p0, p1, frac))
    (x0, x1, dx), (y0, y1, dy) = src
    i00, i10, i01, i11 = image[x0, y0], image[x1, y0], image[x0, y1], image[x1, y1]
    f10 = i10 - i00
    f01 = i01 - i00
    f11 = i00 - i10 - i01 + i11
    out["value"] = i00 + dx * f10 + dy * f01 + dx * dy * f11
    out["gx"] = f10 + dy * f11
    out["gy"] = f01 + dx * f11
    m = mask.astype(np.float64)
    m00, m10, m01, m11 = m[x0, y0], m[x1, y0], m[x0, y1], m[x1, y1]
    mv = m00 + dx * (m10 - m00) + dy * (m01 - m00) + dx * dy * (m00 - m10 - m01 + m11)
    out["mv"] = mv
    out["masked"] = np.trunc(mv) != 0          # <int8> of the interpolated mask truncates toward zero
    return out


def pixel_terms(sd, templ, inp, mask, ii, jj):
    """One _cost_function evaluation restated at pixels (ii, jj): the residual term (0 where masked), the
    gradient terms grad[k, a] = g_a * c_k of corner k (0 off the gradient rows), the cell (l0, m0) each
    pixel feeds, the pixel displacement and the warp's landing flags."""
    xs, ys = sd.shape[1:]
    nx, ny = templ.shape
    xss, yss = nx // xs, ny // ys
    i_shift, j_shift = xss // 2, yss // 2
    xg, yg = _centres(nx, xs), _centres(ny, ys)
    l0 = np.clip((ii - i_shift) // xss, 0, xs - 2)
    m0 = np.clip((jj - j_shift) // yss, 0, ys - 2)
    l1, m1 = l0 + 1, m0 + 1
    xi, yj = ii.astype(np.float64), jj.astype(np.float64)
    xg0, xg1, yg0, yg1 = xg[l0], xg[l1], yg[m0], yg[m1]
    area = (xg1 - xg0) * (yg1 - yg0)
    c = (
        (xg1 * yg1 - xi * yg1 - xg1 * yj + xi * yj) / area,
        (-xg1 * yg0 + xi * yg0 + xg1 * yj - xi * yj) / area,
        (-xg0 * yg1 + xi * yg1 + xg0 * yj - xi * yj) / area,
        (xg0 * yg0 - xi * yg0 - xg0 * yj + xi * yj) / area,
    )
    disp = [sd[a, l0, m0] * c[0] + sd[a, l0, m1] * c[1] + sd[a, l1, m0] * c[2] + sd[a, l1, m1] * c[3]
            for a in (0, 1)]
    w = warp_terms(templ, mask, ii, jj, disp[0], disp[1])
    mm = w["masked"] | (mask[ii, jj] > 0)
    r = w["value"] - inp[ii, jj]
    res = np.where(mm, 0.0, r * r)
    b = np.where(mm, 0.0, 2.0 * (inp[ii, jj] - w["value"]))
    g = (w["gx"] * b, w["gy"] * b)
    # np.unique(l_i, return_index, return_counts): the gradient loops run i_min <= i < i_min + count - 1
    l_i = np.clip((np.arange(nx) - i_shift) // xss, 0, xs - 2)
    vals, first, count = np.unique(l_i, return_index=True, return_counts=True)
    i_max = np.full(xs, nx)
    i_max[vals] = first + count - 1
    grow = ii < i_max[l0]
    grad = np.stack([np.stack([np.where(grow, g[a] * c[k], 0.0) for a in (0, 1)]) for k in range(4)])
    return dict(res=res, grad=grad, l0=l0, m0=m0, grow=grow, contributes=~mm, disp=disp, warp=w)


CORNERS = ((0, 0), (0, 1), (1, 0), (1, 1))   # corner k of cell (l0, m0) is sector (l0 + dl, m0 + dm)


def smooth_terms(sd, nx, ny):
    """The smoothness penalty's terms (_vet.pyx:567-614): the cost terms of the interior sectors, and the
    gradient contributions (before the factor 2 * smooth_gain) as an array (10, 2, xs, ys): contribution c
    of target sector (a, l, m), zero where that neighbour is not interior."""
    _, xs, ys = sd.shape
    xss, yss = nx // xs, ny // ys
    S = lambda dl, dm: sd[:, 1 + dl:xs - 1 + dl, 1 + dm:ys - 1 + dm]   # noqa: E731  (2, xs-2, ys-2) shifted
    dx2 = (S(1, 0) - 2 * S(0, 0) + S(-1, 0)) / float(xss * xss)
    dy2 = (S(0, 1) - 2 * S(0, 0) + S(0, -1)) / float(yss * yss)
    dxy = (S(1, 1) - S(1, -1) - S(-1, 1) + S(-1, -1)) / float(4 * xss * yss)
    cost = dx2 * dx2 + 2 * dxy * dxy + dy2 * dy2
    contrib = np.zeros((10, 2, xs, ys))
    for c, ((dl, dm), t) in enumerate((((0, 0), -2 * dx2), ((1, 0), dx2), ((-1, 0), dx2), ((0, 0), -2 * dy2),
                                       ((0, -1), dy2), ((0, 1), dy2), ((-1, -1), dxy), ((-1, 1), -dxy),
                                       ((1, -1), -dxy), ((1, 1), dxy))):
        contrib[c, :, 1 + dl:xs - 1 + dl, 1 + dm:ys - 1 + dm] = t
    return cost.ravel().tolist(), contrib


def evaluate(sd, templ, inp, mask, gain):
    """Exact sums of one evaluation, per output, with the magnitudes they bound against:
      res, res_abs         residual sum (out[0])
      smooth, smooth_abs   smoothness penalty (out[1]) = gain * sum of the per-sector terms
      grad, grad_abs       residual part of the gradient (2, xs, ys)
      sgrad, sgrad_abs     smoothness part of the gradient, already times 2 * gain
      nterms               terms the oracle adds per gradient sector (its sequential chain)
    plus the per-pixel terms (`px`)."""
    nx, ny = templ.shape
    _, xs, ys = sd.shape
    ii, jj = np.divmod(np.arange(nx * ny), ny)
    px = pixel_terms(sd, templ, inp, mask, ii, jj)
    res = px["res"][px["contributes"]]
    out = dict(px=px, res=math.fsum(res.tolist()), res_abs=math.fsum(res.tolist()), nres=int(res.size))
    cell = px["l0"] * (ys - 1) + px["m0"]
    order = np.argsort(cell, kind="stable")
    starts = np.searchsorted(cell[order], np.arange((xs - 1) * (ys - 1) + 1))
    grows = np.bincount(cell, weights=px["grow"], minlength=(xs - 1) * (ys - 1))
    grad, grad_abs = np.zeros((2, xs, ys)), np.zeros((2, xs, ys))
    nterms = np.zeros((xs, ys), np.int64)
    for k, (dl, dm) in enumerate(CORNERS):
        for l0 in range(xs - 1):
            for m0 in range(ys - 1):
                nterms[l0 + dl, m0 + dm] += int(grows[l0 * (ys - 1) + m0])
    parts = {}
    for k in range(4):
        for a in (0, 1):
            t = px["grad"][k, a][order]
            parts[k, a] = (t.tolist(), np.add.reduceat(np.abs(t), starts[:-1]))
    for a in (0, 1):
        for l in range(xs):
            for m in range(ys):
                seq, mag = [], 0.0
                for k, (dl, dm) in enumerate(CORNERS):
                    l0, m0 = l - dl, m - dm
                    if 0 <= l0 < xs - 1 and 0 <= m0 < ys - 1:
                        cid = l0 * (ys - 1) + m0
                        seq.append(parts[k, a][0][starts[cid]:starts[cid + 1]])
                        mag += parts[k, a][1][cid]
                grad[a, l, m] = math.fsum(itertools.chain(*seq))
                grad_abs[a, l, m] = mag
    out.update(grad=grad, grad_abs=grad_abs, nterms=nterms)
    out.update(smooth_exact(sd, nx, ny, gain))
    return out


def smooth_exact(sd, nx, ny, gain):
    """the smoothness parts of an evaluation: penalty (out[1]) and gradient part, exact, with magnitudes"""
    g = as_c_float(gain)
    _, xs, ys = sd.shape
    cost, contrib = smooth_terms(sd, nx, ny) if g > 0 else ([], np.zeros((10, 2, xs, ys)))
    flat = contrib.reshape(10, -1).T.tolist()
    sgrad = 2 * g * np.array([math.fsum(ts) for ts in flat]).reshape(2, xs, ys)
    sgrad_abs = 2 * g * np.abs(contrib).sum(axis=0)
    return dict(sgrad=sgrad, sgrad_abs=sgrad_abs, smooth=g * math.fsum(cost), smooth_abs=g * math.fsum(cost),
                nsmooth=len(cost))


def as_c_float(gain):
    """smooth_gain as the C float parameter of _cost_function (and of the device entry points) holds it"""
    return float(np.float32(gain))


def add_pairs(a, b):
    """the exact sums of two frame pairs (three frames: (centre, next) + (previous, centre))"""
    out = dict(a)
    for k in ("res", "res_abs", "grad", "grad_abs", "sgrad", "sgrad_abs", "smooth", "smooth_abs"):
        out[k] = a[k] + b[k]
    for k in ("nres", "nterms", "nsmooth"):
        out[k] = a[k] + b[k]
    return out


# slack on every bound: the rounding of the exact sums to float64 (math.fsum rounds once; the gain product,
# the sum of the two gradient parts and that of two frame pairs once more each) and of the magnitudes
SLACK = 4


def within(got, exact, mag, D):
    """|got - exact| <= gamma_{D + SLACK} * mag (1 + 2^-20), element-wise"""
    tol = gamma(np.asarray(D) + SLACK) * np.asarray(mag) * (1 + 2.0 ** -20)
    return np.abs(np.asarray(got) - np.asarray(exact)) <= tol


def oracle_chains(ev):
    """the C oracle adds sequentially: D = the number of terms per output (+ the smoothness part, at most
    ten contributions, and the final additions)"""
    return ev["nres"], ev["nsmooth"] + 1, ev["nterms"] + 1


def check_sums(got_res, got_smooth, got_grad, ev, D):
    """assert the three outputs of an evaluation within the bound of chains D = (res, smooth, grad)"""
    Dr, Ds, Dg = D
    if got_res is not None:
        assert within(got_res, ev["res"], ev["res_abs"], Dr), ("residual", got_res, ev["res"], ev["res_abs"])
    if got_smooth is not None:
        assert within(got_smooth, ev["smooth"], ev["smooth_abs"], Ds), ("smoothness", got_smooth, ev["smooth"])
    if got_grad is not None:
        exact = ev["grad"] + ev["sgrad"]
        # the two parts pass through different chains: the smoothness part through its ten contributions,
        # the product by 2 * gain and the final addition
        tol = gamma(np.asarray(Dg) + SLACK) * ev["grad_abs"] + gamma(12 + SLACK) * ev["sgrad_abs"]
        bad = np.abs(got_grad - exact) > tol * (1 + 2.0 ** -20)
        assert not bad.any(), ("gradient", np.argwhere(bad)[:4].tolist(), got_grad[bad][:4], exact[bad][:4])


# -------------------------------------------------------------------------------------------------- cases
GEOMETRIES = {
    # name: (nx, ny, xs, ys)
    "xs2": (48, 60, 2, 3),                 # one cell spans the frame along x
    "xss1": (16, 12, 16, 12),              # nx == xs: i_shift 0, area 1, every gradient row skipped
    "xss2": (24, 20, 12, 10),
    "xss3": (45, 30, 15, 10),
    "xss15": (45, 30, 3, 2),               # strips capped by xss/2, empty trailing strips
    "pow2_4x16": (64, 96, 16, 6),          # area 64 with unequal sides
    "area105": (60, 42, 4, 6),             # 15 x 7: not a power of two, unequal sides
    "strips1": (128, 128, 64, 64),         # >= 8 SMs cells: one strip
    "bench32": (2048, 2048, 32, 32),       # the default sectors (32, 16, 4, 2) at 2048^2
    "bench16": (2048, 2048, 16, 16),
    "bench4": (2048, 2048, 4, 4),
    "bench2": (2048, 2048, 2, 2),
}
BENCH = ("bench32", "bench16", "bench4", "bench2")

FIELD_CASES = {
    # name: (geometry, displacement, mask, smooth_gain, frames)
    "xs2_sub_clear": ("xs2", "sub", "clear", GAINS[0], 2),
    "xs2_clamp_patch": ("xs2", "clamp", "patch", GAINS[1], 3),
    "xss1_sub_patch": ("xss1", "sub", "patch", GAINS[2], 2),
    "xss1_clamp_all": ("xss1", "clamp", "all", GAINS[1], 2),
    "xss2_clamp_patch": ("xss2", "clamp", "patch", GAINS[2], 3),
    "xss3_sub_patch": ("xss3", "sub", "patch", GAINS[1], 2),
    "xss15_clamp_clear": ("xss15", "clamp", "clear", GAINS[0], 2),
    "xss15_sub_patch": ("xss15", "sub", "patch", GAINS[1], 3),
    "pow2_4x16_integer": ("pow2_4x16", "integer", "patch", GAINS[1], 3),
    "pow2_4x16_clamp": ("pow2_4x16", "clamp", "clear", GAINS[2], 2),
    "area105_sub_patch": ("area105", "sub", "patch", GAINS[2], 2),
    "area105_clamp_all": ("area105", "clamp", "all", GAINS[1], 2),
    "strips1_sub_patch": ("strips1", "sub", "patch", GAINS[1], 2),
    "bench32_sub_patch": ("bench32", "sub", "patch", GAINS[1], 2),
    "bench16_clamp_clear": ("bench16", "clamp", "clear", GAINS[2], 2),
    "bench4_integer_patch": ("bench4", "integer", "patch", GAINS[1], 2),
    "bench2_sub_patch": ("bench2", "sub", "patch", GAINS[0], 2),
}


def _frames(nx, ny, T, rng):
    """smooth-ish frames with detail: a few sinusoids plus noise, values of order 10"""
    x = np.arange(nx)[:, None] / nx
    y = np.arange(ny)[None, :] / ny
    base = 5 + 3 * np.sin(7 * x + 3 * y) + 2 * np.cos(5 * y - 11 * x * y)
    return np.stack([base + (t + 1) * rng.random((nx, ny)) for t in range(T)])


def _mask(kind, nx, ny, rng):
    mask = np.zeros((nx, ny), np.int8)
    if kind == "all":
        mask[:] = 1
    elif kind == "patch":
        for _ in range(4):
            h, w = rng.integers(1, max(2, nx // 4)), rng.integers(1, max(2, ny // 4))
            i, j = rng.integers(0, nx - h + 1), rng.integers(0, ny - w + 1)
            mask[i:i + h, j:j + w] = 1
        mask[rng.random((nx, ny)) < 0.005] = 1
    return mask


def _sector_field(kind, nx, ny, xs, ys, rng):
    if kind == "sub":       # pixel displacements under one pixel (coefficients extrapolate up to ~2x at borders)
        return rng.uniform(-0.2, 0.2, (2, xs, ys))
    if kind == "clamp":     # sources beyond every border: outward at each, half the frame at most
        ramp = (np.linspace(1, -1, xs)[:, None] * np.ones(ys) * nx, np.ones(xs)[:, None] * np.linspace(1, -1, ys) * ny)
        return np.stack(ramp) * rng.uniform(0.25, 0.5, (2, xs, ys))
    if kind == "integer":   # exact -1 everywhere on a power-of-two area: rows nx-2 land on nx-1 exactly
        return np.full((2, xs, ys), -1.0)
    raise KeyError(kind)


def field_case(name):
    """-> (sector displacement (2, xs, ys), images (T, nx, ny), mask int8, smooth_gain, geometry name)"""
    geo, disp, mkind, gain, T = FIELD_CASES[name]
    nx, ny, xs, ys = GEOMETRIES[geo]
    rng = np.random.default_rng(sum(map(ord, name)))
    images = _frames(nx, ny, T, rng)
    return (np.ascontiguousarray(_sector_field(disp, nx, ny, xs, ys, rng)), images,
            _mask(mkind, nx, ny, rng), gain, geo)


def field_branches(name, ev_px):
    """what a whole-field case reaches, from its per-pixel terms"""
    geo, disp, mkind, gain, T = FIELD_CASES[name]
    w = ev_px["warp"]
    got = set()
    for ax in "xy":
        if w[f"{ax}_low"].any() and w[f"{ax}_high"].any():
            got.add(f"clamp {ax} both sides")
        if w[f"{ax}_on_last"].any():
            got.add(f"lands on last {ax}")
    d = np.abs(np.concatenate(ev_px["disp"]))
    if d.max() < 1:
        got.add("|d| < 1")
    if all(np.array_equal(v, np.round(v)) for v in ev_px["disp"]):
        got.add("integer displacements")
    mv = w["mv"]
    if ((mv > 0) & (mv < 1)).any():
        got.add("fractional mask")
    return got


# --------------------------------------------------------------------------------------------------- probes
def probe_points(geo, sms, full=True):
    """Pixels where the index logic turns: the first, last and skipped (last) row of every band, the first
    and last column of every band, the first and last row of every non-empty strip, and the four frame
    corners.  Rows and columns are paired so that each appears at least once.  `full=False` keeps the
    first, second and last bands and strips (for the 2048^2 geometries)."""
    nx, ny, xs, ys = GEOMETRIES[geo]
    p = partition(nx, ny, xs, ys, sms)
    bands = range(p["ncx"]) if full else sorted({0, 1, p["ncx"] - 1} & set(range(p["ncx"])))
    rows = set()
    for l in bands:
        b, e = p["rows"][l]
        rows.update((b, e - 2 if e - b > 1 else b, e - 1))
        sr = strip_rows(p, l)
        for k, (r0, r1) in enumerate(sr):
            if full or k < 2 or k >= len(sr) - 2:
                rows.update((r0, r1))
    cbands = range(p["ncy"]) if full else sorted({0, 1, p["ncy"] - 1} & set(range(p["ncy"])))
    cols = set()
    for m in cbands:
        b, e = p["cols"][m]
        cols.update((b, e - 1))
    rows, cols = sorted(rows), sorted(cols)
    pts = {(0, 0), (0, ny - 1), (nx - 1, 0), (nx - 1, ny - 1)}
    pts.update((r, cols[k % len(cols)]) for k, r in enumerate(rows))
    pts.update((rows[(3 * k) % len(rows)], c) for k, c in enumerate(cols))
    return sorted(pts)


def probe_kind(geo, pt):
    """sub-pixel by default; the frame corners and other pixels on a frame border are pushed out of it
    (the source clamps); two in five other points keep a zero x (or y) field, so that they land on an
    integer row (column): on the last row (column) itself exactly"""
    nx, ny, _, _ = GEOMETRIES[geo]
    i, j = pt
    if i in (0, nx - 1) and j in (0, ny - 1):
        return "clamp"
    h = (7 * i + 13 * j) % 5
    if h == 0:
        return "integer_x"
    if h == 1:
        return "integer_y"
    if i in (0, nx - 1) or j in (0, ny - 1):
        return "clamp"
    return "sub"


def probe_case(geo, pt):
    """-> (sector displacement, template, input, mask) with every pixel masked but pt, and a displacement
    at pt under one pixel so that pt's source footprint keeps weight on pt itself"""
    nx, ny, xs, ys = GEOMETRIES[geo]
    i, j = pt
    kind = probe_kind(geo, pt)
    rng = np.random.default_rng(1000003 * i + 7919 * j + nx + 31 * xs + ys)
    bias = rng.choice([-0.35, 0.35], 2)
    if kind == "clamp":   # outward at a border: x - d < 0 at row 0, > xmi at the last row
        bias = np.array([0.35 if i == 0 else -0.35 if i == nx - 1 else bias[0],
                         0.35 if j == 0 else -0.35 if j == ny - 1 else bias[1]])
    sd = bias[:, None, None] + rng.uniform(-0.05, 0.05, (2, xs, ys))
    if kind == "integer_x":
        sd[0] = 0.0
    elif kind == "integer_y":
        sd[1] = 0.0
    templ, inp = _probe_frames(geo)
    mask = np.ones((nx, ny), np.int8)
    mask[i, j] = 0
    return np.ascontiguousarray(sd), templ, inp, mask


@functools.lru_cache(maxsize=2)
def _probe_frames(geo):
    """template and input shared by a geometry's probes (read-only)"""
    nx, ny, _, _ = GEOMETRIES[geo]
    rng = np.random.default_rng(nx * 7 + ny)
    frames = 10 * rng.random((2, nx, ny))
    frames.flags.writeable = False
    return frames[0], frames[1]


def probe_expect(geo, pt, sd, templ, inp, mask):
    """the single pixel's residual term and the gradient it alone makes: its term in the four sectors of its
    cell, zeros elsewhere (and everywhere when pt is on a band's skipped last row)"""
    _, _, xs, ys = GEOMETRIES[geo]
    t = pixel_terms(sd, templ, inp, mask, np.array([pt[0]]), np.array([pt[1]]))
    assert t["contributes"][0], f"{geo} {pt}: the probe pixel is masked by its own warp"
    grad = np.zeros((2, xs, ys))
    for k, (dl, dm) in enumerate(CORNERS):
        for a in (0, 1):
            grad[a, t["l0"][0] + dl, t["m0"][0] + dm] = t["grad"][k, a, 0]
    return float(t["res"][0]), grad, t


def probe_eval(geo, pt, sd, templ, inp, mask, gain):
    """probe_expect as exact sums with magnitudes (the form check_sums takes), smoothness included"""
    nx, ny, _, _ = GEOMETRIES[geo]
    res, grad, t = probe_expect(geo, pt, sd, templ, inp, mask)
    ev = dict(res=res, res_abs=res, nres=1, grad=grad, grad_abs=np.abs(grad), nterms=(grad != 0).astype(np.int64))
    ev.update(smooth_exact(sd, nx, ny, gain))
    return ev


def probe_branches(geo, pts, sms):
    """what a geometry's probes reach"""
    nx, ny, xs, ys = GEOMETRIES[geo]
    p = partition(nx, ny, xs, ys, sms)
    got = set()
    for pt in pts:
        sd, templ, inp, mask = probe_case(geo, pt)
        t = pixel_terms(sd, templ, inp, mask, np.array([pt[0]]), np.array([pt[1]]))
        w = t["warp"]
        for key in ("x_low", "x_high", "y_low", "y_high", "x_integer", "y_integer", "x_on_last", "y_on_last"):
            if w[key][0]:
                got.add(key)
        if not t["grow"][0]:
            got.add("skipped row")
        l = int(t["l0"][0])
        sr = strip_rows(p, l)
        if pt[0] == sr[-1][0] and len(sr) > 1:
            got.add("last strip first row")
        if p["used"][l] < p["strips"]:
            got.add("band with empty trailing strips")
    return got
