"""The edge grid of the dense LK front end and of the Shi-Tomasi eigenvalue map, with a NumPy classifier
of the branch every case takes.

  front end   csrc/lk_frontend.cu (fused: 64 x 16 pixel tiles staged by TMA in a 68 x 20 box, a two-slot
              ring walked by persistent CTAs, nparts = min(tiles, 4 x SMs)) and the stage kernels of
              csrc/lk_dense.cu (mask_invalid in PAIR / scalar form, morph_open, masked_minmax, quantise)
  eigen map   csrc/lk_dense.cu cov_rowsum (64 x 8 tiles, FMA columns below tail0 = 32 floor(w / 32)),
              box_chain (interior rounds of BOX_U rows while y0 + BOX_R + BOX_U + 2 <= h, then the
              reflected tail; lanes past the last column shadow it) and eig_from_box

Every case names the branches it is there for (`why`); `front_branches` / `eig_branches` compute the
branches a case takes from its shape, contents and the SM count, and the tests assert both that each
case reaches what it names and that the grid as a whole reaches every branch in FRONT_REQUIRED /
EIG_REQUIRED.  tests/test_oracle_lk_frontend_edges.py pins the oracle to cv2 and to the reference on
this grid (CPU); tests/test_lk_frontend_edges_gpu.py holds the kernels to the oracle on it.  Nothing
here imports cv2: the GPU machines do not have it."""
import functools
import math

import numpy as np

from oracle import lucaskanade as ora

FW, FH, HALO = 64, 16, 2                 # lk_frontend.cu: pixel tile, halo
BW, BH = FW + 2 * HALO, FH + 2 * HALO    # TMA box
CR_W, CR_H = 64, 8                       # lk_dense.cu cov_rowsum tile
BOX_R, BOX_U = 64, 8                     # lk_dense.cu box_chain ring depth and rows per round
H100_SXM_SMS = 132                       # the SM count the CPU tests assume (read at run time on the GPU)


# ------------------------------------------------------------------------------------------ front end
def _rand(m, n, seed, zeros=0.35):
    """values in [0, 40) with a share of exact zeros (the frame minimum: the opening's background)"""
    rng = np.random.default_rng(seed)
    a = rng.random((m, n)) * 40.0
    a[rng.random((m, n)) < zeros] = 0.0
    return a


def _seam_positions(size, period):
    """indices period*k - 2 .. period*k + 1 (k >= 1) and the two borders, inside 0 .. size-1"""
    idx = {0, size - 1}
    for k in range(1, size // period + 1):
        idx.update(range(period * k - 2, period * k + 2))
    return sorted(i for i in idx if 0 <= i < size)


def _seam_points(m, n):
    """pixels on every seam row and border row at spread-out columns, and on every seam / border
    column at spread-out rows"""
    pts = set()
    rows, cols = _seam_positions(m, FH), _seam_positions(n, FW)
    for j, r in enumerate(rows):
        pts.update((r, c) for c in range(j % 7, n, 23))
    for j, c in enumerate(cols):
        pts.update((r, c) for r in range(j % 5, m, 11))
    return sorted(pts)


def _cross_probes(a, y, x, axis, sign, survive):
    """Foreground that survives (or dies in) the opening only because of the pixel two away across a
    tile seam: p = (y, x) is the pixel on this side of the seam, c = p + sign*e the centre of a cross on
    the other side, q = p + 2*sign*e the far arm.  With q set, c is eroded and p survives; without it no
    pixel of p's cross is eroded."""
    e = (0, 1) if axis == 1 else (1, 0)
    o = (1, 0) if axis == 1 else (0, 1)
    cy, cx = y + sign * e[0], x + sign * e[1]
    for py, px in ((y, x), (cy, cx), (cy + o[0], cx + o[1]), (cy - o[0], cx - o[1])):
        a[py, px] = 7.0 + (py + px) % 5
    q = (y + 2 * sign * e[0], x + 2 * sign * e[1])
    if survive:
        a[q] = 9.5
    return ((y, x), q, "survive" if survive else "die")


def _opening_frame(m, n):
    a = np.zeros((m, n))
    probes = []
    for k, x in enumerate((FW - 1, 2 * FW - 1, 3 * FW - 1)):          # column seams, p left of the seam
        probes.append(_cross_probes(a, 5 + 6 * k, x, 1, +1, True))
        probes.append(_cross_probes(a, 8 + 6 * k + 20, x, 1, +1, False))
    for k, x in enumerate((FW, 2 * FW)):                              # p right of the seam
        probes.append(_cross_probes(a, 45 + 6 * k, x, 1, -1, k == 0))
        probes.append(_cross_probes(a, 60 - 6 * k, x, 1, -1, k != 0))
    for k, y in enumerate((FH - 1, 2 * FH - 1, 3 * FH - 1)):          # row seams, p above the seam
        probes.append(_cross_probes(a, y, 10 + 30 * k, 0, +1, True))
        probes.append(_cross_probes(a, y, 25 + 30 * k + 100, 0, +1, False))
    for k, y in enumerate((FH, 3 * FH)):                              # p below the seam
        probes.append(_cross_probes(a, y, 170 + 20 * k, 0, -1, True))
        probes.append(_cross_probes(a, y, 230 - 10 * k, 0, -1, False))
    return a, probes


def _checker_mask(m, n):
    return (np.indices((m, n)).sum(0) % 2 == 0)


def _tiles(m, n):
    return math.ceil(n / FW) * math.ceil(m / FH)


def _tile_shape(kind, k, sms):
    """(m, n) of a tall 64-wide (kind 'tall') or short wide ('wide') frame of 4*sms + k tiles, k in
    {-1, 0, 1, 4*sms + 1, 3*(4*sms) + 1} -- partial last tiles"""
    t = 4 * sms + k
    return (FH * t - 3, FW) if kind == "tall" else (FH - 3, FW * t - 2)


_CTA_WHY = {"nparts": {"cta-tiles=1"}, "nparts+1": {"cta-tiles=2"}, "2nparts+1": {"cta-tiles=3", "parity-flip"},
            "4nparts+1": {"cta-tiles=5"}}
_TILE_STEPS = {"nparts-1": lambda p: -1, "nparts": lambda p: 0, "nparts+1": lambda p: 1,
               "2nparts+1": lambda p: p + 1, "4nparts+1": lambda p: 3 * p + 1}


def _fcase(tag, m, n, why, content="rand", buffer_mask=5, opening=3, f32=False, offset=0, user="none", seed=0):
    return tag, dict(m=m, n=n, why=frozenset(why), content=content, buffer_mask=buffer_mask, opening=opening,
                     f32=f32, offset=offset, user=user, seed=seed)


FRONT_CASES = dict([
    # every m and n of the fused path, with buffer_mask 0 .. 5, opening 0 and float32 frames spread over them
    _fcase("s1x2", 1, 2, {"m=1", "n=2", "buffer=0", "box>frame", "det_set=0"}, "rand_nan", buffer_mask=0),
    _fcase("s2x4", 2, 4, {"m=2", "n=4", "buffer=1"}, "rand_nan", buffer_mask=1, seed=1),
    _fcase("s3x62", 3, 62, {"m=3", "n=62", "buffer=2"}, "rand_nan", buffer_mask=2, seed=2),
    _fcase("s15x64", 15, 64, {"m=15", "n=64", "opening=0"}, "rand_nan", buffer_mask=3, opening=0, seed=3),
    _fcase("s16x66", 16, 66, {"m=16", "n=66", "buffer=4"}, "rand_nan", buffer_mask=4, f32=True, seed=4),
    _fcase("s17x68", 17, 68, {"m=17", "n=68", "buffer=5", "path=fused", "f64", "opening=3",
                                       "mask_invalid:pair"}, "rand_nan", seed=5),
    _fcase("s18x128", 18, 128, {"m=18", "n=128", "buffer=3"}, "rand_nan", buffer_mask=3, opening=0, seed=6),
    _fcase("s33x130", 33, 130, {"m=33", "n=130", "f32"}, "rand_nan", buffer_mask=2, f32=True, seed=7),
    _fcase("s33x2", 33, 2, {"m=33,n=2"}, "rand_nan", seed=8),
    _fcase("s1x130", 1, 130, {"m=1,n=130"}, "rand_nan", buffer_mask=0, seed=9),
    _fcase("s18x4", 18, 4, {"m=18,n=4"}, "rand_nan", buffer_mask=1, f32=True, seed=10),
    # tile counts around the persistent grid: one tile per CTA, two, three (the ring's parity flips) and five
    *[_fcase(f"{kind}-{step}", 0, 0, {f"{kind}:tiles={step}"} | (_CTA_WHY.get(step, set()) if kind == "tall" else set()),
             "rand_nan", buffer_mask=5 - i % 3,
             opening=3 * (i % 2 == 0), seed=20 + i + 10 * (kind == "wide"))
      for kind in ("tall", "wide") for i, step in enumerate(_TILE_STEPS)],
    # NaN, +-inf and user-masked finite pixels on seam rows / columns and the border
    _fcase("seam-nonfinite", 70, 260, {"nonfinite@row-seam", "nonfinite@col-seam", "nonfinite@border"},
           "seam_nonfinite", seed=30),
    _fcase("seam-usermask", 70, 260, {"usermask@row-seam", "usermask@col-seam", "usermask@border"},
           user="seams", buffer_mask=3, seed=31),
    _fcase("seam-nonfinite-f32", 70, 260, {"f32+nonfinite"}, "seam_nonfinite", buffer_mask=4, f32=True, seed=32),
    _fcase("opening-seam", 70, 260, {"opening:survive-across-seam", "opening:die-across-seam"}, "opening",
           buffer_mask=0),
    _fcase("usermask-minmax", 70, 260, {"usermask:min+max"}, "extremes", user="extremes", seed=33),
    # the (any_clear, any_masked) combinations of feature/shitomasi.py:139 (a 1-row frame with anything
    # masked and buffer_mask > 0 is left out: there the reference's integer indexing raises IndexError)
    _fcase("nothing-masked", 50, 130, {"clear=1,masked=0", "det_set=1"}, "rand", buffer_mask=5, seed=34),
    _fcase("all-but-one", 50, 130, {"all-but-one", "clear=0,masked=1"}, user="all_but_one", buffer_mask=3, seed=35),
    _fcase("all-buffered", 50, 130, {"all-buffered"}, user="checker", buffer_mask=2, opening=0, seed=36),
    _fcase("rows01-masked", 50, 130, {"rows01-only", "clear=1,masked=1", "det_set=2"}, user="rows01", buffer_mask=4, seed=37),
    # scaling edges
    _fcase("flat", 40, 130, {"flat"}, "flat", buffer_mask=5),
    _fcase("flat-within-1e-8", 40, 130, {"flat<=1e-8"}, "flat_eps", buffer_mask=0),
    _fcase("mostly-min", 40, 130, {"mostly-min"}, "mostly_min", buffer_mask=5, opening=0, seed=38),
    # the stage path: odd widths, odd m*n (scalar mask_invalid), buffer_mask 6, 7, 31, a misaligned frame
    _fcase("stage1x1", 1, 1, {"n=1"}, "rand", buffer_mask=0),
    _fcase("stage3x3", 3, 3, {"n=3", "buffer=7", "mask_invalid:scalar-odd"}, "rand_nan", buffer_mask=7, seed=40),
    _fcase("stage17x63", 17, 63, {"n=63", "buffer=31", "path=stage"}, "rand_nan", buffer_mask=31, seed=41),
    _fcase("stage33x65", 33, 65, {"n=65", "buffer=6"}, "seam_nonfinite", buffer_mask=6, opening=0, user="seams", seed=42),
    _fcase("stage5x129", 5, 129, {"n=129", "stage+f32"}, "rand_nan", buffer_mask=7, f32=True, seed=43),
    _fcase("stage-even-buffer31", 34, 66, {"stage:even-width"}, "rand_nan", buffer_mask=31, user="all_but_one",
           seed=44),
    _fcase("stage-misaligned", 20, 64, {"mask_invalid:misaligned"}, "rand_nan", buffer_mask=5, offset=1, seed=45),
])

FRONT_REQUIRED = frozenset(
    {f"m={m}" for m in (1, 2, 3, 15, 16, 17, 18, 33)} | {f"n={n}" for n in (2, 4, 62, 64, 66, 68, 128, 130)} |
    {f"n={n}" for n in (1, 3, 63, 65, 129)} | {f"buffer={b}" for b in (0, 1, 2, 3, 4, 5, 6, 7, 31)} |
    {"opening=0", "opening=3", "f32", "f64", "path=fused", "path=stage"} |
    {f"{kind}:tiles={s}" for kind in ("tall", "wide") for s in _TILE_STEPS} |
    {"cta-tiles=1", "cta-tiles=2", "cta-tiles=3", "cta-tiles=5", "parity-flip", "box>frame"} |
    {f"{w}@{s}" for w in ("nonfinite", "usermask") for s in ("row-seam", "col-seam", "border")} |
    {"opening:survive-across-seam", "opening:die-across-seam", "usermask:min+max"} |
    {"clear=1,masked=0", "clear=0,masked=1", "clear=1,masked=1", "all-but-one", "all-buffered", "rows01-only"} |
    {"det_set=0", "det_set=1", "det_set=2", "flat", "flat<=1e-8", "mostly-min"} |
    {"mask_invalid:pair", "mask_invalid:scalar-odd", "mask_invalid:misaligned"} |
    {"m=33,n=2", "m=1,n=130", "m=18,n=4", "f32+nonfinite", "stage+f32", "stage:even-width"})


def front_shape(tag, sms=H100_SXM_SMS):
    c = FRONT_CASES[tag]
    kind, _, step = tag.partition("-")
    if step in _TILE_STEPS and kind in ("tall", "wide"):
        return _tile_shape(kind, _TILE_STEPS[step](4 * sms), sms)
    return c["m"], c["n"]


@functools.lru_cache(maxsize=None)
def _front_inputs(tag, sms):
    c = FRONT_CASES[tag]
    m, n = front_shape(tag, sms)
    rng = np.random.default_rng(1000 + c["seed"])
    probes = []
    kind = c["content"]
    if kind in ("rand", "rand_nan"):
        a = _rand(m, n, c["seed"])
        if kind == "rand_nan":
            a[rng.random((m, n)) < 0.01] = np.nan
            a[rng.random((m, n)) < 0.002] = np.inf
    elif kind == "seam_nonfinite":
        a = _rand(m, n, c["seed"])
        for j, (y, x) in enumerate(_seam_points(m, n)):
            a[y, x] = (np.nan, np.inf, -np.inf)[j % 3]
    elif kind == "opening":
        a, probes = _opening_frame(m, n)
    elif kind == "extremes":
        a = 1.0 + _rand(m, n, c["seed"], zeros=0.0)
        a[5, 7], a[61, 200] = -100.0, 500.0
    elif kind == "flat":
        a = np.full((m, n), 3.25)
    elif kind == "flat_eps":
        a = np.full((m, n), 3.25)
        a[rng.random((m, n)) < 0.5] += 5e-9
    elif kind == "mostly_min":
        a = _rand(m, n, c["seed"], zeros=0.97)
    else:
        raise KeyError(kind)
    um = None
    user = c["user"]
    if user == "seams":
        um = np.zeros((m, n), bool)
        for y, x in _seam_points(m, n):
            um[y, x] = True
    elif user == "extremes":
        um = np.zeros((m, n), bool)
        um[5, 7] = um[61, 200] = True
    elif user == "all_but_one":
        um = np.ones((m, n), bool)
        um[0, n // 2] = False       # row 0: the rows the detector's integer indexing keeps decide it
    elif user == "checker":
        um = _checker_mask(m, n)
        a[0, 1] = 100.0             # the maximum on a clear pixel of row 0: only the rows != 1 set holds it
    elif user == "rows01":
        um = np.zeros((m, n), bool)
        um[:2] = True
    if c["f32"]:
        a = a.astype(np.float32)
    return a, um, probes


def front_inputs(tag, sms=H100_SXM_SMS):
    """(frame, user mask or None, opening probes, case) -- the frame is float32 for the f32 cases (the
    device gets it widened to float64 with B200_QUANTISE_F32)"""
    a, um, probes = _front_inputs(tag, sms)
    return a, um, probes, FRONT_CASES[tag]


def masked_frame(a, um):
    """the MaskedArray dense_lucaskanade / shitomasi.detection derive from a frame and a user mask"""
    mk = ~np.isfinite(a) if um is None else (um | ~np.isfinite(a))
    return np.ma.MaskedArray(a, mask=mk)


def _dilated(mask, k):
    return ora.dilate_rect(mask.astype(np.uint8), k).astype(bool) if k > 0 else mask


def _open_keep(fg):
    return ora.morph_open_cross3(fg.astype(np.uint8)).astype(bool)


def front_stats(opened, mask, buffer_mask):
    """the 12 statistics of the opened image: [min, max, count] of the unmasked pixels of all rows
    (set 0), of the rows the detector scales when it masks row 0 (set 1: rows >= 1) or row 1 alone
    (set 1 when anything is masked: rows != 1), of rows >= 2 (set 2); set 3 is [inf, -inf, number of
    pixels whose buffered mask is clear].  An empty set is [nan, nan, 0]."""
    m = mask.shape[0]
    rows = np.arange(m)[:, None]
    any_masked = bool(mask.any())
    v = np.asarray(opened, np.float64)

    def mm(sel):
        s = v[sel]
        return [s.min(), s.max(), float(s.size)] if s.size else [np.nan, np.nan, 0.0]

    buffered = _dilated(mask, buffer_mask) if any_masked else mask
    clear = int((~buffered).sum())
    set1 = (rows != 1) if any_masked else (rows >= 1)
    return np.array(mm(~mask) + mm(~mask & set1) + mm(~mask & (rows >= 2)) +
                    ([np.inf, -np.inf, float(clear)] if clear else [np.nan, np.nan, 0.0]))


def front_branches(tag, sms=H100_SXM_SMS):
    """the branches the front end takes on a case"""
    a, um, probes, c = front_inputs(tag, sms)
    m, n = a.shape
    b, op = c["buffer_mask"], c["opening"]
    out = {f"m={m}", f"n={n}", f"m={m},n={n}", f"buffer={b}", f"opening={op}", "f32" if c["f32"] else "f64"}
    fused = n % 2 == 0 and 0 <= b <= 5 and (c["offset"] * 8) % 16 == 0
    out.add("path=fused" if fused else "path=stage")
    if not fused and n % 2 == 0:
        out.add("stage:even-width")
    if c["f32"]:
        out.add("stage+f32" if not fused else "fused+f32")
    # mask_invalid: PAIR for an even pixel count and a 16-byte aligned frame
    if (m * n) % 2:
        out.add("mask_invalid:scalar-odd")
    elif c["offset"] % 2:
        out.add("mask_invalid:misaligned")
    else:
        out.add("mask_invalid:pair")
    if fused:
        tiles = _tiles(m, n)
        nparts = min(tiles, 4 * sms)
        per_cta = -(-tiles // nparts)
        out.add(f"cta-tiles={per_cta}")
        if [(it >> 1) & 1 for it in range(per_cta)].count(1):
            out.add("parity-flip")
        if m < BH or n < BW:
            out.add("box>frame")
        for kind, shape_ok in (("tall", n == FW), ("wide", math.ceil(m / FH) == 1)):
            for step, f in _TILE_STEPS.items():
                if shape_ok and tiles == 4 * sms + f(4 * sms):
                    out.add(f"{kind}:tiles={step}")
    # where the non-finite and the user-masked pixels lie
    rows, cols = _seam_positions(m, FH), _seam_positions(n, FW)
    for what, sel in (("nonfinite", ~np.isfinite(a)), ("usermask", (um & np.isfinite(a)) if um is not None
                                                        else np.zeros((m, n), bool))):
        ys, xs = np.nonzero(sel)
        if any(y in rows and y % FH in (FH - 2, FH - 1, 0, 1) and 0 < y < m - 1 for y in ys):
            out.add(f"{what}@row-seam")
        if any(x in cols and x % FW in (FW - 2, FW - 1, 0, 1) and 0 < x < n - 1 for x in xs):
            out.add(f"{what}@col-seam")
        if any(y in (0, m - 1) or x in (0, n - 1) for y, x in zip(ys, xs)):
            out.add(f"{what}@border")
    if c["f32"] and (~np.isfinite(a)).any():
        out.add("f32+nonfinite")
    ma = masked_frame(a.astype(np.float64), um)
    mask = np.ma.getmaskarray(ma)
    vals = a[~mask].astype(np.float64)
    minval = vals.min() if vals.size else np.inf
    # opening probes: p's fate flips with the pixel q two away, across a seam
    if op and probes:
        fg = ~mask & (np.asarray(a, np.float64) > minval)
        for p, q, fate in probes:
            assert (p[0] // FH, p[1] // FW) != (q[0] // FH, q[1] // FW), "probe does not cross a seam"
            flip = fg.copy()
            flip[q] = not flip[q]
            now, other = _open_keep(fg)[p], _open_keep(flip)[p]
            if fg[p] and now != other and now == (fate == "survive"):
                out.add(f"opening:{fate}-across-seam")
    if um is not None and vals.size:
        hidden = a[um & np.isfinite(a)]
        if hidden.size and hidden.min() < vals.min() and hidden.max() > vals.max():
            out.add("usermask:min+max")
    # the detector's integer-indexing quirk (feature/shitomasi.py:139)
    any_masked = bool(mask.any())
    buffered = _dilated(mask, b) if (b > 0 and any_masked) else mask
    any_clear = bool((~buffered).any())
    if b > 0:
        out.add(f"clear={int(any_clear)},masked={int(any_masked)}")
        out.add(f"det_set={int(any_clear) + int(any_masked)}")
    else:
        out.add("det_set=0")
    if (~mask).sum() == 1:
        out.add("all-but-one")
    if b > 1 and any_masked and not any_clear and (~mask).any():
        out.add("all-buffered")
    if mask[:2].all() and not mask[2:].any():
        out.add("rows01-only")
    if vals.size and vals.max() - vals.min() <= 1e-8:
        out.add("flat" if vals.max() == vals.min() else "flat<=1e-8")
    if vals.size and (vals == minval).mean() > 0.9:
        out.add("mostly-min")
    return out


# ------------------------------------------------------------------------------------ eigenvalue map
EIG_WIDTHS = (1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 66, 67, 68, 95, 96, 97, 128, 129)
EIG_HEIGHTS = (1, 2, 3, 4, 5, 8, 9, 63, 64, 65, 66, 73, 74, 75, 81, 82, 83, 137, 138, 139, 4099)
_EIG_AT_H = (5, 75, 139)     # every width at: tail only, one interior round, nine rounds
_EIG_AT_W = (3, 64, 97)      # every height at: scalar columns only, no scalar tail, a split and shadow lanes


def _eig_content(kind, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (h, w)).astype(np.uint8)
    if kind == "checker":
        return ((np.indices((h, w)).sum(0) % 2) * 255).astype(np.uint8)
    if kind == "flat":
        return np.full((h, w), 200, np.uint8)
    if kind == "stripes-h":
        return ((np.arange(h)[:, None] % 3 == 0) * 255 * np.ones((1, w))).astype(np.uint8)
    if kind == "stripes-v":
        return ((np.arange(w)[None, :] % 2 == 0) * 255 * np.ones((h, 1))).astype(np.uint8)
    if kind in ("bright-seams", "bright-corners"):
        q = np.zeros((h, w), np.uint8)
        if kind == "bright-corners":
            pts = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)]
        else:
            pts = [(y, x) for y in _seam_positions(h, CR_H) for x in _seam_positions(w, CR_W)
                   if (y % CR_H in (CR_H - 1, 0)) and (x % CR_W in (CR_W - 1, 0))]
        for y, x in pts:
            q[y, x] = 255
        return q
    raise KeyError(kind)


# the cases that declare the chain / column branches (each is also reached elsewhere)
_EIG_BRANCH_WHY = {"random-5x3": {"chain:tail-only", "chain:tail<BOX_U", "tail0=0"},
                   "random-75x64": {"tail0=w", "full-warps"},
                   "checker-139x129": {"chain:interior", "tail0-split", "shadow-lanes", "cov:partial-tile-x",
                                       "cov:partial-tile-y"},
                   "bright-seams-139x129": {"cov:bright-on-seam"}}


def _ecase(h, w, kind="random", why=None):
    tag = f"{kind}-{h}x{w}"
    why = set(why if why is not None else {f"h={h}@w={w}"}) | _EIG_BRANCH_WHY.get(tag, set())
    return tag, dict(h=h, w=w, kind=kind, why=frozenset(why))


EIG_CASES = dict([
    *[_ecase(h, w) for h in _EIG_AT_H for w in EIG_WIDTHS],
    *[_ecase(h, w) for w in _EIG_AT_W for h in EIG_HEIGHTS if h not in _EIG_AT_H],
    # contents: the largest covariance sums, flat, stripes, single bright pixels on the 64 x 8 tile seams
    # and at the corners
    *[_ecase(h, w, kind, {f"{kind}@{h}x{w}"}) for kind in ("checker", "flat", "stripes-h", "stripes-v",
                                                            "bright-seams", "bright-corners")
      for h, w in ((139, 129), (75, 66), (9, 33))],
])

EIG_REQUIRED = frozenset(
    {f"h={h}@w={w}" for h in _EIG_AT_H for w in EIG_WIDTHS} |
    {f"h={h}@w={w}" for w in _EIG_AT_W for h in EIG_HEIGHTS} |
    {f"{k}@{h}x{w}" for k in ("checker", "flat", "stripes-h", "stripes-v", "bright-seams", "bright-corners")
     for h, w in ((139, 129), (75, 66), (9, 33))} |
    {"chain:interior", "chain:tail-only", "chain:tail<BOX_U", "tail0=0", "tail0=w", "tail0-split",
     "shadow-lanes", "full-warps", "cov:partial-tile-x", "cov:partial-tile-y", "cov:bright-on-seam"})


@functools.lru_cache(maxsize=None)
def eig_input(tag):
    c = EIG_CASES[tag]
    return _eig_content(c["kind"], c["h"], c["w"], c["h"] * 1009 + c["w"])


def chain_rounds(h):
    """box_chain: the interior rounds (BOX_U rows each) and the rows its reflected tail loop takes"""
    rounds = max(0, (h - (BOX_R + BOX_U + 2)) // BOX_U + 1)
    return rounds, h - BOX_U * rounds


def eig_branches(tag):
    c = EIG_CASES[tag]
    h, w = c["h"], c["w"]
    out = {f"h={h}@w={w}", f"{c['kind']}@{h}x{w}"}
    rounds, tail = chain_rounds(h)
    out.add("chain:interior" if rounds else "chain:tail-only")
    if tail < BOX_U:
        out.add("chain:tail<BOX_U")
    tail0 = 32 * (w // 32)
    out.add("tail0=0" if tail0 == 0 else "tail0=w" if tail0 == w else "tail0-split")
    out.add("shadow-lanes" if w % 32 else "full-warps")
    if w % CR_W:
        out.add("cov:partial-tile-x")
    if h % CR_H:
        out.add("cov:partial-tile-y")
    q = eig_input(tag)
    ys, xs = np.nonzero(q)
    if c["kind"] == "bright-seams" and any((y % CR_H in (CR_H - 1, 0) and 0 < y < h - 1) or
                                           (x % CR_W in (CR_W - 1, 0) and 0 < x < w - 1) for y, x in zip(ys, xs)):
        out.add("cov:bright-on-seam")
    return out
