"""TEST INFRASTRUCTURE: extended-precision references of the three DARTS entry points
(pysteps_b200/csrc/darts.cu) with a-priori forward-error bounds, and a NumPy restatement of
darts_normal_kernel that matches it bit for bit.  Every reference works on exactly the float64 inputs
the device receives (frames, the twiddle tables of motion.darts.spectrum_tables, the spectrum block,
the coefficients and their tables) and computes in np.longdouble (x87 extended, 64-bit significand).

The bounds are first-order sums of |terms| times a count of roundings, derived at each function;
u = 2^-53 is the unit roundoff of float64.  The factor SLACK = 1 + 2^-10 on every bound covers the
second-order terms, the float64 rounding of the bound's own |.| sums (at most (n + m + T) u relative)
and the longdouble reference's error (its sums round at 2^-64 = u / 2^11 per addition).

Also the edge cases that tests/test_darts_bound.py (CPU) and tests/test_darts_edges_gpu.py (device)
share: the spectra, the normal equations and the syntheses at the kernels' tile and parameter edges."""
import numpy as np
import pytest

LD = np.longdouble
if np.finfo(LD).eps > 2.0 ** -63:
    pytest.skip("np.longdouble is not x87 extended precision here", allow_module_level=True)

U = 2.0 ** -53
SLACK = 1.0 + 2.0 ** -10
NORMAL_ROWS = 512  # B200_DARTS_NORMAL_ROWS
XF = 64            # darts_rows_kernel's frequency tile


def _ld(a):
    return np.asarray(a, dtype=np.float64).astype(LD)


def x_selection(K, n, kx=None):
    """(f, cj) of the block columns kx (default all 2K+1): the x-pass frequency each reads and whether
    it is conjugated (2w > n, w = (kx - K) mod n), as darts_time_kernel reads them"""
    kx = np.arange(2 * K + 1) if kx is None else np.asarray(kx)
    w = (kx - K) % n
    cj = 2 * w > n
    return np.where(cj, n - w, w), cj


# ---- spectrum ---------------------------------------------------------------------------------
def spectrum_gamma(T, m, n):
    """Relative factor of the spectrum bound: |X_device - X| <= spectrum_gamma * S entrywise (complex
    modulus), S the three passes on |frames - c0| and |tw|.

      subtraction  a = frames - c0 in float64 (float32 frames widen exactly):          1
      x pass       P = sum_x a tw_x: n FMAs per component, so each of Re and Im is
                   within n u sum |a| |tw_x.re| (resp. .im), and the pair within
                   n u sum |a| |tw_x| (triangle inequality in R^2):                     n
      t pass       Re Q = sum_t (c.re p.re - c.im p.im) runs 2T FMAs, within
                   2T u sum (|c.re p.re| + |c.im p.im|); with Im alike the modulus is
                   within 2 sqrt(2) T u sum |c| |p| (the worst case has |c.re| = |c.im|
                   and |p.re| = |p.im|); 2 sqrt(2) < 3:                                3T
      y pass       the same over m terms:                                              3m

    P's error enters the t pass through |tw_t|, Q's the y pass through |tw_y|, which is how S
    propagates it.  c = 1 (the subtraction); SLACK covers the rest (module docstring)."""
    return (n + 3 * T + 3 * m + 1) * U * SLACK


def _passes(frames, tw_x, f, cj, tw_t, tw_y, absolute):
    """x, t and y passes on the rows a = frames - frames[0, 0, 0]: in longdouble, or with
    absolute=True on |a| and |tw| in float64 (the bound's sums, whose rounding SLACK covers)"""
    T, m, n = frames.shape
    fs, inv = np.unique(f, return_inverse=True)
    tx = tw_x[fs]
    if absolute:
        a = np.abs(frames.reshape(T * m, n).astype(np.float64) - np.float64(frames[0, 0, 0]))
        Px = (a @ np.abs(tx).T)[:, inv].reshape(T, m, -1)
        Q = np.tensordot(np.abs(tw_t), Px, axes=(1, 0))
        return np.matmul(np.abs(tw_y)[None], Q)
    c0 = LD(np.float64(frames[0, 0, 0]))
    Pr = np.empty((T, m, len(fs)), LD)
    Pi = np.empty((T, m, len(fs)), LD)
    txr, txi = _ld(tx.real).T.copy(), _ld(tx.imag).T.copy()
    for t in range(T):  # one frame at a time: a 2048^2 frame is 64 MB in longdouble
        a = _ld(frames[t]) - c0  # rounds at 2^-64 relative at most (SLACK)
        Pr[t] = a @ txr
        Pi[t] = a @ txi
    Pr, Pi = Pr[:, :, inv], Pi[:, :, inv]
    Pi[:, :, cj] = -Pi[:, :, cj]
    ttr, tti = _ld(tw_t.real), _ld(tw_t.imag)
    Qr = np.tensordot(ttr, Pr, axes=(1, 0)) - np.tensordot(tti, Pi, axes=(1, 0))
    Qi = np.tensordot(ttr, Pi, axes=(1, 0)) + np.tensordot(tti, Pr, axes=(1, 0))
    tyr, tyi = _ld(tw_y.real)[None], _ld(tw_y.imag)[None]
    return np.matmul(tyr, Qr) - np.matmul(tyi, Qi), np.matmul(tyr, Qi) + np.matmul(tyi, Qr)


def spectrum(frames, tw_x, tw_y, tw_t, K, kx=None, ky=None):
    """-> (Xr, Xi, B): the (Kt, len(ky), len(kx)) block of b200_darts_spectrum in longdouble (real
    and imaginary parts) and its bound; kx, ky select block columns and rows (default all)."""
    T, m, n = frames.shape
    f, cj = x_selection(K, n, kx)
    ty = tw_y if ky is None else tw_y[np.asarray(ky)]
    Xr, Xi = _passes(frames, tw_x, f, cj, tw_t, ty, False)
    S = _passes(frames, tw_x, f, cj, tw_t, ty, True)
    return Xr, Xi, spectrum_gamma(T, m, n) * S


def complex_ratio(got, ref_re, ref_im, bound):
    """max over entries of |got - ref| / bound (complex modulus); bound 0 needs got == ref exactly"""
    got = np.asarray(got)
    dr, di = _ld(got.real) - ref_re, _ld(got.imag) - ref_im
    err = np.sqrt(dr * dr + di * di)
    return _ratio(err, bound)


def _ratio(err, bound):
    err = np.asarray(err, LD)
    bound = np.asarray(bound, LD)
    if np.any((bound == 0) & (err != 0)):
        return float("inf")
    nz = bound > 0
    return float((err[nz] / bound[nz]).max()) if nz.any() else 0.0


# ---- normal equations --------------------------------------------------------------------------
def pairs(nc):
    """(c, d) of darts_normal_kernel's pairs: the upper triangle c <= d < nc column by column, then
    d = nc (M^H y) for c = 0 .. nc - 1"""
    d = np.concatenate([np.full(q + 1, q) for q in range(nc)] + [np.full(nc, nc)])
    c = np.concatenate([np.arange(q + 1) for q in range(nc)] + [np.arange(nc)])
    return c, d


def _entries(X, N_x, N_y, N_t, M_x, M_y):
    """(kt, i_, j_, Z, z): rows of M in the reference's (k_t, k_y, k_x) order, the A and B columns'
    integer factors i_, j_ (rows, hw), the spectrum entries Z (rows, hw) they scale, and y's z"""
    X = np.asarray(X)
    kt, ky, kx = (a.ravel() for a in np.meshgrid(np.arange(-N_t, N_t + 1), np.arange(-N_y, N_y + 1),
                                                 np.arange(-N_x, N_x + 1), indexing="ij"))
    mw = 2 * M_x + 1
    q = np.arange((2 * M_y + 1) * mw)
    i_ = ky[:, None] - (q // mw - M_y)[None, :]
    j_ = kx[:, None] - (q % mw - M_x)[None, :]
    Z = X[(kt + N_t)[:, None], i_ + N_y + M_y, j_ + N_x + M_x]
    return kt, i_, j_, Z, X[kt + N_t, ky + N_y + M_y, kx + N_x + M_x]


def columns(X, N_x, N_y, N_t, M_x, M_y, sx, sy):
    """(re, im) float64 (rows, nc + 1) of [M | y] as darts_normal_kernel stages them: (s i) z with
    s = sy for the A columns and sx for the B columns, and kt z for y, each a correctly rounded
    product (no FMA)."""
    kt, i_, j_, Z, z = _entries(X, N_x, N_y, N_t, M_x, M_y)
    s = np.hstack([sy * i_.astype(np.float64), sx * j_.astype(np.float64)])
    Z = np.hstack([Z, Z])
    ktf = kt.astype(np.float64)
    re = np.hstack([s * Z.real, (ktf * z.real)[:, None]])
    im = np.hstack([s * Z.imag, (ktf * z.imag)[:, None]])
    return np.ascontiguousarray(re), np.ascontiguousarray(im)


def normal_restated(X, N_x, N_y, N_t, M_x, M_y, sx, sy, drop_last_partial=False, sel=None):
    """(MM, M^H y) complex128 as b200_darts_normal computes them, bit for bit: per block of 512 rows,
    re += u.re v.re + u.im v.im and im += u.re v.im - u.im v.re in row order from 0.0 (conj(u) v, no
    FMA); the block partials summed in block order; MM's lower triangle conj(upper).
    drop_last_partial: a mutation that leaves out the last block when it is partial.
    sel: compute only these pairs (indices into pairs(nc)) and return (c, d, value) instead."""
    re, im = columns(X, N_x, N_y, N_t, M_x, M_y, sx, sy)
    rows, ld = re.shape
    nc = ld - 1
    c, d = pairs(nc)
    if sel is not None:
        c, d = c[sel], d[sel]
    G = -(-rows // NORMAL_ROWS)
    pad = G * NORMAL_ROWS - rows
    # row r of every block, contiguous: (512, G, nc + 1)
    Br = np.vstack([re, np.zeros((pad, ld))]).reshape(G, NORMAL_ROWS, ld).transpose(1, 0, 2).copy()
    Bi = np.vstack([im, np.zeros((pad, ld))]).reshape(G, NORMAL_ROWS, ld).transpose(1, 0, 2).copy()
    pr = np.zeros((G, len(c)))
    pi = np.zeros((G, len(c)))
    last = rows - (G - 1) * NORMAL_ROWS  # rows of the last block
    for r in range(min(rows, NORMAL_ROWS)):
        k = G if r < last else G - 1  # the blocks that hold a row r
        ur, ui = Br[r, :k][:, c], Bi[r, :k][:, c]
        vr, vi = Br[r, :k][:, d], Bi[r, :k][:, d]
        pr[:k] = pr[:k] + (ur * vr + ui * vi)
        pi[:k] = pi[:k] + (ur * vi - ui * vr)
    if drop_last_partial and pad:
        G -= 1
    sr, si = np.zeros(len(c)), np.zeros(len(c))
    for g in range(G):
        sr = sr + pr[g]
        si = si + pi[g]
    if sel is not None:
        v = np.empty(len(c), dtype=np.complex128)
        v.real, v.imag = sr, si
        return c, d, v
    return _assemble(sr, si, c, d, nc)


def _assemble(sr, si, c, d, nc):
    MM = np.zeros((nc, nc), dtype=np.complex128)
    up = d < nc
    MM.real[c[up], d[up]], MM.imag[c[up], d[up]] = sr[up], si[up]
    lo = up & (c != d)
    MM.real[d[lo], c[lo]], MM.imag[d[lo], c[lo]] = sr[lo], -si[lo]
    Mhy = np.empty(nc, dtype=np.complex128)
    Mhy.real, Mhy.imag = sr[~up], si[~up]
    return MM, Mhy


def normal_gamma(rows):
    """Relative factor of the normal-equation bound: Re and Im of each entry of [M|y]^H [M|y] are
    each within normal_gamma * (|M|^T |M|) of the exact sum over the float64 block X.

      staging      each entry of M is (s i) z: two roundings, so |M - M_exact| <= 2u |M| per
                   component; conj(u) v then errs by 4u (|u.re v.re| + |u.im v.im|) in Re:  4
      the term     two products and one sum, each rounded once:                            2
      row sums     at most 511 additions per block after the first (exact) one:           511
      block sums   G - 1 additions after the first:                                      G - 1

    |u.re v.re| + |u.im v.im| <= |u| |v| (Cauchy-Schwarz), and Im alike, so with G blocks the
    count is 516 + G = 512 + G + 4.  The longdouble reference sums all rows in one sequential
    chain: rows * 2^-64 = rows * 2^-11 u more."""
    G = -(-rows // NORMAL_ROWS)
    return (NORMAL_ROWS + G + 4 + rows * 2.0 ** -11) * U * SLACK


def is_hermitian_bitwise(MM):
    """MM's strict lower triangle is conj of the upper bit for bit, and its diagonal's imaginary part
    is +0.0 (what darts_normal_final_kernel writes: conj(u) u has im = 0 exactly, never -0.0)"""
    lo = np.tril_indices(MM.shape[0], -1)
    low, up = MM[lo], MM[lo[1], lo[0]]
    return (np.array_equal(low.real.view(np.int64), up.real.view(np.int64))
            and np.array_equal(low.imag.view(np.int64), (-up.imag).view(np.int64))
            and not np.diagonal(MM).imag.view(np.int64).any())


def normal_exact(X, N_x, N_y, N_t, M_x, M_y, sx, sy):
    """-> (MMr, MMi, Mhyr, Mhyi, B_MM, B_Mhy): [M|y]^H [M|y] in longdouble from the exact staged
    entries (ld(s) * i) * ld(z), and the per-component bounds of normal_gamma"""
    kt, i_, j_, Z, z = _entries(X, N_x, N_y, N_t, M_x, M_y)
    sx_, sy_ = LD(sx), LD(sy)
    s = np.hstack([sy_ * i_.astype(LD), sx_ * j_.astype(LD)])
    Zr, Zi = _ld(np.hstack([Z.real, Z.real])), _ld(np.hstack([Z.imag, Z.imag]))
    Mr = np.hstack([s * Zr, (kt.astype(LD) * _ld(z.real))[:, None]])
    Mi = np.hstack([s * Zi, (kt.astype(LD) * _ld(z.imag))[:, None]])
    nc = Mr.shape[1] - 1
    Gr = Mr.T @ Mr + Mi.T @ Mi
    Gi = Mr.T @ Mi - Mi.T @ Mr
    A = np.abs(np.asarray(Mr, np.float64) + 1j * np.asarray(Mi, np.float64))
    B = normal_gamma(Mr.shape[0]) * (A.T @ A)
    return Gr[:nc, :nc], Gi[:nc, :nc], Gr[:nc, nc], Gi[:nc, nc], B[:nc, :nc], B[:nc, nc]


def normal_ratio(MM, Mhy, ex):
    """max over Re and Im of MM and M^H y of |got - exact| / bound, for normal_exact's ex"""
    MMr, MMi, Yr, Yi, BM, BY = ex
    MM, Mhy = np.asarray(MM), np.asarray(Mhy)
    return max(_ratio(abs(_ld(MM.real) - MMr), BM), _ratio(abs(_ld(MM.imag) - MMi), BM),
               _ratio(abs(_ld(Mhy.real) - Yr), BY), _ratio(abs(_ld(Mhy.imag) - Yi), BY))


# ---- synthesis ---------------------------------------------------------------------------------
def synth_gamma(h, w):
    """Relative factor of the synthesis bound: |out - Re(ey^T C ex) / (m n)| <= synth_gamma *
    (|ey|^T |C| |ex|) / (m n) per pixel.

      G = sum_a C ey   2h FMAs per component, each within 2h u sum_a |C| |ey| (Cauchy-Schwarz as
                       in normal_gamma); Re(G ex) reads G.re ex.re + G.im ex.im, so G's error
                       enters with |ex.re| + |ex.im| <= sqrt(2) |ex|: 2 sqrt(2) h < 3h       3h
      Re(G ex)         2w FMAs, within 2w u sum_b |G| |ex|:                                 2w
      scale            1 / (m n) rounded once (m n < 2^53 is exact), v * scale once:         2

    Each complex term costs two FMAs per component, hence 2h and 2w rather than h and w."""
    return (3 * h + 2 * w + 2) * U * SLACK


def synthesize(coef, ey, ex, m, n):
    """-> (out, B): (2, m, n) Re(ey^T C ex) / (m n) in longdouble and its bound"""
    eyr, eyi, exr, exi = _ld(ey.real), _ld(ey.imag), _ld(ex.real), _ld(ex.imag)
    out = np.empty((2, m, n), LD)
    B = np.empty((2, m, n))
    for k, C in enumerate(coef):
        Cr, Ci = _ld(C.real), _ld(C.imag)
        Gr = eyr.T @ Cr - eyi.T @ Ci
        Gi = eyr.T @ Ci + eyi.T @ Cr
        out[k] = (Gr @ exr - Gi @ exi) / (LD(m) * LD(n))
        B[k] = (np.abs(ey).T @ np.abs(C) @ np.abs(ex)) / (float(m) * float(n))
    return out, synth_gamma(coef.shape[1], coef.shape[2]) * B


# ---- the edge cases ----------------------------------------------------------------------------
def frames(T, m, n, seed, kind="rain", dtype=np.float64):
    """(T, m, n) frames: "rain" a translating rain field, "offset" 1e4 + rain, "spike" rain with
    frames[0, 0, 0] = -3e9, "noise" uniform in [0, 10) (for 1-pixel axes)"""
    from pysteps_b200 import _synthetic as syn
    if kind == "noise" or min(m, n) < 16:
        R = np.random.default_rng(seed).uniform(0.0, 10.0, (T, m, n))
    else:
        R = syn.rain_frames(m, n, T, seed=seed, dx=2, dy=-1)
    if kind == "offset":
        R = 1e4 + R
    elif kind == "spike":
        R = R.copy()
        R[0, 0, 0] = -3e9
    return R.astype(dtype)


# (name, T, m, n, N_x, N_y, N_t, M_x, M_y, frame kind, dtype)
SPECTRUM_CASES = [
    # fx = min(N_x + M_x, 128) + 1 across darts_rows_kernel's 64-wide frequency tiles
    ("fx64", 3, 40, 256, 61, 3, 1, 2, 2, "rain", np.float64),
    ("fx65", 3, 40, 256, 62, 3, 1, 2, 2, "rain", np.float32),
    ("fx66", 3, 40, 256, 63, 3, 1, 2, 2, "offset", np.float64),
    ("fx128", 3, 40, 256, 125, 3, 1, 2, 2, "spike", np.float64),
    ("fx129", 3, 40, 256, 126, 3, 1, 2, 2, "rain", np.float32),
    # 2w > n: conjugate reads, odd n and even n (which reads the Nyquist column)
    ("alias_odd101", 3, 24, 101, 68, 2, 1, 2, 1, "rain", np.float64),
    ("alias_even96", 3, 24, 96, 58, 2, 1, 2, 1, "offset", np.float32),
    # T m < 64 rows, m < 32, n = 9 < XK; 1-pixel axes
    ("small_20x9", 3, 20, 9, 3, 5, 1, 1, 2, "rain", np.float64),
    ("m1", 4, 1, 50, 10, 0, 1, 2, 0, "noise", np.float64),
    ("n1", 4, 30, 1, 0, 5, 1, 0, 2, "noise", np.float32),
    # time axis: K_t = 15 = 2 (T - 2) + 1 at T = 9, and T = 2 with N_t = 0
    ("t9_nt7", 9, 36, 40, 5, 4, 7, 1, 1, "rain", np.float64),
    ("t2_nt0", 2, 36, 40, 5, 4, 0, 1, 1, "spike", np.float32),
    # darts_cols_kernel tiles: K_y and K_x just either side of 16 and 32
    ("ky15_kx17", 3, 48, 64, 6, 5, 1, 2, 2, "rain", np.float64),
    ("ky17_kx15", 3, 48, 64, 5, 6, 1, 2, 2, "rain", np.float64),
    ("ky31_kx33", 3, 48, 64, 14, 13, 1, 2, 2, "offset", np.float64),
    ("ky33_kx31", 3, 48, 64, 13, 14, 1, 2, 2, "rain", np.float32),
]

# (name, N_x, N_y, N_t, M_x, M_y): normal equations on random blocks
NORMAL_CASES = [
    ("m00", 3, 2, 1, 0, 0),
    ("m55", 3, 2, 1, 5, 5),
    ("m50", 3, 2, 1, 5, 0),
    ("m05", 3, 2, 1, 0, 5),
    ("m31", 3, 2, 1, 3, 1),
    ("rows1_m55", 0, 0, 0, 5, 5),
    ("rows1_m00", 0, 0, 0, 0, 0),
    ("rows27_m55", 1, 1, 1, 5, 5),
    ("rows511_m55", 255, 0, 0, 5, 5),
    ("rows513_m55", 256, 0, 0, 5, 5),
    ("rows513_m21", 256, 0, 0, 2, 1),
]


def random_block(N_x, N_y, N_t, M_x, M_y, seed):
    """a (2N_t+1, 2(N_y+M_y)+1, 2(N_x+M_x)+1) complex block whose parts span 2^-30 .. 2^30 with random
    signs, so that any change of summation order shows in the result"""
    rng = np.random.default_rng(seed)
    shape = (2 * N_t + 1, 2 * (N_y + M_y) + 1, 2 * (N_x + M_x) + 1)

    def part():
        return rng.choice([-1.0, 1.0], shape) * np.exp2(rng.uniform(-30.0, 30.0, shape))

    return part() + 1j * part()


def normal_scales(T, m, n):
    """(sx, sy) = (c1 / T_x, c1 / T_y), c1 = -T_t / (T_x T_y), as DARTS passes them"""
    c1 = -1.0 * T / (n * m)
    return c1 / n, c1 / m


# (h, w, m, n): the synthesis shapes
SYNTH_CASES = [(1, 1, 1, 1), (11, 11, 11, 11), (5, 121, 64, 300), (5, 3, 5, 1000), (121, 7, 130, 40)]


def random_synthesis(h, w, m, n, seed):
    """(coef (2, h, w), ey (h, m), ex (w, n)) complex, random"""
    rng = np.random.default_rng(seed)

    def c(*shape):
        return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)

    return c(2, h, w), c(h, m), c(w, n)
