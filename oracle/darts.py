"""CPU oracle of the DARTS motion method (pysteps/motion/darts.py:22-220): a NumPy restatement of what
csrc/darts.cu computes, on the same twiddle tables (pysteps_b200.motion.darts.twiddles):

  * spectrum: the direct DFT of the frames less frames[0, 0, 0] at the block of NumPy indices the
    reference reads -- x (frequencies 0 .. min(K, n // 2), conjugated for the rest), then t, then y
  * normal: M built whole (the device never forms it), MM = M^H M and M^H y
  * solve: the reference's, from the Gram matrix (pysteps_b200.motion.darts.solve)
  * synthesize: Re(ey^T coef ex) / (m n), the separable inverse DFT of _fill's placement
"""
import numpy as np

from pysteps_b200.motion import darts as _d


def spectrum_from_tables(frames, tw_x, tw_y, tw_t, K):
    """(Kt, Ky, 2K+1) complex128 block of b200_darts_spectrum"""
    T, m, n = frames.shape
    rows = frames.reshape(T * m, n).astype(np.float64)
    if rows.size:
        rows = rows - rows[0, 0]
    P = (rows @ tw_x.real.T) + 1j * (rows @ tw_x.imag.T)
    w = np.arange(-K, K + 1) % n
    cj = 2 * w > n
    f = np.where(cj, n - w, w)
    Px = P.reshape(T, m, -1)[:, :, f]
    Px[:, :, cj] = np.conj(Px[:, :, cj])
    Q = np.tensordot(tw_t, Px, axes=(1, 0))  # (Kt, m, Kx)
    return np.matmul(tw_y[None], Q)


def spectrum(frames, N_x=50, N_y=50, N_t=4, M_x=2, M_y=2):
    T, m, n = frames.shape
    tw_x, tw_y, tw_t, K = _d.spectrum_tables(T, m, n, N_x, N_y, N_t, M_x, M_y)
    return spectrum_from_tables(frames, tw_x, tw_y, tw_t, K)


def normal(X, N_x, N_y, N_t, M_x, M_y, sx, sy):
    """(MM, M^H y) from the block X (Kt, Ky, Kx); rows of M in the reference's (k_t, k_y, k_x) order"""
    kt, ky, kx = (a.ravel() for a in np.meshgrid(np.arange(-N_t, N_t + 1), np.arange(-N_y, N_y + 1),
                                                 np.arange(-N_x, N_x + 1), indexing="ij"))
    mw = 2 * M_x + 1
    q = np.arange((2 * M_y + 1) * mw)
    kpy, kpx = q // mw - M_y, q % mw - M_x
    i_ = ky[:, None] - kpy[None, :]
    j_ = kx[:, None] - kpx[None, :]
    R_ = X[(kt + N_t)[:, None], i_ + N_y + M_y, j_ + N_x + M_x]
    M = np.hstack([(sy * i_) * R_, (sx * j_) * R_])
    y = kt * X[kt + N_t, ky + N_y + M_y, kx + N_x + M_x]
    M_ct = M.conjugate().T
    return M_ct @ M, M_ct @ y


def synthesize(coef, ey, ex, m, n):
    """(2, m, n) float64 from coef (2, h, w) and the tables ey (h, m), ex (w, n)"""
    return np.stack([np.real(ey.T @ c @ ex) for c in coef]) * (1.0 / (float(m) * float(n)))


def DARTS(R, N_x=50, N_y=50, N_t=4, M_x=2, M_y=2, output_type="spatial", lsq_method=2, **_):
    """The whole method for valid arguments -> (field or spectral stack, intermediates dict)"""
    R = np.asarray(np.ma.getdata(R))
    T, m, n = R.shape
    X = spectrum(R, N_x, N_y, N_t, M_x, M_y)
    c1 = -1.0 * T / (n * m)
    MM, Mhy = normal(X, N_x, N_y, N_t, M_x, M_y, c1 / n, c1 / m)
    x = _d.solve(MM, Mhy, lsq_method)
    h, w = 2 * M_y + 1, 2 * M_x + 1
    V, U = x[: h * w].reshape(h, w), x[h * w:].reshape(h, w)
    inter = {"spectrum": X, "MM": MM, "Mhy": Mhy, "x": x}
    if output_type != "spatial":
        return np.stack([U, V]), inter
    rows, cols, ri, ci = _d.fill_tables(M_x, M_y, m, n)
    coef = np.zeros((2, len(rows), len(cols)), dtype=complex)
    coef[0][ri, ci] = U
    coef[1][ri, ci] = V
    return synthesize(coef, _d.twiddles(tuple(rows), m, 1), _d.twiddles(tuple(cols), n, 1), m, n), inter
