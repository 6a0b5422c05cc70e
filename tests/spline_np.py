"""NumPy mirror of the device's imported-trajectory spline (ratinabox_b200/csrc/riab_traj.cuh): the host elimination
factors, the per-column forward sweep / back substitution (riab_trajectory_build) and the evaluation at a time.  Every
step is the same IEEE float64 operation in the same order as the device's, so M equals the device's bit for bit."""
import numpy as np


def factors(x):
    """traj_factors: w (forward multipliers), bp (eliminated diagonal), c (super-diagonal), h (spacings)."""
    x = np.asarray(x, dtype=np.float64)
    T = len(x)
    m = T - 2
    h = x[1:] - x[:-1]
    a = h[:m].copy()
    bp = 2.0 * (h[:m] + h[1:m + 1])
    c = h[1:m + 1].copy()
    h0, h1, hm1, hm2 = h[0], h[1], h[T - 2], h[T - 3]
    bp[0] = (h0 + h1) * (h0 + 2.0 * h1) / h1
    c[0] = (h1 * h1 - h0 * h0) / h1
    a[0] = 0.0
    bp[m - 1] = (hm1 + hm2) * (hm1 + 2.0 * hm2) / hm2
    a[m - 1] = (hm2 * hm2 - hm1 * hm1) / hm2
    c[m - 1] = 0.0
    w = np.zeros(m)
    for j in range(1, m):
        w[j] = a[j] / bp[j - 1]
        bp[j] = bp[j] - w[j] * c[j - 1]
    return w, bp, c, h


def build(x, y):
    """k_traj_build over every column: y (T, ...) -> M (T, ...)."""
    y = np.asarray(y, dtype=np.float64)
    T = y.shape[0]
    m = T - 2
    w, bp, c, h = factors(x)
    M = np.empty_like(y)
    d0 = (y[1] - y[0]) / h[0]
    y1 = y[1]
    r = None
    for j in range(m):
        y2 = y[j + 2]
        d1 = (y2 - y1) / h[j + 1]
        rj = 6.0 * (d1 - d0)
        r = rj if j == 0 else rj - w[j] * r
        M[j + 1] = r
        y1, d0 = y2, d1
    mn = M[m] / bp[m - 1]
    M[m] = mn
    mnn = None
    for j in range(m - 2, -1, -1):
        mnn = mn
        mn = (M[j + 1] - c[j] * mnn) / bp[j]
        M[j + 1] = mn
    M[0] = ((h[0] + h[1]) * mn - h[0] * mnn) / h[1]
    M[T - 1] = ((h[T - 2] + h[T - 3]) * M[m] - h[T - 2] * M[m - 1]) / h[T - 3]
    return M


def segment(x, q):
    """traj_segment: times[k] <= q < times[k+1], clipped to [0, T-2]."""
    return np.clip(np.searchsorted(x, q, side="right") - 1, 0, len(x) - 2)


def evaluate(x, y, M, q):
    """traj_eval at the times q (any shape) -> (*q.shape, *y.shape[1:])."""
    x = np.asarray(x, dtype=np.float64)
    q = np.asarray(q, dtype=np.float64)
    k = segment(x, q)
    ex = (Ellipsis,) + (None,) * (y.ndim - 1)
    x0, x1 = x[k][ex], x[k + 1][ex]
    qq = q[ex]
    h = x1 - x0
    A = x1 - qq
    B = qq - x0
    A3, B3, h6 = A * A * A, B * B * B, 6.0 * h
    M0, M1, y0, y1 = M[k], M[k + 1], y[k], y[k + 1]
    return M0 * A3 / h6 + M1 * B3 / h6 + (y0 / h - M0 * h / 6.0) * A + (y1 / h - M1 * h / 6.0) * B
