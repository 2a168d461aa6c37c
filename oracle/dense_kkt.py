"""Dense reference for one KKT solve (TEST INFRASTRUCTURE ONLY).

The full system of the interior-point step (batch.py:349-372) and of the regularised variant (batch.py:228-310),

    [Q + r I   0        G'     A'  ] [dx]     [rx]
    [0         D + r I  I      0   ] [ds]  = -[rs]
    [G         I        -r I   0   ] [dz]     [rz]
    [A         0        0      -r I] [dy]     [ry]

assembled densely and solved by LU in fp64, then refined with residuals accumulated in np.longdouble. No block
elimination, no Cholesky and no whitening: nothing of the kernels' formulation, so it can judge them. With d spread
over 16 decades the refined solution has a normwise backward error at the level of the longdouble residual.
"""
import numpy as np
import scipy.linalg as sla


def kkt_matrix(Q, G, A, d, reg=0.0):
    n, m = Q.shape[0], G.shape[0]
    e = 0 if A is None else A.shape[0]
    N = n + 2 * m + e
    K = np.zeros((N, N))
    K[:n, :n] = Q + reg * np.eye(n)
    K[:n, n + m:n + 2 * m] = G.T
    K[n:n + m, n:n + m] = np.diag(d + reg)
    K[n:n + m, n + m:n + 2 * m] = np.eye(m)
    K[n + m:n + 2 * m, :n] = G
    K[n + m:n + 2 * m, n:n + m] = np.eye(m)
    K[n + m:n + 2 * m, n + m:n + 2 * m] = -reg * np.eye(m)
    if e > 0:
        K[:n, n + 2 * m:] = A.T
        K[n + 2 * m:, :n] = A
        K[n + 2 * m:, n + 2 * m:] = -reg * np.eye(e)
    return K


def _resid_ld(K, u, rhs):
    """rhs - K u with every product and sum in np.longdouble."""
    return np.asarray(rhs, dtype=np.longdouble) - np.asarray(K, dtype=np.longdouble) @ np.asarray(u, dtype=np.longdouble)


def solve_refined(K, rhs, steps=4):
    lu = sla.lu_factor(K, check_finite=False)
    u = sla.lu_solve(lu, rhs, check_finite=False)
    for _ in range(steps):
        u = u + sla.lu_solve(lu, _resid_ld(K, u, rhs).astype(np.float64), check_finite=False)
    return u


def backward_error(K, u, rhs):
    """Normwise backward error  ||rhs - K u||_inf / (||K||_inf ||u||_inf + ||rhs||_inf)."""
    r = np.abs(_resid_ld(K, u, rhs)).max()
    return float(r / (np.abs(K).sum(1).max() * np.abs(u).max() + np.abs(rhs).max()))


def split(u, n, m, e):
    return u[:n], u[n:n + m], u[n + m:n + 2 * m], (u[n + 2 * m:] if e > 0 else None)


def solve(Q, G, A, d, rx, rs, rz, ry, reg=0.0):
    """(dx, ds, dz, dy, K, rhs) of one system; dy is None without equality constraints."""
    n, m = Q.shape[0], G.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    K = kkt_matrix(Q, G, A if e else None, d, reg)
    rhs = -np.concatenate([rx, rs, rz] + ([ry] if e else []))
    return split(solve_refined(K, rhs), n, m, e) + (K, rhs)


def rel(a, b):
    """||a - b|| / ||b|| (0 for two empty vectors)."""
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    if b.size == 0:
        return 0.0
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
