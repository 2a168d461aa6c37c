"""Seeded problems for the regularised mode (QPFunction kkt_solver=IR_UNOPT): Q only positive semidefinite, or linearly
dependent equality rows. Each returns numpy (Q, p, G, h, A, b), every problem feasible with a bounded optimum."""
import numpy as np


def lp(seed, nz=50, nrand=70, neq=10):
    """LP (Q = 0): `nrand` random rows plus both bounds around an interior point."""
    r = np.random.RandomState(seed)
    G = np.vstack([r.randn(nrand, nz), -np.eye(nz), np.eye(nz)])
    z0 = r.rand(nz)
    h = G @ z0 + r.rand(G.shape[0])
    A = r.randn(neq, nz)
    return np.zeros((nz, nz)), r.randn(nz), G, h, A, A @ z0


def lowrank(seed, nz=60, nrand=40, rank=5, neq=5):
    """Q = F F' of rank `rank` (a sample covariance with fewer samples than assets), both bounds."""
    r = np.random.RandomState(seed)
    F = r.randn(nz, rank)
    G = np.vstack([r.randn(nrand, nz), -np.eye(nz), np.eye(nz)])
    z0 = r.rand(nz)
    h = G @ z0 + r.rand(G.shape[0])
    A = r.randn(neq, nz)
    return F @ F.T, r.randn(nz), G, h, A, A @ z0


def sudoku4_full_A():
    """The full 64-row constraint matrix of the 4x4 sudoku (cells, rows, columns, boxes; rank 40)."""
    n = 4
    idx = lambda i, j, k: (i * n + j) * n + k  # noqa: E731
    rows = [[idx(i, j, k) for k in range(n)] for i in range(n) for j in range(n)]
    rows += [[idx(i, j, k) for j in range(n)] for i in range(n) for k in range(n)]
    rows += [[idx(i, j, k) for i in range(n)] for j in range(n) for k in range(n)]
    rows += [[idx(2 * bi + a, 2 * bj + c, k) for a in range(2) for c in range(2)]
             for bi in range(2) for bj in range(2) for k in range(n)]
    A = np.zeros((len(rows), n ** 3))
    for i, cols in enumerate(rows):
        A[i, cols] = 1.0
    return A


def sudoku4(seed):
    """The OptNet sudoku layer (Q = 0.1 I, z >= 0, the full A z = 1) with a random linear term."""
    r = np.random.RandomState(seed)
    A = sudoku4_full_A()
    return 0.1 * np.eye(64), -r.rand(64), -np.eye(64), np.zeros(64), A, np.ones(A.shape[0])


def spd(seed, nz=40, nineq=30, neq=6):
    """An SPD control case."""
    r = np.random.RandomState(seed)
    M = r.randn(nz, nz)
    G = r.randn(nineq, nz)
    z0 = r.randn(nz)
    A = r.randn(neq, nz)
    return M @ M.T + np.eye(nz), r.randn(nz), G, G @ z0 + r.rand(nineq), A, A @ z0


def large(seed, nz=100, nrand=0):
    """Order ms_pad = 200 with nz = 100: W and chol(Q) do not fit next to the factor (the L2-resident build)."""
    r = np.random.RandomState(seed)
    F = r.randn(nz, 5)
    G = np.vstack([r.randn(nrand, nz), -np.eye(nz), np.eye(nz)])
    z0 = r.rand(nz)
    return F @ F.T, r.randn(nz), G, G @ z0 + r.rand(G.shape[0]), np.zeros((0, nz)), np.zeros(0)


def kkt_residuals(Q, p, G, h, A, b, x, z, s, y):
    """max-norm stationarity, primal inequality, primal equality residuals and |z's| of a returned point."""
    rx = Q @ x + p + G.T @ z + (A.T @ y if A.shape[0] else 0.0)
    return (np.abs(rx).max(), np.abs(G @ x + s - h).max(), np.abs(A @ x - b).max() if A.shape[0] else 0.0,
            abs(z @ s))


def dense_grads(Q, G, A, x, z, s, y, dl):
    """Gradients of dl'z* by implicit differentiation of the true KKT system at (x, z, s, y) with qpth's d =
    max(z, 1e-8) / max(s, 1e-8) (qp.py:148), least-squares solved so that linearly dependent equality rows (a singular
    KKT matrix, dy not unique) still give the unique dx and dz."""
    n, m, e = Q.shape[0], G.shape[0], A.shape[0]
    d = np.maximum(z, 1e-8) / np.maximum(s, 1e-8)
    N = n + 2 * m + e
    K = np.zeros((N, N))
    K[:n, :n] = Q; K[:n, n + m:n + 2 * m] = G.T; K[:n, n + 2 * m:] = A.T
    K[n:n + m, n:n + m] = np.diag(d); K[n:n + m, n + m:n + 2 * m] = np.eye(m)
    K[n + m:n + 2 * m, :n] = G; K[n + m:n + 2 * m, n:n + m] = np.eye(m)
    K[n + 2 * m:, :n] = A
    u = np.linalg.lstsq(K, -np.concatenate([dl, np.zeros(2 * m + e)]), rcond=None)[0]
    dx, dz = u[:n], u[n + m:n + 2 * m]
    return dict(dQ=0.5 * (np.outer(dx, x) + np.outer(x, dx)), dp=dx, dG=np.outer(dz, x) + np.outer(z, dx), dh=-dz)
