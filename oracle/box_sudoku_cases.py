"""The 9x9 OptNet sudoku layer as box QPs (TEST INFRASTRUCTURE ONLY): the reduced constraint matrix, seeded puzzles and
the two cases `oracle/gen_golden_box_sudoku.py` runs through the real reference.

The constraints of a board with n^2 x n^2 cells and n^2 digits are one-hot equalities over the n^6 indicator variables
z[(row * n^2 + col) * n^2 + digit]: every cell holds one digit, and every row, column and box holds every digit once.
Of the 4 n^4 rows only some are independent; `sudoku_matrix` keeps them greedily in that order while the rank grows,
which gives 249 x 729 for n = 3 (and 40 x 64 for n = 2, the shape of OptNet's 4x4 experiment)."""
import numpy as np


def sudoku_constraints(n=3):
    """All 4 n^4 one-hot constraint rows: cells, then rows, columns and boxes (each by digit)."""
    N = n * n
    idx = np.arange(N ** 3).reshape(N, N, N)                # [row, col, digit]
    rows = []
    for r in range(N):
        for c in range(N):
            rows.append(idx[r, c, :])
    for r in range(N):
        for d in range(N):
            rows.append(idx[r, :, d])
    for c in range(N):
        for d in range(N):
            rows.append(idx[:, c, d])
    for br in range(n):
        for bc in range(n):
            for d in range(N):
                rows.append(idx[br * n:(br + 1) * n, bc * n:(bc + 1) * n, d].ravel())
    A = np.zeros((len(rows), N ** 3))
    for i, cols in enumerate(rows):
        A[i, cols] = 1.0
    return A


def sudoku_matrix(n=3):
    """The constraint rows kept in order while the rank grows (full row rank)."""
    A = sudoku_constraints(n)
    basis, keep = [], []
    for i, a in enumerate(A):
        v = a.copy()
        for u in basis:                                      # Gram-Schmidt twice: exact enough for 0/1 rows
            v -= (u @ v) * u
        for u in basis:
            v -= (u @ v) * u
        nv = np.linalg.norm(v)
        if nv > 1e-8:
            basis.append(v / nv)
            keep.append(i)
    return A[keep]


def solved_grid(rs, n=3):
    """The standard pattern with seeded digit, band and in-band row permutations."""
    N = n * n
    g = np.array([[(n * (r % n) + r // n + c) % N for c in range(N)] for r in range(N)])
    bands = rs.permutation(n)
    order = np.concatenate([b * n + rs.permutation(n) for b in bands])
    return rs.permutation(N)[g[order]]


def puzzles(seed, B, n=3, blanks=0.6):
    """B puzzles: one-hot boards (B, n^6) with a seeded fraction of the cells blank, and their solutions."""
    rs = np.random.RandomState(seed)
    N = n * n
    P, Z = np.zeros((B, N ** 3)), np.zeros((B, N ** 3))
    for b in range(B):
        g = solved_grid(rs, n)
        hole = rs.rand(N, N) < blanks
        for r in range(N):
            for c in range(N):
                Z[b, (r * N + c) * N + g[r, c]] = 1.0
                if not hole[r, c]:
                    P[b, (r * N + c) * N + g[r, c]] = 1.0
    return P, Z


def sudoku9_problem():
    """The OptNet sudoku layer at its trained point: p = -puzzle, q = 0.1, z >= 0, A z = 1 with A shared."""
    A = sudoku_matrix(3)
    P, _ = puzzles(91, B=3)
    rs = np.random.RandomState(92)
    n = A.shape[1]
    return dict(q=np.full(n, 0.1), p=-P, A=A, b=np.ones(A.shape[0]), lb=np.zeros(n), ub=None, dl=rs.randn(3, n))


def sudoku9_init_problem():
    """OptNet's initialisation of the layer: A = rand(249, 729) shared, b = A z0 for a z0 > 0 (so feasible)."""
    rs = np.random.RandomState(93)
    m, n = sudoku_matrix(3).shape
    A = rs.rand(m, n)
    z0 = 0.1 + rs.rand(n)
    P, _ = puzzles(94, B=2)
    return dict(q=np.full(n, 0.1), p=-P, A=A, b=A @ z0, lb=np.zeros(n), ub=None, dl=rs.randn(2, n))


SUDOKU_BOX_CASES = {
    "box_sudoku9": sudoku9_problem,
    "box_sudoku9_init": sudoku9_init_problem,
}
