"""Seeded problems for the regularised mode (QPFunction kkt_solver=IR_UNOPT) at orders ms_pad = 8 ceil(neq / 8) + nineq
(rounded up to 8) that the product-form kernels do not take: the generic global-scratch kernels run them. Each returns
numpy (Q, p, G, h, A, b), every problem feasible with a bounded optimum."""
import numpy as np

from . import psd_cases as pc
from .box_sudoku_cases import sudoku_matrix


def lp280(seed):
    """The LP of psd_cases.lp at nz = 100: both bounds, 60 random rows, neq = 10 (order 280)."""
    return pc.lp(seed, nz=100, nrand=60, neq=10)


def lowrank120(seed):
    """A rank-8 Q at nz = 120 with both bounds and 5 equality rows (order 248)."""
    return pc.lowrank(seed, nz=120, nrand=0, rank=8, neq=5)


def lp232(seed):
    """An LP of order 232: inside the product-form kernels' 256 rows, but too large for their shared memory."""
    return pc.lp(seed, nz=60, nrand=100, neq=8)


def lp664(seed):
    """An LP at nz = 300: both bounds, 52 random rows, neq = 8 (order 664)."""
    return pc.lp(seed, nz=300, nrand=52, neq=8)


def lp_dependent(seed):
    """The LP of lp280 with 0/1 equality rows (an assignment-style A, 10 of 100 columns per row on average) whose last
    three rows are sums of the first seven (rank 7), b consistent. (With Q = 0 the equality block of the regularised
    factor is A A' / eps + eps I: rows of dense O(1) entries over 100 columns make A A' / eps so large that the eps of
    the dependent rows falls below its rounding, and the factorization breaks down.)"""
    Q, p, G, h, _, _ = lp280(seed)
    rs = np.random.RandomState(seed)                         # psd_cases.lp's interior point: its first draws replayed
    rs.randn(60, 100)
    z0 = rs.rand(100)
    A = (np.random.RandomState(1000 + seed).rand(10, 100) < 0.1).astype(float)
    A[7], A[8], A[9] = A[0] + A[1], A[2] + A[3], A[4] + A[5] + A[6]
    return Q, p, G, h, A, A @ z0


def sudoku9_lp(seed, B=1):
    """The 9x9 sudoku LP relaxation: Q = 0, z >= 0 and the 249 independent rows of the sudoku constraints = 1, with a
    random linear term (order 992). Returns B problems."""
    A = sudoku_matrix(3)
    n = A.shape[1]
    r = np.random.RandomState(seed)
    return [(np.zeros((n, n)), r.randn(n), -np.eye(n), np.zeros(n), A, np.ones(A.shape[0])) for _ in range(B)]
