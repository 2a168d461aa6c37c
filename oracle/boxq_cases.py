"""Golden-case recipes of the dense-Q box path (BoxQPFunction(dense_Q=True)), shared by `oracle/gen_golden_boxq.py` and
`tests/` (TEST INFRASTRUCTURE ONLY). Every case is a box QP with a dense Q (Q, p, A, b, lb, ub, dl; lb or ub None for
an absent side) whose dense equivalent (`dense_problem`) the real reference solves; the fixtures tests/golden/boxq_*.npz
hold the reference's outputs for it."""
import numpy as np


def _spd(rs, n, B=None, cond_decades=2.0, ridge=1e-2, top=0.0):
    """Random SPD matrices (B, n, n), or one (n, n) when B is None: eigenvalues 10^(top - U(0, cond_decades)) + ridge."""
    def one():
        U, _ = np.linalg.qr(rs.randn(n, n))
        ev = 10.0 ** (top - cond_decades * rs.rand(n)) + ridge
        Q = (U * ev) @ U.T
        return 0.5 * (Q + Q.T)
    return one() if B is None else np.stack([one() for _ in range(B)])


def _feasible_b(rs, A, lo, hi, B, n):
    z0 = lo + (hi - lo) * (0.1 + 0.8 * rs.rand(B, n))
    return np.einsum("en,bn->be", A, z0) if A.ndim == 2 else np.einsum("ben,bn->be", A, z0)


def portfolio_problem():
    """long-only portfolio: covariance Q (batched), 0 <= w <= 1, 1'w = 1."""
    rs = np.random.RandomState(61)
    B, n = 8, 30
    F = rs.randn(B, n, 5)
    Q = np.einsum("bik,bjk->bij", F, F) / 5.0 + np.stack([np.diag(0.05 + 0.1 * rs.rand(n)) for _ in range(B)])
    return dict(Q=Q, p=-0.1 * rs.randn(B, n), A=np.ones((1, n)), b=np.ones(1), lb=np.zeros(n), ub=np.ones(n),
                dl=rs.randn(B, n))


def mpc_problem():
    """condensed MPC: one shared Q, batched p (initial states), input bounds on both sides, no equalities."""
    rs = np.random.RandomState(62)
    B, n = 10, 24
    Q = _spd(rs, n, cond_decades=2.0, ridge=0.05)
    return dict(Q=Q, p=3.0 * rs.randn(B, n), A=np.zeros((0,)), b=np.zeros((0,)), lb=-np.ones(n), ub=np.ones(n),
                dl=rs.randn(B, n))


def ub_odd_problem():
    """upper bounds only, odd nz, neq not a multiple of 8, batched Q and A."""
    rs = np.random.RandomState(63)
    B, n, e = 5, 33, 5
    Q = _spd(rs, n, B, cond_decades=1.5, ridge=0.1)
    ub = 0.5 + rs.rand(B, n)
    A = rs.randn(B, e, n)
    b = _feasible_b(rs, A, ub - 2.0, ub, B, n)
    return dict(Q=Q, p=rs.randn(B, n), A=A, b=b, lb=None, ub=ub, dl=rs.randn(B, n))


def shared_q_problem():
    """one Q shared by the batch, lower bounds only, batched A / b / lb."""
    rs = np.random.RandomState(64)
    B, n, e = 6, 20, 4
    Q = _spd(rs, n, cond_decades=1.0, ridge=0.2)
    lb = -rs.rand(B, n)
    A = rs.randn(B, e, n)
    b = _feasible_b(rs, A, lb, lb + 1.0, B, n)
    return dict(Q=Q, p=2.0 * rs.randn(B, n), A=A, b=b, lb=lb, ub=None, dl=rs.randn(B, n))


def spread_problem():
    """Q with eigenvalues over 6 decades (1e-3 .. 1e3), both bounds, a shared A."""
    rs = np.random.RandomState(65)
    B, n, e = 4, 24, 3
    Q = _spd(rs, n, B, cond_decades=6.0, ridge=0.0, top=3.0)
    A = rs.randn(e, n)
    b = _feasible_b(rs, A, np.zeros(n), np.ones(n), B, n)
    return dict(Q=Q, p=30.0 * rs.randn(B, n), A=A, b=b, lb=np.zeros(n), ub=np.ones(n), dl=rs.randn(B, n))


def dense_problem(bx):
    """The dense equivalent QPFunction (and the reference) solves: Q as given, G = [-I; I] (sides given),
    h = [-lb; ub]. Batched inputs stay batched, shared ones shared."""
    Q = np.asarray(bx["Q"], dtype=np.float64)
    n = Q.shape[-1]
    G, h = [], []
    if bx["lb"] is not None:
        G.append(-np.eye(n)); h.append(-np.asarray(bx["lb"], dtype=np.float64))
    if bx["ub"] is not None:
        G.append(np.eye(n)); h.append(np.asarray(bx["ub"], dtype=np.float64))
    if any(v.ndim == 2 for v in h):
        B = next(v.shape[0] for v in h if v.ndim == 2)
        h = [v if v.ndim == 2 else np.tile(v, (B, 1)) for v in h]
    A = np.asarray(bx["A"], dtype=np.float64)
    has_eq = A.ndim >= 2 and A.shape[-2] > 0
    return dict(Q=Q, p=bx["p"], G=np.concatenate(G), h=np.concatenate(h, -1), A=A if has_eq else np.zeros((0,)),
                b=bx["b"] if has_eq else np.zeros((0,)), dl=bx["dl"])


# name -> builder (fixtures tests/golden/<name>.npz)
BOXQ_CASES = {
    "boxq_portfolio": portfolio_problem,
    "boxq_mpc": mpc_problem,
    "boxq_ub_odd": ub_odd_problem,
    "boxq_shared_q": shared_q_problem,
    "boxq_spread": spread_problem,
}


def map_dense_grads(g, bx):
    """QPFunction / reference gradients (dQ, dp, dG, dh, dA, db) -> dict(dQ, dp, dA, db, dlb, dub)."""
    dQ, dp, _, dh, dA, db = g
    n = np.asarray(bx["Q"]).shape[-1]
    nlb = n if bx["lb"] is not None else 0
    return dict(dQ=dQ, dp=dp, dA=dA, db=db,
                dlb=None if bx["lb"] is None else -dh[..., :nlb], dub=None if bx["ub"] is None else dh[..., nlb:])
