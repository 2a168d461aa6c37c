"""Golden-case recipes of the box-QP path (BoxQPFunction), shared by `oracle/gen_golden_box.py` and `tests/`
(TEST INFRASTRUCTURE ONLY). Every case is a box QP (q, p, A, b, lb, ub, dl; lb or ub None for an absent side) whose
dense equivalent (`dense_problem`) the real reference solves; the fixtures hold the reference's outputs for it.
Kept apart from `oracle.cases.CASES` so that the dense path's golden parametrisations do not change."""
import numpy as np

from oracle.cases import sudoku_structured_problem


def _box(seed, B, n, e, lb, ub, q=None, shared_A=False):
    rs = np.random.RandomState(seed)
    lo = np.zeros(n) if lb is None else lb
    hi = np.ones(n) if ub is None else ub
    z0 = lo + (hi - lo) * (0.1 + 0.8 * rs.rand(B, n))                 # strictly inside the box
    A = rs.randn(e, n) if shared_A else rs.randn(B, e, n)
    b = z0 @ A.T if shared_A else np.einsum("ben,bn->be", A, z0)
    qq = np.ones(n) if q is None else q
    return dict(q=qq, p=rs.randn(B, n) * 2.0, A=A, b=b, lb=None if lb is None else np.asarray(lb, dtype=np.float64),
                ub=None if ub is None else np.asarray(ub, dtype=np.float64), dl=rs.randn(B, n))


def projection_problem():
    """min 1/2 ||z - v||^2 s.t. Az = b, 0 <= z <= 1 (Q = I, p = -v), batched A."""
    return _box(41, B=6, n=30, e=6, lb=np.zeros(30), ub=np.ones(30))


def ub_only_problem():
    rs = np.random.RandomState(42)
    return _box(42, B=5, n=20, e=5, lb=None, ub=1.0 + rs.rand(20), q=0.5 + rs.rand(20), shared_A=True)


def noeq_problem():
    rs = np.random.RandomState(43)
    return _box(43, B=6, n=25, e=0, lb=-rs.rand(25), ub=rs.rand(25), q=0.2 + rs.rand(25))


def odd_problem():
    """odd nz, neq not a multiple of 8, lb only"""
    rs = np.random.RandomState(44)
    return _box(44, B=4, n=37, e=13, lb=rs.randn(37), ub=None, q=0.1 + rs.rand(37))


def sudoku_box():
    """golden case `sudoku_structured` (oracle/cases.py) in box form: q = 0.1, lb = 0."""
    pr = sudoku_structured_problem()
    n = pr["Q"].shape[0]
    return dict(q=np.diag(pr["Q"]).copy(), p=pr["p"], A=pr["A"], b=pr["b"], lb=np.zeros(n), ub=None, dl=pr["dl"])


def dense_problem(bx):
    """The dense equivalent QPFunction (and the reference) solves: Q = diag(q), G = [-I; I] (sides given), h = [-lb; ub].
    Batched inputs stay batched, shared ones shared."""
    q = np.asarray(bx["q"], dtype=np.float64)
    n = q.shape[-1]
    Q = np.stack([np.diag(v) for v in q]) if q.ndim == 2 else np.diag(q)
    G, h = [], []
    if bx["lb"] is not None:
        G.append(-np.eye(n)); h.append(-np.asarray(bx["lb"], dtype=np.float64))
    if bx["ub"] is not None:
        G.append(np.eye(n)); h.append(np.asarray(bx["ub"], dtype=np.float64))
    if any(v.ndim == 2 for v in h):
        B = next(v.shape[0] for v in h if v.ndim == 2)
        h = [v if v.ndim == 2 else np.tile(v, (B, 1)) for v in h]
    A = np.asarray(bx["A"], dtype=np.float64)
    return dict(Q=Q, p=bx["p"], G=np.concatenate(G), h=np.concatenate(h, -1),
                A=A if A.shape[-2] > 0 else np.zeros((0,)), b=bx["b"] if A.shape[-2] > 0 else np.zeros((0,)), dl=bx["dl"])


# name -> builder (fixtures tests/golden/<name>.npz; "sudoku_structured" is the dense path's own fixture)
BOX_CASES = {
    "sudoku_structured": sudoku_box,
    "box_projection": projection_problem,
    "box_ub_only": ub_only_problem,
    "box_noeq": noeq_problem,
    "box_odd": odd_problem,
}


def map_dense_grads(g, bx):
    """QPFunction / reference gradients (dQ, dp, dG, dh, dA, db) -> box gradients dict(dq, dp, dA, db, dlb, dub)."""
    dQ, dp, _, dh, dA, db = g
    n = np.asarray(bx["q"]).shape[-1]
    nlb = n if bx["lb"] is not None else 0
    return dict(dq=np.diagonal(dQ, axis1=-2, axis2=-1).copy(), dp=dp, dA=dA, db=db,
                dlb=None if bx["lb"] is None else -dh[..., :nlb], dub=None if bx["ub"] is None else dh[..., nlb:])
