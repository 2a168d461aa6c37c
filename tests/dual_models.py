"""The backward passes of the numpy models with adjoints of the returned duals (TEST INFRASTRUCTURE ONLY).

QPFunction(duals=True) returns (z, lam, nu), and its backward pass puts the incoming gradients g_lam and g_nu into the rz
and ry slots of the backward's KKT solve:

    [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dlam dnu] = -[g_z; 0; g_lam; g_nu],   D = lam / s (clamped at 1e-8)

with the gradient formulas unchanged (dQ = 1/2 (dx z' + z dx'), dp = dx, dG = dlam z' + lam dx', dh = -dlam,
dA = dnu z' + nu dx', db = -dnu; for the box QP dq = dx o z, dlb = dlam_lb, dub = -dlam_ub). These are the models'
backward passes (oracle/kernel_model.backward_one, oracle/reg_model.backward_one_reg, oracle/box_model.backward_one)
with that right-hand side, written over the models' own solves; with g_lam = g_nu = None they are those functions.

`implicit` is the derivation they rest on, restated without any of it: the unsymmetric Jacobian of the KKT conditions
Qz + p + G'lam + A'nu = 0, diag(lam)(Gz - h) = 0, Az = b in (z, lam, nu), with diag(Gz - h) = -diag(s), solved
densely as J' w = -[g_z; g_lam; g_nu]. The loss gradient is then w' dF/dtheta: dx = w_z, dlam = diag(lam) w_lam,
dnu = w_nu.
"""
import numpy as np

from oracle import box_model as bm
from oracle import dense_kkt as dk
from oracle import kernel_model as km
from oracle import reg_model as rm


def _grads(x, lam, nu, dx, dlam, dnu):
    g = dict(dQ=0.5 * (np.outer(dx, x) + np.outer(x, dx)), dp=dx, dG=np.outer(dlam, x) + np.outer(lam, dx), dh=-dlam,
             dx=dx, dlam=dlam)
    if nu is not None and nu.size:
        g.update(dA=np.outer(dnu, x) + np.outer(nu, dx), db=-dnu, dnu=dnu)
    return g


def _rhs(m, e, glam, gnu):
    rz = np.zeros(m) if glam is None else np.asarray(glam, dtype=np.float64)
    ry = None if e == 0 else (np.zeros(e) if gnu is None else np.asarray(gnu, dtype=np.float64))
    return rz, ry


def backward_one(sol, dl, glam=None, gnu=None):
    """kernel_model.backward_one with the dual adjoints: a kernel_model.solve_one solution."""
    f = sol["f"]
    L = f["L"]
    m, e = f["Gt"].shape[0], f["e"]
    rz, ry = _rhs(m, e, glam, gnu)
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        L22 = km._chol(f["R"] + np.diag(1.0 / d))
        dxt, _, dlam, dnu = km._solve_kkt(f, L22, d, km._tri(L, dl), np.zeros(m), rz, ry)
        dx = km._tri(L, dxt, trans=True)
    return _grads(sol["x"], sol["lam"], sol["nu"], dx, dlam, dnu)


def backward_one_reg(sol, dl, glam=None, gnu=None):
    """reg_model.backward_one_reg with the dual adjoints: the regularised solve and its sol["steps"] refinement steps."""
    f, reg, Q, G, A = sol["f"], sol["reg"], sol["Q"], sol["G"], sol["A"]
    m, e = G.shape[0], f["e"]
    rz, ry = _rhs(m, e, glam, gnu)
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        F = rm._factor(f, d, reg)
        dx, _, dlam, dnu = rm._solve(f, F, reg, Q, G, A, dl, np.zeros(m), rz, ry, sol["steps"])
    return _grads(sol["x"], sol["lam"], sol["nu"], dx, dlam, dnu)


def backward_one_box(sol, dl, glam=None, gnu=None):
    """box_model.backward_one with the dual adjoints (glam in the [lb rows; ub rows] layout)."""
    q, A, var, sgn, nlb = sol["q"], sol["A"], sol["var"], sol["sgn"], sol["nlb"]
    m, e = var.shape[0], A.shape[0]
    rz, ry = _rhs(m, e, glam, gnu)
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        dx, _, dlam, dnu = bm._Sys(q, A, var, sgn, d).solve(dl, np.zeros(m), rz, ry)
    x = sol["x"]
    g = dict(dq=dx * x, dp=dx, dlb=dlam[:nlb] if nlb else None, dub=-dlam[nlb:] if m > nlb else None, dA=None, db=None,
             dx=dx, dlam=dlam, dnu=dnu)
    if e > 0:
        g["dA"] = np.outer(dnu, x) + np.outer(sol["nu"], dx)
        g["db"] = -dnu
    return g


def implicit(Q, G, A, x, lam, s, nu, gz, glam, gnu):
    """The gradients from the unsymmetric Jacobian of the KKT conditions at (x, lam, s, nu), solved densely (LU with
    longdouble-refined residuals, oracle/dense_kkt.solve_refined)."""
    n, m = Q.shape[0], G.shape[0]
    e = 0 if A is None else A.shape[0]
    N = n + m + e
    J = np.zeros((N, N))
    J[:n, :n] = Q
    J[:n, n:n + m] = G.T
    J[n:n + m, :n] = lam[:, None] * G
    J[n:n + m, n:n + m] = -np.diag(s)
    if e:
        J[:n, n + m:] = A.T
        J[n + m:, :n] = A
    g = np.concatenate([gz, glam] + ([gnu] if e else []))
    w = dk.solve_refined(J.T.copy(), -g)
    dx, dlam = w[:n], lam * w[n:n + m]
    dnu = w[n + m:] if e else None
    return _grads(x, lam, nu if e else None, dx, dlam, dnu)


def complementary_qp(seed, nz, nineq, neq):
    """A QP with a known, strictly complementary solution: z*, nu* ~ N(0, 1); min(nineq / 2, nz - neq - 2) (at least
    one) inequality rows active with lam* ~ U(0.1, 1) (s* = 0), the others inactive with s* ~ U(0.1, 1) (lam* = 0);
    h = G z* + s*, b = A z*, p = -(Q z* + G' lam* + A' nu*), Q = M M' / nz + 0.5 I."""
    rs = np.random.RandomState(seed)
    M = rs.randn(nz, nz)
    Q = M @ M.T / nz + 0.5 * np.eye(nz)
    G = rs.randn(nineq, nz) / np.sqrt(nz)
    A = rs.randn(neq, nz) / np.sqrt(nz)
    z = rs.randn(nz)
    nu = rs.randn(neq)
    # fewer active rows than nz - neq: the active rows and A are then linearly independent, so lam and nu are unique
    nact = max(1, min(nineq // 2, nz - neq - 2))
    act = np.zeros(nineq, dtype=bool)
    act[rs.permutation(nineq)[:nact]] = True
    lam = np.where(act, rs.uniform(0.1, 1.0, nineq), 0.0)
    s = np.where(act, 0.0, rs.uniform(0.1, 1.0, nineq))
    h = G @ z + s
    b = A @ z
    p = -(Q @ z + G.T @ lam + A.T @ nu)
    return dict(Q=Q, p=p, G=G, h=h, A=A, b=b, z=z, lam=lam, s=s, nu=nu, active=act)


def complementary_box(seed, n, e, sides):
    """A strictly complementary box QP: q ~ U(0.5, 2), z* with up to n - e - 2 variables at a bound (lb or ub, where
    the side exists; the free variables then give A full row rank, so lam and nu are unique), duals ~ U(0.1, 1) there,
    slack >= 0.1 elsewhere."""
    rs = np.random.RandomState(seed)
    has_lb, has_ub = sides != "ub", sides != "lb"
    q = rs.uniform(0.5, 2.0, n)
    A = rs.randn(e, n) / np.sqrt(n)
    z = rs.randn(n)
    nu = rs.randn(e)
    which = rs.randint(0, 2, n)
    which[rs.permutation(n)[:e + 2]] = 2
    at_lb = (which == 0) & has_lb
    at_ub = (which == 1) & has_ub
    lb = np.where(at_lb, z, z - rs.uniform(0.1, 1.0, n)) if has_lb else None
    ub = np.where(at_ub, z, z + rs.uniform(0.1, 1.0, n)) if has_ub else None
    lam_lb = np.where(at_lb, rs.uniform(0.1, 1.0, n), 0.0)
    lam_ub = np.where(at_ub, rs.uniform(0.1, 1.0, n), 0.0)
    # q z + p - lam_lb + lam_ub + A' nu = 0
    p = -(q * z - lam_lb + lam_ub + A.T @ nu)
    return dict(q=q, p=p, A=A, b=A @ z, lb=lb, ub=ub, z=z)
