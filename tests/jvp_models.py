"""Numpy models of forward mode (TEST INFRASTRUCTURE ONLY): the JVP of (z, lam, nu) at a returned point.

For input tangents dQ, dp, dG, dh, dA, db (None: zero) the JVP is the backward's own KKT solve with the right-hand side
    rx = sym(dQ) z + dp + dG' lam + dA' nu,   rz = dG z - dh,   ry = dA z - db,         sym(dQ) = (dQ + dQ') / 2
    [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [z. s. lam. nu.] = -[rx; 0; rz; ry],   D = clamp(lam, 1e-8) / clamp(s, 1e-8)
and for the box QP rx = dq o z + dp + dA' nu, rz = [dlb; -dub], ry = dA z - db. These models solve that system with
oracle/dense_kkt.solve (refined dense LU), the box model's structured solve, or the regularised model's solve and its
refinement steps: the same solves as tests/dual_models.py, with the tangents' right-hand side.
"""
import numpy as np

from oracle import box_model as bm
from oracle import dense_kkt as dk
from oracle import reg_model as rm


def _z(t, shape):
    return np.zeros(shape) if t is None else np.asarray(t, dtype=np.float64)


def rhs(z, lam, nu, tan):
    """(rx, rz, ry) of one QP; tan: dict of Q, p, G, h, A, b tangents (missing or None: zero)."""
    n, m = z.shape[0], lam.shape[0]
    e = 0 if nu is None else nu.shape[0]
    dQ, dp = _z(tan.get("Q"), (n, n)), _z(tan.get("p"), n)
    dG, dh = _z(tan.get("G"), (m, n)), _z(tan.get("h"), m)
    rx = 0.5 * (dQ + dQ.T) @ z + dp + dG.T @ lam
    rz = dG @ z - dh
    ry = None
    if e:
        dA, db = _z(tan.get("A"), (e, n)), _z(tan.get("b"), e)
        rx = rx + dA.T @ nu
        ry = dA @ z - db
    return rx, rz, ry


def jvp_dense(Q, G, A, z, lam, s, nu, tan):
    """(dz, dlam, dnu) from the refined dense solve with qpth's clamped d."""
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    rx, rz, ry = rhs(z, lam, nu if e else None, tan)
    d = np.maximum(lam, 1e-8) / np.maximum(s, 1e-8)
    dx, _, dlam, dnu, _, _ = dk.solve(Q, G, A if e else None, d, rx, np.zeros(lam.shape[0]), rz, ry)
    return dx, dlam, dnu


def jvp_reg(sol, tan):
    """The regularised model (reg_model) at sol (as tests/dual_models.backward_one_reg takes it) with sol["steps"]
    refinement steps."""
    f, reg, Q, G, A = sol["f"], sol["reg"], sol["Q"], sol["G"], sol["A"]
    m, e = G.shape[0], f["e"]
    rx, rz, ry = rhs(sol["x"], sol["lam"], sol["nu"] if e else None, tan)
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        F = rm._factor(f, d, reg)
        dx, _, dlam, dnu = rm._solve(f, F, reg, Q, G, A, rx, np.zeros(m), rz, ry, sol["steps"])
    return dx, dlam, dnu


def box_rhs(z, nu, nlb, has_ub, tan):
    """(rx, rz, ry) of one box QP; tan: dict of q, p, A, b, lb, ub tangents (missing or None: zero)."""
    n = z.shape[0]
    e = 0 if nu is None else nu.shape[0]
    rx = _z(tan.get("q"), n) * z + _z(tan.get("p"), n)
    rz = np.concatenate(([_z(tan.get("lb"), n)] if nlb else []) + ([-_z(tan.get("ub"), n)] if has_ub else []))
    ry = None
    if e:
        dA = _z(tan.get("A"), (e, n))
        rx = rx + dA.T @ nu
        ry = dA @ z - _z(tan.get("b"), e)
    return rx, rz, ry


def jvp_box(q, A, z, lam, s, nu, nlb, has_ub, tan):
    """(dz, dlam, dnu) from the box model's structured solve, lam in the [lb rows; ub rows] layout."""
    n, e = z.shape[0], A.shape[0]
    var, sgn = bm.rows(n, nlb > 0, has_ub)
    rx, rz, ry = box_rhs(z, nu if e else None, nlb, has_ub, tan)
    with np.errstate(all="ignore"):
        d = np.maximum(lam, 1e-8) / np.maximum(s, 1e-8)
        dx, _, dlam, dnu = bm._Sys(q, A, var, sgn, d).solve(rx, np.zeros(var.shape[0]), rz, ry)
    return dx, dlam, dnu


def implicit_jvp(Q, G, A, z, lam, s, nu, tan, clamp=False):
    """(dz, dlam, dnu) from the unsymmetric Jacobian of Qz + p + G'lam + A'nu = 0, diag(lam)(Gz - h) = 0, Az = b:
    J [z.; lam.; nu.] = -[rx; diag(lam) rz; ry]. clamp: lam and s clamped at 1e-8 in J (the row scaling of the backward's
    system, whose d = lam / s is qpth's clamped one); otherwise the exact derivative of the solution map."""
    n, m = Q.shape[0], G.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    rx, rz, ry = rhs(z, lam, nu if e else None, tan)
    lc, sc = (np.maximum(lam, 1e-8), np.maximum(s, 1e-8)) if clamp else (lam, s)
    N = n + m + e
    J = np.zeros((N, N))
    J[:n, :n] = Q
    J[:n, n:n + m] = G.T
    J[n:n + m, :n] = lc[:, None] * G
    J[n:n + m, n:n + m] = -np.diag(sc)
    if e:
        J[:n, n + m:] = A.T
        J[n + m:, :n] = A
    w = dk.solve_refined(J, -np.concatenate([rx, lc * rz] + ([ry] if e else [])))
    return w[:n], w[n:n + m], (w[n + m:] if e else None)
