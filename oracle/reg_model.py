"""numpy model of the regularised mode, QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) (TEST INFRASTRUCTURE ONLY).

The arithmetic of the kReg kernels (qp_solve.cuh) over kernel_model's whitened formulation: every KKT solve factors the
regularised system [Q+eI 0 G' A'; 0 D+eI I 0; G I -eI 0; A 0 0 -eI] (kernel_model.setup(reg=e): chol(Q + eI),
chol(A~A~' + eI)), while the residuals are those of the TRUE problem, so the loop is an inexact Newton method whose
fixed point is the exact KKT point even when Q is singular or A rank-deficient. `steps` refinement steps against the
true system follow the initial solve and each iteration's combined direction (the kernels' placement; refining the
affine and corrector directions one by one gives the same direction, the refinement being linear).
"""
import numpy as np

from . import kernel_model as km


def _factor(f, d, reg):
    dt = d + reg
    return km._chol(f["R"] + np.diag(1.0 / dt + reg)), dt


def _solve(f, F, reg, Q, G, A, rx, rs, rz, ry, steps):
    """K~ [dx ds dz dy] = -[rx rs rz ry], then `steps` corrections K~ dd = -(K [dx ds dz dy] + r)."""
    L22, dt = F
    e = f["e"]

    def one(rx, rs, rz, ry):
        dxt, ds, dz, dy = km._solve_kkt(f, L22, dt, km._tri(f["L"], rx), rs, rz, ry if e > 0 else None)
        return km._tri(f["L"], dxt, trans=True), ds, dz, dy

    dx, ds, dz, dy = one(rx, rs, rz, ry)
    cx, cs, cz, cy = dx, ds, dz, dy                          # the last correction (the solve itself at first)
    for _ in range(steps):
        # With K = K~ - Delta, the true residual K d + r of d = d0 + c1 + ... + ck is -Delta ck (K~ d0 = -r,
        # K~ cj = Delta c(j-1)): (-reg cx, -reg cs, reg cz, reg cy) of the LAST correction, not of the running total
        cx, cs, cz, cy = one(-reg * cx, -reg * cs, reg * cz, reg * cy if e > 0 else None)
        dx, ds, dz = dx + cx, ds + cs, dz + cz
        if e > 0:
            dy = dy + cy
    return dx, ds, dz, dy


def solve_one_reg(Q, p, G, h, A, b, reg=1e-7, steps=0, eps=1e-12, notImprovedLim=3, maxIter=20, stall_tol=1e-6,
                  tie=1.5, trace=None):
    """The forward kernel's loop (per-QP exits, STALL_TOL / BEST_TIE rules of QPFunction) in the original variables."""
    m, n = G.shape
    f = km.setup(Q, G, A, reg)
    e = f["e"]
    with np.errstate(all="ignore"):
        F = _factor(f, np.ones(m), reg)
        x, s, z, y = _solve(f, F, reg, Q, G, A, p, np.zeros(m), -h, -b if e > 0 else None, steps)
        if s.min() < 0:
            s = s - (s.min() - 1)
        if z.min() < 0:
            z = z - (z.min() - 1)
        best, minres, nNot, iters = None, None, 0, 0
        for it in range(maxIter):
            iters = it + 1
            rx = Q @ x + p + G.T @ z + (A.T @ y if e > 0 else 0.0)
            rz = G @ x + s - h
            ry = A @ x - b if e > 0 else None
            mu = abs((s * z).sum() / m)
            pri = np.linalg.norm(rz) + (np.linalg.norm(ry) if e > 0 else 0.0)
            dual = np.linalg.norm(rx)
            resid = pri + dual + m * mu
            if trace is not None:
                trace.append([pri, dual, mu, resid])
            snap = dict(x=x.copy(), s=s.copy(), z=z.copy(), y=None if y is None else y.copy(), it=it)
            if best is None or resid < minres:
                minres, nNot = resid, 0
                best = snap
            else:
                nNot += 1
                if resid < tie * minres:
                    best = snap
            if (nNot == notImprovedLim and minres < stall_tol) or minres < eps or mu > 1e32:
                break
            if not np.isfinite(resid):
                break
            d = z / s
            F = _factor(f, d, reg)
            dxa, dsa, dza, dya = _solve(f, F, reg, Q, G, A, rx, z, rz, ry, 0)
            alpha = min(km._step(z, dza), km._step(s, dsa), 1.0)
            sig = (((s + alpha * dsa) * (z + alpha * dza)).sum() / (s * z).sum()) ** 3
            rs_c = (-mu * sig + dsa * dza) / s
            # the combined direction solves K~ d = -(r_aff + r_cor); refined as a whole
            dx, ds, dz, dy = _solve(f, F, reg, Q, G, A, rx, z + rs_c, rz, ry, steps)
            alpha = min(0.999 * min(km._step(z, dz), km._step(s, ds)), 1.0)
            x = x + alpha * dx; s = s + alpha * ds; z = z + alpha * dz
            if e > 0:
                y = y + alpha * dy
    return dict(x=best["x"], lam=best["z"], s=best["s"], nu=best["y"], f=f, iters=iters, best_resid=minres,
                best_iter=best["it"], reg=reg, steps=steps, Q=Q, G=G, A=A)


def backward_one_reg(sol, dl):
    """The backward kernel: d = max(lam, 1e-8) / max(s, 1e-8) (qp.py:148), one regularised solve + refinement."""
    f, reg, Q, G, A = sol["f"], sol["reg"], sol["Q"], sol["G"], sol["A"]
    m, e = G.shape[0], f["e"]
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        F = _factor(f, d, reg)
        dx, _, dlam, dnu = _solve(f, F, reg, Q, G, A, dl, np.zeros(m), np.zeros(m), np.zeros(e) if e > 0 else None,
                                  sol["steps"])
    x, lam = sol["x"], sol["lam"]
    g = dict(dQ=0.5 * (np.outer(dx, x) + np.outer(x, dx)), dp=dx, dG=np.outer(dlam, x) + np.outer(lam, dx), dh=-dlam)
    if e > 0:
        g["dA"] = np.outer(dnu, x) + np.outer(sol["nu"], dx)
        g["db"] = -dnu
    return g
