"""numpy model of the ARITHMETIC of the box-constrained kernels in csrc/qp_box.cu (TEST INFRASTRUCTURE ONLY).

Problem: min 1/2 z' diag(q) z + p'z  s.t.  Az = b,  lb <= z <= ub, i.e. the dense QP with Q = diag(q),
G = [-I; I] (only the sides given: "lb rows" then "ub rows") and h = [-lb; ub]. The Mehrotra loop is the one of
`kernel_model.solve_one` (per-QP exits, stall_tol, best_tie, the same trace row), but every KKT solve
    [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dz dy] = -[rx rs rz ry]
eliminates the inequality block instead of whitening:
    H = q + G'DG (diagonal),  r = rx + G'(D rz - rs),  M = A H^-1 A'  (order neq),
    M dy = ry - A H^-1 r,  dx = -H^-1 (r + A'dy),  dz = D (G dx + rz) - rs,  ds = (-rs - dz) / D.
Nothing is whitened, so the dual residual is ||q x + p + G'z + A'y|| directly.
"""
import numpy as np
import scipy.linalg as sla

from oracle.kernel_model import _chol, _step


def rows(nz, has_lb, has_ub):
    """(var, sign) of every inequality row: G[i] = sign[i] * e_var[i]; lb rows first."""
    var = np.concatenate([np.arange(nz)] * (int(has_lb) + int(has_ub))).astype(np.int64)
    sgn = np.concatenate(([-np.ones(nz)] if has_lb else []) + ([np.ones(nz)] if has_ub else []))
    return var, sgn


def dense(q, lb, ub):
    """The dense equivalent (Q, G, h) of one box QP; lb / ub may be None."""
    n = q.shape[-1]
    G, h = [], []
    if lb is not None:
        G.append(-np.eye(n)); h.append(-np.asarray(lb, dtype=np.float64))
    if ub is not None:
        G.append(np.eye(n)); h.append(np.asarray(ub, dtype=np.float64))
    return np.diag(q), np.concatenate(G), np.concatenate(h)


class _Sys:
    """Factor of one Newton matrix: H^-1 and chol(M) for a given d."""

    def __init__(self, q, A, var, sgn, d):
        n = q.shape[0]
        self.A, self.var, self.sgn, self.d = A, var, sgn, d
        self.hinv = 1.0 / (q + np.bincount(var, weights=d, minlength=n))
        self.L = _chol((A * self.hinv) @ A.T) if A.shape[0] > 0 else None

    def solve(self, rx, rs, rz, ry):
        A, var, sgn, d, hinv = self.A, self.var, self.sgn, self.d, self.hinv
        r = rx + np.bincount(var, weights=sgn * (d * rz - rs), minlength=rx.shape[0])
        if self.L is not None:
            u = sla.solve_triangular(self.L, ry - A @ (hinv * r), lower=True, check_finite=False)
            dy = sla.solve_triangular(self.L, u, lower=True, trans=1, check_finite=False)
            dx = -hinv * (r + A.T @ dy)
        else:
            dy = None
            dx = -hinv * r
        dz = d * (sgn * dx[var] + rz) - rs
        ds = (-rs - dz) / d
        return dx, ds, dz, dy


def kkt_solve(q, A, has_lb, has_ub, d, rx, rs, rz, ry):
    """The structured KKT solve for one system (qpb200_box_solve_kkt): (dx, ds, dz, dy), dy None without A."""
    var, sgn = rows(q.shape[0], has_lb, has_ub)
    return _Sys(q, A, var, sgn, d).solve(rx, rs, rz, ry if A.shape[0] > 0 else None)


def solve_one(q, p, A, b, lb, ub, eps=1e-12, notImprovedLim=3, maxIter=20, stall_tol=np.inf, tie=1.0,
              trace=None, kkt_log=None):
    """One box QP; lb / ub arrays or None. trace / kkt_log as in kernel_model.solve_one."""
    n = q.shape[0]
    e = A.shape[0]
    var, sgn = rows(n, lb is not None, ub is not None)
    h = np.concatenate(([-lb] if lb is not None else []) + ([ub] if ub is not None else []))
    m = h.shape[0]

    def gt(v):
        return np.bincount(var, weights=sgn * v, minlength=n)

    def solve(d, rx, rs, rz, ry):
        sysm = _Sys(q, A, var, sgn, d)
        out = sysm.solve(rx, rs, rz, ry)
        if kkt_log is not None:
            kkt_log.append(dict(d=d.copy(), rx=rx.copy(), rs=rs.copy(), rz=rz.copy(),
                                ry=None if ry is None else ry.copy(), dx=out[0], ds=out[1], dz=out[2], dy=out[3]))
        return sysm, out

    with np.errstate(all="ignore"):
        _, (x, s, z, y) = solve(np.ones(m), p, np.zeros(m), -h, -b if e > 0 else None)
        if s.min() < 0:
            s = s - (s.min() - 1)
        if z.min() < 0:
            z = z - (z.min() - 1)
        best, minres, nNot, iters = None, None, 0, 0
        for it in range(maxIter):
            iters = it + 1
            rx = q * x + p + gt(z) + (A.T @ y if e > 0 else 0.0)
            rz = sgn * x[var] + s - h
            ry = A @ x - b if e > 0 else None
            mu = abs((s * z).sum() / m)
            pri = np.linalg.norm(rz) + (np.linalg.norm(ry) if e > 0 else 0.0)
            dual = np.linalg.norm(rx)
            resid = pri + dual + m * mu
            if trace is not None:
                trace.append([pri, dual, mu, resid])
            d = z / s
            cur = dict(x=x.copy(), s=s.copy(), z=z.copy(), y=None if y is None else y.copy(), it=it)
            if best is None or resid < minres:
                best, minres, nNot = cur, resid, 0
            else:
                nNot += 1
                if resid < tie * minres:
                    best = cur
            if (nNot == notImprovedLim and minres < stall_tol) or minres < eps or mu > 1e32:
                break
            if not np.isfinite(resid):
                break
            sysm, (dxa, dsa, dza, dya) = solve(d, rx, z, rz, ry)
            alpha = min(_step(z, dza), _step(s, dsa), 1.0)
            sig = (((s + alpha * dsa) * (z + alpha * dza)).sum() / (s * z).sum()) ** 3
            rs_c = (-mu * sig + dsa * dza) / s
            dxc, dsc, dzc, dyc = sysm.solve(np.zeros(n), rs_c, np.zeros(m), np.zeros(e) if e > 0 else None)
            if kkt_log is not None:
                kkt_log.append(dict(d=d.copy(), rx=np.zeros(n), rs=rs_c.copy(), rz=np.zeros(m),
                                    ry=np.zeros(e) if e > 0 else None, dx=dxc, ds=dsc, dz=dzc, dy=dyc))
            dx, ds, dz = dxa + dxc, dsa + dsc, dza + dzc
            alpha = min(0.999 * min(_step(z, dz), _step(s, ds)), 1.0)
            x = x + alpha * dx; s = s + alpha * ds; z = z + alpha * dz
            if e > 0:
                y = y + alpha * (dya + dyc)
    return dict(x=best["x"], lam=best["z"], s=best["s"], nu=best["y"], iters=iters, best_resid=minres,
                best_iter=best["it"], q=q, A=A, var=var, sgn=sgn, nlb=n if lb is not None else 0)


def backward_one(sol, dl):
    """Gradients of one box QP: dict(dq, dp, dlb, dub, dA, db) (None for absent sides / no A)."""
    q, A, var, sgn, nlb = sol["q"], sol["A"], sol["var"], sol["sgn"], sol["nlb"]
    m = var.shape[0]
    e = A.shape[0]
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        dx, _, dlam, dnu = _Sys(q, A, var, sgn, d).solve(dl, np.zeros(m), np.zeros(m), np.zeros(e) if e > 0 else None)
    x = sol["x"]
    g = dict(dq=dx * x, dp=dx, dlb=dlam[:nlb] if nlb else None, dub=-dlam[nlb:] if m > nlb else None,
             dA=None, db=None, dx=dx, dlam=dlam, dnu=dnu)
    if e > 0:
        g["dA"] = np.outer(dnu, x) + np.outer(sol["nu"], dx)
        g["db"] = -dnu
    return g


def qp_solve(q, p, A, b, lb, ub, dl=None, **opts):
    """Batched wrapper: every given input batched ((B, nz), (B, neq, nz), ...); lb / ub may be None.
    Returns stacked outputs; grads (when dl is given) keyed dq, dp, dlb, dub, dA, db."""
    B = p.shape[0]
    sols = [solve_one(q[i], p[i], A[i], b[i], None if lb is None else lb[i], None if ub is None else ub[i], **opts)
            for i in range(B)]
    e = A.shape[1]
    out = dict(zhat=np.stack([s["x"] for s in sols]), lam=np.stack([s["lam"] for s in sols]),
               slacks=np.stack([s["s"] for s in sols]),
               nus=np.stack([s["nu"] for s in sols]) if e > 0 else None,
               iters=np.array([s["iters"] for s in sols]), best_resids=np.array([s["best_resid"] for s in sols]))
    if dl is not None:
        gs = [backward_one(s, dl[i]) for i, s in enumerate(sols)]
        out["grads"] = {k: (None if gs[0][k] is None else np.stack([g[k] for g in gs]))
                        for k in ("dq", "dp", "dlb", "dub", "dA", "db")}
    return out
