"""numpy model of the ARITHMETIC of the dense-Q box kernels in csrc/qp_boxq.cu (TEST INFRASTRUCTURE ONLY).

Problem: min 1/2 z'Qz + p'z  s.t.  Az = b,  lb <= z <= ub with a dense Q, of which only the lower triangle is read
(`sym_lower`). The dense equivalent is QPFunction's (Q, G = [-I; I], h = [-lb; ub]). The loop is the one of
`oracle.box_model.solve_one`, and the inequality block is eliminated in the same way,
    H = Q + G'DG,  r = rx + G'(D rz - rs),  dz = D (G dx + rz) - rs,  ds = (-rs - dz) / D,
but H is now a dense matrix and [dx; dy] comes from ONE bordered factorization of the quasi-definite matrix
    K = [H A'; A 0] = L diag(I, -I) L',   L = [L11 0; L21 L22],
    L11 = chol(H),  L21 = A L11^-T,  M = L21 L21' (= A H^-1 A'),  L22 = chol(M),
and [dx; dy] = K^-1 [-r; -ry]: a forward sweep with L, the sign of the trailing block flipped, a backward sweep with
L'. `_SysQ` holds those four pieces as the kernels form them (the kernels' staircase holds H's lower triangle, A in the
border rows and -L21 L21' in the trailing block after the partial factorization, negated before it is factored).
"""
import numpy as np
import scipy.linalg as sla

from oracle.box_model import dense as _box_dense, rows
from oracle.kernel_model import _chol, _step


def sym_lower(Q):
    """The symmetric matrix the kernels see: Q's lower triangle, mirrored."""
    return np.tril(Q) + np.tril(Q, -1).T


def dense(Q, lb, ub):
    """The dense equivalent (Q, G, h) of one dense-Q box QP; lb / ub may be None."""
    _, G, h = _box_dense(np.ones(Q.shape[-1]), lb, ub)
    return sym_lower(np.asarray(Q, dtype=np.float64)), G, h


def _tri(L, v, trans=0):
    return sla.solve_triangular(L, v, lower=True, trans=trans, check_finite=False)


class _SysQ:
    """Factor of one Newton matrix for a given d: L11, L21, M, L22 (the last three None without A)."""

    def __init__(self, Q, A, var, sgn, d):
        n = Q.shape[0]
        self.A, self.var, self.sgn, self.d = A, var, sgn, d
        self.H = sym_lower(Q) + np.diag(np.bincount(var, weights=d, minlength=n))
        self.L11 = _chol(self.H)
        if A.shape[0] > 0:
            with np.errstate(all="ignore"):
                self.L21 = _tri(self.L11, A.T).T
            self.M = self.L21 @ self.L21.T
            self.L22 = _chol(self.M)
        else:
            self.L21 = self.M = self.L22 = None

    def solve(self, rx, rs, rz, ry):
        var, sgn, d = self.var, self.sgn, self.d
        r = rx + np.bincount(var, weights=sgn * (d * rz - rs), minlength=rx.shape[0])
        with np.errstate(all="ignore"):
            v1 = _tri(self.L11, -r)
            if self.L22 is not None:
                v2 = -_tri(self.L22, -ry - self.L21 @ v1)        # L v = f, then diag(I, -I)
                dy = _tri(self.L22, v2, 1)
                dx = _tri(self.L11, v1 - self.L21.T @ dy, 1)
            else:
                dy = None
                dx = _tri(self.L11, v1, 1)
            dz = d * (sgn * dx[var] + rz) - rs
            ds = (-rs - dz) / d
        return dx, ds, dz, dy


def kkt_solve(Q, A, has_lb, has_ub, d, rx, rs, rz, ry):
    """The structured KKT solve for one system (qpb200_boxq_solve_kkt): (dx, ds, dz, dy), dy None without A."""
    var, sgn = rows(Q.shape[0], has_lb, has_ub)
    return _SysQ(Q, A, var, sgn, d).solve(rx, rs, rz, ry if A.shape[0] > 0 else None)


def spd(Q):
    """What the forward's prologue tests: chol of Q itself (its lower triangle) breaks down or not."""
    L = _chol(sym_lower(Q))
    return bool(np.all(np.isfinite(np.diag(L))) and np.all(np.diag(L) > 0))


def solve_one(Q, p, A, b, lb, ub, eps=1e-12, notImprovedLim=3, maxIter=20, stall_tol=np.inf, tie=1.0,
              trace=None, kkt_log=None):
    """One dense-Q box QP; lb / ub arrays or None. trace / kkt_log as in kernel_model.solve_one."""
    n = Q.shape[0]
    e = A.shape[0]
    Qs = sym_lower(Q)
    var, sgn = rows(n, lb is not None, ub is not None)
    h = np.concatenate(([-lb] if lb is not None else []) + ([ub] if ub is not None else []))
    m = h.shape[0]

    def gt(v):
        return np.bincount(var, weights=sgn * v, minlength=n)

    def solve(d, rx, rs, rz, ry):
        sysm = _SysQ(Q, A, var, sgn, d)
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
            rx = Qs @ x + p + gt(z) + (A.T @ y if e > 0 else 0.0)
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
                best_iter=best["it"], Q=Q, A=A, var=var, sgn=sgn, nlb=n if lb is not None else 0)


def backward_one(sol, dl, dl_dlam=None, dl_dnu=None):
    """Gradients of one dense-Q box QP: dict(dQ, dp, dlb, dub, dA, db) (None for absent sides / no A), plus the
    solve's dx, dlam, dnu. dl_dlam / dl_dnu: adjoints of the returned duals (None: zero)."""
    Q, A, var, sgn, nlb = sol["Q"], sol["A"], sol["var"], sol["sgn"], sol["nlb"]
    m = var.shape[0]
    e = A.shape[0]
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        rz = np.zeros(m) if dl_dlam is None else dl_dlam
        ry = (np.zeros(e) if dl_dnu is None else dl_dnu) if e > 0 else None
        dx, _, dlam, dnu = _SysQ(Q, A, var, sgn, d).solve(dl, np.zeros(m), rz, ry)
    x = sol["x"]
    g = dict(dQ=0.5 * (np.outer(dx, x) + np.outer(x, dx)), dp=dx, dlb=dlam[:nlb] if nlb else None,
             dub=-dlam[nlb:] if m > nlb else None, dA=None, db=None, dx=dx, dlam=dlam, dnu=dnu)
    if e > 0:
        g["dA"] = np.outer(dnu, x) + np.outer(sol["nu"], dx)
        g["db"] = -dnu
    return g


def jvp_one(sol, dQ=None, dp=None, dA=None, db=None, dlb=None, dub=None):
    """Tangents (dz, dlam, dnu) of one solved QP: the backward's solve with rx = sym(dQ) z + dp + dA' nu,
    rz = [dlb; -dub], ry = dA z - db."""
    Q, A, var, nlb = sol["Q"], sol["A"], sol["var"], sol["nlb"]
    n, m, e = Q.shape[0], var.shape[0], A.shape[0]
    z = sol["x"]
    rx = np.zeros(n)
    if dQ is not None:
        rx += 0.5 * (dQ + dQ.T) @ z
    if dp is not None:
        rx += dp
    rz = np.zeros(m)
    if nlb and dlb is not None:
        rz[:nlb] = dlb
    if m > nlb and dub is not None:
        rz[nlb:] = -dub
    ry = None
    if e > 0:
        ry = np.zeros(e)
        if dA is not None:
            rx += dA.T @ sol["nu"]
            ry += dA @ z
        if db is not None:
            ry -= db
    with np.errstate(all="ignore"):
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        dx, _, dlam, dnu = _SysQ(Q, A, var, sol["sgn"], d).solve(rx, np.zeros(m), rz, ry)
    return dx, dlam, dnu


def qp_solve(Q, p, A, b, lb, ub, dl=None, **opts):
    """Batched wrapper: every given input batched ((B, nz, nz), (B, nz), (B, neq, nz), ...); lb / ub may be None.
    Returns stacked outputs; grads (when dl is given) keyed dQ, dp, dlb, dub, dA, db."""
    B = p.shape[0]
    sols = [solve_one(Q[i], p[i], A[i], b[i], None if lb is None else lb[i], None if ub is None else ub[i], **opts)
            for i in range(B)]
    e = A.shape[1]
    out = dict(zhat=np.stack([s["x"] for s in sols]), lam=np.stack([s["lam"] for s in sols]),
               slacks=np.stack([s["s"] for s in sols]),
               nus=np.stack([s["nu"] for s in sols]) if e > 0 else None,
               iters=np.array([s["iters"] for s in sols]), best_resids=np.array([s["best_resid"] for s in sols]),
               sols=sols)
    if dl is not None:
        gs = [backward_one(s, dl[i]) for i, s in enumerate(sols)]
        out["grads"] = {k: (None if gs[0][k] is None else np.stack([g[k] for g in gs]))
                        for k in ("dQ", "dp", "dlb", "dub", "dA", "db")}
    return out
