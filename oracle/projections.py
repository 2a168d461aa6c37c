"""Closed-form solutions of two box QPs and their exact gradients (TEST INFRASTRUCTURE ONLY): references for the box
solver that share no code with any interior-point method.

    min 1/2 z' diag(q) z + p'z   s.t.   lb <= z <= ub                     (project_box; the projection of v at q = 1,
    min 1/2 z' diag(q) z + p'z   s.t.   1'z = k,  lb <= z <= ub            p = -v, and the capped simplex at lb = 0,
                                                                           ub = 1)
Both are separable given the multiplier nu of 1'z = k:  z_i = clamp((-p_i - nu) / q_i, lb_i, ub_i)  (nu = 0 without the
equality). nu is found by bisection on the monotone map nu -> 1'z, then recomputed exactly from the active sets.

The gradients are those of the implicit function at a strictly complementary solution. With F the free variables and
w = 1[F] / q:  dz/dp = -diag(w) + w w' / 1'w,  dz/dk = w / 1'w,  dz/dlb_i = e_i - w / 1'w (i at its lower bound), and
likewise for ub; q enters as p does, scaled by z. Each function returns z, nu and a `vjp(dl)` giving the box solver's
gradient dict (dq, dp, dA, db, dlb, dub; dA = dnu z' + nu dx' with dnu = -db, as for any equality row)."""
import numpy as np


def _sides(n, lb, ub):
    lo = np.full(n, -np.inf) if lb is None else np.asarray(lb, dtype=np.float64)
    hi = np.full(n, np.inf) if ub is None else np.asarray(ub, dtype=np.float64)
    return lo, hi


def _solution(q, p, lo, hi, nu):
    return np.clip((-p - nu) / q, lo, hi)


def _vjp_factory(q, z, nu, lo, hi, has_eq, lb, ub):
    at_lo = z <= lo
    at_hi = (z >= hi) & ~at_lo
    free = ~(at_lo | at_hi)
    w = np.where(free, 1.0 / q, 0.0)
    sw = w.sum()

    def vjp(dl):
        dl = np.asarray(dl, dtype=np.float64)
        c = (w @ dl) / sw if (has_eq and sw > 0) else 0.0     # the multiplier's share of dl
        dx = -w * dl + (w * c if has_eq else 0.0)
        g = dict(dx=dx, dp=dx, dq=dx * z, dA=None, db=None,
                 dlb=None if lb is None else np.where(at_lo, dl - c, 0.0),
                 dub=None if ub is None else np.where(at_hi, dl - c, 0.0))
        if has_eq:
            db = c
            g["db"] = np.array([db])
            g["dA"] = np.outer([-db], z) + nu * dx[None, :]
        return g

    return vjp


def project_box(q, p, lb, ub):
    """z = argmin 1/2 z'diag(q)z + p'z on lb <= z <= ub (lb / ub may be None). Returns (z, vjp)."""
    q, p = np.asarray(q, dtype=np.float64), np.asarray(p, dtype=np.float64)
    lo, hi = _sides(q.shape[0], lb, ub)
    z = _solution(q, p, lo, hi, 0.0)
    return z, _vjp_factory(q, z, 0.0, lo, hi, False, lb, ub)


def project_capped_simplex(q, p, k, lb, ub, iters=200):
    """z = argmin 1/2 z'diag(q)z + p'z s.t. 1'z = k, lb <= z <= ub (A = 1', b = [k]). Returns (z, nu, vjp)."""
    q, p = np.asarray(q, dtype=np.float64), np.asarray(p, dtype=np.float64)
    lo, hi = _sides(q.shape[0], lb, ub)
    k = float(np.asarray(k).reshape(-1)[0])
    # 1'z(nu) is non-increasing in nu: bracket k, then bisect
    a, b = -1.0, 1.0
    while _solution(q, p, lo, hi, a).sum() < k:
        a *= 2.0
    while _solution(q, p, lo, hi, b).sum() > k:
        b *= 2.0
    for _ in range(iters):
        mid = 0.5 * (a + b)
        if _solution(q, p, lo, hi, mid).sum() > k:
            a = mid
        else:
            b = mid
    nu = 0.5 * (a + b)
    z = _solution(q, p, lo, hi, nu)
    free = (z > lo) & (z < hi)
    if free.any():        # nu exactly from the active sets: sum_F (-p - nu) / q + sum_{not F} z = k
        nu = ((-p[free] / q[free]).sum() + z[~free].sum() - k) / (1.0 / q[free]).sum()
        z = np.where(free, (-p - nu) / q, z)
    return z, nu, _vjp_factory(q, z, nu, lo, hi, True, lb, ub)
