"""References for BoxQPFunction's double backward (TEST INFRASTRUCTURE ONLY).

- A torch model: tests/double_backward_models.py on the dense equivalent, Q = diag_embed(q) (or the dense Q itself),
  G = [-I; I] constant (the sides given), h = [-lb; ub] built from the leaves. The dense gradients are mapped back to
  (q, p, A, b, lb, ub) with torch ops (diagonal, -dh_lb, dh_ub, batch means for un-batched inputs), and torch's own double
  backward through that is the reference.
- A numpy per-QP algebra of the kernels (`box_double_backward_one`), on the structured, eliminated solve
  (H = q + d_lb + d_ub, M = A H^-1 A'), cheap at the widest cluster shapes.
"""
import numpy as np
import torch

from tests import double_backward_models as dbm

NAMES = ("q", "p", "A", "b", "lb", "ub")


def _G(n, has_lb, has_ub, like):
    eye = torch.eye(n, dtype=like.dtype, device=like.device)
    return torch.cat(([-eye] if has_lb else []) + ([eye] if has_ub else []), 0)


def first_backward(ins, point, gz, glam, gnu, shared=(), dense_Q=False):
    """The first-order gradients {name: tensor} of BoxQPFunction at `point` = {z, lam, s, nu} ((B, .) fp64; lam and s in
    the [lb rows; ub rows] layout, nu (B, 0) without equality rows) for the adjoints gz, glam, gnu. ins: {name: tensor
    or None (an absent side)}, batched or, for the names in `shared`, un-batched (their gradient is the batch mean);
    A (B, 0, n) and b (B, 0) without equality rows. Differentiable in ins, gz, glam and gnu."""
    B, n = point["z"].shape
    full = {}
    for k in NAMES:
        x = ins[k]
        full[k] = None if x is None else (x.unsqueeze(0).expand(B, *x.shape) if k in shared else x)
    has_lb, has_ub = full["lb"] is not None, full["ub"] is not None
    Q = full["q"] if dense_Q else torch.diag_embed(full["q"])
    G = _G(n, has_lb, has_ub, point["z"]).unsqueeze(0).expand(B, -1, n)
    h = torch.cat(([-full["lb"]] if has_lb else []) + ([full["ub"]] if has_ub else []), 1)
    z, lam, nu = dbm._Point.apply(point, Q, full["p"], G, h, full["A"], full["b"])
    s = dbm._slack(point["s"], G, h, z)
    g = dbm.dense_grads(Q, G, full["A"], z, lam, s, nu, gz, glam, gnu)
    nlb = n if has_lb else 0
    out = {"q": g["Q"] if dense_Q else torch.diagonal(g["Q"], dim1=-2, dim2=-1), "p": g["p"], "A": g["A"],
           "b": g["b"], "lb": -g["h"][:, :nlb] if has_lb else None, "ub": g["h"][:, nlb:] if has_ub else None}
    return {k: (None if x is None else (x.mean(0) if k in shared else x)) for k, x in out.items()}


def double_backward(ins, point, gz, glam, gnu, omegas, shared=(), dense_Q=False):
    """The reference double backward: the gradients of sum_X <w_X, grad_X> with respect to gz, glam, gnu and the
    inputs. omegas: {name: tensor or None}. Returns {"gz", "glam", "gnu", name: tensor} (fp64, detached; an absent side
    None)."""
    leaves = {k: (None if v is None else v.detach().clone().requires_grad_(True)) for k, v in ins.items()}
    adj = {"gz": gz, "glam": glam, "gnu": gnu}
    adj = {k: (None if v is None else v.detach().clone().requires_grad_(True)) for k, v in adj.items()}
    g = first_backward(leaves, point, adj["gz"], adj["glam"], adj["gnu"], shared, dense_Q)
    phi = sum((omegas[k] * g[k]).sum() for k in NAMES if omegas.get(k) is not None and g[k] is not None)
    keys = [k for k, v in adj.items() if v is not None] + [k for k in NAMES if leaves[k] is not None]
    wrt = [adj[k] if k in adj else leaves[k] for k in keys]
    res = torch.autograd.grad(phi, wrt, allow_unused=True)
    out = {k: (torch.zeros_like(x) if r is None else r) for k, r, x in zip(keys, res, wrt)}
    for k in NAMES:
        out.setdefault(k, None)
    return out


# ---- the structured numpy algebra of qpb200_box_double_backward / qpb200_boxq_double_backward -----------------------

def box_solve(q, A, lam, s, nlb, has_ub, dense_Q=False):
    """solve(rx, rz, ry) -> the (x, lam, nu) parts of -K^-1 [rx; 0; rz; ry] for the box KKT system with the backward's
    clamped D, by elimination: H = q + d_lb + d_ub (dense Q: Q + diag(...)), r = rx - d_lb o rz_lb + d_ub o rz_ub,
    M nu = ry - A H^-1 r with M = A H^-1 A', x = -H^-1 (r + A' nu), lam = [d_lb o (rz_lb - x); d_ub o (rz_ub + x)]."""
    n = q.shape[-1]
    D = np.maximum(lam, 1e-8) / np.maximum(s, 1e-8)
    dl, du = D[:nlb], D[nlb:]
    g = np.zeros(n)
    if nlb:
        g = g + dl
    if has_ub:
        g = g + du
    e = 0 if A is None else A.shape[0]
    if dense_Q:
        H = 0.5 * (q + q.T) + np.diag(g)
        Hinv = lambda r: np.linalg.solve(H, r)
    else:
        h = q + g
        Hinv = lambda r: (r.T / h).T
    M = A @ Hinv(A.T) if e else None

    def solve(rx, rz, ry):
        r = rx.copy()
        if nlb:
            r = r - dl * rz[:nlb]
        if has_ub:
            r = r + du * rz[nlb:]
        if e:
            nu = np.linalg.solve(M, ry - A @ Hinv(r))
            x = -Hinv(r + A.T @ nu)
        else:
            nu, x = None, -Hinv(r)
        lm = np.concatenate(([dl * (rz[:nlb] - x)] if nlb else []) + ([du * (rz[nlb:] + x)] if has_ub else []))
        return x, lm, nu
    return solve


def box_double_backward_one(q, A, z, lam, s, nu, v, om, nlb, has_ub, dense_Q=False):
    """The double backward of one box QP as the kernels compute it: v = (vx, vlam, vnu) of the first backward (the same
    solve), om {name: array or None} the cotangents as each QP sees them (w / B for an un-batched input). Returns
    {"gz", "glam", "gnu", name: array} (per QP; an absent side None)."""
    n = z.shape[0]
    m = lam.shape[0]
    e = 0 if (nu is None or A is None) else nu.shape[0]
    solve = box_solve(q, A if e else None, lam, s, nlb, has_ub, dense_Q)
    vx, vl, vn = v
    w = {k: om.get(k) for k in NAMES}
    sym = lambda M: 0.5 * (M + M.T)
    rx, rz, ry = np.zeros(n), np.zeros(m), np.zeros(e)
    cz, cn = np.zeros(n), np.zeros(e)
    if w["q"] is not None:
        if dense_Q:
            rx, cz = rx + sym(w["q"]) @ z, cz + sym(w["q"]) @ vx
        else:
            rx, cz = rx + w["q"] * z, cz + w["q"] * vx
    if w["p"] is not None:
        rx = rx + w["p"]
    if e and w["A"] is not None:
        rx, ry = rx + w["A"].T @ nu, ry + w["A"] @ z
        cz, cn = cz + w["A"].T @ vn, cn + w["A"] @ vx
    if e and w["b"] is not None:
        ry = ry - w["b"]
    if nlb and w["lb"] is not None:
        rz[:nlb] = w["lb"]
    if has_ub and w["ub"] is not None:
        rz[nlb:] = -w["ub"]
    ux, ul, un = solve(rx, rz, ry)
    sc = np.maximum(s, 1e-8)
    D = np.maximum(lam, 1e-8) / sc
    cD = (ul / D) * (vl / D)
    c_lam = np.where(lam >= 1e-8, cD / sc, 0.0)
    c_s = np.where(s >= 1e-8, -cD * D / sc, 0.0)
    if nlb:
        cz = cz + c_s[:nlb]
    if has_ub:
        cz = cz - c_s[nlb:]
    wx, wl, wn = solve(cz, c_lam, cn)
    t = wl - c_s
    out = dict(gz=ux, glam=ul, gnu=None, p=wx, A=None, b=None,
               q=sym(np.outer(wx, z) + np.outer(ux, vx)) if dense_Q else wx * z + ux * vx,
               lb=t[:nlb] if nlb else None, ub=-t[nlb:] if has_ub else None)
    if e:
        out.update(gnu=un, A=np.outer(wn, z) + np.outer(nu, wx) + np.outer(vn, ux) + np.outer(un, vx), b=-wn)
    return out


def box_double_backward(q, A, z, lam, s, nu, v, om, nlb, has_ub, flags, dense_Q=False):
    """box_double_backward_one over a batch: q, A as the kernels see them (batched or shared numpy arrays), z, lam, s,
    nu, v batched, om {name: array or None} the caller's cotangents, flags {name: un-batched} (cotangent / B in, batch
    sum out). Returns {"gz", "glam", "gnu", name: array}."""
    B = z.shape[0]
    e = 0 if nu is None else nu.shape[1]
    qr = 3 if dense_Q else 2
    res = []
    for i in range(B):
        per = {k: (None if om.get(k) is None else (om[k] / B if flags.get(k) else om[k][i])) for k in NAMES}
        qi = q if q.ndim == qr - 1 else q[i]
        Ai = None if not e else (A if A.ndim == 2 else A[i])
        res.append(box_double_backward_one(qi, Ai, z[i], lam[i], s[i], nu[i] if e else None,
                                           (v[0][i], v[1][i], v[2][i] if e else None), per, nlb, has_ub, dense_Q))
    out = {}
    for k in ("gz", "glam", "gnu") + NAMES:
        xs = [r[k] for r in res]
        if xs[0] is None:
            out[k] = None
        elif flags.get(k):
            acc = np.zeros_like(xs[0])
            for x in xs:
                acc = acc + x
            out[k] = acc
        else:
            out[k] = np.stack(xs)
    return out
