"""A dense torch model of QPFunction's first-order backward, whose own double backward is the reference for the double
backward (TEST INFRASTRUCTURE ONLY).

At a given point (z, lam, s, nu) the first backward solves, with D = clamp(lam, 1e-8) / clamp(s, 1e-8),

    [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] v = -[g_z; 0; g_lam; g_nu]

and returns dQ = sym(vx z'), dp = vx, dG = vlam z' + lam vx', dh = -vlam, dA = vnu z' + nu vx', db = -vnu. Here that is
written in torch ops (`dense_grads`, Q entering as sym(Q)). z, lam and nu come from `_Point`, a custom Function whose
forward returns the given point and whose backward is `dense_grads` again, so that torch can differentiate the backward
as often as it likes; s is the given slack with the derivative of h - G z. torch.autograd.grad of
sum_X <w_X, grad_X> through `first_backward` is then the double backward the kernels are specified to compute. Un-batched
inputs (`shared`) are expanded to the batch and their gradient is the batch mean, as QPFunction's.
"""
import numpy as np
import torch

NAMES = ("Q", "p", "G", "h", "A", "b")


def dense_grads(Q, G, A, z, lam, s, nu, gz, glam, gnu):
    """The six gradients per QP (each (B, ...)) of the backward at (z, lam, s, nu): every argument batched, A and nu
    (B, 0, n) / (B, 0) without equality rows, gnu None there."""
    B, n = z.shape
    m, e = lam.shape[1], nu.shape[1]
    Qs = 0.5 * (Q + Q.transpose(1, 2))
    D = lam.clamp(min=1e-8) / s.clamp(min=1e-8)
    f = dict(dtype=z.dtype, device=z.device)
    Im = torch.eye(m, **f).expand(B, m, m)
    Z = lambda r, c: torch.zeros(B, r, c, **f)
    K = torch.cat([torch.cat([Qs, Z(n, m), G.transpose(1, 2), A.transpose(1, 2)], 2),
                   torch.cat([Z(m, n), torch.diag_embed(D), Im, Z(m, e)], 2),
                   torch.cat([G, Im, Z(m, m), Z(m, e)], 2),
                   torch.cat([A, Z(e, m), Z(e, m), Z(e, e)], 2)], 1)
    rhs = torch.cat([gz, torch.zeros(B, m, **f), glam, gnu if gnu is not None else torch.zeros(B, e, **f)], 1)
    v = torch.linalg.solve(K, -rhs.unsqueeze(2)).squeeze(2)
    vx, vl, vn = v[:, :n], v[:, n + m:n + 2 * m], v[:, n + 2 * m:]
    outer = lambda a, b: a.unsqueeze(2) * b.unsqueeze(1)
    return dict(Q=0.5 * (outer(vx, z) + outer(z, vx)), p=vx, G=outer(vl, z) + outer(lam, vx), h=-vl,
                A=outer(vn, z) + outer(nu, vx), b=-vn)


def _slack(s0, G, h, z):
    """The slack s0 with the derivative of s = h - G z."""
    r = h - torch.matmul(G, z.unsqueeze(2)).squeeze(2)
    return s0 + (r - r.detach())


class _Point(torch.autograd.Function):
    """(z, lam, nu) of the given point as a function of the batched (Q, p, G, h, A, b), with the dense backward."""
    @staticmethod
    def forward(ctx, point, Q, p, G, h, A, b):
        ctx.point = point
        ctx.save_for_backward(Q, p, G, h, A, b)
        return point["z"].clone(), point["lam"].clone(), point["nu"].clone()

    @staticmethod
    def backward(ctx, gz, glam, gnu):
        Q, p, G, h, A, b = ctx.saved_tensors
        pt = ctx.point
        z, lam, nu = _Point.apply(pt, Q, p, G, h, A, b)
        zero = lambda t: torch.zeros_like(t)
        g = dense_grads(Q, G, A, z, lam, _slack(pt["s"], G, h, z), nu, gz if gz is not None else zero(z),
                        glam if glam is not None else zero(lam), gnu if gnu is not None else zero(nu))
        return (None,) + tuple(g[k] for k in NAMES)


def first_backward(ins, point, gz, glam, gnu, shared=()):
    """The first-order gradients {name: tensor} of QPFunction at `point` = {z, lam, s, nu} ((B, .) fp64 tensors), for
    the adjoints gz, glam, gnu (gnu None without equality rows). ins: {name: tensor}, batched or, for the names in
    `shared`, un-batched (their gradient is the batch mean). Differentiable in ins, gz, glam and gnu."""
    B = point["z"].shape[0]
    full = {}
    for k in NAMES:
        x = ins[k]
        full[k] = x.unsqueeze(0).expand(B, *x.shape) if k in shared else x
    z, lam, nu = _Point.apply(point, *(full[k] for k in NAMES))
    s = _slack(point["s"], full["G"], full["h"], z)
    g = dense_grads(full["Q"], full["G"], full["A"], z, lam, s, nu, gz, glam, gnu)
    return {k: (g[k].mean(0) if k in shared else g[k]) for k in NAMES}


def double_backward(ins, point, gz, glam, gnu, omegas, shared=()):
    """The reference double backward: the gradients of sum_X <w_X, grad_X> with respect to gz, glam, gnu and ins.
    omegas: {name: tensor or None}. Returns {"gz", "glam", "gnu", name: tensor} (fp64, detached)."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in ins.items()}
    adj = {"gz": gz, "glam": glam, "gnu": gnu}
    adj = {k: (None if v is None else v.detach().clone().requires_grad_(True)) for k, v in adj.items()}
    g = first_backward(leaves, point, adj["gz"], adj["glam"], adj["gnu"], shared)
    phi = sum((omegas[k] * g[k]).sum() for k in NAMES if omegas.get(k) is not None)
    wrt = [v for v in adj.values() if v is not None] + [leaves[k] for k in NAMES]
    res = torch.autograd.grad(phi, wrt, allow_unused=True)
    keys = [k for k, v in adj.items() if v is not None] + list(NAMES)
    return {k: (torch.zeros_like(x) if r is None else r) for k, r, x in zip(keys, res, wrt)}


def double_backward_one(solve, G, z, lam, s, nu, v, om):
    """The double backward of one QP with a given KKT solve, the algebra of qpb200_double_backward: solve(rx, rz, ry)
    returns the (x, lam, nu) parts of -K^-1 [rx; 0; rz; ry] (nu None without equality rows), v = (vx, vlam, vnu) is the
    first backward's solve with the same `solve`, om {name: array or None}. Returns {"gz", "glam", "gnu", name: array}."""
    n, m = z.shape[0], lam.shape[0]
    e = 0 if nu is None else nu.shape[0]
    vx, vl, vn = v
    w = {k: om.get(k) for k in NAMES}
    sym = lambda M: 0.5 * (M + M.T)
    rx, rz, ry = np.zeros(n), np.zeros(m), np.zeros(e)
    cz, cl, cn = np.zeros(n), np.zeros(m), np.zeros(e)
    if w["Q"] is not None:
        rx, cz = rx + sym(w["Q"]) @ z, cz + sym(w["Q"]) @ vx
    if w["p"] is not None:
        rx = rx + w["p"]
    if w["G"] is not None:
        rx, rz = rx + w["G"].T @ lam, rz + w["G"] @ z
        cz, cl = cz + w["G"].T @ vl, cl + w["G"] @ vx
    if w["h"] is not None:
        rz = rz - w["h"]
    if e and w["A"] is not None:
        rx, ry = rx + w["A"].T @ nu, ry + w["A"] @ z
        cz, cn = cz + w["A"].T @ vn, cn + w["A"] @ vx
    if e and w["b"] is not None:
        ry = ry - w["b"]
    ux, ul, un = solve(rx, rz, ry if e else None)
    sc = np.maximum(s, 1e-8)
    D = np.maximum(lam, 1e-8) / sc
    cD = (ul / D) * (vl / D)
    c_lam = np.where(lam >= 1e-8, cD / sc, 0.0)
    c_s = np.where(s >= 1e-8, -cD * D / sc, 0.0)
    wx, wl, wn = solve(cz - G.T @ c_s, cl + c_lam, cn if e else None)
    t = wl - c_s
    out = dict(gz=ux, glam=ul, Q=sym(np.outer(wx, z) + np.outer(ux, vx)), p=wx,
               G=np.outer(t, z) + np.outer(lam, wx) + np.outer(vl, ux) + np.outer(ul, vx), h=-t)
    if e:
        out.update(gnu=un, A=np.outer(wn, z) + np.outer(nu, wx) + np.outer(vn, ux) + np.outer(un, vx), b=-wn)
    return out
