"""Equality-constrained QPs (nineq == 0, neq > 0) behind `QPFunction`: an EXTENSION of the reference's surface.

The reference cannot run this case - it unpacks `G.size()` (`qpth/qp.py:87`) and takes the minimum of an empty slack
vector (`solvers/pdipm/batch.py:77`) - although its own algebra covers it: without inequalities the optimum is ONE KKT
solve, the one `forward` performs for its initial point (`batch.py:61-67`: `solve_kkt(p, 0, -h, -b)` with d = 1), and
the backward pass is the same solve with `dl_dzhat` on the right-hand side (`qp.py:148-177`). Here both are the
stand-alone `pre_factor_kkt` + `solve_kkt` kernels (`qpth_b200/kkt.py`, C ABI `qpb200_pre_factor_kkt_reg` /
`qpb200_solve_kkt_reg`) with one decoupled dummy inequality row (G = 0, h = 1, d = 1: the reduced matrix gets a unit
diagonal entry for it and nothing else), so no interior-point iteration - and no step length over a slack that never
moves - is involved. Gradient conventions are the reference's: symmetrised dQ, `.mean(0)` for un-batched inputs.
"""
import torch
from torch.autograd import Function

from . import _lib, kkt
from .util import bger, check_shapes, expandParam

_factor = kkt._Factored          # (tests inject a CPU stand-in here)
# Refinement steps of each solve in the regularised mode (kkt_solver=IR_UNOPT): with no Newton loop around it, the one
# regularised solve is off by O(IR_EPS), and each step against the true system takes a factor of about IR_EPS off that.
EQ_IR_STEPS = 2


def _solve(F, Q, A, d, rx, rs, rz, ry, steps):
    """F.solve, then `steps` refinement steps against the true system [Q 0 0 A'; 0 d 1 0; 0 1 0 0; A 0 0 0] (the dummy
    inequality row has G = 0): K~ dd = -(K [dx ds dz dy] + r), one factorization for all of them. Q must be the symmetric
    matrix the factor saw (the mirrored lower triangle of the caller's Q)."""
    dx, ds, dz, dy = F.solve(d, rx, rs, rz, ry)
    for _ in range(steps):
        resx = torch.bmm(Q, dx.unsqueeze(2)).squeeze(2) + torch.bmm(A.transpose(1, 2), dy.unsqueeze(2)).squeeze(2) + rx
        resy = torch.bmm(A, dx.unsqueeze(2)).squeeze(2) + ry
        ex, es, ez, ey = F.solve(d, resx, d * ds + dz + rs, ds + rz, resy)
        dx, ds, dz, dy = dx + ex, ds + es, dz + ez, dy + ey
    return dx, ds, dz, dy


def _target_device(Q_):
    if not torch.cuda.is_available():
        raise _lib.QpthB200Error("qpth_b200: no CUDA device available (there is no CPU fallback).")
    return Q_.device if Q_.is_cuda else torch.device("cuda", torch.cuda.current_device())


class QPEqualityFn(Function):
    @staticmethod
    def forward(ctx, Q_, p_, A_, b_, check_Q_spd, reg=False, duals=False):
        empty = Q_.new_empty(0)
        nBatch, nz, nineq, neq = check_shapes(Q_, p_, empty, empty, A_, b_)
        assert neq > 0 or nineq > 0                         # qp.py:89
        device = _target_device(Q_)
        f64 = dict(dtype=torch.float64, device=device)
        batched = []
        flags = []
        for X, nd in ((Q_, 3), (p_, 2), (A_, 3), (b_, 2)):
            Xe, was_unbatched = expandParam(X.detach().to(**f64), nBatch, nd)
            batched.append(Xe.contiguous())
            flags.append(was_unbatched)
        Q, p, A, b = batched
        # one dummy row: G = 0 (h = 1, d = 1 below); regularised mode: chol(Q + eps I), eps on the constraint blocks
        F = _factor(Q, torch.zeros(nBatch, 1, nz, **f64), A, kkt.IR_EPS if reg else 0.0)
        if check_Q_spd and bool(F.spd.any()):
            raise RuntimeError('Q is not positive semidefinite.' if reg else 'Q is not SPD.')
        one, zero = torch.ones(nBatch, 1, **f64), torch.zeros(nBatch, 1, **f64)
        steps = EQ_IR_STEPS if reg else 0
        # the factor sees only the lower triangle of Q: refine against that matrix, tril(Q) + tril(Q, -1)', so that the
        # strictly upper triangle is never read here either
        Qr = (torch.tril(Q) + torch.tril(Q, -1).transpose(1, 2)) if steps else Q
        zhat, _, _, nus = _solve(F, Qr, A, one, p, zero, -one, -b, steps)   # K [x s z y] = -[p 0 -h -b]
        ctx.F, ctx.flags, ctx.one, ctx.zero = F, flags, one, zero
        ctx.QA, ctx.steps = (Qr, A), steps
        ctx.zhat64, ctx.nus = zhat, nus
        ctx.meta = [(X.device, X.dtype) for X in (Q_, p_, A_, b_)]
        ctx.duals = duals
        ctx.save_for_backward(Q_, p_, A_, b_)
        ctx.set_materialize_grads(False)
        zhat_out = zhat.to(device=Q_.device, dtype=Q_.dtype)
        if not duals:
            return zhat_out
        # duals: no inequality rows (lam is (nBatch, 0)); nu is the dy of the solve
        return zhat_out, Q_.new_zeros(nBatch, 0), nus.to(device=Q_.device, dtype=Q_.dtype)

    @staticmethod
    def jvp(ctx, dQ, dp, dA, db, *_):
        # the backward's solve with rx = sym(dQ) z + dp + dA' nu and ry = dA z - db (the dummy row's rz is 0)
        z, nus = ctx.zhat64, ctx.nus
        T = lambda t: None if t is None else t.detach().to(device=z.device, dtype=torch.float64)
        dQ, dp, dA, db = T(dQ), T(dp), T(dA), T(db)
        rx, ry = torch.zeros_like(z), torch.zeros_like(nus)
        if dQ is not None:
            zc = z.unsqueeze(2)
            rx = rx + 0.5 * (torch.matmul(dQ, zc) + torch.matmul(dQ.transpose(-1, -2), zc)).squeeze(2)
        if dp is not None:
            rx = rx + dp
        if dA is not None:
            rx = rx + torch.matmul(dA.transpose(-1, -2), nus.unsqueeze(2)).squeeze(2)
            ry = ry + torch.matmul(dA, z.unsqueeze(2)).squeeze(2)
        if db is not None:
            ry = ry - db
        dx, _, _, dnu = _solve(ctx.F, *ctx.QA, ctx.one, rx.contiguous(), ctx.zero, ctx.zero, ry.contiguous(), ctx.steps)
        dev, dt = ctx.meta[0]
        dz = dx.to(device=dev, dtype=dt)
        if not ctx.duals:
            return dz
        return dz, torch.zeros(dz.shape[0], 0, device=dev, dtype=dt), dnu.to(device=dev, dtype=dt)

    @staticmethod
    def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
        if torch.is_grad_enabled():          # create_graph=True: gradients that can be differentiated again
            return QPEqualityBackwardFn.apply(ctx, ctx.needs_input_grad[:4], dl_dzhat, dl_dnu,
                                              *ctx.saved_tensors) + (None, None, None)
        return _first_order(ctx, dl_dzhat, dl_dnu, ctx.needs_input_grad[:4])[0] + (None, None, None)


def _first_order(ctx, dl_dzhat, dl_dnu, want):
    """QPEqualityFn's backward at the state `ctx` of its forward: (the gradients of Q, p, A, b, (dx, dnu))."""
    z, nus = ctx.zhat64, ctx.nus
    dl = (torch.zeros_like(z) if dl_dzhat is None
          else dl_dzhat.detach().to(device=z.device, dtype=torch.float64).contiguous().view_as(z))
    # dl/dnu is the ry of the solve: K [dx ds dz dnu] = -[dl 0 0 dl/dnu]
    ry = (torch.zeros_like(nus) if dl_dnu is None
          else dl_dnu.detach().to(device=z.device, dtype=torch.float64).contiguous().view_as(nus))
    dx, _, _, dnu = _solve(ctx.F, *ctx.QA, ctx.one, dl, ctx.zero, ctx.zero, ry, ctx.steps)
    grads = [0.5 * (bger(dx, z) + bger(z, dx)),         # qp.py:175-177
             dx,                                        # qp.py:150
             bger(dnu, z) + bger(nus, dx),              # qp.py:166-167
             -dnu]                                      # qp.py:168
    out = []
    for g, unb, (dev, dt), need in zip(grads, ctx.flags, ctx.meta, want):
        if not need:
            out.append(None)
            continue
        out.append((g.mean(0) if unb else g).to(device=dev, dtype=dt))
    return tuple(out), (dx, dnu)


def _mv(M, x):
    return torch.matmul(M, x.unsqueeze(-1)).squeeze(-1)


class QPEqualityBackwardFn(Function):
    """QPEqualityFn's backward as a differentiable function of (g_z, g_nu, Q, p, A, b), under create_graph=True. Its
    backward is the double backward of qpb200_double_backward without inequality rows (no D, c_lam or c_s terms), with
    the same solves as the first order: u = the JVP for tangents w (the gradients of g_z, g_nu), then the solve of the
    cotangents cz = sym(wQ) vx + wA' vnu, cnu = wA vx of (z, nu), w; dQ = sym(wx z' + ux vx'), dp = wx,
    dA = wnu z' + nu wx' + vnu ux' + unu vx', db = -wnu. The cotangent of a batch mean is w / nBatch per QP, and the
    gradient of an un-batched input the batch sum."""
    @staticmethod
    def forward(ctx, eq, want, g_z, g_nu, Q_, p_, A_, b_):
        out, ctx.v = _first_order(eq, g_z, g_nu, want)
        ctx.eq = eq
        ctx.like = (g_z, g_nu, Q_, p_, A_, b_)
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, wQ, wp, wA, wb):
        from .qp import THIRD_ORDER_ERR
        if torch.is_grad_enabled():
            raise RuntimeError(THIRD_ORDER_ERR)
        need = ctx.needs_input_grad[2:]
        if all(w is None for w in (wQ, wp, wA, wb)) or not any(need):
            return (None,) * 8
        eq = ctx.eq
        z, nus = eq.zhat64, eq.nus
        vx, vn = ctx.v
        B = z.shape[0]
        om = []
        for w, unb in zip((wQ, wp, wA, wb), eq.flags):
            w = None if w is None else w.detach().to(device=z.device, dtype=torch.float64)
            om.append(None if w is None else (w / B if unb else w))
        wQ, wp, wA, wb = om
        rx, ry, cz, cn = torch.zeros_like(z), torch.zeros_like(nus), torch.zeros_like(z), torch.zeros_like(nus)
        if wQ is not None:
            rx = rx + 0.5 * (_mv(wQ, z) + _mv(wQ.transpose(-1, -2), z))
            cz = cz + 0.5 * (_mv(wQ, vx) + _mv(wQ.transpose(-1, -2), vx))
        if wp is not None:
            rx = rx + wp
        if wA is not None:
            rx = rx + _mv(wA.transpose(-1, -2), nus)
            ry = ry + _mv(wA, z)
            cz = cz + _mv(wA.transpose(-1, -2), vn)
            cn = cn + _mv(wA, vx)
        if wb is not None:
            ry = ry - wb
        ux, _, _, un = _solve(eq.F, *eq.QA, eq.one, rx.contiguous(), eq.zero, eq.zero, ry.contiguous(), eq.steps)
        wx, _, _, wn = _solve(eq.F, *eq.QA, eq.one, cz.contiguous(), eq.zero, eq.zero, cn.contiguous(), eq.steps)
        grads = [ux, un,
                 0.5 * ((bger(wx, z) + bger(z, wx)) + (bger(ux, vx) + bger(vx, ux))),
                 wx,
                 bger(wn, z) + bger(nus, wx) + bger(vn, ux) + bger(un, vx),
                 -wn]
        unb = (False, False) + tuple(eq.flags)
        res = []
        for g, X, u, n in zip(grads, ctx.like, unb, need):
            res.append((g.sum(0) if u else g).to(device=X.device, dtype=X.dtype) if (n and X is not None) else None)
        return (None, None) + tuple(res)


def solve_equality_qp(Q_, p_, A_, b_, check_Q_spd=True, reg=False, duals=False):
    """z* of  argmin 1/2 z'Qz + p'z  s.t. Az = b  (differentiable in Q, p, A, b). reg: the regularised mode of
    QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) for a Q that is only positive semidefinite on the null space of A, or
    linearly dependent rows of A. duals: return (z*, lam, nu) as QPFunction(duals=True) does, lam (nBatch, 0)."""
    return QPEqualityFn.apply(Q_, p_, A_, b_, check_Q_spd, reg, duals)
