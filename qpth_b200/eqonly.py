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
    inequality row has G = 0): K~ dd = -(K [dx ds dz dy] + r), one factorization for all of them."""
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
        zhat, _, _, nus = _solve(F, Q, A, one, p, zero, -one, -b, steps)   # K [x s z y] = -[p 0 -h -b]
        ctx.F, ctx.flags, ctx.one, ctx.zero = F, flags, one, zero
        ctx.QA, ctx.steps = (Q, A), steps
        ctx.zhat64, ctx.nus = zhat, nus
        ctx.meta = [(X.device, X.dtype) for X in (Q_, p_, A_, b_)]
        zhat_out = zhat.to(device=Q_.device, dtype=Q_.dtype)
        if not duals:
            return zhat_out
        # duals: no inequality rows (lam is (nBatch, 0)); nu is the dy of the solve
        ctx.set_materialize_grads(False)
        return zhat_out, Q_.new_zeros(nBatch, 0), nus.to(device=Q_.device, dtype=Q_.dtype)

    @staticmethod
    def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
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
        for g, unb, (dev, dt), need in zip(grads, ctx.flags, ctx.meta, ctx.needs_input_grad[:4]):
            if not need:
                out.append(None)
                continue
            out.append((g.mean(0) if unb else g).to(device=dev, dtype=dt))
        return tuple(out) + (None, None, None)


def solve_equality_qp(Q_, p_, A_, b_, check_Q_spd=True, reg=False, duals=False):
    """z* of  argmin 1/2 z'Qz + p'z  s.t. Az = b  (differentiable in Q, p, A, b). reg: the regularised mode of
    QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) for a Q that is only positive semidefinite on the null space of A, or
    linearly dependent rows of A. duals: return (z*, lam, nu) as QPFunction(duals=True) does, lam (nBatch, 0)."""
    return QPEqualityFn.apply(Q_, p_, A_, b_, check_Q_spd, reg, duals)
