"""The reference's stand-alone KKT solvers (qpth/solvers/pdipm/batch.py) on the CUDA kernels, same names and argument
order: `factor_solve_kkt` (:313-346, the LU_FULL variant: one exact solve of the full KKT system) and `solve_kkt_ir`
(:244-310, the IR_UNOPT variant: regularise with eps = 1e-7, solve, refine `niter` times against the residual of
`kkt_resid_reg` :228-241). Both run `qpb200_pre_factor_kkt[_reg]` + `qpb200_solve_kkt[_reg]`: the regularised system
is the same reduced Cholesky with `chol(Q + eps I)` and `W W^T + diag(eps, 1/(d + eps) + eps)`, SPD even for a
PSD-singular Q or a rank-deficient A (where the plain Cholesky path of QPFunction hits a zero pivot). The residual and
the correction loop are a handful of batched mat-vecs in torch on the device: glue, not the hot path.

All tensors fp64 on one CUDA device, batched: Q (B,nz,nz), D (B,nineq,nineq) diagonal (or its diagonal (B,nineq)),
G (B,nineq,nz), A (B,neq,nz) or None / empty, rx (B,nz), rs, rz (B,nineq), ry (B,neq) or None.
Returns (dx, ds, dz, dy) with dy None when neq == 0, like the reference.

These helpers keep the reference's signature and take a SYMMETRIC Q: the kernels read only its lower triangle, while the
residual of kkt_resid_reg (and so the refinement of solve_kkt_ir) multiplies by the whole of Q. QPFunction and the
equality-only path never call them with anything else."""
import ctypes

import torch

from . import _lib

IR_EPS = 1e-7          # batch.py:247
# Refinement steps per KKT solve of QPFunction(kkt_solver=KKTSolvers.IR_UNOPT). The Newton loop uses the residuals of
# the true problem, so the forward pass reaches the exact KKT point with 0 as well (oracle/reg_model.py: residuals
# <= 1e-12 either way); the backward pass is ONE solve, whose O(eps) error only refinement removes: on the rank-5 case
# of oracle/psd_cases.py the gradients move from 1.8e-5 to 1e-6 of the dense implicit-differentiation ones. A step costs
# a W pass pair, two chol(Q) sweeps and one reduced solve more per KKT solve. Each further step solves with the residual
# of the previous correction, so the error never grows with the step count; a second step helps only where one leaves
# more than rounding (SPD Q: the backward solve goes from 1e-7 to 5e-14 with one step, to 3e-15 with two). With a Q that
# is singular (an LP, a low-rank Q), chol(Q + eps I) limits every solve to about 1e-8 .. 2e-7 relative, whatever the count
# (tests/test_reg_refine_cpu.py).
IR_STEPS = 1


def _diag(D):
    return D if D.dim() == 2 else torch.diagonal(D, dim1=1, dim2=2)


class _Factored:
    """pre_factor_kkt[_reg] of one batch of systems; solve() may be called any number of times."""

    def __init__(self, Q, G, A, reg):
        assert Q.is_cuda and Q.dtype == torch.float64, "qpth_b200.kkt: fp64 CUDA tensors"
        self.B, self.nineq, self.nz = G.shape
        self.neq = A.shape[1] if (A is not None and A.numel() > 0) else 0
        self.reg = float(reg)
        self.dev = Q.device
        self.plan = _lib.plan_for(self.nz, self.nineq, self.neq, two=False)
        with torch.cuda.device(self.dev):
            self.L, self.W, self.K, self.scratch, self.spd = _lib.pre_factor(
                self.plan, self.B, self.B, Q.contiguous(), self.nz * self.nz, G.contiguous(), self.nineq * self.nz,
                A.contiguous() if self.neq else None, self.neq * self.nz, self.reg, self.dev, _lib.stream())

    def solve(self, d, rx, rs, rz, ry):
        B = self.B
        f64 = dict(dtype=torch.float64, device=self.dev)
        dx = torch.empty(B, self.nz, **f64); ds = torch.empty(B, self.nineq, **f64); dz = torch.empty(B, self.nineq, **f64)
        dy = torch.empty(B, self.neq, **f64) if self.neq else None
        args = [t.contiguous() for t in (d, rx, rs, rz)] + [ry.contiguous() if self.neq else None]
        P = _lib.ptr
        with torch.cuda.device(self.dev):
            _lib.check(_lib.load().qpb200_solve_kkt_reg(
                ctypes.byref(self.plan), B, *(P(t) for t in args), self.reg, P(self.L), P(self.W), P(self.K), 1,
                P(dx), P(ds), P(dz), P(dy), P(self.scratch), _lib.stream()))
        return dx, ds, dz, dy


def factor_solve_kkt(Q, D, G, A, rx, rs, rz, ry):
    """batch.py:313-346 (KKTSolvers.LU_FULL): the exact solve of
    [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dz dy] = -[rx rs rz ry]."""
    return _Factored(Q, G, A, 0.0).solve(_diag(D), rx, rs, rz, ry)


def factor_solve_kkt_reg(Q_tilde, D_tilde, G, A, rx, rs, rz, ry, eps):
    """batch.py:273-310 with the caller's already regularised Q~ = Q + eps I, D~ = D + eps I: solves
    [Q~ 0 G' A'; 0 D~ I 0; G I -eps I 0; A 0 0 -eps I] [dx ds dz dy] = -[rx rs rz ry] (the sign convention of
    kkt_resid_reg, batch.py:228-241; the reduced matrix is then SPD for any A)."""
    eye = torch.eye(Q_tilde.size(-1), dtype=Q_tilde.dtype, device=Q_tilde.device)
    f = _Factored(Q_tilde - eps * eye, G, A, eps)                 # the kernels add eps themselves
    return f.solve(_diag(D_tilde) - eps, rx, rs, rz, ry)


def kkt_resid_reg(Q, D, G, A, eps, dx, ds, dz, dy, rx, rs, rz, ry):
    """batch.py:228-241, with D given as a diagonal matrix or as its diagonal."""
    d = _diag(D)
    resx = torch.bmm(Q, dx.unsqueeze(2)).squeeze(2) + torch.bmm(G.transpose(1, 2), dz.unsqueeze(2)).squeeze(2) + rx
    if dy is not None:
        resx = resx + torch.bmm(A.transpose(1, 2), dy.unsqueeze(2)).squeeze(2)
    ress = d * ds + dz + rs
    resz = torch.bmm(G, dx.unsqueeze(2)).squeeze(2) + ds - eps * dz + rz
    resy = (torch.bmm(A, dx.unsqueeze(2)).squeeze(2) - eps * dy + ry) if dy is not None else None
    return resx, ress, resz, resy


def solve_kkt_ir(Q, D, G, A, rx, rs, rz, ry, niter=1):
    """batch.py:244-271 (KKTSolvers.IR_UNOPT): regularised solve + `niter` refinement steps. One factorization serves
    all of them."""
    eps = IR_EPS
    d = _diag(D)
    f = _Factored(Q, G, A, eps)
    dx, ds, dz, dy = f.solve(d, rx, rs, rz, ry)
    for _ in range(niter):
        resx, ress, resz, resy = kkt_resid_reg(Q, d, G, A, eps, dx, ds, dz, dy, rx, rs, rz, ry)
        ddx, dds, ddz, ddy = f.solve(d, resx, ress, resz, resy)          # solves  K~ dd = -res
        dx, ds, dz = dx + ddx, ds + dds, dz + ddz
        dy = dy + ddy if dy is not None else None
    return dx, ds, dz, dy
