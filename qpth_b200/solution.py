"""Differentiate a QP solution that was produced elsewhere (SURVEY.md section 8(f), rank 1).

The reference has one such path: `QPFunction(solver=QPSolvers.CVXPY)` solves every sample with CVXPY on the CPU
(`qpth/qp.py:97-120`, `qpth/solvers/cvxpy.py:5-31`), keeps `zhats, nus, lams, slacks`, and its backward first
rebuilds the factors with `pre_factor_kkt` (`qpth/qp.py:142-143`) and then runs the same factor + solve + outer
products as the PDIPM branch (`qpth/qp.py:148-182`).

Here the two halves are separate so that ANY solver can be the front end (warm-started loops, an external
commercial solver, a solution cached from a previous step):

* `QPSolutionFunction()(Q, p, G, h, A, b, zhat, lams, slacks, nus) -> zhat` is an autograd node whose backward is
  `qpb200_pre_factor_kkt` + `qpb200_backward` on the device: exactly the kernels of `QPFunction`'s backward, fed
  with the given primal/dual solution instead of the PDIPM iterate.  Gradient conventions are the reference's
  (batch mean for un-batched inputs, `dA = db = None` without equality constraints, symmetrised dQ); the four
  solution tensors receive no gradient.
* `cvxpy_forward(Q, p, G, h, A, b)` is the reference's CVXPY front end (needs the `cvxpy` package, which is not part
  of this image: it raises ImportError with that message otherwise), and `QPFunction(solver=QPSolvers.CVXPY)`
  chains the two, as `qpth/qp.py` does.

There is no CPU fallback for the backward: without the library or a CUDA device the call raises.
"""
import ctypes

import torch
from torch.autograd import Function

from . import _lib
from .qp import KKTSolvers, check_kkt_solver
from .util import expandParam, extract_nBatch


def pre_factor_state(Q_, p_, G_, h_, A_, b_, zhat, lams, slacks, nus, check_Q_spd=True,
                     kkt_solver=KKTSolvers.LU_PARTIAL):
    """`pre_factor_kkt` on the device + the given solution, packaged as the state `solve_backward` consumes.
    kkt_solver=KKTSolvers.IR_UNOPT: the regularised factors (`qpb200_pre_factor_kkt_reg`), so that the backward pass is
    `qpb200_backward_reg` and Q need only be positive semidefinite."""
    from . import kkt
    from .qp import SPD_ERR, SPD_ERR_REG, _Solved, _dev64, _ptr, _stream
    from .util import check_shapes
    nBatch, nz, nineq, neq = check_shapes(Q_, p_, G_, h_, A_, b_)
    assert neq > 0 or nineq > 0                         # qp.py:89
    if nineq == 0:
        raise RuntimeError('qpth_b200: nineq == 0 is not supported (the reference unpacks G.size() at qp.py:87)')
    lib = _lib.load()
    if not torch.cuda.is_available():
        raise _lib.QpthB200Error("qpth_b200: no CUDA device available (there is no CPU fallback).")
    device = Q_.device if Q_.is_cuda else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        Q, G = _dev64(Q_, device), _dev64(G_, device)
        A = _dev64(A_, device) if neq > 0 else None
        reg = kkt_solver == KKTSolvers.IR_UNOPT
        plan = _lib.plan_for_ir(nz, nineq, neq) if reg else _lib.plan_for(nz, nineq, neq)
        sQ = nz * nz if Q.dim() == 3 else 0
        sG = nineq * nz if G.dim() == 3 else 0
        sA = neq * nz if (A is not None and A.dim() == 3) else 0
        nsys = nBatch if (sQ or sG or sA) else 1
        st = _Solved()
        st.plan, st.nBatch, st.nsys, st.device, st.reg = plan, nBatch, nsys, device, reg
        f64 = dict(dtype=torch.float64, device=device)
        st.L = torch.empty(nsys * plan.L_elems, **f64)
        st.W = torch.empty(nsys * plan.W_elems, **f64)
        st.K = torch.empty(nsys * plan.K_elems, **f64)
        spd = torch.zeros(nsys, dtype=torch.int32, device=device)
        nscr = max(nsys * plan.setup_scratch_elems, nBatch * plan.solve_scratch_elems)
        st.scratch = torch.empty(nscr, **f64) if nscr > 0 else None
        if reg:
            _lib.check(lib.qpb200_pre_factor_kkt_reg(
                ctypes.byref(plan), nsys, _ptr(Q), sQ, _ptr(G), sG, _ptr(A), sA, float(kkt.IR_EPS),
                _ptr(st.L), _ptr(st.W), _ptr(st.K), _ptr(spd), _ptr(st.scratch), _stream()))
        else:
            _lib.check(lib.qpb200_pre_factor_kkt(
                ctypes.byref(plan), nsys, _ptr(Q), sQ, _ptr(G), sG, _ptr(A), sA,
                _ptr(st.L), _ptr(st.W), _ptr(st.K), _ptr(spd), _ptr(st.scratch), _stream()))
        if check_Q_spd and bool(spd.any()):
            raise RuntimeError(SPD_ERR_REG if reg else SPD_ERR)

        def sol(t, cols):
            t = t.detach().to(device=device, dtype=torch.float64)
            if t.dim() == 1:
                t = t.unsqueeze(0)
            if tuple(t.shape) != (nBatch, cols):
                raise RuntimeError("qpth_b200: solution tensor of shape %s, expected (%d, %d)"
                                   % (tuple(t.shape), nBatch, cols))
            return t.contiguous()

        st.zhat = sol(zhat, nz)
        st.lam = sol(lams, nineq)
        st.slacks = sol(slacks, nineq)
        st.nus = sol(nus, neq) if neq > 0 else None
        st.iters = torch.zeros(nBatch, dtype=torch.int32, device=device)
        st.best_resid = torch.zeros(nBatch, **f64)
        st.trace = None
    return st


def QPSolutionFunction(check_Q_spd=True, kkt_solver=KKTSolvers.LU_PARTIAL, duals=False):
    """Returns `f(Q, p, G, h, A, b, zhat, lams, slacks, nus) -> zhat`, differentiable in Q, p, G, h, A, b.

    duals=True: f returns (zhat, lam, nu), the given solution's duals as functions of Q, p, G, h, A, b (nu is (nBatch, 0)
    without equality rows), as QPFunction(duals=True) does; a loss may use all three.

    kkt_solver: KKTSolvers.LU_PARTIAL (the default) needs Q positive definite. KKTSolvers.IR_UNOPT differentiates with
    the regularised KKT solve of QPFunction(kkt_solver=IR_UNOPT), so an LP (Q = 0) or a low-rank Q solved by any solver
    can be differentiated; check_Q_spd then checks that Q is positive semidefinite."""
    check_kkt_solver(kkt_solver)

    class QPSolutionFn(Function):
        @staticmethod
        def forward(ctx, Q_, p_, G_, h_, A_, b_, zhat, lams, slacks, nus):
            ctx.st = pre_factor_state(Q_, p_, G_, h_, A_, b_, zhat, lams, slacks, nus, check_Q_spd, kkt_solver)
            zhats = ctx.st.zhat.to(device=Q_.device, dtype=Q_.dtype)
            ctx.save_for_backward(zhats, Q_, p_, G_, h_, A_, b_)
            ctx.lams, ctx.slacks, ctx.nus = ctx.st.lam, ctx.st.slacks, ctx.st.nus
            if not duals:
                return zhats
            from .qp import dual_outputs
            ctx.set_materialize_grads(False)
            return (zhats,) + dual_outputs(ctx.st, Q_)

        @staticmethod
        def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
            from .qp import solve_backward
            zhats, Q, p, G, h, A, b = ctx.saved_tensors
            nBatch = extract_nBatch(Q, p, G, h, A, b)
            flags = [expandParam(X, nBatch, nd)[1]
                     for X, nd in ((Q, 3), (p, 2), (G, 3), (h, 2), (A, 3), (b, 2))]   # qp.py:131-136
            want = list(ctx.needs_input_grad[:6])
            outs = solve_backward(ctx.st, dl_dzhat, flags, want, dl_dlam, dl_dnu)
            grads = [None if g is None else g.to(device=X.device, dtype=X.dtype)
                     for X, g in zip((Q, p, G, h, A, b), outs)]
            return tuple(grads) + (None, None, None, None)

    def apply(Q_, p_, G_, h_, A_, b_, zhat, lams, slacks, nus):
        # the solution is a constant of this node: detach it, or autograd would walk back into whatever produced it
        sol = [x.detach() if torch.is_tensor(x) else x for x in (zhat, lams, slacks, nus)]
        return QPSolutionFn.apply(Q_, p_, G_, h_, A_, b_, *sol)

    return apply


def cvxpy_forward(Q, p, G, h, A, b):
    """Per-sample CVXPY solve on the CPU (the front end of `qpth/qp.py:97-120`).

    Inputs are already expanded to the batch (as in the reference). Returns (zhats, nus, lams, slacks) as CPU
    fp64 tensors; nus is an empty tensor without equality constraints. Problem statement per sample
    (`qpth/solvers/cvxpy.py:5-31`): minimise 1/2 z'Qz + p'z subject to Az = b, Gz + s = h, s >= 0; the duals are
    those of the equality and of the `Gz + s = h` constraint.
    """
    try:
        import cvxpy as cp
    except ImportError as exc:       # cvxpy is not part of this image; the reference hard-requires it
        raise ImportError("QPSolvers.CVXPY needs the `cvxpy` package (not installed); use "
                          "QPSolvers.PDIPM_BATCHED, or solve elsewhere and call QPSolutionFunction") from exc
    import numpy as np
    nBatch, nz = p.shape[0], p.shape[1]
    nineq = G.shape[1]
    neq = A.shape[1] if (A is not None and A.nelement() > 0) else 0
    zhats = torch.empty(nBatch, nz, dtype=torch.float64)
    lams = torch.empty(nBatch, nineq, dtype=torch.float64)
    slacks = torch.empty(nBatch, nineq, dtype=torch.float64)
    nus = torch.empty(nBatch, neq, dtype=torch.float64) if neq > 0 else torch.Tensor()
    for i in range(nBatch):
        Qi, pi, Gi, hi = (x[i].detach().cpu().double().numpy() for x in (Q, p, G, h))
        z = cp.Variable(nz)
        s = cp.Variable(nineq)
        ineq = Gi @ z + s == hi
        cons = [ineq, s >= 0]
        eq = None
        if neq > 0:
            eq = A[i].detach().cpu().double().numpy() @ z == b[i].detach().cpu().double().numpy()
            cons.insert(0, eq)
        prob = cp.Problem(cp.Minimize(0.5 * cp.quad_form(z, Qi) + pi @ z), cons)
        prob.solve()
        assert 'optimal' in prob.status
        zhats[i] = torch.from_numpy(np.asarray(z.value).ravel())
        lams[i] = torch.from_numpy(np.asarray(ineq.dual_value).ravel())
        slacks[i] = torch.from_numpy(np.asarray(s.value).ravel())
        if neq > 0:
            nus[i] = torch.from_numpy(np.asarray(eq.dual_value).ravel())
    return zhats, nus, lams, slacks
