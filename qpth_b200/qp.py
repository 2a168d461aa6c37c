"""`QPFunction` — drop-in for `qpth.qp.QPFunction` backed by the sm_90a kernels.

Mirrors the reference's autograd boundary (`qpth/qp.py:18-183`): same factory
signature, same broadcasting of un-batched parameters (`qpth/util.py:44-59`),
same error strings, same gradient conventions (batch MEAN for un-batched
inputs, `dA = db = None` when there are no equality constraints, symmetrised
dQ).  The solver behind it is `libqpth_b200.so` (include/qpth_b200.h); there is
no CPU fallback — without the library or without a CUDA device the call raises.

Differences from the reference, all documented in DESIGN.md:
  * every QP is solved with the reference's nBatch=1 semantics (the batch-global
    exit tests and get_step fill value are applied per QP);
  * arithmetic is fp64 on the device whatever the input dtype (fp32 inputs are
    promoted and the results cast back);
  * CPU tensors are accepted: they are copied to the current CUDA device,
    solved there, and the results returned on the CPU;
  * `solver=QPSolvers.CVXPY` (qp.py:97-120) needs the `cvxpy` package for its forward; its backward, and the
    stand-alone `QPSolutionFunction` for solutions produced by any other solver, live in `solution.py`.
"""
import ctypes
from enum import Enum

import torch
from torch.autograd import Function

from . import _lib, kkt
from .util import check_shapes, expandParam, extract_nBatch

INACC_ERR = """
--------
qpth warning: Returning an inaccurate and potentially incorrect solution.

Some residual is large.
Your problem may be infeasible or difficult.

You can try using the CVXPY solver to see if your problem is feasible
and you can use the verbose option to check the convergence status of
our solver while increasing the number of iterations.

Advanced users:
You can also try to enable iterative refinement in the solver:
https://github.com/locuslab/qpth/issues/6
--------
"""


# The reference stops a batch when NO QP improved for `notImprovedLim` consecutive iterations
# (batch.py:127-143).  Applied per QP that rule would abandon QPs that merely pause while still far from
# a solution (resids is not monotone early on); it is therefore only applied once a QP's best residual
# is below STALL_TOL, i.e. when it is stalling at its rounding floor like the rest of its batch would.
STALL_TOL = 1e-6
# The reference returns the argmin-resids iterate (batch.py:126-139).  At the rounding floor successive
# iterates tie to within noise while mu still shrinks ~1000x per iteration, and which one wins decides
# whether the backward pass's 1e-8 clamps (qp.py:148) are saturated.  Among iterates within BEST_TIE of
# the minimum the latest is returned (1.0 restores the literal rule).
BEST_TIE = 1.5
TRACE = False     # keep per-iteration residual traces on st.trace even when verbose != 1 (diagnostics)
# Kernel choice where a shape has several product-form variants (plan.pf2_ok / plan.pf3_ok, e.g. nz = nineq = 100):
#   "latency"    one QP per SM, W / chol(Q) / factor in shared memory: the shortest time for ONE batch <= #SMs;
#   "throughput" three (else two) QPs per SM, W and chol(Q) read from L2: +33 % QPs/s once the GPU is full (a large
#                batch, or several batches in flight on several streams; bench.py at C2 on an H100 SXM, 700 W),
#                but a higher latency for a lone 128-QP batch;
#   "auto"       throughput when the batch alone exceeds the SM count, else latency.
# Set qpth_b200.qp.MODE (or QPTH_B200_MODE) before the call. The variants differ only in the summation order of the
# W / chol(Q) passes: results agree to ~1e-12 relative (tests/test_gpu_parity.py pins 1e-10), not bit for bit.
import os as _os
MODE = _os.environ.get("QPTH_B200_MODE", "auto")
# The reference's DEFAULT options (check_Q_spd=True, verbose=0) make every forward read two flags back from the device
# before it returns ('Q is not SPD.' qp.py:81-85; the inaccurate-solution banner batch.py:205-206): one blocking host
# read per call, which caps a training loop at ~67k QPs/s on an H100 SXM (bench.py e2e.default_options at C2)
# where the asynchronous options reach 198k. LAZY_CHECKS = True keeps the diagnostics but DEFERS them: the flags are
# copied to pinned host memory asynchronously and examined at the next QPFunction call, in backward, or by
# flush_checks() - the error / banner then refers to an EARLIER call. Off by default: the reference raises at once.
LAZY_CHECKS = _os.environ.get("QPTH_B200_LAZY_CHECKS", "0") == "1"
_pending = []
import threading as _threading
_pending_lock = _threading.Lock()      # forward runs on the caller's thread, backward on the autograd engine's


def flush_checks(wait=True):
    """Examine the deferred diagnostics (LAZY_CHECKS) of earlier forward calls; wait=False only those already on the host."""
    while True:
        with _pending_lock:
            if not _pending:
                return
            ev, host, chk, banner = _pending[0]
            if not wait and not ev.query():
                return
            _pending.pop(0)
        ev.synchronize()
        bad_spd, inacc = host.tolist()
        if banner and inacc:
            print(INACC_ERR)
        if chk and bad_spd:
            raise RuntimeError(chk + ' (reported by a deferred check, qpth_b200.qp.LAZY_CHECKS)')


class QPSolvers(Enum):
    PDIPM_BATCHED = 1
    CVXPY = 2


class KKTSolvers(Enum):
    """The reference's KKT solver choice (batch.py:41-44). LU_PARTIAL: the default path (Q positive definite).
    IR_UNOPT: the regularised mode, for Q only positive semidefinite (LPs, low-rank quadratic terms) or linearly dependent
    equality rows: every KKT solve factors the system regularised with kkt.IR_EPS and the Newton loop uses the residuals
    of the true problem. LU_FULL is not provided."""
    LU_FULL = 1
    LU_PARTIAL = 2
    IR_UNOPT = 3


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None and t.numel() > 0 else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev64(t, device):
    """fp64, contiguous, on `device`; un-batched tensors stay un-batched (stride 0 is passed to C)."""
    return t.detach().to(device=device, dtype=torch.float64).contiguous()


class _Solved:
    """State carried from forward to backward (the reference's ctx.Q_LU / S_LU / R / nus / lams / slacks)."""
    __slots__ = ("plan", "nBatch", "nsys", "L", "W", "K", "zhat", "lam", "slacks", "nus",
                 "iters", "best_resid", "scratch", "device", "trace", "reg")


def solve_forward(Q_, p_, G_, h_, A_, b_, eps=1e-12, verbose=0, notImprovedLim=3, maxIter=20,
                  check_Q_spd=True, kkt_solver=KKTSolvers.LU_PARTIAL):
    """pre_factor_kkt + forward on the device. Inputs follow QPFunction's conventions. Returns _Solved."""
    # rank errors exactly as expandParam raises them (util.py:44-50), then every trailing dimension / batch size:
    # pure host logic, done before anything touches the device
    nBatch, nz, nineq, neq = check_shapes(Q_, p_, G_, h_, A_, b_)
    if _pending:
        flush_checks(wait=False)
    assert neq > 0 or nineq > 0                         # qp.py:89
    if nineq == 0:
        raise RuntimeError('qpth_b200: nineq == 0 is not supported (the reference unpacks G.size() at qp.py:87)')
    assert maxIter >= 1
    lib = _lib.load()
    if not torch.cuda.is_available():
        raise _lib.QpthB200Error("qpth_b200: no CUDA device available (there is no CPU fallback).")
    device = Q_.device if Q_.is_cuda else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        Q, p, G, h = (_dev64(t, device) for t in (Q_, p_, G_, h_))
        A = _dev64(A_, device) if neq > 0 else None
        b = _dev64(b_, device) if neq > 0 else None
        # one QP per SM (W, chol(Q) and the factor all in shared memory) has the lower latency; two QPs per SM (W and
        # chol(Q) read from L2) the higher throughput once more QPs are in flight than the GPU has SMs (MODE above)
        reg = kkt_solver == KKTSolvers.IR_UNOPT
        if reg:                      # one QP per SM, 256 threads: the only builds of the regularised kernels (MODE ignored)
            plan = _lib.plan_for_ir(nz, nineq, neq)
        else:
            two = MODE == "throughput" or (MODE == "auto" and nBatch > _lib.sm_count(device.index or 0))
            plan = _lib.plan_for(nz, nineq, neq, two=two)

        def stride(t, nd, per):
            return per if (t is not None and t.dim() == nd) else 0

        sQ, sG = stride(Q, 3, nz * nz), stride(G, 3, nineq * nz)
        sA = stride(A, 3, neq * nz)
        sp, sh, sb = stride(p, 2, nz), stride(h, 2, nineq), stride(b, 2, neq)
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
        st.zhat = torch.empty(nBatch, nz, **f64)
        st.lam = torch.empty(nBatch, nineq, **f64)
        st.slacks = torch.empty(nBatch, nineq, **f64)
        st.nus = torch.empty(nBatch, neq, **f64) if neq > 0 else None
        st.iters = torch.empty(nBatch, dtype=torch.int32, device=device)
        st.best_resid = torch.empty(nBatch, **f64)
        st.trace = torch.full((nBatch, int(maxIter), 4), float('nan'), **f64) if (verbose == 1 or TRACE) else None
        common = (float(eps), float(STALL_TOL), float(BEST_TIE), int(notImprovedLim), int(maxIter))
        if reg:
            common += (float(kkt.IR_EPS), int(kkt.IR_STEPS))
        _lib.check((lib.qpb200_forward_reg if reg else lib.qpb200_forward)(
            ctypes.byref(plan), nBatch, _ptr(p), sp, _ptr(h), sh, _ptr(b), sb,
            _ptr(st.L), _ptr(st.W), _ptr(st.K), 1 if nsys > 1 else 0, *common,
            _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus),
            _ptr(st.iters), _ptr(st.best_resid), _ptr(st.trace), _ptr(st.scratch), _stream()))
        diagnostics(spd, st, check_Q_spd, verbose, SPD_ERR_REG if reg else SPD_ERR)
    return st


SPD_ERR = 'Q is not SPD.'
# the regularised mode factors Q + IR_EPS I: a failed pivot means an eigenvalue of Q below -IR_EPS
SPD_ERR_REG = 'Q is not positive semidefinite.'


def diagnostics(spd, st, check_Q_spd, verbose, spd_err=SPD_ERR):
    """After a forward: 'Q is not SPD.' from the device flags `spd`, the inaccurate-solution banner from st.best_resid,
    and at verbose == 1 the per-iteration lines from st.trace / st.iters."""
    # One host read for both diagnostics (the reference syncs many times per iteration):
    # 'Q is not SPD.' (qp.py:81-85) and the inaccurate-solution banner, printed iff
    # best resids max > 1 and verbose >= 0 (batch.py:141-142,205-206).
    if check_Q_spd or verbose >= 0:
        flags = torch.stack([spd.any(), (st.best_resid.max() > 1.)])
        if LAZY_CHECKS:
            # the two flags travel to a pinned host buffer asynchronously; they are examined (and 'Q is not SPD.' raised,
            # the banner printed) at the next QPFunction call, in this call's backward, or by flush_checks()
            host = torch.empty(2, dtype=flags.dtype).pin_memory()
            host.copy_(flags, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            _pending.append((ev, host, spd_err if check_Q_spd else None, verbose >= 0))
        else:
            bad_spd, inacc = flags.tolist()
            if check_Q_spd and bad_spd:
                raise RuntimeError(spd_err)
            if verbose >= 0 and inacc:
                print(INACC_ERR)
    if verbose == 1:
        # batch.py:115-117: per-iteration batch means; a QP that has already stopped contributes
        # the values of its last iteration (in the reference every QP runs every iteration)
        nBatch = st.iters.shape[0]
        tr = st.trace.cpu()
        for i in range(int(st.iters.max())):
            row = tr[:, i, :]
            last = tr[torch.arange(nBatch), (st.iters.cpu().long() - 1).clamp(min=0), :]
            row = torch.where(torch.isnan(row), last, row)
            print('iter: {}, pri_resid: {:.5e}, dual_resid: {:.5e}, mu: {:.5e}'.format(
                i, row[:, 0].mean(), row[:, 1].mean(), row[:, 2].mean()))


def _adjoint(g, B, n, device):
    """An incoming gradient as a (B, n) fp64 device tensor; None (no gradient reached this output) stays None."""
    if g is None or n == 0:
        return None
    return g.detach().to(device=device, dtype=torch.float64).contiguous().view(B, n)


def dual_outputs(st, like):
    """(lam, nu) of the returned iterate with the dtype and device of `like`; nu is (nBatch, 0) without equality rows."""
    lam = st.lam.to(device=like.device, dtype=like.dtype)
    nu = (st.nus.to(device=like.device, dtype=like.dtype) if st.nus is not None
          else torch.zeros(st.nBatch, 0, device=like.device, dtype=like.dtype))
    return lam, nu


def solve_backward(st, dl_dzhat, mean_flags, want, dl_dlam=None, dl_dnu=None):
    """QPFunctionFn.backward on the device. mean_flags / want: 6-tuples for (Q,p,G,h,A,b). dl_dlam / dl_dnu: the
    gradients of the loss with respect to the returned duals (None: zero); dl_dzhat None: zero."""
    if _pending:
        flush_checks(wait=False)
    lib = _lib.load()
    plan, B, device = st.plan, st.nBatch, st.device
    nz, nineq, neq = plan.nz, plan.nineq, plan.neq
    f64 = dict(dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        dl = _adjoint(dl_dzhat, B, nz, device) if dl_dzhat is not None else torch.zeros(B, nz, **f64)
        glam, gnu = _adjoint(dl_dlam, B, nineq, device), _adjoint(dl_dnu, B, neq, device)
        shapes = [(nz, nz), (nz,), (nineq, nz), (nineq,), (neq, nz), (neq,)]
        outs = []
        for k in range(6):
            if not want[k] or (k >= 4 and neq == 0):
                outs.append(None)
            else:
                shp = shapes[k] if mean_flags[k] else (B,) + shapes[k]
                outs.append(torch.empty(*shp, **f64))
        dxv = torch.empty(B, nz, **f64)
        dlamv = torch.empty(B, nineq, **f64)
        dnuv = torch.empty(B, neq, **f64) if neq > 0 else None
        args = []
        for k in range(6):
            args += [_ptr(outs[k]), 1 if mean_flags[k] else 0]
        reg = getattr(st, "reg", False)             # (solution.py builds _Solved without it: the default path)
        if glam is None and gnu is None:            # no dual was used: the entry point of a zhat-only loss
            fn, adj = (lib.qpb200_backward_reg if reg else lib.qpb200_backward), ()
        else:
            fn, adj = (lib.qpb200_backward_reg_duals if reg else lib.qpb200_backward_duals), (_ptr(glam), _ptr(gnu))
        _lib.check(fn(
            ctypes.byref(plan), B, _ptr(dl), *adj, _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus),
            _ptr(st.L), _ptr(st.W), _ptr(st.K), 1 if st.nsys > 1 else 0, *((float(kkt.IR_EPS), int(kkt.IR_STEPS)) if reg else ()),
            *args, _ptr(dxv), _ptr(dlamv), _ptr(dnuv), _ptr(st.scratch), _stream()))
    return outs


def check_kkt_solver(kkt_solver):
    if kkt_solver == KKTSolvers.LU_FULL:
        raise ValueError("qpth_b200: KKTSolvers.LU_FULL is not provided; use KKTSolvers.LU_PARTIAL (Q positive definite) "
                         "or KKTSolvers.IR_UNOPT (Q positive semidefinite, linearly dependent equality rows)")
    if kkt_solver not in (KKTSolvers.LU_PARTIAL, KKTSolvers.IR_UNOPT):
        raise ValueError("qpth_b200: unknown kkt_solver %r" % (kkt_solver,))


def QPFunction(eps=1e-12, verbose=0, notImprovedLim=3, maxIter=20, solver=QPSolvers.PDIPM_BATCHED,
               check_Q_spd=True, kkt_solver=KKTSolvers.LU_PARTIAL, duals=False):
    """Factory with the reference's signature (`qpth/qp.py:18-20`); returns `Function.apply`.

    duals (an extension): False returns zhat (nBatch, nz), as the reference does. True returns (zhat, lam, nu): the
    inequality duals (nBatch, nineq) and the equality duals (nBatch, neq), or (nBatch, 0) without equality rows, of the
    returned iterate (the values of last_solve(), with zhat's dtype and device), and a loss may use all three: the
    backward pass puts the gradients of lam and nu into the right-hand side of its KKT solve,
    [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dlam dnu] = -[dl/dz; 0; dl/dlam; dl/dnu], and the gradient formulas
    are unchanged. With linearly dependent equality rows (IR_UNOPT) nu is not unique, and the gradient through nu is
    that of the nu returned. Slacks are not an output: s = h - Gz.

    kkt_solver (an extension of the reference's signature): KKTSolvers.LU_PARTIAL, the default, needs Q positive definite.
    KKTSolvers.IR_UNOPT also solves QPs whose Q is only positive semidefinite (LPs with Q = 0, low-rank quadratic terms)
    and QPs whose equality rows are linearly dependent: every KKT solve factors the system regularised with kkt.IR_EPS
    (chol(Q + eps I); eps on the constraint blocks) and refines it kkt.IR_STEPS times, while the residuals are those of
    the true problem, so the returned point is the exact KKT point. check_Q_spd then checks that Q is positive
    SEMIdefinite ('Q is not positive semidefinite.'). IR_UNOPT takes every shape the default mode takes with
    nineq >= 1: up to ms_pad = 8 ceil(neq / 8) + nineq rounded up to 8 of about 200 on the product-form kernels, beyond
    that on the generic global-scratch kernels. With linearly dependent equality rows the equality duals, and so the
    gradients dA and db, are not unique; z*, the inequality duals, the slacks and dQ, dp, dG, dh are. An unbounded or
    infeasible problem gives the inaccurate-solution banner, as in the default mode."""
    check_kkt_solver(kkt_solver)
    if solver == QPSolvers.CVXPY:
        # qp.py:97-120,142-143: per-sample CVXPY solve on the CPU, then pre_factor_kkt + the same backward.
        from .solution import QPSolutionFunction, cvxpy_forward

        def apply_cvxpy(Q_, p_, G_, h_, A_, b_):
            nBatch = extract_nBatch(Q_, p_, G_, h_, A_, b_)
            Q, p, G, h, A, b = (expandParam(X, nBatch, nd)[0]
                                for X, nd in ((Q_, 3), (p_, 2), (G_, 3), (h_, 2), (A_, 3), (b_, 2)))
            zhats, nus, lams, slacks = cvxpy_forward(Q, p, G, h, A, b)
            f = QPSolutionFunction(check_Q_spd, kkt_solver, duals=True) if duals else QPSolutionFunction(check_Q_spd,
                                                                                                          kkt_solver)
            return f(Q_, p_, G_, h_, A_, b_, zhats, lams, slacks, nus)

        return apply_cvxpy
    if solver != QPSolvers.PDIPM_BATCHED:
        assert False                                     # qp.py:121-122

    _last = [None]

    class QPFunctionFn(Function):
        @staticmethod
        def forward(ctx, Q_, p_, G_, h_, A_, b_):
            """Solve a batch of QPs  argmin_z 1/2 z^T Q z + p^T z  s.t. Gz <= h, Az = b.

            Q (nBatch,nz,nz)|(nz,nz); p (nBatch,nz)|(nz); G (nBatch,nineq,nz)|(nineq,nz);
            h (nBatch,nineq)|(nineq); A (nBatch,neq,nz)|(neq,nz)|empty; b (nBatch,neq)|(neq)|empty.
            Returns zhat (nBatch, nz).  (qp.py:23-125)
            """
            st = solve_forward(Q_, p_, G_, h_, A_, b_, eps, verbose, notImprovedLim, maxIter, check_Q_spd, kkt_solver)
            ctx.st = st
            _last[0] = st
            ctx.neq, ctx.nineq, ctx.nz = st.plan.neq, st.plan.nineq, st.plan.nz
            zhats = st.zhat.to(device=Q_.device, dtype=Q_.dtype)
            ctx.save_for_backward(zhats, Q_, p_, G_, h_, A_, b_)
            # parity with the reference's ctx attributes (device fp64 views)
            ctx.lams, ctx.slacks, ctx.nus = st.lam, st.slacks, st.nus
            if not duals:
                return zhats
            ctx.set_materialize_grads(False)       # an unused output's gradient arrives as None: no adjoint is read
            return (zhats,) + dual_outputs(st, Q_)

        @staticmethod
        def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
            zhats, Q, p, G, h, A, b = ctx.saved_tensors
            nBatch = extract_nBatch(Q, p, G, h, A, b)
            flags = [expandParam(X, nBatch, nd)[1]
                     for X, nd in ((Q, 3), (p, 2), (G, 3), (h, 2), (A, 3), (b, 2))]   # qp.py:131-136
            want = list(ctx.needs_input_grad)
            outs = solve_backward(ctx.st, dl_dzhat, flags, want, dl_dlam, dl_dnu)
            grads = []
            for X, g in zip((Q, p, G, h, A, b), outs):
                grads.append(None if g is None else g.to(device=X.device, dtype=X.dtype))
            return tuple(grads)

    def apply(Q_, p_, G_, h_, A_, b_):
        if G_.nelement() == 0 and h_.nelement() == 0 and A_.nelement() > 0:
            # equality-constrained QP: an extension (the reference cannot run nineq == 0); one KKT solve, eqonly.py
            from .eqonly import solve_equality_qp
            return solve_equality_qp(Q_, p_, A_, b_, check_Q_spd, reg=kkt_solver == KKTSolvers.IR_UNOPT, duals=duals)
        return QPFunctionFn.apply(Q_, p_, G_, h_, A_, b_)

    # diagnostics the reference keeps on ctx (nus / lams / slacks) plus per-QP iteration counts
    apply.last_solve = lambda: _last[0]
    return apply
