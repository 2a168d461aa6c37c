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
from ._lib import dev64 as _dev64, ptr as _ptr, stream as _stream
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
    _lib.load()
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
        st.L, st.W, st.K, st.scratch, spd = _lib.pre_factor(plan, nsys, nBatch, Q, sQ, G, sG, A, sA,
                                                             kkt.IR_EPS if reg else None, device, _stream())
        f64 = dict(dtype=torch.float64, device=device)
        st.zhat = torch.empty(nBatch, nz, **f64)
        st.lam = torch.empty(nBatch, nineq, **f64)
        st.slacks = torch.empty(nBatch, nineq, **f64)
        st.nus = torch.empty(nBatch, neq, **f64) if neq > 0 else None
        st.iters = torch.empty(nBatch, dtype=torch.int32, device=device)
        st.best_resid = torch.empty(nBatch, **f64)
        st.trace = torch.full((nBatch, int(maxIter), 4), float('nan'), **f64) if (verbose == 1 or TRACE) else None
        fn, ir = _entry(st, "qpb200_forward", "qpb200_forward_reg")
        _lib.check(fn(
            ctypes.byref(plan), nBatch, _ptr(p), sp, _ptr(h), sh, _ptr(b), sb,
            _ptr(st.L), _ptr(st.W), _ptr(st.K), 1 if nsys > 1 else 0,
            float(eps), float(STALL_TOL), float(BEST_TIE), int(notImprovedLim), int(maxIter), *ir,
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


# ---- pieces of the device wrappers of QPFunction and BoxQPFunction ---------------------------------------------------
def grad_buffers(shapes, flags, want, absent, B, device, order=range(6)):
    """The six input gradients a backward writes: None where not wanted or absent, else fp64 of the input's shape, with
    a batch dimension unless its mean flag is set (an un-batched input). Returns them and the flat (pointer, mean flag)
    argument list of the C ABI in `order`."""
    outs = [None if (not w or a) else torch.empty(*(s if f else (B,) + s), dtype=torch.float64, device=device)
            for s, f, w, a in zip(shapes, flags, want, absent)]
    args = []
    for k in order:
        args += [_ptr(outs[k]), 1 if flags[k] else 0]
    return outs, args


def tangent_args(tangents, ranks, per):
    """Input tangents (fp64 device tensors, which the caller keeps alive) as the flat (pointer, batch stride) argument
    list of the C ABI: None (no tangent) is NULL with stride 0, an un-batched tangent (rank - 1 dimensions) gets stride
    0, a batched one `per` elements."""
    args = []
    for t, r, n in zip(tangents, ranks, per):
        if t is None or t.numel() == 0 or n == 0:
            args += [_ptr(None), 0]
        else:
            args += [_ptr(t), n if t.dim() == r else 0]
    return args


def solve_triple(B, nz, nineq, neq, device):
    """Fresh fp64 (B, nz), (B, nineq) and (B, neq) outputs of a KKT solve; the last is None without equality rows."""
    f64 = dict(dtype=torch.float64, device=device)
    return torch.empty(B, nz, **f64), torch.empty(B, nineq, **f64), torch.empty(B, neq, **f64) if neq > 0 else None


def _entry(st, plain, reg):
    """The C entry point for the mode of `st` and the arguments that follow its nsys flag: `reg` with
    (IR_EPS, IR_STEPS) in the regularised mode (IR_UNOPT), else `plain` and none."""
    lib = _lib.load()
    if getattr(st, "reg", False):                   # (states built outside solve_forward may lack it: the default path)
        return getattr(lib, reg), (float(kkt.IR_EPS), int(kkt.IR_STEPS))
    return getattr(lib, plain), ()


def _point(st):
    """The arguments of the returned point and its factors: zhat, lam, slacks, nus, L, W, K and the nsys flag."""
    return (_ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(st.L), _ptr(st.W), _ptr(st.K),
            1 if st.nsys > 1 else 0)


def _shapes(plan):
    return [(plan.nz, plan.nz), (plan.nz,), (plan.nineq, plan.nz), (plan.nineq,), (plan.neq, plan.nz), (plan.neq,)]


RANKS = (3, 2, 3, 2, 3, 2)        # of (Q, p, G, h, A, b) batched


def solve_backward(st, dl_dzhat, mean_flags, want, dl_dlam=None, dl_dnu=None, keep=False):
    """QPFunctionFn.backward on the device. mean_flags / want: 6-tuples for (Q,p,G,h,A,b). dl_dlam / dl_dnu: the
    gradients of the loss with respect to the returned duals (None: zero); dl_dzhat None: zero. keep: also return the
    solve (dxv, dlamv, dnuv), which the double backward reads."""
    if _pending:
        flush_checks(wait=False)
    plan, B, device = st.plan, st.nBatch, st.device
    nz, nineq, neq = plan.nz, plan.nineq, plan.neq
    with torch.cuda.device(device):
        dl = (_adjoint(dl_dzhat, B, nz, device) if dl_dzhat is not None
              else torch.zeros(B, nz, dtype=torch.float64, device=device))
        glam, gnu = _adjoint(dl_dlam, B, nineq, device), _adjoint(dl_dnu, B, neq, device)
        outs, grads = grad_buffers(_shapes(plan), mean_flags, want, (False,) * 4 + (neq == 0,) * 2, B, device)
        v = solve_triple(B, nz, nineq, neq, device)
        if glam is None and gnu is None:            # no dual was used: the entry point of a zhat-only loss
            (fn, ir), adj = _entry(st, "qpb200_backward", "qpb200_backward_reg"), ()
        else:
            (fn, ir), adj = _entry(st, "qpb200_backward_duals", "qpb200_backward_reg_duals"), (_ptr(glam), _ptr(gnu))
        _lib.check(fn(ctypes.byref(plan), B, _ptr(dl), *adj, *_point(st), *ir, *grads, *(_ptr(x) for x in v),
                      _ptr(st.scratch), _stream()))
    return (outs, v) if keep else outs


def solve_double_backward(st, v, omegas, flags, want, G):
    """The double backward on the device (qpb200_double_backward(_reg)): v = (dxv, dlamv, dnuv) of the first backward at
    the point of `st`; omegas: the cotangents of its six outputs (Q, p, G, h, A, b), each None or shaped as that output;
    flags: the first backward's mean flags (an un-batched input: its cotangent is divided by nBatch, and its second-order
    gradient is the batch sum); want: which of the six gradients to write; G: the forward's G. Returns fp64
    (gg_z, gg_lam, gg_nu, dQ, dp, dG, dh, dA, db): the gradients of g_z, g_lam, g_nu (gg_nu None without equality rows)
    and of the six inputs (None where not wanted)."""
    if _pending:
        flush_checks(wait=False)
    plan, B, device = st.plan, st.nBatch, st.device
    nz, nineq, neq = plan.nz, plan.nineq, plan.neq
    absent = (False,) * 4 + (neq == 0,) * 2
    with torch.cuda.device(device):
        om = [None if (w is None or absent[k]) else (_dev64(w, device) / B if flags[k] else _dev64(w, device))
              for k, w in enumerate(omegas)]
        tans = tangent_args(om, RANKS, (nz * nz, nz, nineq * nz, nineq, neq * nz, neq))
        G64 = _dev64(G, device)
        sG = nineq * nz if G64.dim() == 3 else 0
        outs, grads = grad_buffers(_shapes(plan), flags, want, absent, B, device)
        gg = solve_triple(B, nz, nineq, neq, device)
        work = torch.empty(B * (2 * nz + 3 * nineq + 2 * neq), dtype=torch.float64, device=device)
        fn, ir = _entry(st, "qpb200_double_backward", "qpb200_double_backward_reg")
        _lib.check(fn(ctypes.byref(plan), B, *tans, _ptr(G64), sG, *(_ptr(x) for x in v), *_point(st), *ir,
                      *(_ptr(x) for x in gg), *grads, _ptr(work), _ptr(st.scratch), _stream()))
    return list(gg) + outs


THIRD_ORDER_ERR = ("qpth_b200: third-order derivatives through the QP layer are not provided: the double backward is not "
                   "differentiable (call the second torch.autograd.grad without create_graph=True)")


def _cast(g, like):
    return None if (g is None or like is None) else g.to(device=like.device, dtype=like.dtype)


class BackwardFn(Function):
    """The first-order backward of a QP layer as a differentiable function of the incoming gradients (g_z, g_lam, g_nu)
    and of the layer's six inputs: what its backward runs under create_graph=True. Its forward is
    first(st, g_z, flags, want, g_lam, g_nu), the layer's first-order backward returning (grads, v); its backward is
    second(st, v, omegas, flags, want), the layer's double backward."""
    @staticmethod
    def forward(ctx, first, second, st, flags, want, g_z, g_lam, g_nu, *ins):
        outs, v = first(st, g_z, flags, want, g_lam, g_nu)
        ctx.second, ctx.st, ctx.v, ctx.flags = second, st, v, flags
        ctx.like = (g_z, g_lam, g_nu) + ins
        ctx.set_materialize_grads(False)
        return tuple(_cast(g, X) for X, g in zip(ins, outs))

    @staticmethod
    def backward(ctx, *omegas):
        if torch.is_grad_enabled():
            raise RuntimeError(THIRD_ORDER_ERR)
        need = ctx.needs_input_grad[5:]
        if all(w is None for w in omegas) or not any(need):
            return (None,) * 14
        res = ctx.second(ctx.st, ctx.v, omegas, ctx.flags, need[3:])
        return (None,) * 5 + tuple(_cast(g, X) if n else None for g, X, n in zip(res, ctx.like, need))


def backward_graph(st, flags, want, g_z, g_lam, g_nu, Q, p, G, h, A, b):
    """solve_backward under create_graph=True: gradients of (Q, p, G, h, A, b) that can be differentiated again."""
    return BackwardFn.apply(lambda *a: solve_backward(*a, keep=True),
                            lambda st_, v, om, fl, w: solve_double_backward(st_, v, om, fl, w, G),
                            st, flags, want, g_z, g_lam, g_nu, Q, p, G, h, A, b)


def solve_jvp(st, tangents):
    """The JVP of (zhat, lam, nu) at the returned point on the device. tangents: (dQ, dp, dG, dh, dA, db), each None
    (zero), batched or un-batched as its input. Returns fp64 (dz (B,nz), dlam (B,nineq), dnu (B,neq) or None); one
    qpb200_jvp(_reg) call: the right-hand side kernel and the backward's KKT solve."""
    if _pending:
        flush_checks(wait=False)
    plan, B, device = st.plan, st.nBatch, st.device
    nz, nineq, neq = plan.nz, plan.nineq, plan.neq
    with torch.cuda.device(device):
        tans = [None if t is None else _dev64(t, device) for t in tangents]
        args = tangent_args(tans, RANKS, (nz * nz, nz, nineq * nz, nineq, neq * nz, neq))
        rhs = torch.empty(B * (nz + nineq + neq), dtype=torch.float64, device=device)
        dz, dlam, dnu = solve_triple(B, nz, nineq, neq, device)
        fn, ir = _entry(st, "qpb200_jvp", "qpb200_jvp_reg")
        _lib.check(fn(ctypes.byref(plan), B, *args, *_point(st), *ir, _ptr(rhs), _ptr(dz), _ptr(dlam), _ptr(dnu),
                      _ptr(st.scratch), _stream()))
    return dz, dlam, dnu


def jvp_outputs(dz, dlam, dnu, out, duals):
    """The output tangents of a Function whose outputs have out = (device, dtype): dz, or (dz, dlam, dnu) with duals
    (dnu (B, 0) without equality rows). Every output gets a tensor: forward AD does not take None for an output of
    these Functions."""
    device, dtype = out
    z = dz.to(device=device, dtype=dtype)
    if not duals:
        return z
    nu = (dnu.to(device=device, dtype=dtype) if dnu is not None
          else torch.zeros(dz.shape[0], 0, device=device, dtype=dtype))
    return z, dlam.to(device=device, dtype=dtype), nu


def layer_outputs(ctx, st, ins, duals):
    """The end of a QP layer's forward: keep `st` and the inputs for backward and jvp, and return zhat, or (zhat, lam,
    nu) with duals, with the dtype and device of the first input."""
    X = ins[0]
    ctx.st, ctx.duals = st, duals
    zhats = st.zhat.to(device=X.device, dtype=X.dtype)
    ctx.save_for_backward(zhats, *ins)
    # parity with the reference's ctx attributes (device fp64 views)
    ctx.lams, ctx.slacks, ctx.nus = st.lam, st.slacks, st.nus
    ctx.out = (X.device, X.dtype)
    # an unused output's gradient, and an input without a tangent, arrive as None: nothing zero-filled is read
    ctx.set_materialize_grads(False)
    return (zhats,) + dual_outputs(st, X) if duals else zhats


class QPLayerFn(Function):
    """backward and jvp of QPFunction and QPSolutionFunction, whose forward(ctx, Q, p, G, h, A, b, ...) ends with
    layer_outputs; inputs after the sixth (QPSolutionFunction's solution) are constants."""
    @staticmethod
    def jvp(ctx, *tangents):
        return jvp_outputs(*solve_jvp(ctx.st, tangents[:6]), ctx.out, ctx.duals)

    @staticmethod
    def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
        zhats, Q, p, G, h, A, b = ctx.saved_tensors
        nBatch = extract_nBatch(Q, p, G, h, A, b)
        flags = [expandParam(X, nBatch, nd)[1]
                 for X, nd in ((Q, 3), (p, 2), (G, 3), (h, 2), (A, 3), (b, 2))]   # qp.py:131-136
        want = list(ctx.needs_input_grad[:6])
        if torch.is_grad_enabled():          # create_graph=True: gradients that can be differentiated again
            grads = backward_graph(ctx.st, flags, want, dl_dzhat, dl_dlam, dl_dnu, Q, p, G, h, A, b)
        else:
            outs = solve_backward(ctx.st, dl_dzhat, flags, want, dl_dlam, dl_dnu)
            grads = tuple(_cast(g, X) for X, g in zip((Q, p, G, h, A, b), outs))
        return grads + (None,) * (len(ctx.needs_input_grad) - 6)


# ---- Jacobians: rows z, lam, nu as bits 0, 1, 2; columns one bit per input of the layer's table ---------------------
JAC_WRT = ("p", "h", "b")
JAC_SLOTS = (1, 3, 5)             # their tangents' slots in (dQ, dp, dG, dh, dA, db)


def jacobian_covered(plan):
    """True where qpb200_jacobian covers `plan` (qpb200_jacobian_smem reports its shared memory)."""
    out = ctypes.c_int64(0)
    _lib.check(_lib.load().qpb200_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)))
    return out.value > 0


def _jacobian_kernel(st, rows, cols, J):
    """qpb200_jacobian into J (B, R, C) fp64 on st.device."""
    with torch.cuda.device(st.device):
        _lib.check(_lib.load().qpb200_jacobian(
            ctypes.byref(st.plan), st.nBatch, rows, cols, _ptr(st.lam), _ptr(st.slacks), _ptr(st.L), _ptr(st.W),
            1 if st.nsys > 1 else 0, _ptr(J), _stream()))


def jacobian_columns(st, rows, cols, J, csizes, slots, jvp):
    """J column by column: for column block k (csizes[k] columns), one jvp(st, tangents) per column with an un-batched
    unit tangent (batch stride 0) in slot slots[k] of the six tangents, which gives that column for every QP at once
    (qpb200_jvp, or qpb200_jvp_reg with its refinement steps; the box layouts' JVPs)."""
    rsizes = (st.plan.nz, st.plan.nineq, st.plan.neq)
    c0 = 0
    for k, (n, slot) in enumerate(zip(csizes, slots)):
        if not (cols >> k) & 1:
            continue
        for j in range(n):
            t = torch.zeros(n, dtype=torch.float64, device=st.device)
            t[j] = 1.0
            tans = [None] * 6
            tans[slot] = t
            outs = jvp(st, tans)
            r0 = 0
            for i in range(3):
                if (rows >> i) & 1:
                    J[:, r0:r0 + rsizes[i], c0 + j] = outs[i]
                    r0 += rsizes[i]
        c0 += n


def _jacobian_columns(st, rows, cols, J):
    """jacobian_columns for the columns p, h and b: unit tangents through solve_jvp."""
    jacobian_columns(st, rows, cols, J, (st.plan.nz, st.plan.nineq, st.plan.neq), JAC_SLOTS, solve_jvp)


def jacobian_matrix(st, rows, cols, csizes, fill):
    """J (B, R, C) fp64 on st.device: rows [z; lam; nu] and column blocks of csizes, restricted to the bits of `rows` /
    `cols`, written by fill(st, rows, cols, J): the family's kernel or its column path."""
    if _pending:
        flush_checks(wait=False)
    rsizes = (st.plan.nz, st.plan.nineq, st.plan.neq)
    R = sum(n for i, n in enumerate(rsizes) if (rows >> i) & 1)
    C = sum(n for k, n in enumerate(csizes) if (cols >> k) & 1)
    J = torch.empty(st.nBatch, R, C, dtype=torch.float64, device=st.device)
    fill(st, rows, cols, J)
    return J


def solve_jacobian(st, rows, cols):
    """d(zhat, lam, nu)/d(p, h, b) at the returned point of `st`, per QP: fp64 (B, R, C) on st.device, rows [z; lam; nu]
    and columns [p, h, b] restricted to the bits of `rows` / `cols` (bit 0 z / p, bit 1 lam / h, bit 2 nu / b). One
    qpb200_jacobian call where the kernel covers the plan (the default mode); otherwise, and always in the regularised
    mode (IR_UNOPT), one solve_jvp per column."""
    plan = st.plan
    if plan.neq == 0 and ((rows | cols) & 4):
        raise ValueError("qpth_b200: a Jacobian with respect to b, or of nu, needs equality constraints (neq == 0)")
    fill = _jacobian_kernel if not getattr(st, "reg", False) and jacobian_covered(plan) else _jacobian_columns
    return jacobian_matrix(st, rows, cols, (plan.nz, plan.nineq, plan.neq), fill)


def _qp_table(plan):
    return tuple(zip(JAC_WRT, (plan.nz, plan.nineq, plan.neq)))


def _qp_refusal(nm):
    if nm not in JAC_WRT:
        return ("qpth_b200: jacobian(wrt=...) takes %s, not %r (Jacobians with respect to Q, G and A are not provided)"
                % (JAC_WRT, nm))
    return "qpth_b200: jacobian(wrt='b') needs equality constraints (neq == 0)"


def jacobian_of(st, out, wrt, duals, table=_qp_table, solve=None, refusal=_qp_refusal):
    """The `jacobian` attribute of a QP layer on the state `st` of its last forward, whose output had
    out = (device, dtype). table(st.plan): ((name, columns), ...) of the inputs in column-bit order, columns 0 for one
    the problem lacks; solve(st, rows, cols) -> J; refusal(name): the error for a name the problem does not take. The
    defaults are QPFunction's and QPSolutionFunction's (p, h, b; solve_jacobian). Returns {name: (B, rows, columns)}
    for each name of `wrt` (None: every input the problem has), rows z, or [z; lam; nu] with duals."""
    if st is None:
        raise RuntimeError("qpth_b200: jacobian() needs a forward call of this function first")
    table = table(st.plan)
    present = tuple(nm for nm, n in table if n)
    names = present if wrt is None else ((wrt,) if isinstance(wrt, str) else tuple(wrt))
    if not names:
        raise ValueError("qpth_b200: jacobian(wrt=...) needs at least one of %s" % (present,))
    for nm in names:
        if nm not in present:
            raise ValueError(refusal(nm))
    known = [nm for nm, _ in table]
    cols = sum(1 << known.index(nm) for nm in set(names))
    rows = 1 | ((2 | (4 if st.plan.neq > 0 else 0)) if duals else 0)
    J = (solve or solve_jacobian)(st, rows, cols)
    res, c0 = {}, 0
    for k, (nm, n) in enumerate(table):
        if (cols >> k) & 1:
            res[nm] = J[:, :, c0:c0 + n]
            c0 += n
    device, dtype = out
    return {nm: res[nm].to(device=device, dtype=dtype).contiguous() for nm in names}


JACOBIAN_DOC = """jacobian(wrt=("p", "h", "b"), duals=False) -> {name: tensor}: the Jacobians of the last forward's solution with
    respect to p, h and b, per QP (also for an un-batched p, h or b: the true derivative, not a batch mean). J["p"] is
    (nBatch, nz, nz) = dz*/dp, J["h"] (nBatch, nz, nineq), J["b"] (nBatch, nz, neq); duals=True gives the rows
    [z; lam; nu], (nBatch, nz + nineq + neq, n). They are the negated inverse of the backward's system at the returned
    point, [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] with qpth's clamped D, so J t equals the forward-mode tangent for a
    tangent t of p, h or b. One kernel call (qpb200_jacobian) factors S once per QP and solves for every column; where it
    does not cover the shape, and with KKTSolvers.IR_UNOPT, one JVP per column. The result has the dtype and device of the
    forward's output and is not differentiable. Jacobians with respect to Q, G and A are not provided: they are
    contractions of these blocks with z, lam and nu (e.g. dz/dh_i lam_j gives the dG_ij column)."""


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

    Forward mode (torch.autograd.forward_ad, gradcheck's check_forward_ad) is supported: the tangents of the outputs are
    one solve of the backward's system with -[rx; 0; rz; ry], rx = sym(dQ) z + dp + dG' lam + dA' nu, rz = dG z - dh,
    ry = dA z - db (qpb200_jvp), the exact transpose of the backward pass. The tangent of an un-batched input applies
    to every QP and gives the true derivative, where the backward returns the batch mean.

    The returned callable's `jacobian(wrt=("p", "h", "b"), duals=False)` gives the whole Jacobians of the last forward's
    solution with respect to p, h and b, per QP (its docstring has the details).

    Second order: under `torch.autograd.grad(..., create_graph=True)` the gradients are differentiable again, in the
    incoming gradients of z, lam, nu and in Q, p, G, h, A, b (Hessian-vector products, `torch.autograd.functional.hessian`,
    gradient penalties, meta-learning through the layer). The double backward is the exact derivative of the backward as
    computed (qpth's clamped D included): one JVP solve, one dual backward solve and two bandwidth-bound kernels
    (qpb200_double_backward). The cotangent of an un-batched input's gradient (a batch mean) is shared by every QP, and
    that input's second-order gradient is the batch sum. Without create_graph nothing changes. Third order raises.

    kkt_solver (an extension of the reference's signature): KKTSolvers.LU_PARTIAL, the default, needs Q positive definite.
    KKTSolvers.IR_UNOPT also solves QPs whose Q is only positive semidefinite (LPs with Q = 0, low-rank quadratic terms)
    and QPs whose equality rows are linearly dependent: every KKT solve factors the system regularised with kkt.IR_EPS
    (chol(Q + eps I); eps on the constraint blocks) and refines it kkt.IR_STEPS times, while the residuals are those of
    the true problem, so the returned point is the exact KKT point. check_Q_spd then checks that Q is positive
    SEMIdefinite ('Q is not positive semidefinite.'). IR_UNOPT takes every shape the default mode takes with
    nineq >= 1: up to ms_pad = 8 ceil(neq / 8) + nineq rounded up to 8 of about 200 on the product-form kernels, beyond
    that on the generic global-scratch kernels. With linearly dependent equality rows the equality duals, and so the
    gradients dA and db, are not unique; z*, the inequality duals, the slacks and dQ, dp, dG, dh are. An unbounded or
    infeasible problem gives the inaccurate-solution banner, as in the default mode.

    Only the lower triangle of Q is read, by every kernel and host path behind this function (the equality-only path
    included): the strictly upper triangle may hold anything, NaN included, and the result - z*, the duals, the SPD
    check, every gradient - is that of the symmetric matrix tril(Q) + tril(Q, -1)^T. A forward-mode tangent dQ is read
    in full and enters as sym(dQ) = (dQ + dQ^T) / 2 (tests/test_gpu_q_lower_triangle.py)."""
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

        def no_jacobian(wrt=JAC_WRT, duals=False):
            raise NotImplementedError("qpth_b200: jacobian() is not provided for solver=QPSolvers.CVXPY; solve with "
                                      "CVXPY and call QPSolutionFunction's jacobian() instead")

        apply_cvxpy.jacobian = no_jacobian
        return apply_cvxpy
    if solver != QPSolvers.PDIPM_BATCHED:
        assert False                                     # qp.py:121-122

    _last = [None]
    _jac = [None, None, False]           # the state and (device, dtype) of the last forward; True: it was equality-only

    class QPFunctionFn(QPLayerFn):
        @staticmethod
        def forward(ctx, Q_, p_, G_, h_, A_, b_):
            """Solve a batch of QPs  argmin_z 1/2 z^T Q z + p^T z  s.t. Gz <= h, Az = b.

            Q (nBatch,nz,nz)|(nz,nz); p (nBatch,nz)|(nz); G (nBatch,nineq,nz)|(nineq,nz);
            h (nBatch,nineq)|(nineq); A (nBatch,neq,nz)|(neq,nz)|empty; b (nBatch,neq)|(neq)|empty.
            Returns zhat (nBatch, nz).  (qp.py:23-125)
            """
            st = solve_forward(Q_, p_, G_, h_, A_, b_, eps, verbose, notImprovedLim, maxIter, check_Q_spd, kkt_solver)
            _last[0] = st
            _jac[0], _jac[1] = st, (Q_.device, Q_.dtype)
            ctx.neq, ctx.nineq, ctx.nz = st.plan.neq, st.plan.nineq, st.plan.nz
            return layer_outputs(ctx, st, (Q_, p_, G_, h_, A_, b_), duals)

    def apply(Q_, p_, G_, h_, A_, b_):
        if G_.nelement() == 0 and h_.nelement() == 0 and A_.nelement() > 0:
            # equality-constrained QP: an extension (the reference cannot run nineq == 0); one KKT solve, eqonly.py
            from .eqonly import solve_equality_qp
            _jac[:] = [None, None, True]
            return solve_equality_qp(Q_, p_, A_, b_, check_Q_spd, reg=kkt_solver == KKTSolvers.IR_UNOPT, duals=duals)
        _jac[2] = False
        return QPFunctionFn.apply(Q_, p_, G_, h_, A_, b_)

    def jacobian(wrt=JAC_WRT, duals=False):
        if _jac[2]:
            raise NotImplementedError("qpth_b200: jacobian() is not provided for the equality-only path (nineq == 0); "
                                      "use forward-mode AD (torch.autograd.forward_ad) column by column")
        return jacobian_of(_jac[0], _jac[1], wrt, duals)

    jacobian.__doc__ = JACOBIAN_DOC
    # diagnostics the reference keeps on ctx (nus / lams / slacks) plus per-QP iteration counts
    apply.last_solve = lambda: _last[0]
    apply.jacobian = jacobian
    return apply
