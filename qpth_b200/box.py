"""`BoxQPFunction` — batched differentiable QPs with a diagonal Q and simple bounds.

    min_z 1/2 z' diag(q) z + p'z   s.t.   A z = b,   lb <= z <= ub

The semantics are QPFunction's on the dense equivalent Q = diag(q), G = [-I; I] (only the sides given), h = [-lb; ub]:
the same Mehrotra loop, exit rules (per QP, STALL_TOL, BEST_TIE), residuals, diagnostics, dtype / device handling and
gradient conventions (batch mean for an input passed un-batched). What differs is the KKT solve: with Q diagonal and
every row of G equal to +-e_i the inequality block is eliminated in closed form, so a Newton iteration factors only
M = A H^-1 A' (order neq, H = q + G'DG diagonal) - nothing at all without equality constraints - and needs no
pre_factor_kkt (csrc/qp_box.cu). One CTA solves one QP where A and the vectors fit its 227 KB of shared memory
(qpb200_box_plan.ok); past that, a thread block cluster of 2, 4 or 8 CTAs does, each CTA holding a slice of the
variables (plan.cl_ctas; e.g. the capped-simplex projection over thousands of classes). With more than 128 equality
rows (the 9x9 sudoku layer: nz = 729, neq = 249) the cluster also distributes the factor of M (plan.cl_ctas with
plan.neq_pad > 128), where the dense equivalent's order exceeds 384 or the dense kernels reject it. Shapes none of these
covers run the dense kernels on the dense equivalent instead.

The OptNet sudoku layer (Q = 0.1 I, G = -I, h = 0, a learned A) is one such problem; a differentiable projection
min 1/2 ||z - v||^2 s.t. Az = b, lb <= z <= ub is another (q = 1, p = -v).
"""
import ctypes

import torch
from torch.autograd import Function

from . import _lib
from . import qp as _qp
from .qp import _dev64, _ptr, _stream


def check_box_shapes(q, p, A, b, lb, ub):
    """Validate ranks, trailing dimensions and batch sizes before anything touches the device.
    Returns (nBatch, nz, neq). q, p, lb, ub: (B, nz) | (nz); A: (B, neq, nz) | (neq, nz) | empty; b follows A."""
    if lb is None and ub is None:
        raise ValueError("BoxQPFunction: at least one of lb, ub must be given")
    ins = (("q", q, 2), ("p", p, 2), ("A", A, 3), ("b", b, 2), ("lb", lb, 2), ("ub", ub, 2))
    nBatch = next((int(X.size(0)) for _, X, r in ins if X is not None and X.nelement() > 0 and X.dim() == r), 1)
    for _, X, r in ins:
        if X is not None and X.nelement() > 0 and X.dim() not in (r, r - 1):
            raise RuntimeError("Unexpected number of dimensions.")

    def fail(msg):
        raise RuntimeError("qpth_b200: inconsistent shapes: " + msg)

    if q.nelement() == 0:
        fail("q is empty")
    nz = int(q.size(-1))
    neq = int(A.size(-2)) if (A is not None and A.nelement() > 0 and A.dim() >= 2) else 0
    for name, X, trail, needed in (("p", p, (nz,), True), ("lb", lb, (nz,), lb is not None),
                                   ("ub", ub, (nz,), ub is not None), ("A", A, (neq, nz), neq > 0),
                                   ("b", b, (neq,), neq > 0)):
        if not needed:
            if X is not None and X.nelement() != 0:
                fail("%s given %s but there are no equality constraints" % (name, tuple(X.shape)))
            continue
        if X is None or X.nelement() == 0 or tuple(X.shape[-len(trail):]) != trail:
            fail("%s has shape %s, expected trailing dimensions %s"
                 % (name, None if X is None else tuple(X.shape), trail))
    for name, X, r in ins:
        if X is not None and X.nelement() > 0 and X.dim() == r and X.size(0) != nBatch:
            fail("%s has batch size %d, the batch is %d" % (name, X.size(0), nBatch))
    return nBatch, nz, neq


class _BoxSolved:
    """State carried from forward to backward; lam / slacks are laid out as [lb rows; ub rows]."""
    __slots__ = ("plan", "nBatch", "device", "q", "sq", "A", "sA", "zhat", "lam", "slacks", "nus", "iters",
                 "best_resid", "trace", "dense")


def solve_box_forward(q_, p_, A_, b_, lb_, ub_, eps=1e-12, verbose=0, notImprovedLim=3, maxIter=20, check_Q_spd=True):
    """The box kernels on the device (one CTA per QP, or a cluster of plan.cl_ctas CTAs per QP). Returns _BoxSolved
    (dense = None), or None when neither covers the shape."""
    nBatch, nz, neq = check_box_shapes(q_, p_, A_, b_, lb_, ub_)
    if _qp._pending:
        _qp.flush_checks(wait=False)
    assert maxIter >= 1
    lib = _lib.load()
    if not torch.cuda.is_available():
        raise _lib.QpthB200Error("qpth_b200: no CUDA device available (there is no CPU fallback).")
    plan = _lib.box_plan_for(nz, neq, lb_ is not None, ub_ is not None)
    if not (plan.ok or plan.cl_ctas):
        return None
    device = q_.device if q_.is_cuda else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
        q, p = _dev64(q_, device), _dev64(p_, device)
        lb = _dev64(lb_, device) if lb_ is not None else None
        ub = _dev64(ub_, device) if ub_ is not None else None
        A = _dev64(A_, device) if neq > 0 else None
        b = _dev64(b_, device) if neq > 0 else None

        def stride(t, nd, per):
            return per if (t is not None and t.dim() == nd) else 0

        m = plan.nineq
        st = _BoxSolved()
        st.plan, st.nBatch, st.device, st.dense = plan, nBatch, device, None
        st.q, st.sq, st.A, st.sA = q, stride(q, 2, nz), A, stride(A, 3, neq * nz)
        f64 = dict(dtype=torch.float64, device=device)
        st.zhat = torch.empty(nBatch, nz, **f64)
        st.lam = torch.empty(nBatch, m, **f64)
        st.slacks = torch.empty(nBatch, m, **f64)
        st.nus = torch.empty(nBatch, neq, **f64) if neq > 0 else None
        st.iters = torch.empty(nBatch, dtype=torch.int32, device=device)
        st.best_resid = torch.empty(nBatch, **f64)
        st.trace = torch.full((nBatch, int(maxIter), 4), float('nan'), **f64) if (verbose == 1 or _qp.TRACE) else None
        spd = torch.zeros(nBatch, dtype=torch.int32, device=device)
        _lib.check(lib.qpb200_box_forward(
            ctypes.byref(plan), nBatch, _ptr(q), st.sq, _ptr(p), stride(p, 2, nz), _ptr(A), st.sA,
            _ptr(b), stride(b, 2, neq), _ptr(lb), stride(lb, 2, nz), _ptr(ub), stride(ub, 2, nz),
            float(eps), float(_qp.STALL_TOL), float(_qp.BEST_TIE), int(notImprovedLim), int(maxIter),
            _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(st.iters), _ptr(st.best_resid),
            _ptr(st.trace), _ptr(spd), _stream()))
        _qp.diagnostics(spd, st, check_Q_spd, verbose)
    return st


def solve_box_backward(st, dl_dzhat, mean_flags, want, dl_dlam=None, dl_dnu=None):
    """Gradients (dq, dp, dA, db, dlb, dub) on the device; mean_flags / want: 6-tuples in that order. dl_dlam ([lb rows;
    ub rows]) / dl_dnu: the gradients with respect to the returned duals (None: zero); dl_dzhat None: zero."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    lib = _lib.load()
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    f64 = dict(dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        dl = _qp._adjoint(dl_dzhat, B, nz, device) if dl_dzhat is not None else torch.zeros(B, nz, **f64)
        glam, gnu = _qp._adjoint(dl_dlam, B, m, device), _qp._adjoint(dl_dnu, B, neq, device)
        shapes = [(nz,), (nz,), (neq, nz), (neq,), (nz,), (nz,)]
        outs = []
        for k in range(6):
            absent = (k in (2, 3) and neq == 0) or (k == 4 and not plan.has_lb) or (k == 5 and not plan.has_ub)
            if not want[k] or absent:
                outs.append(None)
            else:
                outs.append(torch.empty(*(shapes[k] if mean_flags[k] else (B,) + shapes[k]), **f64))
        dxv = torch.empty(B, nz, **f64)
        dlamv = torch.empty(B, m, **f64)
        dnuv = torch.empty(B, neq, **f64) if neq > 0 else None
        dq, dp, dA, db, dlb, dub = outs
        mq, mp, mA, mb, mlb, mub = (1 if f else 0 for f in mean_flags)
        if glam is None and gnu is None:            # no dual was used: the entry point of a zhat-only loss
            fn, adj = lib.qpb200_box_backward, ()
        else:
            fn, adj = lib.qpb200_box_backward_duals, (_ptr(glam), _ptr(gnu))
        _lib.check(fn(
            ctypes.byref(plan), B, _ptr(st.q), st.sq, _ptr(st.A), st.sA, _ptr(dl), *adj, _ptr(st.zhat), _ptr(st.lam),
            _ptr(st.slacks), _ptr(st.nus), _ptr(dq), mq, _ptr(dp), mp, _ptr(dlb), mlb, _ptr(dub), mub,
            _ptr(dA), mA, _ptr(db), mb, _ptr(dxv), _ptr(dlamv), _ptr(dnuv), _stream()))
    return outs


# ---- shapes beyond the box kernels: the dense kernels on the dense equivalent ---------------------------------------
def dense_equivalent(q, lb, ub):
    """(Q, G, h) of QPFunction for a box QP: Q = diag(q), G = [-I; I] (sides given), h = [-lb; ub]. Batched where
    q (for Q) or either bound (for h) is batched."""
    nz = q.size(-1)
    Q = torch.diag_embed(q)
    eye = torch.eye(nz, dtype=q.dtype, device=q.device)
    G = torch.cat(([-eye] if lb is not None else []) + ([eye] if ub is not None else []), 0)
    sides = [(-lb) if lb is not None else None, ub]
    sides = [s for s in sides if s is not None]
    if any(s.dim() == 2 for s in sides):
        B = next(s.size(0) for s in sides if s.dim() == 2)
        sides = [s if s.dim() == 2 else s.unsqueeze(0).expand(B, nz) for s in sides]
    h = torch.cat(sides, -1)
    return Q, G, h


def solve_dense_forward(q_, p_, A_, b_, lb_, ub_, eps, verbose, notImprovedLim, maxIter, check_Q_spd):
    A_ = A_ if A_ is not None else torch.empty(0, dtype=q_.dtype, device=q_.device)
    b_ = b_ if b_ is not None else torch.empty(0, dtype=q_.dtype, device=q_.device)
    Q, G, h = dense_equivalent(q_.detach(), None if lb_ is None else lb_.detach(), None if ub_ is None else ub_.detach())
    dst = _qp.solve_forward(Q, p_.detach(), G, h, A_.detach(), b_.detach(), eps, verbose, notImprovedLim, maxIter,
                            check_Q_spd)
    st = _BoxSolved()
    st.plan, st.nBatch, st.device, st.dense = dst.plan, dst.nBatch, dst.device, (dst, h.dim() == 1)
    st.zhat, st.lam, st.slacks, st.nus = dst.zhat, dst.lam, dst.slacks, dst.nus
    st.iters, st.best_resid, st.trace = dst.iters, dst.best_resid, dst.trace
    st.q = st.A = None
    st.sq = st.sA = 0
    return st


def dense_backward(st, dl, mean_flags, want, nlb, has_ub, dl_dlam=None, dl_dnu=None):
    dst, h_shared = st.dense
    mq, mp, mA, mb, mlb, mub = mean_flags
    # the dense equivalent's rows are lam's [lb rows; ub rows]: the dual adjoints pass through as they are
    outs = _qp.solve_backward(dst, dl, (mq, mp, True, h_shared, mA, mb),
                              (want[0], want[1], False, want[4] or want[5], want[2], want[3]), dl_dlam, dl_dnu)
    dQ, dp, _, dh, dA, db = outs
    dq = None if dQ is None else torch.diagonal(dQ, dim1=-2, dim2=-1).contiguous()
    dlb = dub = None
    if dh is not None:
        if want[4] and nlb:
            dlb = -dh[..., :nlb]
            dlb = dlb.mean(0) if (mlb and dlb.dim() == 2) else dlb
        if want[5] and has_ub:
            dub = dh[..., nlb:]
            dub = dub.mean(0) if (mub and dub.dim() == 2) else dub
    return [dq, dp, dA, db, dlb, dub]


def BoxQPFunction(eps=1e-12, verbose=0, notImprovedLim=3, maxIter=20, check_Q_spd=True, duals=False):
    """Factory with QPFunction's options; returns f(q, p, A, b, lb, ub) -> z (nBatch, nz).

    q, p, lb, ub: (nBatch, nz) or (nz); A: (nBatch, neq, nz), (neq, nz) or an empty tensor; b follows A. lb or ub may
    be None (no bound on that side), not both. f.last_solve() returns the state of the last forward: lam, slacks
    ([lb rows; ub rows]), nus, iters, best_resid.

    duals=True: f returns (z, lam, nu) as QPFunction(duals=True) does: lam (nBatch, nineq) in the [lb rows; ub rows]
    layout of last_solve(), nu (nBatch, neq) or (nBatch, 0), and a loss may use all three."""
    _last = [None]

    class BoxQPFunctionFn(Function):
        @staticmethod
        def forward(ctx, q_, p_, A_, b_, lb_, ub_):
            st = solve_box_forward(q_, p_, A_, b_, lb_, ub_, eps, verbose, notImprovedLim, maxIter, check_Q_spd)
            if st is None:
                st = solve_dense_forward(q_, p_, A_, b_, lb_, ub_, eps, verbose, notImprovedLim, maxIter, check_Q_spd)
            ctx.st = st
            _last[0] = st
            zhats = st.zhat.to(device=q_.device, dtype=q_.dtype)
            ctx.save_for_backward(zhats, q_, p_, A_, b_, lb_, ub_)
            ctx.lams, ctx.slacks, ctx.nus = st.lam, st.slacks, st.nus
            if not duals:
                return zhats
            ctx.set_materialize_grads(False)
            return (zhats,) + _qp.dual_outputs(st, q_)

        @staticmethod
        def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
            zhats, q, p, A, b, lb, ub = ctx.saved_tensors
            st = ctx.st
            ins = (q, p, A, b, lb, ub)
            ranks = (2, 2, 3, 2, 2, 2)
            flags = [X is not None and X.nelement() > 0 and X.dim() == r - 1 for X, r in zip(ins, ranks)]
            want = list(ctx.needs_input_grad)
            if st.dense is None:
                outs = solve_box_backward(st, dl_dzhat, flags, want, dl_dlam, dl_dnu)
            else:
                outs = dense_backward(st, dl_dzhat, flags, want, q.size(-1) if lb is not None else 0, ub is not None,
                                      dl_dlam, dl_dnu)
            return tuple(None if (g is None or X is None or not w) else g.to(device=X.device, dtype=X.dtype)
                         for X, g, w in zip(ins, outs, want))

    def apply(q, p, A, b, lb, ub):
        return BoxQPFunctionFn.apply(q, p, A, b, lb, ub)

    apply.last_solve = lambda: _last[0]
    return apply
