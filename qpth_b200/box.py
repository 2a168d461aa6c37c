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

BoxQPFunction(dense_Q=True) takes a dense Q instead (long-only portfolios, condensed MPC with input bounds, metric
projections onto a box): the bounds are eliminated the same way, and each Newton iteration factors the bordered matrix
[Q + G'DG  A'; A  0] of order nz + neq once (csrc/qp_boxq.cu, qpb200_boxq_plan.ok) instead of the dense equivalent's
order 2 nz + neq. Shapes past one CTA run the dense kernels on the dense equivalent.
"""
import ctypes

import torch
from torch.autograd import Function

from . import _lib
from . import qp as _qp
from .qp import _dev64, _ptr, _stream


def check_box_shapes(q, p, A, b, lb, ub, dense_Q=False):
    """Validate ranks, trailing dimensions and batch sizes before anything touches the device.
    Returns (nBatch, nz, neq). q, p, lb, ub: (B, nz) | (nz); A: (B, neq, nz) | (neq, nz) | empty; b follows A.
    dense_Q: q is a dense Q, (B, nz, nz) | (nz, nz)."""
    if lb is None and ub is None:
        raise ValueError("BoxQPFunction: at least one of lb, ub must be given")
    ins = (("Q" if dense_Q else "q", q, 3 if dense_Q else 2), ("p", p, 2), ("A", A, 3), ("b", b, 2), ("lb", lb, 2),
           ("ub", ub, 2))
    nBatch = next((int(X.size(0)) for _, X, r in ins if X is not None and X.nelement() > 0 and X.dim() == r), 1)
    for _, X, r in ins:
        if X is not None and X.nelement() > 0 and X.dim() not in (r, r - 1):
            raise RuntimeError("Unexpected number of dimensions.")

    def fail(msg):
        raise RuntimeError("qpth_b200: inconsistent shapes: " + msg)

    if q.nelement() == 0:
        fail("%s is empty" % ins[0][0])
    nz = int(q.size(-1))
    if dense_Q and int(q.size(-2)) != nz:
        fail("Q has shape %s, expected trailing dimensions (nz, nz)" % (tuple(q.shape),))
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
    """State carried from forward to backward; lam / slacks are laid out as [lb rows; ub rows]. dense_Q: q / sq hold a
    dense Q and its batch stride, and plan is a qpb200_boxq_plan."""
    __slots__ = ("plan", "nBatch", "device", "q", "sq", "A", "sA", "zhat", "lam", "slacks", "nus", "iters",
                 "best_resid", "trace", "dense", "dense_Q")


def solve_box_forward(q_, p_, A_, b_, lb_, ub_, eps=1e-12, verbose=0, notImprovedLim=3, maxIter=20, check_Q_spd=True,
                      dense_Q=False):
    """The box kernels on the device: one CTA per QP, or a cluster of plan.cl_ctas CTAs per QP; dense_Q: the dense-Q
    kernels, one CTA per QP. Returns _BoxSolved (dense = None), or None when they do not cover the shape."""
    nBatch, nz, neq = check_box_shapes(q_, p_, A_, b_, lb_, ub_, dense_Q)
    if _qp._pending:
        _qp.flush_checks(wait=False)
    assert maxIter >= 1
    lib = _lib.load()
    if not torch.cuda.is_available():
        raise _lib.QpthB200Error("qpth_b200: no CUDA device available (there is no CPU fallback).")
    if dense_Q:
        plan = _lib.boxq_plan_for(nz, neq, lb_ is not None, ub_ is not None)
        if not plan.ok:
            return None
    else:
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
        st.plan, st.nBatch, st.device, st.dense, st.dense_Q = plan, nBatch, device, None, dense_Q
        st.q, st.sq = q, (stride(q, 3, nz * nz) if dense_Q else stride(q, 2, nz))
        st.A, st.sA = A, stride(A, 3, neq * nz)
        f64 = dict(dtype=torch.float64, device=device)
        st.zhat = torch.empty(nBatch, nz, **f64)
        st.lam = torch.empty(nBatch, m, **f64)
        st.slacks = torch.empty(nBatch, m, **f64)
        st.nus = torch.empty(nBatch, neq, **f64) if neq > 0 else None
        st.iters = torch.empty(nBatch, dtype=torch.int32, device=device)
        st.best_resid = torch.empty(nBatch, **f64)
        st.trace = torch.full((nBatch, int(maxIter), 4), float('nan'), **f64) if (verbose == 1 or _qp.TRACE) else None
        spd = torch.zeros(nBatch, dtype=torch.int32, device=device)
        fn = lib.qpb200_boxq_forward if dense_Q else lib.qpb200_box_forward
        _lib.check(fn(
            ctypes.byref(plan), nBatch, _ptr(q), st.sq, _ptr(p), stride(p, 2, nz), _ptr(A), st.sA,
            _ptr(b), stride(b, 2, neq), _ptr(lb), stride(lb, 2, nz), _ptr(ub), stride(ub, 2, nz),
            float(eps), float(_qp.STALL_TOL), float(_qp.BEST_TIE), int(notImprovedLim), int(maxIter),
            _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(st.iters), _ptr(st.best_resid),
            _ptr(st.trace), _ptr(spd), _stream()))
        _qp.diagnostics(spd, st, check_Q_spd, verbose)
    return st


def solve_box_backward(st, dl_dzhat, mean_flags, want, dl_dlam=None, dl_dnu=None, keep=False):
    """Gradients (dq, dp, dA, db, dlb, dub) on the device; mean_flags / want: 6-tuples in that order. dl_dlam ([lb rows;
    ub rows]) / dl_dnu: the gradients with respect to the returned duals (None: zero); dl_dzhat None: zero. With a
    dense Q the first is dQ, (B, nz, nz) or (nz, nz) with its mean flag. keep: also return the solve (dxv, dlamv,
    dnuv), which the double backward reads."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    lib = _lib.load()
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    f64 = dict(dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        dl = _qp._adjoint(dl_dzhat, B, nz, device) if dl_dzhat is not None else torch.zeros(B, nz, **f64)
        glam, gnu = _qp._adjoint(dl_dlam, B, m, device), _qp._adjoint(dl_dnu, B, neq, device)
        shapes = [(nz, nz) if st.dense_Q else (nz,), (nz,), (neq, nz), (neq,), (nz,), (nz,)]
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
        if st.dense_Q:
            fn, adj = lib.qpb200_boxq_backward_duals, (_ptr(glam), _ptr(gnu))
        elif glam is None and gnu is None:          # no dual was used: the entry point of a zhat-only loss
            fn, adj = lib.qpb200_box_backward, ()
        else:
            fn, adj = lib.qpb200_box_backward_duals, (_ptr(glam), _ptr(gnu))
        _lib.check(fn(
            ctypes.byref(plan), B, _ptr(st.q), st.sq, _ptr(st.A), st.sA, _ptr(dl), *adj, _ptr(st.zhat), _ptr(st.lam),
            _ptr(st.slacks), _ptr(st.nus), _ptr(dq), mq, _ptr(dp), mp, _ptr(dlb), mlb, _ptr(dub), mub,
            _ptr(dA), mA, _ptr(db), mb, _ptr(dxv), _ptr(dlamv), _ptr(dnuv), _stream()))
    if keep:
        return outs, (dxv, dlamv, dnuv)
    return outs


def solve_box_double_backward(st, v, omegas, flags, want):
    """The double backward on the device (qpb200_box_double_backward / qpb200_boxq_double_backward): v = (dxv, dlamv,
    dnuv) of the first backward at the point of `st`; omegas: the cotangents of its six outputs (dq, dp, dA, db, dlb,
    dub; dQ with a dense Q), each None or shaped as that output; flags: the first backward's mean flags (an un-batched
    input: its cotangent is divided by nBatch, and its second-order gradient is the batch sum); want: which of the six
    gradients to write. Returns fp64 (gg_z, gg_lam, gg_nu, dq, dp, dA, db, dlb, dub): the gradients of g_z, g_lam, g_nu
    (gg_nu None without equality rows) and of the six inputs (None where not wanted or absent)."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    lib = _lib.load()
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    f64 = dict(dtype=torch.float64, device=device)
    absent = (False, False, neq == 0, neq == 0, not plan.has_lb, not plan.has_ub)
    with torch.cuda.device(device):
        om = [None if (w is None or absent[k]) else (_dev64(w, device) / B if flags[k] else w)
              for k, w in enumerate(omegas)]
        per = (nz * nz if st.dense_Q else nz, nz, neq * nz, neq, nz, nz)
        tans = _qp.tangent_args(om, (3 if st.dense_Q else 2, 2, 3, 2, 2, 2), per, device)
        shapes = [(nz, nz) if st.dense_Q else (nz,), (nz,), (neq, nz), (neq,), (nz,), (nz,)]
        outs = []
        for k in range(6):
            if not want[k] or absent[k]:
                outs.append(None)
            else:
                outs.append(torch.empty(*(shapes[k] if flags[k] else (B,) + shapes[k]), **f64))
        gz = torch.empty(B, nz, **f64)
        glam = torch.empty(B, m, **f64)
        gnu = torch.empty(B, neq, **f64) if neq > 0 else None
        work = torch.empty(B * (2 * nz + 3 * m + 2 * neq), **f64)      # QPB200_DOUBLE_BACKWARD_WORK
        args = []
        for t, s in tans:
            args += [_ptr(t), s]
        dq, dp, dA, db, dlb, dub = outs
        grads = []
        for g, k in zip((dq, dp, dlb, dub, dA, db), (0, 1, 4, 5, 2, 3)):   # the ABI's order
            grads += [_ptr(g), 1 if flags[k] else 0]
        fn = lib.qpb200_boxq_double_backward if st.dense_Q else lib.qpb200_box_double_backward
        _lib.check(fn(
            ctypes.byref(plan), B, _ptr(st.q), st.sq, _ptr(st.A), st.sA, *args, *(_ptr(x) for x in v),
            _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(gz), _ptr(glam), _ptr(gnu), *grads,
            _ptr(work), _stream()))
    return [gz, glam, gnu] + outs


class BoxQPBackwardFn(Function):
    """The first-order backward of BoxQPFunction (the box kernels) as a differentiable function of the incoming
    gradients (g_z, g_lam, g_nu) and of (q, p, A, b, lb, ub): what its backward runs under create_graph=True. Its
    forward is the first backward's own solve_box_backward call; its backward is solve_box_double_backward."""
    @staticmethod
    def forward(ctx, st, flags, want, g_z, g_lam, g_nu, q, p, A, b, lb, ub):
        outs, v = solve_box_backward(st, g_z, flags, want, g_lam, g_nu, keep=True)
        ctx.st, ctx.v, ctx.flags = st, v, flags
        ctx.like = (g_z, g_lam, g_nu, q, p, A, b, lb, ub)
        ctx.set_materialize_grads(False)
        return tuple(_qp._cast(g, X) for X, g in zip((q, p, A, b, lb, ub), outs))

    @staticmethod
    def backward(ctx, *omegas):
        if torch.is_grad_enabled():
            raise RuntimeError(_qp.THIRD_ORDER_ERR)
        need = ctx.needs_input_grad[3:]
        if all(w is None for w in omegas) or not any(need):
            return (None,) * 12
        res = solve_box_double_backward(ctx.st, ctx.v, omegas, ctx.flags, need[3:])
        return (None, None, None) + tuple(_qp._cast(g, X) if n else None for g, X, n in zip(res, ctx.like, need))


def solve_box_jvp(st, tangents):
    """The JVP of (zhat, lam, nu) at the returned point on the device. tangents: (dq, dp, dA, db, dlb, dub), each None
    (zero), batched or un-batched as its input (with a dense Q, dQ first). Returns fp64 (dz (B,nz), dlam (B,nineq) in
    the [lb rows; ub rows] layout, dnu (B,neq) or None); one qpb200_box_jvp / qpb200_boxq_jvp call: the right-hand side
    kernel and the backward's solve."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    lib = _lib.load()
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    f64 = dict(dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        per = (nz * nz if st.dense_Q else nz, nz, neq * nz, neq, nz if plan.has_lb else 0, nz if plan.has_ub else 0)
        tans = _qp.tangent_args(tangents, (3 if st.dense_Q else 2, 2, 3, 2, 2, 2), per, device)
        rhs = torch.empty(B * (nz + m + neq), **f64)
        dz = torch.empty(B, nz, **f64)
        dlam = torch.empty(B, m, **f64)
        dnu = torch.empty(B, neq, **f64) if neq > 0 else None
        args = []
        for t, s in tans:
            args += [_ptr(t), s]
        fn = lib.qpb200_boxq_jvp if st.dense_Q else lib.qpb200_box_jvp
        _lib.check(fn(
            ctypes.byref(plan), B, _ptr(st.q), st.sq, _ptr(st.A), st.sA, *args, _ptr(st.zhat), _ptr(st.lam),
            _ptr(st.slacks), _ptr(st.nus), _ptr(rhs), _ptr(dz), _ptr(dlam), _ptr(dnu), _stream()))
    return dz, dlam, dnu


# ---- shapes beyond the box kernels: the dense kernels on the dense equivalent ---------------------------------------
def dense_equivalent(q, lb, ub, dense_Q=False):
    """(Q, G, h) of QPFunction for a box QP: Q = diag(q) (dense_Q: q itself), G = [-I; I] (sides given),
    h = [-lb; ub]. Batched where q (for Q) or either bound (for h) is batched."""
    nz = q.size(-1)
    Q = q if dense_Q else torch.diag_embed(q)
    eye = torch.eye(nz, dtype=q.dtype, device=q.device)
    G = torch.cat(([-eye] if lb is not None else []) + ([eye] if ub is not None else []), 0)
    sides = [(-lb) if lb is not None else None, ub]
    sides = [s for s in sides if s is not None]
    if any(s.dim() == 2 for s in sides):
        B = next(s.size(0) for s in sides if s.dim() == 2)
        sides = [s if s.dim() == 2 else s.unsqueeze(0).expand(B, nz) for s in sides]
    h = torch.cat(sides, -1)
    return Q, G, h


def solve_dense_forward(q_, p_, A_, b_, lb_, ub_, eps, verbose, notImprovedLim, maxIter, check_Q_spd, dense_Q=False):
    A_ = A_ if A_ is not None else torch.empty(0, dtype=q_.dtype, device=q_.device)
    b_ = b_ if b_ is not None else torch.empty(0, dtype=q_.dtype, device=q_.device)
    Q, G, h = dense_equivalent(q_.detach(), None if lb_ is None else lb_.detach(), None if ub_ is None else ub_.detach(),
                               dense_Q)
    dst = _qp.solve_forward(Q, p_.detach(), G, h, A_.detach(), b_.detach(), eps, verbose, notImprovedLim, maxIter,
                            check_Q_spd)
    st = _BoxSolved()
    st.plan, st.nBatch, st.device, st.dense = dst.plan, dst.nBatch, dst.device, (dst, h.dim() == 1)
    st.dense_Q = dense_Q
    st.zhat, st.lam, st.slacks, st.nus = dst.zhat, dst.lam, dst.slacks, dst.nus
    st.iters, st.best_resid, st.trace = dst.iters, dst.best_resid, dst.trace
    st.q = st.A = None
    st.sq = st.sA = 0
    return st


def dense_backward(st, dl, mean_flags, want, nlb, has_ub, dl_dlam=None, dl_dnu=None, dense_Q=False):
    dst, h_shared = st.dense
    mq, mp, mA, mb, mlb, mub = mean_flags
    # the dense equivalent's rows are lam's [lb rows; ub rows]: the dual adjoints pass through as they are
    outs = _qp.solve_backward(dst, dl, (mq, mp, True, h_shared, mA, mb),
                              (want[0], want[1], False, want[4] or want[5], want[2], want[3]), dl_dlam, dl_dnu)
    dQ, dp, _, dh, dA, db = outs
    dq = dQ if (dQ is None or dense_Q) else torch.diagonal(dQ, dim1=-2, dim2=-1).contiguous()
    dlb = dub = None
    if dh is not None:
        if want[4] and nlb:
            dlb = -dh[..., :nlb]
            dlb = dlb.mean(0) if (mlb and dlb.dim() == 2) else dlb
        if want[5] and has_ub:
            dub = dh[..., nlb:]
            dub = dub.mean(0) if (mub and dub.dim() == 2) else dub
    return [dq, dp, dA, db, dlb, dub]


def dense_backward_graph(st, dl, mean_flags, want, ins, dl_dlam=None, dl_dnu=None, dense_Q=False):
    """dense_backward under create_graph=True: (Q, h) of the dense equivalent built from the inputs with torch ops, the
    first backward through qp.QPBackwardFn on the dense state (G constant), and the map back to (dq, dp, dA, db, dlb,
    dub) again with torch ops, so that the gradients can be differentiated once more. Returns them cast to the inputs."""
    dst, h_shared = st.dense
    q, p, A, b, lb, ub = ins
    mq, mp, mA, mb, mlb, mub = mean_flags
    Q, G, h = dense_equivalent(q, lb, ub, dense_Q)
    empty = torch.empty(0, dtype=q.dtype, device=q.device)
    A_ = A if (A is not None and A.nelement() > 0) else empty
    b_ = b if (b is not None and b.nelement() > 0) else empty
    dQ, dp, _, dh, dA, db = _qp.QPBackwardFn.apply(
        dst, (mq, mp, True, h_shared, mA, mb), (want[0], want[1], False, want[4] or want[5], want[2], want[3]),
        dl, dl_dlam, dl_dnu, Q, p, G, h, A_, b_)
    nlb = q.size(-1) if lb is not None else 0
    dq = dQ if (dQ is None or dense_Q) else torch.diagonal(dQ, dim1=-2, dim2=-1)
    dlb = dub = None
    if dh is not None:
        if want[4] and lb is not None:
            dlb = -dh[..., :nlb]
            dlb = dlb.mean(0) if (mlb and dlb.dim() == 2) else dlb
        if want[5] and ub is not None:
            dub = dh[..., nlb:]
            dub = dub.mean(0) if (mub and dub.dim() == 2) else dub
    outs = (dq, dp, dA, db, dlb, dub)
    return tuple(None if (g is None or X is None or not w) else g.to(device=X.device, dtype=X.dtype)
                 for X, g, w in zip(ins, outs, want))


def dense_jvp(st, tangents, nlb, has_ub, dense_Q=False):
    """solve_box_jvp on the dense equivalent: dQ = diag(dq) (dense_Q: dq is dQ), no dG, dh = [-dlb; dub] (a missing
    side's tangent is 0)."""
    dst, _ = st.dense
    dq, dp, dA, db, dlb, dub = tangents
    dQ = dq if (dq is None or dense_Q) else torch.diag_embed(dq)
    dh = None
    if dlb is not None or dub is not None:
        sides = ([None if dlb is None else -dlb] if nlb else []) + ([dub] if has_ub else [])
        like = next(s for s in sides if s is not None)
        sides = [torch.zeros_like(like) if s is None else s for s in sides]
        if any(s.dim() == 2 for s in sides):
            B = next(s.size(0) for s in sides if s.dim() == 2)
            sides = [s if s.dim() == 2 else s.unsqueeze(0).expand(B, s.size(-1)) for s in sides]
        dh = torch.cat(sides, -1)
    return _qp.solve_jvp(dst, (dQ, dp, None, dh, dA, db))


# ---- Jacobians (jacobian() of BoxQPFunction): rows z, lam, nu as bits 0, 1, 2 and columns p, lb, ub, b as bits 0..3 ---
BOX_JAC_WRT = ("p", "lb", "ub", "b")


def box_jacobian_covered(plan, dense_Q=False):
    """True where qpb200_box_jacobian (dense_Q: qpb200_boxq_jacobian) covers a qpb200_box_plan (qpb200_boxq_plan): its
    smem function reports the shared memory."""
    out = ctypes.c_int64(0)
    lib = _lib.load()
    fn = lib.qpb200_boxq_jacobian_smem if dense_Q else lib.qpb200_box_jacobian_smem
    _lib.check(fn(ctypes.byref(plan), ctypes.byref(out)))
    return out.value > 0


def _box_jacobian_kernel(st, rows, cols, J):
    """qpb200_box_jacobian (a dense Q: qpb200_boxq_jacobian) into J (B, R, C) fp64 on st.device."""
    lib = _lib.load()
    with torch.cuda.device(st.device):
        _lib.check((lib.qpb200_boxq_jacobian if st.dense_Q else lib.qpb200_box_jacobian)(
            ctypes.byref(st.plan), st.nBatch, rows, cols, _ptr(st.q), st.sq, _ptr(st.A), st.sA, _ptr(st.lam),
            _ptr(st.slacks), _ptr(J), _stream()))


def _box_jacobian_columns(st, rows, cols, J):
    """J column by column: one solve_box_jvp per column with an un-batched unit tangent of p, lb, ub or b (batch stride
    0), which gives that column for every QP at once."""
    plan = st.plan
    sizes, rsizes = (plan.nz,) * 3 + (plan.neq,), (plan.nz, plan.nineq, plan.neq)
    c0 = 0
    for k in range(4):
        if not (cols >> k) & 1:
            continue
        for j in range(sizes[k]):
            t = torch.zeros(sizes[k], dtype=torch.float64, device=st.device)
            t[j] = 1.0
            tans = [None] * 6
            tans[(1, 4, 5, 3)[k]] = t                    # (dq, dp, dA, db, dlb, dub): dp, dlb, dub or db
            outs = solve_box_jvp(st, tans)
            r0 = 0
            for i in range(3):
                if (rows >> i) & 1:
                    J[:, r0:r0 + rsizes[i], c0 + j] = outs[i]
                    r0 += rsizes[i]
        c0 += sizes[k]


def _box_jacobian_dense(st, rows, cols, nlb, J):
    """The dense fallback: _qp.solve_jacobian on the dense equivalent, whose lam rows are already [lb rows; ub rows];
    h = [-lb; ub] gives J_lb = -J_h[:, :, :nlb] and J_ub = J_h[:, :, nlb:]."""
    dst, _ = st.dense
    n, m, e = dst.plan.nz, dst.plan.nineq, dst.plan.neq
    Jd = _qp.solve_jacobian(dst, rows, (cols & 1) | (2 if cols & 6 else 0) | (4 if cols & 8 else 0))
    src, c0 = 0, 0
    if cols & 1:
        J[:, :, :n] = Jd[:, :, :n]
        src, c0 = n, n
    if cols & 6:
        if cols & 2:
            J[:, :, c0:c0 + n] = -Jd[:, :, src:src + nlb]
            c0 += n
        if cols & 4:
            J[:, :, c0:c0 + n] = Jd[:, :, src + nlb:src + m]
            c0 += n
        src += m
    if cols & 8:
        J[:, :, c0:c0 + e] = Jd[:, :, src:src + e]


def solve_box_jacobian(st, rows, cols, nlb):
    """d(zhat, lam, nu)/d(p, lb, ub, b) at the returned point of `st`, per QP: fp64 (B, R, C) on st.device, rows
    [z; lam; nu] and columns [p, lb, ub, b] restricted to the bits of `rows` / `cols`. nlb: nz if lb was given, else 0.
    One qpb200_box_jacobian (dense Q: qpb200_boxq_jacobian) call where the kernel covers the plan; otherwise one
    solve_box_jvp per column, and on the dense fallback the dense path's solve_jacobian."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    plan = st.plan
    n, m, e = plan.nz, plan.nineq, plan.neq
    R = sum((n, m, e)[i] for i in range(3) if (rows >> i) & 1)
    C = sum((n, n, n, e)[k] for k in range(4) if (cols >> k) & 1)
    J = torch.empty(st.nBatch, R, C, dtype=torch.float64, device=st.device)
    if st.dense is not None:
        _box_jacobian_dense(st, rows, cols, nlb, J)
    elif box_jacobian_covered(plan, st.dense_Q):
        _box_jacobian_kernel(st, rows, cols, J)
    else:
        _box_jacobian_columns(st, rows, cols, J)
    return J


def box_jacobian_of(st, out, sides, wrt, duals):
    """The `jacobian` attribute of BoxQPFunction on the state `st` of its last forward, whose output had
    out = (device, dtype) and sides = (nlb, has_ub). Returns {name: (B, rows, n_name)} for each name of `wrt` (None:
    every input the problem has), rows z, or [z; lam; nu] with duals."""
    if st is None:
        raise RuntimeError("qpth_b200: jacobian() needs a forward call of this function first")
    nlb, has_ub = sides
    n, e = st.plan.nz, st.plan.neq
    present = ("p",) + (("lb",) if nlb else ()) + (("ub",) if has_ub else ()) + (("b",) if e > 0 else ())
    names = present if wrt is None else ((wrt,) if isinstance(wrt, str) else tuple(wrt))
    if not names:
        raise ValueError("qpth_b200: jacobian(wrt=...) needs at least one of %s" % (present,))
    for nm in names:
        if nm in ("q", "Q", "A"):
            raise ValueError(
                "qpth_b200: jacobian(wrt=...) does not take %r; contract the blocks it does give: J_.,q = J_.,p diag(z) "
                "for a diagonal q, J_.,Q_ik = J_.,p_i z_k for a dense Q (which enters as sym(dQ)), and "
                "J_.,A_ck = J_.,p_k nu_c - J_.,b_c z_k" % nm)
        if nm not in BOX_JAC_WRT:
            raise ValueError("qpth_b200: jacobian(wrt=...) takes %s, not %r" % (BOX_JAC_WRT, nm))
        if nm not in present:
            raise ValueError("qpth_b200: jacobian(wrt=%r): this problem has no %s" % (
                nm, "equality constraints (neq == 0)" if nm == "b" else "%s side" % nm))
    cols = sum(1 << BOX_JAC_WRT.index(nm) for nm in set(names))
    rows = 1 | ((2 | (4 if e > 0 else 0)) if duals else 0)
    J = solve_box_jacobian(st, rows, cols, nlb)
    res, c0 = {}, 0
    for k, nm in enumerate(BOX_JAC_WRT):
        if (cols >> k) & 1:
            w = e if nm == "b" else n
            res[nm] = J[:, :, c0:c0 + w]
            c0 += w
    device, dtype = out
    return {nm: res[nm].to(device=device, dtype=dtype).contiguous() for nm in names}


def BoxQPFunction(eps=1e-12, verbose=0, notImprovedLim=3, maxIter=20, check_Q_spd=True, duals=False, dense_Q=False):
    """Factory with QPFunction's options; returns f(q, p, A, b, lb, ub) -> z (nBatch, nz).

    q, p, lb, ub: (nBatch, nz) or (nz); A: (nBatch, neq, nz), (neq, nz) or an empty tensor; b follows A. lb or ub may
    be None (no bound on that side), not both. f.last_solve() returns the state of the last forward: lam, slacks
    ([lb rows; ub rows]), nus, iters, best_resid.

    duals=True: f returns (z, lam, nu) as QPFunction(duals=True) does: lam (nBatch, nineq) in the [lb rows; ub rows]
    layout of last_solve(), nu (nBatch, neq) or (nBatch, 0), and a loss may use all three.

    Forward mode (torch.autograd.forward_ad) is supported as for QPFunction: rx = dq o z + dp + dA' nu, rz = [dlb; -dub],
    ry = dA z - db on the right-hand side of the backward's solve (qpb200_box_jvp; the dense fallback maps the tangents
    to its dense equivalent, dQ = diag(dq), dh = [-dlb; dub]).

    dense_Q=True: the first argument is a dense Q, (nBatch, nz, nz) or (nz, nz) (a 2-D Q is un-batched), of which only
    the lower triangle is read, as in QPFunction's kernels (the dense fallback too): the strictly upper triangle may hold
    anything, NaN included, and the result is that of the symmetric matrix tril(Q) + tril(Q, -1)^T. A tangent dQ is
    read in full and enters as sym(dQ). Everything else is as above, with QPFunction's semantics on
    the dense equivalent (Q, G = [-I; I], h = [-lb; ub]): 'Q is not SPD.' where chol(Q) breaks down, the gradient
    dQ = 1/2 (dx z' + z dx') (the batch mean for an un-batched Q), and the tangent dQ enters forward mode as
    sym(dQ) z. Shapes past the dense-Q kernels (qpb200_boxq_plan.ok) run the dense kernels on the dense equivalent.

    f.jacobian(wrt=None, duals=False) -> {name: tensor}: the whole Jacobians of the last forward's solution with respect
    to p, lb, ub and b, per QP (also for an un-batched input: the true derivative, not a batch mean). wrt=None means
    every input the problem has: p, the sides given, and b when neq > 0. J["p"] is (nBatch, nz, nz) = dz*/dp, J["lb"]
    and J["ub"] (nBatch, nz, nz), J["b"] (nBatch, nz, neq); duals=True gives the rows [z; lam; nu] (lam in the
    [lb rows; ub rows] layout, nu only when neq > 0). They are taken at the returned point with the backward's clamped
    D = [d_lb; d_ub], so J t equals the forward-mode tangent of t: with H = Q + diag(d_lb + d_ub) and
    X = [H A'; A 0]^-1, J_z,p = -X_zz, J_z,b = X_zn, J_z,lb = -J_z,p diag(d_lb), J_z,ub = -J_z,p diag(d_ub), and the
    lam rows are d_lb o (rz_lb - z) and d_ub o (rz_ub + z) of the same column (rz_lb = e_j in lb column j, rz_ub = -e_j
    in ub column j). One kernel call factors once per QP and solves for every column: with a diagonal q
    (qpb200_box_jacobian) M = A H^-1 A', with a dense Q (qpb200_boxq_jacobian) the bordered [H A'; A 0] as the forward
    does. Shapes whose factor or column buffers do not fit one CTA take one JVP per column, and the dense fallback the
    dense path's jacobian. Jacobians with respect to q, Q and A are contractions of these:
    J_.,q = J_.,p diag(z), J_.,Q_ik = J_.,p_i z_k (sym(dQ) enters), J_.,A_ck = J_.,p_k nu_c - J_.,b_c z_k. The result has
    the dtype and device of the forward's output and is not differentiable.

    Second order: under `torch.autograd.grad(..., create_graph=True)` the gradients are differentiable again, in the
    incoming gradients of z, lam, nu and in q (Q), p, A, b, lb, ub (Hessian-vector products,
    `torch.autograd.functional.hessian`, gradient penalties, meta-learning through a sudoku layer or a projection). The
    double backward is the exact derivative of the backward as computed (the clamped D included), on the layout that
    solved the forward: one box JVP solve, one dual backward solve and two bandwidth-bound kernels
    (qpb200_box_double_backward; a dense Q: qpb200_boxq_double_backward). The cotangent of an un-batched input's
    gradient (a batch mean) is shared by every QP, and that input's second-order gradient is the batch sum. The dense
    fallback goes through QPFunction's double backward on the dense equivalent. Without create_graph nothing changes.
    Third order raises."""
    _last = [None]
    _jac = [None, None, None]            # the state, (device, dtype) and (nlb, has_ub) of the last forward

    class BoxQPFunctionFn(Function):
        @staticmethod
        def forward(ctx, q_, p_, A_, b_, lb_, ub_):
            st = solve_box_forward(q_, p_, A_, b_, lb_, ub_, eps, verbose, notImprovedLim, maxIter, check_Q_spd,
                                   dense_Q)
            if st is None:
                st = solve_dense_forward(q_, p_, A_, b_, lb_, ub_, eps, verbose, notImprovedLim, maxIter, check_Q_spd,
                                         dense_Q)
            ctx.st = st
            _last[0] = st
            zhats = st.zhat.to(device=q_.device, dtype=q_.dtype)
            ctx.save_for_backward(zhats, q_, p_, A_, b_, lb_, ub_)
            ctx.lams, ctx.slacks, ctx.nus = st.lam, st.slacks, st.nus
            ctx.out = (q_.device, q_.dtype)
            ctx.sides = (q_.size(-1) if lb_ is not None else 0, ub_ is not None)
            _jac[:] = [st, ctx.out, ctx.sides]
            ctx.set_materialize_grads(False)
            if not duals:
                return zhats
            return (zhats,) + _qp.dual_outputs(st, q_)

        @staticmethod
        def jvp(ctx, dq, dp, dA, db, dlb, dub):
            tangents = (dq, dp, dA, db, dlb, dub)
            st = ctx.st
            if st.dense is not None:
                out = dense_jvp(st, tangents, *ctx.sides, dense_Q=dense_Q)
            else:
                out = solve_box_jvp(st, tangents)
            return _qp.jvp_outputs(*out, ctx.out, duals)

        @staticmethod
        def backward(ctx, dl_dzhat, dl_dlam=None, dl_dnu=None):
            zhats, q, p, A, b, lb, ub = ctx.saved_tensors
            st = ctx.st
            ins = (q, p, A, b, lb, ub)
            ranks = (3 if dense_Q else 2, 2, 3, 2, 2, 2)
            flags = [X is not None and X.nelement() > 0 and X.dim() == r - 1 for X, r in zip(ins, ranks)]
            want = list(ctx.needs_input_grad)
            if torch.is_grad_enabled():          # create_graph=True: gradients that can be differentiated again
                if st.dense is None:
                    return BoxQPBackwardFn.apply(st, flags, want, dl_dzhat, dl_dlam, dl_dnu, *ins)
                return dense_backward_graph(st, dl_dzhat, flags, want, ins, dl_dlam, dl_dnu, dense_Q)
            if st.dense is None:
                outs = solve_box_backward(st, dl_dzhat, flags, want, dl_dlam, dl_dnu)
            else:
                outs = dense_backward(st, dl_dzhat, flags, want, q.size(-1) if lb is not None else 0, ub is not None,
                                      dl_dlam, dl_dnu, dense_Q)
            return tuple(None if (g is None or X is None or not w) else g.to(device=X.device, dtype=X.dtype)
                         for X, g, w in zip(ins, outs, want))

    def apply(q, p, A, b, lb, ub):
        return BoxQPFunctionFn.apply(q, p, A, b, lb, ub)

    def jacobian(wrt=None, duals=False):
        return box_jacobian_of(_jac[0], _jac[1], _jac[2], wrt, duals)

    apply.last_solve = lambda: _last[0]
    apply.jacobian = jacobian
    return apply
