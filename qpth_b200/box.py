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
    _lib.load()
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
        _lib.check(_entry(st, "forward")(
            ctypes.byref(plan), nBatch, _ptr(q), st.sq, _ptr(p), stride(p, 2, nz), _ptr(A), st.sA,
            _ptr(b), stride(b, 2, neq), _ptr(lb), stride(lb, 2, nz), _ptr(ub), stride(ub, 2, nz),
            float(eps), float(_qp.STALL_TOL), float(_qp.BEST_TIE), int(notImprovedLim), int(maxIter),
            _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(st.iters), _ptr(st.best_resid),
            _ptr(st.trace), _ptr(spd), _stream()))
        _qp.diagnostics(spd, st, check_Q_spd, verbose)
    return st


def _entry(st, name):
    """The C entry point `name` of the layout of `st`: qpb200_boxq_<name> with a dense Q, else qpb200_box_<name>."""
    return getattr(_lib.load(), ("qpb200_boxq_" if st.dense_Q else "qpb200_box_") + name)


def _call(st, name, middle, tail):
    """Check the C call `name` of the layout of `st` with its arguments: plan, nBatch, (q, sq, A, sA), `middle`, the
    returned point (zhat, lam, slacks, nus), `tail`, the stream."""
    _lib.check(_entry(st, name)(ctypes.byref(st.plan), st.nBatch, _ptr(st.q), st.sq, _ptr(st.A), st.sA, *middle,
                                _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), *tail, _stream()))


def _grads(st, flags, want):
    """The gradient outputs of the box layouts and their C arguments, in the ABI's order (dq, dp, dlb, dub, dA, db)."""
    plan = st.plan
    nz, neq = plan.nz, plan.neq
    shapes = [(nz, nz) if st.dense_Q else (nz,), (nz,), (neq, nz), (neq,), (nz,), (nz,)]
    absent = (False, False, neq == 0, neq == 0, not plan.has_lb, not plan.has_ub)
    return _qp.grad_buffers(shapes, flags, want, absent, st.nBatch, st.device, (0, 1, 4, 5, 2, 3))


def _ranks(st):
    return (3 if st.dense_Q else 2, 2, 3, 2, 2, 2)


def solve_box_backward(st, dl_dzhat, mean_flags, want, dl_dlam=None, dl_dnu=None, keep=False):
    """Gradients (dq, dp, dA, db, dlb, dub) on the device; mean_flags / want: 6-tuples in that order. dl_dlam ([lb rows;
    ub rows]) / dl_dnu: the gradients with respect to the returned duals (None: zero); dl_dzhat None: zero. With a
    dense Q the first is dQ, (B, nz, nz) or (nz, nz) with its mean flag. keep: also return the solve (dxv, dlamv,
    dnuv), which the double backward reads."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    with torch.cuda.device(device):
        dl = (_qp._adjoint(dl_dzhat, B, nz, device) if dl_dzhat is not None
              else torch.zeros(B, nz, dtype=torch.float64, device=device))
        glam, gnu = _qp._adjoint(dl_dlam, B, m, device), _qp._adjoint(dl_dnu, B, neq, device)
        outs, grads = _grads(st, mean_flags, want)
        v = _qp.solve_triple(B, nz, m, neq, device)
        if glam is None and gnu is None and not st.dense_Q:     # no dual was used: the entry point of a zhat-only loss
            _call(st, "backward", (_ptr(dl),), (*grads, *(_ptr(x) for x in v)))
        else:
            _call(st, "backward_duals", (_ptr(dl), _ptr(glam), _ptr(gnu)), (*grads, *(_ptr(x) for x in v)))
    return (outs, v) if keep else outs


def solve_box_double_backward(st, v, omegas, flags, want):
    """The double backward on the device (qpb200_box_double_backward / qpb200_boxq_double_backward): v = (dxv, dlamv,
    dnuv) of the first backward at the point of `st`; omegas: the cotangents of its six outputs (dq, dp, dA, db, dlb,
    dub; dQ with a dense Q), each None or shaped as that output; flags: the first backward's mean flags (an un-batched
    input: its cotangent is divided by nBatch, and its second-order gradient is the batch sum); want: which of the six
    gradients to write. Returns fp64 (gg_z, gg_lam, gg_nu, dq, dp, dA, db, dlb, dub): the gradients of g_z, g_lam, g_nu
    (gg_nu None without equality rows) and of the six inputs (None where not wanted or absent)."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    absent = (False, False, neq == 0, neq == 0, not plan.has_lb, not plan.has_ub)
    with torch.cuda.device(device):
        om = [None if (w is None or absent[k]) else (_dev64(w, device) / B if flags[k] else _dev64(w, device))
              for k, w in enumerate(omegas)]
        tans = _qp.tangent_args(om, _ranks(st), (nz * nz if st.dense_Q else nz, nz, neq * nz, neq, nz, nz))
        outs, grads = _grads(st, flags, want)
        gg = _qp.solve_triple(B, nz, m, neq, device)
        # QPB200_DOUBLE_BACKWARD_WORK
        work = torch.empty(B * (2 * nz + 3 * m + 2 * neq), dtype=torch.float64, device=device)
        _call(st, "double_backward", (*tans, *(_ptr(x) for x in v)), (*(_ptr(x) for x in gg), *grads, _ptr(work)))
    return list(gg) + outs


def solve_box_jvp(st, tangents):
    """The JVP of (zhat, lam, nu) at the returned point on the device. tangents: (dq, dp, dA, db, dlb, dub), each None
    (zero), batched or un-batched as its input (with a dense Q, dQ first). Returns fp64 (dz (B,nz), dlam (B,nineq) in
    the [lb rows; ub rows] layout, dnu (B,neq) or None); one qpb200_box_jvp / qpb200_boxq_jvp call: the right-hand side
    kernel and the backward's solve."""
    if _qp._pending:
        _qp.flush_checks(wait=False)
    plan, B, device = st.plan, st.nBatch, st.device
    nz, neq, m = plan.nz, plan.neq, plan.nineq
    with torch.cuda.device(device):
        tans = [None if t is None else _dev64(t, device) for t in tangents]
        per = (nz * nz if st.dense_Q else nz, nz, neq * nz, neq, nz if plan.has_lb else 0, nz if plan.has_ub else 0)
        args = _qp.tangent_args(tans, _ranks(st), per)
        rhs = torch.empty(B * (nz + m + neq), dtype=torch.float64, device=device)
        dz, dlam, dnu = _qp.solve_triple(B, nz, m, neq, device)
        _call(st, "jvp", args, (_ptr(rhs), _ptr(dz), _ptr(dlam), _ptr(dnu)))
    return dz, dlam, dnu


# ---- shapes beyond the box kernels: the dense kernels on the dense equivalent ---------------------------------------
def _side_rows(lo, hi):
    """The right-hand side h = [lo; hi] of the sides given (None: absent), batched where either side is."""
    sides = [s for s in (lo, hi) if s is not None]
    if any(s.dim() == 2 for s in sides):
        B = next(s.size(0) for s in sides if s.dim() == 2)
        sides = [s if s.dim() == 2 else s.unsqueeze(0).expand(B, s.size(-1)) for s in sides]
    return torch.cat(sides, -1)


def dense_equivalent(q, lb, ub, dense_Q=False):
    """(Q, G, h) of QPFunction for a box QP: Q = diag(q) (dense_Q: q itself), G = [-I; I] (sides given),
    h = [-lb; ub]. Batched where q (for Q) or either bound (for h) is batched."""
    nz = q.size(-1)
    Q = q if dense_Q else torch.diag_embed(q)
    eye = torch.eye(nz, dtype=q.dtype, device=q.device)
    G = torch.cat(([-eye] if lb is not None else []) + ([eye] if ub is not None else []), 0)
    return Q, G, _side_rows(None if lb is None else -lb, ub)


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


def dense_backward(st, dl, mean_flags, want, ins, dl_dlam=None, dl_dnu=None, dense_Q=False):
    """The backward on the dense equivalent, mapped back to (dq, dp, dA, db, dlb, dub). The dense equivalent's rows are
    lam's [lb rows; ub rows]: the dual adjoints pass through as they are. Without create_graph: qp.solve_backward on
    the stored state. Under create_graph=True: (Q, h) built from the inputs with torch ops, qp.backward_graph on them
    (G constant) and the map back in torch ops, so that the gradients can be differentiated once more."""
    dst, h_shared = st.dense
    q, p, A, b, lb, ub = ins
    mq, mp, mA, mb, mlb, mub = mean_flags
    flags = (mq, mp, True, h_shared, mA, mb)
    dwant = (want[0], want[1], False, want[4] or want[5], want[2], want[3])
    if torch.is_grad_enabled():
        Q, G, h = dense_equivalent(q, lb, ub, dense_Q)
        empty = torch.empty(0, dtype=q.dtype, device=q.device)
        A_ = A if (A is not None and A.nelement() > 0) else empty
        b_ = b if (b is not None and b.nelement() > 0) else empty
        dQ, dp, _, dh, dA, db = _qp.backward_graph(dst, flags, dwant, dl, dl_dlam, dl_dnu, Q, p, G, h, A_, b_)
    else:
        dQ, dp, _, dh, dA, db = _qp.solve_backward(dst, dl, flags, dwant, dl_dlam, dl_dnu)
    nlb = q.size(-1) if lb is not None else 0
    dq = dQ if (dQ is None or dense_Q) else torch.diagonal(dQ, dim1=-2, dim2=-1).contiguous()
    dlb = dub = None
    if dh is not None:
        if want[4] and nlb:
            dlb = -dh[..., :nlb]
            dlb = dlb.mean(0) if (mlb and dlb.dim() == 2) else dlb
        if want[5] and ub is not None:
            dub = dh[..., nlb:]
            dub = dub.mean(0) if (mub and dub.dim() == 2) else dub
    return [dq, dp, dA, db, dlb, dub]


def dense_jvp(st, tangents, nlb, has_ub, dense_Q=False):
    """solve_box_jvp on the dense equivalent: dQ = diag(dq) (dense_Q: dq is dQ), no dG, dh = [-dlb; dub] (a missing
    side's tangent is 0)."""
    dst, _ = st.dense
    dq, dp, dA, db, dlb, dub = tangents
    dQ = dq if (dq is None or dense_Q) else torch.diag_embed(dq)
    dh = None
    if dlb is not None or dub is not None:
        like = dlb if dlb is not None else dub
        dh = _side_rows((torch.zeros_like(like) if dlb is None else -dlb) if nlb else None,
                        (torch.zeros_like(like) if dub is None else dub) if has_ub else None)
    return _qp.solve_jvp(dst, (dQ, dp, None, dh, dA, db))


# ---- Jacobians (jacobian() of BoxQPFunction): rows z, lam, nu as bits 0, 1, 2 and columns p, lb, ub, b as bits 0..3 ---
BOX_JAC_WRT = ("p", "lb", "ub", "b")
BOX_JAC_SLOTS = (1, 4, 5, 3)      # their tangents' slots in (dq, dp, dA, db, dlb, dub)


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
    with torch.cuda.device(st.device):
        _lib.check(_entry(st, "jacobian")(
            ctypes.byref(st.plan), st.nBatch, rows, cols, _ptr(st.q), st.sq, _ptr(st.A), st.sA, _ptr(st.lam),
            _ptr(st.slacks), _ptr(J), _stream()))


def _box_jacobian_columns(st, rows, cols, J):
    """qp.jacobian_columns for the columns p, lb, ub and b: unit tangents through solve_box_jvp."""
    _qp.jacobian_columns(st, rows, cols, J, (st.plan.nz,) * 3 + (st.plan.neq,), BOX_JAC_SLOTS, solve_box_jvp)


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
    n = st.plan.nz
    if st.dense is not None:
        fill = lambda st_, rows_, cols_, J: _box_jacobian_dense(st_, rows_, cols_, nlb, J)   # noqa: E731
    else:
        fill = _box_jacobian_kernel if box_jacobian_covered(st.plan, st.dense_Q) else _box_jacobian_columns
    return _qp.jacobian_matrix(st, rows, cols, (n, n, n, st.plan.neq), fill)


def _box_refusal(nm):
    if nm in ("q", "Q", "A"):
        return ("qpth_b200: jacobian(wrt=...) does not take %r; contract the blocks it does give: "
                "J_.,q = J_.,p diag(z) for a diagonal q, J_.,Q_ik = J_.,p_i z_k for a dense Q (which enters as sym(dQ)), "
                "and J_.,A_ck = J_.,p_k nu_c - J_.,b_c z_k" % nm)
    if nm not in BOX_JAC_WRT:
        return "qpth_b200: jacobian(wrt=...) takes %s, not %r" % (BOX_JAC_WRT, nm)
    return "qpth_b200: jacobian(wrt=%r): this problem has no %s" % (
        nm, "equality constraints (neq == 0)" if nm == "b" else "%s side" % nm)


def box_jacobian_of(st, out, sides, wrt, duals):
    """The `jacobian` attribute of BoxQPFunction on the state `st` of its last forward, whose output had
    out = (device, dtype) and sides = (nlb, has_ub): qp.jacobian_of on the columns p, lb, ub, b (wrt=None: every input
    the problem has)."""
    return _qp.jacobian_of(
        st, out, wrt, duals,
        lambda plan: tuple(zip(BOX_JAC_WRT, (plan.nz, sides[0], plan.nz if sides[1] else 0, plan.neq))),
        lambda st_, rows, cols: solve_box_jacobian(st_, rows, cols, sides[0]), _box_refusal)


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
            _last[0] = st
            ctx.sides = (q_.size(-1) if lb_ is not None else 0, ub_ is not None)
            out = _qp.layer_outputs(ctx, st, (q_, p_, A_, b_, lb_, ub_), duals)
            _jac[:] = [st, ctx.out, ctx.sides]
            return out

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
            if st.dense is not None:
                outs = dense_backward(st, dl_dzhat, flags, want, ins, dl_dlam, dl_dnu, dense_Q)
            elif torch.is_grad_enabled():        # create_graph=True: gradients that can be differentiated again
                return _qp.BackwardFn.apply(lambda *a: solve_box_backward(*a, keep=True), solve_box_double_backward,
                                            st, flags, want, dl_dzhat, dl_dlam, dl_dnu, *ins)
            else:
                outs = solve_box_backward(st, dl_dzhat, flags, want, dl_dlam, dl_dnu)
            return tuple(_qp._cast(g, X) for X, g in zip(ins, outs))

    def apply(q, p, A, b, lb, ub):
        return BoxQPFunctionFn.apply(q, p, A, b, lb, ub)

    def jacobian(wrt=None, duals=False):
        return box_jacobian_of(_jac[0], _jac[1], _jac[2], wrt, duals)

    apply.last_solve = lambda: _last[0]
    apply.jacobian = jacobian
    return apply
