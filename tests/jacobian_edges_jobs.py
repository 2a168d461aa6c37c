"""GPU jobs of tests/test_gpu_jacobian_edges.py, run in one child process with a timeout: python -m
tests.jacobian_edges_jobs <out_dir> writes <out_dir>/<job>.npz (or .err with its traceback) and each job's name to
<out_dir>/progress.txt as it starts. The checks that need the full J run here, on the device or against the numpy
references, and each job saves what they measured (counts, relative errors), not J itself.

- `sweep_*`: the mask sweep. The kernel's C entry point (qp._jacobian_kernel, box._box_jacobian_kernel) writes J into
  a view in the middle of a larger buffer, guard bands of max(4096, 2 C) doubles of SENTINEL on either side and the
  view filled with NaN, for every row mask the problem allows and every non-empty column subset, with per-QP and with
  shared inputs. Per call: NaN left in the view, guard doubles changed, and elements not bit-identical to the same rows
  and columns of the full-mask J. Each warp solves its 8-column block with the same instructions whatever the masks,
  and nothing is reduced across warps, so any difference is a placement or scheduling fault, not rounding.
- `edge_*`: every entry of tests/jacobian_edges.py at a point (lam, s ~ U(0.1, 10)): the full J against the dense
  model (the per-variable model without equality rows), J t against the JVP of batched tangents, g' J against the dual
  backward, the symmetry / box identities; and for the next shape, no coverage and the column path's J_z,p.
- `api_*`: the public jacobian() at converged solves: the default call, wrt out of order and repeated, mixed sharing,
  and a BoxQPFunction forward on the widest both-sided plan.
"""
import itertools
import os
import sys
import traceback

import numpy as np
import torch

from tests import box_jacobian_models as bm
from tests import jacobian_edges as je
from tests import jacobian_models as jm

DEV = "cuda:0"
B = 3
SENTINEL = -1234.5


def _T(a):
    return torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _rel_to(a, b, full):
    """a block against b relative to the whole reference J (J_z,p is ~0 where A is square: z is fixed by A z = b)"""
    return float(np.abs(a - b).max() / max(np.abs(full).max(), 1e-300))


# ---- states at a point ----------------------------------------------------------------------------------------------

def jac_point(shape, seed, Bn=B):
    """wellcond_qp_batch (cond(Q) <= 9) with z, nu ~ N(0, 1), lam, s ~ U(0.1, 10), the random tangents of p, h, b and
    the loss weights of z, lam, nu"""
    from tests.kernel_families import wellcond_qp_batch
    n, m, e = shape
    pr = wellcond_qp_batch(Bn, n, m, e, seed=seed)
    rs = np.random.RandomState(seed + 1)
    pr.update(z=rs.randn(Bn, n), nu=rs.randn(Bn, e), lam=rs.uniform(0.1, 10, (Bn, m)), s=rs.uniform(0.1, 10, (Bn, m)),
              tp=rs.randn(Bn, n), th=rs.randn(Bn, m), tb=rs.randn(Bn, e), glam=rs.randn(Bn, m), gnu=rs.randn(Bn, e))
    return pr


def jac_state(pr, shared):
    """pre_factor_kkt on the default plan (plan_for) and the point's solution; shared: QP 0's Q, G, A for every QP"""
    from qpth_b200.solution import pre_factor_state
    e = pr["A"].shape[1]
    E = torch.empty(0, dtype=torch.float64, device=DEV)
    mat = lambda k: _T(pr[k][0] if shared else pr[k])
    return pre_factor_state(mat("Q"), _T(pr["p"]), mat("G"), _T(pr["h"]), mat("A") if e else E,
                            _T(pr["b"]) if e else E, _T(pr["z"]), _T(pr["lam"]), _T(pr["s"]),
                            _T(pr["nu"]) if e else E)


def box_state(kind, name, shared, Bn=B):
    """(plan, point, state) of a BOX or BOXQ entry (tests/box_jacobian_jobs.point: lam, s ~ U(0.1, 10))"""
    from qpth_b200 import _lib
    from tests.box_jacobian_jobs import point, state
    from tests.boxq_families import check_entry
    dense_Q = kind == "boxq"
    if dense_Q:
        plan = check_entry(name)
    else:
        n, e, sides = je.BOX[name]["shape"]
        plan = _lib.box_plan_for(n, e, *je.sides_flags(sides))
    pt = point(plan, 17, dense_Q, Bn=Bn)
    return plan, pt, state(plan, pt, shared, dense_Q)


def full_masks(kind, plan):
    if kind == "jac":
        return (7, 7) if plan.neq else (3, 3)
    return (7 if plan.neq else 3), 1 | (2 if plan.has_lb else 0) | (4 if plan.has_ub else 0) | (8 if plan.neq else 0)


def _bits(mask):
    return [i for i in range(4) if (mask >> i) & 1]


def _index(mask, widths):
    off = np.cumsum([0] + list(widths))
    return np.concatenate([np.arange(off[i], off[i + 1]) for i in _bits(mask)])


def widths(kind, plan):
    """(row block widths, column block widths) of the full J"""
    n, m, e = plan.nz, plan.nineq, plan.neq
    if kind == "jac":
        return (n, m, e), (n, m, e)
    return (n, m, e), (n, n if plan.has_lb else 0, n if plan.has_ub else 0, e)


def kernel(kind, st, rows, cols, J):
    from qpth_b200 import box, qp
    (qp._jacobian_kernel if kind == "jac" else box._box_jacobian_kernel)(st, rows, cols, J)


# ---- the mask sweep -------------------------------------------------------------------------------------------------

def guarded(kind, st, rows, cols, R, C):
    """The kernel into a NaN-filled (B, R, C) view between guard bands of SENTINEL: (J, NaN left in J, guard doubles
    changed)"""
    G, size = max(4096, 2 * C), st.nBatch * R * C
    buf = torch.full((2 * G + size,), SENTINEL, dtype=torch.float64, device=DEV)
    J = buf[G:G + size].view(st.nBatch, R, C)
    J.fill_(float("nan"))
    kernel(kind, st, rows, cols, J)
    bits = torch.tensor([SENTINEL], dtype=torch.float64).view(torch.int64).item()
    guards = torch.cat([buf[:G], buf[G + size:]]).view(torch.int64)
    return J, int(torch.isnan(J).sum()), int((guards != bits).sum())


def sweep_job(kind, name):
    out = {}
    for shared in (False, True):
        if kind == "jac":
            st = jac_state(jac_point(je.JAC[name]["shape"], 31), shared)
        else:
            _, _, st = box_state(kind, name, shared)
        R0, C0 = full_masks(kind, st.plan)
        rw, cw = widths(kind, st.plan)
        Jfull, nan, guard = guarded(kind, st, R0, C0, len(_index(R0, rw)), len(_index(C0, cw)))
        res = [(R0, C0, nan, guard, 0)]
        for rows, cols in itertools.product(range(1, R0 + 1), range(1, C0 + 1)):
            if (rows & ~R0) or (cols & ~C0) or (rows, cols) == (R0, C0):
                continue
            ri = torch.tensor(_index(rows, rw), device=DEV)
            ci = torch.tensor(_index(cols, cw), device=DEV)
            J, nan, guard = guarded(kind, st, rows, cols, len(ri), len(ci))
            ref = Jfull.index_select(1, ri).index_select(2, ci)
            res.append((rows, cols, nan, guard, int((J.view(torch.int64) != ref.view(torch.int64)).sum())))
        torch.cuda.synchronize()
        out["shared" if shared else "batched"] = np.array(res, dtype=np.int64)
    return out


# ---- the edge shapes against the references -------------------------------------------------------------------------

def jac_edge_job(name):
    from qpth_b200 import qp
    ent = je.JAC[name]
    n, m, e = ent["shape"]
    pr = jac_point(ent["shape"], 41)
    st = jac_state(pr, False)
    out = dict(covered=qp.jacobian_covered(st.plan), layout=np.array(je.jac_plan_layout(st.plan)))
    J = qp.solve_jacobian(st, *full_masks("jac", st.plan))
    tans = (None, _T(pr["tp"]), None, _T(pr["th"]), None, _T(pr["tb"]) if e else None)
    dz, dlam, dnu = qp.solve_jvp(st, tans)
    grads = qp.solve_backward(st, _T(pr["dl"]), (False,) * 6, (False, True, False, True, False, bool(e)),
                              _T(pr["glam"]), _T(pr["gnu"]) if e else None)
    t = torch.cat([_T(pr["tp"]), _T(pr["th"])] + ([_T(pr["tb"])] if e else []), 1)
    jvp = torch.cat([dz, dlam] + ([dnu] if e else []), 1)
    g = torch.cat([_T(pr["dl"]), _T(pr["glam"])] + ([_T(pr["gnu"])] if e else []), 1)
    gJ = torch.cat([grads[1], grads[3]] + ([grads[5]] if e else []), 1)
    err = dict(ref=[], jvp=[], grad=[], sym=[])
    for i in range(B):
        Ji = J[i].cpu().numpy()
        if i == 0 or je.order("jac", ent["shape"]) <= 3000:
            Jd = jm.dense_jacobian(pr["Q"][i], pr["G"][i], pr["A"][i] if e else None, pr["lam"][i], pr["s"][i])
            err["ref"].append(_rel(Ji, Jd))
        err["jvp"].append(_rel((J[i] @ t[i]).cpu().numpy(), jvp[i].cpu().numpy()))
        err["grad"].append(_rel((g[i] @ J[i]).cpu().numpy(), gJ[i].cpu().numpy()))
        err["sym"].append(jm.symmetry_residuals(Ji, n, m, e) / np.abs(Ji).max())
    out.update({"err_" + k: np.array(v) for k, v in err.items()})
    if ent["next"] is not None:
        rc, nplan = je.jac_plan(*ent["next"])
        out["next_rc"] = np.array(rc)
        if rc == 0:
            out["next_covered"] = qp.jacobian_covered(nplan)
            # the column path on one QP, the columns of p only
            npr = jac_point(ent["next"], 43, Bn=1)
            nst = jac_state(npr, False)
            Jzp = qp.solve_jacobian(nst, 1, 1)[0].cpu().numpy()
            nn = ent["next"][0]
            Jd = jm.dense_jacobian(npr["Q"][0], npr["G"][0], npr["A"][0] if ent["next"][2] else None, npr["lam"][0],
                                   npr["s"][0])
            out["next_err"] = np.array(_rel_to(Jzp, Jd[:nn, :nn], Jd))
    return out


def box_reference(kind, plan, pt, i):
    """the high-precision reference of QP i: the dense model, or the per-variable one without equality rows"""
    n, e = plan.nz, plan.neq
    nlb = n if plan.has_lb else 0
    if kind == "box" and e == 0:
        return bm.diagonal_box_jacobian(pt["q"][i], pt["lam"][i], pt["s"][i], nlb, bool(plan.has_ub))
    Q = pt["q"][i] if kind == "boxq" else np.diag(pt["q"][i])
    return bm.dense_box_jacobian(Q, pt["A"][i] if e else None, pt["lam"][i], pt["s"][i], nlb, bool(plan.has_ub))


def box_edge_job(kind, name):
    from qpth_b200 import box
    tab = je.BOX if kind == "box" else je.BOXQ
    ent = tab[name]
    n, e, sides = ent["shape"]
    Bn = 1 if (kind == "box" and e == 0 and n > 1000) else B      # the widest J: 5760 x 5760 and more per QP
    plan, pt, st = box_state(kind, name, False, Bn)
    nlb, has_ub = (n if plan.has_lb else 0), bool(plan.has_ub)
    out = dict(covered=box.box_jacobian_covered(plan, kind == "boxq"), fwd=np.array(je.box_forward(plan))
               if kind == "box" else np.array("boxq"))
    R0, C0 = full_masks(kind, plan)
    J = box.solve_box_jacobian(st, R0, C0, nlb)
    tp, tb = _T(pt["tp"][:Bn]), _T(pt["tb"][:Bn]) if e else None
    tlb, tub = (_T(pt["tlb"][:Bn]) if nlb else None), (_T(pt["tub"][:Bn]) if has_ub else None)
    dz, dlam, dnu = box.solve_box_jvp(st, (None, tp, None, tb, tlb, tub))
    grads = box.solve_box_backward(st, _T(pt["dl"][:Bn]), (False,) * 6, (False, True, False, bool(e), True, True),
                                   _T(pt["glam"][:Bn]), _T(pt["gnu"][:Bn]) if e else None)
    t = torch.cat([x for x in (tp, tlb, tub, tb) if x is not None], 1)
    jvp = torch.cat([dz, dlam] + ([dnu] if e else []), 1)
    g = torch.cat([_T(pt["dl"][:Bn]), _T(pt["glam"][:Bn])] + ([_T(pt["gnu"][:Bn])] if e else []), 1)
    gJ = torch.cat([x for x in (grads[1], grads[4] if nlb else None, grads[5] if has_ub else None,
                                grads[3] if e else None) if x is not None], 1)
    err = dict(ref=[], jvp=[], grad=[], ident=[])
    m = plan.nineq
    for i in range(Bn):
        Ji = J[i].cpu().numpy()
        if i == 0 or e == 0 or n + 2 * m + e <= 3000:
            err["ref"].append(_rel(Ji, box_reference(kind, plan, pt, i)))
        err["jvp"].append(_rel((J[i] @ t[i]).cpu().numpy(), jvp[i].cpu().numpy()))
        err["grad"].append(_rel((g[i] @ J[i]).cpu().numpy(), gJ[i].cpu().numpy()))
        d = jm.clamped_d(pt["lam"][i], pt["s"][i])
        err["ident"].append(bm.identity_residuals(Ji, n, m, e, nlb, has_ub, d) / np.abs(Ji[:n]).max())
        del Ji
    out.update({"err_" + k: np.array(v) for k, v in err.items()})
    del J
    if ent["next"] is not None:
        from qpth_b200 import _lib
        from tests.box_jacobian_jobs import point, state
        nn, ne, ns = ent["next"]
        nplan = _lib.box_plan_for(nn, ne, *je.sides_flags(ns))
        out["next_covered"] = box.box_jacobian_covered(nplan)
        npt = point(nplan, 19, Bn=1)
        Jzp = box.solve_box_jacobian(state(nplan, npt, False), 1, 1, nn if nplan.has_lb else 0)[0].cpu().numpy()
        Jr = box_reference("box", nplan, npt, 0)
        out["next_err"] = np.array(_rel_to(Jzp, Jr[:nn, :nn], Jr))
    torch.cuda.synchronize()
    return out


# ---- the public API at converged solves -----------------------------------------------------------------------------

def _qp_problem(n, m, e, seed):
    from tests.kernel_families import wellcond_qp_batch
    return wellcond_qp_batch(B, n, m, e, seed=seed)


def _same(a, b):
    return bool(a.shape == b.shape and torch.equal(a.contiguous().view(torch.int64), b.contiguous().view(torch.int64)))


def _default_and_order(f, names, n):
    """f.jacobian() and every single wrt against the z rows of f.jacobian(duals=True), and wrt out of order with a
    repeat: 1 where bit-identical (names: every input the problem has, the default wrt)"""
    full = f.jacobian(wrt=names, duals=True)
    res = [all(_same(v, full[k][:, :n]) for k, v in f.jacobian().items()) and list(f.jacobian()) == list(names)]
    for k in names:
        res.append(_same(f.jacobian(wrt=k)[k], full[k][:, :n]))
    rev = tuple(reversed(names))
    wrt = rev + (rev[0],)
    J = f.jacobian(wrt=wrt, duals=True)
    res.append(list(J) == list(rev) and all(_same(J[k], full[k]) for k in rev))
    return np.array(res)


def api_qp_job():
    """QPFunction and QPSolutionFunction: the default call and the wrt order"""
    from qpth_b200 import QPFunction
    from qpth_b200.solution import QPSolutionFunction
    n, m, e = 30, 20, 6
    pr = _qp_problem(n, m, e, 3)
    x = [_T(pr[k]) for k in ("Q", "p", "G", "h", "A", "b")]
    f = QPFunction(verbose=-1)
    f(*x)
    out = dict(qpfunction=_default_and_order(f, ("p", "h", "b"), n))
    st = f.last_solve()
    g = QPSolutionFunction()
    g(*x, st.zhat, st.lam, st.slacks, st.nus)
    out["solution"] = _default_and_order(g, ("p", "h", "b"), n)
    return out


def api_box_job():
    """BoxQPFunction, diagonal and dense Q: the default call and the wrt order"""
    from qpth_b200 import BoxQPFunction
    from tests.box_jacobian_jobs import _problem
    out = {}
    for dense_Q, (n, e, sides) in ((False, (40, 7, "both")), (True, (30, 5, "both")), (False, (24, 0, "ub"))):
        pr = _problem(n, e, sides, 6, dense_Q)
        E = torch.empty(0, dtype=torch.float64, device=DEV)
        f = BoxQPFunction(dense_Q=dense_Q, verbose=-1)
        f(_T(pr["q"]), _T(pr["p"]), _T(pr["A"]) if e else E, _T(pr["b"][0]) if e else E,
          None if pr["lb"] is None else _T(pr["lb"]), None if pr["ub"] is None else _T(pr["ub"]))
        names = ("p",) + (("lb",) if pr["lb"] is not None else ()) + (("ub",) if pr["ub"] is not None else ()) \
            + (("b",) if e else ())
        out["%s_%d_%d_%s" % ("dense" if dense_Q else "diag", n, e, sides)] = _default_and_order(f, names, n)
    return out


def api_mixed_qp_job(q_shared):
    """QPFunction with Q shared and G, A batched (q_shared), or Q batched and G, A shared: J at the returned point
    against the dense model and against the column path on the same state"""
    from qpth_b200 import QPFunction
    from qpth_b200.qp import _jacobian_columns
    n, m, e = 30, 20, 6
    pr = _qp_problem(n, m, e, 7 + q_shared)
    shared = ("Q",) if q_shared else ("G", "A")
    for k in shared:                      # h = G z0 + s0 and b = A z0 stay feasible with QP 0's G and A: s0 > 0 per QP
        pr[k] = np.broadcast_to(pr[k][0], pr[k].shape).copy()
    x = [_T(pr[k][0] if k in shared else pr[k]) for k in ("Q", "p", "G", "h", "A", "b")]
    f = QPFunction(verbose=-1)
    f(*x)
    st = f.last_solve()
    J = f.jacobian(duals=True)
    J = torch.cat([J[k] for k in ("p", "h", "b")], 2)
    Jc = torch.empty_like(J)
    _jacobian_columns(st, 7, 7, Jc)
    lam, s = st.lam.cpu().numpy(), st.slacks.cpu().numpy()
    ref, col = [], []
    for i in range(B):
        Jd = jm.dense_jacobian(pr["Q"][i], pr["G"][i], pr["A"][i], lam[i], s[i])
        ref.append(_rel(J[i].cpu().numpy(), Jd))
        col.append(_rel(Jc[i].cpu().numpy(), Jd))
    return dict(nsys=np.array(st.nsys), err_ref=np.array(ref), err_col=np.array(col))


def api_mixed_box_job(q_shared):
    """BoxQPFunction with q shared and A batched (q_shared), or q batched and A shared"""
    from qpth_b200 import BoxQPFunction
    from tests.box_jacobian_jobs import _problem
    n, e = 40, 7
    pr = _problem(n, e, "both", 8 + q_shared)
    rs = np.random.RandomState(9)
    A = rs.randn(B, e, n) / np.sqrt(n) if q_shared else pr["A"]
    z0 = rs.uniform(-0.5, 0.5, (B, n))
    b = np.einsum("bij,bj->bi", A, z0) if q_shared else pr["b"][0]
    q = pr["q"][0] if q_shared else pr["q"]
    f = BoxQPFunction(verbose=-1)
    f(_T(q), _T(pr["p"]), _T(A), _T(b), _T(pr["lb"]), _T(pr["ub"]))
    st = f.last_solve()
    J = f.jacobian(duals=True)
    J = torch.cat([J[k] for k in ("p", "lb", "ub", "b")], 2).cpu().numpy()
    lam, s = st.lam.cpu().numpy(), st.slacks.cpu().numpy()
    ref = []
    for i in range(B):
        qi = q if q_shared else q[i]
        Ai = A[i] if q_shared else A
        ref.append(_rel(J[i], bm.dense_box_jacobian_refined(np.diag(qi), Ai, lam[i], s[i], n, True)))
    return dict(sq=np.array(st.sq), sA=np.array(st.sA), err_ref=np.array(ref))


def api_box_edge_job():
    """One BoxQPFunction forward on the (2616, 0, both) cl4 plan at B = 2, then jacobian(duals=True), against the
    per-variable reference at the returned point"""
    from qpth_b200 import BoxQPFunction, box
    from tests.box_jacobian_jobs import _problem
    n = 2616
    pr = _problem(n, 0, "both", 12, Bn=2)
    E = torch.empty(0, dtype=torch.float64, device=DEV)
    f = BoxQPFunction(verbose=-1)
    f(_T(pr["q"]), _T(pr["p"]), E, E, _T(pr["lb"]), _T(pr["ub"]))
    st = f.last_solve()
    out = dict(fwd=np.array(je.box_forward(st.plan)), dense=np.array(st.dense is not None),
               covered=np.array(box.box_jacobian_covered(st.plan)))
    Jd = f.jacobian(duals=True)
    lam, s = st.lam.cpu().numpy(), st.slacks.cpu().numpy()
    err, err_z, dspan = [], [], []
    for i in range(2):
        Ji = torch.cat([Jd[k][i] for k in ("p", "lb", "ub")], 1).cpu().numpy()
        Jr = bm.diagonal_box_jacobian(pr["q"][i], lam[i], s[i], n, True)
        err.append(_rel(Ji, Jr))
        err_z.append(_rel(Ji[:n], Jr[:n]))
        d = jm.clamped_d(lam[i], s[i])
        dspan.append(d.max() / d.min())
        del Ji, Jr
    out.update(err_ref=np.array(err), err_z=np.array(err_z), dspan=np.array(dspan))
    return out


def jobs():
    out = [("sweep_jac_" + k, sweep_job, ("jac", k)) for k, v in je.JAC.items() if v["sweep"]]
    out += [("sweep_box_" + k, sweep_job, ("box", k)) for k, v in je.BOX.items() if v["sweep"]]
    out += [("sweep_boxq_" + k, sweep_job, ("boxq", k)) for k, v in je.BOXQ.items() if v["sweep"]]
    out += [("edge_jac_" + k, jac_edge_job, (k,)) for k in je.JAC]
    out += [("edge_box_" + k, box_edge_job, ("box", k)) for k in je.BOX]
    out += [("edge_boxq_" + k, box_edge_job, ("boxq", k)) for k in je.BOXQ]
    out += [("api_qp", api_qp_job, ()), ("api_box", api_box_job, ())]
    out += [("api_mixed_qp_%d" % q, api_mixed_qp_job, (q,)) for q in (1, 0)]
    out += [("api_mixed_box_%d" % q, api_mixed_box_job, (q,)) for q in (1, 0)]
    out += [("api_box_edge", api_box_edge_job, ())]
    return out


def main(out_dir):
    import time
    for name, fn, args in jobs():
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        t0 = time.time()
        try:
            np.savez(os.path.join(out_dir, name + ".npz"), **fn(*args))
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())
        with open(os.path.join(out_dir, "times.txt"), "a") as fh:
            fh.write("%s %.2f\n" % (name, time.time() - t0))


def run_child(out_dir, timeout_s=900):
    """main() in a child process; returns "" or why it did not finish."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.jacobian_edges_jobs", out_dir], cwd=root, timeout=timeout_s,
                           capture_output=True, text=True)
        if r.returncode != 0:
            return "child exited with %d: %s" % (r.returncode, (r.stderr or "")[-2000:])
    except subprocess.TimeoutExpired:
        prog = os.path.join(out_dir, "progress.txt")
        last = open(prog).read().split()[-1:] if os.path.exists(prog) else []
        return "child killed after %d s, last job started: %s" % (timeout_s, last)
    return ""


if __name__ == "__main__":
    main(sys.argv[1])
