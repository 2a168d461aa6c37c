"""GPU jobs of tests/test_gpu_box_jacobian.py, run in one child process with a timeout (qpb200_box_jacobian is new to
the device). Each job writes <name>.npz, or <name>.err with its traceback; progress.txt lists the jobs started.

- `entry`: a box-family entry (tests/box_families.py) at the point of test_gpu_duals._box_point, with per-QP and with
  shared q and A: the full Jacobian [z; lam; nu] x [p, lb, ub, b] by solve_box_jacobian (the kernel where it covers
  the plan, else the columns), the column path itself, the JVP of random batched tangents and the dual backward.
- `boxq`: every dense-Q family entry the forward kernels run, the same way with a dense SPD Q.
- `wide`: the widest cluster entries (one QP, J_z,p by the column path) against a batched JVP.
- `dense`: a family entry no box kernel runs, through BoxQPFunction (the dense fallback), with its returned point.
- `conv` / `convq`: converged BoxQPFunction solutions with a diagonal / dense Q (the clamps act).
- `cd`: a strictly complementary batch (tests/dual_models.complementary_box) and its central differences.
- `roundtrip`: fp32 and CPU inputs.
"""
import os
import sys
import traceback

import numpy as np
import torch

DEV = "cuda:0"
# box-family entries run at a point: every layout, the kernel-covered entries and the column-path ones whose dense model
# is small enough to form (WIDE: the eight-CTA entries of 5000 variables and more, and dm8_slice, run the column path on
# one QP for J_z,p only, checked against a batched JVP and its symmetry)
ENTRY_NAMES = ("one_mid_lb", "one_mid_both", "one_mid_ub", "one_full", "one_neq120", "one_wide", "cl2_mid_forced",
               "cl2_mid", "cl2_mid_lb", "cl2_past_one_wide", "cl2_past_one_neq", "cl2_full", "cl4_mid_forced",
               "cl4_mid", "cl4_mid_480", "cl4_mid_lb", "cl4_full", "cl8_mid_forced", "cl8_full", "cl8_empty_9",
               "cl8_empty_5", "dm2_mid_forced", "dm2_boundary", "dm2_full", "dm4_mid_forced", "dm4_mid", "dm4_sudoku",
               "dm4_full", "dm8_mid_forced", "dm8_full")
WIDE_NAMES = ("cl8_mid", "cl8_mid_box", "cl8_widest", "cl8_widest_lb", "dm8_slice")
DENSE_NAMES = ("dense_mid", "dense_boundary")
B = 3


def _T(a):
    return torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)


def point(plan, seed, dense_Q=False, Bn=B):
    """test_gpu_duals._box_point (dense_Q: boxq_edges_child's Q = F F' / n + 0.5 I), plus the random tangents"""
    rs = np.random.RandomState(seed)
    n, e, m = plan.nz, plan.neq, plan.nineq
    B = Bn
    F = rs.randn(B, n, n) if dense_Q else None
    q = (F @ F.transpose(0, 2, 1) / n + 0.5 * np.eye(n)) if dense_Q else 0.5 + rs.rand(B, n)
    pt = dict(q=q, A=rs.randn(B, e, n) / np.sqrt(n), z=rs.randn(B, n), nu=rs.randn(B, e),
              lam=rs.uniform(0.1, 10, (B, m)), s=rs.uniform(0.1, 10, (B, m)), dl=rs.randn(B, n), glam=rs.randn(B, m),
              gnu=rs.randn(B, e))
    pt.update(tp=rs.randn(B, n), tlb=rs.randn(B, n), tub=rs.randn(B, n), tb=rs.randn(B, e))
    return pt


def state(plan, pt, shared, dense_Q=False):
    from qpth_b200.box import _BoxSolved
    n, e = plan.nz, plan.neq
    st = _BoxSolved()
    st.plan, st.nBatch, st.device, st.dense, st.dense_Q = plan, pt["z"].shape[0], torch.device(DEV), None, dense_Q
    st.q, st.sq = (_T(pt["q"][0]), 0) if shared else (_T(pt["q"]), n * n if dense_Q else n)
    st.A, st.sA = ((_T(pt["A"][0]), 0) if shared else (_T(pt["A"]), e * n)) if e else (None, 0)
    st.zhat, st.lam, st.slacks = _T(pt["z"]), _T(pt["lam"]), _T(pt["s"])
    st.nus = _T(pt["nu"]) if e else None
    return st


def masks(plan):
    cols = 1 | (2 if plan.has_lb else 0) | (4 if plan.has_ub else 0) | (8 if plan.neq else 0)
    return (7 if plan.neq else 3), cols


def entry_job(name):
    from tests.box_families import ENTRIES, check_entry, knob
    ent = ENTRIES[name]
    with knob(ent["knob"]):
        return point_job(check_entry(name), False)


def boxq_entry_job(name):
    from tests.boxq_families import ENTRIES, check_entry
    return point_job(check_entry(name), True)


def point_job(plan, dense_Q):
    """The full Jacobian at a point by solve_box_jacobian (the kernel where it covers the plan, else the columns), the
    column path itself, shared q / Q and A, the JVP of batched tangents and the dual backward."""
    from qpth_b200 import box
    pt = point(plan, 11, dense_Q)
    nlb = plan.nz if plan.has_lb else 0
    rows, cols = masks(plan)
    out = dict(covered=box.box_jacobian_covered(plan, dense_Q), q=pt["q"], A=pt["A"], lam=pt["lam"], s=pt["s"],
               tp=pt["tp"], tlb=pt["tlb"], tub=pt["tub"], tb=pt["tb"], dl=pt["dl"], glam=pt["glam"], gnu=pt["gnu"])
    st = state(plan, pt, False, dense_Q)
    J = box.solve_box_jacobian(st, rows, cols, nlb)
    Jc = torch.empty_like(J)
    box._box_jacobian_columns(st, rows, cols, Jc)
    e = plan.neq
    tans = (None, _T(pt["tp"]), None, _T(pt["tb"]) if e else None, _T(pt["tlb"]) if plan.has_lb else None,
            _T(pt["tub"]) if plan.has_ub else None)
    dz, dlam, dnu = box.solve_box_jvp(st, tans)
    grads = box.solve_box_backward(st, _T(pt["dl"]), (False,) * 6, (False, True, False, bool(e), True, True),
                                   _T(pt["glam"]), _T(pt["gnu"]) if e else None)
    Js = box.solve_box_jacobian(state(plan, pt, True, dense_Q), rows, cols, nlb)
    torch.cuda.synchronize()
    c = lambda t: np.zeros(0) if t is None else t.cpu().numpy()
    out.update(J=c(J), Jc=c(Jc), J_shared=c(Js), dz=c(dz), dlam=c(dlam), dnu=c(dnu), grad_dp=c(grads[1]),
               grad_db=c(grads[3]), grad_dlb=c(grads[4]), grad_dub=c(grads[5]))
    return out


def wide_job(name):
    """One QP of a wide entry: J_z,p by solve_box_jacobian (the column path there) and the JVP of a tangent of p."""
    from qpth_b200 import box
    from tests.box_families import ENTRIES, check_entry, knob
    ent = ENTRIES[name]
    with knob(ent["knob"]):
        plan = check_entry(name)
        pt = point(plan, 13, Bn=1)
        st = state(plan, pt, False)
        J = box.solve_box_jacobian(st, 1, 1, plan.nz if plan.has_lb else 0)
        dz, _, _ = box.solve_box_jvp(st, (None, _T(pt["tp"]), None, None, None, None))
        torch.cuda.synchronize()
        return dict(covered=box.box_jacobian_covered(plan), J=J[0].cpu().numpy(), tp=pt["tp"][0],
                    dz=dz[0].cpu().numpy())


def _problem(n, e, sides, seed, dense_Q=False, Bn=B):
    rs = np.random.RandomState(seed)
    if dense_Q:
        F = rs.randn(Bn, n, n)
        q = F @ F.transpose(0, 2, 1) / n + 0.1 * np.eye(n)
    else:
        q = rs.uniform(0.5, 2.0, (Bn, n))
    A = rs.randn(e, n) / np.sqrt(n)
    z0 = rs.uniform(-0.5, 0.5, (Bn, n))
    return dict(q=q, p=rs.randn(Bn, n), A=A, b=z0 @ A.T, lb=-0.5 * np.ones(n) if sides != "ub" else None,
                ub=0.5 * np.ones(n) if sides != "lb" else None)


def solve_job(n, e, sides, dense_Q, seed=5):
    """BoxQPFunction forward + jacobian(duals=True) at a converged point; the column path on the same state."""
    from qpth_b200 import box
    pr = _problem(n, e, sides, seed, dense_Q)
    f = box.BoxQPFunction(dense_Q=dense_Q, verbose=-1)
    E = torch.empty(0, dtype=torch.float64, device=DEV)
    f(_T(pr["q"]), _T(pr["p"]), _T(pr["A"]) if e else E, _T(pr["b"][0]) if e else E,
      None if pr["lb"] is None else _T(pr["lb"]), None if pr["ub"] is None else _T(pr["ub"]))
    st = f.last_solve()
    Jd = f.jacobian(duals=True)
    J = torch.cat(list(Jd.values()), dim=2)
    out = dict(J=J.cpu().numpy(), names=np.array(list(Jd)), lam=st.lam.cpu().numpy(), s=st.slacks.cpu().numpy(),
               q=pr["q"], A=pr["A"], dense=st.dense is not None)
    if st.dense is None:
        rows, cols = masks(st.plan)
        Jc = torch.empty_like(J)
        box._box_jacobian_columns(st, rows, cols, Jc)
        out["Jc"] = Jc.cpu().numpy()
        out["covered"] = box.box_jacobian_covered(st.plan, dense_Q)
    return out


def dense_job(name):
    from tests.box_families import ENTRIES, check_entry, knob
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    with knob(ent["knob"]):
        check_entry(name)
        return solve_job(n, e, sides, False)


def cd_job(n, e, sides):
    """Central differences of (z, lam, nu) in p, lb, ub, b on a strictly complementary QP, and the clamped J."""
    from qpth_b200 import box
    from tests.dual_models import complementary_box
    pr = complementary_box(7, n, e, sides)
    names = ["p"] + (["lb"] if pr["lb"] is not None else []) + (["ub"] if pr["ub"] is not None else []) + ["b"]
    f = box.BoxQPFunction(duals=True, verbose=-1)

    def run(vals):
        z, lam, nu = f(_T(pr["q"]), vals["p"], _T(pr["A"]), vals["b"], vals.get("lb"), vals.get("ub"))
        return torch.cat([z[0], lam[0], nu[0]]).cpu().numpy()

    base = {k: _T(pr[k]) for k in names}
    run(base)
    J = f.jacobian(duals=True)
    J = torch.cat([J[k] for k in names], dim=2)[0].cpu().numpy()
    h = 1e-6
    cols = []
    for k in names:
        for j in range(base[k].numel()):
            v1, v2 = dict(base), dict(base)
            v1[k], v2[k] = base[k].clone(), base[k].clone()
            v1[k][j] += h
            v2[k][j] -= h
            cols.append((run(v1) - run(v2)) / (2 * h))
    return dict(J=J, Jfd=np.stack(cols, axis=1))


def roundtrip_job():
    """fp32 CUDA and fp64 CPU inputs: dtype and device of the result, against fp64 CUDA."""
    from qpth_b200 import box
    pr = _problem(12, 3, "both", 9)
    out = {}
    for tag, dt, dev in (("f64", torch.float64, DEV), ("f32", torch.float32, DEV), ("cpu", torch.float64, "cpu")):
        f = box.BoxQPFunction(verbose=-1)
        T = lambda a: torch.tensor(a, dtype=dt, device=dev)
        f(T(pr["q"]), T(pr["p"]), T(pr["A"]), T(pr["b"][0]), T(pr["lb"]), T(pr["ub"]))
        J = f.jacobian(wrt=("p", "ub"), duals=True)
        out[tag] = torch.cat([J["p"], J["ub"]], dim=2).double().cpu().numpy()
        out[tag + "_meta"] = np.array([str(J["p"].dtype), J["p"].device.type, str(J["p"].requires_grad)])
    return out


CONVERGED = [(64, 40, "lb", False), (31, 13, "both", False), (40, 0, "ub", False), (30, 5, "both", True),
             (24, 0, "both", True)]
CD = [(9, 3, "both"), (10, 2, "lb")]


def jobs():
    from tests.boxq_families import kernel_entries
    out = [("entry_" + nm, entry_job, (nm,)) for nm in ENTRY_NAMES]
    out += [("boxq_" + nm, boxq_entry_job, (nm,)) for nm in kernel_entries()]
    out += [("wide_" + nm, wide_job, (nm,)) for nm in WIDE_NAMES]
    out += [("dense_" + nm, dense_job, (nm,)) for nm in DENSE_NAMES]
    out += [("conv_%d_%d_%s_%d" % c, solve_job, c) for c in CONVERGED]
    out += [("cd_%d_%d_%s" % c, cd_job, c) for c in CD]
    out += [("roundtrip", roundtrip_job, ())]
    return out


def main(out_dir):
    for name, fn, args in jobs():
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        try:
            np.savez(os.path.join(out_dir, name + ".npz"), **fn(*args))
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


def run_child(out_dir, timeout_s=900):
    """main() in a child process; returns "" or why it did not finish."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.box_jacobian_jobs", out_dir], cwd=root, timeout=timeout_s,
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
