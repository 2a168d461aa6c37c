"""GPU runs of the Jacobians (jacobian() of QPSolutionFunction and QPFunction) for every kernel family of
tests/kernel_families.py, the regularised mode and converged solutions, shared by tests/test_gpu_jacobian.py and its child
process:  python -m tests.jacobian_jobs <out_dir>  writes <out_dir>/<job>.npz (or .err) and each job's name to
<out_dir>/progress.txt as it starts. Every job runs in the child process: a fault there fails only the Jacobian tests.

Family jobs, at the family's dual_point (lam, s ~ U(0.1, 10)) with the family's plan: J with per-QP factors ("J") and
with Q, G, A shared ("J_shared", QP 0's matrices), the JVP for random batched tangents of p, h, b ("dz", "dlam", "dnu")
and the gradients of g_z'z + g_lam'lam + g_nu'nu ("grad_dp", "grad_dh", "grad_db"). J is (B, nz + nineq + neq, n_wrt),
rows [z; lam; nu], columns [p, h, b]; "covered": whether qpb200_jacobian ran (else the column-by-column JVPs).
"""
import os
import sys
import traceback

import numpy as np

from tests.duals_jobs import dual_point, solution_backward_duals
from tests.jvp_jobs import solution_jvp, tangents
from tests.kernel_families import cases, family_env, family_plan, seed_for

DEV = "cuda:0"
REG_SHAPES = [(24, 19, 5), (50, 50, 10), (100, 100, 0)]
CONVERGED_SHAPES = [(100, 100, 0), (50, 50, 10), (10, 5, 0)]


def wrt_of(neq):
    return ("p", "h", "b") if neq else ("p", "h")


def solution_jacobian(pr, plan=None, shared=False, kkt_solver=None):
    """QPSolutionFunction at the point of `pr` (Q, G, A of QP 0 for every QP when shared) and its jacobian(duals=True),
    the blocks concatenated in the order p, h, b."""
    import torch
    from qpth_b200 import _lib
    from qpth_b200.qp import KKTSolvers
    from qpth_b200.solution import QPSolutionFunction
    neq = pr["A"].shape[1]
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64, device=DEV)
    E = torch.Tensor().to(DEV).double()
    x = {k: T(pr[k][0] if (shared and k in "QGA") else pr[k]) for k in ("Q", "p", "G", "h")}
    x["A"] = T(pr["A"][0] if shared else pr["A"]) if neq else E
    x["b"] = T(pr["b"]) if neq else E
    sol = [T(pr[k]) for k in ("z", "lam", "s")] + [T(pr["nu"]) if neq else E]
    saved = _lib.plan_for
    if plan is not None:
        _lib.plan_for = lambda *a, **k: plan
    try:
        f = QPSolutionFunction(kkt_solver=kkt_solver or KKTSolvers.LU_PARTIAL, duals=True)
        f(*(x[k] for k in ("Q", "p", "G", "h", "A", "b")), *sol)
        J = f.jacobian(wrt=wrt_of(neq), duals=True)
    finally:
        _lib.plan_for = saved
    return torch.cat([J[k] for k in wrt_of(neq)], dim=2).cpu().numpy()


def family_job(fam, shape):
    from qpth_b200.qp import jacobian_covered
    pr = dual_point(fam, shape)
    tan = tangents(pr, seed_for(fam, shape, 9))
    tan = {k: (tan[k] if k in "phb" else None) for k in tan}
    with family_env(fam):
        plan = family_plan(fam, shape)
        out = dict(covered=np.array(jacobian_covered(plan)))
        out["J"] = solution_jacobian(pr, plan)
        out["J_shared"] = solution_jacobian(pr, plan, shared=True)
        dz, dlam, dnu = solution_jvp(pr, tan, plan=plan)
        grads = solution_backward_duals(pr, "all", plan=plan)
    out.update(dz=dz, dlam=dlam, tp=tan["p"], th=tan["h"])
    if shape[2]:
        out.update(dnu=dnu, tb=tan["b"])
    out.update({"grad_" + k: grads[k] for k in ("dp", "dh", "db") if grads.get(k) is not None})
    return out


def reg_job(shape):
    """The column-by-column path of the regularised mode (IR_UNOPT) at a well-conditioned point."""
    from qpth_b200 import _lib
    from qpth_b200.qp import KKTSolvers
    plan = _lib.plan_for_ir(*shape)
    return dict(J=solution_jacobian(reg_point(shape), plan, kkt_solver=KKTSolvers.IR_UNOPT))


def reg_point(shape):
    """The point of a regularised-mode job: random_qp_batch (Q positive definite) with lam, s ~ U(0.1, 10)."""
    from tests.kernel_families import backward_point
    return backward_point(shape, 4, 1234 + sum(shape))


def converged_job(shape):
    """QPFunction at a converged solution (the clamps act, D spans many decades): the kernel's J and the column-by-column
    J at the same state."""
    import torch
    from qpth_b200 import QPFunction
    from qpth_b200.qp import _jacobian_columns
    from tests.kernel_families import wellcond_qp_batch
    nz, nineq, neq = shape
    pr = wellcond_qp_batch(8, nz, nineq, neq, seed=sum(shape))
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64, device=DEV)
    E = torch.Tensor().to(DEV).double()
    f = QPFunction(verbose=-1)
    f(T(pr["Q"]), T(pr["p"]), T(pr["G"]), T(pr["h"]), T(pr["A"]) if neq else E, T(pr["b"]) if neq else E)
    st = f.last_solve()
    J = f.jacobian(wrt=wrt_of(neq), duals=True)
    J = torch.cat([J[k] for k in wrt_of(neq)], dim=2)
    rows, cols = 3 if not neq else 7, 3 if not neq else 7
    Jc = torch.empty_like(J)
    _jacobian_columns(st, rows, cols, Jc)
    return dict(J=J.cpu().numpy(), Jc=Jc.cpu().numpy(), lam=st.lam.cpu().numpy(), s=st.slacks.cpu().numpy(),
                Q=pr["Q"], G=pr["G"], A=pr["A"])


def jobs():
    out = [("jac_%s_%dx%dx%d" % ((fam,) + tuple(shape)), family_job, (fam, shape)) for fam, shape in cases()]
    out += [("jacreg_%dx%dx%d" % s, reg_job, (s,)) for s in REG_SHAPES]
    out += [("jacconv_%dx%dx%d" % s, converged_job, (s,)) for s in CONVERGED_SHAPES]
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
        r = subprocess.run([sys.executable, "-m", "tests.jacobian_jobs", out_dir], cwd=root, timeout=timeout_s,
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
