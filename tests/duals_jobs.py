"""GPU runs of the dual outputs (QPSolutionFunction(duals=True)) for every kernel family of tests/kernel_families.py, shared
by tests/test_gpu_duals.py and its child process. The families marked `child` run in the child process, so that a fault
there fails only their own tests:  python -m tests.duals_jobs <out_dir>  writes <out_dir>/<job>.npz (or .err) and each
job's name to <out_dir>/progress.txt as it starts.

At the family's backward_point (lam, s ~ U(0.1, 10): the clamps do nothing) with random g_lam, g_nu, each job runs the
backward of one loss per variant and returns its six gradients as "<variant>_<gradient>":
  all   g_z'z + g_lam'lam + g_nu'nu            z     g_z'z with duals=True (lam, nu unused: NULL adjoints)
  base  g_z'z with duals=False                 lam   g_lam'lam alone (dl_dzhat arrives as None)
  nu    g_nu'nu alone (equality rows only)
"""
import os
import sys
import traceback

import numpy as np

from tests.kernel_families import BWD_B, GRAD_NAMES, backward_point, family_env, family_plan, seed_for


def dual_point(fam, shape, B=BWD_B):
    nz, nineq, neq = shape
    pr = backward_point(shape, B, seed_for(fam, shape, 4), fam)
    rs = np.random.RandomState(seed_for(fam, shape, 5))
    pr.update(glam=rs.randn(B, nineq), gnu=rs.randn(B, neq))
    return pr


def variants(neq):
    return ("all", "z", "base", "lam") + (("nu",) if neq else ())


def solution_backward_duals(pr, variant, batched=None, plan=None, dev="cuda:0", kkt_solver=None):
    """QPSolutionFunction at the point of `pr` and the backward of the variant's loss. batched: {name: bool} (default all
    batched); un-batched inputs take QP 0's value. Returns {gradient name: array or None}."""
    import torch
    from qpth_b200 import _lib
    from qpth_b200.qp import KKTSolvers
    from qpth_b200.solution import QPSolutionFunction
    batched = batched or {k: True for k in "QpGhAb"}
    neq = pr["A"].shape[1]
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64, device=dev)
    t = {}
    for k in ("Q", "p", "G", "h", "A", "b"):
        v = pr[k] if batched[k] else pr[k][0]
        t[k] = T(v).requires_grad_(True) if (neq or k not in "Ab") else torch.Tensor().to(dev).double()
    sol = [T(pr[k]) for k in ("z", "lam", "s")] + [T(pr["nu"]) if neq else torch.Tensor().to(dev).double()]
    saved = _lib.plan_for
    if plan is not None:
        _lib.plan_for = lambda *a, **k: plan
    try:
        f = QPSolutionFunction(kkt_solver=kkt_solver or KKTSolvers.LU_PARTIAL, duals=variant != "base")
        out = f(t["Q"], t["p"], t["G"], t["h"], t["A"], t["b"], *sol)
        if variant == "base":
            loss = (out * T(pr["dl"])).sum()
        else:
            z, lam, nu = out
            assert lam.shape == tuple(pr["lam"].shape) and nu.shape == (pr["lam"].shape[0], neq)
            assert torch.equal(lam, sol[1]) and (neq == 0 or torch.equal(nu, sol[3]))
            terms = dict(all=[(z, "dl"), (lam, "glam")] + ([(nu, "gnu")] if neq else []), z=[(z, "dl")],
                         lam=[(lam, "glam")], nu=[(nu, "gnu")])[variant]
            loss = sum((x * T(pr[k])).sum() for x, k in terms)
        loss.backward()
    finally:
        _lib.plan_for = saved
    return {n: (t[k].grad.cpu().numpy() if t[k].grad is not None else None) for n, k in zip(GRAD_NAMES, "QpGhAb")}


def dual_backward_on_gpu(fam, shape):
    """Every variant at the family's point, with the family's plan: {"<variant>_<gradient>": array}."""
    pr = dual_point(fam, shape)
    out = {}
    with family_env(fam):
        plan = family_plan(fam, shape)
        for v in variants(shape[2]):
            g = solution_backward_duals(pr, v, plan=plan)
            out.update({"%s_%s" % (v, k): a for k, a in g.items() if a is not None})
    return out


def job_name(fam, shape):
    return "duals_%s_%dx%dx%d" % ((fam,) + tuple(shape))


def main(out_dir):
    from tests.kernel_families import cases
    for fam, shape in cases(child=True):
        name = job_name(fam, shape)
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        try:
            np.savez(os.path.join(out_dir, name + ".npz"), **dual_backward_on_gpu(fam, shape))
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


def run_child(out_dir, timeout_s=600):
    """main() in a child process; returns "" or why it did not finish."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.duals_jobs", out_dir], cwd=root, timeout=timeout_s,
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
