"""GPU runs of forward mode (torch.autograd.forward_ad through QPSolutionFunction) for every kernel family of
tests/kernel_families.py, shared by tests/test_gpu_jvp.py and its child process. The families marked `child` run in the
child process, so that a fault there fails only their own tests:  python -m tests.jvp_jobs <out_dir>  writes
<out_dir>/<job>.npz (or .err) and each job's name to <out_dir>/progress.txt as it starts.

At the family's backward_point (tests/duals_jobs.dual_point: lam, s ~ U(0.1, 10), so the clamps do nothing) with random
tangents of every input (dQ not symmetric), each job returns the JVP (dz, dlam, dnu) and the gradients of the loss
g_z'z + g_lam'lam + g_nu'nu (the backward with dual adjoints, "grad_<name>"), for the transpose identity.
"""
import os
import sys
import traceback

import numpy as np

from tests.duals_jobs import dual_point, solution_backward_duals
from tests.kernel_families import family_env, family_plan, seed_for

INPUTS = ("Q", "p", "G", "h", "A", "b")


def tangents(pr, seed, batched=None):
    """Random tangents of the inputs of `pr` (None for an empty input); batched[k] False: one un-batched tangent."""
    rs = np.random.RandomState(seed)
    batched = batched or {k: True for k in INPUTS}
    out = {}
    for k in INPUTS:
        v = pr[k] if batched[k] else pr[k][0]
        out[k] = rs.randn(*v.shape) if v.size else None
    return out


def solution_jvp(pr, tan, plan=None, dev="cuda:0", kkt_solver=None, duals=True, batched=None):
    """QPSolutionFunction at the point of `pr` with the tangents `tan` through torch.autograd.forward_ad: (dz, dlam,
    dnu) as arrays (dlam, dnu None with duals=False)."""
    import torch
    import torch.autograd.forward_ad as fwAD
    from qpth_b200 import _lib
    from qpth_b200.qp import KKTSolvers
    from qpth_b200.solution import QPSolutionFunction
    batched = batched or {k: True for k in INPUTS}
    neq = pr["A"].shape[1]
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64, device=dev)
    E = torch.Tensor().to(dev).double()
    sol = [T(pr[k]) for k in ("z", "lam", "s")] + [T(pr["nu"]) if neq else E]
    saved = _lib.plan_for
    if plan is not None:
        _lib.plan_for = lambda *a, **k: plan
    try:
        f = QPSolutionFunction(kkt_solver=kkt_solver or KKTSolvers.LU_PARTIAL, duals=duals)
        with fwAD.dual_level():
            x = {}
            for k in INPUTS:
                if k in "Ab" and not neq:
                    x[k] = E
                    continue
                v = T(pr[k] if batched[k] else pr[k][0])
                x[k] = fwAD.make_dual(v, T(tan[k])) if tan.get(k) is not None else v
            out = f(*(x[k] for k in INPUTS), *sol)
            outs = out if duals else (out,)
            tl = [fwAD.unpack_dual(o).tangent for o in outs]
    finally:
        _lib.plan_for = saved
    res = [t.cpu().numpy() for t in tl]
    return res if duals else [res[0], None, None]


def jvp_on_gpu(fam, shape):
    """The JVP and the dual backward at the family's point, with the family's plan."""
    pr = dual_point(fam, shape)
    tan = tangents(pr, seed_for(fam, shape, 6))
    with family_env(fam):
        plan = family_plan(fam, shape)
        dz, dlam, dnu = solution_jvp(pr, tan, plan=plan)
        z_only = solution_jvp(pr, tan, plan=plan, duals=False)[0]
        grads = solution_backward_duals(pr, "all", plan=plan)
    out = dict(dz=dz, dlam=dlam, z_only=z_only)
    if shape[2]:
        out["dnu"] = dnu
    out.update({"grad_" + k: v for k, v in grads.items() if v is not None})
    return out


def job_name(fam, shape):
    return "jvp_%s_%dx%dx%d" % ((fam,) + tuple(shape))


def main(out_dir):
    from tests.kernel_families import cases
    for fam, shape in cases(child=True):
        name = job_name(fam, shape)
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        try:
            np.savez(os.path.join(out_dir, name + ".npz"), **jvp_on_gpu(fam, shape))
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


def run_child(out_dir, timeout_s=600):
    """main() in a child process; returns "" or why it did not finish."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.jvp_jobs", out_dir], cwd=root, timeout=timeout_s,
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

