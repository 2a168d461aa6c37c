"""GPU runs of the double backward (create_graph=True through QPSolutionFunction, then a second grad) for every kernel family
of tests/kernel_families.py, shared by tests/test_gpu_double_backward.py and its child process. The families marked
`child` run in the child process, so that a fault there fails only their own tests:  python -m tests.double_backward_jobs
<out_dir>  writes <out_dir>/<job>.npz (or .err) and each job's name to <out_dir>/progress.txt as it starts.

At the family's dual point (tests/duals_jobs.dual_point) with seeded adjoints (g_z, g_lam, g_nu) and cotangents w_X, each
job returns the gradients of sum <w_X, grad_X> with respect to g_z, g_lam, g_nu and every input, for each sharing of
SHARED (un-batched inputs take QP 0's value).
"""
import os
import sys
import traceback

import numpy as np

from tests.duals_jobs import dual_point
from tests.kernel_families import family_env, family_plan, seed_for

NAMES = ("Q", "p", "G", "h", "A", "b")
ADJ = ("gz", "glam", "gnu")
# every input batched; Q, G, A shared (the sums of k_ggrad_sum); p, h, b shared (the sums of k_ggrad_sum_vec)
SHARED = {"batched": (), "shared_QGA": ("Q", "G", "A"), "shared_phb": ("p", "h", "b")}


def case_data(fam, shape, sharing):
    """(pr, inputs, adjoints, cotangents) as arrays; an input or adjoint absent without equality rows is None."""
    shared = SHARED[sharing]
    pr = dual_point(fam, shape)
    e = shape[2]
    ins = {k: (None if (k in "Ab" and not e) else (pr[k][0] if k in shared else pr[k])) for k in NAMES}
    adj = dict(gz=pr["dl"], glam=pr["glam"], gnu=pr["gnu"] if e else None)
    rs = np.random.RandomState(seed_for(fam, shape, 7) + list(SHARED).index(sharing))
    om = {k: (None if ins[k] is None else rs.randn(*ins[k].shape)) for k in NAMES}
    return pr, ins, adj, om


def second_order(f, ins, sol, adj, om, plan=None, dev="cuda:0"):
    """Through `f` (QPSolutionFunction(duals=True) or alike) at the solution `sol`: first order of
    <g_z, z> + <g_lam, lam> + <g_nu, nu> with create_graph=True, then the gradients of sum <om_X, grad_X> with respect to
    the adjoints and the inputs. ins / adj / om: arrays or None. Returns {name: array}."""
    import torch
    from qpth_b200 import _lib
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), device=dev)
    E = torch.Tensor().to(dev).double()
    lv = {k: (E if ins[k] is None else T(ins[k]).requires_grad_(True)) for k in NAMES}
    ad = {k: (None if adj[k] is None else T(adj[k]).requires_grad_(True)) for k in ADJ}
    sol = [T(x) if np.size(x) else E for x in sol]
    saved = _lib.plan_for
    if plan is not None:
        _lib.plan_for = lambda *a, **k: plan
    try:
        z, lam, nu = f(*(lv[k] for k in NAMES), *sol)
        loss = (ad["gz"] * z).sum() + (ad["glam"] * lam).sum() + ((ad["gnu"] * nu).sum() if ad["gnu"] is not None else 0.0)
        want = [k for k in NAMES if lv[k].requires_grad]
        g1 = torch.autograd.grad(loss, [lv[k] for k in want], create_graph=True)
        phi = sum((T(om[k]) * g).sum() for k, g in zip(want, g1) if om.get(k) is not None)
        keys = [k for k in ADJ if ad[k] is not None] + want
        g2 = torch.autograd.grad(phi, [ad[k] for k in ADJ if ad[k] is not None] + [lv[k] for k in want],
                                 allow_unused=True)
    finally:
        _lib.plan_for = saved
    return {k: g.detach().cpu().numpy() for k, g in zip(keys, g2) if g is not None}


def on_gpu(fam, shape, sharing):
    from qpth_b200.solution import QPSolutionFunction
    pr, ins, adj, om = case_data(fam, shape, sharing)
    sol = [pr["z"], pr["lam"], pr["s"], pr["nu"]]
    with family_env(fam):
        plan = family_plan(fam, shape)
        return second_order(QPSolutionFunction(duals=True), ins, sol, adj, om, plan)


def job_name(fam, shape, sharing):
    return "db_%s_%dx%dx%d_%s" % ((fam,) + tuple(shape) + (sharing,))


def main(out_dir):
    from tests.kernel_families import cases
    for fam, shape in cases(child=True):
        for sharing in SHARED:
            name = job_name(fam, shape, sharing)
            with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
                fh.write(name + "\n")
            try:
                np.savez(os.path.join(out_dir, name + ".npz"), **on_gpu(fam, shape, sharing))
            except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
                with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                    fh.write(traceback.format_exc())


def run_child(out_dir, timeout_s=600):
    """main() in a child process; returns "" or why it did not finish."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.double_backward_jobs", out_dir], cwd=root, timeout=timeout_s,
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
