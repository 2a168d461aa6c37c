"""Child process of tests/test_gpu_zz_fallback_families.py and of the per-family tests: runs every job of one job list of
tests/fallback_jobs.py on cuda:0 and writes <out_dir>/<job>.npz (or <job>.err with the traceback).
Usage: python -m tests.gpu_child <out_dir> [job list, default `jobs`]."""
import os
import subprocess
import sys
import traceback

import numpy as np


def _run_eq_only(cfg, dev="cuda:0"):
    import torch
    from qpth_b200 import QPFunction
    from tests.fallback_jobs import eq_only_problem
    pr = eq_only_problem(**cfg)
    t = {k: torch.tensor(pr[k], dtype=torch.float64, device=dev, requires_grad=True) for k in ("Q", "p", "A", "b")}
    e = torch.Tensor().to(dev).double()
    z = QPFunction(verbose=-1)(t["Q"], t["p"], e, e, t["A"], t["b"])
    z.backward(torch.tensor(pr["dl"], dtype=torch.float64, device=dev))
    return dict(zhat=z.detach().cpu().numpy(), grads=[t[k].grad.cpu().numpy() for k in ("Q", "p", "A", "b")])


def _save(out_dir, name, out):
    rec = {k: np.asarray(out[k]) for k in ("zhat", "lam", "slacks", "iters") if out.get(k) is not None}
    if out.get("nus") is not None:
        rec["nus"] = np.asarray(out["nus"])
    for i, g in enumerate(out.get("grads") or ()):
        if g is not None:
            rec["grad%d" % i] = np.asarray(g)
    np.savez(os.path.join(out_dir, name + ".npz"), **rec)


def main(out_dir, which="jobs"):
    from oracle.cases import load_case
    from qpth_b200 import qp as qpmod
    from qpth_b200.problems import random_qp_batch
    from tests import fallback_jobs, kernel_families
    from tests.test_gpu_parity import _run
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    for name, kind, payload, env, mode in getattr(fallback_jobs, which)():
        saved = {k: os.environ.get(k) for k in env}
        try:
            os.environ.update(env)
            qpmod.MODE = mode or "auto"
            if kind == "call":               # (function of tests/kernel_families.py, kwargs) -> dict of arrays
                fn, kw = payload
                np.savez(os.path.join(out_dir, name + ".npz"), **getattr(kernel_families, fn)(**kw))
            else:
                if kind == "eq_only":
                    out = _run_eq_only(payload)
                else:
                    prob = load_case(payload, golden)[0] if kind == "golden" else random_qp_batch(**payload)
                    out = _run(prob)
                _save(out_dir, name, out)
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")


def run(out_dir, which="jobs", timeout_s=240):
    """Run one job list in a child process; returns "" or why it did not finish (the parent fails the jobs without a
    result with this note)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.gpu_child", out_dir, which], cwd=root, timeout=timeout_s,
                           capture_output=True, text=True)
        if r.returncode != 0:
            return "child exited with %d: %s" % (r.returncode, (r.stderr or "")[-2000:])
    except subprocess.TimeoutExpired:
        return "child killed after %d s (a job hung)" % timeout_s
    return ""


def load(out_dir, note, job):
    """The arrays job `job` wrote, or pytest.fail with its traceback / the child's note."""
    import pytest
    path = os.path.join(out_dir, job + ".npz")
    if not os.path.exists(path):
        err = os.path.join(out_dir, job + ".err")
        why = open(err).read()[-3000:] if os.path.exists(err) else ("no result: " + (note or "job never ran"))
        pytest.fail("%s: %s" % (job, why), pytrace=False)
    return dict(np.load(path))


if __name__ == "__main__":
    main(sys.argv[1], *sys.argv[2:3])
