"""The Newton trajectory of every kernel family against oracle/kernel_model.py (the kernels' formulation in numpy, itself
checked against the dense KKT solve and the reference in tests/test_oracle.py).

A converged z* hides a wrong step: the iteration corrects itself and only takes longer. Below convergence it cannot.
For maxIter in {1, 2, 3, 5, 20} and eps in {1e-12, 1e-6}, on well-conditioned random_qp_batch shapes, and once per family
with Q, G, A, h, b shared by the batch (the edge entries: wellcond_qp_batch, eps = 1e-12 only, batched only):
  * every trace row [||rz|| + ||ry||, ||L r~x||, mu, resid] against the model's, row-relative l2 error <= 1e-9 while the
    model's resid >= 1e-3. Below that the iterates sit close to the rounding floor: a 1e-15 relative perturbation of p
    and h moves the model's own rows by up to 1.5e-8 at resid ~1e-6 and 1e-3 at resid ~1e-9 (measured at these
    shapes), so rows with 1e-6 <= resid < 1e-3 get 1e-9 * (1e-3 / resid) and later ones none;
  * truncated runs (maxIter < 20): the returned z, lam, s, nu within 1e-9 relative and the same iteration count;
  * full runs: iteration counts within +-1 (the eps exit sits at the rounding floor);
  * best_resid is the smallest resid of the trace, as the reference reports it.
"""
import numpy as np
import pytest

from oracle import kernel_model as km
from tests import gpu_child
from tests.fallback_jobs import TRAJ_B, traj_job_name, traj_runs, traj_unbatched
from tests.kernel_families import cases, family_env, family_plan, trajectory_on_gpu, trajectory_problem
from tests.parity import rel_rows

pytestmark = pytest.mark.gpu


def _variants(child):
    return [(fam, s, u) for fam, s in cases(child=child, forward=True) for u in traj_unbatched(fam, s)]


def _ids(vs):
    return ["%s-%dx%dx%d%s" % ((fam,) + tuple(s) + ("-unbatched" if u else "",)) for fam, s, u in vs]


def _model(fam, shape, unbatched, maxIter, eps):
    from qpth_b200.qp import BEST_TIE, STALL_TOL
    pr = trajectory_problem(fam, shape, TRAJ_B, unbatched)
    out = []
    for i in range(TRAJ_B):
        arg = [pr[k] if np.asarray(pr[k]).ndim == nd else pr[k][i]
               for k, nd in (("Q", 2), ("p", 1), ("G", 2), ("h", 1), ("A", 2), ("b", 1))]
        tr = []
        o = km.solve_one(*arg, eps=eps, maxIter=maxIter, stall_tol=STALL_TOL, tie=BEST_TIE, trace=tr)
        o["trace"] = np.array(tr)
        out.append(o)
    return out


def _row_tol(resid):
    return 1e-9 if resid >= 1e-3 else (1e-9 * 1e-3 / resid if resid >= 1e-6 else np.inf)


def check_run(fam, shape, unbatched, maxIter, eps, out, worst):
    neq = shape[2]
    for i, m in enumerate(_model(fam, shape, unbatched, maxIter, eps)):
        it = int(out["iters"][i])
        tr = out["trace"][i]
        if maxIter < 20:
            assert it == m["iters"], (i, it, m["iters"])
        else:
            assert abs(it - m["iters"]) <= 1, (i, it, m["iters"])
        # rows past the last iteration stay unwritten; the last one may be NaN (a step off the rounding floor ends a
        # solve in both the kernels and the model, which then return the best earlier iterate)
        assert np.isfinite(tr[:it - 1]).all() and np.isnan(tr[it:]).all()
        assert out["best_resid"][i] == np.nanmin(tr[:it, 3])
        assert m["best_resid"] == np.nanmin(m["trace"][:, 3])
        for k in range(min(it, m["iters"])):
            if not m["trace"][k, 3] >= 1e-6:
                continue
            err = np.linalg.norm(tr[k] - m["trace"][k]) / np.linalg.norm(m["trace"][k])
            if m["trace"][k, 3] >= 1e-3:
                worst["trace"] = max(worst["trace"], err)
            assert err <= _row_tol(m["trace"][k, 3]), (i, k, err, m["trace"][k])
        if maxIter < 20:
            pairs = [("zhat", m["x"]), ("lam", m["lam"]), ("slacks", m["s"])] + ([("nus", m["nu"])] if neq else [])
            for key, ref in pairs:
                e = rel_rows(out[key][i], ref).max()
                worst["iterate"] = max(worst["iterate"], e)
                assert e <= 1e-9, (i, key, e)
            e = abs(out["best_resid"][i] - m["best_resid"]) / m["best_resid"]
            assert e <= 1e-9 or m["best_resid"] < 1e-3, (i, e)


def _check_all(fam, shape, unbatched, get):
    from tests.test_gpu_parity import _report
    worst = dict(trace=0.0, iterate=0.0)
    for maxIter, eps in traj_runs(fam):
        check_run(fam, shape, unbatched, maxIter, eps, get(maxIter, eps), worst)
    _report("traj[%s %s%s]" % (fam, shape, " unbatched" if unbatched else ""), worst)


@pytest.mark.parametrize("fam,shape,unbatched", _variants(False), ids=_ids(_variants(False)))
def test_trajectory_matches_model(fam, shape, unbatched):
    _check_all(fam, shape, unbatched,
               lambda maxIter, eps: trajectory_on_gpu(fam, shape, TRAJ_B, unbatched, maxIter, eps))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("trajectory_families"))
    return out_dir, gpu_child.run(out_dir, "family_trajectory_jobs")


@pytest.mark.parametrize("fam,shape,unbatched", _variants(True), ids=_ids(_variants(True)))
def test_trajectory_matches_model_new_dispatch(fam, shape, unbatched, child_results):
    """Families with a dispatch branch that had never run before these tests (the resident 512-thread forward among
    them): solved in the child process."""
    with family_env(fam):
        family_plan(fam, shape)
    _check_all(fam, shape, unbatched,
               lambda maxIter, eps: gpu_child.load(*child_results, traj_job_name(fam, shape, unbatched, maxIter, eps)))
