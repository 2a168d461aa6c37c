"""Jacobians of (z, lam, nu) with respect to (p, h, b) on the GPU (jacobian() of QPFunction and QPSolutionFunction).

The kernel (qpb200_jacobian) runs here for the first time on a device, so every job runs in one child process
(tests/jacobian_jobs.py) and each test reads its job's output:
- every family and shape of tests/kernel_families.py at its dual_point: J against the dense model
  (tests/jacobian_models.dense_jacobian) within 1e-10 per-QP relative, with per-QP and with shared factors; J t against
  the JVP of random batched tangents of p, h, b; g' J against the dual backward's dp, dh, db; the symmetry identities.
  The global-scratch shapes, which the kernel does not cover, check the column-by-column path the same way;
- the column-by-column path of IR_UNOPT against the dense model;
- converged QPFunction solutions (the clamps act): the kernel against the column-by-column path.
In-process: central differences of z, lam, nu on a strictly complementary batch, and fp32 / CPU inputs.
"""
import os
import tempfile

import numpy as np
import pytest
import torch

from tests import dual_models as dm
from tests import jacobian_models as jm
from tests.duals_jobs import dual_point
from tests.jacobian_jobs import CONVERGED_SHAPES, REG_SHAPES, jobs, reg_point, run_child
from tests.kernel_families import cases, ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_OUT = {}
UNCOVERED = ("global_scratch", "edge_generic_full")


@pytest.fixture(scope="module")
def out_dir():
    if "dir" not in _OUT:
        d = tempfile.mkdtemp(prefix="jacobian_jobs_")
        _OUT["dir"], _OUT["why"] = d, run_child(d)
    return _OUT["dir"]


def _load(out_dir, name):
    path = os.path.join(out_dir, name + ".npz")
    if not os.path.exists(path):
        err = os.path.join(out_dir, name + ".err")
        pytest.fail(open(err).read() if os.path.exists(err) else "no output: %s" % _OUT.get("why"))
    return dict(np.load(path))


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("fam,shape", cases(), ids=ids(cases()))
def test_family_jacobian(out_dir, fam, shape):
    n, m, e = shape
    got = _load(out_dir, "jac_%s_%dx%dx%d" % ((fam,) + tuple(shape)))
    pr = dual_point(fam, shape)
    B = pr["z"].shape[0]
    A = lambda i: pr["A"][i] if e else None
    for i in range(B):
        Jd = jm.dense_jacobian(pr["Q"][i], pr["G"][i], A(i), pr["lam"][i], pr["s"][i])
        assert got["J"][i].shape == Jd.shape
        assert _rel(got["J"][i], Jd) < 1e-10, (i, _rel(got["J"][i], Jd))
        Js = jm.dense_jacobian(pr["Q"][0], pr["G"][0], A(0), pr["lam"][i], pr["s"][i])
        assert _rel(got["J_shared"][i], Js) < 1e-10, (i, _rel(got["J_shared"][i], Js))
        J = got["J"][i]
        assert jm.symmetry_residuals(J, n, m, e) < 1e-10 * np.abs(J).max()
        t = np.concatenate([got["tp"][i], got["th"][i]] + ([got["tb"][i]] if e else []))
        jvp = np.concatenate([got["dz"][i], got["dlam"][i]] + ([got["dnu"][i]] if e else []))
        assert _rel(J @ t, jvp) < 1e-10
        g = np.concatenate([pr["dl"][i], pr["glam"][i]] + ([pr["gnu"][i]] if e else []))
        grads = np.concatenate([got["grad_dp"][i], got["grad_dh"][i]] + ([got["grad_db"][i]] if e else []))
        assert _rel(g @ J, grads) < 1e-10
    # orders above 256 (the global-scratch plans): the staircase of S alone exceeds the shared memory, so these shapes
    # check the column-by-column path the same way
    assert bool(got["covered"]) == (fam not in UNCOVERED)


@pytest.mark.parametrize("shape", REG_SHAPES)
def test_reg_columns(out_dir, shape):
    n, m, e = shape
    got = _load(out_dir, "jacreg_%dx%dx%d" % shape)
    pr = reg_point(shape)
    for i in range(pr["z"].shape[0]):
        Jd = jm.dense_jacobian(pr["Q"][i], pr["G"][i], pr["A"][i] if e else None, pr["lam"][i], pr["s"][i])
        # the regularised solve with its refinement step (kkt.IR_STEPS) against the exact inverse
        assert _rel(got["J"][i], Jd) < 1e-6, (i, _rel(got["J"][i], Jd))


@pytest.mark.parametrize("shape", CONVERGED_SHAPES)
def test_converged_kernel_vs_columns(out_dir, shape):
    n, m, e = shape
    got = _load(out_dir, "jacconv_%dx%dx%d" % shape)
    for i in range(got["J"].shape[0]):
        d = jm.clamped_d(got["lam"][i], got["s"][i])
        Jd = jm.dense_jacobian(got["Q"][i], got["G"][i], got["A"][i] if e else None, got["lam"][i], got["s"][i])
        tol = max(1e-8, 10 * _rel(got["Jc"][i], Jd))
        err = _rel(got["J"][i], got["Jc"][i])
        print("converged %s QP %d: D spans %.1e .. %.1e, kernel vs columns %.2e (tol %.1e)"
              % (shape, i, d.min(), d.max(), err, tol))
        assert err < tol


def test_jobs_cover_every_case():
    names = [nm for nm, _, _ in jobs()]
    assert len(names) == len(set(names)) == len(cases()) + len(REG_SHAPES) + len(CONVERGED_SHAPES)


@pytest.mark.parametrize("neq", [0, 3])
def test_central_differences(neq):
    """Central differences within 1e-5 of the exact implicit derivative, J within 1e-7 of the implicit derivative with
    qpth's 1e-8 clamps (the function the kernel computes; tests/test_gpu_duals.py explains the two references)."""
    from qpth_b200 import QPFunction
    from tests import jvp_models as jvm
    prs = [dm.complementary_qp(71 + i, 10, 9, neq) for i in range(3)]
    t = {k: torch.tensor(np.stack([pr[k] for pr in prs]), dtype=torch.float64, device=DEV)
         for k in ("Q", "p", "G", "h", "A", "b")}
    E = torch.Tensor().to(DEV).double()
    f = QPFunction(verbose=-1, duals=True)

    def solve(x):
        z, lam, nu = f(x["Q"], x["p"], x["G"], x["h"], x["A"] if neq else E, x["b"] if neq else E)
        return torch.cat([z, lam, nu], dim=1)

    solve(t)
    wrt = ("p", "h", "b") if neq else ("p", "h")
    J = f.jacobian(wrt=wrt, duals=True)
    eps = 1e-6
    for k in wrt:
        for j in range(t[k].shape[1]):
            xp, xm = dict(t), dict(t)
            xp[k] = t[k].clone(); xp[k][:, j] += eps
            xm[k] = t[k].clone(); xm[k][:, j] -= eps
            fd = ((solve(xp) - solve(xm)) / (2 * eps)).cpu().numpy()
            Jj = J[k][:, :, j].cpu().numpy()
            for i, pr in enumerate(prs):
                unit = np.zeros(t[k].shape[1]); unit[j] = 1.0
                refs = [np.concatenate([v for v in jvm.implicit_jvp(pr["Q"], pr["G"], pr["A"] if neq else None, pr["z"],
                                                                      pr["lam"], pr["s"], pr["nu"], {k: unit}, clamp=c)
                                        if v is not None]) for c in (False, True)]
                assert np.abs(fd[i] - refs[0]).max() < 1e-5, (k, j, i)
                assert np.abs(Jj[i] - refs[1]).max() < 1e-7, (k, j, i)


def test_dtype_device_round_trip():
    from qpth_b200 import QPFunction
    pr = dm.complementary_qp(5, 8, 6, 2)
    for dev, dtype in (("cpu", torch.float32), (DEV, torch.float32), ("cpu", torch.float64)):
        x = [torch.tensor(pr[k], dtype=dtype, device=dev) for k in ("Q", "p", "G", "h", "A", "b")]
        f = QPFunction(verbose=-1)
        f(*x)
        J = f.jacobian(wrt=("p", "b"), duals=True)
        assert set(J) == {"p", "b"}
        assert J["p"].shape == (1, 16, 8) and J["b"].shape == (1, 16, 2)
        assert J["p"].dtype == dtype and J["p"].device.type == torch.device(dev).type
        assert not J["p"].requires_grad
