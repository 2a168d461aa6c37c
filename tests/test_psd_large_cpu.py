"""The regularised mode (QPFunction kkt_solver=KKTSolvers.IR_UNOPT) beyond the product-form kernels, without a GPU: which
plan each shape gets, the numpy model of the kernels' arithmetic (oracle/reg_model.py) on the large cases against scipy
HiGHS and the dense implicit differentiation, and the routing of QPSolutionFunction(kkt_solver=IR_UNOPT)."""
import contextlib
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import psd_cases as pc, psd_large_cases as lc, reg_model as rm

EPS, STEPS = 1e-7, 1


def _lib():
    from qpth_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libqpth_b200.so not built")
    return _lib


def _plan(fn, *shape):
    L = _lib()
    p = L.Plan()
    return getattr(L.load(), fn)(*shape, ctypes.byref(p)), p


def test_every_shape_the_default_mode_takes_has_a_regularised_plan():
    """Over the shape grid of test_capi_cpu: wherever plan_init_reg refuses a shape with nineq >= 1 that plan_init
    accepts, plan_init gives it a global-scratch plan, which forward_reg / backward_reg run."""
    checked = 0
    for nz in (1, 7, 8, 10, 31, 64, 100, 200, 500, 1000):
        for nineq in (0, 1, 5, 50, 200, 500, 1000):
            for neq in (0, 1, 9, 100):
                if nineq == 0:
                    continue
                rc, p = _plan("qpb200_plan_init", nz, nineq, neq)
                if rc != 0:
                    continue
                rr, _ = _plan("qpb200_plan_init_reg", nz, nineq, neq)
                if rr != 0:
                    assert rr == 4
                    assert (p.tiny, p.pf, p.smem_resident) == (0, 0, 0), (nz, nineq, neq)
                    assert p.solve_scratch_elems > 0
                    checked += 1
    assert checked > 10


def test_plan_helper():
    L = _lib()
    p = L.plan_for_ir(200, 200, 0)
    assert p.pf == 1 and p.pf_threads == 256
    for shape in ((50, 250, 10), (100, 260, 10), (729, 729, 249)):
        p = L.plan_for_ir(*shape)
        assert (p.tiny, p.pf, p.smem_resident) == (0, 0, 0), shape
    with pytest.raises(L.QpthB200Error, match="too large"):
        L.plan_for_reg(50, 250, 10)
    with pytest.raises(L.QpthB200Error, match="too large"):
        L.plan_for_ir(729, 729, 324)                  # the unreduced 9x9 sudoku: the default mode refuses it too


def test_case_orders():
    L = _lib()
    for make, order in ((lc.lp280, 280), (lc.lowrank120, 248), (lc.lp232, 232), (lc.lp664, 664),
                        (lc.lp_dependent, 280)):
        Q, p, G, h, A, b = make(0)
        plan = L.plan_for_ir(Q.shape[0], G.shape[0], A.shape[0])
        assert plan.ms_pad == order and plan.pf == 0 and plan.smem_resident == 0
    Q, p, G, h, A, b = lc.sudoku9_lp(0)[0]
    assert L.plan_for_ir(Q.shape[0], G.shape[0], A.shape[0]).ms_pad == 992
    assert np.linalg.matrix_rank(lc.lp_dependent(0)[4]) == 7


@pytest.mark.parametrize("make", [lc.lp280, lc.lp_dependent, lc.lp232])
def test_model_lp_matches_highs(make):
    from scipy.optimize import linprog
    Q, p, G, h, A, b = case = make(0)
    sol = rm.solve_one_reg(*case, reg=EPS, steps=STEPS)
    res = linprog(p, A_ub=G, b_ub=h, A_eq=A, b_eq=b, bounds=(None, None), method="highs")
    assert res.status == 0
    assert abs(p @ sol["x"] - res.fun) <= 1e-9 * abs(res.fun)
    assert np.linalg.norm(sol["x"] - res.x) <= 1e-7 * np.linalg.norm(res.x)
    assert max(pc.kkt_residuals(*case, sol["x"], sol["lam"], sol["s"], sol["nu"])) <= 1e-10


def test_model_lowrank120_gradients_match_dense_kkt():
    Q, p, G, h, A, b = case = lc.lowrank120(0)
    sol = rm.solve_one_reg(*case, reg=EPS, steps=STEPS)
    assert max(pc.kkt_residuals(*case, sol["x"], sol["lam"], sol["s"], sol["nu"])) <= 1e-10
    dl = np.random.RandomState(5).randn(Q.shape[0])
    g = rm.backward_one_reg(sol, dl)
    gd = pc.dense_grads(Q, G, A, sol["x"], sol["lam"], sol["s"], sol["nu"], dl)
    for k in gd:
        assert np.abs(g[k] - gd[k]).max() <= 1e-5 * max(np.abs(gd[k]).max(), 1e-8), k


class _CpuTorch:
    """torch as solution.py / qp.py see it on a machine without a GPU: a CUDA device is "available" and is the CPU."""
    cuda = SimpleNamespace(is_available=lambda: True, device=lambda d: contextlib.nullcontext(), current_device=lambda: 0)

    @staticmethod
    def device(*args):
        return torch.device("cpu")

    def __getattr__(self, name):
        return getattr(torch, name)


class _DenseLib:
    """Stand-in for the library: records the entry points called; pre_factor_kkt_reg flags the PSD check on request."""

    def __init__(self, calls, bad_spd=False):
        self.calls, self.bad_spd = calls, bad_spd

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            if name == "qpb200_pre_factor_kkt_reg" and self.bad_spd:
                ctypes.cast(args[12], ctypes.POINTER(ctypes.c_int))[0] = 1
            return 0
        return fn


def test_solution_function_routes_to_the_regularised_entry_points(monkeypatch):
    """QPSolutionFunction(kkt_solver=IR_UNOPT): the plan helper, pre_factor_kkt_reg with kkt.IR_EPS, the PSD message
    of the regularised mode, and backward_reg with IR_EPS and IR_STEPS in the backward pass."""
    import qpth_b200.qp as qp
    from qpth_b200 import KKTSolvers, QPSolutionFunction, _lib as L, kkt, solution
    calls = []
    plan = L.Plan()
    plan.nz, plan.nineq, plan.neq = 4, 3, 0
    plan.L_elems = plan.W_elems = plan.K_elems = plan.solve_scratch_elems = 1
    monkeypatch.setattr(L, "load", lambda: _DenseLib(calls))
    monkeypatch.setattr(L, "plan_for_ir", lambda *s: calls.append(("plan_for_ir", s)) or plan)
    monkeypatch.setattr(L, "plan_for", lambda *s, **k: pytest.fail("default plan used"))
    for mod in (qp, solution):
        monkeypatch.setattr(mod, "torch", _CpuTorch())
    monkeypatch.setattr(qp, "_stream", lambda: None)
    Q = torch.zeros(4, 4, dtype=torch.float64, requires_grad=True)
    p = torch.ones(4, dtype=torch.float64, requires_grad=True)
    G = -torch.eye(3, 4, dtype=torch.float64)
    h = torch.zeros(3, dtype=torch.float64)
    e = torch.Tensor()
    z = torch.zeros(1, 4, dtype=torch.float64)
    lam = torch.ones(1, 3, dtype=torch.float64)
    zo = QPSolutionFunction(kkt_solver=KKTSolvers.IR_UNOPT)(Q, p, G, h, e, e, z, lam, lam, e)
    assert [c[0] for c in calls] == ["plan_for_ir", "qpb200_pre_factor_kkt_reg"]
    assert calls[1][1][8] == kkt.IR_EPS
    calls.clear()
    zo.sum().backward()
    (name, args), = calls
    assert name == "qpb200_backward_reg" and args[11:13] == (kkt.IR_EPS, kkt.IR_STEPS)
    # a failed pivot of chol(Q + eps I) reports the message of the regularised mode
    monkeypatch.setattr(L, "load", lambda: _DenseLib(calls, bad_spd=True))
    with pytest.raises(RuntimeError, match="Q is not positive semidefinite."):
        QPSolutionFunction(kkt_solver=KKTSolvers.IR_UNOPT)(Q, p, G, h, e, e, z, lam, lam, e)
    QPSolutionFunction(check_Q_spd=False, kkt_solver=KKTSolvers.IR_UNOPT)(Q, p, G, h, e, e, z, lam, lam, e)
    with pytest.raises(ValueError, match="IR_UNOPT"):
        QPSolutionFunction(kkt_solver=KKTSolvers.LU_FULL)


def test_cvxpy_branch_passes_kkt_solver_on(monkeypatch):
    from qpth_b200 import KKTSolvers, QPFunction, QPSolvers, solution
    seen = []
    monkeypatch.setattr(solution, "cvxpy_forward", lambda *a: (None, None, None, None))
    monkeypatch.setattr(solution, "QPSolutionFunction", lambda *a: seen.append(a) or (lambda *x: None))
    Q, p = torch.eye(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    G, h, e = torch.ones(2, 3, dtype=torch.float64), torch.ones(2, dtype=torch.float64), torch.Tensor()
    QPFunction(solver=QPSolvers.CVXPY, kkt_solver=KKTSolvers.IR_UNOPT)(Q, p, G, h, e, e)
    QPFunction(solver=QPSolvers.CVXPY)(Q, p, G, h, e, e)
    assert seen == [(True, KKTSolvers.IR_UNOPT), (True, KKTSolvers.LU_PARTIAL)]
