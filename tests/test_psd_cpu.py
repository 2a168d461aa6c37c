"""The regularised mode (QPFunction kkt_solver=KKTSolvers.IR_UNOPT) without a GPU: the numpy model of the kernels'
arithmetic (oracle/reg_model.py) against scipy HiGHS, the KKT residuals and the dense implicit differentiation; central
finite differences; the host logic (enum, errors, plans, the equality-only route) and the C ABI exports."""
import os

import numpy as np
import pytest
import torch

from oracle import psd_cases as pc, reg_model as rm

EPS, STEPS = 1e-7, 1


def _kkt_ok(case, sol, tol=1e-10):
    r = pc.kkt_residuals(*case, sol["x"], sol["lam"], sol["s"], sol["nu"])
    assert max(r) <= tol, r


@pytest.mark.parametrize("seed", [0, 1])
def test_model_lp_matches_highs(seed):
    from scipy.optimize import linprog
    for case in (pc.lp(seed), pc.lp(seed, nz=10, nrand=6, neq=2)):
        Q, p, G, h, A, b = case
        sol = rm.solve_one_reg(*case, reg=EPS, steps=STEPS)
        res = linprog(p, A_ub=G, b_ub=h, A_eq=A, b_eq=b, bounds=(None, None), method="highs")
        assert res.status == 0
        assert abs(p @ sol["x"] - res.fun) <= 1e-9 * abs(res.fun)
        assert np.linalg.norm(sol["x"] - res.x) <= 1e-7 * np.linalg.norm(res.x)
        _kkt_ok(case, sol)


@pytest.mark.parametrize("steps", [0, 1])
@pytest.mark.parametrize("make", [pc.lowrank, pc.sudoku4, pc.spd])
def test_model_kkt_residuals(make, steps):
    case = make(0)
    sol = rm.solve_one_reg(*case, reg=EPS, steps=steps)
    _kkt_ok(case, sol)
    assert sol["best_resid"] < 1e-11


def test_sudoku_full_A_is_rank_deficient_and_solved():
    A = pc.sudoku4_full_A()
    assert A.shape == (64, 64) and np.linalg.matrix_rank(A) == 40
    case = pc.sudoku4(3)
    sol = rm.solve_one_reg(*case, reg=EPS, steps=STEPS)
    _kkt_ok(case, sol)


@pytest.mark.parametrize("make", [pc.lowrank, pc.spd])
def test_model_gradients_match_dense_kkt(make):
    Q, p, G, h, A, b = make(0)
    sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=EPS, steps=STEPS)
    dl = np.random.RandomState(5).randn(Q.shape[0])
    g = rm.backward_one_reg(sol, dl)
    gd = pc.dense_grads(Q, G, A, sol["x"], sol["lam"], sol["s"], sol["nu"], dl)
    for k in gd:
        assert np.abs(g[k] - gd[k]).max() <= 1e-6 * max(np.abs(gd[k]).max(), 1e-8), k


def test_finite_differences_lowrank():
    """d(dl'z*)/dp and /dh by central differences of the model's forward on the rank-5 case (strictly complementary
    solution: every active row has lam >> s)."""
    Q, p, G, h, A, b = pc.lowrank(0)
    sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=EPS, steps=STEPS)
    act = sol["s"] < 1e-6
    assert np.all(sol["lam"][act] > 1e-4) and np.all(sol["lam"][~act] < 1e-8)
    dl = np.random.RandomState(9).randn(Q.shape[0])
    g = rm.backward_one_reg(sol, dl)
    r = np.random.RandomState(4)
    step = 1e-5
    for key, arr in (("dp", p), ("dh", h)):
        v = r.randn(arr.size)
        plus, minus = arr + step * v, arr - step * v
        args_p = (Q, plus, G, h, A, b) if key == "dp" else (Q, p, G, plus, A, b)
        args_m = (Q, minus, G, h, A, b) if key == "dp" else (Q, p, G, minus, A, b)
        fd = (dl @ rm.solve_one_reg(*args_p, reg=EPS, steps=STEPS)["x"]
              - dl @ rm.solve_one_reg(*args_m, reg=EPS, steps=STEPS)["x"]) / (2 * step)
        assert abs(fd - g[key] @ v) <= 1e-4 * max(abs(fd), 1.0), key   # (qpth's 1e-8 clamps: not exactly the derivative)


def test_kkt_solvers_enum_and_lu_full():
    import qpth_b200
    from qpth_b200 import KKTSolvers, QPFunction
    assert qpth_b200.KKTSolvers is KKTSolvers
    assert (KKTSolvers.LU_FULL.value, KKTSolvers.LU_PARTIAL.value, KKTSolvers.IR_UNOPT.value) == (1, 2, 3)
    with pytest.raises(ValueError, match="IR_UNOPT"):
        QPFunction(kkt_solver=KKTSolvers.LU_FULL)
    from qpth_b200 import kkt
    assert kkt.IR_EPS == 1e-7 and kkt.IR_STEPS in (0, 1)


def _lib():
    from qpth_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libqpth_b200.so not built")
    return _lib


def test_c_abi_exports():
    lib = _lib().load()
    for name in ("qpb200_plan_init_reg", "qpb200_forward_reg", "qpb200_backward_reg"):
        assert hasattr(lib, name)
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "qpth_b200.h")).read()
    for name in ("qpb200_plan_init_reg(", "qpb200_forward_reg(", "qpb200_backward_reg("):
        assert name in header


def test_reg_plans():
    L = _lib()
    # tiny shapes: the product-form kernels, not the one-warp ones of the default path
    d, r = L.plan_for(10, 24, 2), L.plan_for_reg(10, 24, 2)
    assert d.tiny == 1 and r.tiny == 0 and r.pf == 1
    for shape in ((50, 170, 10), (64, 64, 64), (100, 200, 0), (200, 200, 0)):
        p = L.plan_for_reg(*shape)
        assert p.pf == 1 and p.pf_threads == 256 and p.pf_two == 0 and p.pf_three == 0
    assert L.plan_for_reg(100, 200, 0).pf_global == 1 and L.plan_for_reg(64, 64, 64).pf_global == 0
    # default plans are untouched by the regularised ones
    assert L.plan_for(200, 200, 0).pf_threads == 512
    with pytest.raises(L.QpthB200Error, match="too large"):
        L.plan_for_reg(50, 250, 10)                   # ms_pad = 264 > 256


class RegDenseFactor:
    """CPU stand-in for kkt._Factored with reg: [Q+rI 0 G' A'; 0 D+rI I 0; G I -rI 0; A 0 0 -rI] u = -r."""

    def __init__(self, Q, G, A, reg):
        self.Q, self.G, self.A = (t.detach().cpu().numpy() for t in (Q, G, A))
        self.reg = reg
        self.spd = torch.tensor([int(np.linalg.eigvalsh(q + reg * np.eye(len(q))).min() <= 0) for q in self.Q])

    def solve(self, d, rx, rs, rz, ry):
        d, rx, rs, rz, ry = (t.detach().cpu().numpy() for t in (d, rx, rs, rz, ry))
        B, m, n = self.G.shape
        e, r = self.A.shape[1], self.reg
        out = []
        for i in range(B):
            K = np.zeros((n + 2 * m + e,) * 2)
            K[:n, :n] = self.Q[i] + r * np.eye(n); K[:n, n + m:n + 2 * m] = self.G[i].T; K[:n, n + 2 * m:] = self.A[i].T
            K[n:n + m, n:n + m] = np.diag(d[i] + r); K[n:n + m, n + m:n + 2 * m] = np.eye(m)
            K[n + m:n + 2 * m, :n] = self.G[i]; K[n + m:n + 2 * m, n:n + m] = np.eye(m)
            K[n + m:n + 2 * m, n + m:n + 2 * m] = -r * np.eye(m)
            K[n + 2 * m:, :n] = self.A[i]; K[n + 2 * m:, n + 2 * m:] = -r * np.eye(e)
            out.append(np.linalg.solve(K, -np.concatenate([rx[i], rs[i], rz[i], ry[i]])))
        s = torch.tensor(np.stack(out))
        return s[:, :n], s[:, n:n + m], s[:, n + m:n + 2 * m], s[:, n + 2 * m:]


def test_equality_only_route(monkeypatch):
    """nineq == 0 with IR_UNOPT: the regularised factor plus refinement, dependent rows of A and a singular Q."""
    from qpth_b200 import KKTSolvers, QPFunction, eqonly, kkt
    seen = []
    monkeypatch.setattr(eqonly, "_factor", lambda Q, G, A, reg: seen.append(reg) or RegDenseFactor(Q, G, A, reg))
    monkeypatch.setattr(eqonly, "_target_device", lambda Q_: torch.device("cpu"))
    r = np.random.RandomState(2)
    nz = 12
    F = r.randn(nz, 8)
    A = r.randn(4, nz)
    A = np.vstack([A, A[:1]])
    Q = torch.tensor(F @ F.T, requires_grad=True)
    p = torch.tensor(r.randn(nz), requires_grad=True)
    At = torch.tensor(A)
    b = torch.tensor(A @ r.randn(nz))
    e = torch.Tensor()
    z = QPFunction(kkt_solver=KKTSolvers.IR_UNOPT)(Q, p, e, e, At, b)
    assert seen == [kkt.IR_EPS]
    K = np.block([[Q.detach().numpy(), A.T], [A, np.zeros((5, 5))]])
    sol = np.linalg.lstsq(K, np.concatenate([-p.detach().numpy(), b.numpy()]), rcond=None)[0]
    assert np.abs(z.detach().numpy() - sol[:nz]).max() <= 1e-9 * np.abs(sol[:nz]).max()
    dl = torch.tensor(r.randn(1, nz))
    (z * dl).sum().backward()
    dsol = np.linalg.lstsq(K, np.concatenate([-dl.numpy()[0], np.zeros(5)]), rcond=None)[0][:nz]
    assert np.abs(p.grad.numpy() - dsol).max() <= 1e-7 * np.abs(dsol).max()
    with pytest.raises(RuntimeError, match="Q is not SPD."):
        QPFunction()(torch.zeros(nz, nz), p.detach(), e, e, At, b)
    with pytest.raises(RuntimeError, match="positive semidefinite"):
        QPFunction(kkt_solver=KKTSolvers.IR_UNOPT)(-torch.eye(nz, dtype=torch.float64), p.detach(), e, e, At, b)
