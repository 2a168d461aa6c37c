"""QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) beyond the product-form kernels: LPs and low-rank QPs of order ms_pad
above what qpb200_plan_init_reg takes run on the generic global-scratch kernels (k_forward / k_solve_kkt with kReg).
Checked against the numpy model of the kernels' arithmetic (oracle/reg_model.py), scipy HiGHS, the KKT residuals of the
returned point, the dense implicit differentiation (oracle/psd_cases.dense_grads) and the default mode. Tolerances are
those of tests/test_gpu_psd.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import kernel_model as km, psd_cases as pc, psd_large_cases as lc, reg_model as rm

pytestmark = pytest.mark.gpu

GRAD_TOL = 1e-5


def _qpth():
    from qpth_b200 import KKTSolvers, QPFunction, _lib, kkt
    return QPFunction, KKTSolvers, kkt, _lib


def _global_plan(case):
    """The plan IR_UNOPT uses for a case, asserted to be the global-scratch one."""
    _, _, _, L = _qpth()
    Q, p, G, h, A, b = case
    plan = L.plan_for_ir(Q.shape[0], G.shape[0], A.shape[0])
    assert plan.pf == 0 and plan.smem_resident == 0 and plan.tiny == 0
    return plan


def _t(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda", requires_grad=grad)


def _run(cases, dl, shared=False, **opts):
    """Solve a batch of numpy cases with IR_UNOPT; returns (z, lam, s, grads dict, last solve)."""
    QPFunction, KKTSolvers, _, _ = _qpth()
    _global_plan(cases[0])
    if shared:
        Q, p, G, h, A, b = cases[0]
        ins = [_t(Q, True), _t(np.stack([c[1] for c in cases]), True), _t(G, True), _t(h, True), _t(A, True), _t(b, True)]
    else:
        ins = [_t(np.stack([c[k] for c in cases]), True) for k in range(6)]
    f = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT, **opts)
    z = f(*ins)
    (z * torch.tensor(dl, device="cuda")).sum().backward()
    st = f.last_solve()
    grads = {k: ins[i].grad.cpu().numpy() for i, k in enumerate(("dQ", "dp", "dG", "dh")) if ins[i].grad is not None}
    return z.detach().cpu().numpy(), st.lam.cpu().numpy(), st.slacks.cpu().numpy(), grads, st


def _rel(a, b, floor=1e-8):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


CASES = {
    "lp280": lc.lp280,
    "lowrank120": lc.lowrank120,
    "lp232": lc.lp232,
    "lp664": lc.lp664,
    "lp_dependent": lc.lp_dependent,
}
GRAD_PINNED = ("lowrank120",)     # LPs: inactive rows below eps after qpth's 1e-8 clamp (see test_gpu_psd.GRAD_PINNED)


@pytest.mark.parametrize("name", list(CASES))
def test_matches_model_and_kkt(name):
    _, _, kkt, L = _qpth()
    cases = [CASES[name](s) for s in range(2)]
    Q0, _, G0, _, A0, _ = cases[0]
    if name == "lp232":                            # inside 256 rows, but refused by the product-form plan
        with pytest.raises(L.QpthB200Error, match="too large"):
            L.plan_for_reg(Q0.shape[0], G0.shape[0], A0.shape[0])
    nz = Q0.shape[0]
    dl = np.random.RandomState(7).randn(len(cases), nz)
    z, lam, s, grads, st = _run(cases, dl)
    assert st.plan.pf == 0 and st.plan.smem_resident == 0
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=kkt.IR_EPS, steps=kkt.IR_STEPS)
        assert _rel(z[i], sol["x"]) <= 1e-8
        assert _rel(lam[i], sol["lam"]) <= 1e-8
        assert _rel(s[i], sol["s"]) <= 1e-8
        nu = st.nus[i].cpu().numpy() if st.nus is not None else None
        r = pc.kkt_residuals(Q, p, G, h, A, b, z[i], lam[i], s[i], nu)
        assert max(r) <= 1e-9, r
        for k in ("dQ", "dp", "dG", "dh"):
            assert np.isfinite(grads[k][i]).all(), k
        if name in GRAD_PINNED:
            g = rm.backward_one_reg(sol, dl[i])
            gd = pc.dense_grads(Q, G, A, z[i], lam[i], s[i], nu, dl[i])
            for k in ("dQ", "dp", "dG", "dh"):
                assert _rel(grads[k][i], g[k]) <= GRAD_TOL, k
                assert _rel(grads[k][i], gd[k]) <= GRAD_TOL, k


@pytest.mark.parametrize("name", ["lp280", "lp664", "lp_dependent"])
def test_lp_optimum_matches_highs(name):
    from scipy.optimize import linprog
    cases = [CASES[name](s) for s in range(2)]
    z = _run(cases, np.zeros((2, cases[0][0].shape[0])))[0]
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        res = linprog(p, A_ub=G, b_ub=h, A_eq=A, b_eq=b, bounds=(None, None), method="highs")
        assert res.status == 0
        assert abs(p @ z[i] - res.fun) <= 1e-9 * abs(res.fun)
        assert np.linalg.norm(z[i] - res.x) <= 1e-7 * np.linalg.norm(res.x)


def test_sudoku9_lp_relaxation_matches_highs():
    """The 9x9 sudoku LP relaxation (Q = 0, z >= 0, 249 independent rows, order 992) with random linear terms: the
    optimum is degenerate, so the objective and the KKT residuals are compared, not the point."""
    from scipy.optimize import linprog
    cases = lc.sudoku9_lp(0, B=2)
    plan = _global_plan(cases[0])
    assert plan.ms_pad == 992
    z, lam, s, grads, st = _run(cases, np.random.RandomState(2).randn(2, 729))
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        res = linprog(p, A_ub=G, b_ub=h, A_eq=A, b_eq=b, bounds=(None, None), method="highs")
        assert res.status == 0
        assert abs(p @ z[i] - res.fun) <= 1e-9 * abs(res.fun)
        r = pc.kkt_residuals(Q, p, G, h, A, b, z[i], lam[i], s[i], st.nus[i].cpu().numpy())
        assert max(r) <= 1e-9, r
        for k in ("dp", "dh"):
            assert np.isfinite(grads[k][i]).all(), k


@pytest.mark.parametrize("shape", [(120, 260, 0), (121, 257, 3)])
def test_spd_problem_agrees_with_default_mode(shape):
    QPFunction, KKTSolvers, _, _ = _qpth()
    nz, nineq, neq = shape
    cases = [pc.spd(s, nz=nz, nineq=nineq, neq=neq) for s in range(3)]
    _global_plan(cases[0])
    ins = [torch.tensor(np.stack([c[k] for c in cases]), device="cuda") for k in range(6)]
    if neq == 0:
        ins[4] = ins[5] = torch.empty(0, dtype=torch.float64, device="cuda")
    z0 = QPFunction(verbose=-1)(*ins)
    z1 = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(*ins)
    assert _rel(z1.cpu().numpy(), z0.cpu().numpy()) <= 1e-8


def test_shared_inputs_mean_gradients():
    """Q, G, h, A, b shared, p batched: the shared inputs get the batch mean of the per-QP gradients."""
    _, _, kkt, _ = _qpth()
    base = lc.lowrank120(0)
    r = np.random.RandomState(3)
    cases = [(base[0], base[1] + 0.1 * r.randn(base[1].size)) + base[2:] for _ in range(4)]
    dl = r.randn(4, base[0].shape[0])
    z, lam, s, grads, _ = _run(cases, dl, shared=True)
    per = []
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=kkt.IR_EPS, steps=kkt.IR_STEPS)
        per.append(rm.backward_one_reg(sol, dl[i]))
    for k in ("dQ", "dG", "dh"):
        assert _rel(grads[k], np.mean([g[k] for g in per], 0)) <= GRAD_TOL, k
    assert _rel(grads["dp"], np.stack([g["dp"] for g in per])) <= GRAD_TOL


def test_refinement_steps(monkeypatch):
    """IR_STEPS = 0 and 2 follow the model too."""
    _, _, kkt, _ = _qpth()
    for steps in (0, 2):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        cases = [lc.lowrank120(s) for s in range(2)]
        dl = np.random.RandomState(1).randn(2, 120)
        z, lam, s, grads, _ = _run(cases, dl)
        for i, (Q, p, G, h, A, b) in enumerate(cases):
            sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=kkt.IR_EPS, steps=steps)
            assert _rel(z[i], sol["x"]) <= 1e-8
            g = rm.backward_one_reg(sol, dl[i])
            assert _rel(grads["dp"][i], g["dp"]) <= GRAD_TOL


def test_psd_check():
    QPFunction, KKTSolvers, _, _ = _qpth()
    case = lc.lp280(0)
    _global_plan(case)
    Q, p, G, h, A, b = (torch.tensor(a, device="cuda") for a in case)
    with pytest.raises(RuntimeError, match="Q is not SPD."):
        QPFunction(verbose=-1)(Q, p, G, h, A, b)
    Qn = Q.clone()
    Qn[0, 0] = -1e-3
    with pytest.raises(RuntimeError, match="Q is not positive semidefinite."):
        QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(Qn, p, G, h, A, b)


def test_verbose_trace(capsys):
    QPFunction, KKTSolvers, _, _ = _qpth()
    case = lc.lp280(0)
    _global_plan(case)
    QPFunction(verbose=1, kkt_solver=KKTSolvers.IR_UNOPT)(*[torch.tensor(a, device="cuda") for a in case])
    out = capsys.readouterr().out
    assert "iter: 0, pri_resid:" in out
    last = [ln for ln in out.splitlines() if ln.startswith("iter:")][-1]
    assert float(last.split("dual_resid: ")[1].split(",")[0]) <= 1e-9


def test_c_abi_plan_checks():
    """forward_reg takes a global-scratch plan only with scratch (else QPB200_ERR_BAD_ARG = 1), and still refuses the
    one-warp plans (QPB200_ERR_TOO_LARGE = 4). Both return before any launch."""
    _, _, kkt, L = _qpth()
    lib = L.load()
    buf = torch.zeros(1 << 16, dtype=torch.float64, device="cuda")
    ib = torch.zeros(16, dtype=torch.int32, device="cuda")
    P = ctypes.c_void_p(buf.data_ptr())
    I = ctypes.c_void_p(ib.data_ptr())

    def fwd(plan, scratch):
        return lib.qpb200_forward_reg(ctypes.byref(plan), 1, P, 0, P, 0, P, 0, P, P, P, 0, 1e-12, 1e-6, 1.5, 3, 20,
                                      float(kkt.IR_EPS), 1, P, P, P, P, I, P, None, scratch, None)
    g = L.plan_for(100, 260, 10, two=False)
    assert (g.tiny, g.pf, g.smem_resident) == (0, 0, 0)
    assert fwd(g, None) == 1
    tiny = L.plan_for(10, 24, 2)
    assert tiny.tiny == 1
    assert fwd(tiny, P) == 4


def _highs_point(case):
    from scipy.optimize import linprog
    Q, p, G, h, A, b = case
    res = linprog(p, A_ub=G, b_ub=h, A_eq=A, b_eq=b, bounds=(None, None), method="highs")
    assert res.status == 0
    return res.x, -res.ineqlin.marginals, np.maximum(res.ineqlin.residual, 0.0), -res.eqlin.marginals


@pytest.mark.parametrize("which", ["product_form", "global_scratch"])
def test_solution_function_on_highs_lp_solutions(which):
    """QPSolutionFunction(kkt_solver=IR_UNOPT) differentiates an LP solved by HiGHS (duals from its marginals): dp and
    dh agree with reg_model.backward_one_reg at the same point. (The default mode raises 'Q is not SPD.' there.)"""
    from qpth_b200 import KKTSolvers, QPSolutionFunction, _lib as L, kkt
    cases = [pc.lp(s) if which == "product_form" else lc.lp280(s) for s in range(2)]
    Q0, _, G0, _, A0, _ = cases[0]
    plan = L.plan_for_ir(Q0.shape[0], G0.shape[0], A0.shape[0])
    assert plan.pf == (1 if which == "product_form" else 0)
    pts = [_highs_point(c) for c in cases]
    ins = [_t(np.stack([c[k] for c in cases]), k in (1, 3)) for k in range(6)]
    sol = [torch.tensor(np.stack([pt[k] for pt in pts]), device="cuda") for k in range(4)]
    z = QPSolutionFunction(kkt_solver=KKTSolvers.IR_UNOPT)(*ins, sol[0], sol[1], sol[2], sol[3])
    assert torch.equal(z.detach(), sol[0])
    dl = np.random.RandomState(4).randn(2, Q0.shape[0])
    (z * torch.tensor(dl, device="cuda")).sum().backward()
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        x, lam, s, nu = pts[i]
        state = dict(x=x, lam=lam, s=s, nu=nu, f=km.setup(Q, G, A, kkt.IR_EPS), reg=kkt.IR_EPS, steps=kkt.IR_STEPS,
                     Q=Q, G=G, A=A)
        g = rm.backward_one_reg(state, dl[i])
        # At an LP vertex dz*/dp = 0: dp is the rounding-level remainder of the regularised solve (about 1e-6 |dl|), so
        # both gradients are compared relative to the scale of dl rather than to their own
        scale = np.abs(dl[i]).max()
        assert _rel(ins[1].grad[i].cpu().numpy(), g["dp"], floor=scale) <= GRAD_TOL
        assert _rel(ins[3].grad[i].cpu().numpy(), g["dh"], floor=scale) <= GRAD_TOL
