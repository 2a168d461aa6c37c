"""QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) on the device: QPs with a positive SEMIdefinite Q (LPs, low-rank Q) or
linearly dependent equality rows (the 4x4 sudoku layer with its full 64-row A), against the numpy model of the kernels'
arithmetic (oracle/reg_model.py), scipy HiGHS for the LPs, the KKT residuals of the returned point, and the gradients of
the dense implicit differentiation of the true KKT system (oracle/psd_cases.dense_grads)."""
import numpy as np
import pytest
import torch

from oracle import psd_cases as pc, reg_model as rm

pytestmark = pytest.mark.gpu


def _qpth():
    from qpth_b200 import KKTSolvers, QPFunction, kkt
    return QPFunction, KKTSolvers, kkt


def _run(cases, dl, shared=False, **opts):
    """Solve a batch of numpy cases with IR_UNOPT; returns (z, lam, s, grads dict, last solve)."""
    QPFunction, KKTSolvers, _ = _qpth()
    t = lambda a: torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda", requires_grad=True)  # noqa: E731
    if shared:
        Q, p, G, h, A, b = cases[0]
        ins = [t(Q), t(np.stack([c[1] for c in cases])), t(G), t(h), t(A), t(b)]
    else:
        ins = [t(np.stack([c[k] for c in cases])) for k in range(6)]
    if ins[4].numel() == 0:
        ins[4] = torch.empty(0, dtype=torch.float64, device="cuda")
        ins[5] = torch.empty(0, dtype=torch.float64, device="cuda")
    f = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT, **opts)
    z = f(*ins)
    (z * torch.tensor(dl, device="cuda")).sum().backward()
    st = f.last_solve()
    grads = {k: ins[i].grad.cpu().numpy() for i, k in enumerate(("dQ", "dp", "dG", "dh")) if ins[i].grad is not None}
    return z.detach().cpu().numpy(), st.lam.cpu().numpy(), st.slacks.cpu().numpy(), grads, st


def _rel(a, b, floor=1e-8):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


CASES = {
    "lp": lambda s: pc.lp(s),
    "lowrank": lambda s: pc.lowrank(s),
    "sudoku4": lambda s: pc.sudoku4(s),
    "tiny_lp": lambda s: pc.lp(s, nz=10, nrand=4, neq=2),
    "spd": lambda s: pc.spd(s),
    "large": lambda s: pc.large(s),
}
# Gradients pinned where the backward solve is well conditioned: LPs and the sudoku layer have inactive rows with
# d = 1e-8 / s below eps (qpth's clamp, qp.py:148), where the regularised backward solve, and the gradient itself, move
# with the last bits of the returned point (the model's and the kernels' points agree to 1e-8, not bit for bit).
GRAD_PINNED = ("lowrank", "spd", "large")
GRAD_TOL = 1e-5


@pytest.mark.parametrize("name", list(CASES))
def test_matches_model_and_kkt(name):
    _, _, kkt = _qpth()
    cases = [CASES[name](s) for s in range(3)]
    nz = cases[0][0].shape[0]
    dl = np.random.RandomState(7).randn(3, nz)
    z, lam, s, grads, st = _run(cases, dl)
    if name == "large":
        assert st.plan.pf_global == 1
    elif name == "tiny_lp":
        assert st.plan.tiny == 0 and st.plan.ms_pad <= 32
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


@pytest.mark.parametrize("name", ["lp", "tiny_lp"])
def test_lp_optimum_matches_highs(name):
    from scipy.optimize import linprog
    cases = [CASES[name](s) for s in range(3)]
    z = _run(cases, np.zeros((3, cases[0][0].shape[0])))[0]
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        res = linprog(p, A_ub=G, b_ub=h, A_eq=A, b_eq=b, bounds=(None, None), method="highs")
        assert res.status == 0
        assert abs(p @ z[i] - res.fun) <= 1e-9 * abs(res.fun)
        assert np.linalg.norm(z[i] - res.x) <= 1e-7 * np.linalg.norm(res.x)


def test_shared_inputs_mean_gradients():
    """Q, G, h, A, b shared, p batched: the shared inputs get the batch mean of the per-QP gradients."""
    _, _, kkt = _qpth()
    cases = [pc.lowrank(0)] * 4
    r = np.random.RandomState(3)
    cases = [(c[0], c[1] + 0.1 * r.randn(c[1].size)) + c[2:] for c in cases]
    dl = r.randn(4, cases[0][0].shape[0])
    z, lam, s, grads, _ = _run(cases, dl, shared=True)
    per = []
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=kkt.IR_EPS, steps=kkt.IR_STEPS)
        per.append(rm.backward_one_reg(sol, dl[i]))
    for k in ("dQ", "dG", "dh"):
        assert _rel(grads[k], np.mean([g[k] for g in per], 0)) <= GRAD_TOL, k
    assert _rel(grads["dp"], np.stack([g["dp"] for g in per])) <= GRAD_TOL


def test_spd_problem_agrees_with_default_mode():
    QPFunction, KKTSolvers, _ = _qpth()
    cases = [pc.spd(s) for s in range(4)]
    ins = [torch.tensor(np.stack([c[k] for c in cases]), device="cuda") for k in range(6)]
    z0 = QPFunction(verbose=-1)(*ins)
    z1 = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(*ins)
    assert _rel(z1.cpu().numpy(), z0.cpu().numpy()) <= 1e-8


def test_refinement_steps(monkeypatch):
    """IR_STEPS = 0 and 2 follow the model too."""
    _, _, kkt = _qpth()
    for steps in (0, 2):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        cases = [pc.lowrank(s) for s in range(2)]
        dl = np.random.RandomState(1).randn(2, 60)
        z, lam, s, grads, _ = _run(cases, dl)
        for i, (Q, p, G, h, A, b) in enumerate(cases):
            sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=kkt.IR_EPS, steps=steps)
            assert _rel(z[i], sol["x"]) <= 1e-8
            g = rm.backward_one_reg(sol, dl[i])
            assert _rel(grads["dp"][i], g["dp"]) <= GRAD_TOL


def test_psd_check_and_default_mode_errors():
    QPFunction, KKTSolvers, _ = _qpth()
    Q, p, G, h, A, b = (torch.tensor(a, device="cuda") for a in pc.lp(0))
    with pytest.raises(RuntimeError, match="Q is not SPD."):
        QPFunction(verbose=-1)(Q, p, G, h, A, b)
    QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(Q, p, G, h, A, b)
    Qn = Q.clone()
    Qn[0, 0] = -1e-3
    with pytest.raises(RuntimeError, match="Q is not positive semidefinite."):
        QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(Qn, p, G, h, A, b)
    QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT, check_Q_spd=False)(Qn, p, G, h, A, b)


def test_verbose_trace(capsys):
    QPFunction, KKTSolvers, _ = _qpth()
    ins = [torch.tensor(a, device="cuda") for a in pc.lp(0)]
    QPFunction(verbose=1, kkt_solver=KKTSolvers.IR_UNOPT)(*ins)
    out = capsys.readouterr().out
    assert "iter: 0, pri_resid:" in out
    last = [ln for ln in out.splitlines() if ln.startswith("iter:")][-1]
    assert float(last.split("dual_resid: ")[1].split(",")[0]) <= 1e-9


def test_fp32_and_cpu_inputs():
    QPFunction, KKTSolvers, _ = _qpth()
    case = pc.sudoku4(0)                      # (a rank-5 Q rounded to fp32 is no longer positive semidefinite)
    ref = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(*[torch.tensor(a, device="cuda") for a in case])
    zc = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(*[torch.tensor(a) for a in case])
    assert zc.device.type == "cpu" and zc.dtype == torch.float64
    assert torch.equal(zc, ref.cpu())
    z32 = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(*[torch.tensor(a, dtype=torch.float32, device="cuda")
                                                                    for a in case])
    assert z32.dtype == torch.float32
    assert _rel(z32.double().cpu().numpy(), ref.cpu().numpy()) <= 1e-5


def test_equality_only_with_dependent_rows():
    """nineq == 0: the regularised one-solve route of eqonly.py, A with a repeated row, Q singular off null(A)."""
    QPFunction, KKTSolvers, _ = _qpth()
    r = np.random.RandomState(2)
    nz = 12
    F = r.randn(nz, 8)
    A = r.randn(4, nz)
    A = np.vstack([A, A[:1]])
    b = A @ r.randn(nz)
    p = r.randn(nz)
    Q = F @ F.T
    e = torch.empty(0, dtype=torch.float64, device="cuda")
    z = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT)(*(torch.tensor(a, device="cuda") for a in (Q, p)), e, e,
                                                              *(torch.tensor(a, device="cuda") for a in (A, b)))
    K = np.block([[Q, A.T], [A, np.zeros((5, 5))]])
    ref = np.linalg.lstsq(K, np.concatenate([-p, b]), rcond=None)[0][:nz]
    assert _rel(z.cpu().numpy(), ref) <= 1e-8
