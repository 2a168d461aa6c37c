"""The kReg kernels of QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) below convergence, family by family
(tests/reg_families.py: the smallest product-form plans, the resident and the L2 product-form builds, the generic
global-scratch kernels), each on an SPD-Q, a low-rank-Q and an LP case.

Backward at a chosen point (QPSolutionFunction with random z, nu and lam, s ~ U(0.1, 10), so that qpth's 1e-8 clamps
are inactive), IR_STEPS in {0, 1, 2, 3}:
  * every gradient against oracle/reg_model.backward_one_reg at the same step count;
  * dQ, dp, dG, dh against the refined dense solve of the TRUE KKT system (oracle/dense_kkt.py), within
    max(1e-12, 10 x the model's own error there);
  * the kernels' error against the dense solve does not grow with the step count (a step built from the running total
    instead of the last correction multiplies it by 10 to 1e7 at the second step).
The model's own error (max over the four gradients, relative to their max-norm) at k = 0 / >= 1 is about 2e-7 / 1e-14
on the SPD cases and 1e-7 / 1e-8 .. 2e-7 on the low-rank and LP cases: only the SPD cases can tell a refinement error at
rounding level; on the others (chol(Q + eps I) ~ sqrt(eps) I on Q's null space) it must exceed the floor of ~1e-7.
On the SPD cases of the four families the error from k = 1 on is held to 1e-12. On the SPD cases of the edge entries
it is held to max(1e-12, 10 x the model's error at that k): some of them have many equality rows or a small A Q^-1 A'
(for example 64 rows at nz = 97, or 129 rows at nz = 208). One step contracts less there, and the model's own error at k = 1 is up to 1.1e-11 (measured:
9.6e-12 at 39/144/17, 7.8e-12 at 97/9/64, 3.8e-12 at 208/57/129, 1.1e-11 at 4/193/0). From k = 2 on it is below 1e-13.

Forward trajectories (every family but the backward_only one of tests/reg_families.py): maxIter in {1, 2, 3, 5, 20}, eps in {1e-12, 1e-6}, IR_STEPS in {0, 1, 2}, qp.TRACE on:
  * each trace row [pri, dual, mu, resid] against reg_model.solve_one_reg(trace=...), row-relative l2 error within
    ROW_TOL[case] while the model's resid >= 1e-3, ROW_TOL[case] x 1e-3 / resid for 1e-6 <= resid < 1e-3, and
    unchecked below (the iterates sit at the rounding floor there);
  * truncated runs: z, lam, s, nu within ROW_TOL[case] relative, the same iteration count; full runs converge as far
    as the model (the eps = 1e-12 exit sits at the rounding floor, so their counts may differ); best_resid is the smallest
    resid of the trace.
ROW_TOL is 10 x the model's own spread: perturbing p and h by 1e-15 relative (three sign draws, seeds 0 and 1,
IR_STEPS 0 .. 2) moves the model's rows by the amounts in MODEL_SPREAD (max over rows with resid >= 1e-3, and of
row error x resid / 1e-3 over 1e-6 <= resid < 1e-3).
"""
import numpy as np
import pytest
import torch

from oracle import dense_kkt as dk, kernel_model as km, reg_model as rm
from tests.reg_families import CASES, FAMILIES, family_plan, ids, problem

pytestmark = pytest.mark.gpu

B = 2
# (rows with resid >= 1e-3, rows with 1e-6 <= resid < 1e-3 scaled by resid / 1e-3)
MODEL_SPREAD = {
    ("pf_small", "spd"): (1.6e-12, 1.3e-11),
    ("pf_small", "lowrank"): (2.3e-7, 3.2e-7),
    ("pf_small", "lp"): (1.0e-7, 5.9e-7),
    ("pf_resident", "spd"): (2.2e-11, 5.4e-11),
    ("pf_resident", "lowrank"): (5.3e-6, 6.4e-6),
    ("pf_resident", "lp"): (9.9e-7, 1.8e-6),
    ("pf_l2", "spd"): (6.5e-11, 2.1e-10),
    ("pf_l2", "lowrank"): (2.3e-7, 1.0e-7),
    ("pf_l2", "lp"): (3.1e-6, 2.1e-6),
    ("global_scratch", "spd"): (9.7e-11, 4.5e-10),
    ("global_scratch", "lowrank"): (5.7e-7, 7.6e-7),
    ("global_scratch", "lp"): (7.2e-7, 5.1e-7),
    ("edge_pf_res_full", "spd"): (2.8e-13, 3.0e-12),
    ("edge_pf_res_full", "lp"): (8.3e-6, 1.3e-5),
    ("edge_pf_res_order", "spd"): (9.9e-12, 6.1e-12),
    ("edge_pf_res_order", "lp"): (7.9e-5, 3.8e-5),
    ("edge_gs_pf_res", "spd"): (1.3e-12, 2.8e-12),
    ("edge_sf_pf_res", "spd"): (3.5e-12, 4.2e-12),
    ("edge_l2_full", "spd"): (2.0e-12, 4.1e-12),
    ("edge_l2_order", "spd"): (2.5e-12, 4.0e-12),
    ("edge_l2_wide", "spd"): (2.1e-12, 9.7e-12),
}


def _row_tol(case, resid):
    a, b = MODEL_SPREAD[case]
    ta, tb = max(10 * a, 1e-10), max(10 * b, 1e-10)
    return ta if resid >= 1e-3 else (tb * 1e-3 / resid if resid >= 1e-6 else np.inf)


def _qpth():
    from qpth_b200 import KKTSolvers, QPFunction, QPSolutionFunction, kkt, qp
    return QPFunction, QPSolutionFunction, KKTSolvers, kkt, qp


def _t(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda", requires_grad=grad)


def _rel(a, b, floor=1e-300):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


def _point(case, seed):
    Q, p, G, h, A, b = case
    r = np.random.RandomState(50 + seed)
    n, m, e = Q.shape[0], G.shape[0], A.shape[0]
    return r.randn(n), r.uniform(0.1, 10, m), r.uniform(0.1, 10, m), r.randn(e), r.randn(n)


def _dense_grads(case, x, lam, s, nu, dl):
    """Gradients from the refined dense solve of the true KKT system at the point (d = lam / s, clamps inactive)."""
    Q, p, G, h, A, b = case
    m, e = G.shape[0], A.shape[0]
    dx, _, dz, _, _, _ = dk.solve(Q, G, A, lam / s, dl, np.zeros(m), np.zeros(m), np.zeros(e), reg=0.0)
    return dict(dQ=0.5 * (np.outer(dx, x) + np.outer(x, dx)), dp=dx, dG=np.outer(dz, x) + np.outer(lam, dx), dh=-dz)


def _model_grads(case, x, lam, s, nu, dl, steps, eps):
    Q, p, G, h, A, b = case
    st = dict(x=x, lam=lam, s=s, nu=nu if A.shape[0] else None, f=km.setup(Q, G, A, eps), reg=eps, steps=steps,
              Q=Q, G=G, A=A)
    return rm.backward_one_reg(st, dl)


def _backward_on_gpu(cases, pts, shared):
    """Gradients of sum(dl * z) through QPSolutionFunction(kkt_solver=IR_UNOPT) at the given points."""
    _, QPSolutionFunction, KKTSolvers, _, _ = _qpth()
    neq = cases[0][4].shape[0]
    keys = ("dQ", "dp", "dG", "dh", "dA", "db")
    if shared:
        ins = [_t(cases[0][k], k != 4 or neq > 0) if k != 1 else _t(np.stack([c[1] for c in cases]), True)
               for k in range(6)]
    else:
        ins = [_t(np.stack([c[k] for c in cases]), k < 4 or neq > 0) for k in range(6)]
    sol = [_t(np.stack([pt[k] for pt in pts])) for k in range(4)]
    z = QPSolutionFunction(kkt_solver=KKTSolvers.IR_UNOPT)(*ins, *sol)
    (z * _t(np.stack([pt[4] for pt in pts]))).sum().backward()
    return {k: ins[i].grad.cpu().numpy() for i, k in enumerate(keys) if ins[i].grad is not None}


@pytest.mark.parametrize("case", CASES, ids=ids(CASES))
def test_backward_at_chosen_point(case, monkeypatch):
    _, _, _, kkt, _ = _qpth()
    fam, kind = case
    cases = [problem(fam, kind, s) for s in range(B)]
    family_plan(fam, cases[0])
    neq = cases[0][4].shape[0]
    pts = [_point(c, i) for i, c in enumerate(cases)]
    dense = [_dense_grads(c, pt[0], pt[1], pt[2], pt[3], pt[4]) for c, pt in zip(cases, pts)]
    errs, model_errs, worst = [], [], dict(model=0.0)
    for steps in range(4):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        g = _backward_on_gpu(cases, pts, shared=False)
        assert set(g) == {"dQ", "dp", "dG", "dh"} | ({"dA", "db"} if neq else set())
        err = merr = 0.0
        for i, (c, pt) in enumerate(zip(cases, pts)):
            gm = _model_grads(c, *pt, steps, kkt.IR_EPS)
            model_err = max(_rel(gm[k], dense[i][k]) for k in dense[i])
            merr = max(merr, model_err)
            tol = max(1e-12, 10 * model_err)
            for k in g:
                assert _rel(g[k][i], gm[k]) <= tol, (steps, i, k, _rel(g[k][i], gm[k]), tol)
            for k in dense[i]:
                assert _rel(g[k][i], dense[i][k]) <= tol, (steps, i, k, _rel(g[k][i], dense[i][k]), tol)
            err = max(err, max(_rel(g[k][i], dense[i][k]) for k in dense[i]))
            worst["model"] = max(worst["model"], max(_rel(g[k][i], gm[k]) for k in g))
        errs.append(err)
        model_errs.append(merr)
    _report("reg_bwd[%s %s]" % case, dict(worst, **{"dense_k%d" % k: e for k, e in enumerate(errs)}))
    for k in range(3):
        assert errs[k + 1] <= 2 * errs[k] + 1e-13, errs
    if kind == "spd" and "pair" not in FAMILIES[fam]:
        assert max(errs[1:]) <= 1e-12 < errs[0], errs
    elif kind == "spd":                    # edge entries: the bound the model's own error allows (module docstring)
        assert errs[0] > 1e-12, errs
        for k in range(1, 4):
            assert errs[k] <= max(1e-12, 10 * model_errs[k]), (k, errs, model_errs)


@pytest.mark.parametrize("fam", list(FAMILIES))
def test_backward_shared_inputs_mean(fam, monkeypatch):
    """Q, G, h, A, b shared and p batched (B = 3), IR_STEPS = 2: the shared inputs get the batch mean of the per-QP
    gradients of the model, within 1e-12. Edge entries: within max(1e-12, 10 x the model's error against the dense solve),
    the bound of test_backward_at_chosen_point (at order 1056 the refinement contracts slowly, reg_families.py)."""
    _, _, _, kkt, _ = _qpth()
    monkeypatch.setattr(kkt, "IR_STEPS", 2)
    base = problem(fam, "spd", 0)
    family_plan(fam, base)
    r = np.random.RandomState(8)
    cases = [(base[0], base[1] + 0.1 * r.randn(base[1].size)) + base[2:] for _ in range(3)]
    pts = [_point(base, i) for i in range(3)]
    g = _backward_on_gpu(cases, pts, shared=True)
    per = [_model_grads(c, *pt, 2, kkt.IR_EPS) for c, pt in zip(cases, pts)]
    tol = 1e-12
    if "pair" in FAMILIES[fam]:
        for c, pt, gm in zip(cases, pts, per):
            dense = _dense_grads(c, *pt)
            tol = max(tol, 10 * max(_rel(gm[k], dense[k]) for k in dense))
    for k in g:
        want = np.stack([q[k] for q in per]) if k == "dp" else np.mean([q[k] for q in per], 0)
        assert _rel(g[k], want) <= tol, (k, _rel(g[k], want), tol)


def _forward_on_gpu(cases, shared, **opts):
    QPFunction, _, KKTSolvers, _, _ = _qpth()
    neq = cases[0][4].shape[0]
    if shared:
        ins = [_t(cases[0][k]) if k != 1 else _t(np.stack([c[1] for c in cases])) for k in range(6)]
    else:
        ins = [_t(np.stack([c[k] for c in cases])) for k in range(6)]
    if neq == 0:
        ins[4] = ins[5] = torch.empty(0, dtype=torch.float64, device="cuda")
    f = QPFunction(verbose=-1, kkt_solver=KKTSolvers.IR_UNOPT, **opts)
    z = f(*ins).cpu().numpy()
    st = f.last_solve()
    return (z, st.lam.cpu().numpy(), st.slacks.cpu().numpy(), None if st.nus is None else st.nus.cpu().numpy(),
            st.iters.cpu().numpy(), st.best_resid.cpu().numpy(), st.trace.cpu().numpy())


def _report(name, errs):
    from tests.test_gpu_parity import _report as rep
    rep(name, errs)


def _check_forward(case, cases, out, maxIter, eps, steps, reg, worst=None):
    from qpth_b200.qp import BEST_TIE, STALL_TOL
    worst = {} if worst is None else worst
    z, lam, s, nu, iters, best, trace = out
    for i, (Q, p, G, h, A, b) in enumerate(cases):
        tr = []
        m = rm.solve_one_reg(Q, p, G, h, A, b, reg=reg, steps=steps, eps=eps, maxIter=maxIter, stall_tol=STALL_TOL,
                             tie=BEST_TIE, trace=tr)
        tr = np.array(tr)
        k = min(len(tr), int(iters[i]))
        for it in range(k):
            tol = _row_tol(case, tr[it, 3])
            err = np.linalg.norm(trace[i, it] - tr[it]) / np.linalg.norm(tr[it])
            if tr[it, 3] >= 1e-3:
                worst["trace"] = max(worst.get("trace", 0.0), err)
            assert err <= tol, (i, it, err, tol, trace[i, it], tr[it])
        assert best[i] == np.nanmin(trace[i, :int(iters[i]), 3])
        if maxIter < 20:
            assert int(iters[i]) == m["iters"], (i, int(iters[i]), m["iters"])
            tol = _row_tol(case, tr[m["best_iter"], 3])
            if np.isfinite(tol):
                worst["iterate"] = max(worst.get("iterate", 0.0), _rel(z[i], m["x"]))
                assert _rel(z[i], m["x"]) <= tol
                assert _rel(lam[i], m["lam"]) <= tol
                assert _rel(s[i], m["s"]) <= tol
                if nu is not None:
                    assert _rel(nu[i], m["nu"]) <= tol
        else:
            # the eps = 1e-12 exit sits at the rounding floor, where the iteration counts may part: both converge
            assert best[i] <= max(1e-9, 10 * m["best_resid"]), (i, best[i], m["best_resid"])


FWD_CASES = [c for c in CASES if not FAMILIES[c[0]].get("backward_only")]
FWD_FAMILIES = [f for f in FAMILIES if not FAMILIES[f].get("backward_only")]


@pytest.mark.parametrize("case", FWD_CASES, ids=ids(FWD_CASES))
def test_forward_trajectory(case, monkeypatch):
    _, _, _, kkt, qp = _qpth()
    fam, kind = case
    monkeypatch.setattr(qp, "TRACE", True)
    cases = [problem(fam, kind, s) for s in range(B)]
    family_plan(fam, cases[0])
    worst = {}
    for steps in (0, 1, 2):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        for eps in (1e-12, 1e-6):
            for maxIter in (1, 2, 3, 5, 20):
                out = _forward_on_gpu(cases, False, eps=eps, maxIter=maxIter)
                _check_forward(case, cases, out, maxIter, eps, steps, kkt.IR_EPS, worst)
    _report("reg_traj[%s %s]" % case, worst)


@pytest.mark.parametrize("fam", FWD_FAMILIES)
def test_forward_trajectory_shared_inputs(fam, monkeypatch):
    """Q, G, h, A, b shared (one system for the batch), p batched, IR_STEPS = 2, truncated at 3 iterations."""
    _, _, _, kkt, qp = _qpth()
    case = (fam, "spd")
    monkeypatch.setattr(qp, "TRACE", True)
    monkeypatch.setattr(kkt, "IR_STEPS", 2)
    base = problem(fam, "spd", 0)
    family_plan(fam, base)
    r = np.random.RandomState(6)
    cases = [(base[0], base[1] + 0.1 * r.randn(base[1].size)) + base[2:] for _ in range(3)]
    for maxIter in (3, 20):
        out = _forward_on_gpu(cases, True, maxIter=maxIter)
        _check_forward(case, cases, out, maxIter, 1e-12, 2, kkt.IR_EPS)
