"""The refinement of the regularised mode (QPFunction kkt_solver=IR_UNOPT) in the numpy model of the kernels'
arithmetic (oracle/reg_model.py), without a GPU.

Every KKT solve of that mode factors K~ = K + Delta (eps = 1e-7 on the four diagonal blocks) and refines against the
true K. Refinement step j must solve K~ cj = Delta c(j-1) from the LAST correction, so that the total is
sum_j (K~^-1 Delta)^j d0; a step built from the running total instead computes (I + K~^-1 Delta)^k d0, which undoes the
first step's gain at the second and loses accuracy from the third on. Checked here at a chosen point (lam, s ~
U(0.1, 10): qpth's 1e-8 clamps inactive) against a refined dense solve of the true system (oracle/dense_kkt.py).

Measured with the model (largest relative 2-norm error of dx, ds, dz at k = 0, 1, 2 steps; the same from there on;
a step built from the running total gives 2.4e-7, 4.3e-7, 1.4e-6 for spd, lowrank, lp at k = 2 and grows by that
much per further step):
  spd        (nz, nineq, neq) = (40, 30, 6)    2.4e-7, 4.8e-14, 3.0e-15
  large                         (100, 200, 0)  3.6e-7, 9.3e-9,  9.3e-9
  lowrank120                    (120, 240, 5)  4.5e-7, 1.0e-8,  1.0e-8
  lowrank                       (60, 160, 5)   4.1e-7, 4.1e-8,  4.1e-8
  lp                            (50, 170, 10)  1.3e-6, 2.2e-7,  2.2e-7
The LP row is the floor of Q = 0: chol(Q + eps I) = sqrt(eps) I makes W ~ G / 3e-4 and limits every solve to about
2e-7 relative, whatever the step count; so only cases with a moderately conditioned Q can tell a refinement error.
"""
import numpy as np
import pytest

from oracle import dense_kkt as dk, kernel_model as km, psd_cases as pc, psd_large_cases as lc, reg_model as rm

EPS = 1e-7

CASES = {
    "spd": lambda: pc.spd(0),
    "large": lambda: pc.large(0),
    "lowrank120": lambda: lc.lowrank120(0),
    "lowrank": lambda: pc.lowrank(0),
    "lp": lambda: pc.lp(0),
}


def _point(case, seed=11):
    Q, p, G, h, A, b = case
    r = np.random.RandomState(seed)
    m, n = G.shape
    lam, s = r.uniform(0.1, 10, m), r.uniform(0.1, 10, m)
    return lam, s, r.randn(n)


def _model_dx(case, d, rhs, steps):
    """dx of the model's backward solve (rx = rhs, rs = rz = ry = 0) with `steps` refinement steps."""
    Q, p, G, h, A, b = case
    m, e = G.shape[0], A.shape[0]
    f = km.setup(Q, G, A, EPS)
    with np.errstate(all="ignore"):
        F = rm._factor(f, d, EPS)
        return rm._solve(f, F, EPS, Q, G, A, rhs, np.zeros(m), np.zeros(m), np.zeros(e) if e else None, steps)


def _true(case, d, rhs):
    Q, p, G, h, A, b = case
    m, e = G.shape[0], A.shape[0]
    return dk.solve(Q, G, A, d, rhs, np.zeros(m), np.zeros(m), np.zeros(e), reg=0.0)


@pytest.mark.parametrize("name", list(CASES))
def test_refinement_error_does_not_grow(name):
    """The error of dx, ds, dz against the true solve never grows from k to k + 1 steps (k = 0 .. 4; 1 % slack for
    rounding once converged), and on the SPD case it reaches rounding level from two steps on."""
    case = CASES[name]()
    lam, s, rhs = _point(case)
    d = lam / s
    tx, ts, tz, _, _, _ = _true(case, d, rhs)
    errs = []
    for k in range(6):
        dx, ds, dz, _ = _model_dx(case, d, rhs, k)
        errs.append(max(dk.rel(dx, tx), dk.rel(ds, ts), dk.rel(dz, tz)))
    for k in range(5):
        assert errs[k + 1] <= 1.01 * errs[k] + 1e-15, (k, errs)
    assert errs[1] < errs[0] or name == "lp", errs           # (the LP floor: see the module docstring)
    if name == "spd":
        assert max(errs[2:]) <= 1e-13, errs
        assert errs[0] >= 1e-8, errs                          # one solve alone is off by O(eps): the test can tell


def test_steps_zero_and_one_unchanged():
    """k = 0 and 1 are the unrefined solve and one step against its own residual, as before the fix: the first step's
    residual is that of the solution itself."""
    case = pc.spd(1)
    Q, p, G, h, A, b = case
    lam, s, rhs = _point(case)
    d = lam / s
    m, e = G.shape[0], A.shape[0]
    f = km.setup(Q, G, A, EPS)
    F = rm._factor(f, d, EPS)
    L22, dt = F

    def one(rx, rs, rz, ry):
        dxt, ds, dz, dy = km._solve_kkt(f, L22, dt, km._tri(f["L"], rx), rs, rz, ry)
        return km._tri(f["L"], dxt, trans=True), ds, dz, dy

    d0 = one(rhs, np.zeros(m), np.zeros(m), np.zeros(e))
    c = one(-EPS * d0[0], -EPS * d0[1], EPS * d0[2], EPS * d0[3])
    got0 = _model_dx(case, d, rhs, 0)
    got1 = _model_dx(case, d, rhs, 1)
    for a, b_ in zip(got0, d0):
        assert np.array_equal(a, b_)
    for a, x, y in zip(got1, d0, c):
        assert np.array_equal(a, x + y)


@pytest.mark.parametrize("steps", [0, 1, 2])
@pytest.mark.parametrize("name", ["spd", "lowrank", "lp"])
def test_trace_rows_are_true_residuals(name, steps):
    """solve_one_reg(trace=...): row it is [pri, dual, mu, resid] of the TRUE problem at the iterate it. Replayed by
    re-running the loop truncated at it + 1 iterations, whose returned point is then the last (best) iterate or an
    earlier one with the recorded best_resid."""
    case = CASES[name]()
    Q, p, G, h, A, b = case
    m = G.shape[0]
    tr = []
    full = rm.solve_one_reg(Q, p, G, h, A, b, reg=EPS, steps=steps, trace=tr)
    assert len(tr) == full["iters"]
    for it in range(len(tr)):
        sub = []
        sol = rm.solve_one_reg(Q, p, G, h, A, b, reg=EPS, steps=steps, trace=sub, maxIter=it + 1)
        assert sub == tr[:it + 1]                             # truncation does not change the earlier rows
        x, z, s, y = sol["x"], sol["lam"], sol["s"], sol["nu"]
        row = tr[sol["best_iter"]]
        rx = Q @ x + p + G.T @ z + (A.T @ y if A.shape[0] else 0.0)
        pri = np.linalg.norm(G @ x + s - h) + (np.linalg.norm(A @ x - b) if A.shape[0] else 0.0)
        mu = abs(s @ z / m)
        scale = 1.0 + np.abs(p).max() + np.abs(h).max()
        assert abs(row[0] - pri) <= 1e-12 * scale * (1 + row[0]), (it, row[0], pri)
        assert abs(row[1] - np.linalg.norm(rx)) <= 1e-12 * scale * (1 + row[1]) * (1 + np.abs(Q).max()), it
        assert abs(row[2] - mu) <= 1e-14 * max(mu, 1.0), it
        assert row[3] == pytest.approx(row[0] + row[1] + m * row[2], rel=1e-14)
        assert sol["best_resid"] == min(r[3] for r in sub)
    assert tr[-1][3] <= 1e-9 or full["best_resid"] <= 1e-9


def test_reg_family_plans():
    """The cases of tests/reg_families.py land in their families (the GPU tests assert the same before they solve)."""
    from tests.reg_families import CASES, family_plan, problem
    for fam, kind in CASES:
        family_plan(fam, problem(fam, kind, 0))
