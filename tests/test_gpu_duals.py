"""The dual outputs, duals=True, of QPFunction, QPSolutionFunction, BoxQPFunction and the equality-only path on the GPU.

- Every family of tests/kernel_families.py at its backward_point with random g_lam, g_nu (tests/duals_jobs.py): every
  gradient against the formulas applied to oracle/dense_kkt.solve with rz = g_lam and ry = g_nu, within 1e-10 (the
  bound of test_gpu_backward_families.py); with only z used, and with duals=False, the gradients are bit-identical;
  the gradient of g_z'z + g_lam'lam + g_nu'nu is the sum of the three separate ones within 1e-12, or 10 x the error
  against the dense solve where that is larger.
- Batch means of un-batched inputs for the three sharings of test_gpu_backward_families.MEAN_SHARING, within 1e-12.
- Every family of tests/reg_families.py at IR_STEPS 0 .. 3, as test_gpu_reg_families.test_backward_at_chosen_point:
  against the model with the dual adjoints (tests/dual_models.py) and the refined dense solve within
  max(1e-12, 10 x the model's error there), and the error against the dense solve does not grow with the step count.
- Every entry of tests/box_families.py: the box kernels at a chosen point against the box model with the dual
  adjoints within 1e-10, NULL adjoints bit-identical to qpb200_box_backward, linearity; the `dense` entries
  (BoxQPFunction on the dense equivalent) against QPFunction(duals=True) on the dense equivalent.
- End to end: QPFunction, QPSolutionFunction, BoxQPFunction and the equality-only path with duals=True on seeded
  strictly complementary batches (tests/dual_models.py), with and without equality rows: central differences (step
  1e-5) of a loss on z, lam and nu within 1e-5 of the exact implicit derivative, and for the dense path the backward
  within 1e-7 of the implicit derivative with qpth's 1e-8 clamps (_qp_fd says why these are two references).
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import box_model as bm
from oracle import dense_kkt as dk
from tests import dual_models as dm
from tests.duals_jobs import (dual_backward_on_gpu, dual_point, job_name, run_child, solution_backward_duals,
                              variants)
from tests.kernel_families import GRAD_NAMES, cases, family_env, family_plan, ids
from tests.parity import rel_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _reference(pr, i, glam=True, gnu=True):
    """Per-QP gradients from the dense solve with rx = dl, rz = g_lam, ry = g_nu."""
    neq = pr["A"].shape[1]
    d = pr["lam"][i] / pr["s"][i]
    m = d.shape[0]
    dx, _, dlam, dnu, _, _ = dk.solve(pr["Q"][i], pr["G"][i], pr["A"][i], d, pr["dl"][i], np.zeros(m),
                                      pr["glam"][i] if glam else np.zeros(m),
                                      (pr["gnu"][i] if gnu else np.zeros(neq)) if neq else None)
    z, lam = pr["z"][i], pr["lam"][i]
    g = dict(dQ=0.5 * (np.outer(dx, z) + np.outer(z, dx)), dp=dx, dG=np.outer(dlam, z) + np.outer(lam, dx), dh=-dlam)
    if neq:
        g.update(dA=np.outer(dnu, z) + np.outer(pr["nu"][i], dx), db=-dnu)
    return g


def _check_family(fam, shape, got):
    pr = dual_point(fam, shape)
    B = pr["z"].shape[0]
    refs = [_reference(pr, i) for i in range(B)]
    for n in GRAD_NAMES:
        if n not in refs[0]:
            assert all(("%s_%s" % (v, n)) not in got for v in variants(shape[2])), n
            continue
        e = rel_rows(got["all_" + n], np.stack([r[n] for r in refs])).max()
        assert e <= 1e-10, (n, e)
        assert np.array_equal(got["z_" + n], got["base_" + n]), n        # NULL adjoints: the existing call
        # linearity holds to the rounding of the solves: 1e-12, or 10 x the solve's own error against the dense solve
        # where the family's conditioning makes that larger (random_qp_batch families: measured up to 1.5e-11)
        total = got["z_" + n] + got["lam_" + n] + (got["nu_" + n] if shape[2] else 0.0)
        lin = np.abs(got["all_" + n] - total).max() / np.abs(got["all_" + n]).max()
        assert lin <= max(1e-12, 10 * e), (n, lin, e)


@pytest.mark.parametrize("fam,shape", cases(child=False), ids=ids(cases(child=False)))
def test_family_dual_backward(fam, shape):
    _check_family(fam, shape, dual_backward_on_gpu(fam, shape))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("duals_families"))
    return out_dir, run_child(out_dir)


@pytest.mark.parametrize("fam,shape", cases(child=True), ids=ids(cases(child=True)))
def test_family_dual_backward_in_child(fam, shape, child_results):
    from tests import gpu_child
    with family_env(fam):
        family_plan(fam, shape)
    _check_family(fam, shape, gpu_child.load(*child_results, job_name(fam, shape)))


@pytest.mark.parametrize("sharing", ["QGAh_unbatched", "Q_unbatched_G_batched", "p_b_unbatched"])
def test_batch_mean_with_dual_adjoints(sharing):
    from tests.test_gpu_backward_families import MEAN_SHARING
    B, shape = 37, (100, 100, 8)
    bat = MEAN_SHARING[sharing]
    pr = dual_point("pf_one_setup_fast", shape, B)
    for k, v in bat.items():
        if not v:
            pr[k] = np.broadcast_to(pr[k][:1], pr[k].shape).copy()
    got = solution_backward_duals(pr, "all", bat)
    refs = [_reference(pr, i) for i in range(B)]
    for n, k in zip(GRAD_NAMES, "QpGhAb"):
        per = np.stack([r[n] for r in refs])
        if bat[k]:
            assert rel_rows(got[n], per).max() <= 1e-10, n
        else:
            scale = np.mean([np.linalg.norm(x) for x in per])
            assert np.linalg.norm(got[n] - per.mean(0)) / scale <= 1e-12, n


# ---- the regularised mode ------------------------------------------------------------------------------------------------

def _reg_cases():
    from tests.reg_families import CASES
    return CASES


@pytest.mark.parametrize("case", _reg_cases(), ids=["%s-%s" % c for c in _reg_cases()])
def test_reg_family_dual_backward(case, monkeypatch):
    from qpth_b200 import KKTSolvers, kkt
    from oracle import kernel_model as km
    from tests.reg_families import FAMILIES, family_plan as reg_plan, problem
    from tests.test_gpu_reg_families import B, _point, _rel
    fam, kind = case
    probs = [problem(fam, kind, s) for s in range(B)]
    reg_plan(fam, probs[0])
    n, m, e = probs[0][0].shape[0], probs[0][2].shape[0], probs[0][4].shape[0]
    pts = [_point(c, i) for i, c in enumerate(probs)]
    rs = np.random.RandomState(77)
    glam, gnu = rs.randn(B, m), rs.randn(B, e)
    pr = dict(Q=np.stack([c[0] for c in probs]), p=np.stack([c[1] for c in probs]), G=np.stack([c[2] for c in probs]),
              h=np.stack([c[3] for c in probs]), A=np.stack([c[4] for c in probs]), b=np.stack([c[5] for c in probs]),
              z=np.stack([pt[0] for pt in pts]), lam=np.stack([pt[1] for pt in pts]), s=np.stack([pt[2] for pt in pts]),
              nu=np.stack([pt[3] for pt in pts]), dl=np.stack([pt[4] for pt in pts]), glam=glam, gnu=gnu)
    dense = []
    for i in range(B):
        g = _reference(pr, i)
        dense.append({k: g[k] for k in ("dQ", "dp", "dG", "dh")})        # dA, db: not unique for dependent rows
    errs, model_errs = [], []
    for steps in range(4):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        got = solution_backward_duals(pr, "all", kkt_solver=KKTSolvers.IR_UNOPT)
        err = merr = 0.0
        for i in range(B):
            st = dict(x=pr["z"][i], lam=pr["lam"][i], s=pr["s"][i], nu=pr["nu"][i] if e else None,
                      f=km.setup(pr["Q"][i], pr["G"][i], pr["A"][i], kkt.IR_EPS), reg=kkt.IR_EPS, steps=steps,
                      Q=pr["Q"][i], G=pr["G"][i], A=pr["A"][i])
            gm = dm.backward_one_reg(st, pr["dl"][i], glam[i], gnu[i] if e else None)
            model_err = max(_rel(gm[k], dense[i][k]) for k in dense[i])
            merr = max(merr, model_err)
            tol = max(1e-12, 10 * model_err)
            for k in GRAD_NAMES:
                if got[k] is not None:
                    assert _rel(got[k][i], gm[k]) <= tol, (steps, i, k, _rel(got[k][i], gm[k]), tol)
            for k in dense[i]:
                assert _rel(got[k][i], dense[i][k]) <= tol, (steps, i, k, _rel(got[k][i], dense[i][k]), tol)
            err = max(err, max(_rel(got[k][i], dense[i][k]) for k in dense[i]))
        errs.append(err)
        model_errs.append(merr)
    for k in range(3):
        assert errs[k + 1] <= 2 * errs[k] + 1e-13, errs
    if kind == "spd" and "pair" not in FAMILIES[fam]:
        assert max(errs[1:]) <= 1e-12, errs


# ---- the box QP ----------------------------------------------------------------------------------------------------------

def _box_names():
    from tests.box_families import ENTRIES
    return list(ENTRIES)


def _box_point(plan, B, seed):
    rs = np.random.RandomState(seed)
    n, e, m = plan.nz, plan.neq, plan.nineq
    return dict(q=0.5 + rs.rand(B, n), A=rs.randn(B, e, n) / np.sqrt(n), z=rs.randn(B, n), nu=rs.randn(B, e),
                lam=rs.uniform(0.1, 10, (B, m)), s=rs.uniform(0.1, 10, (B, m)), dl=rs.randn(B, n), glam=rs.randn(B, m),
                gnu=rs.randn(B, e))


def _box_backward(plan, pt, dl, glam, gnu, legacy=False):
    """qpb200_box_backward_duals (legacy: qpb200_box_backward) at the point: (dx, dlam, dnu, dq, dp, dlb, dub, dA, db)."""
    from qpth_b200 import _lib
    lib = _lib.load()
    B, n = pt["z"].shape
    e, m = plan.neq, plan.nineq
    T = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if (t is not None and t.numel()) else ctypes.c_void_p(0)
    ins = {k: T(pt[k]) for k in ("q", "A", "z", "nu", "lam", "s")}
    f64 = dict(dtype=torch.float64, device=DEV)
    outs = [torch.empty(B, *s, **f64) for s in ((n,), (m,), (e,), (n,), (n,), (n,), (n,), (e, n), (e,))]
    dxv, dlamv, dnuv, dq, dp, dlb, dub, dA, db = outs
    if not plan.has_lb:
        dlb = None
    if not plan.has_ub:
        dub = None
    grads = [P(dq), 0, P(dp), 0, P(dlb), 0, P(dub), 0, P(dA), 0, P(db), 0]
    common = (ctypes.byref(plan), B, P(ins["q"]), n, P(ins["A"]), e * n)
    tail = (P(ins["z"]), P(ins["lam"]), P(ins["s"]), P(ins["nu"]), *grads, P(dxv), P(dlamv), P(dnuv), ctypes.c_void_p(0))
    adj = [None if a is None else T(a) for a in (dl, glam, gnu)]       # (kept alive until the kernels have run)
    if legacy:
        _lib.check(lib.qpb200_box_backward(*common, P(adj[0]), *tail))
    else:
        _lib.check(lib.qpb200_box_backward_duals(*common, *(P(a) for a in adj), *tail))
    torch.cuda.synchronize()
    return [None if o is None else o.cpu().numpy() for o in (dxv, dlamv, dnuv, dq, dp, dlb, dub, dA, db)]


@pytest.mark.parametrize("name", _box_names())
def test_box_entry_dual_backward(name):
    from tests.box_families import ENTRIES, check_entry, knob, layout, sides_flags
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    with knob(ent["knob"]):
        plan = check_entry(name)
        if layout(plan) == "dense":
            _check_box_dense(n, e, sides)
            return
        B = 2
        pt = _box_point(plan, B, 600 + n + e)
        gnu = pt["gnu"] if e else None
        full = _box_backward(plan, pt, pt["dl"], pt["glam"], gnu)
        nul = _box_backward(plan, pt, pt["dl"], None, None)
        old = _box_backward(plan, pt, pt["dl"], None, None, legacy=True)
        zero = np.zeros_like(pt["dl"])
        lam_only = _box_backward(plan, pt, zero, pt["glam"], None)
        nu_only = _box_backward(plan, pt, zero, None, gnu) if e else None
    lb, ub = sides_flags(sides)
    var, sgn = bm.rows(n, lb, ub)
    names = ("dx", "dlam", "dnu", "dq", "dp", "dlb", "dub", "dA", "db")
    for i in range(B):
        sol = dict(x=pt["z"][i], lam=pt["lam"][i], s=pt["s"][i], nu=pt["nu"][i], q=pt["q"][i], A=pt["A"][i], var=var,
                   sgn=sgn, nlb=n if lb else 0)
        gm = dm.backward_one_box(sol, pt["dl"][i], pt["glam"][i], gnu[i] if e else None)
        for k, g in zip(names, full):
            if g is None or gm.get(k) is None or (k in ("dnu", "dA", "db") and not e):
                continue
            err = np.abs(g[i] - gm[k]).max() / max(np.abs(gm[k]).max(), 1e-300)
            assert err <= 1e-10, (k, i, err)
    for k, a, b in zip(names, nul, old):
        assert (a is None and b is None) or np.array_equal(a, b), k
    for k, f, a, b, c in zip(names, full, nul, lam_only, nu_only or [None] * 9):
        if f is None or (k in ("dnu", "dA", "db") and not e):
            continue
        total = a + b + (c if c is not None else 0.0)
        assert np.abs(f - total).max() <= 1e-12 * np.abs(f).max(), k


def _check_box_dense(n, e, sides):
    """BoxQPFunction(duals=True) on a shape no box kernel takes (the dense kernels on the dense equivalent) against
    QPFunction(duals=True) on the dense equivalent: the same duals and the same gradients of a loss on z, lam, nu."""
    from qpth_b200 import BoxQPFunction, QPFunction
    from qpth_b200.box import dense_equivalent
    from tests.box_util import random_box
    bx = random_box(700 + n, 2, n, e, sides)
    T = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV, requires_grad=True)
    q, p = T(bx["q"]), T(bx["p"])
    A = T(bx["A"]) if e else torch.Tensor().to(DEV).double()
    b = T(bx["b"]) if e else torch.Tensor().to(DEV).double()
    lb = T(bx["lb"]) if bx.get("lb") is not None else None
    ub = T(bx["ub"]) if bx.get("ub") is not None else None
    z, lam, nu = BoxQPFunction(verbose=-1, duals=True)(q, p, A, b, lb, ub)
    rs = np.random.RandomState(9)
    gz, gl, gn = (torch.tensor(rs.randn(*x.shape), dtype=torch.float64, device=DEV) for x in (z, lam, nu))
    ((z * gz).sum() + (lam * gl).sum() + (nu * gn).sum()).backward()
    got = [x.grad.clone() for x in (q, p, A, b, lb, ub) if x is not None and x.requires_grad]
    q2, p2, A2, b2, lb2, ub2 = (None if x is None else x.detach().clone().requires_grad_(x.requires_grad)
                                for x in (q, p, A, b, lb, ub))
    Q, G, h = dense_equivalent(q2, lb2, ub2)
    z2, lam2, nu2 = QPFunction(verbose=-1, duals=True)(Q, p2, G, h, A2, b2)
    assert torch.equal(lam, lam2) and torch.equal(nu, nu2)
    ((z2 * gz).sum() + (lam2 * gl).sum() + (nu2 * gn).sum()).backward()
    want = [x.grad for x in (q2, p2, A2, b2, lb2, ub2) if x is not None and x.requires_grad]
    for g, w in zip(got, want):
        assert torch.allclose(g, w, rtol=1e-10, atol=1e-12)


# ---- end to end: central differences ----------------------------------------------------------------------------------

# Central-difference step: the GPU solves stop at resid < 1e-12, so lam and nu carry ~1e-11 of noise, 1e-6 of the
# difference at this step; the truncation error, O(t^2), is below 4e-7 here (at 1e-4 it reaches 3e-5 for G). Every
# margin of the active set is 0.1, far beyond the step.
T_FD = 1e-5


def _fd_check(fwd, inputs, adj, tol=1e-5):
    """fwd(dict of tensors) -> (z, lam, nu); <grad, V> against central differences of the loss along a random V."""
    x = {k: v.clone().requires_grad_(True) for k, v in inputs.items()}
    outs = fwd(x)
    sum(((o * a).sum() for o, a in zip(outs, adj))).backward()
    rs = np.random.RandomState(4)
    for k, v in inputs.items():
        V = torch.tensor(rs.randn(*v.shape), dtype=v.dtype, device=v.device)
        if k == "Q":
            V = 0.5 * (V + V.transpose(-1, -2))
        with torch.no_grad():
            lo = fwd(dict(inputs, **{k: v - T_FD * V}))
            hi = fwd(dict(inputs, **{k: v + T_FD * V}))
            fd = sum(((h - l) * a).sum() for h, l, a in zip(hi, lo, adj)).item() / (2 * T_FD)
        an = (x[k].grad * V).sum().item()
        assert abs(fd - an) <= tol * max(1.0, abs(an)), (k, fd, an)


def _adj(z, lam, nu):
    rs = np.random.RandomState(12)
    return [torch.tensor(rs.randn(*t.shape), dtype=torch.float64, device=DEV) for t in (z, lam, nu)]


def _implicit_directional(prs, adj, k, V):
    """<grad_k, V> of the loss from the dense implicit derivative at the exact solutions of `prs`: (exact, clamped).
    exact: the unsymmetric Jacobian with the true lam and s (active s = 0, inactive lam = 0), the derivative of the
    solution map itself. clamped: the same with lam and s clamped at 1e-8, which is the backward's d = lam / s of
    qp.py:148 (and dG takes the unclamped lam): the function the kernels are specified to compute."""
    gz, gl, gn = (a.cpu().numpy() for a in adj)
    V = V.cpu().numpy()
    out = []
    for clamp in (False, True):
        tot = 0.0
        for i, pr in enumerate(prs):
            lam, s = (np.maximum(pr["lam"], 1e-8), np.maximum(pr["s"], 1e-8)) if clamp else (pr["lam"], pr["s"])
            g = dm.implicit(pr["Q"], pr["G"], pr["A"], pr["z"], lam, s, pr["nu"], gz[i], gl[i],
                            gn[i] if pr["A"].shape[0] else None)
            g["dG"] = np.outer(g["dlam"], pr["z"]) + np.outer(pr["lam"], g["dx"])
            tot += float(np.sum(g["d" + k] * V[i]))
        out.append(tot)
    return out


def _qp_fd(neq, solution_function):
    """QPFunction(duals=True) (or QPSolutionFunction(duals=True) at the exact solution) on strictly complementary
    batches. Along a random direction V of each input:
      - the central difference of the loss, the GPU forward re-solving the perturbed problems, against the exact implicit
        derivative within 1e-5: the derivation holds end to end;
      - the backward's <grad, V> against the clamped implicit derivative within 1e-7: the kernels compute the specified
        gradient.
    The two references differ by the bias of qpth's 1e-8 clamps (qp.py:148), which a converged point always hits (active
    s ~ 1e-13, inactive lam ~ 1e-13). It grows with |dlam| / lam of the active rows, so an adjoint on lam shows it more
    than one on z alone: on the neq = 3 batch it is 8.2e-5 of a directional derivative of 1.39 (G), 5.8e-5 of 31.7 (h)."""
    from qpth_b200 import QPFunction, QPSolutionFunction
    prs = [dm.complementary_qp(31 + i, 10, 9, neq) for i in range(3)]
    t = {k: torch.tensor(np.stack([pr[k] for pr in prs]), dtype=torch.float64, device=DEV)
         for k in ("Q", "p", "G", "h", "A", "b", "z", "lam", "s", "nu")}
    ins = {k: t[k] for k in ("Q", "p", "G", "h") + (("A", "b") if neq else ())}
    E = torch.Tensor().to(DEV).double()
    f = QPFunction(verbose=-1, duals=True)

    def fwd(x):
        return f(x["Q"], x["p"], x["G"], x["h"], x.get("A", E), x.get("b", E))
    x = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
    if solution_function:
        z, lam, nu = QPSolutionFunction(duals=True)(x["Q"], x["p"], x["G"], x["h"], x.get("A", E), x.get("b", E),
                                                    t["z"], t["lam"], t["s"], t["nu"] if neq else E)
    else:
        z, lam, nu = fwd(x)
        st = f.last_solve()
        assert torch.equal(lam, st.lam) and (neq == 0 or torch.equal(nu, st.nus))
    assert lam.shape == t["lam"].shape and nu.shape == (3, neq)
    assert (z - t["z"]).abs().max() < 1e-9 and (lam - t["lam"]).abs().max() < 1e-8
    adj = _adj(z, lam, nu)
    sum(((o * a).sum() for o, a in zip((z, lam, nu), adj))).backward()
    rs = np.random.RandomState(4)
    for k, v in ins.items():
        V = torch.tensor(rs.randn(*v.shape), dtype=v.dtype, device=v.device)
        if k == "Q":
            V = 0.5 * (V + V.transpose(-1, -2))
        with torch.no_grad():
            lo = fwd(dict(ins, **{k: v - T_FD * V}))
            hi = fwd(dict(ins, **{k: v + T_FD * V}))
            fd = sum(((h - l) * a).sum() for h, l, a in zip(hi, lo, adj)).item() / (2 * T_FD)
        an = (x[k].grad * V).sum().item()
        exact, clamped = _implicit_directional(prs, adj, k, V)
        assert abs(fd - exact) <= 1e-5 * max(1.0, abs(exact)), (k, fd, exact)
        assert abs(an - clamped) <= 1e-7 * max(1.0, abs(clamped)), (k, an, clamped)


@pytest.mark.parametrize("neq", [0, 3])
def test_qpfunction_duals_match_central_differences(neq):
    _qp_fd(neq, solution_function=False)


@pytest.mark.parametrize("neq", [0, 3])
def test_solution_function_duals_match_central_differences(neq):
    """QPSolutionFunction(duals=True) at the exact solution; the central differences re-solve with QPFunction."""
    _qp_fd(neq, solution_function=True)


@pytest.mark.parametrize("shape", [(12, 0, "both"), (10, 3, "lb"), (9, 2, "ub")])
def test_box_duals_match_central_differences(shape):
    from qpth_b200 import BoxQPFunction
    n, e, sides = shape
    prs = [dm.complementary_box(41 + i, n, e, sides) for i in range(3)]
    T = lambda k: torch.tensor(np.stack([pr[k] for pr in prs]), dtype=torch.float64, device=DEV)
    ins = {k: T(k) for k in ("q", "p") + (("A", "b") if e else ()) + (("lb",) if sides != "ub" else ())
           + (("ub",) if sides != "lb" else ())}
    E = torch.Tensor().to(DEV).double()
    f = BoxQPFunction(verbose=-1, duals=True)

    def fwd(x):
        return f(x["q"], x["p"], x.get("A", E), x.get("b", E), x.get("lb"), x.get("ub"))
    z, lam, nu = fwd(ins)
    assert lam.shape == (3, (2 if sides == "both" else 1) * n) and nu.shape == (3, e)
    assert torch.equal(lam, f.last_solve().lam)
    _fd_check(fwd, ins, _adj(z, lam, nu))


def test_equality_only_duals_match_central_differences():
    from qpth_b200 import QPFunction
    rs = np.random.RandomState(21)
    B, n, e = 3, 8, 3
    L = rs.randn(B, n, n)
    ins = {k: torch.tensor(v, dtype=torch.float64, device=DEV) for k, v in
           dict(Q=L @ L.transpose(0, 2, 1) + 0.5 * np.eye(n), p=rs.randn(B, n), A=rs.randn(B, e, n),
                b=rs.randn(B, e)).items()}
    E = torch.Tensor().to(DEV).double()
    f = QPFunction(verbose=-1, duals=True)

    def fwd(x):
        return f(x["Q"], x["p"], E, E, x["A"], x["b"])
    z, lam, nu = fwd(ins)
    assert lam.shape == (B, 0) and nu.shape == (B, e)
    _fd_check(fwd, ins, _adj(z, lam, nu))
