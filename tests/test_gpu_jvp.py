"""Forward mode (torch.autograd.forward_ad) of QPFunction, QPSolutionFunction, BoxQPFunction and the equality-only path
on the GPU.

- Every family of tests/kernel_families.py (tests/jvp_jobs.py; the `child` families in a child process): the JVP
  against the dense model (tests/jvp_models.jvp_dense) within 1e-10, duals=False gives the same dz bit for bit, and the
  transpose identity sum_b <(g_z, g_lam, g_nu), JVP(t)> = sum_X <grad_X, t_X> against the existing dual backward at
  the same point within 1e-10 relative.
- Every family of tests/reg_families.py at IR_STEPS 0 .. 3: within max(1e-12, 10 x the model's own error) of the
  regularised model and of the refined dense solve (dz and dlam; nu is not unique for dependent rows).
- Every entry of tests/box_families.py: qpb200_box_jvp against the box model and by the transpose identity against
  qpb200_box_backward_duals within 1e-10; the `dense` entries against QPFunction's JVP on the dense equivalent.
- End to end on strictly complementary batches: central differences of z, lam and nu within 1e-5 of the exact implicit
  derivative, and the JVP within 1e-7 of the implicit derivative with qpth's 1e-8 clamps (the function the kernels are
  specified to compute; tests/test_gpu_duals.py explains the two references); gradcheck with check_forward_ad.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from oracle import box_model as bm
from tests import dual_models as dm
from tests import jvp_models as jm
from tests.duals_jobs import dual_point, solution_backward_duals
from tests.jvp_jobs import INPUTS, job_name, jvp_on_gpu, run_child, solution_jvp, tangents
from tests.kernel_families import GRAD_NAMES, cases, family_env, family_plan, ids, seed_for
from tests.parity import rel_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _check_family(fam, shape, got):
    pr = dual_point(fam, shape)
    tan = tangents(pr, seed_for(fam, shape, 6))
    B, neq = pr["z"].shape[0], shape[2]
    refs = []
    for i in range(B):
        ti = {k: (None if tan[k] is None else tan[k][i]) for k in INPUTS}
        refs.append(jm.jvp_dense(pr["Q"][i], pr["G"][i], pr["A"][i], pr["z"][i], pr["lam"][i], pr["s"][i],
                                 pr["nu"][i], ti))
    for j, k in enumerate(("dz", "dlam") + (("dnu",) if neq else ())):
        e = rel_rows(got[k], np.stack([r[j] for r in refs])).max()
        assert e <= 1e-10, (k, e)
    assert np.array_equal(got["dz"], got["z_only"])
    # transpose identity: the JVP against the gradients of g_z'z + g_lam'lam + g_nu'nu at the same point
    lhs = np.sum(pr["dl"] * got["dz"]) + np.sum(pr["glam"] * got["dlam"])
    terms = [np.sum(got["grad_" + n] * tan[k]) for n, k in zip(GRAD_NAMES, INPUTS) if "grad_" + n in got]
    if neq:
        lhs += np.sum(pr["gnu"] * got["dnu"])
    rhs = sum(terms)
    scale = max(abs(lhs), sum(abs(t) for t in terms))
    assert abs(lhs - rhs) <= 1e-10 * scale, (lhs, rhs)


@pytest.mark.parametrize("fam,shape", cases(child=False), ids=ids(cases(child=False)))
def test_family_jvp(fam, shape):
    _check_family(fam, shape, jvp_on_gpu(fam, shape))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("jvp_families"))
    return out_dir, run_child(out_dir)


@pytest.mark.parametrize("fam,shape", cases(child=True), ids=ids(cases(child=True)))
def test_family_jvp_in_child(fam, shape, child_results):
    from tests import gpu_child
    with family_env(fam):
        family_plan(fam, shape)
    _check_family(fam, shape, gpu_child.load(*child_results, job_name(fam, shape)))


def test_unbatched_tangents_carry_the_factor_B():
    """Un-batched inputs: their tangent applies to every QP (the true derivative), while the backward returns the batch
    mean, so the transpose identity carries a factor B for them."""
    B, shape = 37, (100, 100, 8)
    pr = dual_point("pf_one_setup_fast", shape, B)
    bat = dict(Q=False, p=True, G=False, h=False, A=True, b=False)
    for k, v in bat.items():
        if not v:
            pr[k] = np.broadcast_to(pr[k][:1], pr[k].shape).copy()
    tan = tangents(pr, 5, bat)
    dz, dlam, dnu = solution_jvp(pr, tan, batched=bat)
    for i in range(B):
        ti = {k: (tan[k] if not bat[k] else tan[k][i]) for k in INPUTS}
        ref = jm.jvp_dense(pr["Q"][i], pr["G"][i], pr["A"][i], pr["z"][i], pr["lam"][i], pr["s"][i], pr["nu"][i], ti)
        for g, r in zip((dz[i], dlam[i], dnu[i]), ref):
            assert np.abs(g - r).max() <= 1e-10 * np.abs(r).max()
    grads = solution_backward_duals(pr, "all", bat)
    lhs = np.sum(pr["dl"] * dz) + np.sum(pr["glam"] * dlam) + np.sum(pr["gnu"] * dnu)
    terms = [np.sum(grads[n] * tan[k]) * (1 if bat[k] else B) for n, k in zip(GRAD_NAMES, INPUTS)]
    assert abs(lhs - sum(terms)) <= 1e-10 * sum(abs(t) for t in terms)


# ---- the regularised mode ------------------------------------------------------------------------------------------------

def _reg_cases():
    from tests.reg_families import CASES
    return CASES


@pytest.mark.parametrize("case", _reg_cases(), ids=["%s-%s" % c for c in _reg_cases()])
def test_reg_family_jvp(case, monkeypatch):
    from oracle import kernel_model as km
    from qpth_b200 import KKTSolvers, kkt
    from tests.reg_families import family_plan as reg_plan, problem
    from tests.test_gpu_reg_families import B, _point, _rel
    fam, kind = case
    probs = [problem(fam, kind, s) for s in range(B)]
    reg_plan(fam, probs[0])
    e = probs[0][4].shape[0]
    pts = [_point(c, i) for i, c in enumerate(probs)]
    pr = dict(Q=np.stack([c[0] for c in probs]), p=np.stack([c[1] for c in probs]), G=np.stack([c[2] for c in probs]),
              h=np.stack([c[3] for c in probs]), A=np.stack([c[4] for c in probs]), b=np.stack([c[5] for c in probs]),
              z=np.stack([pt[0] for pt in pts]), lam=np.stack([pt[1] for pt in pts]), s=np.stack([pt[2] for pt in pts]),
              nu=np.stack([pt[3] for pt in pts]))
    tan = tangents(pr, 91)
    dense = []
    for i in range(B):
        ti = {k: (None if tan[k] is None else tan[k][i]) for k in INPUTS}
        dense.append(jm.jvp_dense(pr["Q"][i], pr["G"][i], pr["A"][i], pr["z"][i], pr["lam"][i], pr["s"][i],
                                  pr["nu"][i], ti)[:2])             # nu. is not unique for dependent rows
    for steps in range(4):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        got = solution_jvp(pr, tan, kkt_solver=KKTSolvers.IR_UNOPT)
        for i in range(B):
            ti = {k: (None if tan[k] is None else tan[k][i]) for k in INPUTS}
            st = dict(x=pr["z"][i], lam=pr["lam"][i], s=pr["s"][i], nu=pr["nu"][i] if e else None,
                      f=km.setup(pr["Q"][i], pr["G"][i], pr["A"][i], kkt.IR_EPS), reg=kkt.IR_EPS, steps=steps,
                      Q=pr["Q"][i], G=pr["G"][i], A=pr["A"][i])
            model = jm.jvp_reg(st, ti)
            model_err = max(_rel(model[j], dense[i][j]) for j in range(2))
            tol = max(1e-12, 10 * model_err)
            for j in range(3 if e else 2):
                assert _rel(got[j][i], model[j]) <= tol, (steps, i, j, _rel(got[j][i], model[j]), tol)
            for j in range(2):
                assert _rel(got[j][i], dense[i][j]) <= tol, (steps, i, j, _rel(got[j][i], dense[i][j]), tol)


# ---- the box QP ----------------------------------------------------------------------------------------------------------

def _box_names():
    from tests.box_families import ENTRIES
    return list(ENTRIES)


BOX_INPUTS = ("q", "p", "A", "b", "lb", "ub")


def _box_jvp(plan, pt, tan):
    """qpb200_box_jvp at the point: (dz, dlam, dnu)."""
    from qpth_b200 import _lib
    lib = _lib.load()
    B, n = pt["z"].shape
    e, m = plan.neq, plan.nineq
    T = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if (t is not None and t.numel()) else ctypes.c_void_p(0)
    ins = {k: T(pt[k]) for k in ("q", "A", "z", "nu", "lam", "s")}
    tt = {k: (None if tan.get(k) is None else T(tan[k])) for k in BOX_INPUTS}
    per = dict(q=n, p=n, A=e * n, b=e, lb=n, ub=n)
    args = []
    for k in BOX_INPUTS:
        args += [P(tt[k]), per[k] if tt[k] is not None else 0]
    f64 = dict(dtype=torch.float64, device=DEV)
    rhs = torch.empty(B * (n + m + e), **f64)
    dz, dlam, dnu = torch.empty(B, n, **f64), torch.empty(B, m, **f64), torch.empty(B, e, **f64)
    _lib.check(lib.qpb200_box_jvp(ctypes.byref(plan), B, P(ins["q"]), n, P(ins["A"]), e * n, *args, P(ins["z"]),
                                  P(ins["lam"]), P(ins["s"]), P(ins["nu"]), P(rhs), P(dz), P(dlam), P(dnu),
                                  ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    return dz.cpu().numpy(), dlam.cpu().numpy(), dnu.cpu().numpy()


@pytest.mark.parametrize("name", _box_names())
def test_box_entry_jvp(name):
    from tests.box_families import ENTRIES, check_entry, knob, layout, sides_flags
    from tests.test_gpu_duals import _box_backward, _box_point
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    lb, ub = sides_flags(sides)
    with knob(ent["knob"]):
        plan = check_entry(name)
        if layout(plan) == "dense":
            _check_box_dense(n, e, sides)
            return
        B = 2
        pt = _box_point(plan, B, 800 + n + e)
        rs = np.random.RandomState(n + e)
        tan = dict(q=rs.randn(B, n), p=rs.randn(B, n), A=rs.randn(B, e, n) if e else None, b=rs.randn(B, e) if e else None,
                   lb=rs.randn(B, n) if lb else None, ub=rs.randn(B, n) if ub else None)
        got = _box_jvp(plan, pt, tan)
        gnu = pt["gnu"] if e else None
        grads = _box_backward(plan, pt, pt["dl"], pt["glam"], gnu)
    nlb = n if lb else 0
    for i in range(B):
        ti = {k: (None if tan[k] is None else tan[k][i]) for k in BOX_INPUTS}
        ref = jm.jvp_box(pt["q"][i], pt["A"][i], pt["z"][i], pt["lam"][i], pt["s"][i], pt["nu"][i], nlb, ub, ti)
        for j in range(3 if e else 2):
            err = np.abs(got[j][i] - ref[j]).max() / max(np.abs(ref[j]).max(), 1e-300)
            assert err <= 1e-10, (j, i, err)
    # transpose identity with qpb200_box_backward_duals: (dx, dlam, dnu, dq, dp, dlb, dub, dA, db)
    lhs = np.sum(pt["dl"] * got[0]) + np.sum(pt["glam"] * got[1]) + (np.sum(gnu * got[2]) if e else 0.0)
    gx = dict(q=grads[3], p=grads[4], lb=grads[5], ub=grads[6], A=grads[7], b=grads[8])
    terms = [np.sum(gx[k] * tan[k]) for k in BOX_INPUTS if tan[k] is not None]
    assert abs(lhs - sum(terms)) <= 1e-10 * max(abs(lhs), sum(abs(t) for t in terms)), (lhs, sum(terms))


def _check_box_dense(n, e, sides):
    """BoxQPFunction's JVP on a shape no box kernel takes (the dense kernels on the dense equivalent) against
    QPFunction's JVP on the dense equivalent with the mapped tangents."""
    from qpth_b200 import BoxQPFunction, QPFunction
    from qpth_b200.box import dense_equivalent
    from tests.box_util import random_box
    bx = random_box(700 + n, 2, n, e, sides)
    T = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV)
    rs = np.random.RandomState(3)
    ins = dict(q=T(bx["q"]), p=T(bx["p"]), A=T(bx["A"]) if e else None, b=T(bx["b"]) if e else None,
               lb=T(bx["lb"]) if bx.get("lb") is not None else None, ub=T(bx["ub"]) if bx.get("ub") is not None else None)
    tan = {k: (None if v is None else T(rs.randn(*v.shape))) for k, v in ins.items()}
    E = torch.Tensor().to(DEV).double()
    with fwAD.dual_level():
        x = {k: (None if v is None else fwAD.make_dual(v, tan[k])) for k, v in ins.items()}
        outs = BoxQPFunction(verbose=-1, duals=True)(x["q"], x["p"], x["A"] if e else E, x["b"] if e else E, x["lb"],
                                                     x["ub"])
        got = [fwAD.unpack_dual(o).tangent for o in outs]
        Q, G, h = dense_equivalent(x["q"], x["lb"], x["ub"])
        outs2 = QPFunction(verbose=-1, duals=True)(Q, x["p"], G.detach(), h, x["A"] if e else E, x["b"] if e else E)
        want = [fwAD.unpack_dual(o).tangent for o in outs2]
    for g, w in zip(got, want):
        assert torch.allclose(g, w, rtol=1e-10, atol=1e-12)


# ---- end to end ------------------------------------------------------------------------------------------------------------

T_FD = 1e-5          # the step of tests/test_gpu_duals.py (its T_FD note applies here)


def _fd_vs_jvp(fwd, ins, exact, clamped, jvp_tol=1e-7):
    """fwd(dict) -> outputs. For a random tangent of every input at once: central differences against `exact` within
    1e-5, the JVP through forward_ad against `clamped` within jvp_tol (both lists of arrays per output)."""
    rs = np.random.RandomState(4)
    tan = {k: torch.tensor(rs.randn(*v.shape), dtype=v.dtype, device=v.device) for k, v in ins.items()}
    if "Q" in tan:          # the forward reads one triangle of Q (chol(Q)): differences need a symmetric direction
        tan["Q"] = 0.5 * (tan["Q"] + tan["Q"].transpose(-1, -2))
    with fwAD.dual_level():
        outs = fwd({k: fwAD.make_dual(v, tan[k]) for k, v in ins.items()})
        outs = outs if isinstance(outs, tuple) else (outs,)
        jv = [fwAD.unpack_dual(o).tangent for o in outs]
    assert all(t is not None for t in jv)
    with torch.no_grad():
        hi = fwd({k: v + T_FD * tan[k] for k, v in ins.items()})
        lo = fwd({k: v - T_FD * tan[k] for k, v in ins.items()})
        hi, lo = (o if isinstance(o, tuple) else (o,) for o in (hi, lo))
    tn = {k: v.cpu().numpy() for k, v in tan.items()}
    ex, cl = exact(tn), clamped(tn)
    for j, (h, l, g) in enumerate(zip(hi, lo, jv)):
        if h.numel() == 0:                  # lam without inequality rows, nu without equality rows
            assert g.shape == h.shape
            continue
        fd = ((h - l) / (2 * T_FD)).cpu().numpy()
        scale = max(1.0, np.abs(ex[j]).max()) if ex[j].size else 1.0
        assert np.abs(fd - ex[j]).max() <= 1e-5 * scale, (j, np.abs(fd - ex[j]).max())
        assert np.abs(g.cpu().numpy() - cl[j]).max() <= jvp_tol * scale, (j, np.abs(g.cpu().numpy() - cl[j]).max())
    return tan, jv


def _implicit_all(prs, neq, duals, clamp):
    def f(tn):
        outs = [[], [], []]
        for i, pr in enumerate(prs):
            ti = {k: tn[k][i] for k in tn}
            dz, dl, dn = jm.implicit_jvp(pr["Q"], pr["G"], pr["A"], pr["z"], pr["lam"], pr["s"], pr["nu"], ti, clamp)
            outs[0].append(dz)
            outs[1].append(dl)
            outs[2].append(dn if neq else np.zeros(0))
        res = [np.stack(o) for o in outs]
        return res if duals else res[:1]
    return f


@pytest.mark.parametrize("duals", [False, True])
@pytest.mark.parametrize("neq", [0, 3])
@pytest.mark.parametrize("solver", ["LU_PARTIAL", "IR_UNOPT", "solution"])
def test_qpfunction_jvp_matches_central_differences(solver, neq, duals):
    from qpth_b200 import KKTSolvers, QPFunction, QPSolutionFunction
    prs = [dm.complementary_qp(31 + i, 10, 9, neq) for i in range(3)]
    t = {k: torch.tensor(np.stack([pr[k] for pr in prs]), dtype=torch.float64, device=DEV)
         for k in ("Q", "p", "G", "h", "A", "b", "z", "lam", "s", "nu")}
    ins = {k: t[k] for k in ("Q", "p", "G", "h") + (("A", "b") if neq else ())}
    E = torch.Tensor().to(DEV).double()
    kkt = KKTSolvers.IR_UNOPT if solver == "IR_UNOPT" else KKTSolvers.LU_PARTIAL
    f = QPFunction(verbose=-1, duals=duals, kkt_solver=kkt)
    if solver == "solution":
        g = QPSolutionFunction(duals=duals)
        fwd_jvp = lambda x: g(x["Q"], x["p"], x["G"], x["h"], x.get("A", E), x.get("b", E), t["z"], t["lam"], t["s"],
                              t["nu"] if neq else E)
    else:
        fwd_jvp = lambda x: f(x["Q"], x["p"], x["G"], x["h"], x.get("A", E), x.get("b", E))
    solve = QPFunction(verbose=-1, duals=duals)

    def fwd(x):
        # the JVP from the function under test; central differences always re-solve with QPFunction
        if any(fwAD.unpack_dual(v).tangent is not None for v in x.values()):
            return fwd_jvp(x)
        return solve(x["Q"], x["p"], x["G"], x["h"], x.get("A", E), x.get("b", E))
    _fd_vs_jvp(fwd, ins, _implicit_all(prs, neq, duals, False), _implicit_all(prs, neq, duals, True),
               jvp_tol=1e-6 if solver == "IR_UNOPT" else 1e-7)


@pytest.mark.parametrize("duals", [False, True])
@pytest.mark.parametrize("shape", [(12, 0, "both"), (10, 3, "lb"), (9, 2, "ub")])
def test_box_jvp_matches_central_differences(shape, duals):
    from qpth_b200 import BoxQPFunction
    n, e, sides = shape
    prs = [dm.complementary_box(41 + i, n, e, sides) for i in range(3)]
    T = lambda k: torch.tensor(np.stack([pr[k] for pr in prs]), dtype=torch.float64, device=DEV)
    keys = ("q", "p") + (("A", "b") if e else ()) + (("lb",) if sides != "ub" else ()) + (("ub",) if sides != "lb" else ())
    ins = {k: T(k) for k in keys}
    E = torch.Tensor().to(DEV).double()
    f = BoxQPFunction(verbose=-1, duals=duals)

    def fwd(x):
        return f(x["q"], x["p"], x.get("A", E), x.get("b", E), x.get("lb"), x.get("ub"))
    st_outs = fwd(ins)
    st = f.last_solve()
    nlb = n if sides != "ub" else 0

    def refs(clamp):
        def r(tn):
            outs = [[], [], []]
            for i, pr in enumerate(prs):
                Q, G, _ = bm.dense(pr["q"], pr["lb"], pr["ub"])
                ti = dict(Q=np.diag(tn["q"][i]), p=tn["p"][i], A=tn["A"][i] if e else None, b=tn["b"][i] if e else None)
                hs = ([-tn["lb"][i]] if nlb else []) + ([tn["ub"][i]] if sides != "lb" else [])
                ti["h"] = np.concatenate(hs)
                lam = st.lam[i].cpu().numpy()
                s = st.slacks[i].cpu().numpy()
                act = lam > s
                lam, s = np.where(act, lam, 0.0), np.where(act, 0.0, s)      # the exact complementary pair
                nu = st.nus[i].cpu().numpy() if e else np.zeros(0)
                dz, dl, dn = jm.implicit_jvp(Q, G, pr["A"], pr["z"], lam, s, nu, ti, clamp)
                outs[0].append(dz)
                outs[1].append(dl)
                outs[2].append(dn if e else np.zeros(0))
            res = [np.stack(o) for o in outs]
            return res if duals else res[:1]
        return r
    assert st_outs is not None
    _fd_vs_jvp(fwd, ins, refs(False), refs(True))


@pytest.mark.parametrize("duals", [False, True])
def test_equality_only_jvp_matches_central_differences(duals):
    from qpth_b200 import QPFunction
    rs = np.random.RandomState(21)
    B, n, e = 3, 8, 3
    L = rs.randn(B, n, n)
    ins = {k: torch.tensor(v, dtype=torch.float64, device=DEV) for k, v in
           dict(Q=L @ L.transpose(0, 2, 1) + 0.5 * np.eye(n), p=rs.randn(B, n), A=rs.randn(B, e, n),
                b=rs.randn(B, e)).items()}
    E = torch.Tensor().to(DEV).double()
    f = QPFunction(verbose=-1, duals=duals)

    def fwd(x):
        return f(x["Q"], x["p"], E, E, x["A"], x["b"])
    z0 = fwd(ins)
    z0 = z0[0] if duals else z0
    nu0 = f(ins["Q"], ins["p"], E, E, ins["A"], ins["b"])[2] if duals else None

    def ref(tn):
        outs = [[], [], []]
        Qn, An = ins["Q"].cpu().numpy(), ins["A"].cpu().numpy()
        for i in range(B):
            nu = nu0[i].cpu().numpy() if duals else _nu(Qn[i], ins["p"][i].cpu().numpy(), An[i], ins["b"][i].cpu().numpy())
            K = np.block([[Qn[i], An[i].T], [An[i], np.zeros((e, e))]])
            z = z0[i].cpu().numpy()
            rx = 0.5 * (tn["Q"][i] + tn["Q"][i].T) @ z + tn["p"][i] + tn["A"][i].T @ nu
            ry = tn["A"][i] @ z - tn["b"][i]
            w = np.linalg.solve(K, -np.concatenate([rx, ry]))
            outs[0].append(w[:n]); outs[1].append(np.zeros(0)); outs[2].append(w[n:])
        res = [np.stack(o) for o in outs]
        return res if duals else res[:1]
    _fd_vs_jvp(fwd, ins, ref, ref, jvp_tol=1e-9)


def _nu(Q, p, A, b):
    n, e = Q.shape[0], A.shape[0]
    K = np.block([[Q, A.T], [A, np.zeros((e, e))]])
    return np.linalg.solve(K, np.concatenate([-p, b]))[n:]


def test_gradcheck_forward_ad():
    """torch.autograd.gradcheck in forward mode on a small batched problem, duals=True: every output's Jacobian from
    the JVP against finite differences of the forward. Q stays fixed: the forward reads only chol(Q), one triangle,
    while the JVP takes the symmetrised dQ (checked against symmetric directions above)."""
    from qpth_b200 import QPFunction
    prs = [dm.complementary_qp(61 + i, 6, 5, 2) for i in range(2)]
    Q = torch.tensor(np.stack([pr["Q"] for pr in prs]), dtype=torch.float64, device=DEV)
    ins = tuple(torch.tensor(np.stack([pr[k] for pr in prs]), dtype=torch.float64, device=DEV, requires_grad=True)
                for k in ("p", "G", "h", "A", "b"))
    f = QPFunction(verbose=-1, duals=True)
    # tolerance: the 1e-8 clamps bias the JVP of lam by up to ~1e-4 against the exact derivative (test_gpu_duals.py)
    assert torch.autograd.gradcheck(lambda *x: f(Q, *x), ins, eps=1e-6, atol=2e-4, rtol=1e-3, check_forward_ad=True,
                                    check_backward_ad=False, check_batched_forward_grad=False)
