"""BoxQPFunction(dense_Q=True) on the GPU: the dense-Q box kernels (csrc/qp_boxq.cu) against the real reference's
fixtures, against QPFunction on the dense equivalent, against the diagonal box kernels, and below convergence against
the numpy model of their arithmetic (oracle/boxq_model.py)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import boxq_model as qm, dense_kkt
from oracle.box_model import rows
from oracle.boxq_cases import BOXQ_CASES
from tests.boxq_util import GRAD_KEYS, KEYS, batched, load_boxq_case, random_boxq, run_boxq, run_dense
from tests.parity import GTOL, ZTOL, rel_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("boxq_child"))
    r = subprocess.run([sys.executable, "-m", "tests.boxq_child", out], cwd=ROOT, timeout=300, capture_output=True,
                       text=True)
    return out, "" if r.returncode == 0 else "child exited with %d: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.parametrize("job", ["portfolio"] + ["first_%s_%d" % (s, e) for s in ("lb", "ub", "both") for e in (0, 13)])
def test_first_runs_in_child_process(child_results, job):
    from tests.gpu_child import load
    out_dir, note = child_results
    rec = load(out_dir, note, job)
    assert np.isfinite(rec["zhat"]).all() and (rec["iters"] >= 1).all()


def _close(a, b, tol, floor=0.0):
    return rel_rows(a, b, floor=floor).max() <= tol


@pytest.mark.parametrize("name", list(BOXQ_CASES))
def test_boxq_matches_reference_golden(name, golden_dir):
    from qpth_b200 import _lib
    bx, gold = load_boxq_case(name, golden_dir)
    n, A = np.asarray(bx["Q"]).shape[-1], np.asarray(bx["A"])
    e = A.shape[-2] if A.ndim >= 2 else 0
    assert _lib.boxq_plan_for(n, e, bx["lb"] is not None, bx["ub"] is not None).ok == 1
    out = run_boxq(bx)
    assert not out["dense"]
    assert rel_rows(out["zhat"], gold["zhat"]).max() <= ZTOL, name
    assert np.allclose(out["lam"], gold["lam"], rtol=1e-6, atol=1e-8 * max(1.0, np.abs(gold["lam"]).max())), name
    if "nus" in gold:
        assert rel_rows(out["nus"], gold["nus"]).max() <= ZTOL, name
    g = out["grads"]
    nlb = n if bx["lb"] is not None else 0
    ref = dict(dQ=gold["dQ"], dp=gold["dp"], dA=gold.get("dA"), db=gold.get("db"),
               dlb=None if bx["lb"] is None else -gold["dh"][..., :nlb],
               dub=None if bx["ub"] is None else gold["dh"][..., nlb:])
    for k in GRAD_KEYS:
        if ref[k] is None:
            continue
        mine = g[k]
        r = ref[k]
        if mine.shape != r.shape:        # an un-batched input's gradient is the batch mean; the side h is batched
            r = r.mean(0)
        assert mine.shape == r.shape, (k, mine.shape, r.shape)
        assert rel_rows(mine, r, floor=1e-4).max() <= GTOL, (name, k, rel_rows(mine, r, floor=1e-4).max())


EQUIV = [(s, e, n, sh, B) for s in ("lb", "ub", "both") for e, n in ((0, 20), (13, 31), (40, 64))
         for sh, B in (((), 5), (("Q", "A", "b", "lb", "ub"), 5))] + [("both", 1, 100, ("A", "b", "lb", "ub"), 600),
                                                                       ("ub", 13, 37, ("p",), 4)]


def _model_outputs(bx, B):
    """z* and the gradients of the numpy model (fp64, the same algorithm; batch means for un-batched inputs)."""
    bb = batched(bx, B)
    out = qm.qp_solve(bb["Q"], bb["p"], bb["A"], bb["b"], bb["lb"], bb["ub"], dl=bx["dl"])
    g = dict(out["grads"])
    for k, key in zip(GRAD_KEYS, KEYS):
        if g[k] is not None and bx[key] is not None and np.asarray(bx[key]).ndim == (3 if k in ("dQ", "dA") else 2) - 1:
            g[k] = g[k].mean(0)
    return out["zhat"], g


@pytest.mark.parametrize("sides,e,n,shared,B", EQUIV)
def test_boxq_matches_dense_qpfunction(sides, e, n, shared, B):
    """z* within 1e-8 and gradients within 1e-6 of QPFunction on the dense equivalent. Where QPFunction's own error
    exceeds that (its reduced KKT matrix has order 2 nz + neq: at nz = 100 with both bounds it was measured up to 3e-10
    in z* from the fp64 model, which the dense-Q kernels match to 1e-16), the model decides, at the same tolerances."""
    bx = random_boxq(100 + e + n, B, n, e, sides, shared)
    a, d = run_boxq(bx), run_dense(bx)
    assert not a["dense"]
    ref = None
    if not _close(a["zhat"], d["zhat"], 1e-8):
        ref = _model_outputs(bx, B)
        assert _close(a["zhat"], ref[0], 1e-8)
        assert rel_rows(a["zhat"], ref[0]).max() < rel_rows(d["zhat"], ref[0]).max()
    for k in GRAD_KEYS:
        if d["grads"][k] is None or np.asarray(d["grads"][k]).size == 0:
            assert a["grads"][k] is None, k
            continue
        assert a["grads"][k].shape == d["grads"][k].shape, k
        if not _close(a["grads"][k], d["grads"][k], 1e-6, floor=1e-4):
            ref = ref or _model_outputs(bx, B)
            assert _close(a["grads"][k], ref[1][k], 1e-6, floor=1e-4), k


@pytest.mark.parametrize("sides,e,n", [("both", 13, 31), ("lb", 0, 20), ("ub", 40, 64)])
def test_diagonal_q_matches_box_kernels(sides, e, n):
    from tests.box_util import random_box, run_box
    bx = random_box(7 + n, 4, n, e, sides)
    bq = dict(bx, Q=np.stack([np.diag(v) for v in bx["q"]]))
    a, d = run_boxq(bq), run_box(bx)
    assert _close(a["zhat"], d["zhat"], 1e-9)
    assert _close(a["grads"]["dp"], d["grads"]["dp"], 1e-7, floor=1e-4)
    dq = np.diagonal(a["grads"]["dQ"], axis1=-2, axis2=-1)
    assert _close(dq, d["grads"]["dq"], 1e-7, floor=1e-4)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if (t is not None and t.numel()) else ctypes.c_void_p(0)


@pytest.mark.parametrize("sides,e,n", [("lb", 40, 64), ("ub", 13, 37), ("both", 0, 25), ("both", 7, 9)])
def test_boxq_solve_kkt_matches_dense_refined_solve(sides, e, n):
    from qpth_b200 import _lib
    rs = np.random.RandomState(e + n)
    B = 6
    hl, hu = sides != "ub", sides != "lb"
    plan = _lib.boxq_plan_for(n, e, hl, hu)
    m = plan.nineq
    bx = random_boxq(e + n, B, n, e if e else 1, sides)
    Q, A = bx["Q"], rs.randn(B, e, n)
    d = 10.0 ** rs.uniform(-8, 8, (B, m))
    rx, rs_, rz, ry = rs.randn(B, n), rs.randn(B, m), rs.randn(B, m), rs.randn(B, e)
    ins = [torch.tensor(v, dtype=torch.float64, device=DEV).contiguous() for v in (Q, A, d, rx, rs_, rz, ry)]
    out = [torch.empty(B, k, dtype=torch.float64, device=DEV) for k in (n, m, m, e)]
    tQ, tA = ins[:2]
    _lib.check(_lib.load().qpb200_boxq_solve_kkt(ctypes.byref(plan), B, _ptr(tQ), n * n, _ptr(tA), e * n,
                                                 *(_ptr(v) for v in ins[2:]), *(_ptr(o) for o in out),
                                                 ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in out]
    var, sgn = rows(n, hl, hu)
    G = np.zeros((m, n)); G[np.arange(m), var] = sgn
    for i in range(B):
        ref = dense_kkt.solve(qm.sym_lower(Q[i]), G, A[i], d[i], rx[i], rs_[i], rz[i], ry[i])
        mod = qm.kkt_solve(Q[i], A[i], hl, hu, d[i], rx[i], rs_[i], rz[i], ry[i])
        for k in range(4 if e else 3):
            err, merr = dense_kkt.rel(got[k][i], ref[k]), dense_kkt.rel(mod[k], ref[k])
            assert err <= max(10 * merr, 1e-10 if k != 1 else 1e-8), (i, k, err, merr)


@pytest.mark.parametrize("maxIter", [1, 2, 3, 5, 20])
@pytest.mark.parametrize("sides,e,n", [("lb", 40, 64), ("both", 13, 31), ("ub", 0, 20)])
def test_boxq_trajectory_matches_model(maxIter, sides, e, n):
    from qpth_b200 import qp as qpmod
    B = 3
    bx = random_boxq(300 + n, B, n, e, sides)
    old = qpmod.TRACE
    qpmod.TRACE = True
    try:
        out = run_boxq(bx, requires=False, maxIter=maxIter)
    finally:
        qpmod.TRACE = old
    bb = batched(bx, B)
    for i in range(B):
        tr = []
        sol = qm.solve_one(bb["Q"][i], bb["p"][i], bb["A"][i], bb["b"][i], None if bb["lb"] is None else bb["lb"][i],
                           None if bb["ub"] is None else bb["ub"][i], maxIter=maxIter,
                           stall_tol=qpmod.STALL_TOL, tie=qpmod.BEST_TIE, trace=tr)
        assert out["iters"][i] == sol["iters"], (i, out["iters"][i], sol["iters"])
        k = sol["iters"]
        np.testing.assert_allclose(out["trace"][i, :k], np.array(tr), rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(out["best_resid"][i], sol["best_resid"], rtol=1e-6, atol=1e-10)
        np.testing.assert_allclose(out["zhat"][i], sol["x"], rtol=1e-6, atol=1e-8)


@pytest.mark.parametrize("shared", [("Q",), ("p",), ("A", "b"), ("lb", "ub"), ("Q", "A", "b", "lb", "ub")])
def test_batch_means_of_unbatched_inputs(shared):
    B, n, e = 6, 23, 5
    bx = random_boxq(55, B, n, e, "both", shared)
    a, d = run_boxq(bx), run_dense(bx)
    for k in GRAD_KEYS:
        assert a["grads"][k].shape == d["grads"][k].shape, k
        assert _close(a["grads"][k], d["grads"][k], 1e-6, floor=1e-4), k


def test_duals_end_to_end_against_central_differences():
    from qpth_b200 import BoxQPFunction
    B, n, e = 2, 9, 2
    bx = random_boxq(77, B, n, e, "both")
    f = BoxQPFunction(verbose=-1, dense_Q=True, duals=True)
    t = {k: torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=DEV) for k in KEYS}
    rs = np.random.RandomState(3)
    wz, wl, wn = (torch.tensor(rs.randn(*s), device=DEV) for s in ((B, n), (B, 2 * n), (B, e)))

    def loss(p):
        z, lam, nu = f(t["Q"], p, t["A"], t["b"], t["lb"], t["ub"])
        return (wz * z).sum() + (wl * lam).sum() + (wn * nu).sum()

    p = t["p"].clone().requires_grad_(True)
    loss(p).backward()
    h = 1e-6
    num = np.zeros((B, n))
    for i in range(B):
        for j in range(n):
            pp, pm = t["p"].clone(), t["p"].clone()
            pp[i, j] += h; pm[i, j] -= h
            num[i, j] = (loss(pp).item() - loss(pm).item()) / (2 * h)
    assert rel_rows(p.grad.cpu().numpy(), num).max() < 1e-5


def _box_G(n):
    var, sgn = rows(n, True, True)
    G = np.zeros((2 * n, n))
    G[np.arange(2 * n), var] = sgn
    return G


def test_jvp_matches_model_and_transposes_the_backward():
    import torch.autograd.forward_ad as fwAD
    from qpth_b200 import BoxQPFunction
    from tests import jvp_models as jm
    from tests.test_gpu_boxq_edges import dlam_floor
    B, n, e = 3, 14, 3
    bx = random_boxq(88, B, n, e, "both")
    rs = np.random.RandomState(8)
    tang = dict(Q=rs.randn(B, n, n), p=rs.randn(B, n), A=rs.randn(B, e, n), b=rs.randn(B, e), lb=rs.randn(B, n),
                ub=rs.randn(B, n))
    f = BoxQPFunction(verbose=-1, dense_Q=True, duals=True)
    prim = {k: torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=DEV) for k in KEYS}
    with fwAD.dual_level():
        duals_in = [fwAD.make_dual(prim[k], torch.tensor(tang[k], device=DEV)) for k in KEYS]
        z, lam, nu = f(*duals_in)
        dz, dlam, dnu = (fwAD.unpack_dual(v).tangent.cpu().numpy() for v in (z, lam, nu))
    st = f.last_solve()
    for i in range(B):
        sol = dict(Q=bx["Q"][i], A=bx["A"][i], var=rows(n, True, True)[0], sgn=rows(n, True, True)[1], nlb=n,
                   x=st.zhat[i].cpu().numpy(), lam=st.lam[i].cpu().numpy(), s=st.slacks[i].cpu().numpy(),
                   nu=st.nus[i].cpu().numpy())
        mz, ml, mn = qm.jvp_one(sol, dQ=tang["Q"][i], dp=tang["p"][i], dA=tang["A"][i], db=tang["b"][i],
                                dlb=tang["lb"][i], dub=tang["ub"][i])
        assert rel_rows(dz[i], mz).max() < 1e-8 and rel_rows(dnu[i], mn).max() < 1e-8
        # dlam = d (G dz + rz) carries d up to 1e8 at the converged point, so kernels and model both round it to ~1e-8:
        # the refined dense solve decides, with the bound of tests/test_gpu_boxq_edges.py
        G = _box_G(n)
        dh = np.concatenate([-tang["lb"][i], tang["ub"][i]])
        ref = jm.jvp_dense(qm.sym_lower(bx["Q"][i]), G, bx["A"][i], sol["x"], sol["lam"], sol["s"], sol["nu"],
                           dict(Q=tang["Q"][i], p=tang["p"][i], h=dh, A=tang["A"][i], b=tang["b"][i]))
        d = np.maximum(sol["lam"], 1e-8) / np.maximum(sol["s"], 1e-8)
        bound = max(10 * dense_kkt.rel(ml, ref[1]), 1e-10, dlam_floor(d, G, ref[0], -dh, ref[1]))
        assert dense_kkt.rel(dlam[i], ref[1]) <= bound, (i, dense_kkt.rel(dlam[i], ref[1]), bound)
    # transpose identity: <g, JVP(t)> = sum_X <grad_X, t_X> for batched inputs
    g = rs.randn(B, n)
    ins = {k: prim[k].clone().requires_grad_(True) for k in KEYS}
    z2 = BoxQPFunction(verbose=-1, dense_Q=True)(*(ins[k] for k in KEYS))
    z2.backward(torch.tensor(g, device=DEV))
    lhs = float((g * dz).sum())
    rhs = sum(float((ins[k].grad.cpu().numpy() * tang[k]).sum()) for k in KEYS)
    assert abs(lhs - rhs) <= 1e-8 * max(1.0, abs(lhs))


def test_gradcheck_forward_ad_tiny():
    from qpth_b200 import BoxQPFunction
    bx = random_boxq(5, 2, 4, 1, "both")
    f = BoxQPFunction(verbose=-1, dense_Q=True)
    ins = [torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=DEV, requires_grad=(k != "Q")) for k in KEYS]
    assert torch.autograd.gradcheck(lambda *a: f(*a), tuple(ins), check_forward_ad=True, check_backward_ad=True,
                                    check_undefined_grad=False, atol=1e-6, rtol=1e-4)


def test_spd_check_and_verbose_output(capsys):
    from qpth_b200 import BoxQPFunction
    from qpth_b200 import qp as qpmod
    bx = random_boxq(9, 2, 10, 2, "both")
    bad = bx["Q"].copy()
    bad[1] -= 2.0 * np.eye(10) * np.abs(np.linalg.eigvalsh(bad[1])).max()
    t = {k: torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=DEV) for k in KEYS}
    old = qpmod.LAZY_CHECKS
    qpmod.LAZY_CHECKS = False
    try:
        with pytest.raises(RuntimeError, match="Q is not SPD."):
            BoxQPFunction(verbose=-1, dense_Q=True)(torch.tensor(bad, device=DEV), *(t[k] for k in KEYS[1:]))
        BoxQPFunction(verbose=-1, dense_Q=True, check_Q_spd=False)(torch.tensor(bad, device=DEV),
                                                                   *(t[k] for k in KEYS[1:]))
        capsys.readouterr()
        BoxQPFunction(verbose=1, dense_Q=True)(*(t[k] for k in KEYS))
        lines = capsys.readouterr().out
        capsys.readouterr()
        _ = run_dense(bx, verbose=1)
        ref = capsys.readouterr().out
    finally:
        qpmod.LAZY_CHECKS = old
    assert lines.count("\n") == ref.count("\n") and lines.count("\n") >= 2


def test_plan_edges_below_convergence_and_fallback():
    from qpth_b200 import _lib
    from tests.test_boxq_cpu import LARGEST
    for (n, e, sides) in LARGEST:
        hl, hu = sides != "ub", sides != "lb"
        assert _lib.boxq_plan_for(n, e, hl, hu).ok == 1
        bx = random_boxq(n + e, 2, n, e, sides)
        out = run_boxq(bx, requires=False, maxIter=2)
        bb = batched(bx, 2)
        for i in range(2):
            sol = qm.solve_one(bb["Q"][i], bb["p"][i], bb["A"][i], bb["b"][i],
                               None if bb["lb"] is None else bb["lb"][i], None if bb["ub"] is None else bb["ub"][i],
                               maxIter=2)
            np.testing.assert_allclose(out["zhat"][i], sol["x"], rtol=1e-6, atol=1e-8)
    n, e, sides = LARGEST[0]
    bx = random_boxq(3, 2, n + 8, e, sides)
    assert _lib.boxq_plan_for(n + 8, e, sides != "ub", sides != "lb").ok == 0
    a, d = run_boxq(bx), run_dense(bx)
    assert a["dense"]
    assert rel_rows(a["zhat"], d["zhat"]).max() < 1e-12
    for k in ("dQ", "dp"):
        assert rel_rows(a["grads"][k], d["grads"][k], floor=1e-4).max() < 1e-12, k
