"""The box-QP cluster kernels (csrc/qp_box.cu: one thread block cluster of 2, 4 or 8 CTAs per QP) on the GPU: against the
one-CTA kernels and the numpy model below convergence (forced with QPB200_BOX_CLUSTER), against QPFunction on the dense
equivalent and the real reference where the dense path still runs, and against closed-form projections past it."""
import contextlib
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import box_model as bm, dense_kkt
from oracle.box_wide_cases import WIDE_BOX_CASES
from oracle.projections import project_box, project_capped_simplex
from tests.box_util import GRAD_KEYS, random_box, run_box
from tests.parity import rel_rows
from tests.test_box_cluster_cpu import check_wide_golden, load_wide
from tests.test_box_cpu import _batched
from tests.test_gpu_box import _dense_run

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def cluster_knob(C):
    old = os.environ.get("QPB200_BOX_CLUSTER")
    if C is None:
        os.environ.pop("QPB200_BOX_CLUSTER", None)
    else:
        os.environ["QPB200_BOX_CLUSTER"] = str(C)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("QPB200_BOX_CLUSTER", None)
        else:
            os.environ["QPB200_BOX_CLUSTER"] = old


def _plan(n, e, sides):
    from qpth_b200 import _lib
    return _lib.box_plan_for(n, e, sides != "ub", sides != "lb")


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("box_cluster_child"))
    env = {k: v for k, v in os.environ.items() if k != "QPB200_BOX_CLUSTER"}
    r = subprocess.run([sys.executable, "-m", "tests.box_cluster_child", out], cwd=ROOT, timeout=300,
                       capture_output=True, text=True, env=env)
    return out, "" if r.returncode == 0 else "child exited with %d: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.parametrize("job", ["forced_2", "forced_4", "forced_8", "wide"])
def test_first_runs_in_child_process(child_results, job):
    from tests.gpu_child import load
    out_dir, note = child_results
    rec = load(out_dir, note, job)
    assert np.isfinite(rec["zhat"]).all() and (rec["iters"] >= 1).all()
    if "kkt_dx" in rec:
        assert np.isfinite(rec["kkt_dx"]).all()


# ---- the cluster kernels against the one-CTA kernels and the model, below convergence ----------------------------------
@pytest.mark.parametrize("maxIter", [1, 2, 3, 5, 20])
@pytest.mark.parametrize("sides,e,n", [("lb", 40, 64), ("both", 13, 31), ("ub", 0, 20)])
@pytest.mark.parametrize("C", [2, 4, 8])
def test_cluster_trajectory_matches_one_cta_and_model(C, maxIter, sides, e, n):
    from qpth_b200 import qp as qpmod
    bx = random_box(9 + e, 4, n, e, sides)
    old = qpmod.TRACE
    qpmod.TRACE = True
    try:
        with cluster_knob(None):
            assert _plan(n, e, sides).ok == 1 and _plan(n, e, sides).cl_ctas == 0
            one = run_box(bx, maxIter=maxIter, requires=False)
        with cluster_knob(C):
            assert _plan(n, e, sides).cl_ctas == C
            out = run_box(bx, maxIter=maxIter, requires=False)
    finally:
        qpmod.TRACE = old
    t = _batched(bx, 4)
    for i in range(4):
        tr = []
        sol = bm.solve_one(t["q"][i], t["p"][i], t["A"][i], t["b"][i], None if t["lb"] is None else t["lb"][i],
                           None if t["ub"] is None else t["ub"][i], maxIter=maxIter, stall_tol=qpmod.STALL_TOL,
                           tie=qpmod.BEST_TIE, trace=tr)
        assert out["iters"][i] == sol["iters"] == one["iters"][i]
        tr = np.array(tr)
        for ref in (tr, one["trace"][i, :len(tr)]):
            assert np.allclose(out["trace"][i, :len(tr)], ref, rtol=1e-8, atol=1e-12, equal_nan=True), i
        for ref in (sol["best_resid"], one["best_resid"][i]):
            assert abs(out["best_resid"][i] - ref) <= 1e-8 * abs(ref) + 1e-13
        assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9
        assert rel_rows(out["zhat"][i], one["zhat"][i]).max() < 1e-9


# ---- against the dense path and the real reference -------------------------------------------------------------------
@pytest.mark.parametrize("n,e,sides", [(480, 64, "both"), (450, 100, "lb")])
def test_cluster_matches_dense_qpfunction(n, e, sides):
    """Shapes that took the dense fallback before the cluster kernels existed (the dense path stops near nz = 500 with
    both sides; (600, 64) and (1000, 1) are past it and are checked against the reference's fixture and closed forms)"""
    p = _plan(n, e, sides)
    assert p.ok == 0 and p.cl_ctas >= 2
    bx = random_box(200 + n + e, 3, n, e, sides)
    a, d = run_box(bx), _dense_run(bx)
    assert rel_rows(a["zhat"], d["zhat"]).max() < 1e-8
    for k in GRAD_KEYS:
        if d["grads"][k] is None or np.asarray(d["grads"][k]).size == 0:
            assert a["grads"][k] is None, k
            continue
        assert rel_rows(a["grads"][k], d["grads"][k], floor=1e-4).max() < 1e-6, k


@pytest.mark.parametrize("name", list(WIDE_BOX_CASES))
def test_cluster_matches_reference_golden_and_model(name, golden_dir):
    """the real reference at the tolerances of tests/test_box_cluster_cpu.py (where the model meets the same fixture),
    and the model itself tightly"""
    bx, gold = load_wide(name, golden_dir)
    n, e = bx["q"].shape[-1], bx["A"].shape[-2]
    p = _plan(n, e, "both")
    assert p.ok == 0 and p.cl_ctas >= 2
    out = run_box(bx)
    check_wide_golden(out, gold, bx)
    B = bx["p"].shape[0]
    t = _batched(bx, B)
    mod = bm.qp_solve(t["q"], t["p"], t["A"], t["b"], t["lb"], t["ub"], dl=bx["dl"], stall_tol=1e-6, tie=1.5)
    assert (out["iters"] == mod["iters"]).all()
    assert rel_rows(out["zhat"], mod["zhat"]).max() < 1e-9
    for k in ("dp", "db", "dA"):
        assert rel_rows(out["grads"][k], mod["grads"][k], floor=1e-4).max() < 1e-7, k


# ---- past the dense limit: closed-form projections ---------------------------------------------------------------------
def _closed_form_case(kind, n, B, seed):
    rs = np.random.RandomState(seed)
    v = 3.0 * rs.randn(B, n) / np.sqrt(np.log(n))
    lb, ub = np.zeros(n), np.ones(n)
    k = 0.1 * n
    bx = dict(q=np.ones(n), p=-v, lb=lb, ub=ub, dl=rs.randn(B, n))
    if kind == "simplex":
        bx.update(A=np.ones((1, n)), b=np.full(1, k))
    else:
        bx.update(A=np.zeros((0,)), b=np.zeros((0,)))
    refs = []
    for i in range(B):
        if kind == "simplex":
            z, nu, vjp = project_capped_simplex(bx["q"], bx["p"][i], k, lb, ub)
        else:
            z, vjp = project_box(bx["q"], bx["p"][i], lb, ub)
        refs.append((z, vjp(bx["dl"][i])))
    return bx, refs


@pytest.mark.parametrize("kind,n", [("simplex", 1000), ("simplex", 6000), ("box", 5000)])
def test_cluster_beyond_dense_limit_matches_closed_form(kind, n):
    """z* within 1e-8 of the closed form, or within 10x the model's own distance to it where the interior-point exit
    rules stop earlier (without equality rows the stall rule ends at a residual near 1e-9: z* is then 1e-6 off)"""
    from qpth_b200 import _lib
    from qpth_b200 import qp as qpmod
    e = 1 if kind == "simplex" else 0
    p = _plan(n, e, "both")
    assert p.ok == 0 and p.cl_ctas >= 2
    assert _lib.load().qpb200_plan_init(n, 2 * n, e, ctypes.byref(_lib.Plan())) == 4     # the dense path rejects it
    B = 2
    bx, refs = _closed_form_case(kind, n, B, 17 + n)
    out = run_box(bx)
    t = _batched(bx, B)
    A = np.ones((1, n)) if e else np.zeros((0, n))
    for i in range(B):
        z, g = refs[i]
        sol = bm.solve_one(t["q"][i], t["p"][i], t["A"][i], t["b"][i], t["lb"][i], t["ub"][i],
                           stall_tol=qpmod.STALL_TOL, tie=qpmod.BEST_TIE)
        assert out["iters"][i] == sol["iters"], i
        assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9, i
        assert np.abs(out["zhat"][i] - z).max() <= max(1e-8, 10 * np.abs(sol["x"] - z).max()), i
        d = np.maximum(out["lam"][i], 1e-8) / np.maximum(out["slacks"][i], 1e-8)
        m = d.shape[0]
        mod = bm.kkt_solve(bx["q"], A, True, True, d, bx["dl"][i], np.zeros(m), np.zeros(m), np.zeros(e))
        dx = out["grads"]["dp"][i]
        assert dense_kkt.rel(dx, g["dx"]) <= max(10 * dense_kkt.rel(mod[0], g["dx"]), 1e-10), i


# ---- the stand-alone KKT solve on a cluster plan -------------------------------------------------------------------
@pytest.mark.parametrize("sides,e,n", [("both", 8, 1000), ("lb", 3, 1500)])
def test_cluster_solve_kkt_matches_dense_refined_solve(sides, e, n):
    from qpth_b200 import _lib
    plan = _plan(n, e, sides)
    assert plan.ok == 0 and plan.cl_ctas >= 2
    rs = np.random.RandomState(e + n)
    B = 2
    hl, hu = sides != "ub", sides != "lb"
    m = plan.nineq
    q, A = 0.1 + rs.rand(B, n), rs.randn(B, e, n)
    d = 10.0 ** rs.uniform(-8, 8, (B, m))
    rx, rs_, rz, ry = rs.randn(B, n), rs.randn(B, m), rs.randn(B, m), rs.randn(B, e)
    ins = [torch.tensor(v, dtype=torch.float64, device=DEV).contiguous() for v in (q, A, d, rx, rs_, rz, ry)]
    out = [torch.empty(B, k, dtype=torch.float64, device=DEV) for k in (n, m, m, e)]

    def ptr(t):
        return ctypes.c_void_p(t.data_ptr())
    _lib.check(_lib.load().qpb200_box_solve_kkt(ctypes.byref(plan), B, ptr(ins[0]), n, ptr(ins[1]), e * n,
                                                *(ptr(v) for v in ins[2:]), *(ptr(o) for o in out),
                                                ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in out]
    var, sgn = bm.rows(n, hl, hu)
    G = np.zeros((m, n)); G[np.arange(m), var] = sgn
    for i in range(B):
        ref = dense_kkt.solve(np.diag(q[i]), G, A[i], d[i], rx[i], rs_[i], rz[i], ry[i])
        mod = bm.kkt_solve(q[i], A[i], hl, hu, d[i], rx[i], rs_[i], rz[i], ry[i])
        for k in range(4):
            err, merr = dense_kkt.rel(got[k][i], ref[k]), dense_kkt.rel(mod[k], ref[k])
            assert err <= max(10 * merr, 1e-10 if k != 1 else 1e-8), (i, k, err, merr)


# ---- batch means, the SPD check and verbose output on cluster plans --------------------------------------------------
@pytest.mark.parametrize("sides,e,n,C", [("both", 13, 31, 4), ("both", 1, 1000, None), ("ub", 0, 20, 8)])
def test_cluster_batch_means(sides, e, n, C):
    B = 5
    with cluster_knob(C):
        assert _plan(n, e, sides).cl_ctas >= 2
        for shared in (("q", "A", "b", "lb", "ub"), ("p",)):
            sb = random_box(31 + e, B, n, e, sides, shared=shared)
            full = dict(_batched(sb, B), dl=sb["dl"])
            a, f = run_box(sb), run_box(full)
            for k in GRAD_KEYS:
                if f["grads"][k] is None:
                    continue
                key = dict(zip(GRAD_KEYS, ("q", "p", "A", "b", "lb", "ub")))[k]
                if key in shared:
                    assert a["grads"][k].shape == f["grads"][k].shape[1:], k
                    assert rel_rows(a["grads"][k], f["grads"][k].mean(0)).max() < 1e-12, k
                else:
                    assert rel_rows(a["grads"][k], f["grads"][k]).max() < 1e-12, k


def test_cluster_spd_check_and_verbose_output(capsys):
    bx = random_box(5, 3, 12, 4, "both")
    bad = dict(bx, q=bx["q"].copy())
    bad["q"][1, 3] = -0.5
    with cluster_knob(2):
        assert _plan(12, 4, "both").cl_ctas == 2
        with pytest.raises(RuntimeError, match="Q is not SPD"):
            run_box(bad, requires=False)
        run_box(bad, requires=False, check_Q_spd=False)
        capsys.readouterr()
        run_box(bx, requires=False, verbose=1)
        cl_lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("iter:")]
    with cluster_knob(None):
        run_box(bx, requires=False, verbose=1)
        one_lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("iter:")]
    assert len(cl_lines) == len(one_lines) > 0

    def nums(ln):
        return [float(x) for x in ln.replace(",", " ").split() if x[0].isdigit()]
    for a, b in zip(cl_lines, one_lines):
        assert np.allclose(nums(a), nums(b), rtol=1e-8, atol=1e-12), (a, b)
