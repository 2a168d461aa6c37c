"""The distributed-M box kernels (csrc/qp_box.cu k_box_*_dm: neq_pad > 128, M spread over a cluster of 2, 4 or 8 CTAs)
on the GPU: against the numpy model below convergence (forced with QPB200_BOX_CLUSTER on small shapes), against a
refined dense KKT solve, against QPFunction on the dense equivalent (the 9x9 sudoku layer and a mid-size shape), and
against the real reference's sudoku fixtures."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import box_model as bm, dense_kkt
from oracle.box_sudoku_cases import SUDOKU_BOX_CASES, sudoku9_init_problem
from tests.box_util import GRAD_KEYS, random_box, run_box
from tests.parity import GTOL, ZTOL, rel_rows
from tests.test_box_cpu import _batched
from tests.test_box_dm_cpu import SUDOKU_GTOL, SUDOKU_ZTOL, check_sudoku_golden, load_sudoku
from tests.test_gpu_box import _dense_run
from tests.test_gpu_box_cluster import cluster_knob

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = [("ub", 130, 150), ("both", 136, 160), ("lb", 180, 200)]


def _plan(n, e, sides):
    from qpth_b200 import _lib
    return _lib.box_plan_for(n, e, sides != "ub", sides != "lb")


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("box_dm_child"))
    env = {k: v for k, v in os.environ.items() if k != "QPB200_BOX_CLUSTER"}
    r = subprocess.run([sys.executable, "-m", "tests.box_dm_child", out], cwd=ROOT, timeout=300,
                       capture_output=True, text=True, env=env)
    return out, "" if r.returncode == 0 else "child exited with %d: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.parametrize("job", ["forced_2", "forced_4", "forced_8", "sudoku9"])
def test_first_runs_in_child_process(child_results, job):
    from tests.gpu_child import load
    out_dir, note = child_results
    rec = load(out_dir, note, job)
    assert np.isfinite(rec["zhat"]).all() and (rec["iters"] >= 1).all()
    if "kkt_dx" in rec:
        assert np.isfinite(rec["kkt_dx"]).all()


# ---- forced onto small shapes: the model below convergence ------------------------------------------------------------
@pytest.mark.parametrize("maxIter", [1, 2, 3, 5, 20])
@pytest.mark.parametrize("sides,e,n", SMALL)
@pytest.mark.parametrize("C", [2, 4, 8])
def test_dm_trajectory_matches_model(C, maxIter, sides, e, n):
    from qpth_b200 import qp as qpmod
    bx = random_box(5 + e, 2, n, e, sides)
    old = qpmod.TRACE
    qpmod.TRACE = True
    try:
        with cluster_knob(C):
            assert _plan(n, e, sides).cl_ctas == C
            out = run_box(bx, maxIter=maxIter, requires=False)
    finally:
        qpmod.TRACE = old
    t = _batched(bx, 2)
    for i in range(2):
        tr = []
        sol = bm.solve_one(t["q"][i], t["p"][i], t["A"][i], t["b"][i], None if t["lb"] is None else t["lb"][i],
                           None if t["ub"] is None else t["ub"][i], maxIter=maxIter, stall_tol=qpmod.STALL_TOL,
                           tie=qpmod.BEST_TIE, trace=tr)
        assert out["iters"][i] == sol["iters"]
        tr = np.array(tr)
        assert np.allclose(out["trace"][i, :len(tr)], tr, rtol=1e-8, atol=1e-12, equal_nan=True), i
        assert abs(out["best_resid"][i] - sol["best_resid"]) <= 1e-8 * abs(sol["best_resid"]) + 1e-13
        assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9


@pytest.mark.parametrize("sides,e,n", SMALL)
@pytest.mark.parametrize("C", [2, 4, 8])
def test_dm_solve_kkt_matches_dense_refined_solve(C, sides, e, n):
    from qpth_b200 import _lib
    with cluster_knob(C):
        plan = _plan(n, e, sides)
        assert plan.cl_ctas == C and plan.neq_pad > 128
        rs = np.random.RandomState(e + n + C)
        B = 2
        hl, hu = sides != "ub", sides != "lb"
        m = plan.nineq
        q, A = 0.1 + rs.rand(B, n), rs.randn(B, e, n)
        d = 10.0 ** rs.uniform(-8, 8, (B, m))
        rx, rs_, rz, ry = rs.randn(B, n), rs.randn(B, m), rs.randn(B, m), rs.randn(B, e)
        ins = [torch.tensor(v, dtype=torch.float64, device=DEV).contiguous() for v in (q, A, d, rx, rs_, rz, ry)]
        out = [torch.empty(B, k, dtype=torch.float64, device=DEV) for k in (n, m, m, e)]

        def ptr(v):
            return ctypes.c_void_p(v.data_ptr())
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


# ---- chosen by the plan: against QPFunction on the dense equivalent ---------------------------------------------------
def _mid_problem():
    """nz = 600, neq = 249, lb only (dense order 856): random shared A, batched p"""
    bx = random_box(77, 3, 600, 249, "lb", shared=("q", "A", "b", "lb"))
    return bx


@pytest.mark.parametrize("name", ["sudoku9_init", "mid"])
def test_dm_matches_dense_qpfunction(name):
    """z* to ZTOL and every gradient to GTOL (floored as tests/parity.py does), including the batch means of the shared
    A and b"""
    bx = sudoku9_init_problem() if name == "sudoku9_init" else _mid_problem()
    n, e = np.asarray(bx["q"]).shape[-1], np.asarray(bx["A"]).shape[-2]
    with cluster_knob(None):
        p = _plan(n, e, "lb")
        assert p.ok == 0 and p.cl_ctas in (2, 4, 8) and p.neq_pad > 128
        a, d = run_box(bx), _dense_run(bx)
    assert rel_rows(a["zhat"], d["zhat"]).max() < ZTOL
    for k in GRAD_KEYS:
        if d["grads"][k] is None or np.asarray(d["grads"][k]).size == 0:
            assert a["grads"][k] is None, k
            continue
        assert a["grads"][k].shape == np.asarray(d["grads"][k]).shape, k
        assert rel_rows(a["grads"][k], d["grads"][k], floor=1e-4).max() < GTOL, k


@pytest.mark.parametrize("name", list(SUDOKU_BOX_CASES))
def test_dm_matches_sudoku_reference_golden_and_model(name, golden_dir):
    bx, gold = load_sudoku(name, golden_dir)
    n, e = bx["q"].shape[-1], bx["A"].shape[-2]
    with cluster_knob(None):
        assert _plan(n, e, "lb").cl_ctas in (2, 4, 8)
        out = run_box(bx)
    check_sudoku_golden(out, gold, bx, SUDOKU_ZTOL, SUDOKU_GTOL)
    # At convergence the stall rule may fire one iteration apart from the model's (the last bits of the factor of an
    # order-249 M differ); test_dm_trajectory_matches_model pins the iterates below convergence.
    B = bx["p"].shape[0]
    t = _batched(bx, B)
    mod = bm.qp_solve(t["q"], t["p"], t["A"], t["b"], t["lb"], t["ub"], dl=bx["dl"], stall_tol=1e-6, tie=1.5)
    assert (np.abs(out["iters"] - mod["iters"]) <= 1).all()
    assert rel_rows(out["zhat"], mod["zhat"]).max() < SUDOKU_ZTOL
    assert rel_rows(out["grads"]["dp"], mod["grads"]["dp"], floor=1e-4).max() < SUDOKU_GTOL
