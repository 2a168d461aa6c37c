"""The box-QP kernels (csrc/qp_box.cu) at the edges of their plans, on the GPU: every edge entry of tests/box_families.py
(the last bytes of shared memory, neq_pad 120 on one CTA and 128 on a cluster, empty cluster slices, the widest nz, the
largest distributed M, and both sides of the dense / distributed-M switch) below convergence against the numpy model,
in the stand-alone KKT solve and the backward against a refined dense solve of the full KKT system, and against
QPFunction on the dense equivalent and closed-form projections. Every test asserts its entry's plan before it solves.

The refined dense solve (oracle/dense_kkt.py) is O(order^3) in fp64 plus long-double residuals, so the KKT and backward
checks take it up to dense KKT order nz + 2 nineq + neq = 3600. Past that, shapes without equality rows are checked
against the model, whose solve is then elementwise and exact to rounding; (2000, 312, lb) keeps only its trajectory,
batch-free gradient identities and first run."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import box_model as bm, dense_kkt
from oracle.projections import project_box
from tests.box_edges_child import kkt_inputs, run_kkt
from tests.box_families import ENTRIES, check_entry, edges, knob, layout, sides_flags
from tests.box_util import GRAD_KEYS, random_box, run_box
from tests.parity import GTOL, ZTOL, rel_rows
from tests.test_box_cpu import _batched
from tests.test_gpu_box import _dense_run

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_DENSE_ORDER = 3600

EDGES = edges()
BOX_EDGES = [k for k in EDGES if ENTRIES[k]["layout"] != "dense"]
SPLIT_EDGES = [k for k in BOX_EDGES if ENTRIES[k]["layout"] != "one"]
EMPTY_SLICES = ("cl8_empty_9", "cl8_empty_5")

# Entries whose 20-iteration runs end at the rounding floor of the residual, where the summation order decides the exit
# tests, and how far kernels and model were measured apart there (one H100): the most iterations and the largest
# difference of a trace row or the best residual. At (2000, 312, lb) the kernels' primal residual floor is 4.8e-13 and
# passes eps = 1e-12 at iteration 14, the model's is 1.9e-12 and runs on to 16 (trace rows up to 1.9e-12 apart); at
# (1089, 264, lb) the two stop at 13 and 14 for the same reason; the other two differ by up to 6.7e-13. Every other
# entry, and every entry below 20 iterations, is held to the exact iteration count, atol 1e-12 in the trace and 1e-13 in
# the best residual.
AT_FLOOR = {"cl2_full": dict(iters=0, atol=1e-12), "dm4_full": dict(iters=1, atol=1e-12),
            "dm8_full": dict(iters=0, atol=1e-12), "dm8_slice": dict(iters=2, atol=5e-12)}
# The widest entry at which the model ends one iterate short of the kernels: its last step fails on an exact ds = 0
# that the kernels' fused multiply-add does not produce, and its best iterate is then 1.1e-8 from theirs.
MODEL_SHORT = ("cl2_past_one_wide",)


def _order(name):
    n, e, sides = ENTRIES[name]["shape"]
    return n + 2 * n * sum(sides_flags(sides)) + e


def _has_ref(name):
    """a reference KKT solve exists: the refined dense one, or the model's elementwise one without equality rows"""
    return _order(name) <= MAX_DENSE_ORDER or ENTRIES[name]["shape"][1] == 0


def _kkt_ref(q, A, hl, hu, d, rx, rs, rz, ry):
    """(reference, model) solutions of one KKT system; the reference is the refined dense solve where its order allows,
    else (no equality rows) the model itself"""
    n, e = q.shape[0], A.shape[0]
    mod = bm.kkt_solve(q, A, hl, hu, d, rx, rs, rz, ry)
    m = d.shape[0]
    if n + 2 * m + e > MAX_DENSE_ORDER:
        assert e == 0
        return mod, mod
    var, sgn = bm.rows(n, hl, hu)
    G = np.zeros((m, n)); G[np.arange(m), var] = sgn
    return dense_kkt.solve(np.diag(q), G, A if e else None, d, rx, rs, rz, ry if e else None)[:4], mod


def _trace_run(bx, maxIter):
    from qpth_b200 import qp as qpmod
    old = qpmod.TRACE
    qpmod.TRACE = True
    try:
        return run_box(bx, maxIter=maxIter, requires=False)
    finally:
        qpmod.TRACE = old


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("box_edges_child"))
    env = {k: v for k, v in os.environ.items() if k != "QPB200_BOX_CLUSTER"}
    timeout_s = 600
    try:
        r = subprocess.run([sys.executable, "-m", "tests.box_edges_child", out], cwd=ROOT, timeout=timeout_s,
                           capture_output=True, text=True, env=env)
    except subprocess.TimeoutExpired:
        prog = os.path.join(out, "progress.txt")
        last = open(prog).read().split()[-1:] if os.path.exists(prog) else []
        return out, "child killed after %d s (the last entry it started: %s)" % (timeout_s, last[0] if last else "none")
    return out, "" if r.returncode == 0 else "child exited with %d: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.parametrize("name", EDGES)
def test_first_runs_in_child_process(child_results, name):
    from tests.gpu_child import load
    out_dir, note = child_results
    rec = load(out_dir, note, name)
    assert np.isfinite(rec["zhat"]).all() and (rec["iters"] >= 1).all()
    assert np.isfinite(rec["grad_dp"]).all()
    if ENTRIES[name]["layout"] != "dense":
        assert np.isfinite(rec["kkt_dx"]).all()


# ---- below convergence against the model ------------------------------------------------------------------------------
@pytest.mark.parametrize("maxIter", [1, 2, 5, 20])
@pytest.mark.parametrize("name", BOX_EDGES)
def test_edge_trajectory_matches_model(name, maxIter):
    """iterations, trace rows, best residual and z* against the model; the forced empty-slice entries also against the
    same problem on one CTA"""
    from qpth_b200 import qp as qpmod
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    B = 2
    bx = random_box(500 + n + e, B, n, e, sides)
    with knob(ent["knob"]):
        check_entry(name)
        out = _trace_run(bx, maxIter)
    one = None
    if name in EMPTY_SLICES:
        with knob(None):
            assert layout(_plan(n, e, sides)) == "one"
            one = _trace_run(bx, maxIter)
    t = _batched(bx, B)
    for i in range(B):
        tr = []
        sol = bm.solve_one(t["q"][i], t["p"][i], t["A"][i], t["b"][i], None if t["lb"] is None else t["lb"][i],
                           None if t["ub"] is None else t["ub"][i], maxIter=maxIter, stall_tol=qpmod.STALL_TOL,
                           tie=qpmod.BEST_TIE, trace=tr)
        tr = np.array(tr)
        floor = AT_FLOOR.get(name) if maxIter == 20 else None
        if floor is None:
            assert out["iters"][i] == sol["iters"], (i, out["iters"][i], sol["iters"])
            atol, resid_atol = 1e-12, 1e-13
        else:
            assert abs(int(out["iters"][i]) - sol["iters"]) <= floor["iters"], (i, out["iters"][i], sol["iters"])
            atol = resid_atol = floor["atol"]
            tr = tr[:int(out["iters"][i])]                   # the rows both ran
        assert abs(out["best_resid"][i] - sol["best_resid"]) <= 1e-8 * abs(sol["best_resid"]) + resid_atol, i
        refs = [tr] + ([] if one is None else [one["trace"][i, :len(tr)]])
        for ref in refs:
            assert np.allclose(out["trace"][i, :len(tr)], ref, rtol=1e-8, atol=atol, equal_nan=True), i
        assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9
        if one is not None:
            assert out["iters"][i] == one["iters"][i]
            assert abs(out["best_resid"][i] - one["best_resid"][i]) <= 1e-8 * abs(one["best_resid"][i]) + 1e-13
            assert rel_rows(out["zhat"][i], one["zhat"][i]).max() < 1e-9


def _plan(n, e, sides):
    from qpth_b200 import _lib
    return _lib.box_plan_for(n, e, *sides_flags(sides))


# ---- the stand-alone KKT solve ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [k for k in BOX_EDGES if _has_ref(k)])
def test_edge_solve_kkt_matches_refined_solve(name):
    """d = 10^U(-8, 8): error <= max(10x the model's own error, 1e-10), 1e-8 for ds"""
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    hl, hu = sides_flags(sides)
    B = 2
    with knob(ent["knob"]):
        plan = check_entry(name)
        ins = kkt_inputs(plan, B, 7 + n + e)
        got = run_kkt(plan, ins)
    q, A, d, rx, rs, rz, ry = ins
    for i in range(B):
        ref, mod = _kkt_ref(q[i], A[i], hl, hu, d[i], rx[i], rs[i], rz[i], ry[i])
        for k in range(4 if e else 3):
            err, merr = dense_kkt.rel(got[k][i], ref[k]), dense_kkt.rel(mod[k], ref[k])
            assert err <= max(10 * merr, 1e-10 if k != 1 else 1e-8), (i, k, err, merr)


# ---- the backward at the kernels' own solution ------------------------------------------------------------------------
@pytest.mark.parametrize("name", SPLIT_EDGES)
def test_edge_backward_at_own_solution(name):
    """dx, dnu (= -db) and dlam (from dlb / dub) against the reference solve at d = lam / s of the kernels' solution,
    bounded by 10x the model's own error there; dq = dx o z and dA = -db z' + nu dx' from the kernels' own outputs"""
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    hl, hu = sides_flags(sides)
    B = 2
    bx = random_box(600 + n + e, B, n, e, sides)
    with knob(ent["knob"]):
        check_entry(name)
        out = run_box(bx)
    t = _batched(bx, B)
    g = out["grads"]
    for i in range(B):
        x = out["zhat"][i]
        dx = g["dp"][i]
        assert rel_rows(g["dq"][i], dx * x).max() < 1e-13
        if e:
            assert rel_rows(g["dA"][i], np.outer(-g["db"][i], x) + np.outer(out["nus"][i], dx)).max() < 1e-13
        if not _has_ref(name):
            continue
        d = np.maximum(out["lam"][i], 1e-8) / np.maximum(out["slacks"][i], 1e-8)
        m = d.shape[0]
        ref, mod = _kkt_ref(t["q"][i], t["A"][i], hl, hu, d, bx["dl"][i], np.zeros(m), np.zeros(m), np.zeros(e))

        def bound(k):
            return max(10 * dense_kkt.rel(mod[k], ref[k]), 1e-10)
        assert dense_kkt.rel(dx, ref[0]) <= bound(0), (i, dense_kkt.rel(dx, ref[0]), bound(0))
        if e:
            assert dense_kkt.rel(-g["db"][i], ref[3]) <= bound(3), i
        dlam = np.concatenate(([g["dlb"][i]] if hl else []) + ([-g["dub"][i]] if hu else []))
        assert dense_kkt.rel(dlam, ref[2]) <= bound(2), (i, dense_kkt.rel(dlam, ref[2]), bound(2))


# ---- batch means ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cl4_full", "dm2_full"])
def test_edge_batch_means(name):
    """every input passed un-batched: its gradient is the batch mean of the all-batched run (dm2_full has 232 equality
    rows, so k_box_mean_outer runs with more than 128 rows)"""
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    B = 4
    with knob(ent["knob"]):
        check_entry(name)
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


# ---- the dense / distributed-M switch ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["dense_boundary", "dm2_boundary"])
def test_dense_dm_boundary(name):
    """dense order 384 runs the dense kernels, 392 the distributed-M kernels: both against QPFunction on the dense
    equivalent (z* to ZTOL, gradients to GTOL) and the model. The dm side runs the model's arithmetic: iterations exact,
    z* to 1e-9. The dense side factors the whole KKT system: one iteration apart is allowed, z* to ZTOL."""
    from qpth_b200 import qp as qpmod
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    B = 3
    bx = random_box(700 + n, B, n, e, sides)
    with knob(ent["knob"]):
        check_entry(name)
        a, d = run_box(bx), _dense_run(bx)
    assert rel_rows(a["zhat"], d["zhat"]).max() < ZTOL
    for k in GRAD_KEYS:
        if d["grads"][k] is None or np.asarray(d["grads"][k]).size == 0:
            assert a["grads"][k] is None, k
            continue
        assert rel_rows(a["grads"][k], d["grads"][k], floor=1e-4).max() < GTOL, k
    t = _batched(bx, B)
    mod = bm.qp_solve(t["q"], t["p"], t["A"], t["b"], t["lb"], t["ub"], dl=bx["dl"], stall_tol=qpmod.STALL_TOL,
                      tie=qpmod.BEST_TIE)
    if ent["layout"] == "dense":
        assert (np.abs(a["iters"] - mod["iters"]) <= 1).all(), (a["iters"], mod["iters"])
        assert rel_rows(a["zhat"], mod["zhat"]).max() < ZTOL
    else:
        assert (a["iters"] == mod["iters"]).all(), (a["iters"], mod["iters"])
        assert rel_rows(a["zhat"], mod["zhat"]).max() < 1e-9
        assert rel_rows(a["grads"]["dp"], mod["grads"]["dp"], floor=1e-4).max() < GTOL


# ---- the widest nz: closed-form projections --------------------------------------------------------------------------
@pytest.mark.parametrize("name", [k for k in BOX_EDGES if ENTRIES[k]["shape"][1] == 0])
def test_widest_matches_projection(name):
    """q = 1, p = -v: the projection of v onto the box. z* within 1e-8 of the closed form, or within 10x the model's own
    distance to it where the exit rules stop earlier (without equality rows the stall rule ends at a residual near
    1e-9); dx against the closed-form gradient within 10x the model's error at the kernels' d"""
    from qpth_b200 import qp as qpmod
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    hl, hu = sides_flags(sides)
    B = 2
    rs = np.random.RandomState(17 + n)
    v = 3.0 * rs.randn(B, n) / np.sqrt(np.log(n))
    lb, ub = (np.zeros(n) if hl else None), (np.ones(n) if hu else None)
    bx = dict(q=np.ones(n), p=-v, lb=lb, ub=ub, A=np.zeros((0,)), b=np.zeros((0,)), dl=rs.randn(B, n))
    with knob(ent["knob"]):
        check_entry(name)
        out = run_box(bx)
    for i in range(B):
        z, vjp = project_box(bx["q"], bx["p"][i], lb, ub)
        sol = bm.solve_one(bx["q"], bx["p"][i], np.zeros((0, n)), np.zeros(0), lb, ub, stall_tol=qpmod.STALL_TOL,
                           tie=qpmod.BEST_TIE)
        assert out["iters"][i] == sol["iters"], i
        dz_mod, dz_own = np.abs(sol["x"] - z).max(), np.abs(out["zhat"][i] - z).max()
        if name in MODEL_SHORT:     # the closed form decides: the kernels at least as close to it as the model
            assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9 or dz_own <= dz_mod, (i, dz_own, dz_mod)
        else:
            assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9, i
        assert dz_own <= max(1e-8, 10 * dz_mod), i
        d = np.maximum(out["lam"][i], 1e-8) / np.maximum(out["slacks"][i], 1e-8)
        m = d.shape[0]
        mod = bm.kkt_solve(bx["q"], np.zeros((0, n)), hl, hu, d, bx["dl"][i], np.zeros(m), np.zeros(m), None)
        gx = vjp(bx["dl"][i])["dx"]
        assert dense_kkt.rel(out["grads"]["dp"][i], gx) <= max(10 * dense_kkt.rel(mod[0], gx), 1e-10), i


# ---- past the edges ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(7009, 0, "both"), (1000, 353, "lb")])
def test_past_the_edges_raises_before_any_launch(shape):
    """one variable past the widest cl8 slice, one equality row past the largest distributed M: no path takes them, and
    BoxQPFunction raises from the plan, before it allocates or launches anything"""
    from qpth_b200 import BoxQPFunction
    from qpth_b200._lib import QpthB200Error
    n, e, sides = shape
    hl, hu = sides_flags(sides)
    f64 = dict(dtype=torch.float64, device="cuda:0")
    q, p = torch.ones(1, n, **f64), torch.zeros(1, n, **f64)
    A = torch.randn(1, e, n, **f64) if e else torch.empty(0, **f64)
    b = torch.zeros(1, e, **f64) if e else torch.empty(0, **f64)
    lb = torch.zeros(1, n, **f64) if hl else None
    ub = torch.ones(1, n, **f64) if hu else None
    with knob(None):
        with pytest.raises(QpthB200Error, match="too large|TOO_LARGE"):
            BoxQPFunction(verbose=-1)(q, p, A, b, lb, ub)
