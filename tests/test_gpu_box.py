"""BoxQPFunction on the GPU: the box kernels (csrc/qp_box.cu) against the real reference's fixtures, against QPFunction
on the dense equivalent, and below convergence against the numpy model of their arithmetic (oracle/box_model.py)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import box_model as bm, dense_kkt
from oracle.box_cases import BOX_CASES, map_dense_grads
from tests.box_util import BOX_KEYS, GRAD_KEYS, load_box_case, random_box, run_box
from tests.parity import rel_rows
from tests.test_box_cpu import _batched, check_box_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("box_child"))
    r = subprocess.run([sys.executable, "-m", "tests.box_child", out], cwd=ROOT, timeout=300, capture_output=True,
                       text=True)
    return out, "" if r.returncode == 0 else "child exited with %d: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.parametrize("job", ["sudoku"] + ["first_%s_%d" % (s, e) for s in ("lb", "ub", "both") for e in (0, 13)])
def test_first_runs_in_child_process(child_results, job):
    from tests.gpu_child import load
    out_dir, note = child_results
    rec = load(out_dir, note, job)
    assert np.isfinite(rec["zhat"]).all() and (rec["iters"] >= 1).all()


@pytest.mark.parametrize("name", list(BOX_CASES))
def test_box_matches_reference_golden(name, golden_dir):
    from qpth_b200 import _lib
    bx, gold = load_box_case(name, golden_dir)
    n, e = np.asarray(bx["q"]).shape[-1], np.asarray(bx["A"]).shape[-2] if np.asarray(bx["A"]).size else 0
    assert _lib.box_plan_for(n, e, bx["lb"] is not None, bx["ub"] is not None).ok == 1
    check_box_golden(run_box(bx), gold, bx, name)


def _dense_run(bx, **opts):
    from qpth_b200 import QPFunction
    from qpth_b200.box import dense_equivalent
    t = {k: (None if bx[k] is None else torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=DEV))
         for k in BOX_KEYS}
    Q, G, h = dense_equivalent(t["q"], t["lb"], t["ub"])
    ins = dict(Q=Q, p=t["p"], G=G, h=h, A=t["A"], b=t["b"])
    for v in ins.values():
        if v.numel():
            v.requires_grad_(True)
    f = QPFunction(**dict(dict(verbose=-1), **opts))
    z = f(*(ins[k] for k in ("Q", "p", "G", "h", "A", "b")))
    z.backward(torch.tensor(np.asarray(bx["dl"]), dtype=torch.float64, device=DEV))
    g = tuple(None if (v.grad is None) else v.grad.cpu().numpy() for v in ins.values())
    st = f.last_solve()
    return dict(zhat=z.detach().cpu().numpy(), iters=st.iters.cpu().numpy(), grads=map_dense_grads(g, bx))


EQUIV = [(s, e, n, sh, B) for s in ("lb", "ub", "both") for e, n in ((0, 20), (13, 31), (40, 64))
         for sh, B in (((), 5), (("q", "A", "b", "lb", "ub"), 5), (("p",), 3))] + [("lb", 40, 64, ("q", "A", "b", "lb"), 300)]


@pytest.mark.parametrize("sides,e,n,shared,B", EQUIV)
def test_box_matches_dense_qpfunction(sides, e, n, shared, B):
    bx = random_box(100 + e + n, B, n, e, sides, shared)
    a, d = run_box(bx), _dense_run(bx)
    assert rel_rows(a["zhat"], d["zhat"]).max() < 1e-8
    for k in GRAD_KEYS:
        if d["grads"][k] is None or np.asarray(d["grads"][k]).size == 0:
            assert a["grads"][k] is None, k
            continue
        assert a["grads"][k].shape == d["grads"][k].shape, k
        assert rel_rows(a["grads"][k], d["grads"][k], floor=1e-4).max() < 1e-6, k


def test_fallback_past_kernel_limit():
    from qpth_b200 import _lib
    bx = random_box(7, 3, 150, 130, "ub")
    assert _lib.box_plan_for(150, 130, False, True).ok == 0
    a, d = run_box(bx), _dense_run(bx)
    assert rel_rows(a["zhat"], d["zhat"]).max() < 1e-12
    for k in ("dq", "dp", "dA", "db", "dub"):
        assert rel_rows(a["grads"][k], d["grads"][k], floor=1e-4).max() < 1e-12, k


# ---- below convergence against the model ---------------------------------------------------------------------------
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if (t is not None and t.numel()) else ctypes.c_void_p(0)


@pytest.mark.parametrize("sides,e,n", [("lb", 40, 64), ("ub", 13, 37), ("both", 0, 25), ("both", 7, 9)])
def test_box_solve_kkt_matches_dense_refined_solve(sides, e, n):
    from qpth_b200 import _lib
    rs = np.random.RandomState(e + n)
    B = 6
    hl, hu = sides != "ub", sides != "lb"
    plan = _lib.box_plan_for(n, e, hl, hu)
    m = plan.nineq
    q, A = 0.1 + rs.rand(B, n), rs.randn(B, e, n)
    d = 10.0 ** rs.uniform(-8, 8, (B, m))
    rx, rs_, rz, ry = rs.randn(B, n), rs.randn(B, m), rs.randn(B, m), rs.randn(B, e)
    ins = [torch.tensor(v, dtype=torch.float64, device=DEV).contiguous() for v in (q, A, d, rx, rs_, rz, ry)]
    out = [torch.empty(B, k, dtype=torch.float64, device=DEV) for k in (n, m, m, e)]
    tq, tA = ins[:2]
    _lib.check(_lib.load().qpb200_box_solve_kkt(ctypes.byref(plan), B, _ptr(tq), n, _ptr(tA), e * n,
                                                *(_ptr(v) for v in ins[2:]), *(_ptr(o) for o in out),
                                                ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in out]
    var, sgn = bm.rows(n, hl, hu)
    G = np.zeros((m, n)); G[np.arange(m), var] = sgn
    for i in range(B):
        ref = dense_kkt.solve(np.diag(q[i]), G, A[i], d[i], rx[i], rs_[i], rz[i], ry[i])
        mod = bm.kkt_solve(q[i], A[i], hl, hu, d[i], rx[i], rs_[i], rz[i], ry[i])
        for k in range(4 if e else 3):
            err, merr = dense_kkt.rel(got[k][i], ref[k]), dense_kkt.rel(mod[k], ref[k])
            assert err <= max(10 * merr, 1e-10 if k != 1 else 1e-8), (i, k, err, merr)


@pytest.mark.parametrize("maxIter", [1, 2, 3, 5, 20])
@pytest.mark.parametrize("sides,e,n", [("lb", 40, 64), ("both", 13, 31), ("ub", 0, 20)])
def test_box_trajectory_matches_model(maxIter, sides, e, n):
    from qpth_b200 import qp as qpmod
    bx = random_box(9 + e, 4, n, e, sides)
    old = qpmod.TRACE
    qpmod.TRACE = True
    try:
        out = run_box(bx, maxIter=maxIter, requires=False)
    finally:
        qpmod.TRACE = old
    t = _batched(bx, 4)
    for i in range(4):
        tr = []
        sol = bm.solve_one(t["q"][i], t["p"][i], t["A"][i], t["b"][i], None if t["lb"] is None else t["lb"][i],
                           None if t["ub"] is None else t["ub"][i], maxIter=maxIter, stall_tol=qpmod.STALL_TOL,
                           tie=qpmod.BEST_TIE, trace=tr)
        assert out["iters"][i] == sol["iters"]
        tr = np.array(tr)
        assert np.allclose(out["trace"][i, :len(tr)], tr, rtol=1e-8, atol=1e-12, equal_nan=True), i
        assert abs(out["best_resid"][i] - sol["best_resid"]) <= 1e-8 * abs(sol["best_resid"]) + 1e-13
        assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9


@pytest.mark.parametrize("sides,e,n", [("lb", 40, 64), ("both", 13, 31), ("ub", 0, 20)])
def test_box_backward_and_batch_means(sides, e, n):
    """The backward's KKT solve at the kernels' own solution against the refined dense solve (bounded by 10x the model's
    own error on the same system: d = lam / s spans up to 16 decades there), the gradients formed from it exactly, and
    every input passed un-batched against the batch mean of the all-batched run."""
    B = 37
    bx = random_box(21 + e, B, n, e, sides)
    out = run_box(bx)
    t = _batched(bx, B)
    hl, hu = t["lb"] is not None, t["ub"] is not None
    var, sgn = bm.rows(n, hl, hu)
    G = np.zeros((var.shape[0], n)); G[np.arange(var.shape[0]), var] = sgn
    for i in range(B):
        d = np.maximum(out["lam"][i], 1e-8) / np.maximum(out["slacks"][i], 1e-8)
        m = d.shape[0]
        ref = dense_kkt.solve(np.diag(t["q"][i]), G, t["A"][i], d, bx["dl"][i], np.zeros(m), np.zeros(m), np.zeros(e))
        mod = bm.kkt_solve(t["q"][i], t["A"][i], hl, hu, d, bx["dl"][i], np.zeros(m), np.zeros(m), np.zeros(e))
        dx = out["grads"]["dp"][i]
        assert dense_kkt.rel(dx, ref[0]) <= max(10 * dense_kkt.rel(mod[0], ref[0]), 1e-10), i
        sol = dict(x=out["zhat"][i], lam=out["lam"][i], s=out["slacks"][i], nu=None if e == 0 else out["nus"][i],
                   q=t["q"][i], A=t["A"][i], nlb=n if hl else 0, var=var, sgn=sgn)

        if e:
            assert dense_kkt.rel(-out["grads"]["db"][i], ref[3]) <= max(10 * dense_kkt.rel(mod[3], ref[3]), 1e-10), i
            assert rel_rows(out["grads"]["dA"][i], np.outer(-out["grads"]["db"][i], sol["x"]) + np.outer(sol["nu"], dx)).max() < 1e-13
        assert rel_rows(out["grads"]["dq"][i], dx * sol["x"]).max() < 1e-13
        dlam = np.concatenate(([out["grads"]["dlb"][i]] if hl else []) + ([-out["grads"]["dub"][i]] if hu else []))
        assert dense_kkt.rel(dlam, ref[2]) <= max(10 * dense_kkt.rel(mod[2], ref[2]), 1e-10), i
    for shared in (("q", "A", "b", "lb", "ub"), ("p",)):
        sb = random_box(21 + e, B, n, e, sides, shared=shared)
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


def test_spd_check_and_verbose_output(capsys):
    bx = random_box(5, 3, 12, 4, "both")
    bad = dict(bx, q=bx["q"].copy())
    bad["q"][1, 3] = -0.5
    with pytest.raises(RuntimeError, match="Q is not SPD"):
        run_box(bad, requires=False)
    run_box(bad, requires=False, check_Q_spd=False)
    capsys.readouterr()
    run_box(bx, requires=False, verbose=1)
    box_lines = [l for l in capsys.readouterr().out.splitlines() if l.startswith("iter:")]
    from qpth_b200 import QPFunction
    from qpth_b200.box import dense_equivalent
    t = {k: (None if bx[k] is None else torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=DEV))
         for k in BOX_KEYS}
    Q, G, h = dense_equivalent(t["q"], t["lb"], t["ub"])
    QPFunction(verbose=1)(Q, t["p"], G, h, t["A"], t["b"])
    dense_lines = [l for l in capsys.readouterr().out.splitlines() if l.startswith("iter:")]
    assert len(box_lines) == len(dense_lines) > 0

    def nums(l):
        return [float(x) for x in l.replace(",", " ").split() if x[0].isdigit()]
    for a, b in zip(box_lines, dense_lines):
        assert np.allclose(nums(a), nums(b), rtol=1e-5, atol=1e-9), (a, b)
