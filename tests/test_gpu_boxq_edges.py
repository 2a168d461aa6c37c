"""The dense-Q box-QP kernels (csrc/qp_boxq.cu, the DenseQ family of qp_box_loop.cuh) at the edges of their plan, on
the GPU: every entry of tests/boxq_families.py (the widest nz, every byte of shared memory, the most equality rows, the
equality tile boundary, tiny shapes and the benchmark's shapes with their sharing) against references that share
nothing with the bordered factorization:
  a. qpb200_boxq_solve_kkt against the refined dense solve of the full KKT system (oracle/dense_kkt.py);
  b. the forward below and at convergence against the numpy model of its arithmetic (oracle/boxq_model.py);
  c. qpb200_boxq_backward_duals at a chosen point against the refined dense solve, all nine outputs;
  d. qpb200_boxq_jvp against tests/jvp_models.jvp_dense, and its transpose against (c);
  e. the gradients of BoxQPFunction(dense_Q=True, duals=True), and of QPFunction on the dense equivalent, at each
     path's own solution against the refined dense solve there;
  f. batch means of un-batched inputs under dual adjoints; g. forward AD through BoxQPFunction;
  h. one step past the plan: the dense path, against QPFunction on the dense equivalent.
Every test asserts its entry's plan (check_entry) before it solves. The first run of every entry happens in a child
process (tests/boxq_edges_child.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import boxq_model as qm, dense_kkt
from oracle.box_model import rows
from tests import jvp_models as jm
from tests.boxq_edges_child import (GRAD_NAMES, TANGENTS, kkt_inputs, point, run_backward, run_jvp, run_kkt,
                                    tangents)
from tests.boxq_families import ENTRIES, check_entry, dense_entries, kernel_entries, problem, sides_flags
from tests.boxq_util import KEYS, batched, random_boxq
from tests.parity import rel_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = kernel_entries()
CHILD_TIMEOUT_S = 600

# Entries whose 20-iteration runs end at the rounding floor of the residual, where the summation order decides the exit
# tests, with how far kernels and model were measured apart there (one H100): the most iterations and the largest
# difference of a trace row or of the best residual. Every other entry, and every entry below 20 iterations, is held to
# the exact iteration count and AT_TOL.
AT_FLOOR = {}
AT_TOL = dict(rtol=1e-8, atol=1e-11)
# Entries at which one corrector solve gives an exact ds = 0, where qpth's step rule takes -s / 0 = -inf as the step
# (batch.py:212) and the next iterate is NaN; the kernels' fused multiply-add and the model's separate roundings meet
# such a zero at different iterations, and whichever meets it first stops there. (84, 83, lb): the model's 8th residual
# is NaN, the kernels' 2.6e-13 (below eps); (1, 1, lb): on one QP the model's 2nd residual is NaN and the kernels' 3rd,
# on the other the kernels' 4th and the model's 5th. There the rows before the first NaN row are held to AT_TOL and the
# one that went on must end with a best residual no larger; where both meet it at the same row, the QP is held to
# everything below.
ZERO_STEP = ("most_eq_lb", "tiny_1_1")
EPS = np.finfo(np.float64).eps


def _rel(a, b):
    """max |a - b| / max |b| (0 for two empty arrays)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if b.size == 0:
        return 0.0
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _G(n, hl, hu):
    var, sgn = rows(n, hl, hu)
    G = np.zeros((var.shape[0], n))
    G[np.arange(var.shape[0]), var] = sgn
    return G


def _clamped_d(lam, s):
    return np.maximum(lam, 1e-8) / np.maximum(s, 1e-8)


def _grads(x, nu, dx, dlam, dnu, nlb, e):
    """the nine outputs of the backward from its solve (tests/dual_models._grads, box layout)"""
    m = dlam.shape[0]
    g = dict(dx=dx, dlam=dlam, dQ=0.5 * (np.outer(dx, x) + np.outer(x, dx)), dp=dx, dlb=dlam[:nlb] if nlb else None,
             dub=-dlam[nlb:] if m > nlb else None, dnu=None, dA=None, db=None)
    if e:
        g.update(dnu=dnu, dA=np.outer(dnu, x) + np.outer(nu, dx), db=-dnu)
    return g


def dlam_floor(d, G, dx, rz, dlam):
    """Ten roundings of dx carried into dlam = d (G dx + rz), relative to ||dlam||: where an active row has d near 1e8
    the formula amplifies them by d, in the kernels and the model alike, and which of the two rounds luckier decides
    their ratio, not their accuracy"""
    return 10 * EPS * np.linalg.norm(d * (np.abs(G @ dx) + np.abs(rz))) / max(np.linalg.norm(dlam), 1e-300)


def _refined(Q, A, hl, hu, d, rx, rz, ry):
    """(dx, ds, dz, dy) of the full KKT system with rs = 0, refined (oracle/dense_kkt.solve), and the model's"""
    n, e = Q.shape[0], A.shape[0]
    m = d.shape[0]
    ref = dense_kkt.solve(qm.sym_lower(Q), _G(n, hl, hu), A if e else None, d, rx, np.zeros(m), rz,
                          ry if e else None)[:4]
    mod = qm.kkt_solve(Q, A, hl, hu, d, rx, np.zeros(m), rz, ry if e else None)
    return ref, mod


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("boxq_edges_child"))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.boxq_edges_child", out], cwd=ROOT, timeout=CHILD_TIMEOUT_S,
                           capture_output=True, text=True)
    except subprocess.TimeoutExpired:
        prog = os.path.join(out, "progress.txt")
        last = open(prog).read().split()[-1:] if os.path.exists(prog) else []
        return out, "child killed after %d s (the last entry it started: %s)" % (CHILD_TIMEOUT_S,
                                                                                last[0] if last else "none")
    return out, "" if r.returncode == 0 else "child exited with %d: %s" % (r.returncode, r.stderr[-2000:])


@pytest.mark.parametrize("name", list(ENTRIES))
def test_first_runs_in_child_process(child_results, name):
    from tests.gpu_child import load
    out_dir, note = child_results
    rec = load(out_dir, note, name)
    assert np.isfinite(rec["zhat"]).all() and (rec["iters"] >= 1).all()
    assert bool(rec["dense"]) == (not ENTRIES[name]["edge"]["ok"])
    assert np.isfinite(rec["grad_dp"]).all() and np.isfinite(rec["grad_dQ"]).all()
    if ENTRIES[name]["edge"]["ok"]:
        assert np.isfinite(rec["jvp_dz"]).all() and np.isfinite(rec["kkt_dx"]).all()


# ---- a. the stand-alone KKT solve -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", KERNEL)
def test_solve_kkt_matches_refined_solve(name):
    """B = 3, d = 10^U(-8, 8): error <= max(10x the model's own error, 1e-10), 1e-8 for ds"""
    n, e, sides = ENTRIES[name]["shape"]
    hl, hu = sides_flags(sides)
    plan = check_entry(name)
    ins = kkt_inputs(plan, 3, 7 + n + e)
    got = run_kkt(plan, ins)
    Q, A, d, rx, rs, rz, ry = ins
    G = _G(n, hl, hu)
    for i in range(3):
        ref = dense_kkt.solve(qm.sym_lower(Q[i]), G, A[i] if e else None, d[i], rx[i], rs[i], rz[i],
                              ry[i] if e else None)
        mod = qm.kkt_solve(Q[i], A[i], hl, hu, d[i], rx[i], rs[i], rz[i], ry[i] if e else None)
        for k in range(4 if e else 3):
            err, merr = dense_kkt.rel(got[k][i], ref[k]), dense_kkt.rel(mod[k], ref[k])
            assert err <= max(10 * merr, 1e-10 if k != 1 else 1e-8), (i, k, err, merr)


def _first_nan_row(trace):
    bad = np.flatnonzero(~np.isfinite(trace).all(1))
    return int(bad[0]) if bad.size else len(trace)


# ---- b. below and at convergence against the model --------------------------------------------------------------------
@pytest.mark.parametrize("maxIter", [1, 2, 3, 20])
@pytest.mark.parametrize("name", KERNEL)
def test_trajectory_matches_model(name, maxIter):
    """iterations exact, trace rows, best residual and z* against the model"""
    from qpth_b200 import qp as qpmod
    from tests.boxq_util import run_boxq
    n, e, sides = ENTRIES[name]["shape"]
    B = 2
    bx = problem(name, B, 300 + n + e)
    check_entry(name)
    old = qpmod.TRACE
    qpmod.TRACE = True
    try:
        out = run_boxq(bx, requires=False, maxIter=maxIter)
    finally:
        qpmod.TRACE = old
    assert not out["dense"]
    bb = batched(bx, B)
    for i in range(B):
        tr = []
        sol = qm.solve_one(bb["Q"][i], bb["p"][i], bb["A"][i], bb["b"][i], None if bb["lb"] is None else bb["lb"][i],
                           None if bb["ub"] is None else bb["ub"][i], maxIter=maxIter, stall_tol=qpmod.STALL_TOL,
                           tie=qpmod.BEST_TIE, trace=tr)
        tr = np.array(tr)
        ki = int(out["iters"][i])
        k, kk = _first_nan_row(tr), _first_nan_row(out["trace"][i, :ki])
        if name in ZERO_STEP and kk != k:
            j = min(k, kk)
            assert np.allclose(out["trace"][i, :j], tr[:j], **AT_TOL), (i, np.abs(out["trace"][i, :j] - tr[:j]).max())
            if kk > k:      # the one that went on ends no worse
                assert ki >= sol["iters"] and out["best_resid"][i] <= sol["best_resid"], (i, k, kk)
            else:
                assert ki <= sol["iters"] and sol["best_resid"] <= out["best_resid"][i], (i, k, kk)
            continue
        floor = AT_FLOOR.get(name) if maxIter == 20 else None
        tol = AT_TOL
        if floor is None:
            assert out["iters"][i] == sol["iters"], (i, out["iters"][i], sol["iters"])
        else:
            assert abs(int(out["iters"][i]) - sol["iters"]) <= floor["iters"], (i, out["iters"][i], sol["iters"])
            tol = dict(rtol=1e-8, atol=floor["atol"])
            tr = tr[:int(out["iters"][i])]
        gap = np.abs(out["trace"][i, :len(tr)] - tr).max()
        assert np.allclose(out["trace"][i, :len(tr)], tr, equal_nan=True, **tol), (i, gap)
        assert abs(out["best_resid"][i] - sol["best_resid"]) <= tol["rtol"] * sol["best_resid"] + tol["atol"], \
            (i, out["best_resid"][i], sol["best_resid"])
        assert rel_rows(out["zhat"][i], sol["x"]).max() < 1e-9, (i, rel_rows(out["zhat"][i], sol["x"]).max())


# ---- c. the backward with dual adjoints at a chosen point -------------------------------------------------------------
@pytest.mark.parametrize("name", KERNEL)
def test_dual_backward_at_a_point(name):
    """All nine outputs against the refined dense solve within 1e-10 (lam, s ~ U(0.1, 10)); linear in (dl, glam, gnu)
    within 1e-12; NULL dual adjoints exactly as zero-filled ones; lam, s ~ 10^U(-12, 0) (d clamped to [1e-8, 1e8])
    within 10x the model's own error"""
    n, e, sides = ENTRIES[name]["shape"]
    hl, hu = sides_flags(sides)
    nlb = n if hl else 0
    plan = check_entry(name)
    B = 2
    pt = point(plan, B, 600 + n + e)
    gnu = pt["gnu"] if e else None
    zero = np.zeros_like(pt["dl"])
    full = run_backward(plan, pt, pt["dl"], pt["glam"], gnu)
    nul = run_backward(plan, pt, pt["dl"], None, None)
    zer = run_backward(plan, pt, pt["dl"], np.zeros_like(pt["glam"]), np.zeros_like(gnu) if e else None)
    lam_only = run_backward(plan, pt, zero, pt["glam"], None)
    nu_only = run_backward(plan, pt, zero, None, gnu) if e else None
    for i in range(B):
        d = _clamped_d(pt["lam"][i], pt["s"][i])
        ref, _ = _refined(pt["Q"][i], pt["A"][i], hl, hu, d, pt["dl"][i], pt["glam"][i], gnu[i] if e else None)
        want = _grads(pt["z"][i], pt["nu"][i], ref[0], ref[2], ref[3], nlb, e)
        for k in GRAD_NAMES:
            assert (full[k] is None) == (want[k] is None), k
            if want[k] is not None:
                assert _rel(full[k][i], want[k]) <= 1e-10, (k, i, _rel(full[k][i], want[k]))
    for k in GRAD_NAMES:
        if full[k] is None:
            continue
        assert np.array_equal(nul[k], zer[k]), k
        total = nul[k] + lam_only[k] + (nu_only[k] if e else 0.0)
        assert np.abs(full[k] - total).max() <= 1e-12 * np.abs(full[k]).max(), k
    ptw = point(plan, B, 650 + n + e, wide=True)
    gnu = ptw["gnu"] if e else None
    got = run_backward(plan, ptw, ptw["dl"], ptw["glam"], gnu)
    var, sgn = rows(n, hl, hu)
    for i in range(B):
        d = _clamped_d(ptw["lam"][i], ptw["s"][i])
        assert d.min() >= 1e-8 * (1 - 1e-15) and d.max() <= 1e8 * (1 + 1e-15)
        ref, _ = _refined(ptw["Q"][i], ptw["A"][i], hl, hu, d, ptw["dl"][i], ptw["glam"][i], gnu[i] if e else None)
        sol = dict(Q=ptw["Q"][i], A=ptw["A"][i], var=var, sgn=sgn, nlb=nlb, lam=ptw["lam"][i], s=ptw["s"][i],
                   x=ptw["z"][i], nu=ptw["nu"][i])
        mod = qm.backward_one(sol, ptw["dl"][i], ptw["glam"][i], gnu[i] if e else None)
        for k, j in (("dx", 0), ("dlam", 2)) + ((("dnu", 3),) if e else ()):
            err, merr = dense_kkt.rel(got[k][i], ref[j]), dense_kkt.rel(mod[k], ref[j])
            assert err <= max(10 * merr, 1e-10), (k, i, err, merr)


# ---- d. forward mode at a chosen point ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", KERNEL)
def test_jvp_at_a_point(name):
    """Every tangent batched (dQ not symmetric) against jvp_dense on the dense equivalent within 1e-10; each tangent
    alone sums to the full result; stride-0 tangents exactly as broadcast ones; the transpose of the backward"""
    n, e, sides = ENTRIES[name]["shape"]
    hl, hu = sides_flags(sides)
    plan = check_entry(name)
    B = 2
    pt = point(plan, B, 800 + n + e)
    tan = tangents(plan, B, n + e)
    got = run_jvp(plan, pt, tan)
    parts = [run_jvp(plan, pt, {k: tan[k]}) for k in TANGENTS if tan[k] is not None]
    un = {k: (None if v is None else v[0]) for k, v in tan.items()}
    s0 = run_jvp(plan, pt, un)
    bc = run_jvp(plan, pt, {k: (None if v is None else np.broadcast_to(v, (B,) + v.shape)) for k, v in un.items()})
    gnu = pt["gnu"] if e else None
    grads = run_backward(plan, pt, pt["dl"], pt["glam"], gnu)
    G = _G(n, hl, hu)
    for i in range(B):
        dh = np.concatenate(([-tan["lb"][i]] if hl else []) + ([tan["ub"][i]] if hu else []))
        ti = dict(Q=tan["Q"][i], p=tan["p"][i], h=dh, A=tan["A"][i] if e else None, b=tan["b"][i] if e else None)
        ref = jm.jvp_dense(qm.sym_lower(pt["Q"][i]), G, pt["A"][i] if e else None, pt["z"][i], pt["lam"][i],
                           pt["s"][i], pt["nu"][i] if e else None, ti)
        for j in range(3 if e else 2):
            assert _rel(got[j][i], ref[j]) <= 1e-10, (j, i, _rel(got[j][i], ref[j]))
    for j in range(3 if e else 2):
        total = sum(p[j] for p in parts)
        assert np.abs(got[j] - total).max() <= 1e-12 * np.abs(got[j]).max(), j
        assert np.array_equal(s0[j], bc[j]), j
    lhs = np.sum(pt["dl"] * got[0]) + np.sum(pt["glam"] * got[1]) + (np.sum(gnu * got[2]) if e else 0.0)
    gx = dict(Q=grads["dQ"], p=grads["dp"], A=grads["dA"], b=grads["db"], lb=grads["dlb"], ub=grads["dub"])
    terms = [np.sum(gx[k] * tan[k]) for k in TANGENTS if tan[k] is not None]
    assert abs(lhs - sum(terms)) <= 1e-10 * max(abs(lhs), sum(abs(t) for t in terms)), (lhs, sum(terms))


# ---- e. converged gradients at each path's own solution ----------------------------------------------------------------
def _tensors(bx, requires=True):
    t = {}
    for k in KEYS:
        v = bx[k]
        if v is None:
            t[k] = None
        elif np.asarray(v).size == 0:
            t[k] = torch.Tensor().to(DEV).double()
        else:
            t[k] = torch.tensor(np.ascontiguousarray(v), dtype=torch.float64, device=DEV, requires_grad=requires)
    return t


def _loss(z, lam, nu, gz, gl, gn):
    T = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV)
    return (z * T(gz)).sum() + (lam * T(gl)).sum() + ((nu * T(gn)).sum() if gn.size else 0.0)


def run_box_duals(bx, gz, gl, gn):
    """BoxQPFunction(dense_Q=True, duals=True) forward and the backward of <gz, z> + <gl, lam> + <gn, nu>"""
    from qpth_b200 import BoxQPFunction
    t = _tensors(bx)
    f = BoxQPFunction(verbose=-1, dense_Q=True, duals=True)
    z, lam, nu = f(*(t[k] for k in KEYS))
    _loss(z, lam, nu, gz, gl, gn).backward()
    st = f.last_solve()
    c = lambda v: None if v is None else v.detach().cpu().numpy()
    return dict(z=c(z), lam=c(lam), s=c(st.slacks), nu=c(nu), dense=st.dense is not None,
                grads={k: (None if (t[k] is None or t[k].grad is None) else c(t[k].grad)) for k in KEYS})


def run_qpf_duals(bx, gz, gl, gn):
    """QPFunction(duals=True) on the dense equivalent, the same loss; the gradient of h mapped to lb / ub"""
    from qpth_b200 import QPFunction
    from qpth_b200.box import dense_equivalent
    t = _tensors(bx, requires=False)
    Q, G, h = dense_equivalent(t["Q"], t["lb"], t["ub"], dense_Q=True)
    ins = dict(Q=Q.clone(), p=t["p"], G=G, h=h.clone(), A=t["A"], b=t["b"])
    for k in ("Q", "p", "h", "A", "b"):
        if ins[k].numel():
            ins[k].requires_grad_(True)
    f = QPFunction(verbose=-1, duals=True)
    z, lam, nu = f(*(ins[k] for k in ("Q", "p", "G", "h", "A", "b")))
    _loss(z, lam, nu, gz, gl, gn).backward()
    st = f.last_solve()
    c = lambda v: None if v is None else v.detach().cpu().numpy()
    g = {k: (c(ins[k].grad) if ins[k].grad is not None else None) for k in ("Q", "p", "A", "b")}
    dh = c(ins["h"].grad)
    nlb = Q.shape[-1] if t["lb"] is not None else 0
    g["lb"] = -dh[..., :nlb] if nlb else None
    g["ub"] = dh[..., nlb:] if t["ub"] is not None else None
    return dict(z=c(z), lam=c(lam), s=c(st.slacks), nu=c(nu), grads=g, h_batched=h.dim() == 2)


def own_solution_errors(name, out, bx, gz, gl, gn, h_batched=None):
    """Per QP: (output, error, bound) of dx, dlam, dnu (where a batched input shows them) against the refined solve at
    d = clamp(lam) / clamp(s) of the returned point; the bound is max(10x the model's error there, 1e-10, and for dlam
    dlam_floor). Asserts dQ and dA from the returned outputs."""
    n, e, sides = ENTRIES[name]["shape"]
    hl, hu = sides_flags(sides)
    B = gz.shape[0]
    bb = batched(bx, B)
    g = out["grads"]
    shown = {k: bx[k] is not None and np.asarray(bx[k]).ndim == (3 if k in ("Q", "A") else 2) for k in KEYS}
    lam_shown = h_batched if h_batched is not None else all(shown[k] for k in ("lb", "ub") if bx[k] is not None)
    errs = []
    dQ_mean = np.zeros((n, n))
    for i in range(B):
        x, dx = out["z"][i], g["p"][i]
        d = _clamped_d(out["lam"][i], out["s"][i])
        ref, mod = _refined(bb["Q"][i], bb["A"][i], hl, hu, d, gz[i], gl[i], gn[i] if e else None)
        got = [(0, dx)]
        if lam_shown:
            got.append((2, np.concatenate(([g["lb"][i]] if hl else []) + ([-g["ub"][i]] if hu else []))))
        if e and shown["b"]:
            got.append((3, -g["b"][i]))
        floor = {0: 0.0, 2: dlam_floor(d, _G(n, hl, hu), ref[0], gl[i], ref[2]), 3: 0.0}
        errs.append([(k, dense_kkt.rel(v, ref[k]), max(10 * dense_kkt.rel(mod[k], ref[k]), 1e-10, floor[k]))
                     for k, v in got])
        dQ = 0.5 * (np.outer(dx, x) + np.outer(x, dx))
        dQ_mean += dQ / B
        if shown["Q"]:
            assert _rel(g["Q"][i], dQ) <= 1e-13, (i, _rel(g["Q"][i], dQ))
        if e and shown["A"] and shown["b"]:
            dA = np.outer(-g["b"][i], x) + np.outer(out["nu"][i], dx)
            assert _rel(g["A"][i], dA) <= 1e-13, (i, _rel(g["A"][i], dA))
    if not shown["Q"]:
        assert _rel(g["Q"], dQ_mean) <= 1e-12, _rel(g["Q"], dQ_mean)
    return errs


@pytest.mark.parametrize("name", KERNEL)
def test_converged_gradients_at_own_solution(name):
    """BoxQPFunction(dense_Q=True, duals=True) and QPFunction(duals=True) on the dense equivalent, a loss on z, lam and
    nu: each path's dx, dlam and dnu against the refined solve at its own returned point, within max(10x the model's
    error there, 1e-10; for dlam also dlam_floor); dQ = 1/2 (dx z' + z dx') and dA = dnu z' + nu dx' from each path's own outputs"""
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    hl, hu = sides_flags(sides)
    B = 3
    bx = problem(name, B, (7 if ent["gen"] == "bench" else 900) + n + e)
    check_entry(name)
    rs = np.random.RandomState(n + e)
    gz, gl, gn = rs.randn(B, n), rs.randn(B, n * (hl + hu)), rs.randn(B, e)
    box = run_box_duals(bx, gz, gl, gn)
    assert not box["dense"]
    qpf = run_qpf_duals(bx, gz, gl, gn)
    for path, out, hb in (("dense_Q", box, None), ("QPFunction", qpf, qpf["h_batched"])):
        for i, errs in enumerate(own_solution_errors(name, out, bx, gz, gl, gn, hb)):
            for k, err, bound in errs:
                assert err <= bound, (path, i, k, err, bound)


# ---- f. batch means under dual adjoints --------------------------------------------------------------------------------
@pytest.mark.parametrize("shared", [("Q",), ("p",), ("A", "b"), ("lb", "ub")])
@pytest.mark.parametrize("name", ["full_both", "most_eq_lb"])
def test_batch_means_with_dual_adjoints(name, shared):
    """an input passed un-batched: its gradient is the batch mean of the all-batched run within 1e-12, the others equal
    (qpb200_internal_mean_outer for dQ, qpb200_internal_box_means for the rest, with glam and gnu nonzero)"""
    n, e, sides = ENTRIES[name]["shape"]
    hl, hu = sides_flags(sides)
    B = 4
    check_entry(name)
    sb = random_boxq(31 + e, B, n, e, sides, shared)
    full = dict(batched(sb, B), dl=sb["dl"])
    rs = np.random.RandomState(5)
    gz, gl, gn = rs.randn(B, n), rs.randn(B, n * (hl + hu)), rs.randn(B, e)
    a, f = run_box_duals(sb, gz, gl, gn), run_box_duals(full, gz, gl, gn)
    for k in KEYS:
        if f["grads"][k] is None:
            assert a["grads"][k] is None, k
            continue
        if k in shared:
            assert a["grads"][k].shape == f["grads"][k].shape[1:], k
            assert _rel(a["grads"][k], f["grads"][k].mean(0)) <= 1e-12, (k, _rel(a["grads"][k], f["grads"][k].mean(0)))
        else:
            assert _rel(a["grads"][k], f["grads"][k]) <= 1e-12, k


# ---- g. forward AD -------------------------------------------------------------------------------------------------------
def test_forward_ad_matches_the_entry_point():
    """torch.autograd.forward_ad through BoxQPFunction(dense_Q=True, duals=True) at (144, 32, both) with Q, A, b, lb
    and ub shared and their tangents un-batched: qpb200_boxq_jvp with the tangents broadcast, within 1e-12"""
    import torch.autograd.forward_ad as fwAD
    from qpth_b200 import BoxQPFunction
    name = "full_both"
    n, e, sides = ENTRIES[name]["shape"]
    plan = check_entry(name)
    B = 3
    shared = ("Q", "A", "b", "lb", "ub")
    bx = random_boxq(55, B, n, e, sides, shared)
    rs = np.random.RandomState(6)
    tan = dict(Q=rs.randn(n, n), p=rs.randn(B, n), A=rs.randn(e, n), b=rs.randn(e), lb=rs.randn(n), ub=rs.randn(n))
    t = _tensors(bx, requires=False)
    f = BoxQPFunction(verbose=-1, dense_Q=True, duals=True)
    with fwAD.dual_level():
        x = [fwAD.make_dual(t[k], torch.tensor(tan[k], dtype=torch.float64, device=DEV)) for k in KEYS]
        got = [fwAD.unpack_dual(o).tangent.cpu().numpy() for o in f(*x)]
    st = f.last_solve()
    bb = batched(bx, B)
    pt = dict(Q=bb["Q"], A=bb["A"], z=st.zhat.cpu().numpy(), nu=st.nus.cpu().numpy(), lam=st.lam.cpu().numpy(),
              s=st.slacks.cpu().numpy())
    want = run_jvp(plan, pt, {k: (v if v.ndim == (3 if k in ("Q", "A") else 2) else np.broadcast_to(v, (B,) + v.shape))
                              for k, v in tan.items()})
    for j in range(3):
        assert _rel(got[j], want[j]) <= 1e-12, (j, _rel(got[j], want[j]))


# ---- h. past the plan: the dense path ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", dense_entries())
def test_past_the_edge_takes_the_dense_path(name):
    """BoxQPFunction(dense_Q=True, duals=True) one step past an edge runs the dense kernels on the dense equivalent:
    lam and nu exactly QPFunction's there, the gradients of a loss on z, lam, nu and the JVP within 1e-10"""
    import torch.autograd.forward_ad as fwAD
    from qpth_b200 import BoxQPFunction, QPFunction
    from qpth_b200.box import dense_equivalent
    n, e, sides = ENTRIES[name]["shape"]
    plan = check_entry(name)
    assert not plan.ok
    bx = random_boxq(700 + n, 2, n, e, sides)
    f = BoxQPFunction(verbose=-1, dense_Q=True, duals=True)
    t = _tensors(bx)
    z, lam, nu = f(*(t[k] for k in KEYS))
    assert f.last_solve().dense is not None
    rs = np.random.RandomState(9)
    gz, gl, gn = (torch.tensor(rs.randn(*v.shape), dtype=torch.float64, device=DEV) for v in (z, lam, nu))
    ((z * gz).sum() + (lam * gl).sum() + (nu * gn).sum()).backward()
    got = [t[k].grad.clone() for k in KEYS if t[k] is not None and t[k].requires_grad]
    t2 = _tensors(bx)
    Q, G, h = dense_equivalent(t2["Q"], t2["lb"], t2["ub"], dense_Q=True)
    z2, lam2, nu2 = QPFunction(verbose=-1, duals=True)(Q, t2["p"], G, h, t2["A"], t2["b"])
    assert torch.equal(lam, lam2) and torch.equal(nu, nu2)
    ((z2 * gz).sum() + (lam2 * gl).sum() + (nu2 * gn).sum()).backward()
    want = [t2[k].grad for k in KEYS if t2[k] is not None and t2[k].requires_grad]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert torch.allclose(g, w, rtol=1e-10, atol=1e-12)
    p = _tensors(bx, requires=False)
    tan = {k: (None if v is None or not v.numel() else torch.tensor(rs.randn(*v.shape), dtype=torch.float64,
                                                                     device=DEV)) for k, v in p.items()}
    with fwAD.dual_level():
        x = {k: (v if tan[k] is None else fwAD.make_dual(v, tan[k])) for k, v in p.items()}
        outs = BoxQPFunction(verbose=-1, dense_Q=True, duals=True)(*(x[k] for k in KEYS))
        jv = [fwAD.unpack_dual(o).tangent for o in outs]
        Q, G, h = dense_equivalent(x["Q"], x["lb"], x["ub"], dense_Q=True)
        outs2 = QPFunction(verbose=-1, duals=True)(Q, x["p"], G.detach(), h, x["A"], x["b"])
        jw = [fwAD.unpack_dual(o).tangent for o in outs2]
    for g, w in zip(jv, jw):
        assert (g is None and w is None) or torch.allclose(g, w, rtol=1e-10, atol=1e-12)
