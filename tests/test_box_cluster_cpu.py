"""Box QPs beyond one CTA without a GPU: the plans of the thread block cluster kernels (csrc/qp_box.cu), the closed-form
projections of oracle/projections.py against the numpy model and the dense interior-point oracle, and the real
reference's `box_wide` fixture against the model."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import box_model as bm, pdipm_oracle as orc
from oracle.box_cases import dense_problem, map_dense_grads
from oracle.box_wide_cases import WIDE_BOX_CASES
from oracle.cases import checksum, proj
from oracle.projections import project_box, project_capped_simplex
from tests.parity import GTOL, ZTOL, rel_rows
from tests.test_box_cpu import _batched

MAX_SMEM = 232448


def _plan(n, e, lb, ub):
    from qpth_b200 import _lib
    return _lib.box_plan_for(n, e, lb, ub)


@pytest.fixture
def no_knob(monkeypatch):
    monkeypatch.delenv("QPB200_BOX_CLUSTER", raising=False)


def test_cluster_plans(no_knob):
    p = _plan(600, 64, True, True)
    assert p.ok == 0 and p.cl_ctas >= 2 and p.cl_slice * p.cl_ctas >= 600
    assert p.cl_smem_bytes <= MAX_SMEM
    assert _plan(150, 130, False, True).cl_ctas == 0          # neq_pad > 128: the dense kernels
    p = _plan(6000, 1, True, True)
    assert p.ok == 0 and p.cl_ctas in (2, 4, 8) and 0 < p.cl_smem_bytes <= MAX_SMEM
    assert p.cl_slice * p.cl_ctas >= 6000
    p = _plan(2000, 1, True, True)                             # the capped simplex over 2000 classes
    assert p.cl_ctas in (2, 4, 8) and p.cl_smem_bytes <= MAX_SMEM
    for n, e, lb, ub in ((64, 40, True, False), (600, 64, True, True), (37, 13, True, True)):
        p = _plan(n, e, lb, ub)
        assert p.ok == 1 or p.cl_ctas, (n, e)
        if p.ok:
            assert p.cl_ctas == 0 and p.smem_bytes <= MAX_SMEM   # one CTA wherever it covers the shape


def test_cluster_size_is_the_smallest_that_fits(no_knob):
    from qpth_b200 import _lib
    for n, e in ((600, 64), (1000, 1), (3000, 8), (6000, 1), (5000, 0)):
        p = _plan(n, e, True, True)
        assert p.cl_ctas, (n, e)
        if p.cl_ctas > 2:                                      # half the cluster would not fit
            q = _lib.BoxPlan()
            os.environ["QPB200_BOX_CLUSTER"] = str(p.cl_ctas // 2)
            try:
                assert _lib.load().qpb200_box_plan_init(n, e, 1, 1, ctypes.byref(q)) == 0
            finally:
                del os.environ["QPB200_BOX_CLUSTER"]
            assert q.cl_ctas == p.cl_ctas                      # the knob's size does not fit: the normal choice


def test_past_every_path_is_too_large(no_knob):
    from qpth_b200 import _lib
    lib = _lib.load()
    for n, e, lb, ub in ((20000, 1, 1, 1), (12000, 1, 1, 1), (5000, 200, 1, 1), (2048, 128, 1, 1)):
        assert lib.qpb200_box_plan_init(n, e, lb, ub, ctypes.byref(_lib.BoxPlan())) == 4, (n, e)
    # the dense path still takes neq_pad > 128 where it fits
    assert lib.qpb200_box_plan_init(150, 130, 0, 1, ctypes.byref(_lib.BoxPlan())) == 0


def test_cluster_knob_changes_the_plan_and_the_cache_sees_it(monkeypatch):
    monkeypatch.delenv("QPB200_BOX_CLUSTER", raising=False)
    a = _plan(64, 40, True, False)
    assert a.ok == 1 and a.cl_ctas == 0
    for C in (2, 4, 8):
        monkeypatch.setenv("QPB200_BOX_CLUSTER", str(C))
        p = _plan(64, 40, True, False)
        assert p.ok == 1 and p.cl_ctas == C and p.cl_slice == -(-64 // C) and p.cl_smem_bytes <= MAX_SMEM
    monkeypatch.setenv("QPB200_BOX_CLUSTER", "3")               # not a cluster size: ignored
    assert _plan(64, 40, True, False).cl_ctas == 0
    monkeypatch.delenv("QPB200_BOX_CLUSTER")
    assert _plan(64, 40, True, False).cl_ctas == 0


def test_cluster_plan_checks():
    from qpth_b200 import _lib
    lib = _lib.load()
    bad = _lib.BoxPlan()
    assert lib.qpb200_box_plan_init(600, 64, 1, 1, ctypes.byref(bad)) == 0
    bad.cl_ctas = 3
    assert lib.qpb200_box_solve_kkt(ctypes.byref(bad), 1, None, 0, None, 0, None, None, None, None, None,
                                    None, None, None, None, None) == 1
    bad.cl_ctas = 0
    assert lib.qpb200_box_solve_kkt(ctypes.byref(bad), 1, None, 0, None, 0, None, None, None, None, None,
                                    None, None, None, None, None) == 4


def test_header_and_signatures_keep_the_existing_entries():
    from qpth_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "qpth_b200.h")).read()
    body = re.search(r"typedef struct qpb200_box_plan \{(.*?)\} qpb200_box_plan;", hdr, re.S).group(1)
    fields = re.findall(r"\b(?:int|int64_t)\s+([\w, ]+);", body)
    names = [f.strip() for grp in fields for f in grp.split(",")]
    assert names == ["nz", "neq", "neq_pad", "nineq", "has_lb", "has_ub", "threads", "smem_bytes", "ok",
                     "cl_ctas", "cl_slice", "cl_smem_bytes"]
    assert [f[0] for f in _lib.BoxPlan._fields_] == names
    assert ctypes.sizeof(_lib.BoxPlan) == 64
    for name in ("qpb200_box_plan_init", "qpb200_box_forward", "qpb200_box_backward", "qpb200_box_solve_kkt"):
        assert re.search(r"\bint " + name + r"\(", hdr), name
        assert name in _lib.SIGNATURES, name
    assert len(_lib.SIGNATURES["qpb200_box_forward"][1]) == 28
    assert len(_lib.SIGNATURES["qpb200_box_backward"][1]) == 27
    assert len(_lib.SIGNATURES["qpb200_box_solve_kkt"][1]) == 16


# ---- closed-form projections -------------------------------------------------------------------------------------------
def _problem(kind, n, seed, sides="both"):
    rs = np.random.RandomState(seed)
    q = 0.5 + rs.rand(n)
    p = 2.0 * rs.randn(n)
    lb = -rs.rand(n) if sides in ("lb", "both") else None
    ub = 0.5 + rs.rand(n) if sides in ("ub", "both") else None
    if kind == "simplex":
        lo = 0.0 if lb is None else lb.sum()
        k = lo + 0.3 * n if ub is None else lo + 0.4 * ((ub.sum() if lb is None else (ub - lb).sum()))
        A, b = np.ones((1, n)), np.array([k])
    else:
        A, b = np.zeros((0, n)), np.zeros(0)
    return q, p, A, b, lb, ub, rs.randn(n)


def _closed(kind, q, p, A, b, lb, ub):
    if kind == "simplex":
        z, nu, vjp = project_capped_simplex(q, p, b[0], lb, ub)
    else:
        z, vjp = project_box(q, p, lb, ub)
    return z, vjp


@pytest.mark.parametrize("kind,sides", [("box", "both"), ("box", "lb"), ("box", "ub"), ("simplex", "both"),
                                        ("simplex", "lb")])
def test_projections_match_model_and_dense_oracle(kind, sides):
    n = 17
    for seed in range(3):
        q, p, A, b, lb, ub, dl = _problem(kind, n, 50 + seed, sides)
        z, vjp = _closed(kind, q, p, A, b, lb, ub)
        if kind == "simplex":
            assert abs(z.sum() - b[0]) < 1e-12
        g = vjp(dl)
        sol = bm.solve_one(q, p, A, b, lb, ub, stall_tol=1e-6, tie=1.5)
        assert np.abs(sol["x"] - z).max() < 1e-8
        gm = bm.backward_one(sol, dl)
        for k in ("dq", "dp", "dlb", "dub", "dA", "db"):
            if g[k] is None:
                assert gm[k] is None, k
                continue
            assert rel_rows(gm[k], g[k], floor=1e-4).max() < 1e-6, (k, seed)
        Q, G, h = bm.dense(q, lb, ub)
        ref = orc.qp_solve(Q[None], p[None], G[None], h[None], A[None] if A.size else np.zeros((0,)),
                           b[None] if b.size else np.zeros((0,)), dl[None], per_qp=True)
        assert np.abs(ref["zhat"][0] - z).max() < 1e-8
        assert rel_rows(ref["grads"][1][0], g["dp"], floor=1e-4).max() < 1e-6


def test_capped_simplex_jvp_matches_finite_differences():
    n = 12
    q, p, A, b, lb, ub, dl = _problem("simplex", n, 7)
    z, vjp = _closed("simplex", q, p, A, b, lb, ub)
    g = vjp(dl)
    h = 1e-7
    for name, val, idx in (("dp", p, 3), ("dq", q, 5), ("dlb", lb, None), ("dub", ub, None), ("db", b, 0)):
        if idx is None:       # a bound that is active, if any
            act = np.nonzero(g[name])[0]
            if act.size == 0:
                continue
            idx = act[0]
        vp, vm = val.copy(), val.copy()
        vp[idx] += h; vm[idx] -= h
        args = dict(q=q, p=p, b=b, lb=lb, ub=ub)
        key = {"dp": "p", "dq": "q", "dlb": "lb", "dub": "ub", "db": "b"}[name]
        zp = _closed("simplex", **dict(args, A=A, **{key: vp}))[0]
        zm = _closed("simplex", **dict(args, A=A, **{key: vm}))[0]
        fd = dl @ (zp - zm) / (2 * h)
        assert abs(g[name].reshape(-1)[idx] - fd) < 1e-6 * max(1.0, abs(fd)), name


# ---- the real reference's box_wide fixture against the model ------------------------------------------------------------
def load_wide(name, golden_dir):
    bx = WIDE_BOX_CASES[name]()
    gold = dict(np.load(os.path.join(golden_dir, name + ".npz")))
    cs = checksum(dense_problem(bx))
    assert abs(cs - float(gold["input_checksum"])) <= 1e-9 * abs(cs), "golden inputs no longer reproduce from the seed"
    return bx, gold


# The reference (dense KKT factorization) and the box formulation stop at different last iterates: z* agrees to 1.2e-8
# and the gradients to 1.3e-5 between the model and the reference at box_wide, while the reference moves by 1e-14 under
# a 1e-15 perturbation of its inputs (sens_* in the fixture). With 1200 bounds, the d = lam / s of weakly active ones
# differs between those iterates, and the backward passes that on. Both bounds sit about 2x above what was measured.
WIDE_ZTOL, WIDE_GTOL = 2.5e-8, 3e-5


def check_wide_golden(out, gold, bx, ztol=WIDE_ZTOL, gtol=WIDE_GTOL):
    """z*, lam, slacks, nus and the box gradients (batch means for the shared q, lb, ub; dA through its projection)"""
    n = np.asarray(bx["q"]).shape[-1]
    for k in ("zhat", "lam", "slacks", "nus"):
        assert rel_rows(out[k], gold[k]).max() <= ztol, k
    g = out["grads"]
    ref = dict(dq=gold["dq"], dp=gold["dp"], db=gold["db"], dlb=-gold["dh"][..., :n], dub=gold["dh"][..., n:])
    for k, v in ref.items():
        assert g[k].shape == v.shape, k
        assert rel_rows(g[k], v, floor=1e-4).max() <= gtol, k
    assert rel_rows(g["dA"] @ proj(n), gold["dA_proj"], floor=1e-4).max() <= gtol


@pytest.mark.parametrize("name", list(WIDE_BOX_CASES))
def test_model_matches_wide_reference_golden(name, golden_dir):
    bx, gold = load_wide(name, golden_dir)
    B = np.asarray(bx["p"]).shape[0]
    t = _batched(bx, B)
    out = bm.qp_solve(t["q"], t["p"], t["A"], t["b"], t["lb"], t["ub"], dl=bx["dl"], stall_tol=1e-6, tie=1.5)
    g = out["grads"]
    for k in ("dq", "dlb", "dub"):      # shared in the case
        g[k] = g[k].mean(0)
    check_wide_golden(dict(out, grads=g), gold, bx)
