"""Dense-Q box QPs without a GPU: the numpy model of csrc/qp_boxq.cu (oracle/boxq_model.py) against the reference's
fixtures, the iteration model of the dense path and the refined dense KKT solve; the plan (qpb200_boxq_plan_init);
the exports; the shape checks of BoxQPFunction(dense_Q=True)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import box_model as bm, boxq_model as qm, dense_kkt
from oracle.boxq_cases import BOXQ_CASES
from tests.boxq_util import batched, load_boxq_case, random_boxq
from tests.parity import GTOL, ZTOL, rel_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the largest shape one CTA holds for each bound pattern, with one equality row: (nz, neq, sides)
LARGEST = [(192, 1, "lb"), (192, 1, "ub"), (184, 1, "both")]


def _sides(s):
    return s != "ub", s != "lb"


@pytest.mark.parametrize("name", list(BOXQ_CASES))
def test_model_matches_reference_fixtures(name, golden_dir):
    bx, gold = load_boxq_case(name, golden_dir)
    B = np.asarray(bx["p"]).shape[0]
    bb = batched(bx, B)
    out = qm.qp_solve(bb["Q"], bb["p"], bb["A"], bb["b"], bb["lb"], bb["ub"], dl=bx["dl"])
    assert rel_rows(out["zhat"], gold["zhat"]).max() <= ZTOL
    g = out["grads"]
    n = bb["Q"].shape[-1]
    nlb = n if bx["lb"] is not None else 0
    for k, ref in (("dQ", gold["dQ"]), ("dp", gold["dp"])):
        mine = g[k] if g[k].shape == ref.shape else g[k].mean(0)
        assert rel_rows(mine, ref, floor=1e-4).max() <= GTOL, k
    if bx["lb"] is not None:
        ref = -gold["dh"][..., :nlb]
        assert rel_rows(g["dlb"], ref if ref.ndim == 2 else np.broadcast_to(ref, g["dlb"].shape), floor=1e-4).max() \
            <= GTOL or rel_rows(g["dlb"].mean(0), ref, floor=1e-4).max() <= GTOL


@pytest.mark.parametrize("sides,e,n", [("both", 3, 12), ("lb", 0, 9), ("ub", 5, 17)])
def test_model_matches_dense_iteration_model(sides, e, n):
    from oracle import kernel_model as km
    hl, hu = _sides(sides)
    bx = random_boxq(21 + n, 2, n, e, sides)
    bb = batched(bx, 2)
    for i in range(2):
        Q, G, h = qm.dense(bb["Q"][i], None if bb["lb"] is None else bb["lb"][i],
                           None if bb["ub"] is None else bb["ub"][i])
        a = qm.solve_one(bb["Q"][i], bb["p"][i], bb["A"][i], bb["b"][i], None if bb["lb"] is None else bb["lb"][i],
                         None if bb["ub"] is None else bb["ub"][i])
        d = km.solve_one(Q, bb["p"][i], G, h, bb["A"][i], bb["b"][i])
        assert rel_rows(a["x"], d["x"]).max() < 1e-8


@pytest.mark.parametrize("sides,e,n", [("both", 3, 12), ("lb", 0, 9), ("ub", 7, 20), ("both", 16, 30)])
def test_model_kkt_matches_refined_dense_solve(sides, e, n):
    hl, hu = _sides(sides)
    rs = np.random.RandomState(n + e)
    Q = random_boxq(n, 1, n, 1, sides)["Q"][0]
    A = rs.randn(e, n)
    var, sgn = bm.rows(n, hl, hu)
    m = var.shape[0]
    G = np.zeros((m, n)); G[np.arange(m), var] = sgn
    for _ in range(3):
        d = 10.0 ** rs.uniform(-8, 8, m)
        rx, rs_, rz, ry = rs.randn(n), rs.randn(m), rs.randn(m), rs.randn(e)
        mod = qm.kkt_solve(Q, A, hl, hu, d, rx, rs_, rz, ry)
        ref = dense_kkt.solve(Q, G, A, d, rx, rs_, rz, ry)
        for k in (0, 2) + ((3,) if e else ()):
            assert dense_kkt.rel(mod[k], ref[k]) < 1e-6, k


def test_model_with_diagonal_q_matches_box_model():
    from tests.box_util import random_box
    bx = random_box(4, 3, 15, 4, "both")
    for i in range(3):
        a = qm.solve_one(np.diag(bx["q"][i]), bx["p"][i], bx["A"][i], bx["b"][i], bx["lb"][i], bx["ub"][i])
        d = bm.solve_one(bx["q"][i], bx["p"][i], bx["A"][i], bx["b"][i], bx["lb"][i], bx["ub"][i])
        assert a["iters"] == d["iters"] and rel_rows(a["x"], d["x"]).max() < 1e-12


def test_model_factor_pieces():
    """L diag(I, -I) L' reproduces [H A'; A 0]."""
    rs = np.random.RandomState(2)
    n, e = 12, 3
    Q = random_boxq(1, 1, n, 1, "both")["Q"][0]
    A = rs.randn(e, n)
    var, sgn = bm.rows(n, True, True)
    s = qm._SysQ(Q, A, var, sgn, 10.0 ** rs.uniform(-8, 8, 2 * n))
    L = np.block([[s.L11, np.zeros((n, e))], [s.L21, s.L22]])
    K = np.block([[s.H, A.T], [A, np.zeros((e, e))]])
    assert np.abs(L @ np.diag(np.r_[np.ones(n), -np.ones(e)]) @ L.T - K).max() <= 1e-8 * np.abs(K).max()


def test_shape_errors():
    from qpth_b200.box import check_box_shapes
    Q, p = torch.zeros(3, 5, 5), torch.zeros(3, 5)
    lb = torch.zeros(5)
    e = torch.Tensor()
    assert check_box_shapes(Q, p, e, e, lb, None, dense_Q=True) == (3, 5, 0)
    assert check_box_shapes(Q[0], p, e, e, lb, None, dense_Q=True) == (3, 5, 0)
    with pytest.raises(RuntimeError, match="trailing dimensions"):
        check_box_shapes(torch.zeros(3, 5, 4), p, e, e, lb, None, dense_Q=True)
    with pytest.raises(RuntimeError, match="batch size"):
        check_box_shapes(torch.zeros(2, 5, 5), p, e, e, lb, None, dense_Q=True)
    with pytest.raises(RuntimeError, match="Unexpected number of dimensions"):
        check_box_shapes(torch.zeros(5), p, e, e, lb, None, dense_Q=True)
    with pytest.raises(ValueError):
        check_box_shapes(Q, p, e, e, None, None, dense_Q=True)


# ---- the plan ---------------------------------------------------------------------------------------------------------
def _plan(n, e, hl, hu):
    from qpth_b200 import _lib
    p = _lib.BoxQPlan()
    rc = _lib.load().qpb200_boxq_plan_init(n, e, int(hl), int(hu), ctypes.byref(p))
    return rc, p


def test_plan_grid():
    for n in (1, 7, 8, 9, 31, 64, 100, 127, 128, 150, 184, 192, 200, 256, 300):
        for e in (0, 1, 7, 8, 13, 40, 64, 128):
            for hl, hu in ((1, 0), (0, 1), (1, 1)):
                rc, p = _plan(n, e, hl, hu)
                assert rc == 0
                order = ((n + 7) // 8 + (e + 7) // 8) * 8
                assert (p.order, p.threads, p.nineq) == (order, 256, (hl + hu) * n)
                assert p.ok == int(order <= 256 and p.smem_bytes <= 232448)
    assert _plan(10, 0, 0, 0)[0] == 2          # QPB200_ERR_NO_CONSTRAINTS
    assert _plan(0, 1, 1, 1)[0] == 1


@pytest.mark.parametrize("n,e,sides", LARGEST)
def test_plan_largest_shape_and_the_next(n, e, sides):
    hl, hu = _sides(sides)
    rc, p = _plan(n, e, hl, hu)
    assert rc == 0 and p.ok == 1
    slack = 232448 - p.smem_bytes
    assert 0 <= slack < 20000, slack            # shared memory binds, not the 256 rows of the sweeps
    assert _plan(n + 8, e, hl, hu)[1].ok == 0
    assert _plan(n + 1, e, hl, hu)[1].ok == 0


def test_header_and_signatures_export_the_entry_points():
    from qpth_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "qpth_b200.h")).read()
    for name in ("qpb200_boxq_plan_init", "qpb200_boxq_forward", "qpb200_boxq_backward_duals", "qpb200_boxq_jvp",
                 "qpb200_boxq_solve_kkt"):
        assert re.search(r"\b%s\(" % name, hdr), name
        assert name in _lib.SIGNATURES
        if os.path.exists(_lib.LIB_PATH):
            assert hasattr(_lib.load(), name)
    fields = [f for f, _ in _lib.BoxQPlan._fields_]
    assert fields == ["nz", "neq", "neq_pad", "nineq", "has_lb", "has_ub", "order", "threads", "smem_bytes", "ok"]
