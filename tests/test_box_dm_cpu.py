"""Box QPs with neq_pad > 128 without a GPU: the plans of the distributed-M kernels (csrc/qp_box.cu k_box_*_dm), the
index-level model of their factorization and sweeps (oracle/dm_model.py), the 9x9 sudoku generator, and the real
reference's sudoku fixtures against the box model."""
import ctypes
import os

import numpy as np
import pytest

from oracle import box_model as bm, dm_model
from oracle.box_cases import dense_problem
from oracle.box_sudoku_cases import SUDOKU_BOX_CASES, puzzles, sudoku_constraints, sudoku_matrix
from oracle.cases import checksum, proj
from tests.parity import rel_rows
from tests.test_box_cpu import _batched

MAX_SMEM = 232448


def _plan(n, e, lb, ub):
    from qpth_b200 import _lib
    return _lib.box_plan_for(n, e, lb, ub)


@pytest.fixture
def no_knob(monkeypatch):
    monkeypatch.delenv("QPB200_BOX_CLUSTER", raising=False)


# ---- plans -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,e,lb,ub", [(729, 249, True, False), (729, 249, True, True), (1000, 249, True, False)])
def test_sudoku_shapes_get_the_distributed_kernels(no_knob, n, e, lb, ub):
    p = _plan(n, e, lb, ub)
    assert p.ok == 0 and p.neq_pad > 128
    assert p.cl_ctas in (2, 4, 8) and 0 < p.cl_smem_bytes <= MAX_SMEM
    assert p.cl_slice * p.cl_ctas >= n


def test_smallest_cluster_that_fits(no_knob):
    from qpth_b200 import _lib
    p = _plan(729, 249, True, False)
    assert p.cl_ctas == 4                                    # the 9x9 sudoku layer: half of M does not fit one CTA
    q = _lib.BoxPlan()
    os.environ["QPB200_BOX_CLUSTER"] = "2"
    try:
        assert _lib.load().qpb200_box_plan_init(729, 249, 1, 0, ctypes.byref(q)) == 0
    finally:
        del os.environ["QPB200_BOX_CLUSTER"]
    assert q.cl_ctas == 4                                    # the knob's size does not fit: the normal choice


def test_pinned_shapes_keep_their_path(no_knob):
    from qpth_b200 import _lib
    lib = _lib.load()
    assert _plan(150, 130, False, True).cl_ctas == 0          # dense order 288: the dense kernels
    for n, e in ((5000, 200), (2048, 128)):
        assert lib.qpb200_box_plan_init(n, e, 1, 1, ctypes.byref(_lib.BoxPlan())) == 4, (n, e)


def test_dense_order_threshold(no_knob):
    """neq_pad > 128: these kernels past dense order 384 (measured on an H100: parity at 384, 2.2x faster at 504)"""
    from qpth_b200 import _lib
    for n, e, lb, ub in ((150, 130, False, True), (200, 180, True, False), (300, 200, True, False),
                         (160, 136, True, True), (600, 249, True, False)):
        d = _lib.Plan()
        assert _lib.load().qpb200_plan_init(n, (int(lb) + int(ub)) * n, e, ctypes.byref(d)) == 0
        assert (_plan(n, e, lb, ub).cl_ctas != 0) == (d.ms_pad > 384), (n, e, d.ms_pad)


def test_knob_forces_the_family_on_small_shapes(monkeypatch):
    for n, e, lb, ub in ((150, 130, False, True), (160, 136, True, True), (200, 180, True, False)):
        for C in (2, 4, 8):
            monkeypatch.setenv("QPB200_BOX_CLUSTER", str(C))
            p = _plan(n, e, lb, ub)
            assert p.cl_ctas == C and p.cl_slice == -(-n // C) and p.cl_smem_bytes <= MAX_SMEM


# ---- the distributed factorization ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,C", [(136, 2), (136, 4), (136, 8), (256, 4), (40, 8), (16, 8), (24, 4)])
def test_distributed_factor_model_solves(n, C):
    """n / 8 < C: ranks without block rows (and, in the kernels, without variables) take part in every barrier"""
    rs = np.random.RandomState(n + C)
    X = rs.randn(n, n + 5)
    M = X @ X.T / n + np.diag(rs.rand(n))
    h, h2 = rs.randn(n), rs.randn(n)
    w, w2 = dm_model.solve(M, h, C, refactor_rhs=h2)
    for v, rhs in ((w, h), (w2, h2)):
        ref = np.linalg.solve(M, rhs)
        assert np.abs(v - ref).max() <= 1e-10 * np.abs(ref).max()


def test_distributed_layout_covers_the_staircase():
    """every element (r, c <= 8 (r >> 3) + 7) of the staircase has one owner and one local slot, and the ranks'
    storage adds up to the staircase's"""
    from oracle import pf_model
    for nts, C in ((17, 2), (32, 4), (31, 8), (3, 8)):
        total = 0
        for r in range(C):
            R = dm_model.Rank(C, r, nts)
            slots = {R.at(8 * i + rr, c) for i in R.own() for rr in range(8) for c in range(8 * i + 8)}
            assert len(slots) == 8 * sum(8 * i + 8 for i in R.own())
            total += R.S.size
        assert total == pf_model.elems(nts)
        assert dm_model.stair_doubles(nts, C) >= pf_model.elems(nts) / C


# ---- the sudoku generator and the reference's fixtures -----------------------------------------------------------------
def test_sudoku_matrix():
    for n, shape in ((2, (40, 64)), (3, (249, 729))):
        A = sudoku_matrix(n)
        assert A.shape == shape and np.linalg.matrix_rank(A) == shape[0]
        assert np.linalg.matrix_rank(sudoku_constraints(n)) == shape[0]   # nothing independent was dropped
    P, Z = puzzles(91, 3)
    A = sudoku_matrix(3)
    assert np.abs(A @ Z.T - 1.0).max() == 0.0 and ((P == 0) | (Z == 1)).all()


def load_sudoku(name, golden_dir):
    bx = SUDOKU_BOX_CASES[name]()
    gold = dict(np.load(os.path.join(golden_dir, name + ".npz")))
    cs = checksum(dense_problem(bx))
    assert abs(cs - float(gold["input_checksum"])) <= 1e-9 * abs(cs), "golden inputs no longer reproduce from the seed"
    return bx, gold


# The model and the reference stop at different last iterates, as at box_wide: on box_sudoku9_init z* agrees to 1e-9
# and the gradients to 1.5e-5, while the reference moves by 2e-13 under a 1e-15 perturbation of its inputs (sens_*).
# The bounds are box_wide's (tests/test_box_cluster_cpu.py), about 2x above what was measured.
# The trained layer (box_sudoku9: p = -puzzle, an LP-like problem with many degenerate bounds) has no unique duals:
# the reference's own lam, nus, dh, db and dA move by 30 % to 70 % under that perturbation (sens_dh, sens_db,
# sens_dA_proj), so only z*, the slacks, dq and dp are compared where sens_dh says so.
SUDOKU_ZTOL, SUDOKU_GTOL = 2.5e-8, 3e-5
UNDETERMINED = 1e-3


def check_sudoku_golden(out, gold, bx, ztol=SUDOKU_ZTOL, gtol=SUDOKU_GTOL):
    n = np.asarray(bx["q"]).shape[-1]
    duals = float(gold["sens_dh"]) < UNDETERMINED
    for k in ("zhat", "slacks") + (("lam", "nus") if duals else ()):
        assert rel_rows(out[k], gold[k]).max() <= ztol, k
    g = out["grads"]
    ref = dict(dq=gold["dq"], dp=gold["dp"])
    if duals:
        ref.update(db=gold["db"], dlb=-gold["dh"][..., :n])
    for k, v in ref.items():
        assert g[k].shape == v.shape, k
        assert rel_rows(g[k], v, floor=1e-4).max() <= gtol, k
    if duals:
        assert rel_rows(g["dA"] @ proj(n), gold["dA_proj"], floor=1e-4).max() <= gtol


@pytest.mark.parametrize("name", list(SUDOKU_BOX_CASES))
def test_model_matches_sudoku_reference_golden(name, golden_dir):
    bx, gold = load_sudoku(name, golden_dir)
    if name == "box_sudoku9":
        assert float(gold["sens_dh"]) > UNDETERMINED and float(gold["sens_zhat"]) < 1e-7
    B = np.asarray(bx["p"]).shape[0]
    t = _batched(bx, B)
    out = bm.qp_solve(t["q"], t["p"], t["A"], t["b"], t["lb"], t["ub"], dl=bx["dl"], stall_tol=1e-6, tie=1.5)
    g = out["grads"]
    for k in ("dq", "dlb", "dA", "db"):      # shared in the cases
        g[k] = g[k].mean(0)
    check_sudoku_golden(dict(out, grads=g), gold, bx)
