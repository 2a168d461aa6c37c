"""Box-QP path without a GPU: the numpy model of the kernels' arithmetic (oracle/box_model.py) against the reference's
algorithm on the dense equivalents and against the real reference's fixtures, its KKT directions against the dense
solve, and the host logic of BoxQPFunction (shape checks, plans, the kernel-or-dense choice, the C ABI)."""
import ctypes
import re

import numpy as np
import pytest
import torch

from oracle import box_model as bm, dense_kkt, pdipm_oracle as orc
from oracle.box_cases import BOX_CASES, dense_problem, map_dense_grads
from tests.box_util import GRAD_KEYS, load_box_case, random_box
from tests.parity import GTOL, ZTOL, check_against_golden, rel_rows


def _batched(bx, B):
    out = {}
    for k, nd in (("q", 2), ("p", 2), ("A", 3), ("b", 2), ("lb", 2), ("ub", 2)):
        v = bx[k]
        if v is None or np.asarray(v).size == 0:
            out[k] = v if v is None else np.zeros((B, 0, np.asarray(bx["q"]).shape[-1])) if k == "A" else np.zeros((B, 0))
            continue
        v = np.asarray(v, dtype=np.float64)
        out[k] = v if v.ndim == nd else np.broadcast_to(v, (B,) + v.shape).copy()
    return out


def _model(bx, **opts):
    B = np.asarray(bx["p"]).shape[0]
    t = _batched(bx, B)
    return bm.qp_solve(t["q"], t["p"], t["A"], t["b"], t["lb"], t["ub"], dl=bx["dl"], **opts), t


def _mean_like(g, ref_shape):
    return g.mean(0) if (g is not None and g.ndim == len(ref_shape) + 1) else g


@pytest.mark.parametrize("sides", ["lb", "ub", "both"])
@pytest.mark.parametrize("e", [0, 5])
@pytest.mark.parametrize("shared", [(), ("q", "A", "b", "lb", "ub")])
def test_model_matches_pdipm_oracle_on_dense_equivalent(sides, e, shared):
    bx = random_box(3, 4, 11, e, sides, shared)
    out, t = _model(bx)
    dp = dense_problem(dict(t, dl=bx["dl"]))
    ref = orc.qp_solve(dp["Q"], dp["p"], dp["G"], dp["h"], t["A"], t["b"], bx["dl"], per_qp=True)
    assert rel_rows(out["zhat"], ref["zhat"]).max() < 1e-9
    g = map_dense_grads(ref["grads"], bx)
    for k in GRAD_KEYS:
        if g[k] is None or out["grads"][k] is None:
            assert (g[k] is None or np.asarray(g[k]).size == 0) and out["grads"][k] is None, k
            continue
        assert rel_rows(out["grads"][k], g[k], floor=1e-4).max() < 1e-7, k


def check_box_golden(out, gold, bx, what, ztol=ZTOL, gtol=GTOL):
    """z*, lam, slacks, nus as tests/parity.py checks them; every box gradient against the reference's dense gradients
    mapped to the box inputs (dq = diag(dQ), dlb = -dh_lb, dub = dh_ub), batch means where the input is shared."""
    res = dict(zhat=out["zhat"], lam=out["lam"], slacks=out["slacks"], nus=out["nus"])
    errs = check_against_golden(res, gold, True, ztol=ztol, gtol=gtol, what=what)
    ref = map_dense_grads(tuple(gold.get(k) for k in ("dQ", "dp", "dG", "dh", "dA", "db")), bx)
    for k in GRAD_KEYS:
        g = out["grads"][k]
        if ref[k] is None or np.asarray(ref[k]).size == 0:
            assert g is None or np.asarray(g).size == 0, (what, k)
            continue
        g = _mean_like(g, np.asarray(ref[k]).shape)
        errs[k] = rel_rows(g, ref[k], floor=1e-4).max()
        assert errs[k] <= gtol, (what, k, errs[k])
    return errs


def _shared_like_gold(out, bx):
    """the model runs everything batched: reduce the gradients of shared inputs to their batch mean"""
    g = dict(out["grads"])
    for gk, k in zip(GRAD_KEYS, ("q", "p", "A", "b", "lb", "ub")):
        v = bx[k]
        if g[gk] is not None and v is not None and np.asarray(v).ndim == {"A": 2}.get(k, 1) and np.asarray(v).size:
            g[gk] = g[gk].mean(0)
    return dict(out, grads=g)


@pytest.mark.parametrize("name", list(BOX_CASES))
def test_model_matches_reference_golden(name, golden_dir):
    bx, gold = load_box_case(name, golden_dir)
    out, _ = _model(bx, stall_tol=1e-6, tie=1.5)
    check_box_golden(_shared_like_gold(out, bx), gold, bx, name)


def test_model_kkt_directions_match_dense_solve():
    rs = np.random.RandomState(5)
    for sides in ("lb", "ub", "both"):
        for e in (0, 7):
            n = 13
            q = 0.1 + rs.rand(n)
            A = rs.randn(e, n)
            var, sgn = bm.rows(n, sides != "ub", sides != "lb")
            m = var.shape[0]
            G = np.zeros((m, n)); G[np.arange(m), var] = sgn
            d = 10.0 ** rs.uniform(-8, 8, m)
            rx, rs_, rz, ry = rs.randn(n), rs.randn(m), rs.randn(m), rs.randn(e)
            got = bm.kkt_solve(q, A, sides != "ub", sides != "lb", d, rx, rs_, rz, ry)
            ref = dense_kkt.solve(np.diag(q), G, A, d, rx, rs_, rz, ry)
            for k, (a, r) in enumerate(zip(got, ref[:4])):
                if r is None:
                    continue
                assert dense_kkt.rel(a, r) < (1e-8 if k == 1 else 1e-10), (sides, e, k, dense_kkt.rel(a, r))


# ---- host logic ----------------------------------------------------------------------------------------------------
def _t(*shape):
    return torch.zeros(*shape, dtype=torch.float64) if shape != (0,) else torch.Tensor().double()


def test_shape_errors_before_device():
    from qpth_b200.box import check_box_shapes
    n, e = 6, 2
    ok = dict(q=_t(n), p=_t(3, n), A=_t(e, n), b=_t(e), lb=_t(n), ub=None)
    assert check_box_shapes(**ok) == (3, n, e)
    assert check_box_shapes(**dict(ok, A=_t(0), b=_t(0))) == (3, n, 0)
    assert check_box_shapes(**dict(ok, lb=None, ub=_t(3, n))) == (3, n, e)
    with pytest.raises(ValueError):
        check_box_shapes(**dict(ok, lb=None))
    for bad in (dict(p=_t(3, n + 1)), dict(lb=_t(n + 1)), dict(A=_t(e, n + 1)), dict(b=_t(e + 1)),
                dict(ub=_t(4, n)), dict(b=_t(4, e)), dict(A=_t(0), b=_t(e))):
        with pytest.raises(RuntimeError, match="inconsistent shapes"):
            check_box_shapes(**dict(ok, **bad))
    with pytest.raises(RuntimeError, match="Unexpected number of dimensions"):
        check_box_shapes(**dict(ok, q=_t(1, 3, n)))


def test_exports_declared_in_header_and_signatures():
    import os
    from qpth_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "qpth_b200.h")).read()
    for name in ("qpb200_box_plan_init", "qpb200_box_forward", "qpb200_box_backward", "qpb200_box_solve_kkt"):
        assert re.search(r"\bint " + name + r"\(", hdr), name
        assert name in _lib.SIGNATURES, name
        lib = _lib.load()
        assert hasattr(lib, name)


def test_box_plan_and_kernel_choice():
    from qpth_b200 import _lib
    p = _lib.box_plan_for(64, 40, True, False)       # the sudoku shape
    assert p.ok == 1 and p.neq_pad == 40 and p.nineq == 64 and p.threads == 128
    assert p.smem_bytes <= 76 * 1024                 # three QPs per SM
    assert _lib.box_plan_for(37, 13, True, True).nineq == 74
    assert _lib.box_plan_for(50, 0, False, True).ok == 1
    assert _lib.box_plan_for(150, 130, False, True).ok == 0     # neq_pad > 128: the dense kernels
    assert _lib.box_plan_for(600, 64, True, True).ok == 0       # A beyond shared memory
    bad = _lib.BoxPlan()
    assert _lib.load().qpb200_box_plan_init(10, 2, 0, 0, ctypes.byref(bad)) == 2    # no bound at all
    bad.ok = 0
    assert _lib.load().qpb200_box_solve_kkt(ctypes.byref(bad), 1, None, 0, None, 0, None, None, None, None, None,
                                            None, None, None, None, None) == 4


def test_dense_equivalent_layout():
    from qpth_b200.box import dense_equivalent
    q = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)
    lb = torch.tensor([[-1.0, -2.0, -3.0], [0.0, 0.0, 0.0]], dtype=torch.float64)
    ub = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)
    Q, G, h = dense_equivalent(q, lb, ub)
    assert torch.equal(Q, torch.diag(q))
    assert torch.equal(G, torch.cat([-torch.eye(3), torch.eye(3)]).double())
    assert h.shape == (2, 6) and torch.equal(h[0], torch.tensor([1.0, 2, 3, 1, 2, 3]).double())
    Q, G, h = dense_equivalent(q, None, ub)
    assert G.shape == (3, 3) and torch.equal(h, ub)
