"""BoxQPFunction's Jacobians of (z, lam, nu) with respect to (p, lb, ub, b) without a GPU.

- The numpy model of the kernel's blocked algorithm (tests/box_jacobian_models.blocked_box_jacobian: H^-1, the
  product-form factor of M = A H^-1 A', 8-column block sweeps, the lb / ub columns and lam rows as diagonal scalings)
  against the dense model on the dense equivalent, and the identities J_z,p = J_z,p', J_z,b = -J_nu,p',
  J_nu,b = J_nu,b', J_z,lb = -J_z,p diag(d_lb), J_z,ub = -J_z,p diag(d_ub).
- The host logic of jacobian() / solve_box_jacobian with the C calls replaced by the dense model: block order and
  shapes, dtype, every error, and the three dispatch branches (kernel, column path, dense fallback with h -> lb, ub).
- qpb200_box_jacobian_smem over the box-family entries, and the argument checks of qpb200_box_jacobian (both return
  before any device work).
- The ptxas report of k_box_jacobian: registers, no stack, no spills.
"""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from tests import box_jacobian_models as bm
from tests import jacobian_models as jm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (nz, neq, sides): odd nz, neq not a multiple of 8, neq = 0, a full tile, each side alone and both
SHAPES = [(13, 5, "both"), (9, 0, "lb"), (16, 8, "ub"), (21, 11, "both"), (21, 11, "lb"), (30, 17, "ub"),
          (7, 0, "both")]


def _flags(sides):
    return sides != "ub", sides != "lb"


def _case(shape, seed, spread):
    n, e, sides = shape
    has_lb, has_ub = _flags(sides)
    nlb = n if has_lb else 0
    m = nlb + (n if has_ub else 0)
    rs = np.random.RandomState(seed)
    q = rs.uniform(0.5, 2.0, n)
    A = rs.randn(e, n) / np.sqrt(n) if e else None
    if spread:       # d = lam / s over 1e-8 .. 1e8
        lam, s = 10 ** rs.uniform(-4, 4, m), 10 ** rs.uniform(-4, 4, m)
    else:
        lam, s = rs.uniform(0.1, 10, m), rs.uniform(0.1, 10, m)
    return q, A, lam, s, nlb, has_ub


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_blocked_model_matches_dense(shape, spread):
    n, e, _ = shape
    q, A, lam, s, nlb, has_ub = _case(shape, n + e, spread)
    m = lam.shape[0]
    Jr = bm.dense_box_jacobian_refined(np.diag(q), A, lam, s, nlb, has_ub)
    Jb = bm.blocked_box_jacobian(q, A, lam, s, nlb, has_ub)
    C = n * (1 + bool(nlb) + has_ub) + e
    assert Jb.shape == Jr.shape == (n + m + e, C)
    _check_against_refined(Jb, Jr, n, m, e, nlb, has_ub, jm.clamped_d(lam, s), spread)
    if not spread:
        assert np.abs(bm.dense_box_jacobian(np.diag(q), A, lam, s, nlb, has_ub) - Jr).max() < 1e-13 * np.abs(Jr).max()


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_bordered_model_matches_dense(shape, spread):
    """The dense-Q kernel's arithmetic (bordered factor, sweeps with the trailing block negated) on a dense SPD Q."""
    n, e, _ = shape
    q, A, lam, s, nlb, has_ub = _case(shape, n + e, spread)
    m = lam.shape[0]
    F = np.random.RandomState(n + 2 * e).randn(n, n)
    Q = F @ F.T / n + 0.5 * np.eye(n)
    Jr = bm.dense_box_jacobian_refined(Q, A, lam, s, nlb, has_ub)
    Jq = bm.bordered_box_jacobian(Q, A, lam, s, nlb, has_ub)
    assert Jq.shape == Jr.shape
    _check_against_refined(Jq, Jr, n, m, e, nlb, has_ub, jm.clamped_d(lam, s), spread)


def _check_against_refined(J, Jr, n, m, e, nlb, has_ub, d, spread):
    """Against the dense model with its inverse refined on long-double residuals. With d spread over 1e-8 .. 1e8 K is
    conditioned so that fp64 arithmetic in any order leaves ~1e-11 of max|J| (the refined reference converges; both
    blocked models land there), hence 1e-10 for those cases and 1e-12 otherwise."""
    scale = np.abs(Jr).max()
    tol = 1e-10 if spread else 1e-12
    assert np.abs(J - Jr).max() < tol * scale, np.abs(J - Jr).max() / scale
    assert bm.identity_residuals(J, n, m, e, nlb, has_ub, d) < 1e-12 * scale


def test_dense_model_is_the_jvp():
    """A column of the dense box model is the JVP of that input's unit tangent on the dense equivalent
    (tests/jvp_models.jvp_dense, dh = [-dlb; dub])."""
    from tests import jvp_models as jvm
    n, e = 9, 3
    q, A, lam, s, nlb, has_ub = _case((n, e, "both"), 3, False)
    m = lam.shape[0]
    rs = np.random.RandomState(4)
    z, nu = rs.randn(n), rs.randn(e)
    J = bm.dense_box_jacobian(np.diag(q), A, lam, s, nlb, has_ub)
    G = bm.dense_G(n, nlb, has_ub)
    for c0, k, mk in ((0, n, lambda u: {"p": u}), (n, n, lambda u: {"h": np.concatenate([-u, np.zeros(n)])}),
                      (2 * n, n, lambda u: {"h": np.concatenate([np.zeros(n), u])}), (3 * n, e, lambda u: {"b": u})):
        for j in range(k):
            u = np.zeros(k)
            u[j] = 1.0
            ref = np.concatenate(jvm.jvp_dense(np.diag(q), G, A, z, lam, s, nu, mk(u)))
            assert np.abs(J[:, c0 + j] - ref).max() < 1e-12 * np.abs(J).max()
    assert J.shape == (n + m + e, 3 * n + e)


# ---- host logic with the C calls replaced by the dense model ----------------------------------------------------------

def _state(B, shape, seed, dense_Q=False):
    """A _BoxSolved on the CPU with the real plan of the shape, and the dense model of every QP."""
    from qpth_b200 import _lib
    from qpth_b200.box import _BoxSolved
    n, e, sides = shape
    st = _BoxSolved()
    st.plan = (_lib.boxq_plan_for if dense_Q else _lib.box_plan_for)(n, e, *_flags(sides))
    st.nBatch, st.device, st.dense, st.dense_Q = B, torch.device("cpu"), None, dense_Q
    cases = [_case(shape, seed + i, False) for i in range(B)]
    st.lam = torch.tensor(np.stack([c[2] for c in cases]))
    st.slacks = torch.tensor(np.stack([c[3] for c in cases]))
    st.model = np.stack([bm.dense_box_jacobian(np.diag(c[0]), c[1], c[2], c[3], c[4], c[5]) for c in cases])
    return st


def _select(J, n, m, e, nlb, has_ub, rows, cols):
    off = np.cumsum((0, n, m, e))
    ri = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(3) if (rows >> i) & 1])
    widths = [n, n if nlb else 0, n if has_ub else 0, e]
    co = np.cumsum([0] + widths)
    ci = np.concatenate([np.arange(co[k], co[k + 1]) for k in range(4) if (cols >> k) & 1])
    return J[:, ri][:, :, ci]


@pytest.fixture
def dense_lib(monkeypatch):
    """solve_box_jacobian's three branches on the dense model: the kernel writes the selected blocks, solve_box_jvp
    returns the columns, and the dense path's solve_jacobian gives the [p, h, b] columns of the dense equivalent."""
    from qpth_b200 import box
    from qpth_b200 import qp as _qp
    calls = {"kernel": 0, "jvp": 0, "dense": 0, "covered": True, "dense_Q": []}

    def kernel(st, rows, cols, J):
        calls["kernel"] += 1
        p = st.plan
        J.copy_(torch.tensor(_select(st.model, p.nz, p.nineq, p.neq, p.nz if p.has_lb else 0, p.has_ub, rows, cols)))

    def jvp(st, tans):
        calls["jvp"] += 1
        p = st.plan
        n, m, e = p.nz, p.nineq, p.neq
        widths = [n, n if p.has_lb else 0, n if p.has_ub else 0, e]
        co = np.cumsum([0] + widths)
        t = np.zeros(co[-1])
        for k, slot in enumerate((1, 4, 5, 3)):
            if tans[slot] is not None:
                assert tans[slot].dim() == 1          # an un-batched unit tangent: one call gives the column of every QP
                t[co[k]:co[k + 1]] = tans[slot].numpy()
        out = torch.tensor(st.model @ t)
        return out[:, :n], out[:, n:n + m], (out[:, n + m:] if e else None)

    def dense_solve(dst, rows, cols):
        calls["dense"] += 1
        n, m, e, nlb = dst.n, dst.m, dst.e, dst.nlb
        Jm = dst.model                                # [p, lb, ub, b] -> [p, h, b], h = [-lb; ub]
        h = np.concatenate(([-Jm[:, :, n:n + nlb]] if nlb else []) + ([Jm[:, :, n + nlb:n + m]] if m > nlb else []),
                           axis=2)
        Jh = np.concatenate([Jm[:, :, :n], h, Jm[:, :, n + m:]], axis=2)
        off = np.cumsum((0, n, m, e))
        ri = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(3) if (rows >> i) & 1])
        ci = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(3) if (cols >> i) & 1])
        return torch.tensor(Jh[:, ri][:, :, ci])

    monkeypatch.setattr(box, "_box_jacobian_kernel", kernel)
    monkeypatch.setattr(box, "solve_box_jvp", jvp)
    def covered(plan, dense_Q=False):
        calls["dense_Q"].append(dense_Q)
        return calls["covered"]

    monkeypatch.setattr(box, "box_jacobian_covered", covered)
    monkeypatch.setattr(_qp, "solve_jacobian", dense_solve)
    return calls


@pytest.fixture(autouse=True)
def _model_slot(monkeypatch):
    """Give _BoxSolved a `model` slot for these tests (the dense model of each QP)."""
    from qpth_b200 import box

    class _ModelSolved(box._BoxSolved):
        __slots__ = ("model",)

    monkeypatch.setattr(box, "_BoxSolved", _ModelSolved)


MASKS = [(1, 1), (7, 15), (2, 8), (5, 2), (3, 6), (1, 4), (7, 9)]


@pytest.mark.parametrize("path", ["kernel", "columns"])
@pytest.mark.parametrize("rows,cols", MASKS)
def test_solve_box_jacobian_order(dense_lib, path, rows, cols):
    from qpth_b200.box import solve_box_jacobian
    dense_lib["covered"] = path == "kernel"
    n, e = 11, 3
    st = _state(3, (n, e, "both"), 1)
    J = solve_box_jacobian(st, rows, cols, n)
    ref = _select(st.model, n, 2 * n, e, n, True, rows, cols)
    assert J.dtype == torch.float64 and tuple(J.shape) == ref.shape
    assert np.abs(J.numpy() - ref).max() < 1e-13
    ncols = sum((n, n, n, e)[k] for k in range(4) if (cols >> k) & 1)
    assert (dense_lib["kernel"], dense_lib["jvp"]) == ((1, 0) if path == "kernel" else (0, ncols))


@pytest.mark.parametrize("covered", [True, False])
def test_dense_Q_dispatch(dense_lib, covered):
    """A dense Q takes qpb200_boxq_jacobian where it covers the plan, else one JVP per column."""
    from qpth_b200.box import solve_box_jacobian
    dense_lib["covered"] = covered
    st = _state(2, (8, 2, "lb"), 2, dense_Q=True)
    J = solve_box_jacobian(st, 7, 1 | 2 | 8, 8)
    assert (dense_lib["kernel"], dense_lib["jvp"]) == ((1, 0) if covered else (0, 18))
    assert dense_lib["dense_Q"] == [True]
    assert np.abs(J.numpy() - _select(st.model, 8, 8, 2, 8, False, 7, 11)).max() < 1e-13


@pytest.mark.parametrize("sides", ["both", "lb", "ub"])
@pytest.mark.parametrize("rows,cols", [(7, 15), (1, 4), (3, 2), (5, 9)])
def test_dense_fallback_maps_h(dense_lib, sides, rows, cols):
    """The dense fallback: J_lb = -J_h[:, :, :nlb], J_ub = J_h[:, :, nlb:], lam rows as they are."""
    from qpth_b200.box import solve_box_jacobian
    n, e = 10, 3
    has_lb, has_ub = _flags(sides)
    cols &= 1 | (2 if has_lb else 0) | (4 if has_ub else 0) | 8
    if not cols:
        cols = 1
    ref_state = _state(2, (n, e, sides), 3)

    class _Dense:
        pass

    dst = _Dense()
    dst.plan = type("P", (), dict(nz=n, nineq=ref_state.plan.nineq, neq=e))()
    dst.n, dst.m, dst.e, dst.nlb, dst.model = n, ref_state.plan.nineq, e, n if has_lb else 0, ref_state.model
    st = ref_state
    st.dense, st.plan = (dst, True), dst.plan
    J = solve_box_jacobian(st, rows, cols, dst.nlb)
    ref = _select(ref_state.model, n, dst.m, e, dst.nlb, has_ub, rows, cols)
    assert dense_lib["dense"] == 1 and dense_lib["kernel"] == 0 and dense_lib["jvp"] == 0
    assert tuple(J.shape) == ref.shape and np.abs(J.numpy() - ref).max() < 1e-13


@pytest.mark.parametrize("duals", [False, True])
def test_box_jacobian_of_blocks(dense_lib, duals):
    from qpth_b200.box import box_jacobian_of
    n, e = 10, 2
    st = _state(2, (n, e, "both"), 4)
    out = box_jacobian_of(st, (torch.device("cpu"), torch.float32), (n, True), ("b", "ub", "p"), duals)
    assert list(out) == ["b", "ub", "p"]
    R = n + 2 * n + e if duals else n
    assert tuple(out["p"].shape) == (2, R, n) and tuple(out["ub"].shape) == (2, R, n)
    assert tuple(out["b"].shape) == (2, R, e)
    assert out["p"].dtype == torch.float32 and not out["p"].requires_grad
    full = st.model[:, :R]
    tol = 1e-5 * np.abs(full).max()
    assert np.abs(out["p"].double().numpy() - full[:, :, :n]).max() < tol
    assert np.abs(out["ub"].double().numpy() - full[:, :, 2 * n:3 * n]).max() < tol
    assert np.abs(out["b"].double().numpy() - full[:, :, 3 * n:]).max() < tol
    every = box_jacobian_of(st, (torch.device("cpu"), torch.float64), (n, True), None, duals)
    assert list(every) == ["p", "lb", "ub", "b"]


def test_box_jacobian_of_defaults_without_b(dense_lib):
    from qpth_b200.box import box_jacobian_of
    st = _state(1, (6, 0, "ub"), 5)
    cpu = (torch.device("cpu"), torch.float64)
    out = box_jacobian_of(st, cpu, (0, True), None, True)
    assert list(out) == ["p", "ub"] and tuple(out["ub"].shape) == (1, 12, 6)    # duals without equality rows


def test_box_jacobian_errors(dense_lib):
    from qpth_b200.box import box_jacobian_of
    st = _state(1, (6, 0, "ub"), 6)
    cpu = (torch.device("cpu"), torch.float64)
    with pytest.raises(ValueError, match="equality"):
        box_jacobian_of(st, cpu, (0, True), ("p", "b"), False)
    with pytest.raises(ValueError, match="lb side"):
        box_jacobian_of(st, cpu, (0, True), ("lb",), False)
    for nm in ("q", "Q", "A"):
        with pytest.raises(ValueError, match=r"J_\.,q = J_\.,p diag\(z\)"):
            box_jacobian_of(st, cpu, (0, True), (nm,), False)
    with pytest.raises(ValueError, match="'h'"):
        box_jacobian_of(st, cpu, (0, True), ("h",), False)
    with pytest.raises(ValueError):
        box_jacobian_of(st, cpu, (0, True), (), False)
    with pytest.raises(RuntimeError, match="forward"):
        box_jacobian_of(None, cpu, (0, True), ("p",), False)


def test_function_attribute():
    from qpth_b200 import BoxQPFunction
    with pytest.raises(RuntimeError, match="forward"):
        BoxQPFunction().jacobian()
    with pytest.raises(RuntimeError, match="forward"):
        BoxQPFunction(dense_Q=True).jacobian(wrt="p")


def test_pending_checks_are_flushed(dense_lib, monkeypatch):
    from qpth_b200 import qp as _qp
    from qpth_b200.box import solve_box_jacobian
    seen = []
    monkeypatch.setattr(_qp, "_pending", [object()])
    monkeypatch.setattr(_qp, "flush_checks", lambda wait=True: seen.append(wait))
    solve_box_jacobian(_state(1, (5, 0, "lb"), 7), 1, 1, 5)
    assert seen == [False]


# ---- C ABI: coverage and argument checks (no device work) -----------------------------------------------------------

def _box_smem(plan):
    from qpth_b200 import _lib
    out = ctypes.c_int64(-1)
    assert _lib.load().qpb200_box_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)) == 0
    return out.value


# Coverage per box-family entry: every OneCta and Cluster entry and the distributed-M entries whose M and one warp's
# buffers fit (neq_pad up to 25 tiles at nz 249); not dm2_full and past (neq_pad 232..352: M alone exceeds 227 KB),
# nor the eight-CTA slices past about 3300 variables (one warp's nz_pad x 8 buffer)
UNCOVERED_ENTRIES = {"dm2_full", "dm4_mid", "dm4_sudoku", "dm4_full", "dm8_full", "dm8_slice", "cl8_mid",
                     "cl8_mid_box", "cl8_widest", "cl8_widest_lb"}


def test_box_jacobian_smem_entries():
    from qpth_b200 import _lib
    from tests.box_families import ENTRIES, knob, sides_flags
    for name, ent in ENTRIES.items():
        n, e, sides = ent["shape"]
        with knob(ent["knob"]):
            plan = _lib.box_plan_for(n, e, *sides_flags(sides))
        smem = _box_smem(plan)
        assert (smem > 0) == (name not in UNCOVERED_ENTRIES), (name, smem)
        assert smem <= 232448 - 1024


def test_box_jacobian_smem_edges():
    """The widest covered nz (one warp's buffers beside H^-1 and d) and the most equality rows at nz = neq."""
    from qpth_b200 import _lib
    cov = lambda n, e, sides: _box_smem(_lib.box_plan_for(n, e, *_flags(sides))) > 0
    assert cov(2616, 0, "both") and not cov(2617, 0, "both")
    assert cov(2880, 0, "lb") and not cov(2881, 0, "lb")
    most = max(k for k in range(190, 210) if _box_smem(_lib.box_plan_for(k, k, True, False)) > 0)
    assert most == 200 and _box_smem(_lib.box_plan_for(201, 201, True, False)) == 0


def _boxq_smem(plan):
    from qpth_b200 import _lib
    out = ctypes.c_int64(-1)
    assert _lib.load().qpb200_boxq_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)) == 0
    return out.value


def test_boxq_jacobian_smem_entries():
    """Every dense-Q family entry the forward kernels run (plan.ok) is covered. (The kernel needs less shared memory than
    the forward and covers some plans past ok too; BoxQPFunction never reaches it there: those run the dense fallback.)"""
    from tests.boxq_families import ENTRIES, plan_init
    for name, ent in ENTRIES.items():
        rc, plan = plan_init(*ent["shape"])
        assert rc == 0, name
        smem = _boxq_smem(plan)
        assert smem > 0 or not plan.ok, (name, smem)
        assert smem <= 232448


def test_boxq_jacobian_smem_grid():
    """Over a grid of shapes, qpb200_boxq_jacobian covers every plan with ok = 1."""
    from qpth_b200 import _lib
    seen = {True: 0, False: 0}
    for n in list(range(1, 40, 3)) + list(range(40, 220, 11)):
        for e in sorted({0, 1, 7, 8, 9, n // 2, n}):
            for sides in ("lb", "ub", "both"):
                plan = _lib.BoxQPlan()
                rc = _lib.load().qpb200_boxq_plan_init(n, e, *_flags(sides), ctypes.byref(plan))
                if rc:
                    continue
                assert _boxq_smem(plan) > 0 or not plan.ok, (n, e, sides)
                seen[bool(plan.ok)] += 1
    assert seen[True] > 100 and seen[False] > 10


def test_boxq_jacobian_arg_checks():
    from qpth_b200 import _lib
    lib = _lib.load()
    plan = _lib.boxq_plan_for(12, 3, True, True)
    plan0 = _lib.boxq_plan_for(12, 0, True, False)
    big = _lib.BoxQPlan()
    assert lib.qpb200_boxq_plan_init(250, 0, 1, 1, ctypes.byref(big)) == 0 and _boxq_smem(big) == 0
    P = ctypes.c_void_p(16)                                 # never dereferenced: every check returns first
    N = ctypes.c_void_p(0)
    f = lib.qpb200_boxq_jacobian
    ok = lambda pl=plan, B=2, r=7, c=15: (ctypes.byref(pl), B, r, c)
    assert lib.qpb200_boxq_jacobian_smem(None, ctypes.byref(ctypes.c_int64())) == 1
    assert lib.qpb200_boxq_jacobian_smem(ctypes.byref(plan), None) == 1
    for i in (0, 2, 4, 5, 6):                               # Q, A, lam, slacks, J
        args = [P, 0, P, 0, P, P, P]
        args[i] = N
        assert f(*ok(), *args, N) == 1, i
    assert f(None, 2, 7, 15, P, 0, P, 0, P, P, P, N) == 1
    assert f(*ok(B=0), P, 0, P, 0, P, P, P, N) == 1         # nbatch < 1
    assert f(*ok(r=0), P, 0, P, 0, P, P, P, N) == 1         # empty masks
    assert f(*ok(c=0), P, 0, P, 0, P, P, P, N) == 1
    assert f(*ok(r=8), P, 0, P, 0, P, P, P, N) == 1         # unknown bits
    assert f(*ok(c=16), P, 0, P, 0, P, P, P, N) == 1
    assert f(*ok(), P, -1, P, 0, P, P, P, N) == 1           # negative stride
    assert f(*ok(plan0, r=4, c=1), P, 0, N, 0, P, P, P, N) == 1    # nu rows, neq == 0
    assert f(*ok(plan0, r=1, c=8), P, 0, N, 0, P, P, P, N) == 1    # b columns, neq == 0
    assert f(*ok(plan0, r=1, c=4), P, 0, N, 0, P, P, P, N) == 1    # ub columns, no ub side
    assert f(*ok(big, r=1, c=1), P, 0, N, 0, P, P, P, N) == 4      # not covered


def test_box_jacobian_arg_checks():
    from qpth_b200 import _lib
    lib = _lib.load()
    plan = _lib.box_plan_for(12, 3, True, True)
    plan0 = _lib.box_plan_for(12, 0, True, False)
    big = _lib.box_plan_for(7008, 0, True, True)
    P = ctypes.c_void_p(16)                                 # never dereferenced: every check returns first
    N = ctypes.c_void_p(0)
    f = lib.qpb200_box_jacobian
    ok = lambda pl=plan, B=2, r=7, c=15: (ctypes.byref(pl), B, r, c)
    assert lib.qpb200_box_jacobian_smem(None, ctypes.byref(ctypes.c_int64())) == 1
    assert lib.qpb200_box_jacobian_smem(ctypes.byref(plan), None) == 1
    for i in (0, 2, 4, 5, 6):                               # q, A, lam, slacks, J
        args = [P, 0, P, 0, P, P, P]
        args[i] = N
        assert f(*ok(), *args, N) == 1, i
    assert f(None, 2, 7, 15, P, 0, P, 0, P, P, P, N) == 1
    assert f(*ok(B=0), P, 0, P, 0, P, P, P, N) == 1         # nbatch < 1
    assert f(*ok(r=0), P, 0, P, 0, P, P, P, N) == 1         # empty masks
    assert f(*ok(c=0), P, 0, P, 0, P, P, P, N) == 1
    assert f(*ok(r=8), P, 0, P, 0, P, P, P, N) == 1         # unknown bits
    assert f(*ok(c=16), P, 0, P, 0, P, P, P, N) == 1
    assert f(*ok(), P, -1, P, 0, P, P, P, N) == 1           # negative stride
    assert f(*ok(plan0, r=4, c=1), P, 0, N, 0, P, P, P, N) == 1    # nu rows, neq == 0
    assert f(*ok(plan0, r=1, c=8), P, 0, N, 0, P, P, P, N) == 1    # b columns, neq == 0
    assert f(*ok(plan0, r=1, c=4), P, 0, N, 0, P, P, P, N) == 1    # ub columns, no ub side
    assert f(*ok(big, r=1, c=1), P, 0, N, 0, P, P, P, N) == 4      # not covered


# ---- ptxas report ------------------------------------------------------------------------------------------------------
# k_box_jacobian with nvcc 12.9 for sm_90a: registers at most this, and no stack frame or spills in it or its subroutines
BOX_JAC_REGISTERS = 106


def test_box_jacobian_ptxas_report():
    from tests.test_local_memory_cpu import _nvcc, parse_ptxas
    from qpth_b200 import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    (src, defs, tag), = [u for u in build.UNITS if u[0] == "qp_jac.cu"]
    with tempfile.TemporaryDirectory() as tmp:
        cmd = ([nvcc] + build.GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
               + defs + ["-c", "-o", os.path.join(tmp, tag + ".o"), os.path.join(ROOT, "qpth_b200", "csrc", src)])
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    rep = parse_ptxas(r.stderr)
    (entry, funcs), = [(k, v) for k, v in rep.items() if "k_box_jacobian" in k]
    assert all(f[1:] == (0, 0, 0) for f in funcs), funcs
    blocks = r.stderr.split("Compiling entry function")
    (blk,) = [b for b in blocks if "k_box_jacobian" in b.split("\n")[0]]
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", blk)]
    assert regs and max(regs) <= BOX_JAC_REGISTERS, regs


# k_boxq_jacobian with nvcc 12.9 for sm_90a: registers at most this, no stack frame and no spills in the kernel or in the
# subroutines it adds (jac_ssolve_bordered); the factorization's subroutines are the forward's own
BOXQ_JAC_REGISTERS = 114


def test_boxq_jacobian_ptxas_report():
    from tests.test_local_memory_cpu import _nvcc, parse_ptxas
    from qpth_b200 import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    (src, defs, tag), = [u for u in build.UNITS if u[0] == "qp_boxq.cu"]
    with tempfile.TemporaryDirectory() as tmp:
        cmd = ([nvcc] + build.GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
               + defs + ["-c", "-o", os.path.join(tmp, tag + ".o"), os.path.join(ROOT, "qpth_b200", "csrc", src)])
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    rep = parse_ptxas(r.stderr)
    (entry, funcs), = [(k, v) for k, v in rep.items() if "k_boxq_jacobian" in k]
    mine = [f for f in funcs if "k_boxq_jacobian" in f[0] or "jac_ssolve" in f[0]]
    assert mine and all(f[1:] == (0, 0, 0) for f in mine), funcs
    blocks = r.stderr.split("Compiling entry function")
    (blk,) = [b for b in blocks if "k_boxq_jacobian" in b.split("\n")[0]]
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", blk)]
    assert regs and max(regs) <= BOXQ_JAC_REGISTERS, regs
