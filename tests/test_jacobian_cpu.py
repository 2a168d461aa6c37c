"""Jacobians of (z, lam, nu) with respect to (p, h, b) without a GPU.

- The numpy model of the kernel's blocked algorithm (tests/jacobian_models.blocked_jacobian: W, L, lam, s in; product-form
  factor of S, 8-column block sweeps) against the dense model (np.linalg.solve of the backward's system with identity
  right-hand sides) within 1e-12, with neq not a multiple of 8 and lam, s spread over 1e-8 .. 1e8; the symmetry
  identities J_z,p = J_z,p', J_lam,h = J_lam,h', J_z,h = -J_lam,p', J_z,b = -J_nu,p', J_lam,b = J_nu,h'.
- The host logic of jacobian() / solve_jacobian with the C call replaced by the dense model: shapes, row and column
  order, dtype, un-batched inputs, every error, and the column-by-column path's assembly.
- qpb200_jacobian_smem over a shape grid and the argument checks of qpb200_jacobian (both return before any device work).
- The ptxas report of csrc/qp_jac.cu: registers, no stack, no spills.
"""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from tests import jacobian_models as jm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(10, 5, 0), (13, 9, 3), (20, 17, 11), (24, 16, 5), (16, 8, 8)]


def _qp(rs, n, m, e):
    M = rs.randn(n, n)
    return M @ M.T / n + 0.5 * np.eye(n), rs.randn(m, n) / np.sqrt(n), rs.randn(e, n) / np.sqrt(n)


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_blocked_model_matches_dense(shape, spread):
    n, m, e = shape
    rs = np.random.RandomState(sum(shape) + spread)
    Q, G, A = _qp(rs, n, m, e)
    if spread:
        lam, s = 10 ** rs.uniform(-8, 8, m), 10 ** rs.uniform(-8, 8, m)
    else:
        lam, s = rs.uniform(0.1, 10, m), rs.uniform(0.1, 10, m)
    Jd = jm.dense_jacobian(Q, G, A, lam, s)
    L, W = jm.factors(Q, G, A)
    assert W.shape == ((e + 7) // 8 * 8 + m, n)
    Jb = jm.blocked_jacobian(L, W, lam, s, e)
    scale = np.abs(Jd).max()
    assert Jb.shape == Jd.shape == (n + m + e, n + m + e)
    assert np.abs(Jb - Jd).max() < 1e-12 * scale
    assert jm.symmetry_residuals(Jd, n, m, e) < 1e-12 * scale
    assert jm.symmetry_residuals(Jb, n, m, e) < 1e-12 * scale


def test_dense_model_is_the_jvp():
    """A column of the dense model is the JVP of that input's unit tangent (tests/jvp_models.jvp_dense)."""
    from tests import jvp_models as jvm
    rs = np.random.RandomState(3)
    n, m, e = 9, 7, 3
    Q, G, A = _qp(rs, n, m, e)
    z, nu, lam, s = rs.randn(n), rs.randn(e), rs.uniform(0.1, 1, m), rs.uniform(0.1, 1, m)
    J = jm.dense_jacobian(Q, G, A, lam, s)
    for name, c0, k in (("p", 0, n), ("h", n, m), ("b", n + m, e)):
        for j in range(k):
            u = np.zeros(k)
            u[j] = 1.0
            ref = np.concatenate(jvm.jvp_dense(Q, G, A, z, lam, s, nu, {name: u}))
            assert np.abs(J[:, c0 + j] - ref).max() < 1e-12 * np.abs(J).max()


# ---- host logic with the C call replaced by the dense model ----------------------------------------------------------

def _state(B, n, m, e, seed, shared=False):
    """A _Solved on the CPU with the real plan of the shape, and the dense model of every QP."""
    from qpth_b200 import _lib
    from qpth_b200.qp import _Solved
    class _DenseSolved(_Solved):
        __slots__ = ("dense",)

    rs = np.random.RandomState(seed)
    st = _DenseSolved()
    st.plan, st.nBatch, st.nsys, st.device, st.reg = _lib.plan_for(n, m, e), B, 1 if shared else B, \
        torch.device("cpu"), False
    mats = [_qp(rs, n, m, e) for _ in range(1 if shared else B)] * (B if shared else 1)
    lam, s = rs.uniform(0.1, 10, (B, m)), rs.uniform(0.1, 10, (B, m))
    st.lam, st.slacks = torch.tensor(lam), torch.tensor(s)
    st.dense = np.stack([jm.dense_jacobian(Q, G, A, lam[i], s[i]) for i, (Q, G, A) in enumerate(mats)])
    return st


def _select(J, n, m, e, rows, cols):
    sizes = (n, m, e)
    off = np.cumsum((0,) + sizes)
    ri = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(3) if (rows >> i) & 1])
    ci = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(3) if (cols >> i) & 1])
    return J[:, ri][:, :, ci]


@pytest.fixture
def dense_lib(monkeypatch):
    """solve_jacobian's two paths on the dense model: the kernel writes the selected blocks, solve_jvp returns the
    columns; `covered` chooses between them."""
    from qpth_b200 import qp
    calls = {"kernel": 0, "jvp": 0, "covered": True}

    def kernel(st, rows, cols, J):
        calls["kernel"] += 1
        J.copy_(torch.tensor(_select(st.dense, st.plan.nz, st.plan.nineq, st.plan.neq, rows, cols)))

    def jvp(st, tans):
        calls["jvp"] += 1
        n, m, e = st.plan.nz, st.plan.nineq, st.plan.neq
        t = np.zeros(n + m + e)
        for k, (c0, c1) in zip((1, 3, 5), ((0, n), (n, n + m), (n + m, n + m + e))):
            if tans[k] is not None:
                assert tans[k].dim() == 1          # an un-batched unit tangent: one call gives the column of every QP
                t[c0:c1] = tans[k].numpy()
        out = torch.tensor(st.dense @ t)
        return out[:, :n], out[:, n:n + m], (out[:, n + m:] if e else None)

    monkeypatch.setattr(qp, "_jacobian_kernel", kernel)
    monkeypatch.setattr(qp, "solve_jvp", jvp)
    monkeypatch.setattr(qp, "jacobian_covered", lambda plan: calls["covered"])
    return calls


@pytest.mark.parametrize("covered", [True, False])
@pytest.mark.parametrize("rows,cols", [(1, 1), (7, 7), (2, 4), (5, 2), (3, 6)])
def test_solve_jacobian_order(dense_lib, covered, rows, cols):
    from qpth_b200.qp import solve_jacobian
    dense_lib["covered"] = covered
    n, m, e = 11, 9, 3
    st = _state(3, n, m, e, 1)
    J = solve_jacobian(st, rows, cols)
    ref = _select(st.dense, n, m, e, rows, cols)
    assert J.dtype == torch.float64 and tuple(J.shape) == ref.shape
    assert np.abs(J.numpy() - ref).max() < 1e-13
    ncols = sum((n, m, e)[i] for i in range(3) if (cols >> i) & 1)
    assert (dense_lib["kernel"], dense_lib["jvp"]) == ((1, 0) if covered else (0, ncols))


def test_regularised_state_takes_the_columns(dense_lib):
    from qpth_b200.qp import solve_jacobian
    st = _state(2, 8, 6, 0, 2)
    st.reg = True
    solve_jacobian(st, 3, 3)
    assert dense_lib["kernel"] == 0 and dense_lib["jvp"] == 14


@pytest.mark.parametrize("duals", [False, True])
def test_jacobian_of_blocks(dense_lib, duals):
    from qpth_b200.qp import jacobian_of
    n, m, e = 10, 7, 2
    st = _state(2, n, m, e, 3, shared=True)
    out = jacobian_of(st, (torch.device("cpu"), torch.float32), ("b", "p"), duals)
    assert list(out) == ["b", "p"]
    R = n + m + e if duals else n
    assert tuple(out["p"].shape) == (2, R, n) and tuple(out["b"].shape) == (2, R, e)
    assert out["p"].dtype == torch.float32 and not out["p"].requires_grad
    full = st.dense[:, :R]
    assert np.abs(out["p"].double().numpy() - full[:, :, :n]).max() < 1e-5 * np.abs(full).max()
    assert np.abs(out["b"].double().numpy() - full[:, :, n + m:]).max() < 1e-5 * np.abs(full).max()
    # shared Q, G, A: the QPs differ only through lam and s, and each gets its own Jacobian
    assert not np.allclose(out["p"][0].numpy(), out["p"][1].numpy())


def test_jacobian_errors(dense_lib):
    from qpth_b200.qp import jacobian_of
    st = _state(1, 6, 4, 0, 4)
    cpu = (torch.device("cpu"), torch.float64)
    with pytest.raises(ValueError, match="equality"):
        jacobian_of(st, cpu, ("p", "b"), False)
    with pytest.raises(ValueError, match="'Q'"):
        jacobian_of(st, cpu, ("Q",), False)
    with pytest.raises(ValueError):
        jacobian_of(st, cpu, (), False)
    with pytest.raises(RuntimeError, match="forward"):
        jacobian_of(None, cpu, ("p",), False)
    assert tuple(jacobian_of(st, cpu, "h", True)["h"].shape) == (1, 10, 4)    # duals without equality rows: [z; lam]


def test_function_attributes(monkeypatch):
    from qpth_b200 import QPFunction, QPSolutionFunction, eqonly
    from qpth_b200.qp import QPSolvers
    with pytest.raises(RuntimeError, match="forward"):
        QPFunction().jacobian()
    with pytest.raises(RuntimeError, match="forward"):
        QPSolutionFunction().jacobian(wrt=("p",))
    with pytest.raises(NotImplementedError, match="CVXPY"):
        QPFunction(solver=QPSolvers.CVXPY).jacobian()
    monkeypatch.setattr(eqonly, "solve_equality_qp", lambda Q, p, A, b, *a, **k: torch.zeros(1, 4))
    f = QPFunction()
    f(torch.eye(4), torch.zeros(4), torch.Tensor(), torch.Tensor(), torch.ones(1, 4), torch.ones(1))
    with pytest.raises(NotImplementedError, match="equality-only"):
        f.jacobian()


# ---- C ABI: coverage and argument checks (no device work) -----------------------------------------------------------

def _smem(n, m, e):
    from qpth_b200 import _lib
    plan = _lib.Plan()
    _lib.check(_lib.load().qpb200_plan_init(n, m, e, ctypes.byref(plan)))
    out = ctypes.c_int64(-1)
    assert _lib.load().qpb200_jacobian_smem(ctypes.byref(plan), ctypes.byref(out)) == 0
    return plan, out.value


# (shape, covered): C2, C3, tiny shapes; the edge pair of nz = nineq (the staircase of order 200 leaves room for one
# column block, order 208 for none); orders past the product-form kernels
GRID = [((100, 100, 0), True), ((50, 50, 10), True), ((10, 5, 0), True), ((24, 19, 5), True), ((31, 21, 0), True),
        ((200, 200, 0), True), ((201, 201, 0), False), ((120, 260, 0), False), ((133, 920, 129), False),
        ((1000, 9, 100), True)]


@pytest.mark.parametrize("shape,covered", GRID)
def test_jacobian_smem_grid(shape, covered):
    _, smem = _smem(*shape)
    assert (smem > 0) == covered, (shape, smem)
    assert smem <= 232448 - 1024


def test_jacobian_smem_edge_pair():
    """The largest covered nz = nineq order, and the next one."""
    last = max(k for k in range(190, 210) if _smem(k, k, 0)[1] > 0)
    assert last == 200 and _smem(201, 201, 0)[1] == 0
    assert _smem(200, 200, 0)[1] == 220672


def test_jacobian_arg_checks():
    from qpth_b200 import _lib
    lib = _lib.load()
    plan, _ = _smem(12, 8, 3)
    plan0, _ = _smem(12, 8, 0)
    big, _ = _smem(201, 201, 0)
    P = ctypes.c_void_p(16)                                 # never dereferenced: every check returns first
    N = ctypes.c_void_p(0)
    ok = (P, P, P, P, 1, P, N)
    assert lib.qpb200_jacobian_smem(None, ctypes.byref(ctypes.c_int64())) == 1
    assert lib.qpb200_jacobian_smem(ctypes.byref(plan), None) == 1
    for i in range(4):
        args = list(ok)
        args[i] = N
        assert lib.qpb200_jacobian(ctypes.byref(plan), 2, 7, 7, *args[:4], 1, P, N) == 1
    assert lib.qpb200_jacobian(ctypes.byref(plan), 2, 7, 7, P, P, P, P, 1, N, N) == 1      # J
    assert lib.qpb200_jacobian(None, 2, 7, 7, P, P, P, P, 1, P, N) == 1
    assert lib.qpb200_jacobian(ctypes.byref(plan), 0, 7, 7, P, P, P, P, 1, P, N) == 1     # nbatch < 1
    assert lib.qpb200_jacobian(ctypes.byref(plan), 2, 0, 7, P, P, P, P, 1, P, N) == 1     # empty masks
    assert lib.qpb200_jacobian(ctypes.byref(plan), 2, 7, 0, P, P, P, P, 1, P, N) == 1
    assert lib.qpb200_jacobian(ctypes.byref(plan), 2, 8, 7, P, P, P, P, 1, P, N) == 1     # unknown bit
    assert lib.qpb200_jacobian(ctypes.byref(plan0), 2, 4, 1, P, P, P, P, 1, P, N) == 1    # nu rows, neq == 0
    assert lib.qpb200_jacobian(ctypes.byref(plan0), 2, 1, 4, P, P, P, P, 1, P, N) == 1    # b columns, neq == 0
    assert lib.qpb200_jacobian(ctypes.byref(big), 2, 3, 3, P, P, P, P, 1, P, N) == 4      # not covered


# ---- ptxas report of the Jacobian unit ------------------------------------------------------------------------------
# k_jacobian with nvcc 12.9 for sm_90a: registers at most this, and no stack frame or spills in it or its subroutines
JAC_REGISTERS = 106


def test_jacobian_ptxas_report():
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
    (entry, funcs), = [(k, v) for k, v in rep.items() if "k_jacobian" in k]
    assert all(f[1:] == (0, 0, 0) for f in funcs), funcs
    regs = [int(x) for x in re.findall(r"Used (\d+) registers", r.stderr)]
    assert regs and max(regs) <= JAC_REGISTERS, regs
