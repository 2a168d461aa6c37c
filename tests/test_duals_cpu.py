"""The dual outputs of QPFunction / BoxQPFunction (duals=True) on the CPU: the derivation their backward pass rests on,
the host logic of the equality-only path, and the C ABI boundary of the three new entry points.

- The models' backward passes with dual adjoints (tests/dual_models.py) against the unsymmetric implicit derivative of
  the KKT conditions, solved densely, at 1e-9; and against central differences of a loss on z, lam and nu at 1e-5, the
  models re-solving the perturbed problems tightly. The problems are strictly complementary (active lam >= 0.1,
  inactive s >= 0.1), so lam and nu are differentiable there.
- The equality-only path (qpth_b200/eqonly.py) with the dense stand-in of tests/test_eqonly_cpu.py: the gradients of a
  loss on z and nu against autograd through the closed-form KKT solution.
- qpb200_backward_duals, qpb200_backward_reg_duals, qpb200_box_backward_duals are declared, exported and typed, and
  refuse bad arguments with QPB200_ERR_BAD_ARG before anything reaches the device.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import box_model as bm
from oracle import kernel_model as km
from oracle import reg_model as rm
from tests import dual_models as dm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(8, 10, 3), (12, 15, 0), (10, 9, 4)]
BOX_SHAPES = [(9, 3, "both"), (10, 0, "lb"), (7, 2, "ub")]


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _adjoints(seed, n, m, e):
    rs = np.random.RandomState(seed + 7)
    return rs.randn(n), rs.randn(m), (rs.randn(e) if e else None)


def _solve_dense(pr, reg=False):
    if reg:
        return rm.solve_one_reg(pr["Q"], pr["p"], pr["G"], pr["h"], pr["A"], pr["b"], steps=3, eps=1e-14, maxIter=40,
                                stall_tol=1e-6)
    return km.solve_one(pr["Q"], pr["p"], pr["G"], pr["h"], pr["A"], pr["b"], eps=1e-14, maxIter=40, stall_tol=1e-6,
                        tie=1.5)


def _check_complementary(sol, pr):
    act = pr["active"]
    assert np.abs(sol["x"] - pr["z"]).max() < 1e-9
    assert sol["lam"][act].min() >= 0.1 - 1e-9 and sol["s"][~act].min() >= 0.1 - 1e-9


@pytest.mark.parametrize("reg", [False, True], ids=["dense", "reg_spd"])
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_model_matches_implicit_derivative(shape, reg):
    """dx, dlam, dnu and every gradient against J' w = -[g_z; g_lam; g_nu], J the unsymmetric Jacobian at the model's
    iterate after three iterations: lam and s there lie between 1e-4 and 10, so d = lam / s is well conditioned and
    the 1e-8 clamps do nothing (at the converged point d spans 14 decades and the model's own rounding is ~1e-7, which
    the central differences below tolerate)."""
    n, m, e = shape
    seed = 11 * n + m + e
    pr = dm.complementary_qp(seed, n, m, e)
    args = tuple(pr[k] for k in ("Q", "p", "G", "h", "A", "b"))
    sol = rm.solve_one_reg(*args, steps=3, maxIter=3, eps=0.0) if reg else km.solve_one(*args, maxIter=3, eps=0.0)
    assert min(sol["lam"].min(), sol["s"].min()) >= 1e-4
    gz, glam, gnu = _adjoints(seed, n, m, e)
    got = (dm.backward_one_reg if reg else dm.backward_one)(sol, gz, glam, gnu)
    ref = dm.implicit(pr["Q"], pr["G"], pr["A"], sol["x"], sol["lam"], sol["s"], sol["nu"], gz, glam, gnu)
    for k in ("dx", "dlam", "dQ", "dp", "dG", "dh") + (("dnu", "dA", "db") if e else ()):
        assert _rel(got[k], ref[k]) <= 1e-9, (k, _rel(got[k], ref[k]))


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_model_without_adjoints_is_the_oracle_backward(shape):
    """g_lam = g_nu = None is the oracle's backward pass, bit for bit."""
    n, m, e = shape
    pr = dm.complementary_qp(5 + n, n, m, e)
    sol = _solve_dense(pr)
    gz = np.random.RandomState(1).randn(n)
    a, b = dm.backward_one(sol, gz), km.backward_one(sol, gz)
    for k in b:
        assert np.array_equal(a[k], b[k]), k


INPUTS = ("Q", "p", "G", "h", "A", "b")


def _loss(sol, gz, glam, gnu):
    out = gz @ sol["x"] + glam @ sol["lam"]
    if gnu is not None:
        out += gnu @ sol["nu"]
    return out


@pytest.mark.parametrize("reg", [False, True], ids=["dense", "reg_spd"])
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_model_matches_central_differences(shape, reg):
    """<grad, V> against (L(theta + t V) - L(theta - t V)) / 2t, t = 1e-6, for a random direction V of each input
    (symmetric for Q), L = g_z'z + g_lam'lam + g_nu'nu of a tight solve."""
    n, m, e = shape
    seed = 13 * n + m + e
    pr = dm.complementary_qp(seed, n, m, e)
    sol = _solve_dense(pr, reg)
    _check_complementary(sol, pr)
    gz, glam, gnu = _adjoints(seed, n, m, e)
    g = (dm.backward_one_reg if reg else dm.backward_one)(sol, gz, glam, gnu)
    rs = np.random.RandomState(seed + 3)
    t = 1e-6
    for k, gk in zip(INPUTS, ("dQ", "dp", "dG", "dh", "dA", "db")):
        if pr[k].size == 0:
            continue
        V = rs.randn(*pr[k].shape)
        if k == "Q":
            V = 0.5 * (V + V.T)
        lo, hi = dict(pr), dict(pr)
        lo[k], hi[k] = pr[k] - t * V, pr[k] + t * V
        fd = (_loss(_solve_dense(hi, reg), gz, glam, gnu) - _loss(_solve_dense(lo, reg), gz, glam, gnu)) / (2 * t)
        an = float(np.sum(g[gk] * V))
        assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (k, fd, an)


def _solve_box(pr):
    return bm.solve_one(pr["q"], pr["p"], pr["A"], pr["b"], pr["lb"], pr["ub"], eps=1e-14, maxIter=40, stall_tol=1e-6,
                        tie=1.5)


@pytest.mark.parametrize("shape", BOX_SHAPES, ids=["%dx%dx%s" % s for s in BOX_SHAPES])
def test_box_model_matches_implicit_derivative_and_central_differences(shape):
    n, e, sides = shape
    seed = 17 * n + e
    pr = dm.complementary_box(seed, n, e, sides)
    sol = _solve_box(pr)
    assert np.abs(sol["x"] - pr["z"]).max() < 1e-9
    m = sol["lam"].shape[0]
    assert np.maximum(sol["lam"], sol["s"]).min() >= 0.1 - 1e-9           # strictly complementary
    gz, glam, gnu = _adjoints(seed, n, m, e)
    got = dm.backward_one_box(sol, gz, glam, gnu)
    # the implicit derivative at the third iterate (see test_model_matches_implicit_derivative)
    early = bm.solve_one(pr["q"], pr["p"], pr["A"], pr["b"], pr["lb"], pr["ub"], maxIter=3, eps=0.0)
    assert min(early["lam"].min(), early["s"].min()) >= 1e-4
    Q, G, _ = bm.dense(pr["q"], pr["lb"], pr["ub"])
    g3 = dm.backward_one_box(early, gz, glam, gnu)
    ref = dm.implicit(Q, G, pr["A"], early["x"], early["lam"], early["s"], early["nu"], gz, glam, gnu)
    for k in ("dx", "dlam") + (("dnu",) if e else ()):
        assert _rel(g3[k], ref[k]) <= 1e-9, (k, _rel(g3[k], ref[k]))
    nlb = n if pr["lb"] is not None else 0
    rs = np.random.RandomState(seed + 3)
    t = 1e-6
    grads = dict(q=got["dq"], p=got["dp"], A=got["dA"], b=got["db"], lb=got["dlb"], ub=got["dub"])
    for k in ("q", "p", "A", "b", "lb", "ub"):
        if pr[k] is None or pr[k].size == 0:
            continue
        V = rs.randn(*pr[k].shape)
        lo, hi = dict(pr), dict(pr)
        lo[k], hi[k] = pr[k] - t * V, pr[k] + t * V
        fd = (_loss(_solve_box(hi), gz, glam, gnu) - _loss(_solve_box(lo), gz, glam, gnu)) / (2 * t)
        an = float(np.sum(grads[k] * V))
        assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (k, fd, an)
    assert nlb == (got["dlb"].shape[0] if got["dlb"] is not None else 0)


# ---- the equality-only path -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shared", [False, True])
def test_equality_only_nu_adjoint_matches_the_closed_form(shared, monkeypatch):
    from qpth_b200 import QPFunction, eqonly
    from tests.test_eqonly_cpu import DenseFactor
    monkeypatch.setattr(eqonly, "_factor", DenseFactor)
    monkeypatch.setattr(eqonly, "_target_device", lambda Q_: torch.device("cpu"))
    rs = np.random.RandomState(5)
    B, nz, neq = 4, 9, 4
    L = rs.randn(nz, nz) if shared else rs.randn(B, nz, nz)
    Q = torch.tensor(L @ np.swapaxes(L, -1, -2) + 0.1 * np.eye(nz), requires_grad=True)
    p = torch.tensor(rs.randn(B, nz), requires_grad=True)
    A = torch.tensor(rs.randn(neq, nz) if shared else rs.randn(B, neq, nz), requires_grad=True)
    b = torch.tensor(rs.randn(B, neq), requires_grad=True)
    gz, gnu = torch.tensor(rs.randn(B, nz)), torch.tensor(rs.randn(B, neq))
    e = torch.Tensor().double()
    z, lam, nu = QPFunction(verbose=-1, duals=True)(Q, p, e, e, A, b)
    assert lam.shape == (B, 0) and nu.shape == (B, neq) and lam.dtype == nu.dtype == z.dtype
    ((z * gz).sum() + (nu * gnu).sum()).backward()
    got = [t.grad.clone() for t in (Q, p, A, b)]
    for t in (Q, p, A, b):
        t.grad = None
    Qb = Q.expand(B, nz, nz) if shared else Q
    Ab = A.expand(B, neq, nz) if shared else A
    K = torch.cat([torch.cat([Qb, Ab.transpose(1, 2)], 2), torch.cat([Ab, torch.zeros(B, neq, neq).double()], 2)], 1)
    sol = torch.linalg.solve(K, torch.cat([-p, b], 1).unsqueeze(-1)).squeeze(-1)
    zc, nuc = sol[:, :nz], sol[:, nz:]
    assert torch.allclose(z, zc, rtol=1e-10, atol=1e-12) and torch.allclose(nu, nuc, rtol=1e-10, atol=1e-12)
    ((zc * gz).sum() + (nuc * gnu).sum()).backward()
    dQ = 0.5 * (Q.grad + Q.grad.transpose(-1, -2)) / (B if shared else 1)
    dA = A.grad / (B if shared else 1)
    for g, r in zip(got, (dQ, p.grad, dA, b.grad)):
        assert g.shape == r.shape and torch.allclose(g, r, rtol=1e-9, atol=1e-11)
    # only nu used: dl_dzhat arrives as None and is taken as zero
    for t in (Q, p, A, b):
        t.grad = None
    z, lam, nu = QPFunction(verbose=-1, duals=True)(Q, p, e, e, A, b)
    (nu * gnu).sum().backward()
    assert all(torch.isfinite(t.grad).all() for t in (Q, p, A, b))


# ---- the C ABI ----------------------------------------------------------------------------------------------------------

NEW = ("qpb200_backward_duals", "qpb200_backward_reg_duals", "qpb200_box_backward_duals")


@pytest.fixture(scope="module")
def lib():
    from qpth_b200 import _lib, build
    build.build()
    return _lib.load()


def test_new_symbols_declared_exported_typed(lib):
    from qpth_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "qpth_b200.h")).read()
    for name in NEW:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        base = name.replace("_duals", "")
        # the arguments of the counterpart plus dl_dlam and dl_dnu, after dl_dzhat
        assert len(_lib.SIGNATURES[name][1]) == len(_lib.SIGNATURES[base][1]) + 2, name


def test_bad_arguments_are_refused_before_any_launch(lib):
    """Every call here fails its argument checks, which run before any CUDA call: on a machine without a GPU a check
    that came too late would return QPB200_ERR_CUDA instead. The pointers are never dereferenced."""
    from qpth_b200 import _lib
    P = ctypes.c_void_p(16)                      # a non-NULL pointer the checks see but never read
    N = None
    plan = _lib.plan_for(20, 15, 0)              # neq == 0: dl_dnu must be NULL
    plan_eq = _lib.plan_for(20, 15, 5)
    outs = [N, 0] * 6

    def dense(fn, pl, B, dl, glam, gnu, extra=()):
        return fn(ctypes.byref(pl), B, dl, glam, gnu, P, P, P, P, P, P, P, 1, *extra, *outs, P, P, P, P, N)

    for fn, extra in ((lib.qpb200_backward_duals, ()), (lib.qpb200_backward_reg_duals, (1e-7, 1))):
        assert dense(fn, plan, 2, P, N, P, extra) == 1          # dl_dnu without equality rows
        assert dense(fn, plan, 0, P, P, N, extra) == 1          # empty batch
        assert dense(fn, plan, 2, N, P, N, extra) == 1          # dl_dzhat is required (zeros when only duals are used)
    assert lib.qpb200_backward_duals(ctypes.byref(plan_eq), 2, P, P, P, P, P, P, N, P, P, P, 1, *outs, P, P, P, P, N) == 1
    assert lib.qpb200_backward_reg_duals(ctypes.byref(plan), 2, P, P, N, P, P, P, P, P, P, P, 1, -1.0, 1, *outs, P, P,
                                         P, P, N) == 1          # reg_eps < 0
    bp = _lib.box_plan_for(10, 0, True, True)
    bp_eq = _lib.box_plan_for(10, 3, True, True)

    def box(pl, B, dl, glam, gnu, A=P, nus=P):
        return lib.qpb200_box_backward_duals(ctypes.byref(pl), B, P, 0, A, 0, dl, glam, gnu, P, P, P, nus, *outs, P, P,
                                             P, N)

    assert box(bp, 2, P, P, P) == 1                             # dl_dnu without equality rows
    assert box(bp, 0, P, P, N) == 1
    assert box(bp, 2, N, P, N) == 1
    assert box(bp_eq, 2, P, P, P, nus=N) == 1                   # neq > 0 needs nus
    assert lib.qpb200_box_backward_duals(None, 2, P, 0, P, 0, P, P, N, P, P, P, P, *outs, P, P, P, N) == 1
