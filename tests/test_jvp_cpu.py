"""Forward mode of QPFunction / BoxQPFunction on the CPU: the models it rests on, the equality-only path's host logic, and
the C ABI boundary of qpb200_jvp, qpb200_jvp_reg and qpb200_box_jvp.

- The JVP models (tests/jvp_models.py: the backward's system with rx = sym(dQ) z + dp + dG' lam + dA' nu, rz = dG z - dh,
  ry = dA z - db) against central differences of tight re-solves within 1e-5, on the strictly complementary problems of
  tests/dual_models.py.
- The transpose identity sum <(g_z, g_lam, g_nu), JVP(t)> = sum_X <grad_X, t_X> against the backward models
  dual_models.backward_one, backward_one_reg and backward_one_box within 1e-12, and its factor B for un-batched inputs
  (their tangent applies to every QP, while the backward returns the batch mean).
- The equality-only path (qpth_b200/eqonly.py) with the dense stand-in of tests/test_eqonly_cpu.py through
  torch.autograd.forward_ad: None tangents, shared tangents, fp32 and CPU inputs, duals=True and False, against forward
  mode through the closed-form KKT solution.
- The three entry points are declared, exported and typed, and refuse bad arguments with QPB200_ERR_BAD_ARG before
  anything reaches the device.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from oracle import box_model as bm
from oracle import kernel_model as km
from oracle import reg_model as rm
from tests import dual_models as dm
from tests import jvp_models as jm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(8, 10, 3), (12, 15, 0), (10, 9, 4)]
BOX_SHAPES = [(9, 3, "both"), (10, 0, "lb"), (7, 2, "ub")]
INPUTS = ("Q", "p", "G", "h", "A", "b")
GRADS = ("dQ", "dp", "dG", "dh", "dA", "db")


def _solve(pr, reg=False):
    args = tuple(pr[k] for k in INPUTS)
    if reg:
        return rm.solve_one_reg(*args, steps=3, eps=1e-14, maxIter=40, stall_tol=1e-6)
    return km.solve_one(*args, eps=1e-14, maxIter=40, stall_tol=1e-6, tie=1.5)


def _tangents(pr, seed, keys=INPUTS):
    rs = np.random.RandomState(seed)
    return {k: (rs.randn(*pr[k].shape) if pr[k] is not None and pr[k].size else None) for k in keys}


def _outs(sol, e):
    return [sol["x"], sol["lam"]] + ([sol["nu"]] if e else [])


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_model_matches_central_differences(shape):
    """The JVP of z, lam and nu along a tangent of every input at once (Q symmetric: the models read one triangle)."""
    n, m, e = shape
    pr = dm.complementary_qp(23 * n + m + e, n, m, e)
    sol = _solve(pr)
    tan = _tangents(pr, n + m)
    tan["Q"] = 0.5 * (tan["Q"] + tan["Q"].T)
    got = jm.jvp_dense(pr["Q"], pr["G"], pr["A"], sol["x"], sol["lam"], sol["s"], sol["nu"], tan)
    t = 1e-6
    hi = {k: (pr[k] + t * tan[k] if tan[k] is not None else pr[k]) for k in INPUTS}
    lo = {k: (pr[k] - t * tan[k] if tan[k] is not None else pr[k]) for k in INPUTS}
    for g, h, l in zip(got, _outs(_solve(hi), e), _outs(_solve(lo), e)):
        fd = (h - l) / (2 * t)
        assert np.abs(fd - g).max() <= 1e-5 * max(1.0, np.abs(g).max()), np.abs(fd - g).max()


def _pairing(jvp, g, e):
    return sum(float(np.sum(a * b)) for a, b in zip(jvp[:3 if e else 2], g))


@pytest.mark.parametrize("reg", [False, True], ids=["dense", "reg"])
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_transpose_identity_with_the_backward_models(shape, reg):
    n, m, e = shape
    seed = 29 * n + m + e
    pr = dm.complementary_qp(seed, n, m, e)
    rs = np.random.RandomState(seed)
    gz, glam, gnu = rs.randn(n), rs.randn(m), (rs.randn(e) if e else None)
    tan = _tangents(pr, seed + 1)
    if reg:
        sol = rm.solve_one_reg(*(pr[k] for k in INPUTS), steps=2, maxIter=3, eps=0.0)
        sol["steps"] = 2
        jvp = jm.jvp_reg(sol, tan)
        grads = dm.backward_one_reg(sol, gz, glam, gnu)
    else:
        sol = km.solve_one(*(pr[k] for k in INPUTS), maxIter=3, eps=0.0)
        jvp = jm.jvp_dense(pr["Q"], pr["G"], pr["A"], sol["x"], sol["lam"], sol["s"], sol["nu"], tan)
        grads = dm.backward_one(sol, gz, glam, gnu)
    lhs = _pairing(jvp, [gz, glam] + ([gnu] if e else []), e)
    terms = [float(np.sum(grads[g] * tan[k])) for g, k in zip(GRADS, INPUTS) if tan[k] is not None and g in grads]
    assert abs(lhs - sum(terms)) <= 1e-12 * max(abs(lhs), sum(abs(x) for x in terms)), (lhs, sum(terms))


@pytest.mark.parametrize("shape", BOX_SHAPES, ids=["%dx%dx%s" % s for s in BOX_SHAPES])
def test_box_transpose_identity_and_central_differences(shape):
    n, e, sides = shape
    pr = dm.complementary_box(31 * n + e, n, e, sides)
    args = (pr["q"], pr["p"], pr["A"], pr["b"], pr["lb"], pr["ub"])
    sol = bm.solve_one(*args, eps=1e-14, maxIter=40, stall_tol=1e-6, tie=1.5)
    nlb, has_ub = (n if pr["lb"] is not None else 0), pr["ub"] is not None
    keys = ("q", "p", "A", "b", "lb", "ub")
    tan = _tangents(pr, n + e, keys)
    # the identity at the third iterate, where d = lam / s is well conditioned (at the converged point it spans 14
    # decades and the two solves agree only to their rounding there, ~1e-10)
    early = bm.solve_one(*args, maxIter=3, eps=0.0)
    ej = jm.jvp_box(pr["q"], pr["A"], early["x"], early["lam"], early["s"], early["nu"], nlb, has_ub, tan)
    rs = np.random.RandomState(n)
    m = sol["lam"].shape[0]
    gz, glam, gnu = rs.randn(n), rs.randn(m), (rs.randn(e) if e else None)
    var, sgn = bm.rows(n, nlb > 0, has_ub)
    g = dm.backward_one_box(dict(early, q=pr["q"], A=pr["A"], var=var, sgn=sgn, nlb=nlb), gz, glam, gnu)
    lhs = _pairing(ej, [gz, glam] + ([gnu] if e else []), e)
    terms = [float(np.sum(g["d" + k] * tan[k])) for k in keys if tan[k] is not None]
    assert abs(lhs - sum(terms)) <= 1e-12 * max(abs(lhs), sum(abs(x) for x in terms)), (lhs, sum(terms))
    jvp = jm.jvp_box(pr["q"], pr["A"], sol["x"], sol["lam"], sol["s"], sol["nu"], nlb, has_ub, tan)
    t = 1e-6
    hi = [a + t * tan[k] if tan[k] is not None else a for a, k in zip(args, keys)]
    lo = [a - t * tan[k] if tan[k] is not None else a for a, k in zip(args, keys)]
    sh = bm.solve_one(*hi, eps=1e-14, maxIter=40, stall_tol=1e-6, tie=1.5)
    sl = bm.solve_one(*lo, eps=1e-14, maxIter=40, stall_tol=1e-6, tie=1.5)
    for gv, h, l in zip(jvp, _outs(sh, e), _outs(sl, e)):
        fd = (h - l) / (2 * t)
        assert np.abs(fd - gv).max() <= 1e-5 * max(1.0, np.abs(gv).max()), np.abs(fd - gv).max()


def test_unbatched_tangents_carry_the_factor_B():
    """One shared tangent for a batch of QPs: sum_b <g_b, JVP_b(t)> = B <mean_b grad_b, t>, the mean being what the
    backward returns for an un-batched input."""
    n, m, e, B = 8, 10, 3, 4
    prs = [dm.complementary_qp(70 + i, n, m, e) for i in range(B)]
    rs = np.random.RandomState(3)
    tan = dict(G=rs.randn(m, n), b=rs.randn(e))           # the shared tangents; the others are absent
    lhs, grads = 0.0, []
    for pr in prs:
        sol = km.solve_one(*(pr[k] for k in INPUTS), maxIter=3, eps=0.0)
        gz, glam, gnu = rs.randn(n), rs.randn(m), rs.randn(e)
        lhs += _pairing(jm.jvp_dense(pr["Q"], pr["G"], pr["A"], sol["x"], sol["lam"], sol["s"], sol["nu"], tan),
                        [gz, glam, gnu], e)
        grads.append(dm.backward_one(sol, gz, glam, gnu))
    mean = {k: np.mean([g[k] for g in grads], 0) for k in ("dG", "db")}
    rhs = B * (np.sum(mean["dG"] * tan["G"]) + np.sum(mean["db"] * tan["b"]))
    assert abs(lhs - rhs) <= 1e-12 * abs(rhs)


# ---- the equality-only path -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("duals", [False, True])
@pytest.mark.parametrize("shared", [False, True])
def test_equality_only_jvp_matches_the_closed_form(shared, duals, dtype, monkeypatch):
    from qpth_b200 import QPFunction, eqonly
    from tests.test_eqonly_cpu import DenseFactor
    monkeypatch.setattr(eqonly, "_factor", DenseFactor)
    monkeypatch.setattr(eqonly, "_target_device", lambda Q_: torch.device("cpu"))
    rs = np.random.RandomState(8)
    B, nz, neq = 3, 7, 3
    L = rs.randn(nz, nz) if shared else rs.randn(B, nz, nz)
    T = lambda a: torch.tensor(a, dtype=dtype)
    ins = dict(Q=T(L @ np.swapaxes(L, -1, -2) + 0.5 * np.eye(nz)), p=T(rs.randn(B, nz)),
               A=T(rs.randn(neq, nz) if shared else rs.randn(B, neq, nz)), b=T(rs.randn(B, neq)))
    # Q symmetric (the factor reads one triangle); p has no tangent: it arrives as None
    tan = dict(Q=T(np.swapaxes(L, -1, -2) + L), A=T(rs.randn(*ins["A"].shape)), b=T(rs.randn(B, neq)))
    e = torch.Tensor().to(dtype)
    f = QPFunction(verbose=-1, duals=duals)
    with fwAD.dual_level():
        x = {k: fwAD.make_dual(v, tan[k]) if k in tan else v for k, v in ins.items()}
        outs = f(x["Q"], x["p"], e, e, x["A"], x["b"])
        outs = outs if duals else (outs,)
        got = [fwAD.unpack_dual(o).tangent for o in outs]

    def closed(Q, p, A, b):
        Qb, Ab = Q.expand(B, nz, nz), A.expand(B, neq, nz)
        K = torch.cat([torch.cat([Qb, Ab.transpose(1, 2)], 2), torch.cat([Ab, torch.zeros(B, neq, neq)], 2)], 1)
        s = torch.linalg.solve(K, torch.cat([-p, b], 1).unsqueeze(-1)).squeeze(-1)
        return s[:, :nz], s[:, nz:]
    d64 = {k: v.double() for k, v in ins.items()}
    with fwAD.dual_level():
        x = {k: fwAD.make_dual(v, tan[k].double()) if k in tan else v for k, v in d64.items()}
        zc, nuc = (fwAD.unpack_dual(o).tangent for o in closed(x["Q"], x["p"], x["A"], x["b"]))
    want = [zc, torch.zeros(B, 0, dtype=torch.float64), nuc] if duals else [zc]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == dtype and g.device.type == "cpu" and g.shape == w.shape
        tol = 1e-9 if dtype == torch.float64 else 1e-3
        assert torch.allclose(g.double(), w, rtol=tol, atol=tol)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------

NEW = ("qpb200_jvp", "qpb200_jvp_reg", "qpb200_box_jvp")


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
    # the tangents (pointer, stride) x 6 replace the gradients (pointer, mean flag) x 6 of the backward; the adjoints
    # become the rhs work buffer
    assert len(_lib.SIGNATURES["qpb200_jvp"][1]) == len(_lib.SIGNATURES["qpb200_backward_duals"][1]) - 2
    assert len(_lib.SIGNATURES["qpb200_jvp_reg"][1]) == len(_lib.SIGNATURES["qpb200_jvp"][1]) + 2


def test_bad_arguments_are_refused_before_any_launch(lib):
    """Every call here fails its argument checks, which run before any CUDA call: on a machine without a GPU a check
    that came too late would return QPB200_ERR_CUDA instead. The pointers are never dereferenced."""
    from qpth_b200 import _lib
    P = ctypes.c_void_p(16)
    N = None
    plan = _lib.plan_for(20, 15, 0)
    plan_eq = _lib.plan_for(20, 15, 5)

    def dense(pl, B=2, tans=None, rhs=P, dnu=N, extra=(), fn=None):
        tans = tans or [N, 0] * 6
        fn = fn or lib.qpb200_jvp
        return fn(ctypes.byref(pl), B, *tans, P, P, P, P, P, P, P, 1, *extra, rhs, P, P, dnu, P, N)

    for fn, extra in ((lib.qpb200_jvp, ()), (lib.qpb200_jvp_reg, (1e-7, 1))):
        assert dense(plan, dnu=P, extra=extra, fn=fn) == 1                              # dnu without equality rows
        assert dense(plan, tans=[N, 0] * 4 + [P, 0, N, 0], extra=extra, fn=fn) == 1     # dA without equality rows
        assert dense(plan, B=0, extra=extra, fn=fn) == 1                                # empty batch
        assert dense(plan, rhs=N, extra=extra, fn=fn) == 1                              # no work buffer
        assert dense(plan, tans=[P, -1] + [N, 0] * 5, extra=extra, fn=fn) == 1          # negative stride
        assert dense(plan_eq, extra=extra, fn=fn) == 1                                  # neq > 0 needs dnu
    assert dense(plan, extra=(-1.0, 1), fn=lib.qpb200_jvp_reg) == 1                     # reg_eps < 0
    bp = _lib.box_plan_for(10, 0, True, False)
    bp_eq = _lib.box_plan_for(10, 3, True, True)

    def box(pl, B=2, tans=None, rhs=P, dnu=N, nus=P):
        tans = tans or [N, 0] * 6
        return lib.qpb200_box_jvp(ctypes.byref(pl), B, P, 0, P, 0, *tans, P, P, P, nus, rhs, P, P, dnu, N)

    assert box(bp, dnu=P) == 1                                                          # dnu without equality rows
    assert box(bp, tans=[N, 0] * 5 + [P, 0]) == 1                                       # dub without an ub side
    assert box(bp, B=0) == 1
    assert box(bp, rhs=N) == 1
    assert box(bp_eq, dnu=P, nus=N) == 1                                                # neq > 0 needs nus
    assert lib.qpb200_box_jvp(None, 2, P, 0, P, 0, *([N, 0] * 6), P, P, P, P, P, P, P, N, N) == 1
