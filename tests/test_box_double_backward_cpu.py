"""Second order of BoxQPFunction on the CPU: the model it rests on, the algebra the kernels implement, the host logic, and
the C ABI boundary of qpb200_box_double_backward / qpb200_boxq_double_backward.

- The torch model (tests/box_double_backward_models.py) against central differences of the first-order box gradient
  (the dense first-order gradient of tests/dual_models.backward_one on the dense equivalent, mapped back) at re-solved
  points, on strictly complementary problems.
- The structured numpy algebra of the kernels against the model within 1e-10: diagonal and dense Q, lb / ub / both,
  neq = 0 and > 0, every input batched and each sharing.
- BoxQPFunction's host logic with the box solves replaced by CPU stand-ins: create_graph routing, None cotangents,
  dtype casts, sums for un-batched inputs, first order unchanged, third order raising; the dense fallback by
  gradgradcheck through QPFunction's stand-ins.
- The entry points are declared, exported and typed, refuse bad arguments before any launch, the version is still 103,
  the right-hand side kernels' shared memory fits every plan, and the new kernels' ptxas report.
"""
import ctypes
import os
import re
import subprocess
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle import kernel_model as km
from tests import box_double_backward_models as bdm
from tests import dual_models as dm
from tests.test_double_backward_cpu import stand_ins  # noqa: F401  (QPFunction's dense stand-ins, a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = bdm.NAMES
SIDES = ("both", "lb", "ub")


def _T(a):
    return torch.tensor(np.asarray(a, dtype=np.float64))


def _dense(pr):
    """(Q, G, h) of the dense equivalent of one box problem (numpy)"""
    n = pr["q"].shape[-1]
    Q = pr["q"] if pr["q"].ndim == 2 else np.diag(pr["q"])
    G = np.concatenate(([-np.eye(n)] if pr["lb"] is not None else []) + ([np.eye(n)] if pr["ub"] is not None else []))
    h = np.concatenate(([-pr["lb"]] if pr["lb"] is not None else []) + ([pr["ub"]] if pr["ub"] is not None else []))
    return Q, G, h


def _box_grads(pr, gz, glam, gnu, eps=1e-15):
    """the first-order box gradients of one problem at a tight re-solve of its dense equivalent"""
    n, e = pr["q"].shape[-1], pr["A"].shape[0]
    Q, G, h = _dense(pr)
    sol = km.solve_one(Q, pr["p"], G, h, pr["A"], pr["b"], eps=eps, maxIter=60, stall_tol=1e-7, tie=1.5)
    g = dm.backward_one(sol, gz, glam, gnu)
    nlb = n if pr["lb"] is not None else 0
    return dict(q=np.diag(g["dQ"]), p=g["dp"], A=g["dA"] if e else None, b=g["db"] if e else None,
                lb=-g["dh"][:nlb] if nlb else None, ub=g["dh"][nlb:] if pr["ub"] is not None else None), sol


@pytest.mark.parametrize("shape", [(8, 3, "both"), (9, 0, "lb"), (10, 2, "ub")], ids=["8x3_both", "9x0_lb", "10x2_ub"])
def test_model_matches_central_differences(shape):
    """d/de <w, grad(theta + e t)> by central differences of the first-order box gradient at re-solved points, against
    <model's second-order gradient, t>, along a direction t of every input and of the adjoints."""
    n, e, sides = shape
    pr = dm.complementary_box(3 * n + e, n, e, sides)
    m = n * ((pr["lb"] is not None) + (pr["ub"] is not None))
    rs = np.random.RandomState(n + e)
    gz, glam, gnu = rs.randn(n), rs.randn(m), (rs.randn(e) if e else None)
    keys = [k for k in NAMES if pr[k] is not None and np.size(pr[k])]
    om = {k: rs.randn(*np.shape(pr[k])) for k in keys}
    tan = {k: rs.randn(*np.shape(pr[k])) for k in keys}
    tg = dict(gz=rs.randn(n), glam=rs.randn(m), gnu=rs.randn(e) if e else None)

    def phi(h):
        x = dict(pr)
        x.update({k: pr[k] + h * tan[k] for k in keys})
        g, _ = _box_grads(x, gz + h * tg["gz"], glam + h * tg["glam"], None if gnu is None else gnu + h * tg["gnu"])
        return sum(np.sum(om[k] * g[k]) for k in keys)

    h = 1e-5
    fd = (phi(h) - phi(-h)) / (2 * h)
    _, sol = _box_grads(pr, gz, glam, gnu)
    ins = {k: (_T(pr[k])[None] if pr[k] is not None else None) for k in NAMES}
    if e == 0:
        ins["A"], ins["b"] = torch.zeros(1, 0, n, dtype=torch.float64), torch.zeros(1, 0, dtype=torch.float64)
    pt = dict(z=_T(sol["x"])[None], lam=_T(sol["lam"])[None], s=_T(sol["s"])[None],
              nu=_T(sol["nu"])[None] if e else torch.zeros(1, 0, dtype=torch.float64))
    r = bdm.double_backward(ins, pt, _T(gz)[None], _T(glam)[None], _T(gnu)[None] if e else None,
                            {k: (_T(om[k])[None] if k in om else None) for k in NAMES})
    an = sum(float((r[k][0] * _T(tan[k])).sum()) for k in keys)
    an += float((r["gz"][0] * _T(tg["gz"])).sum()) + float((r["glam"][0] * _T(tg["glam"])).sum())
    if e:
        an += float((r["gnu"][0] * _T(tg["gnu"])).sum())
    # 1e-5: the re-solved points are interior-point points, whose D at the active bounds is large but finite
    assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (fd, an)


# ---- the structured algebra against the model -----------------------------------------------------------------------

def _point(n, e, sides, dense_Q, B=3, seed=1, clamp=False):
    rs = np.random.RandomState(seed)
    nlb, has_ub = (n if sides != "ub" else 0), sides != "lb"
    m = n * (int(sides != "ub") + int(has_ub))
    q = (lambda F: F @ F.transpose(0, 2, 1) / n + 0.5 * np.eye(n))(rs.randn(B, n, n)) if dense_Q else 0.5 + rs.rand(B, n)
    pt = dict(q=q, A=rs.randn(B, e, n) / np.sqrt(n), z=rs.randn(B, n), nu=rs.randn(B, e),
              lam=rs.uniform(0.1, 10, (B, m)), s=rs.uniform(0.1, 10, (B, m)), dl=rs.randn(B, n), glam=rs.randn(B, m),
              gnu=rs.randn(B, e), nlb=nlb, has_ub=has_ub)
    if clamp:                        # one clamped slack and one clamped dual: the clamps' derivative conventions
        pt["s"][1, 0], pt["lam"][2, 0] = 1e-9, 1e-9
    return pt, rs


def _algebra_and_model(n, e, sides, dense_Q, shared, clamp=False):
    B = 3
    pt, rs = _point(n, e, sides, dense_Q, B, clamp=clamp)
    nlb, has_ub = pt["nlb"], pt["has_ub"]
    shp = dict(q=(n, n) if dense_Q else (n,), p=(n,), A=(e, n), b=(e,), lb=(n,), ub=(n,))
    absent = dict(A=e == 0, b=e == 0, lb=not nlb, ub=not has_ub)
    om = {k: None if absent.get(k) else rs.randn(*(shp[k] if k in shared else (B,) + shp[k])) for k in NAMES}
    q = pt["q"][0] if "q" in shared else pt["q"]
    A = (pt["A"][0] if "A" in shared else pt["A"]) if e else None
    sv = [bdm.box_solve(q if "q" in shared else q[i], (A if "A" in shared else A[i]) if e else None, pt["lam"][i],
                        pt["s"][i], nlb, has_ub, dense_Q)(pt["dl"][i], pt["glam"][i], pt["gnu"][i]) for i in range(B)]
    v = (np.stack([x[0] for x in sv]), np.stack([x[1] for x in sv]), np.stack([x[2] for x in sv]) if e else None)
    flags = {k: k in shared for k in NAMES}
    got = bdm.box_double_backward(q, A, pt["z"], pt["lam"], pt["s"], pt["nu"] if e else None, v, om, nlb, has_ub,
                                  flags, dense_Q)
    zeros = lambda k, s: _T(np.zeros(shp[k] if k in shared else (B,) + shp[k]))
    ins = dict(q=_T(q), p=zeros("p", shared), A=_T(A) if e else torch.zeros(B, 0, n, dtype=torch.float64),
               b=zeros("b", shared) if e else torch.zeros(B, 0, dtype=torch.float64),
               lb=zeros("lb", shared) if nlb else None, ub=zeros("ub", shared) if has_ub else None)
    sh = tuple(k for k in shared if not absent.get(k))
    mpt = dict(z=_T(pt["z"]), lam=_T(pt["lam"]), s=_T(pt["s"]),
               nu=_T(pt["nu"]) if e else torch.zeros(B, 0, dtype=torch.float64))
    ref = bdm.double_backward(ins, mpt, _T(pt["dl"]), _T(pt["glam"]), _T(pt["gnu"]) if e else None,
                              {k: (None if x is None else _T(x)) for k, x in om.items()}, sh, dense_Q)
    return got, ref


SHARINGS = {"batched": (), "shared_qA": ("q", "A"), "shared_pbs": ("p", "b", "lb", "ub")}


@pytest.mark.parametrize("shared", list(SHARINGS), ids=list(SHARINGS))
@pytest.mark.parametrize("e", [0, 3])
@pytest.mark.parametrize("sides", SIDES)
@pytest.mark.parametrize("dense_Q", [False, True], ids=["diag", "dense"])
def test_algebra_matches_the_model(dense_Q, sides, e, shared):
    got, ref = _algebra_and_model(7, e, sides, dense_Q, SHARINGS[shared])
    for k in ("gz", "glam", "gnu") + NAMES:
        if got[k] is None:
            assert ref.get(k) is None or ref[k].numel() == 0, k
            continue
        r = ref[k].numpy()
        assert np.abs(got[k] - r).max() <= 1e-10 * max(1.0, np.abs(r).max()), k


@pytest.mark.parametrize("dense_Q", [False, True], ids=["diag", "dense"])
def test_algebra_matches_the_model_at_the_clamps(dense_Q):
    """a clamped slack and a clamped dual (1e-9): c_lam and c_s vanish where torch's clamp passes no gradient. D spans
    eleven decades there, so the dense model's own solve is the looser side."""
    got, ref = _algebra_and_model(7, 3, "both", dense_Q, (), clamp=True)
    for k in ("gz", "glam", "gnu") + NAMES:
        r = ref[k].numpy()
        assert np.abs(got[k] - r).max() <= 1e-6 * max(1.0, np.abs(r).max()), k


# ---- BoxQPFunction's host logic with CPU stand-ins -----------------------------------------------------------------

class _BoxPlan:
    def __init__(self, n, e, has_lb, has_ub):
        self.nz, self.neq, self.has_lb, self.has_ub = n, e, int(has_lb), int(has_ub)
        self.nineq = n * (int(has_lb) + int(has_ub))


@pytest.fixture
def box_stand_ins(monkeypatch):
    """solve_box_forward, solve_box_backward and solve_box_double_backward on the CPU: the dense model's solver on the
    dense equivalent, the structured solves of box_double_backward_models."""
    from qpth_b200 import box
    calls = []

    def fwd(q_, p_, A_, b_, lb_, ub_, *a, **k):
        dense_Q = bool(a[5]) if len(a) > 5 else bool(k.get("dense_Q", False))   # solve_box_forward's 12th argument
        nB, n, e = box.check_box_shapes(q_, p_, A_, b_, lb_, ub_, dense_Q)
        ex = lambda X, nd: None if X is None else (X.detach().double() if X.dim() == nd else
                                                    X.detach().double().unsqueeze(0).expand(nB, *X.shape))
        q, p, lb, ub = ex(q_, 3 if dense_Q else 2), ex(p_, 2), ex(lb_, 2), ex(ub_, 2)
        A = ex(A_, 3) if e else None
        b = ex(b_, 2) if e else None
        st = types.SimpleNamespace(plan=_BoxPlan(n, e, lb_ is not None, ub_ is not None), nBatch=nB, dense=None,
                                   dense_Q=dense_Q, q=q, A=A, device=torch.device("cpu"))
        sols = []
        for i in range(nB):
            pr = dict(q=q[i].numpy(), p=p[i].numpy(), lb=None if lb is None else lb[i].numpy(),
                      ub=None if ub is None else ub[i].numpy())
            Q, G, h = _dense(pr)
            sols.append(km.solve_one(Q, pr["p"], G, h, A[i].numpy() if e else np.zeros((0, n)),
                                     b[i].numpy() if e else np.zeros(0), eps=1e-14, maxIter=40, stall_tol=1e-6,
                                     tie=1.5))
        st.zhat = _T(np.stack([s_["x"] for s_ in sols]))
        st.lam = _T(np.stack([s_["lam"] for s_ in sols]))
        st.slacks = _T(np.stack([s_["s"] for s_ in sols]))
        st.nus = _T(np.stack([s_["nu"] for s_ in sols])) if e else None
        st.iters = torch.zeros(nB, dtype=torch.int32)
        st.best_resid = torch.zeros(nB, dtype=torch.float64)
        st.trace = None
        return st

    def solves(st):
        P = st.plan
        return [bdm.box_solve(st.q[i].numpy(), st.A[i].numpy() if P.neq else None, st.lam[i].numpy(),
                              st.slacks[i].numpy(), P.nz if P.has_lb else 0, bool(P.has_ub), st.dense_Q)
                for i in range(st.nBatch)]

    def bwd(st, dl, flags, want, glam=None, gnu=None, keep=False):
        calls.append("backward")
        P, B = st.plan, st.nBatch
        n, e, m, nlb = P.nz, P.neq, P.nineq, (P.nz if P.has_lb else 0)
        f = lambda g, k: np.zeros((B, k)) if g is None else g.detach().double().reshape(B, k).numpy()
        gz_, gl_, gn_ = f(dl, n), f(glam, m), f(gnu, e)
        vs = [s(gz_[i], gl_[i], gn_[i]) for i, s in enumerate(solves(st))]
        vx, vl = _T(np.stack([x[0] for x in vs])), _T(np.stack([x[1] for x in vs]))
        vn = _T(np.stack([x[2] for x in vs])) if e else None
        z = st.zhat
        outer = lambda a, b: a.unsqueeze(2) * b.unsqueeze(1)
        g = [0.5 * (outer(vx, z) + outer(z, vx)) if st.dense_Q else vx * z, vx,
             outer(vn, z) + outer(st.nus, vx) if e else None, -vn if e else None, vl[:, :nlb] if nlb else None,
             -vl[:, nlb:] if P.has_ub else None]
        outs = [None if (not want[k] or g[k] is None) else (g[k].mean(0) if flags[k] else g[k]) for k in range(6)]
        return (outs, (vx, vl, vn)) if keep else outs

    def dbl(st, v, omegas, flags, want):
        calls.append("double_backward")
        P = st.plan
        e = P.neq
        om = {k: None if w is None else w.detach().double().numpy() for k, w in zip(NAMES, omegas)}
        res = bdm.box_double_backward(st.q.numpy() if not flags[0] else st.q[0].numpy(),
                                      (st.A.numpy() if not flags[2] else st.A[0].numpy()) if e else None,
                                      st.zhat.numpy(), st.lam.numpy(), st.slacks.numpy(),
                                      st.nus.numpy() if e else None, tuple(None if x is None else x.numpy() for x in v),
                                      om, P.nz if P.has_lb else 0, bool(P.has_ub), dict(zip(NAMES, flags)), st.dense_Q)
        out = [None if res[k] is None else _T(res[k]) for k in ("gz", "glam", "gnu")]
        return out + [None if (res[k] is None or not want[i]) else _T(res[k]) for i, k in enumerate(NAMES)]

    monkeypatch.setattr(box, "solve_box_forward", fwd)
    monkeypatch.setattr(box, "solve_box_backward", bwd)
    monkeypatch.setattr(box, "solve_box_double_backward", dbl)
    return calls


def _box_problem(n, e, sides, B, seed, dense_Q=False, same=False):
    """B strictly complementary problems (same: B copies of one, so that un-batched inputs keep every QP strictly
    complementary)"""
    prs = [dm.complementary_box(seed + (0 if same else 31 * i), n, e, sides) for i in range(B)]
    ins = {k: (None if prs[0][k] is None else _T(np.stack([pr[k] for pr in prs]))) for k in NAMES}
    if dense_Q:
        rs = np.random.RandomState(seed)
        F = rs.randn(B, n, n)
        ins["q"] = _T(np.stack([np.diag(pr["q"]) for pr in prs]) + 0.1 * (F @ F.transpose(0, 2, 1)) / n)
    return ins


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("shared", [(), ("q", "A", "lb"), ("p", "b", "ub")], ids=["batched", "shared_qAlb", "shared_pbub"])
@pytest.mark.parametrize("case", [(8, 3, "both", False), (9, 0, "lb", False), (7, 2, "both", True)],
                         ids=["8x3_both", "9x0_lb", "7x2_denseQ"])
def test_box_second_order_through_the_host_logic(box_stand_ins, case, shared, dtype):
    from qpth_b200 import BoxQPFunction
    n, e, sides, dense_Q = case
    B = 3
    ins = _box_problem(n, e, sides, B, 4, dense_Q, same=bool(shared))
    if e == 0:
        ins["A"], ins["b"] = torch.Tensor().double(), torch.Tensor().double()
    ins = {k: (None if v is None else (v[0] if k in shared and v.numel() else v)) for k, v in ins.items()}
    leaves = {k: (None if v is None else v.to(dtype).clone().requires_grad_(v.numel() > 0)) for k, v in ins.items()}
    keys = [k for k in NAMES if leaves[k] is not None and leaves[k].requires_grad]
    rs = np.random.RandomState(4)
    f = BoxQPFunction(verbose=-1, duals=True, dense_Q=dense_Q)
    z, lam, nu = f(*(leaves[k] for k in NAMES))
    wz, wl = torch.tensor(rs.randn(B, n), dtype=dtype), torch.tensor(rs.randn(*lam.shape), dtype=dtype)
    loss = (wz * z).sum() + (wl * lam).sum()
    g1 = torch.autograd.grad(loss, [leaves[k] for k in keys], create_graph=True)
    assert box_stand_ins == ["backward"]
    g0 = torch.autograd.grad(loss, [leaves[k] for k in keys], retain_graph=True)
    for a, b_ in zip(g1, g0):                            # first order unchanged under create_graph=True
        assert a.dtype == dtype and torch.equal(a.detach(), b_)
    om = {k: torch.tensor(rs.randn(*leaves[k].shape), dtype=dtype) for k in keys}
    om_none = keys[1]                                     # a None cotangent: that gradient is not in phi
    phi = sum((om[k] * g).sum() for k, g in zip(keys, g1) if k != om_none)
    g2 = torch.autograd.grad(phi, [leaves[k] for k in keys], retain_graph=True, allow_unused=True)
    assert box_stand_ins[1:] == ["backward", "double_backward"]
    st = f.last_solve()
    pt = dict(z=st.zhat, lam=st.lam, s=st.slacks, nu=st.nus if e else torch.zeros(B, 0, dtype=torch.float64))
    mins = {k: (None if v is None else (v if v.numel() else (torch.zeros(B, 0, n, dtype=torch.float64) if k == "A"
                                                             else torch.zeros(B, 0, dtype=torch.float64))))
            for k, v in ins.items()}
    sh = tuple(k for k in shared if mins[k] is not None and mins[k].numel())
    ref = bdm.double_backward(mins, pt, wz.double(), wl.double(), None,
                              {k: (om[k].double() if (k in om and k != om_none) else None) for k in NAMES}, sh,
                              dense_Q)
    tol = 1e-9 if dtype == torch.float64 else 2e-3
    for k, a in zip(keys, g2):
        r = ref[k]
        assert a is not None and a.dtype == dtype and a.shape == leaves[k].shape, k
        assert torch.allclose(a.double(), r, rtol=tol, atol=tol * max(1.0, float(r.abs().max()))), k
    with pytest.raises(RuntimeError, match="third-order"):
        torch.autograd.grad(phi, [leaves[k] for k in keys], create_graph=True)


def test_without_create_graph_the_first_order_calls_are_made(box_stand_ins):
    from qpth_b200 import BoxQPFunction
    ins = _box_problem(6, 2, "both", 2, 9)
    leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
    z = BoxQPFunction(verbose=-1)(*(leaves[k] for k in NAMES))
    z.sum().backward()
    assert box_stand_ins == ["backward"]
    assert all(leaves[k].grad is not None and leaves[k].grad.grad_fn is None for k in NAMES)


@pytest.mark.parametrize("shared", [False, True])
def test_dense_fallback_gradgradcheck(stand_ins, monkeypatch, shared):  # noqa: F811
    """The dense fallback (no box kernel covers the shape) under create_graph: QPFunction's double backward on the
    dense equivalent, mapped back with torch ops, passes gradgradcheck (QPFunction's solves replaced by dense
    stand-ins)."""
    from qpth_b200 import BoxQPFunction, box, qp
    monkeypatch.setattr(box, "solve_box_forward", lambda *a, **k: None)
    inner = qp.solve_forward

    def fwd(*a, **k):
        st = inner(*a, **k)
        st.device, st.iters, st.best_resid, st.trace = torch.device("cpu"), None, None, None
        return st
    monkeypatch.setattr(qp, "solve_forward", fwd)
    B = 2
    prs = [dm.complementary_box(41 if shared else 41 + i, 6, 2, "both") for i in range(B)]
    T = lambda k: _T(prs[0][k]) if (shared and k in ("A", "b", "lb")) else _T(np.stack([p_[k] for p_ in prs]))
    ins = tuple(T(k).requires_grad_(True) for k in NAMES)
    f = BoxQPFunction(verbose=-1, duals=True)

    def fn(*a):
        z, lam, nu = f(*a)
        return z, lam
    assert torch.autograd.gradgradcheck(fn, ins, atol=1e-5, rtol=1e-4)
    assert B == ins[1].shape[0]


# ---- the C ABI -----------------------------------------------------------------------------------------------------

NEW = ("qpb200_box_double_backward", "qpb200_boxq_double_backward")


@pytest.fixture(scope="module")
def lib():
    from qpth_b200 import _lib, build
    build.build()
    return _lib.load()


def test_symbols_declared_exported_typed_and_version(lib):
    from qpth_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "qpth_b200.h")).read()
    for name in NEW:
        assert re.search(r"\b%s\s*\(" % name, hdr), name
        assert hasattr(lib, name) and name in _lib.SIGNATURES, name
        # plan, B, q / Q and A with strides, six (w, stride), v, the point, gg, six (grad, sum), work, stream
        assert len(_lib.SIGNATURES[name][1]) == 2 + 4 + 12 + 3 + 4 + 3 + 12 + 2, name
    assert lib.qpb200_version() == 103


def _box_plan(lib, n, e, lb, ub, dense_Q=False):
    from qpth_b200 import _lib
    p = _lib.BoxQPlan() if dense_Q else _lib.BoxPlan()
    fn = lib.qpb200_boxq_plan_init if dense_Q else lib.qpb200_box_plan_init
    assert fn(n, e, lb, ub, ctypes.byref(p)) == 0
    return p


@pytest.mark.parametrize("dense_Q", [False, True], ids=["box", "boxq"])
def test_bad_arguments_are_refused_before_any_launch(lib, dense_Q):
    """Every call fails its argument checks, which run before any CUDA call (without a GPU a late check would return
    QPB200_ERR_CUDA). The pointers are never dereferenced."""
    P, N = ctypes.c_void_p(16), None
    plan = _box_plan(lib, 20, 0, 1, 0, dense_Q)          # lb only, no equality rows
    plan_eq = _box_plan(lib, 20, 5, 1, 1, dense_Q)
    fn = lib.qpb200_boxq_double_backward if dense_Q else lib.qpb200_box_double_backward

    def call(pl, B=2, oms=None, v=(P, P, N), gg=(P, P, N), grads=None, work=P, q=P):
        oms = oms or [N, 0] * 6
        grads = grads or [N, 0] * 6
        return fn(ctypes.byref(pl), B, q, 0, P, 0, *oms, *v, P, P, P, P, *gg, *grads, work, N)

    assert call(plan, gg=(P, P, P)) == 1                                   # gg_nu without equality rows
    assert call(plan, oms=[N, 0] * 2 + [P, 0] + [N, 0] * 3) == 1           # wA without equality rows
    assert call(plan, oms=[N, 0] * 3 + [P, 0] + [N, 0] * 2) == 1           # wb without equality rows
    assert call(plan, grads=[N, 0] * 4 + [P, 0, N, 0]) == 1                # dA without equality rows
    assert call(plan, grads=[N, 0] * 5 + [P, 0]) == 1                      # db without equality rows
    assert call(plan, oms=[N, 0] * 5 + [P, 0]) == 1                        # wub with no ub side
    assert call(plan, grads=[N, 0] * 3 + [P, 0] + [N, 0] * 2) == 1         # dub with no ub side
    assert call(plan, B=0) == 1
    assert call(plan, work=N) == 1
    assert call(plan, q=N) == 1
    assert call(plan, v=(N, P, N)) == 1
    assert call(plan, v=(P, N, N)) == 1
    assert call(plan, oms=[P, -1] + [N, 0] * 5) == 1                       # a negative stride
    assert call(plan, oms=[N, 0, P, -3] + [N, 0] * 4) == 1
    assert call(plan_eq, gg=(P, P, P)) == 1                                # neq > 0 needs dnuv
    assert call(plan_eq, v=(P, P, P)) == 1                                 # ... and gg_nu
    assert call(plan_eq, v=(P, P, P), gg=(P, P, P), q=N) == 1
    lb_only = _box_plan(lib, 20, 5, 0, 1, dense_Q)                         # ub only: wlb / dlb refused
    assert call(lb_only, v=(P, P, P), gg=(P, P, P), oms=[N, 0] * 4 + [P, 0, N, 0]) == 1
    assert call(lb_only, v=(P, P, P), gg=(P, P, P), grads=[N, 0] * 2 + [P, 0] + [N, 0] * 3) == 1


def box_jvp_smem_bytes(n, e, threads=256):
    """k_box_ggrad_rhs's dynamic shared memory (qp_box.cu box_jvp_smem_bytes): vx (n), vnu and the cnu accumulator (e),
    the column partials of jvp::contract (threads / 32 warps x 128 doubles)"""
    r8 = lambda v: (v + 7) & ~7
    return (r8(n) + 2 * r8(e) + (threads // 32) * 128) * 8


def boxq_jvp_smem_bytes(n, e, threads=256):
    """k_boxq_ggrad_rhs's (qp_boxq.cu boxq_jvp_smem_bytes): vx and cz (n), vnu and cnu (e), the column partials"""
    r8 = lambda v: (v + 7) & ~7
    return (2 * r8(n) + 2 * r8(e) + (threads // 32) * 128) * 8


def test_ggrad_rhs_shared_memory_fits_every_plan(lib):
    """k_box_ggrad_rhs over every shape qpb200_box_plan_init accepts (nz up to 16384, neq up to 4096), and
    k_boxq_ggrad_rhs over every qpb200_boxq_plan with ok = 1, stay within the 227 KB a CTA can have."""
    from qpth_b200 import _lib
    worst = 0
    for n in (1, 7, 8, 100, 729, 1000, 4096, 11008, 16383, 16384, 16385):
        for e in (0, 1, 8, 249, 1000, 4095, 4096, 4097):
            p = _lib.BoxPlan()
            if lib.qpb200_box_plan_init(n, e, 1, 1, ctypes.byref(p)) != 0:
                continue
            worst = max(worst, box_jvp_smem_bytes(n, e))
    assert 0 < worst <= 227 * 1024, worst
    assert box_jvp_smem_bytes(16384, 4096) == 200 * 1024
    worst = 0
    for n in range(1, 257, 3):
        for e in range(0, 257, 5):
            p = _lib.BoxQPlan()
            assert lib.qpb200_boxq_plan_init(n, e, 1, 1, ctypes.byref(p)) == 0
            if p.ok:
                worst = max(worst, boxq_jvp_smem_bytes(n, e))
    assert 0 < worst <= 227 * 1024, worst


# ---- ptxas report of the new kernels --------------------------------------------------------------------------------
# nvcc 12.9 for sm_90a: registers at most these, and no stack frame or spills
GG_REGISTERS = {("qp_box.cu", "k_box_ggrad_rhs"): 64, ("qp_box.cu", "k_box_ggrad_out"): 40,
                ("qp_box.cu", "k_box_ggrad_sum_vec"): 32, ("qp_boxq.cu", "k_boxq_ggrad_rhs"): 64}


@pytest.mark.parametrize("unit", ["qp_box.cu", "qp_boxq.cu"])
def test_ggrad_ptxas_report(unit):
    from tests.test_local_memory_cpu import _nvcc, parse_ptxas
    from qpth_b200 import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    (src, defs, tag), = [u for u in build.UNITS if u[0] == unit]
    with tempfile.TemporaryDirectory() as tmp:
        cmd = ([nvcc] + build.GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
               + defs + ["-c", "-o", os.path.join(tmp, tag + ".o"), os.path.join(ROOT, "qpth_b200", "csrc", src)])
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    rep = parse_ptxas(r.stderr)
    regs = {}
    entry = None
    for line in r.stderr.splitlines():
        mt = re.search(r"Compiling entry function '(\w+)'", line)
        if mt:
            entry = mt.group(1)
        mt = re.search(r"Used (\d+) registers", line)
        if mt and entry:
            regs[entry] = int(mt.group(1))
    for (u, name), limit in GG_REGISTERS.items():
        if u != unit:
            continue
        (entry, funcs), = [(k, v) for k, v in rep.items() if re.search(r"%d%sE" % (len(name), name), k)]
        assert all(f[1:] == (0, 0, 0) for f in funcs), funcs
        assert regs[entry] <= limit, (name, regs[entry])
