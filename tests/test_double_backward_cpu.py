"""Second order of QPFunction / QPSolutionFunction on the CPU: the model it rests on, the algebra the kernels implement,
the host logic, and the C ABI boundary of qpb200_double_backward(_reg).

- The dense torch model (tests/double_backward_models.py) against central differences of the dense first-order
  gradient (tests/dual_models.backward_one at tight re-solves) within 1e-6, on strictly complementary problems.
- `algebra`, the double backward as qpb200_double_backward computes it (one JVP solve, k_ggrad_rhs's cotangents, one
  dual backward solve, the bilinear terms), written with dense solves, against the model within 1e-10, batched and with
  un-batched inputs.
- QPFunction's host logic with solve_forward, solve_backward and solve_double_backward replaced by dense stand-ins:
  torch.autograd.grad with create_graph=True, the mean / sum conventions, None cotangents, first order bit-identical
  under create_graph=True, third order raising; the equality-only path (torch on the host) by gradgradcheck.
- The entry points are declared, exported and typed, refuse bad arguments before any launch, the version is 103,
  k_ggrad_rhs's shared memory fits every shape qpb200_plan_init takes, and the new kernels' ptxas report.
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
from tests import double_backward_models as dbm
from tests import dual_models as dm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = dbm.NAMES
SHAPES = [(8, 10, 3), (12, 15, 0), (10, 9, 4)]


def _T(a):
    return torch.tensor(np.asarray(a, dtype=np.float64))


def _problem(n, m, e, B=1, seed=0):
    """A batch of complementary_qp problems and their solutions as torch tensors (B, ...)."""
    prs = [dm.complementary_qp(seed + 97 * i + 23 * n + m + e, n, m, e) for i in range(B)]
    ins = {k: _T(np.stack([pr[k] for pr in prs])) for k in NAMES}
    pt = {k: _T(np.stack([pr[k] for pr in prs])) for k in ("z", "lam", "s", "nu")}
    return ins, pt


def _omegas(ins, rs, keys=NAMES, shared=()):
    out = {}
    for k in NAMES:
        if k not in keys or ins[k].numel() == 0:
            out[k] = None
        else:
            shp = ins[k].shape[1:] if k in shared else ins[k].shape
            out[k] = _T(rs.randn(*shp))
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_model_matches_central_differences(shape):
    """d/de <w, grad(theta + e t)> by central differences of the dense first-order gradient at re-solved points, against
    <model's second-order gradient, t>, along a direction t of every input (Q symmetric) and of the adjoints."""
    n, m, e = shape
    pr = dm.complementary_qp(23 * n + m + e, n, m, e)
    rs = np.random.RandomState(n + 3 * m)
    gz, glam, gnu = rs.randn(n), rs.randn(m), (rs.randn(e) if e else None)
    om = {k: rs.randn(*np.shape(pr[k])) if np.size(pr[k]) else None for k in NAMES}
    tan = {k: rs.randn(*np.shape(pr[k])) if np.size(pr[k]) else None for k in NAMES}
    tan["Q"] = tan["Q"] + tan["Q"].T
    tg = dict(gz=rs.randn(n), glam=rs.randn(m), gnu=rs.randn(e) if e else None)

    def phi(eps):
        x = {k: (pr[k] + eps * tan[k] if tan[k] is not None else pr[k]) for k in NAMES}
        sol = km.solve_one(*(x[k] for k in NAMES), eps=1e-15, maxIter=60, stall_tol=1e-7, tie=1.5)
        g = dm.backward_one(sol, gz + eps * tg["gz"], glam + eps * tg["glam"],
                            None if gnu is None else gnu + eps * tg["gnu"])
        return sum(np.sum(om[k] * g["d" + k]) for k in NAMES if om[k] is not None)

    h = 1e-5
    fd = (phi(h) - phi(-h)) / (2 * h)
    ins = {k: _T(pr[k])[None] if np.size(pr[k]) else _T(np.zeros((1, 0) + np.shape(pr[k])[1:])) for k in NAMES}
    if e == 0:
        ins["A"], ins["b"] = torch.zeros(1, 0, n, dtype=torch.float64), torch.zeros(1, 0, dtype=torch.float64)
    pt = {k: _T(pr[k])[None] for k in ("z", "lam", "s")}
    pt["nu"] = _T(pr["nu"])[None] if e else torch.zeros(1, 0, dtype=torch.float64)
    r = dbm.double_backward(ins, pt, _T(gz)[None], _T(glam)[None], _T(gnu)[None] if e else None,
                            {k: (None if om[k] is None else _T(om[k])[None]) for k in NAMES})
    an = sum(float((r[k][0] * _T(tan[k])).sum()) for k in NAMES if tan[k] is not None)
    an += float((r["gz"][0] * _T(tg["gz"])).sum()) + float((r["glam"][0] * _T(tg["glam"])).sum())
    if e:
        an += float((r["gnu"][0] * _T(tg["gnu"])).sum())
    assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (fd, an)


# ---- the algebra of qpb200_double_backward, with dense solves ---------------------------------------------------------

def _kkt(Q, G, A, lam, s):
    B, m, n = G.shape
    e = A.shape[1]
    Qs = 0.5 * (Q + Q.transpose(1, 2))
    D = lam.clamp(min=1e-8) / s.clamp(min=1e-8)
    K = torch.zeros(B, n + 2 * m + e, n + 2 * m + e, dtype=torch.float64)
    K[:, :n, :n] = Qs
    K[:, :n, n + m:n + 2 * m] = G.transpose(1, 2)
    K[:, :n, n + 2 * m:] = A.transpose(1, 2)
    K[:, n:n + m, n:n + m] = torch.diag_embed(D)
    K[:, n:n + m, n + m:n + 2 * m] = torch.eye(m)
    K[:, n + m:n + 2 * m, :n] = G
    K[:, n + m:n + 2 * m, n:n + m] = torch.eye(m)
    K[:, n + 2 * m:, :n] = A
    return K, D


def _ksolve(K, n, m, rx, rz, ry):
    """(x, lam, nu) parts of -K^-1 [rx; 0; rz; ry]."""
    B = rx.shape[0]
    rhs = torch.cat([rx, torch.zeros(B, m, dtype=rx.dtype), rz, ry], 1)
    v = torch.linalg.solve(K, -rhs.unsqueeze(2)).squeeze(2)
    return v[:, :n], v[:, n + m:n + 2 * m], v[:, n + 2 * m:]


def _mv(M, x):
    return torch.matmul(M, x.unsqueeze(-1)).squeeze(-1)


def _outer(a, b):
    return a.unsqueeze(2) * b.unsqueeze(1)


def algebra(Q, G, A, z, lam, s, nu, v, omegas, flags):
    """The double backward as the kernels compute it: (gz, glam, gnu, dQ, dp, dG, dh, dA, db), with batched Q, G, A
    (B, ...), v = (vx, vlam, vnu), omegas shaped as the first-order gradients and flags their mean flags."""
    B, m, n = G.shape
    e = A.shape[1]
    K, D = _kkt(Q, G, A, lam, s)
    vx, vl, vn = v
    w = [None if om is None else (om / B if f else om) for om, f in zip(omegas, flags)]
    zero = lambda k: torch.zeros(B, k, dtype=torch.float64)
    sym = lambda M: 0.5 * (M + M.transpose(-1, -2))
    wQ, wp, wG, wh, wA, wb = w
    rx, rz, ry = zero(n), zero(m), zero(e)
    cz, cl, cn = zero(n), zero(m), zero(e)
    if wQ is not None:
        rx, cz = rx + _mv(sym(wQ), z), cz + _mv(sym(wQ), vx)
    if wp is not None:
        rx = rx + wp
    if wG is not None:
        rx, rz = rx + _mv(wG.transpose(-1, -2), lam), rz + _mv(wG, z)
        cz, cl = cz + _mv(wG.transpose(-1, -2), vl), cl + _mv(wG, vx)
    if wh is not None:
        rz = rz - wh
    if wA is not None:
        rx, ry = rx + _mv(wA.transpose(-1, -2), nu), ry + _mv(wA, z)
        cz, cn = cz + _mv(wA.transpose(-1, -2), vn), cn + _mv(wA, vx)
    if wb is not None:
        ry = ry - wb
    ux, ul, un = _ksolve(K, n, m, rx, rz, ry)
    sc = s.clamp(min=1e-8)
    cD = (ul / D) * (vl / D)
    c_lam = torch.where(lam >= 1e-8, cD / sc, torch.zeros_like(cD))
    c_s = torch.where(s >= 1e-8, -cD * D / sc, torch.zeros_like(cD))
    cz = cz - _mv(G.transpose(1, 2), c_s)
    cl = cl + c_lam
    wx, wl, wn = _ksolve(K, n, m, cz, cl, cn)
    t = wl - c_s
    g = [sym(_outer(wx, z) + _outer(ux, vx)), wx, _outer(t, z) + _outer(lam, wx) + _outer(vl, ux) + _outer(ul, vx),
         -t, _outer(wn, z) + _outer(nu, wx) + _outer(vn, ux) + _outer(un, vx), -wn]
    return [ux, ul, un] + [x.sum(0) if f else x for x, f in zip(g, flags)]


@pytest.mark.parametrize("shared", [(), ("Q", "G", "A"), ("p", "h", "b")], ids=["batched", "shared_QGA", "shared_phb"])
@pytest.mark.parametrize("shape", SHAPES, ids=["%dx%dx%d" % s for s in SHAPES])
def test_algebra_matches_the_model(shape, shared):
    n, m, e = shape
    B = 3
    ins, pt = _problem(n, m, e, B, seed=5)
    # one point with a clamped slack and one with a clamped dual: the clamps' derivative conventions
    pt["s"][1, 0], pt["lam"][2, 0] = 1e-9, 1e-9
    rs = np.random.RandomState(11 + n)
    ins = {k: (v[0] if k in shared else v) for k, v in ins.items()}
    gz, glam = _T(rs.randn(B, n)), _T(rs.randn(B, m))
    gnu = _T(rs.randn(B, e)) if e else None
    om = _omegas({k: (v.unsqueeze(0).expand(B, *v.shape) if k in shared else v) for k, v in ins.items()}, rs,
                 shared=shared)
    ref = dbm.double_backward(ins, pt, gz, glam, gnu, om, shared)
    full = {k: (v.unsqueeze(0).expand(B, *v.shape) if k in shared else v) for k, v in ins.items()}
    K, _ = _kkt(full["Q"], full["G"], full["A"], pt["lam"], pt["s"])
    v = _ksolve(K, n, m, gz, glam, gnu if e else torch.zeros(B, 0, dtype=torch.float64))
    flags = [k in shared for k in NAMES]
    got = algebra(full["Q"], full["G"], full["A"], pt["z"], pt["lam"], pt["s"], pt["nu"], v,
                  [om[k] for k in NAMES], flags)
    keys = ["gz", "glam", "gnu"] + list(NAMES)
    for k, x in zip(keys, got):
        if k in ref and ref[k].numel():
            scale = max(1.0, float(ref[k].abs().max()))
            assert float((x - ref[k]).abs().max()) <= 1e-10 * scale, k


# ---- QPFunction's host logic with dense stand-ins --------------------------------------------------------------------

class _Plan:
    def __init__(self, n, m, e):
        self.nz, self.nineq, self.neq = n, m, e


@pytest.fixture
def stand_ins(monkeypatch):
    """solve_forward, solve_backward and solve_double_backward on the CPU with dense solves (model points)."""
    from qpth_b200 import qp
    calls = []

    def fwd(Q_, p_, G_, h_, A_, b_, *a, **k):
        nB, n, m, e = qp.check_shapes(Q_, p_, G_, h_, A_, b_)
        exp = lambda X, nd: qp.expandParam(X.detach().double(), nB, nd)[0]
        Q, p, G, h = exp(Q_, 3), exp(p_, 2), exp(G_, 3), exp(h_, 2)
        A = exp(A_, 3) if e else torch.zeros(nB, 0, n, dtype=torch.float64)
        b = exp(b_, 2) if e else torch.zeros(nB, 0, dtype=torch.float64)
        sols = [km.solve_one(*(x[i].numpy() for x in (Q, p, G, h)), A[i].numpy() if e else np.zeros((0, n)),
                             b[i].numpy() if e else np.zeros(0), eps=1e-14, maxIter=40, stall_tol=1e-6, tie=1.5)
                for i in range(nB)]
        st = types.SimpleNamespace(plan=_Plan(n, m, e), nBatch=nB, Q=Q, G=G, A=A, reg=False)
        st.zhat = _T(np.stack([s_["x"] for s_ in sols]))
        st.lam = _T(np.stack([s_["lam"] for s_ in sols]))
        st.slacks = _T(np.stack([s_["s"] for s_ in sols]))
        st.nus = _T(np.stack([s_["nu"] for s_ in sols])) if e else None
        return st

    def bwd(st, dl, flags, want, glam=None, gnu=None, keep=False):
        calls.append("backward")
        n, m, e = st.plan.nz, st.plan.nineq, st.plan.neq
        B = st.nBatch
        K, _ = _kkt(st.Q, st.G, st.A, st.lam, st.slacks)
        z0 = lambda k: torch.zeros(B, k, dtype=torch.float64)
        f = lambda g, k: z0(k) if g is None else g.detach().double().reshape(B, k)
        v = _ksolve(K, n, m, f(dl, n), f(glam, m), f(gnu, e))
        vx, vl, vn = v
        z, lam, nu = st.zhat, st.lam, st.nus if e else z0(0)
        g = [0.5 * (_outer(vx, z) + _outer(z, vx)), vx, _outer(vl, z) + _outer(lam, vx), -vl,
             _outer(vn, z) + _outer(nu, vx), -vn]
        outs = [None if (not want[k] or (k >= 4 and e == 0)) else (g[k].mean(0) if flags[k] else g[k])
                for k in range(6)]
        return (outs, (vx, vl, vn if e else None)) if keep else outs

    def dbl(st, v, omegas, flags, want, G):
        calls.append("double_backward")
        e = st.plan.neq
        vx, vl, vn = v
        nu = st.nus if e else torch.zeros(st.nBatch, 0, dtype=torch.float64)
        om = [None if (w is None or (k >= 4 and e == 0)) else w.detach().double() for k, w in enumerate(omegas)]
        res = algebra(st.Q, st.G, st.A, st.zhat, st.lam, st.slacks, nu,
                      (vx, vl, vn if e else torch.zeros(st.nBatch, 0, dtype=torch.float64)), om, flags)
        res = [None if (k >= 3 and not want[k - 3]) else r for k, r in enumerate(res)]
        if e == 0:
            res[2] = res[7] = res[8] = None
        return res

    monkeypatch.setattr(qp, "solve_forward", fwd)
    monkeypatch.setattr(qp, "solve_backward", bwd)
    monkeypatch.setattr(qp, "solve_double_backward", dbl)
    return calls


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("shared", [(), ("Q", "G", "A", "h")], ids=["batched", "shared"])
@pytest.mark.parametrize("shape", [(8, 10, 3), (9, 12, 0)], ids=["8x10x3", "9x12x0"])
def test_qpfunction_second_order_through_the_host_logic(stand_ins, shape, shared, dtype):
    from qpth_b200 import QPFunction
    n, m, e = shape
    B = 3
    ins, pt = _problem(n, m, e, B, seed=2)
    ins = {k: (v[0] if k in shared else v) for k, v in ins.items()}
    if e == 0:
        ins["A"], ins["b"] = torch.Tensor().double(), torch.Tensor().double()
    leaves = {k: v.to(dtype).clone().requires_grad_(v.numel() > 0) for k, v in ins.items()}
    rs = np.random.RandomState(4)
    f = QPFunction(verbose=-1, duals=True)
    z, lam, nu = f(*(leaves[k] for k in NAMES))
    wz, wl = torch.tensor(rs.randn(B, n), dtype=dtype), torch.tensor(rs.randn(B, m), dtype=dtype)
    # with batched inputs the adjoint g_z = wz + 2 z also depends on z, so the second order flows through the first
    # backward again; with un-batched ones that backward returns a batch mean, not the model's derivative: g_z = wz
    sq = not shared
    loss = (wz * z).sum() + (wl * lam).sum() + ((z ** 2).sum() if sq else 0.0)
    want = [k for k in NAMES if leaves[k].requires_grad]
    g1 = torch.autograd.grad(loss, [leaves[k] for k in want], create_graph=True)
    assert stand_ins == ["backward"]
    g0 = torch.autograd.grad(loss, [leaves[k] for k in want], retain_graph=True)
    for a, b_ in zip(g1, g0):                            # first order unchanged under create_graph=True
        assert a.dtype == dtype and torch.equal(a.detach(), b_)
    om = {k: torch.tensor(rs.randn(*leaves[k].shape), dtype=dtype) for k in want}
    phi = sum((om[k] * g).sum() for k, g in zip(want, g1))
    g2 = torch.autograd.grad(phi, [leaves[k] for k in want], retain_graph=True)
    # the double backward, then (batched) the first backward again for its gradient of g_z through z
    assert stand_ins[1:] == ["backward", "double_backward"] + (["backward"] if sq else [])
    # the reference: the model at the returned point; the loss's adjoints g_z = wz + 2 z, g_lam = wl depend on z
    st_pt = dict(z=z.detach().double(), lam=lam.detach().double(), s=None, nu=nu.detach().double())
    from qpth_b200 import qp
    st = qp.solve_forward(*(ins[k] for k in NAMES))
    st_pt["s"] = st.slacks
    st_pt["z"], st_pt["lam"] = st.zhat, st.lam
    st_pt["nu"] = st.nus if e else torch.zeros(B, 0, dtype=torch.float64)
    mins = {k: (v if v.numel() else (torch.zeros(B, 0, n, dtype=torch.float64) if k == "A"
                                     else torch.zeros(B, 0, dtype=torch.float64))) for k, v in ins.items()}
    lv = {k: v.clone().requires_grad_(True) for k, v in mins.items()}
    zz, ll, nn = dbm._Point.apply(st_pt, *(lv[k].unsqueeze(0).expand(B, *lv[k].shape) if k in want and k in shared
                                           else lv[k]
                                           for k in NAMES))
    L = (wz.double() * zz).sum() + (wl.double() * ll).sum() + ((zz ** 2).sum() if sq else 0.0)
    r1 = torch.autograd.grad(L, [lv[k] for k in want], create_graph=True)
    r1 = [(g / B if k in shared else g) for k, g in zip(want, r1)]   # the first backward returns the batch mean
    ph = sum((om[k].double() * g).sum() for k, g in zip(want, r1))
    r2 = torch.autograd.grad(ph, [lv[k] for k in want])
    tol = 1e-9 if dtype == torch.float64 else 2e-3
    for k, a, b_ in zip(want, g2, r2):
        assert a.dtype == dtype and a.shape == leaves[k].shape
        assert torch.allclose(a.double(), b_, rtol=tol, atol=tol * max(1.0, float(b_.abs().max()))), k
    with pytest.raises(RuntimeError, match="third-order"):
        torch.autograd.grad(phi, [leaves[k] for k in want], create_graph=True)


@pytest.mark.parametrize("shared", [False, True])
def test_equality_only_gradgradcheck(shared, monkeypatch):
    from qpth_b200 import QPFunction, eqonly
    from tests.test_eqonly_cpu import DenseFactor
    monkeypatch.setattr(eqonly, "_factor", DenseFactor)
    monkeypatch.setattr(eqonly, "_target_device", lambda Q_: torch.device("cpu"))
    rs = np.random.RandomState(6)
    B, nz, neq = 3, 5, 2
    M = torch.tensor(rs.randn(nz, nz) if shared else rs.randn(B, nz, nz), requires_grad=True)
    p = torch.tensor(rs.randn(B, nz), requires_grad=True)
    A = torch.tensor(rs.randn(neq, nz) if shared else rs.randn(B, neq, nz), requires_grad=True)
    b = torch.tensor(rs.randn(neq) if shared else rs.randn(B, neq), requires_grad=True)
    e = torch.Tensor().double()
    f = QPFunction(verbose=-1, duals=True)

    def fn(M, p, A, b):                      # Q = M M' + I: symmetric perturbations only (one triangle is read)
        z, _, nu = f(M @ M.transpose(-1, -2) + torch.eye(nz, dtype=torch.float64), p, e, e, A, b)
        return z, nu
    assert torch.autograd.gradgradcheck(fn, (M, p, A, b), atol=1e-6, rtol=1e-5)
    z, nu = fn(M, p, A, b)
    g = torch.autograd.grad((z ** 2).sum() + nu.sum(), p, create_graph=True)[0]
    with pytest.raises(RuntimeError, match="third-order"):
        torch.autograd.grad(g.sum(), p, create_graph=True)


# ---- the C ABI -----------------------------------------------------------------------------------------------------

NEW = ("qpb200_double_backward", "qpb200_double_backward_reg")


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
    assert "QPB200_DOUBLE_BACKWARD_WORK" in hdr
    assert lib.qpb200_version() == 103
    # (w, stride) x 6, G and its stride, v x 3 in place of the JVP's tangents, rhs and outputs; reg adds reg_eps, ir_steps
    assert len(_lib.SIGNATURES["qpb200_double_backward_reg"][1]) == len(_lib.SIGNATURES["qpb200_double_backward"][1]) + 2


def test_bad_arguments_are_refused_before_any_launch(lib):
    """Every call fails its argument checks, which run before any CUDA call (without a GPU a late check would return
    QPB200_ERR_CUDA). The pointers are never dereferenced."""
    from qpth_b200 import _lib
    P, N = ctypes.c_void_p(16), None
    plan = _lib.plan_for(20, 15, 0)
    plan_eq = _lib.plan_for(20, 15, 5)

    def call(pl, B=2, oms=None, G=P, sG=0, v=(P, P, N), gg=(P, P, N), grads=None, work=P, reg=None):
        oms = oms or [N, 0] * 6
        grads = grads or [N, 0] * 6
        fn = lib.qpb200_double_backward_reg if reg else lib.qpb200_double_backward
        return fn(ctypes.byref(pl), B, *oms, G, sG, *v, P, P, P, P, P, P, P, 1, *(reg or ()), *gg, *grads, work, P, N)

    for reg in (None, (1e-7, 1)):
        assert call(plan, reg=reg, gg=(P, P, P)) == 1                               # gg_nu without equality rows
        assert call(plan, reg=reg, oms=[N, 0] * 4 + [P, 0, N, 0]) == 1              # wA without equality rows
        assert call(plan, reg=reg, grads=[N, 0] * 4 + [P, 0, N, 0]) == 1            # dA without equality rows
        assert call(plan, reg=reg, B=0) == 1
        assert call(plan, reg=reg, work=N) == 1
        assert call(plan, reg=reg, G=N) == 1
        assert call(plan, reg=reg, sG=-1) == 1
        assert call(plan, reg=reg, v=(N, P, N)) == 1
        assert call(plan, reg=reg, oms=[P, -1] + [N, 0] * 5) == 1
        assert call(plan_eq, reg=reg, gg=(P, P, P)) == 1                            # neq > 0 needs dnuv
        assert call(plan_eq, reg=reg, v=(P, P, P)) == 1                             # ... and gg_nu
    assert call(plan, reg=(-1.0, 1)) == 1


def ggrad_smem_bytes(n, m, e, threads=256):
    """k_ggrad_rhs's dynamic shared memory: jvp_smem_bytes (qp_kernels.cu), vx, cz, c_s/vlam, clam, vnu, cnu and the
    column partials of jvp::contract (threads / 32 warps x 128 doubles)."""
    r8 = lambda v: (v + 7) & ~7
    return (2 * (r8(n) + r8(m) + r8(e)) + (threads // 32) * 128) * 8


def test_ggrad_shared_memory_fits_every_plan(lib):
    """Over a grid of shapes up to 4096 x 4096 x 4096: wherever qpb200_plan_init takes the shape, k_ggrad_rhs's shared
    memory is within the 227 KB a CTA can have."""
    from qpth_b200 import _lib
    worst = 0
    vals = [1, 7, 8, 100, 1000, 2048, 4095, 4096, 4097]
    for n in vals:
        for m in vals:
            for e in [0] + vals:
                p = _lib.Plan()
                if lib.qpb200_plan_init(n, m, e, ctypes.byref(p)) != 0:
                    continue
                worst = max(worst, ggrad_smem_bytes(n, m, e))
    assert 0 < worst <= 227 * 1024, worst
    assert ggrad_smem_bytes(4096, 4096, 4096) == 200 * 1024


# ---- ptxas report of the new kernels --------------------------------------------------------------------------------
# nvcc 12.9 for sm_90a: registers at most these, and no stack frame or spills
GG_REGISTERS = {"k_ggrad_rhs": 80, "k_ggrad_out": 40, "k_ggrad_sum": 80, "k_ggrad_sum_vec": 32}


def test_ggrad_ptxas_report():
    from tests.test_local_memory_cpu import _nvcc, parse_ptxas
    from qpth_b200 import build
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    (src, defs, tag), = [u for u in build.UNITS if u[0] == "qp_kernels.cu"]
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
    for name, limit in GG_REGISTERS.items():
        (entry, funcs), = [(k, v) for k, v in rep.items() if re.search(r"%d%sE" % (len(name), name), k)]
        assert all(f[1:] == (0, 0, 0) for f in funcs), funcs
        assert regs[entry] <= limit, (name, regs[entry])
