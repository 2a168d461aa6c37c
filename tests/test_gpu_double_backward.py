"""Second order of QPFunction and QPSolutionFunction on the GPU (qpb200_double_backward and its _reg variant).

- Model agreement: every family of tests/kernel_families.py (tests/double_backward_jobs.py; the `child` families in a
  child process), at its dual point, through QPSolutionFunction with create_graph=True: the gradients of
  sum <w_X, grad_X> with respect to (g_z, g_lam, g_nu) and every input against the dense model
  (tests/double_backward_models.py) within 1e-10 per-QP relative, with every input batched, with un-batched Q, G, A and
  with un-batched p, h, b. The equality-only path within 1e-10 (1e-9 with IR_UNOPT).
- Every family of tests/reg_families.py (KKTSolvers.IR_UNOPT) at IR_STEPS 0 .. 3: within max(1e-12, 10 x the model's own
  error) of the same algebra with the regularised model's solves (oracle/reg_model), the model's error taken against the
  exact dense solve.
- Identities: the gradient of g is solve_jvp with tangents w (w / B for un-batched inputs) bit for bit; the Hessian of a
  scalar of z(p) is symmetric, its blocks between different QPs are zero, and on a strictly complementary batch the
  p-Hessian of 1/2 ||z||^2 is J'J from jacobian() within 1e-6.
- End to end on strictly complementary batches: central differences of first-order gradients in the Q, G, A, h and b
  directions, and gradgradcheck.
- First order under create_graph=True is bit-identical to first order without it; third order raises.
"""
import numpy as np
import pytest
import torch

from tests import double_backward_models as dbm
from tests import dual_models as dm
from tests.double_backward_jobs import ADJ, SHARED, case_data, job_name, on_gpu, run_child, second_order
from tests.kernel_families import cases, family_env, family_plan, ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAMES = dbm.NAMES


def _T(a, dev=DEV):
    return torch.tensor(np.asarray(a, dtype=np.float64), device=dev)


def _rel_per_qp(got, ref, batched=True):
    g, r = got.detach().double().cpu(), ref.detach().double().cpu()
    if not batched:
        return float((g - r).abs().max() / max(float(r.abs().max()), 1e-300))
    g, r = g.reshape(g.shape[0], -1), r.reshape(r.shape[0], -1)
    return float(((g - r).abs().max(1).values / r.abs().max(1).values.clamp(min=1e-300)).max())


def _model(pr, ins, adj, om, shared):
    """The dense model (tests/double_backward_models.py) at the family point for the inputs of case_data."""
    B, n = pr["z"].shape
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64))
    cpu = {}
    for k in NAMES:
        if ins[k] is not None:
            cpu[k] = T(ins[k])
        else:                                          # no equality rows
            cpu[k] = torch.zeros(*((() if k in shared else (B,)) + ((0, n) if k == "A" else (0,))), dtype=torch.float64)
    pt = {k: T(pr[k]) for k in ("z", "lam", "s", "nu")}
    return dbm.double_backward(cpu, pt, *(None if adj[k] is None else T(adj[k]) for k in ADJ),
                               {k: (None if v is None else T(v)) for k, v in om.items()}, shared)


def _check_family(fam, shape, sharing, got):
    shared = SHARED[sharing]
    pr, ins, adj, om = case_data(fam, shape, sharing)
    ref = _model(pr, ins, adj, om, shared)
    want = [k for k in ADJ if adj[k] is not None] + [k for k in NAMES if ins[k] is not None]
    assert sorted(got) == sorted(want), (sorted(got), want)
    for k in want:
        err = _rel_per_qp(torch.tensor(got[k]), ref[k], batched=k not in shared)
        assert err <= 1e-10, (k, err)


@pytest.mark.parametrize("sharing", list(SHARED))
@pytest.mark.parametrize("fam,shape", cases(child=False), ids=ids(cases(child=False)))
def test_family_matches_the_model(fam, shape, sharing):
    _check_family(fam, shape, sharing, on_gpu(fam, shape, sharing))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("double_backward_families"))
    return out_dir, run_child(out_dir, timeout_s=900)


@pytest.mark.parametrize("sharing", list(SHARED))
@pytest.mark.parametrize("fam,shape", cases(child=True), ids=ids(cases(child=True)))
def test_family_matches_the_model_in_child(fam, shape, sharing, child_results):
    from tests import gpu_child
    with family_env(fam):
        family_plan(fam, shape)
    _check_family(fam, shape, sharing, gpu_child.load(*child_results, job_name(fam, shape, sharing)))


def _reg_cases():
    from tests.reg_families import CASES
    return CASES


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("case", _reg_cases(), ids=["%s-%s" % c for c in _reg_cases()])
def test_reg_family_matches_the_regularised_model(case, monkeypatch):
    """KKTSolvers.IR_UNOPT at IR_STEPS 0 .. 3 against the same algebra with the regularised model's solves and refinement
    steps (oracle/reg_model), within max(1e-12, 10 x that model's own error against the exact dense solve)."""
    from oracle import dense_kkt as dk
    from oracle import kernel_model as km
    from oracle import reg_model as rm
    from qpth_b200 import KKTSolvers, kkt
    from qpth_b200.solution import QPSolutionFunction
    from tests.reg_families import family_plan as reg_plan, problem
    from tests.test_gpu_reg_families import B, _point
    fam, kind = case
    probs = [problem(fam, kind, s) for s in range(B)]
    reg_plan(fam, probs[0])
    e = probs[0][4].shape[0]
    pts = [_point(c, i) for i, c in enumerate(probs)]
    pr = {k: np.stack([c[j] for c in probs]) for j, k in enumerate(NAMES)}
    pr.update(z=np.stack([q[0] for q in pts]), lam=np.stack([q[1] for q in pts]), s=np.stack([q[2] for q in pts]),
              nu=np.stack([q[3] for q in pts]))
    rs = np.random.RandomState(77)
    n, m = pr["z"].shape[1], pr["lam"].shape[1]
    adj = dict(gz=rs.randn(B, n), glam=rs.randn(B, m), gnu=rs.randn(B, e) if e else None)
    ins = {k: (None if (k in "Ab" and not e) else pr[k]) for k in NAMES}
    om = {k: (None if ins[k] is None else rs.randn(*ins[k].shape)) for k in NAMES}
    sol = [pr["z"], pr["lam"], pr["s"], pr["nu"]]

    def reference(i, solve):
        v = solve(adj["gz"][i], adj["glam"][i], adj["gnu"][i] if e else None)
        return dbm.double_backward_one(solve, pr["G"][i], pr["z"][i], pr["lam"][i], pr["s"][i],
                                       pr["nu"][i] if e else None, v, {k: (None if om[k] is None else om[k][i])
                                                                      for k in NAMES})

    def exact(i):
        d = np.maximum(pr["lam"][i], 1e-8) / np.maximum(pr["s"][i], 1e-8)

        def solve(rx, rz, ry):
            dx, _, dz, dy, _, _ = dk.solve(pr["Q"][i], pr["G"][i], pr["A"][i], d, rx, np.zeros(m), rz, ry, reg=0.0)
            return dx, dz, dy
        return solve

    def regularised(i, steps):
        f = km.setup(pr["Q"][i], pr["G"][i], pr["A"][i], kkt.IR_EPS)
        d = np.maximum(pr["lam"][i], 1e-8) / np.maximum(pr["s"][i], 1e-8)
        F = rm._factor(f, d, kkt.IR_EPS)

        def solve(rx, rz, ry):
            with np.errstate(all="ignore"):
                dx, _, dz, dy = rm._solve(f, F, kkt.IR_EPS, pr["Q"][i], pr["G"][i], pr["A"][i], rx, np.zeros(m), rz, ry,
                                          steps)
            return dx, dz, dy
        return solve

    dense = [reference(i, exact(i)) for i in range(B)]
    unique = ("gz", "glam", "Q", "p", "G", "h")           # nu, and so gnu, dA and db, are not unique for dependent rows
    for steps in range(4):
        monkeypatch.setattr(kkt, "IR_STEPS", steps)
        got = second_order(QPSolutionFunction(kkt_solver=KKTSolvers.IR_UNOPT, duals=True), ins, sol, adj, om)
        for i in range(B):
            model = reference(i, regularised(i, steps))
            tol = max(1e-12, 10 * max(_rel(model[k], dense[i][k]) for k in unique))
            for k, g in got.items():
                assert _rel(g[i], model[k]) <= tol, (steps, i, k, _rel(g[i], model[k]), tol)


@pytest.mark.parametrize("reg", [False, True], ids=["lu_partial", "ir_unopt"])
@pytest.mark.parametrize("shared", [False, True])
def test_equality_only_matches_the_model(shared, reg):
    """The torch double backward of the equality-only path against the model; with IR_UNOPT its solves are the
    regularised ones with EQ_IR_STEPS refinement steps, whose error against the exact solve is far below the bound."""
    from qpth_b200 import KKTSolvers, QPFunction
    rs = np.random.RandomState(9)
    B, n, e = 4, 12, 5
    M = rs.randn(n, n) if shared else rs.randn(B, n, n)
    Q = _T(M @ np.swapaxes(M, -1, -2) / n + np.eye(n)).requires_grad_(True)
    p = _T(rs.randn(B, n)).requires_grad_(True)
    A = _T(rs.randn(e, n) if shared else rs.randn(B, e, n)).requires_grad_(True)
    b = _T(rs.randn(B, e)).requires_grad_(True)
    emp = torch.Tensor().double().to(DEV)
    kkt_solver = KKTSolvers.IR_UNOPT if reg else KKTSolvers.LU_PARTIAL
    z, _, nu = QPFunction(verbose=-1, duals=True, kkt_solver=kkt_solver)(Q, p, emp, emp, A, b)
    gz, gnu = _T(rs.randn(B, n)).requires_grad_(True), _T(rs.randn(B, e)).requires_grad_(True)
    g1 = torch.autograd.grad((gz * z).sum() + (gnu * nu).sum(), (Q, p, A, b), create_graph=True)
    om = [_T(rs.randn(*x.shape)) for x in (Q, p, A, b)]
    g2 = torch.autograd.grad(sum((w * g).sum() for w, g in zip(om, g1)), (gz, gnu, Q, p, A, b))
    sh = ("Q", "A") if shared else ()
    ins = dict(Q=Q.detach().cpu(), p=p.detach().cpu(), G=torch.zeros(*(() if shared else (B,)), 0, n, dtype=torch.float64),
               h=torch.zeros(B, 0, dtype=torch.float64), A=A.detach().cpu(), b=b.detach().cpu())
    pt = dict(z=z.detach().cpu(), lam=torch.zeros(B, 0, dtype=torch.float64), s=torch.zeros(B, 0, dtype=torch.float64),
              nu=nu.detach().cpu())
    ref = dbm.double_backward(ins, pt, gz.detach().cpu(), torch.zeros(B, 0, dtype=torch.float64),
                              gnu.detach().cpu(), dict(zip(("Q", "p", "A", "b"), (w.cpu() for w in om))),
                              sh + (("G",) if shared else ()))
    for k, g in zip(("gz", "gnu", "Q", "p", "A", "b"), g2):
        assert _rel_per_qp(g, ref[k], batched=k not in sh) <= (1e-9 if reg else 1e-10), k


def _complementary(B, n, m, e, seed, dev=DEV):
    prs = [dm.complementary_qp(seed + i, n, m, e) for i in range(B)]
    return {k: _T(np.stack([pr[k] for pr in prs]), dev) for k in NAMES}


def test_gradient_of_g_is_the_jvp_bit_for_bit():
    """grad g = solve_jvp with tangents w, w / B for the un-batched inputs, bit for bit (the same qpb200_jvp call)."""
    from qpth_b200 import qp
    B, n, m, e = 6, 30, 25, 5
    ins = _complementary(B, n, m, e, 40)
    ins["Q"], ins["G"] = ins["Q"][0], ins["G"][0]
    rs = np.random.RandomState(3)
    st = qp.solve_forward(*(ins[k] for k in NAMES), verbose=-1)
    flags = [k in ("Q", "G") for k in NAMES]
    outs, v = qp.solve_backward(st, _T(rs.randn(B, n)), flags, [True] * 6, _T(rs.randn(B, m)), _T(rs.randn(B, e)),
                                keep=True)
    om = [_T(rs.randn(*o.shape)) for o in outs]
    res = qp.solve_double_backward(st, v, om, flags, [True] * 6, ins["G"])
    jvp = qp.solve_jvp(st, [w / B if f else w for w, f in zip(om, flags)])
    for a, b_ in zip(res[:3], jvp):
        assert torch.equal(a, b_)


def test_hessian_is_symmetric_and_matches_jacobian():
    from qpth_b200 import QPFunction
    B, n, m, e = 3, 12, 10, 3
    ins = _complementary(B, n, m, e, 70)
    f = QPFunction(verbose=-1, eps=1e-14, maxIter=40)
    other = [ins[k] for k in ("Q",)]

    def loss(p):
        z = f(other[0], p, ins["G"], ins["h"], ins["A"], ins["b"])
        return 0.5 * (z ** 2).sum()
    H = torch.autograd.functional.hessian(loss, ins["p"])          # (B, n, B, n)
    Hm = H.reshape(B * n, B * n)
    assert float((Hm - Hm.T).abs().max()) <= 1e-10 * float(Hm.abs().max())
    loss(ins["p"])
    J = f.jacobian(wrt="p")["p"]                                     # (B, n, n)
    for i in range(B):
        JtJ = J[i].T @ J[i]
        # H - J'J is sum_i z_i d2z_i/dp2, which the interior-point point's D keeps nonzero: 2.0e-7 measured on an H100,
        # so the bound is 1e-6, not 1e-7
        assert float((H[i, :, i, :] - JtJ).abs().max()) <= 1e-6 * max(1.0, float(JtJ.abs().max()))
        for j in range(B):                            # the QPs are independent: the off-diagonal blocks are exactly zero
            if j != i:
                assert not H[i, :, j, :].any(), (i, j)


@pytest.mark.parametrize("direction", ["Q", "G", "A", "h", "b"])
def test_central_differences_of_first_order_gradients(direction):
    """d/de <w, grad(theta + e t)> by central differences of QPFunction's first-order gradients against the double
    backward, on a strictly complementary batch (tight solves: the forward's error stays below the step)."""
    from qpth_b200 import QPFunction
    B, n, m, e = 4, 15, 12, 4
    ins = _complementary(B, n, m, e, 90)
    rs = np.random.RandomState(17)
    t = _T(rs.randn(*ins[direction].shape))
    if direction == "Q":
        t = t + t.transpose(1, 2)
    gz = _T(rs.randn(B, n))
    om = {k: _T(rs.randn(*ins[k].shape)) for k in NAMES}
    f = QPFunction(verbose=-1, eps=1e-15, maxIter=60)

    def grads(x, create):
        lv = {k: x[k].clone().requires_grad_(True) for k in NAMES}
        z = f(*(lv[k] for k in NAMES))
        g = torch.autograd.grad((gz * z).sum() + 0.5 * (z ** 2).sum(), [lv[k] for k in NAMES], create_graph=create)
        return lv, g

    def phi(eps):
        x = dict(ins)
        x[direction] = ins[direction] + eps * t
        _, g = grads(x, False)
        return sum(float((om[k] * gk).sum()) for k, gk in zip(NAMES, g))
    h = 1e-5
    fd = (phi(h) - phi(-h)) / (2 * h)
    lv, g = grads(ins, True)
    ph = sum((om[k] * gk).sum() for k, gk in zip(NAMES, g))
    an = float((torch.autograd.grad(ph, lv[direction])[0] * t).sum())
    assert abs(fd - an) <= 1e-5 * max(1.0, abs(an)), (fd, an)


def test_gradgradcheck():
    from qpth_b200 import QPFunction
    B, n, m, e = 2, 5, 4, 1
    ins = _complementary(B, n, m, e, 123)
    f = QPFunction(verbose=-1, eps=1e-15, maxIter=60)
    Q = ins["Q"]

    def fn(p, h, b):
        return f(Q, p, ins["G"], h, ins["A"], b)
    args = tuple(ins[k].clone().requires_grad_(True) for k in ("p", "h", "b"))
    assert torch.autograd.gradgradcheck(fn, args, eps=1e-6, atol=1e-5, rtol=1e-4)


def test_first_order_unchanged_and_third_order_raises():
    from qpth_b200 import QPFunction
    B, n, m, e = 8, 40, 30, 6
    ins = _complementary(B, n, m, e, 55)
    ins["Q"] = ins["Q"][0]
    f = QPFunction(verbose=-1, duals=True)
    rs = np.random.RandomState(2)
    wz, wl, wn = _T(rs.randn(B, n)), _T(rs.randn(B, m)), _T(rs.randn(B, e))

    def run(create):
        lv = {k: ins[k].clone().requires_grad_(True) for k in NAMES}
        z, lam, nu = f(*(lv[k] for k in NAMES))
        loss = (wz * z).sum() + (wl * lam).sum() + (wn * nu).sum()
        return lv, torch.autograd.grad(loss, [lv[k] for k in NAMES], create_graph=create)
    _, g0 = run(False)
    lv, g1 = run(True)
    for a, b_ in zip(g0, g1):
        assert a.grad_fn is None and b_.grad_fn is not None
        assert torch.equal(a, b_.detach())
    with pytest.raises(RuntimeError, match="third-order"):
        torch.autograd.grad(g1[1].square().sum(), lv["p"], create_graph=True)
