"""Only the lower triangle of Q is read, by every entry point that takes a dense Q.

The public header, QPFunction's, QPSolutionFunction's and BoxQPFunction's docstrings and util.copy_lower_ promise it,
and callers rely on it: copy_lower_ moves only the lower strips of Q and leaves the destination's upper part as it was.
Every case runs the same inputs four times (kernel_families.VARIANTS): with the symmetric matrix
tril(Q) + tril(Q, -1)^T, with it again (the control: a difference there is nondeterminism, not the poison), with the
strictly upper triangle NaN, and with it finite garbage, -1e3 lower^T + N(0, 1) (which catches reads that fmin, fmax or a
comparison would hide from NaN). Every output is compared bit for bit with np.array_equal: z, lam, slacks, nu, iters,
best_resid, the trace, every gradient of a backward with adjoints on z, lam and nu, the JVP, and the stand-alone KKT
solve with its packed L buffer. The poisoned runs use check_Q_spd=True with deferred checks off, so a poisoned pivot
would raise 'Q is not SPD.'.

Cases: every family of tests/kernel_families.py (the `child` ones in the child process of tests/gpu_child.py) with Q,
G, A batched (nsys = B) and un-batched (nsys = 1), plus pre_factor_kkt + solve_kkt at reg 0 and 1e-7; every case of
tests/reg_families.py under IR_UNOPT; the equality-only path and QPSolutionFunction under both KKT solvers;
BoxQPFunction(dense_Q=True) at its plan's largest shapes, odd nz, a shared Q and the dense fallback; OptNetQP's L;
qpb200_qp_host; and util.copy_lower_ into a poisoned device buffer (the Q-band path of bench.py's e2e leg)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from tests import gpu_child, reg_families as rf
from tests.fallback_jobs import EQ_ONLY, eq_only_problem, lower_triangle_job_name, lower_triangle_jobs
from tests.kernel_families import (FAMILIES, VARIANTS, adjoints, backward_point, cases, compare_variants, eq_outputs,
                                   family_env, family_plan, ids, leaf, lower_triangle_runs, poison, q_variants,
                                   qp_outputs)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B = 2

PARENT_CASES = cases(child=False, forward=True)
CHILD_CASES = cases(child=True, forward=True)


@pytest.fixture(autouse=True)
def eager_checks(monkeypatch):
    """'Q is not SPD.' raised by the call that meets it."""
    from qpth_b200 import qp
    monkeypatch.setattr(qp, "LAZY_CHECKS", False)


def _add(rec, run, variant, outs):
    rec.update({"%s__%s__%s" % (run, variant, k): np.asarray(v) for k, v in outs.items()})


def _runs(fam):
    return ["qp_batched", "qp_unbatched"] + ([] if FAMILIES[fam].get("forward_only") else ["kkt", "kkt_reg"])


def test_every_family_is_covered():
    """A family added to either table without a case here fails."""
    assert {f for f, _ in PARENT_CASES} | {f for f, _ in CHILD_CASES} == set(FAMILIES)
    assert {name for name, *_ in lower_triangle_jobs()} == {lower_triangle_job_name(f, s) for f, s in CHILD_CASES}
    assert {f for f, _ in rf.CASES} == set(rf.FAMILIES)


@pytest.mark.parametrize("fam,shape", PARENT_CASES, ids=ids(PARENT_CASES))
def test_qpfunction_family(fam, shape):
    assert compare_variants(lower_triangle_runs(fam, shape, B)) == sorted(_runs(fam))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("lower_triangle"))
    return out_dir, gpu_child.run(out_dir, "lower_triangle_jobs", timeout_s=900)


@pytest.mark.parametrize("fam,shape", CHILD_CASES, ids=ids(CHILD_CASES))
def test_qpfunction_family_in_child(fam, shape, child_results):
    with family_env(fam):
        family_plan(fam, shape)
    rec = gpu_child.load(*child_results, lower_triangle_job_name(fam, shape))
    assert compare_variants(rec) == sorted(_runs(fam))


@pytest.mark.parametrize("case", rf.CASES, ids=rf.ids(rf.CASES))
def test_ir_unopt_family(case):
    from qpth_b200 import KKTSolvers
    fam, kind = case
    cs = [rf.problem(fam, kind, s) for s in range(B)]
    rf.family_plan(fam, cs[0])
    pr = {k: np.stack([c[i] for c in cs]) for i, k in enumerate(("Q", "p", "G", "h", "A", "b"))}
    adj = adjoints(pr, 11)
    rec = {}
    for v, Q in q_variants(pr["Q"], 12).items():
        _add(rec, "reg", v, qp_outputs(dict(pr, Q=Q), adj, KKTSolvers.IR_UNOPT))
    assert compare_variants(rec) == ["reg"]


@pytest.mark.parametrize("solver", ["LU_PARTIAL", "IR_UNOPT"])
@pytest.mark.parametrize("name", list(EQ_ONLY))
def test_equality_only(name, solver):
    from qpth_b200 import KKTSolvers
    pr = eq_only_problem(**EQ_ONLY[name])
    rs = np.random.RandomState(13)
    Bq, nz = pr["p"].shape
    adj = dict(z=rs.randn(Bq, nz), nu=rs.randn(*pr["b"].shape))
    tan = {k: rs.randn(*np.shape(pr[k])) for k in ("Q", "p", "A", "b")}
    rec = {}
    for v, Q in q_variants(pr["Q"], 14).items():
        _add(rec, "eq", v, eq_outputs(dict(pr, Q=Q), adj, tan, getattr(KKTSolvers, solver)))
    assert compare_variants(rec) == ["eq"]


def _tangents(pr, keys, seed):
    rs = np.random.RandomState(seed)
    return {k: rs.randn(*np.shape(pr[k])) for k in keys if pr.get(k) is not None and np.size(pr[k])}


SOLUTION_SHAPES = [(24, 19, 5), (50, 50, 10), (99, 93, 3)]


@pytest.mark.parametrize("solver", ["LU_PARTIAL", "IR_UNOPT"])
@pytest.mark.parametrize("shape", SOLUTION_SHAPES, ids=["%dx%dx%d" % s for s in SOLUTION_SHAPES])
def test_solution_function(shape, solver):
    """QPSolutionFunction at a given solution: the backward with duals and the JVP."""
    from qpth_b200 import KKTSolvers, QPSolutionFunction
    pr = backward_point(shape, 3, 31)
    keys = ("Q", "p", "G", "h", "A", "b")
    adj = adjoints(pr, 32)
    tan = _tangents(pr, keys, 33)
    sol = [torch.tensor(pr[k], dtype=torch.float64, device=DEV) for k in ("z", "lam", "s", "nu")]
    T = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV)
    rec = {}
    for v, Q in q_variants(pr["Q"], 34).items():
        f = QPSolutionFunction(check_Q_spd=True, kkt_solver=getattr(KKTSolvers, solver), duals=True)
        t = {k: leaf(Q if k == "Q" else pr[k], DEV, True) for k in keys}
        z, lam, nu = f(*(t[k] for k in keys), *sol)
        ((z * T(adj["z"])).sum() + (lam * T(adj["lam"])).sum() + (nu * T(adj["nu"])).sum()).backward()
        out = {"d" + k: t[k].grad.cpu().numpy() for k in keys}
        with fwAD.dual_level():
            zd, ld, nd = f(*(fwAD.make_dual(t[k].detach(), T(tan[k])) for k in keys), *sol)
            out.update({"jvp_" + k: fwAD.unpack_dual(o).tangent.cpu().numpy() for k, o in (("z", zd), ("lam", ld), ("nu", nd))})
        _add(rec, "solution", v, out)
    assert compare_variants(rec) == ["solution"]


# (nz, neq, sides, inputs passed un-batched): the three largest shapes of the plan (tests/test_boxq_cpu.py LARGEST), an
# nz that is not a multiple of 8 with and without equality rows, a shared Q, and a shape past the plan (the dense
# fallback: QPFunction's kernels on the dense equivalent)
BOXQ_CASES = [(192, 1, "lb", ()), (192, 1, "ub", ()), (184, 1, "both", ()), (37, 0, "both", ()), (37, 13, "lb", ()),
              (23, 5, "both", ("Q",)), (200, 1, "lb", ())]


def _boxq_outputs(bx, adj, tan):
    """BoxQPFunction(dense_Q=True, duals=True, check_Q_spd=True) with qp.TRACE on: the outputs, every gradient of a
    backward with adjoints on z, lam and nu, and the JVP."""
    from qpth_b200 import BoxQPFunction, qp as qpmod
    from tests.boxq_util import KEYS
    e = torch.Tensor().to(DEV).double()
    t = {k: (None if bx[k] is None else (leaf(bx[k], DEV, True) if np.size(bx[k]) else e)) for k in KEYS}
    T = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV)
    f = BoxQPFunction(verbose=-1, dense_Q=True, duals=True, check_Q_spd=True)
    saved = qpmod.TRACE
    qpmod.TRACE = True
    try:
        z, lam, nu = f(*(t[k] for k in KEYS))
    finally:
        qpmod.TRACE = saved
    st = f.last_solve()
    out = dict(z=z.detach().cpu().numpy(), lam=lam.detach().cpu().numpy(), nu=nu.detach().cpu().numpy(),
               slacks=st.slacks.cpu().numpy(), iters=st.iters.cpu().numpy(), best_resid=st.best_resid.cpu().numpy(),
               trace=st.trace.cpu().numpy())
    loss = (z * T(adj["z"])).sum() + (lam * T(adj["lam"])).sum()
    if nu.numel():
        loss = loss + (nu * T(adj["nu"])).sum()
    loss.backward()
    out.update({"d" + k: t[k].grad.cpu().numpy() for k in KEYS if t[k] is not None and t[k].grad is not None})
    with fwAD.dual_level():
        outs = f(*(None if t[k] is None else (fwAD.make_dual(t[k].detach(), T(tan[k])) if k in tan else t[k].detach())
                   for k in KEYS))
        out.update({"jvp_" + k: fwAD.unpack_dual(o).tangent.cpu().numpy() for k, o in zip(("z", "lam", "nu"), outs)
                    if o.numel()})
    return out


def _boxq_kkt(plan, Q, A, seed):
    """qpb200_boxq_solve_kkt for random d and right-hand sides."""
    from qpth_b200 import _lib
    n, e, m = plan.nz, plan.neq, plan.nineq
    rs = np.random.RandomState(seed)
    d = 10.0 ** rs.uniform(-8, 8, (B, m))
    vec = [torch.tensor(v, dtype=torch.float64, device=DEV).contiguous()
           for v in (d, rs.randn(B, n), rs.randn(B, m), rs.randn(B, m), rs.randn(B, e))]
    tQ = torch.tensor(np.ascontiguousarray(Q), dtype=torch.float64, device=DEV)
    tA = torch.tensor(np.asarray(A).reshape(B, e, n) if e else np.zeros((B, 0, n)), dtype=torch.float64, device=DEV)
    out = [torch.empty(B, k, dtype=torch.float64, device=DEV) for k in (n, m, m, e)]
    P = lambda x: ctypes.c_void_p(x.data_ptr()) if x.numel() else ctypes.c_void_p(0)
    _lib.check(_lib.load().qpb200_boxq_solve_kkt(ctypes.byref(plan), B, P(tQ), n * n if tQ.dim() == 3 else 0, P(tA),
                                                 e * n, *(P(v) for v in vec), *(P(o) for o in out), ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    return {"kkt_" + k: o.cpu().numpy() for k, o in zip(("dx", "ds", "dz", "dy"), out) if o.numel()}


@pytest.mark.parametrize("n,e,sides,shared", BOXQ_CASES,
                         ids=["%d-%d-%s%s" % (n, e, s, "-sharedQ" if sh else "") for n, e, s, sh in BOXQ_CASES])
def test_boxq_dense(n, e, sides, shared):
    from qpth_b200 import _lib
    from tests.boxq_util import KEYS, random_boxq
    plan = _lib.boxq_plan_for(n, e, sides != "ub", sides != "lb")
    assert plan.ok == (0 if n == 200 else 1)
    bx = random_boxq(n + e, B, n, e, sides, shared)
    adj = dict(z=np.random.RandomState(1).randn(B, n), lam=np.random.RandomState(2).randn(B, plan.nineq),
               nu=np.random.RandomState(3).randn(B, e))
    tan = _tangents(bx, KEYS, 4)
    rec = {}
    for v, Q in q_variants(bx["Q"], 5).items():
        out = _boxq_outputs(dict(bx, Q=Q), adj, tan)
        if plan.ok:
            out.update(_boxq_kkt(plan, Q, bx["A"], 6))
        _add(rec, "boxq", v, out)
    assert compare_variants(rec) == ["boxq"]


def test_optnet_layer_reads_the_lower_triangle_of_L():
    """OptNetQP with the strictly upper triangle of L zero ("sym" and its control), NaN and garbage: the Q and h the
    layer builds, z and every gradient bit-identical; dL zero above the diagonal."""
    from qpth_b200 import _lib
    from qpth_b200.layers import OptNetQP
    n, m, Bl, eps = 20, 15, 4, 1e-4
    rs = np.random.RandomState(21)
    Lt = np.tril(rs.randn(n, n)) + 2.0 * np.eye(n)
    fixed = dict(G=rs.randn(m, n), z0=rs.randn(n), s0=rs.uniform(0.5, 1.5, m), p=rs.randn(Bl, n))
    dl = torch.tensor(rs.randn(Bl, n), dtype=torch.float64, device=DEV)
    Ls = dict(sym=Lt, sym_again=Lt.copy(), nan=poison(Lt, "nan", rs), garbage=poison(Lt, "garbage", rs))
    P = lambda x: ctypes.c_void_p(x.data_ptr())
    rec = {}
    for v in VARIANTS:
        t = dict({k: leaf(a, DEV, True) for k, a in fixed.items()}, L=leaf(Ls[v], DEV, True))
        Q = torch.empty(n, n, dtype=torch.float64, device=DEV)
        h = torch.empty(m, dtype=torch.float64, device=DEV)
        _lib.check(_lib.load().qpb200_optnet_construct(n, m, P(t["L"]), P(t["G"]), P(t["z0"]), P(t["s0"]), float(eps),
                                                       P(Q), P(h), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        z = OptNetQP(eps=eps)(t["L"], t["G"], t["z0"], t["s0"], t["p"])
        z.backward(dl)
        out = dict(Q=Q.cpu().numpy(), h=h.cpu().numpy(), z=z.detach().cpu().numpy(),
                   **{"d" + k: x.grad.cpu().numpy() for k, x in t.items()})
        assert np.array_equal(np.triu(out["dL"], 1), np.zeros((n, n))), v
        _add(rec, "optnet", v, out)
    assert compare_variants(rec) == ["optnet"]


def test_qp_host():
    """qpb200_qp_host with the poison in the host Q."""
    from qpth_b200 import _lib
    from qpth_b200.problems import random_qp_batch
    Bh, n, m, e = 4, 20, 15, 5
    pr = random_qp_batch(Bh, n, m, e, seed=2)
    c = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    rec = {}
    for v, Q in q_variants(pr["Q"], 3).items():
        ins = dict({k: c(pr[k]) for k in ("p", "G", "h", "A", "b", "dl")}, Q=c(Q))
        out = dict(z=np.empty((Bh, n)), dQ=np.empty((Bh, n, n)), dp=np.empty((Bh, n)), dG=np.empty((Bh, m, n)),
                   dh=np.empty((Bh, m)), dA=np.empty((Bh, e, n)), db=np.empty((Bh, e)), spd=np.ones(Bh, dtype=np.int32))
        _lib.check(_lib.load().qpb200_qp_host(0, Bh, n, m, e, *(P(ins[k]) for k in ("Q", "p", "G", "h", "A", "b", "dl")),
                                              1e-12, 3, 20, *(P(out[k]) for k in ("z", "dQ", "dp", "dG", "dh", "dA", "db",
                                                                                  "spd"))))
        assert not out["spd"].any(), v
        _add(rec, "host", v, out)
    assert compare_variants(rec) == ["host"]


@pytest.mark.parametrize("mode", ["latency", "throughput"])
@pytest.mark.parametrize("band", [20, 30])
def test_copy_lower_into_a_poisoned_buffer(band, mode, monkeypatch):
    """util.copy_lower_ from pinned host memory into a device buffer whose every entry is NaN (or garbage) first, then
    QPFunction at C2 (100, 100, 0): z and every gradient as with a full copy. Band 30 does not divide nz = 100."""
    from qpth_b200 import qp, util
    from qpth_b200.problems import random_qp_batch
    monkeypatch.setattr(qp, "MODE", mode)
    Bc = 4
    pr = random_qp_batch(Bc, 100, 100, 0, seed=17)
    pr["Q"] = torch.tensor(q_variants(pr["Q"], 0)["sym"]).pin_memory()
    adj = adjoints(pr, 18)
    rec = {}
    for v, fill in (("sym", None), ("sym_again", None), ("nan", float("nan")), ("garbage", -1e3)):
        if fill is None:
            Qd = pr["Q"].to(DEV)
        else:
            Qd = torch.full((Bc, 100, 100), fill, dtype=torch.float64, device=DEV)
            util.copy_lower_(Qd, pr["Q"], band=band)
        _add(rec, "copy_lower", v, qp_outputs(dict(pr, Q=Qd), adj))
    assert compare_variants(rec) == ["copy_lower"]
