"""pre_factor_kkt[_reg] + solve_kkt[_reg] (the stand-alone KKT solve of kkt.py and eqonly.py) on every kernel family,
against the refined dense solve of the full KKT system (oracle/dense_kkt.py).

d = 10^U(-8, 8), random right-hand sides, reg = 0 and reg = 1e-7, batched systems (sF = 1) and one system shared by the
batch (sF = 0). Per system: normwise backward error <= 1e-14, and relative error <= 1e-10 for dx, dz, dy and <= 1e-8
for ds (ds = (-rs - dz) / d divides by d).

The relative bounds hold where the kernels' formulation (Cholesky of the reduced system W W^T + D^-1, the same in
oracle/kernel_model.py) is that accurate. Where nineq is far above nz, R = G Q^-1 G^T has rank nz only and with d over
16 decades the full system's condition number reaches 1e14: at 20/120/0 and 24/116/4 the model itself is off by up to
4e-7 from the dense solve, at 120/260/0 by up to 2e-10 (with a backward error still ~1e-20). The kernels use that
formulation and differ from the model only in FMA use and summation order, so their error there is rounding noise of
the same size, which varies ~10x from system to system. Each block is held to max(bound, 10 x the model's largest
error on the batch's systems (for ds and for the other blocks separately): that leaves every well-conditioned shape at
1e-10 / 1e-8.

The normwise backward error is held to 1e-14, except on three edge entries of kernel_families.py (MODEL_BERR). They
have fewer than 10 inequality rows next to hundreds of columns. With d over 16 decades, the formulation itself leaves a
larger backward error there: the model's (measured) is 1.0e-10 at 213/8/0, 9.4e-13 at 880/1/128 and 3.7e-14 at
740/1/0. On those three the bound is max(1e-14, 10 x the model's largest backward error on the batch's systems).
"""
import numpy as np
import pytest

from oracle import dense_kkt as dk
from oracle import kernel_model as km
from tests import gpu_child
from tests.fallback_jobs import KKT_B, KKT_VARIANTS, kkt_job_name
from tests.kernel_families import cases, family_env, family_plan, ids, kkt_inputs, kkt_on_gpu

pytestmark = pytest.mark.gpu

BERR, XTOL, STOL = 1e-14, 1e-10, 1e-8
# edge entries whose backward error is held to max(BERR, 10 x the model's) (module docstring); every other family to BERR
MODEL_BERR = ("edge_gs_pf_res", "edge_512_wide", "edge_two_wide")


def _report(name, errs):
    from tests.test_gpu_parity import _report as rep
    rep(name, errs)


def check_kkt(fam, shape, shared, reg, out):
    neq = shape[2]
    x = kkt_inputs(fam, shape, KKT_B, shared)
    assert int(np.asarray(out["spd"]).sum()) == 0
    refs, merr = [], dict(x=0.0, s=0.0, b=0.0)   # the model's largest error: dx, dz, dy / ds / backward error
    for i in range(KKT_B):
        j = 0 if shared else i
        args = (x["Q"][j], x["G"][j], x["A"][j], x["d"][i], x["rx"][i], x["rs"][i], x["rz"][i], x["ry"][i] if neq else None)
        refs.append(dk.solve(*args, reg=reg))
        m = km.kkt_solve(*args, reg=reg)
        for k, (a, b) in enumerate(zip(m, refs[-1][:4])):
            if b is not None:
                merr["s" if k == 1 else "x"] = max(merr["s" if k == 1 else "x"], dk.rel(a, b))
        mu = np.concatenate([m[0], m[1], m[2]] + ([m[3]] if neq else []))
        merr["b"] = max(merr["b"], dk.backward_error(refs[-1][4], mu, refs[-1][5]))
    worst = dict(berr=0.0, dx=0.0, ds=0.0, dz=0.0, dy=0.0, model_x=merr["x"], model_s=merr["s"], model_berr=merr["b"])
    for i, ref in enumerate(refs):
        u = np.concatenate([out["dx"][i], out["ds"][i], out["dz"][i]] + ([out["dy"][i]] if neq else []))
        berr = dk.backward_error(ref[4], u, ref[5])
        worst["berr"] = max(worst["berr"], berr)
        tol_b = max(BERR, 10 * merr["b"]) if fam in MODEL_BERR else BERR
        assert berr <= tol_b, (i, berr, tol_b)
        for k, name in enumerate(("dx", "ds", "dz", "dy")):
            if ref[k] is None:
                continue
            err = dk.rel(out[name][i], ref[k])
            worst[name] = max(worst[name], err)
            tol = max(STOL, 10 * merr["s"]) if name == "ds" else max(XTOL, 10 * merr["x"])
            assert err <= tol, (i, name, err, tol)
    _report("kkt[%s %s %s %s]" % (fam, shape, "shared" if shared else "batched", reg), worst)


@pytest.mark.parametrize("shared,reg", KKT_VARIANTS)
@pytest.mark.parametrize("fam,shape", cases(child=False), ids=ids(cases(child=False)))
def test_solve_kkt_matches_dense_solve(fam, shape, shared, reg):
    check_kkt(fam, shape, shared, reg, kkt_on_gpu(fam, shape, KKT_B, shared, reg))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("kkt_families"))
    return out_dir, gpu_child.run(out_dir, "family_kkt_jobs")


@pytest.mark.parametrize("shared,reg", KKT_VARIANTS)
@pytest.mark.parametrize("fam,shape", cases(child=True), ids=ids(cases(child=True)))
def test_solve_kkt_matches_dense_solve_new_dispatch(fam, shape, shared, reg, child_results):
    """The 192- and 512-thread solve_kkt builds and the regularised solve on a 512-thread plan (which runs the
    256-thread build): solved in the child process."""
    with family_env(fam):
        family_plan(fam, shape)
    check_kkt(fam, shape, shared, reg, gpu_child.load(*child_results, kkt_job_name(fam, shape, shared, reg)))


@pytest.mark.parametrize("fam,shape", [("pf_global_512", (200, 200, 0)), ("pf_one_setup_fast", (100, 100, 0)),
                                       ("pf_one_setup_pf", (50, 50, 10))])
def test_kkt_module_entry_points(fam, shape):
    """kkt.factor_solve_kkt and kkt.solve_kkt_ir (the reference's stand-alone solvers; latency-mode plans) at C4 size,
    where the regularised solve of a 512-thread plan runs, and at the C2 / C3 shapes. The exact solve against the dense
    one. The refined solve converges to the system kkt_resid_reg measures, [Q 0 G' A'; 0 D I 0; G I -eps I 0;
    A 0 0 -eps I]: against the dense solve of that system (two refinement steps leave ~1e-14 there in fp64)."""
    import torch
    from qpth_b200 import kkt
    nz, nineq, neq = shape
    x = kkt_inputs(fam, shape, KKT_B, False)
    x["d"] = 10.0 ** np.random.RandomState(5).uniform(-2, 2, x["d"].shape)      # refinement contracts by ~eps / lambda_min
    t = {k: torch.tensor(v, dtype=torch.float64, device="cuda:0") for k, v in x.items()}
    A, ry = (t["A"], t["ry"]) if neq else (None, None)
    with family_env(fam):
        family_plan(fam, shape)
        exact = kkt.factor_solve_kkt(t["Q"], t["d"], t["G"], A, t["rx"], t["rs"], t["rz"], ry)
        ir = kkt.solve_kkt_ir(t["Q"], t["d"], t["G"], A, t["rx"], t["rs"], t["rz"], ry, niter=2)
    eps, n, m = kkt.IR_EPS, nz, nineq
    for i in range(KKT_B):
        Ai = x["A"][i] if neq else None
        ref = dk.solve(x["Q"][i], x["G"][i], Ai, x["d"][i], x["rx"][i], x["rs"][i], x["rz"][i], x["ry"][i] if neq else None)
        Kir = dk.kkt_matrix(x["Q"][i], x["G"][i], Ai, x["d"][i], eps)
        Kir[:n, :n] -= eps * np.eye(n)
        Kir[n:n + m, n:n + m] -= eps * np.eye(m)
        ref_ir = dk.split(dk.solve_refined(Kir, ref[5]), n, m, neq)
        for k in range(4):
            if ref[k] is None:
                continue
            tol = STOL if k == 1 else XTOL
            assert dk.rel(exact[k][i].cpu().numpy(), ref[k]) <= tol, ("exact", i, k)
            assert dk.rel(ir[k][i].cpu().numpy(), ref_ir[k]) <= tol, ("ir", i, k)
