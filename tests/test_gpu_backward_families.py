"""The backward pass of every kernel family at a chosen, well-conditioned primal-dual point, and the batch-mean reduction
of gradients of un-batched inputs.

At a converged point d = lam / s spans ~16 decades and the reference's 1e-8 clamps (qp.py:148) put noise into the
gradients, so the converged-output tests can only hold them to 1e-6. Here QPSolutionFunction is fed random z and nu,
and lam, s ~ U(0.1, 10): the clamps do nothing, d is well conditioned, and every gradient is compared at 1e-10
relative with the outer-product formulas (qp.py:157-176) applied to dx, dlam, dnu of the refined dense solve of
[Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dlam dnu] = -[dl 0 0 0] (oracle/dense_kkt.py).
"""
import numpy as np
import pytest
import torch

from oracle import dense_kkt as dk
from tests.kernel_families import cases, family_env, family_plan, ids, seed_for
from tests.parity import rel_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAMES = ("dQ", "dp", "dG", "dh", "dA", "db")


def _point(shape, B, seed):
    from qpth_b200.problems import random_qp_batch
    nz, nineq, neq = shape
    pr = random_qp_batch(B, nz, nineq, neq, seed=seed)
    rs = np.random.RandomState(seed + 1)
    pr.update(z=rs.randn(B, nz), nu=rs.randn(B, neq), lam=rs.uniform(0.1, 10, (B, nineq)),
              s=rs.uniform(0.1, 10, (B, nineq)))
    return pr


def _per_qp_reference(pr, i):
    """Per-QP gradients (qp.py:157-176) from the dense solve; fully batched inputs."""
    neq = pr["A"].shape[1]
    d = pr["lam"][i] / pr["s"][i]
    m = d.shape[0]
    dx, _, dlam, dnu, _, _ = dk.solve(pr["Q"][i], pr["G"][i], pr["A"][i], d, pr["dl"][i], np.zeros(m), np.zeros(m),
                                      np.zeros(neq) if neq else None)
    z, lam = pr["z"][i], pr["lam"][i]
    g = dict(dQ=0.5 * (np.outer(dx, z) + np.outer(z, dx)), dp=dx, dG=np.outer(dlam, z) + np.outer(lam, dx), dh=-dlam)
    if neq:
        g.update(dA=np.outer(dnu, z) + np.outer(pr["nu"][i], dx), db=-dnu)
    return g


def _backward(pr, batched, plan=None, monkeypatch=None):
    """QPSolutionFunction + backward(dl). batched: {name: bool} for Q, p, G, h, A, b (un-batched inputs take QP 0's
    value). plan: force this plan (a several-QPs-per-SM one) on pre_factor_kkt and the backward."""
    from qpth_b200 import _lib
    from qpth_b200.solution import QPSolutionFunction
    if plan is not None:
        monkeypatch.setattr(_lib, "plan_for", lambda *a, **k: plan)
    neq = pr["A"].shape[1]
    t = {}
    for k in ("Q", "p", "G", "h", "A", "b"):
        v = pr[k] if batched[k] else pr[k][0]
        t[k] = torch.tensor(v, dtype=torch.float64, device=DEV, requires_grad=True) if (neq or k not in "Ab") \
            else torch.Tensor().to(DEV).double()
    sol = [torch.tensor(pr[k], dtype=torch.float64, device=DEV) for k in ("z", "lam", "s")]
    nu = torch.tensor(pr["nu"], dtype=torch.float64, device=DEV) if neq else torch.Tensor().to(DEV).double()
    z = QPSolutionFunction()(t["Q"], t["p"], t["G"], t["h"], t["A"], t["b"], sol[0], sol[1], sol[2], nu)
    z.backward(torch.tensor(pr["dl"], dtype=torch.float64, device=DEV))
    return {n: (t[k].grad.cpu().numpy() if t[k].grad is not None else None) for n, k in zip(NAMES, "QpGhAb")}


ALL_BATCHED = dict(Q=True, p=True, G=True, h=True, A=True, b=True)


@pytest.mark.parametrize("fam,shape", cases(), ids=ids(cases()))
def test_backward_matches_dense_solve(fam, shape, monkeypatch):
    from tests.test_gpu_parity import _report
    B = 4
    pr = _point(shape, B, seed_for(fam, shape, 4))
    with family_env(fam):
        plan = family_plan(fam, shape)
        got = _backward(pr, ALL_BATCHED, plan, monkeypatch)
    refs = [_per_qp_reference(pr, i) for i in range(B)]
    worst = {}
    for n in NAMES:
        if n not in refs[0]:
            assert got[n] is None, n
            continue
        e = rel_rows(got[n], np.stack([r[n] for r in refs])).max()
        worst[n] = e
        assert e <= 1e-10, (n, e)
    _report("bwd[%s %s]" % (fam, shape), worst)


MEAN_SHARING = {
    "QGAh_unbatched": dict(Q=False, p=True, G=False, h=False, A=False, b=True),
    "Q_unbatched_G_batched": dict(Q=False, p=True, G=True, h=True, A=True, b=True),
    "p_b_unbatched": dict(Q=True, p=False, G=True, h=True, A=True, b=False),
}


@pytest.mark.parametrize("sharing", sorted(MEAN_SHARING))
def test_batch_mean_of_unbatched_gradients(sharing):
    """B = 37 at 100/100/8: the 32 x 64 output tiles of k_mean_outer (4 x 2 tiles for dQ, dG; 1 x 2 for dA) and its
    16-QP chunks with a partial last one (37 = 16 + 16 + 5); mixed sharing included (Q un-batched, G batched: nsys = B
    with a zero Q stride). The reference gradient of an un-batched input is the mean of the per-QP gradients; the error
    is measured against the mean per-QP gradient norm (the scale the kernel's summation rounds at) and held to 1e-12."""
    from tests.test_gpu_parity import _report
    B, shape = 37, (100, 100, 8)
    bat = MEAN_SHARING[sharing]
    pr = _point(shape, B, 900)
    for k, v in bat.items():             # un-batched inputs: every QP sees QP 0's value
        if not v:
            pr[k] = np.broadcast_to(pr[k][:1], pr[k].shape).copy()
    got = _backward(pr, bat)
    refs = [_per_qp_reference(pr, i) for i in range(B)]
    worst = {}
    for n, k in zip(NAMES, "QpGhAb"):
        per = np.stack([r[n] for r in refs])
        if bat[k]:
            e = rel_rows(got[n], per).max()
            assert e <= 1e-10, (n, e)
        else:
            assert got[n].shape == per.shape[1:], n
            scale = np.mean([np.linalg.norm(x) for x in per])
            e = np.linalg.norm(got[n] - per.mean(0)) / scale
            assert e <= 1e-12, (n, e)
        worst[n] = e
    _report("mean[%s]" % sharing, worst)
