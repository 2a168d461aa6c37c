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

from oracle import dense_kkt as dk
from tests import gpu_child
from tests.fallback_jobs import bwd_job_name
from tests.kernel_families import (BWD_B, GRAD_NAMES as NAMES, backward_on_gpu, backward_point, cases, family_env,
                                   family_plan, ids, seed_for, solution_backward)
from tests.parity import rel_rows

pytestmark = pytest.mark.gpu


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


def check_backward(fam, shape, got):
    from tests.test_gpu_parity import _report
    pr = backward_point(shape, BWD_B, seed_for(fam, shape, 4), fam)
    refs = [_per_qp_reference(pr, i) for i in range(BWD_B)]
    worst = {}
    for n in NAMES:
        if n not in refs[0]:
            assert got.get(n) is None, n
            continue
        e = rel_rows(got[n], np.stack([r[n] for r in refs])).max()
        worst[n] = e
        assert e <= 1e-10, (n, e)
    _report("bwd[%s %s]" % (fam, shape), worst)


@pytest.mark.parametrize("fam,shape", cases(child=False), ids=ids(cases(child=False)))
def test_backward_matches_dense_solve(fam, shape):
    check_backward(fam, shape, backward_on_gpu(fam, shape))


@pytest.fixture(scope="module")
def child_results(tmp_path_factory):
    out_dir = str(tmp_path_factory.mktemp("backward_families"))
    return out_dir, gpu_child.run(out_dir, "family_backward_jobs")


@pytest.mark.parametrize("fam,shape", cases(child=True), ids=ids(cases(child=True)))
def test_backward_matches_dense_solve_new_dispatch(fam, shape, child_results):
    """The families whose dispatch branches had never run before these tests, and the edge entries: solved in the child
    process."""
    with family_env(fam):
        family_plan(fam, shape)
    check_backward(fam, shape, gpu_child.load(*child_results, bwd_job_name(fam, shape)))


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
    pr = backward_point(shape, B, 900)
    for k, v in bat.items():             # un-batched inputs: every QP sees QP 0's value
        if not v:
            pr[k] = np.broadcast_to(pr[k][:1], pr[k].shape).copy()
    got = solution_backward(pr, bat)
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
