"""Second-order gradients through BoxQPFunction on the GPU (qpb200_box_double_backward, qpb200_boxq_double_backward).

The kernels are new to the device, so every job runs in one child process (tests/box_double_backward_jobs.py) and each
test reads its job's output:
- every box-family entry (one, cl2/4/8, dm2/4/8, the edges, dm4_sudoku) at a point, in three sharings (all batched; q
  and A shared; p, b, lb, ub shared): the double backward within 1e-10 per-QP relative of the structured numpy algebra
  (tests/box_double_backward_models.box_double_backward, tied to the torch model by the CPU tests), and of the torch
  model itself where its dense KKT system is small; the gradients of g bit-identical to the JVP with the cotangents as
  tangents;
- every dense-Q family entry the kernels run, the same way;
- the dense fallback entries through BoxQPFunction under create_graph, against the torch model at the returned point;
- the p-Hessian of a scalar of z(p): symmetric, with exactly zero blocks between different QPs; on strictly
  complementary batches the p-Hessian of 1/2 ||z||^2 against J'J from jacobian();
- central differences of the first-order gradients, gradgradcheck, first order bit-identical under create_graph, and
  fp32 / CPU inputs.
"""
import os
import tempfile

import numpy as np
import pytest
import torch

from tests import box_double_backward_models as bdm
from tests.box_double_backward_jobs import DENSE_NAMES, ENTRY_NAMES, NAMES, SHARINGS, run_child
from tests.boxq_families import kernel_entries

pytestmark = pytest.mark.gpu
_OUT = {}
MODEL_MAX = 400          # the torch model forms the dense KKT system of order nz + 2 nineq + neq: small entries only


@pytest.fixture(scope="module")
def out_dir():
    if "dir" not in _OUT:
        d = tempfile.mkdtemp(prefix="box_double_backward_jobs_")
        _OUT["dir"], _OUT["why"] = d, run_child(d)
    return _OUT["dir"]


def _load(out_dir, name):
    path = os.path.join(out_dir, name + ".npz")
    if not os.path.exists(path):
        err = os.path.join(out_dir, name + ".err")
        pytest.fail(open(err).read() if os.path.exists(err) else "no output: %s" % _OUT.get("why"))
    return dict(np.load(path))


def _per_qp_rel(a, b, batched):
    """max over QPs of max|a - b| / max(max|b|, 1) (one block when un-batched)"""
    if not batched:
        return float(np.abs(a - b).max() / max(np.abs(b).max(), 1.0))
    return max(float(np.abs(a[i] - b[i]).max() / max(np.abs(b[i]).max(), 1.0)) for i in range(a.shape[0]))


def _check_point(o, plan, dense_Q):
    n, e, m = plan.nz, plan.neq, plan.nineq
    nlb = n if plan.has_lb else 0
    for tag, shared in SHARINGS.items():
        flags = {k: k in shared for k in NAMES}
        q = o["q"][0] if "q" in shared else o["q"]
        A = (o["A"][0] if "A" in shared else o["A"]) if e else None
        om = {k: (None if o[tag + "_om_" + k].size == 0 else o[tag + "_om_" + k]) for k in NAMES}
        v = (o[tag + "_vx"], o[tag + "_vlam"], o[tag + "_vnu"] if e else None)
        solve = [bdm.box_solve(q if q.ndim == (2 if dense_Q else 1) else q[i],
                               (A if A.ndim == 2 else A[i]) if e else None, o["lam"][i], o["s"][i], nlb,
                               bool(plan.has_ub), dense_Q) for i in range(3)]
        vref = [solve[i](o["dl"][i], o["glam"][i], o["gnu"][i] if e else np.zeros(0)) for i in range(3)]
        assert _per_qp_rel(v[0], np.stack([r[0] for r in vref]), True) <= 1e-10, (tag, "vx")
        ref = bdm.box_double_backward(q, A, o["z"], o["lam"], o["s"], o["nu"] if e else None, v, om, nlb,
                                      bool(plan.has_ub), flags, dense_Q)
        for k in ("gz", "glam", "gnu") + NAMES:
            got = o[tag + "_" + k]
            if ref[k] is None:
                assert got.size == 0, (tag, k)
                continue
            assert _per_qp_rel(got, ref[k], not flags.get(k)) <= 1e-10, (tag, k, _per_qp_rel(got, ref[k], True))
        # the gradients of g are the JVP with the cotangents as tangents, bit for bit
        for k, j in (("gz", "jz"), ("glam", "jlam"), ("gnu", "jnu")):
            assert np.array_equal(o[tag + "_" + k], o[tag + "_" + j]), (tag, k)
        if n + 2 * m + e <= MODEL_MAX:
            _check_model(o, tag, shared, plan, dense_Q, flags)


def _check_model(o, tag, shared, plan, dense_Q, flags):
    """the torch model (the reference the numpy algebra is tied to) at the same point"""
    e = plan.neq
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    B, n = o["z"].shape
    ins = dict(q=T(o["q"][0] if "q" in shared else o["q"]), p=T(np.zeros((n,) if "p" in shared else (B, n))),
               A=T(o["A"][0] if "A" in shared else o["A"]) if e else torch.zeros(B, 0, n, dtype=torch.float64),
               b=T(np.zeros((e,) if "b" in shared else (B, e))) if e else torch.zeros(B, 0, dtype=torch.float64))
    for k, has in (("lb", plan.has_lb), ("ub", plan.has_ub)):
        ins[k] = T(np.zeros((n,) if k in shared else (B, n))) if has else None
    sh = tuple(k for k in shared if ins.get(k) is not None and not (k in ("A", "b") and not e))
    pt = dict(z=T(o["z"]), lam=T(o["lam"]), s=T(o["s"]), nu=T(o["nu"]) if e else torch.zeros(B, 0, dtype=torch.float64))
    om = {k: (None if o[tag + "_om_" + k].size == 0 else T(o[tag + "_om_" + k])) for k in NAMES}
    ref = bdm.double_backward(ins, pt, T(o["dl"]), T(o["glam"]), T(o["gnu"]) if e else None, om, sh, dense_Q)
    for k in ("gz", "glam", "gnu") + NAMES:
        got = o[tag + "_" + k]
        if ref.get(k) is None or got.size == 0:
            continue
        assert _per_qp_rel(got, ref[k].numpy(), not flags.get(k)) <= 1e-10, (tag, "model", k)


@pytest.mark.parametrize("name", ENTRY_NAMES)
def test_entry_double_backward(out_dir, name):
    from tests.box_families import ENTRIES, check_entry, knob
    with knob(ENTRIES[name]["knob"]):
        plan = check_entry(name)
    _check_point(_load(out_dir, "entry_" + name), plan, False)


@pytest.mark.parametrize("name", kernel_entries())
def test_boxq_entry_double_backward(out_dir, name):
    from tests.boxq_families import check_entry
    _check_point(_load(out_dir, "boxq_" + name), check_entry(name), True)


@pytest.mark.parametrize("name", DENSE_NAMES)
def test_dense_fallback_double_backward(out_dir, name):
    o = _load(out_dir, "dense_" + name)
    assert bool(o["dense"])
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    B, n = o["z"].shape
    e = o["in_A"].shape[0] if o["in_A"].size else 0
    shared = ("A", "b", "lb", "ub")
    ins = {k: (None if o["in_" + k].size == 0 else T(o["in_" + k])) for k in NAMES}
    if not e:
        ins["A"], ins["b"] = torch.zeros(B, 0, n, dtype=torch.float64), torch.zeros(B, 0, dtype=torch.float64)
    pt = dict(z=T(o["z"]), lam=T(o["lam"]), s=T(o["s"]), nu=T(o["nu"]) if e else torch.zeros(B, 0, dtype=torch.float64))
    keys = [str(k) for k in o["keys"]]
    om = {k: (T(o["om_" + k]) if k in keys else None) for k in NAMES}
    ref = bdm.double_backward(ins, pt, T(o["gz"]), T(o["glam"]), T(o["gnu"]) if e else None, om,
                              tuple(k for k in shared if ins[k] is not None), False)
    for k in keys:
        assert _per_qp_rel(o["g2_" + k], ref[k].numpy(), k not in shared) <= 1e-8, k


def test_hessian_symmetric_and_block_diagonal(out_dir):
    H = _load(out_dir, "hess")["H"]
    B, n = H.shape[:2]
    Hm = H.reshape(B * n, B * n)
    assert np.abs(Hm - Hm.T).max() <= 1e-10 * max(1.0, np.abs(Hm).max())
    for i in range(B):
        for j in range(B):
            if i != j:
                assert not H[i, :, j, :].any(), (i, j)


@pytest.mark.parametrize("job", ["jtj_9_3_both", "jtj_10_2_lb"])
def test_p_hessian_is_jtj_on_complementary_batches(out_dir, job):
    o = _load(out_dir, job)
    H, JtJ = o["H"], o["JtJ"]
    for i in range(JtJ.shape[0]):
        assert np.abs(H[i, :, i, :] - JtJ[i]).max() <= 1e-6 * max(1.0, np.abs(JtJ[i]).max()), i


def test_central_differences_gradgradcheck_and_first_order(out_dir):
    o = _load(out_dir, "cd")
    an, fd = float(o["an"]), float(o["fd"])
    assert abs(an - fd) <= 1e-5 * max(1.0, abs(an)), (an, fd)
    assert bool(o["same"])
    assert bool(o["gradgradcheck"])


def test_fp32_and_cpu_inputs_round_trip(out_dir):
    o = _load(out_dir, "roundtrip")
    assert list(o["f32_meta"]) == ["torch.float32", "cuda"]
    assert list(o["cpu_meta"]) == ["torch.float64", "cpu"]
    assert np.abs(o["cpu"] - o["f64"]).max() <= 1e-12 * max(1.0, np.abs(o["f64"]).max())
    assert np.abs(o["f32"] - o["f64"]).max() <= 1e-3 * max(1.0, np.abs(o["f64"]).max())
