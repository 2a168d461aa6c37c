"""Jacobians of (z, lam, nu) with respect to (p, lb, ub, b) on the GPU (jacobian() of BoxQPFunction).

The kernels (qpb200_box_jacobian, qpb200_boxq_jacobian) are new to the device, so every job runs in one child process
(tests/box_jacobian_jobs.py) and each test reads its job's output:
- box-family entries of every layout at a point: J against the dense model (tests/box_jacobian_models) within 1e-10
  per-QP relative, with per-QP and with shared q and A; the kernel against the column path; J t against the JVP of
  random batched tangents of p, lb, ub, b; g' J against the dual backward; the identities; the coverage flag;
- every dense-Q family entry the forward kernels run, the same way (qpb200_boxq_jacobian);
- the widest cluster entries, which take the column path: J_z,p against a JVP, and its symmetry;
- the dense fallback entries against the dense model at their returned point;
- converged BoxQPFunction solutions, diagonal and dense Q (the clamps act): against the dense model, and the kernel
  against the column path;
- central differences on strictly complementary batches, and fp32 / CPU inputs.
"""
import os
import tempfile

import numpy as np
import pytest

from tests import box_jacobian_models as bm
from tests import jacobian_models as jm
from tests.box_jacobian_jobs import CD, CONVERGED, DENSE_NAMES, ENTRY_NAMES, WIDE_NAMES, run_child
from tests.boxq_families import kernel_entries

pytestmark = pytest.mark.gpu
_OUT = {}
# the entries whose M or column buffers do not fit one CTA: they take the column path (qpb200_box_jacobian_smem = 0;
# tests/test_box_jacobian_cpu.UNCOVERED_ENTRIES)
UNCOVERED = ("dm2_full", "dm4_mid", "dm4_sudoku", "dm4_full", "dm8_full")


@pytest.fixture(scope="module")
def out_dir():
    if "dir" not in _OUT:
        d = tempfile.mkdtemp(prefix="box_jacobian_jobs_")
        _OUT["dir"], _OUT["why"] = d, run_child(d)
    return _OUT["dir"]


def _load(out_dir, name):
    path = os.path.join(out_dir, name + ".npz")
    if not os.path.exists(path):
        err = os.path.join(out_dir, name + ".err")
        pytest.fail(open(err).read() if os.path.exists(err) else "no output: %s" % _OUT.get("why"))
    return dict(np.load(path))


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _sides(name):
    from tests.box_families import ENTRIES
    n, e, sides = ENTRIES[name]["shape"]
    return n, e, (n if sides != "ub" else 0), sides != "lb"


@pytest.mark.parametrize("name", ENTRY_NAMES)
def test_entry_jacobian(out_dir, name):
    got = _load(out_dir, "entry_" + name)
    assert bool(got["covered"]) == (name not in UNCOVERED)
    _check_point(got, *_sides(name), dense_Q=False)


@pytest.mark.parametrize("name", kernel_entries())
def test_boxq_entry_jacobian(out_dir, name):
    """Every dense-Q family entry the forward kernels run is covered by qpb200_boxq_jacobian."""
    from tests.boxq_families import ENTRIES
    got = _load(out_dir, "boxq_" + name)
    assert bool(got["covered"])
    n, e, sides = ENTRIES[name]["shape"]
    _check_point(got, n, e, (n if sides != "ub" else 0), sides != "lb", dense_Q=True)


def _check_point(got, n, e, nlb, has_ub, dense_Q):
    m = nlb + (n if has_ub else 0)
    A = lambda i: got["A"][i] if e else None
    Qm = (lambda i: got["q"][i]) if dense_Q else (lambda i: np.diag(got["q"][i]))
    B = got["J"].shape[0]
    for i in range(B):
        assert _rel(got["J"][i], got["Jc"][i]) < 1e-10, (i, _rel(got["J"][i], got["Jc"][i]))
    # the dense model is an order-(n + 2m + e) solve: past order 3000 the first QP only
    for i in (range(B) if n + 2 * m + e <= 3000 else [0]):
        J = got["J"][i]
        Jd = bm.dense_box_jacobian(Qm(i), A(i), got["lam"][i], got["s"][i], nlb, has_ub)
        assert J.shape == Jd.shape
        assert _rel(J, Jd) < 1e-10, (i, _rel(J, Jd))
        Js = bm.dense_box_jacobian(Qm(0), A(0), got["lam"][i], got["s"][i], nlb, has_ub)
        assert _rel(got["J_shared"][i], Js) < 1e-10
        d = jm.clamped_d(got["lam"][i], got["s"][i])
        assert bm.identity_residuals(J, n, m, e, nlb, has_ub, d) < 1e-10 * np.abs(J[:n]).max()
        t = np.concatenate([got["tp"][i]] + ([got["tlb"][i]] if nlb else []) + ([got["tub"][i]] if has_ub else [])
                           + ([got["tb"][i]] if e else []))
        jvp = np.concatenate([got["dz"][i], got["dlam"][i]] + ([got["dnu"][i]] if e else []))
        assert _rel(J @ t, jvp) < 1e-10
        g = np.concatenate([got["dl"][i], got["glam"][i]] + ([got["gnu"][i]] if e else []))
        grads = np.concatenate([got["grad_dp"][i]] + ([got["grad_dlb"][i]] if nlb else [])
                               + ([got["grad_dub"][i]] if has_ub else []) + ([got["grad_db"][i]] if e else []))
        assert _rel(g @ J, grads) < 1e-10


@pytest.mark.parametrize("name", WIDE_NAMES)
def test_wide_entry_columns(out_dir, name):
    """The column path on the widest cluster plans (the kernel does not cover them): J_z,p t against the JVP of t, and
    J_z,p symmetric."""
    got = _load(out_dir, "wide_" + name)
    assert not bool(got["covered"])
    J = got["J"]
    assert _rel(J @ got["tp"], got["dz"]) < 1e-10
    assert np.abs(J - J.T).max() < 1e-10 * np.abs(J).max()


@pytest.mark.parametrize("name", DENSE_NAMES)
def test_dense_fallback_jacobian(out_dir, name):
    got = _load(out_dir, "dense_" + name)
    n, e, nlb, has_ub = _sides(name)
    assert bool(got["dense"])
    for i in range(got["J"].shape[0]):
        Jd = bm.dense_box_jacobian(np.diag(got["q"][i]), got["A"] if e else None, got["lam"][i], got["s"][i], nlb,
                                   has_ub)
        assert _rel(got["J"][i], Jd) < 1e-10, (i, _rel(got["J"][i], Jd))


@pytest.mark.parametrize("case", CONVERGED, ids=["%d_%d_%s_%d" % c for c in CONVERGED])
def test_converged_jacobian(out_dir, case):
    n, e, sides, dense_Q = case
    got = _load(out_dir, "conv_%d_%d_%s_%d" % case)
    nlb, has_ub = (n if sides != "ub" else 0), sides != "lb"
    assert list(got["names"]) == ["p"] + (["lb"] if nlb else []) + (["ub"] if has_ub else []) + (["b"] if e else [])
    assert bool(got["covered"])
    for i in range(got["J"].shape[0]):
        Q = got["q"][i] if dense_Q else np.diag(got["q"][i])
        Jd = bm.dense_box_jacobian(Q, got["A"] if e else None, got["lam"][i], got["s"][i], nlb, has_ub)
        # converged: d spans many decades, and the dense model's order-(n + 2m + e) solve loses digits with it
        col_err = _rel(got["Jc"][i], Jd)
        assert col_err < 1e-6, (i, col_err)
        # the clamps act at a converged point: the kernel agrees with the column path to the column path's own accuracy
        assert _rel(got["J"][i], got["Jc"][i]) < max(1e-8, 10 * col_err), (i, _rel(got["J"][i], got["Jc"][i]))


@pytest.mark.parametrize("case", CD, ids=["%d_%d_%s" % c for c in CD])
def test_central_differences(out_dir, case):
    got = _load(out_dir, "cd_%d_%d_%s" % case)
    assert _rel(got["Jfd"], got["J"]) < 1e-5, _rel(got["Jfd"], got["J"])


def test_dtype_device_roundtrip(out_dir):
    got = _load(out_dir, "roundtrip")
    assert list(got["f64_meta"]) == ["torch.float64", "cuda", "False"]
    assert list(got["f32_meta"]) == ["torch.float32", "cuda", "False"]
    assert list(got["cpu_meta"]) == ["torch.float64", "cpu", "False"]
    assert _rel(got["cpu"], got["f64"]) < 1e-12
    assert _rel(got["f32"], got["f64"]) < 1e-4
