"""The Jacobian kernels at the edges of their plans, on the GPU (k_jacobian, k_box_jacobian, k_boxq_jacobian).

Every job runs in one child process (tests/jacobian_edges_jobs.py) and each test reads what its job measured:
- the mask sweep: every row and column mask through the C entry points into a NaN-filled view between sentinel guard
  bands, per-QP and shared inputs: every element written, nothing written outside, bit-identical to the full-mask J;
- every entry of tests/jacobian_edges.py: its layout (nblk, shared memory, blocks) and coverage, J against the dense
  model (or the per-variable long-double model without equality rows) within 1e-10 per-QP relative, J t against the
  JVP, g' J against the dual backward, the identities; the next shape is not covered and its column path's J_z,p
  agrees (relative to the whole reference J);
- the public jacobian(): the default call is the z rows of duals=True bit for bit, wrt order and repeats, mixed
  sharing against the dense model, and a BoxQPFunction forward on the widest both-sided plan.
"""
import os
import tempfile
import time

import numpy as np
import pytest

from tests import jacobian_edges as je
from tests.jacobian_edges_jobs import B, jobs, run_child

pytestmark = pytest.mark.gpu
_OUT = {}
TOL = 1e-10


@pytest.fixture(scope="module")
def out_dir():
    if "dir" not in _OUT:
        d = tempfile.mkdtemp(prefix="jacobian_edges_jobs_")
        t0 = time.time()
        _OUT["dir"], _OUT["why"] = d, run_child(d)
        print("jacobian edges child: %.1f s" % (time.time() - t0))
    return _OUT["dir"]


def _load(out_dir, name):
    path = os.path.join(out_dir, name + ".npz")
    if not os.path.exists(path):
        err = os.path.join(out_dir, name + ".err")
        pytest.fail(open(err).read() if os.path.exists(err) else "no output: %s" % _OUT.get("why"))
    return dict(np.load(path))


SWEEPS = [nm for nm, _, _ in jobs() if nm.startswith("sweep_")]


@pytest.mark.parametrize("name", SWEEPS)
def test_mask_sweep(out_dir, name):
    got = _load(out_dir, name)
    for sharing in ("batched", "shared"):
        res = got[sharing]
        assert len(res) > 1
        bad = [tuple(int(v) for v in r) for r in res if r[2] or r[3] or r[4]]
        # (rows, cols, NaN left in the view, guard doubles changed, elements not bit-identical to the full-mask J)
        assert not bad, (sharing, bad)


def _check_errors(got, what):
    for k in what:
        assert np.all(got["err_" + k] < TOL), (k, got["err_" + k])


@pytest.mark.parametrize("name", list(je.JAC))
def test_jac_edge(out_dir, name):
    ent = je.JAC[name]
    got = _load(out_dir, "edge_jac_" + name)
    assert bool(got["covered"])
    assert tuple(int(v) for v in got["layout"]) == (ent["nblk"], ent["smem"], ent["blocks"])
    assert len(got["err_ref"]) == (B if je.order("jac", ent["shape"]) <= 3000 else 1)
    _check_errors(got, ("ref", "jvp", "grad", "sym"))
    if ent["next"] is not None:
        if int(got["next_rc"]) == 0:
            assert not bool(got["next_covered"])
            assert float(got["next_err"]) < TOL
        else:
            assert ent["shape"][0] == 1056 and int(got["next_rc"]) == 4      # no plan past the widest nz


@pytest.mark.parametrize("name", list(je.BOX))
def test_box_edge(out_dir, name):
    ent = je.BOX[name]
    got = _load(out_dir, "edge_box_" + name)
    assert bool(got["covered"])
    assert str(got["fwd"]) == ent["fwd"]
    _check_errors(got, ("ref", "jvp", "grad", "ident"))
    if ent["next"] is not None:
        assert not bool(got["next_covered"])
        assert float(got["next_err"]) < TOL


@pytest.mark.parametrize("name", list(je.BOXQ))
def test_boxq_edge(out_dir, name):
    got = _load(out_dir, "edge_boxq_" + name)
    assert bool(got["covered"])
    _check_errors(got, ("ref", "jvp", "grad", "ident"))
    assert len(got["err_ref"]) == B


@pytest.mark.parametrize("job", ["api_qp", "api_box"])
def test_default_call_and_wrt_order(out_dir, job):
    got = _load(out_dir, job)
    for k, v in got.items():
        # [default call, each single wrt..., reversed wrt with a repeat]
        assert v.all(), (k, v)


@pytest.mark.parametrize("q_shared", [1, 0])
def test_mixed_sharing_qp(out_dir, q_shared):
    got = _load(out_dir, "api_mixed_qp_%d" % q_shared)
    assert int(got["nsys"]) == B
    # converged: d spans many decades, and the dense model's solve loses digits with it; the kernel agrees with it to
    # the column path's own accuracy
    for ref, col in zip(got["err_ref"], got["err_col"]):
        assert col < 1e-6 and ref < max(1e-8, 10 * col), (ref, col)


@pytest.mark.parametrize("q_shared", [1, 0])
def test_mixed_sharing_box(out_dir, q_shared):
    got = _load(out_dir, "api_mixed_box_%d" % q_shared)
    assert (int(got["sq"]) == 0) == bool(q_shared) and (int(got["sA"]) == 0) != bool(q_shared)
    # converged: against the refined dense model, to the accuracy a d spread over many decades leaves
    assert np.all(got["err_ref"] < 1e-7), got["err_ref"]


def test_box_edge_forward(out_dir):
    got = _load(out_dir, "api_box_edge")
    assert str(got["fwd"]) == "cl4" and not bool(got["dense"]) and bool(got["covered"])
    print("converged (2616, 0, both): d spans %s" % got["dspan"])
    # the z rows (1 / H and d / H per variable) to 1e-10; the lam rows d o (rz - z) cancel where d ~ 1e16 (an active
    # bound at a converged point), as they do in the backward, so the whole J to 1e-6
    assert np.all(got["err_z"] < TOL), got["err_z"]
    assert np.all(got["err_ref"] < 1e-6), got["err_ref"]

