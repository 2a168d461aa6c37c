"""The plan table of the Jacobian kernels' edges (tests/jacobian_edges.py) without a GPU.

- Every figure of every entry: the shared memory qpb200_jacobian_smem / qpb200_box_jacobian_smem /
  qpb200_boxq_jacobian_smem reports, and nblk and the block count of the Python mirror of the kernels' layouts.
- The next shape of each edge is not covered (smem 0) or has no plan; the forward plan each box entry reaches.
- The mirror against the C smem functions over a grid of shapes of each kernel.
- The per-variable model without equality rows (box_jacobian_models.diagonal_box_jacobian) against the dense model.
- The GPU job list (tests/jacobian_edges_jobs.py) covers every entry.
"""
import numpy as np
import pytest

from tests import box_jacobian_models as bm
from tests import jacobian_edges as je


@pytest.mark.parametrize("name", list(je.JAC))
def test_jac_entry(name):
    ent = je.JAC[name]
    rc, plan = je.jac_plan(*ent["shape"])
    assert rc == 0
    assert je.jac_smem(plan) == ent["smem"]
    assert je.jac_plan_layout(plan) == (ent["nblk"], ent["smem"], ent["blocks"])
    if ent["next"] is not None:
        rc, nplan = je.jac_plan(*ent["next"])
        assert rc == 4 if ent["shape"][0] == 1056 else (rc == 0 and je.jac_smem(nplan) == 0), (ent["next"], rc)


def test_jac_widest_nz_has_no_plan_past_it():
    """1056 is the widest nz any plan takes, with or without equality rows"""
    for m, e in ((1, 0), (8, 132), (8, 0), (1, 8)):
        assert je.jac_plan(1056, m, e)[0] == 0
        assert je.jac_plan(1057, m, e)[0] == 4


@pytest.mark.parametrize("name", list(je.BOX))
def test_box_entry(name):
    ent = je.BOX[name]
    n, e, sides = ent["shape"]
    rc, plan = je.box_plan(n, e, sides)
    assert rc == 0
    smem = je.box_smem(plan)
    assert smem == ent["smem"]
    assert je.box_layout(n, e, *je.sides_flags(sides)) == (ent["nblk"], ent["smem"], ent["blocks"])
    # the forward plan that reaches the kernel
    assert je.box_forward(plan) == ent["fwd"]
    assert bool(plan.ok) == (ent["fwd"] == "one")
    assert plan.cl_ctas == (0 if ent["fwd"] == "one" else int(ent["fwd"][2:]))
    assert (plan.neq_pad > 128) == ent["fwd"].startswith("dm")
    if e == 0:                   # shared memory within 256..448 bytes of the cap
        assert 256 <= je.JAC_MAX_SMEM - smem <= 448
    if ent["next"] is not None:
        rc, nplan = je.box_plan(*ent["next"])
        assert rc == 0 and je.box_smem(nplan) == 0


@pytest.mark.parametrize("name", list(je.BOXQ))
def test_boxq_entry(name):
    from tests.boxq_families import ENTRIES, check_entry
    ent = je.BOXQ[name]
    assert ENTRIES[name]["shape"] == ent["shape"]
    plan = check_entry(name)
    assert je.boxq_smem(plan) == ent["smem"]
    assert je.boxq_layout(*ent["shape"][:2], *je.sides_flags(ent["shape"][2])) == (ent["nblk"], ent["smem"],
                                                                                    ent["blocks"])


def test_every_kernel_has_few_warp_entries_in_the_sweep():
    """the sweep runs each kernel with its fewest buffers (one warp; two for k_boxq_jacobian) and with all eight"""
    from tests.boxq_families import ENTRIES, kernel_entries
    for tab in (je.JAC, je.BOX, je.BOXQ):
        swept = {v["nblk"] for v in tab.values() if v["sweep"]}
        assert 8 in swept and min(swept) == min(v["nblk"] for v in tab.values())
    assert min(je.boxq_layout(*ENTRIES[k]["shape"][:2], *je.sides_flags(ENTRIES[k]["shape"][2]))[0]
               for k in kernel_entries()) == 2
    assert min(v["nblk"] for v in je.BOX.values()) == min(v["nblk"] for v in je.JAC.values()) == 1


def test_jac_mirror_grid():
    seen = set()
    for n in (1, 7, 8, 9, 17, 45, 100, 199, 200, 201, 320, 640, 1056):
        for m in (1, 8, 13, 61, 120, 199, 208, 209, 260):
            for e in (0, 1, 3, 8, 17, 40, 129, 184):
                rc, plan = je.jac_plan(n, m, e)
                if rc:
                    continue
                nb, smem, _ = je.jac_plan_layout(plan)
                assert smem == je.jac_smem(plan), (n, m, e)
                seen.add(nb)
    assert {0, 1, 3, 8} <= seen, seen


def test_box_mirror_grid():
    seen = set()
    for n in (1, 5, 8, 31, 64, 200, 201, 600, 1000, 2616, 2617, 2880, 2881, 4000):
        for e in (0, 1, 9, 40, 120, 129, 160, 200, 201, 250):
            for sides in ("lb", "ub", "both"):
                rc, plan = je.box_plan(n, e, sides)
                if rc:
                    continue
                nb, smem, _ = je.box_layout(n, e, *je.sides_flags(sides))
                assert smem == je.box_smem(plan), (n, e, sides)
                seen.add(nb)
    assert {0, 1, 8} <= seen, seen


def test_boxq_mirror_grid():
    from tests.boxq_families import plan_init
    seen = set()
    for n in list(range(1, 40, 3)) + list(range(40, 260, 11)):
        for e in sorted({0, 1, 7, 8, 9, n // 2, n}):
            for sides in ("lb", "ub", "both"):
                rc, plan = plan_init(n, e, sides)
                if rc:
                    continue
                nb, smem, _ = je.boxq_layout(n, e, *je.sides_flags(sides))
                assert smem == je.boxq_smem(plan), (n, e, sides)
                seen.add(nb)
    assert {0, 2, 8} <= seen, seen


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("sides", ["lb", "ub", "both"])
@pytest.mark.parametrize("n", [1, 9, 24])
def test_diagonal_model_matches_dense(n, sides, spread):
    rs = np.random.RandomState(n + len(sides) + spread)
    has_lb, has_ub = je.sides_flags(sides)
    nlb = n if has_lb else 0
    m = nlb + (n if has_ub else 0)
    q = rs.uniform(0.5, 2.0, n)
    if spread:        # d over 1e-8 .. 1e8: the refined dense model is the reference
        lam, s = 10 ** rs.uniform(-4, 4, m), 10 ** rs.uniform(-4, 4, m)
    else:
        lam, s = rs.uniform(0.1, 10, m), rs.uniform(0.1, 10, m)
    Jv = bm.diagonal_box_jacobian(q, lam, s, nlb, has_ub)
    Jd = bm.dense_box_jacobian_refined(np.diag(q), None, lam, s, nlb, has_ub)
    assert Jv.shape == Jd.shape == (n + m, n * (1 + has_lb + has_ub))
    assert np.abs(Jv - Jd).max() < 1e-13 * np.abs(Jd).max()
    if not spread:
        assert np.abs(Jv - bm.dense_box_jacobian(np.diag(q), None, lam, s, nlb, has_ub)).max() < 1e-13 * np.abs(Jd).max()


def test_jobs_cover_every_entry():
    from tests.jacobian_edges_jobs import jobs
    names = [nm for nm, _, _ in jobs()]
    assert len(names) == len(set(names))
    for tab, kind in ((je.JAC, "jac"), (je.BOX, "box"), (je.BOXQ, "boxq")):
        for k, v in tab.items():
            assert "edge_%s_%s" % (kind, k) in names
            assert ("sweep_%s_%s" % (kind, k) in names) == v["sweep"]
