"""The kernel-family table (tests/kernel_families.py) against the planner, on the CPU: every shape of every family plans
to that family under its knobs, and each family's shapes cover the edges the kernels pad (odd nz, nineq and neq that
are not multiples of 8)."""
import pytest

from tests.kernel_families import FAMILIES, cases, family_env, family_plan, ids


@pytest.fixture(scope="module")
def lib():
    from qpth_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.mark.parametrize("fam,shape", cases(forward=True), ids=ids(cases(forward=True)))
def test_family_shapes_plan_to_their_family(fam, shape, lib):
    with family_env(fam):
        family_plan(fam, shape)


@pytest.mark.parametrize("fam", sorted(f for f in FAMILIES if "edge" not in FAMILIES[f]))
def test_family_shapes_cover_padding_edges(fam):
    """(The edge entries are single shapes chosen by the planner's limits; tests/test_plan_edges_cpu.py checks them.)"""
    shapes = FAMILIES[fam]["shapes"]
    assert len(shapes) >= 2
    assert any(nz % 2 for nz, _, _ in shapes)
    assert any(nineq % 8 for _, nineq, _ in shapes)
    assert any(neq % 8 for _, _, neq in shapes)


def test_plan_cache_tells_the_coop_knob_apart(lib):
    """QPB200_COOP selects between two kernel families at the same shape: the cached plans must differ."""
    with family_env("r1_fast"):
        fast = family_plan("r1_fast", (100, 100, 0))
    with family_env("r1_coop"):
        coop = family_plan("r1_coop", (100, 100, 0))
    assert (fast.coop, coop.coop) == (0, 1)
