"""The entries of tests/box_families.py stay on their edges, and the table covers every box-QP layout the planner can
give a shape, without a GPU (plans only: nothing runs on a device).

A layout that no entry has is a set of kernels that no edge or below-convergence test runs; a planner change that
creates one, or moves an entry off its edge, fails here.
"""
import ctypes
import os

import pytest

from tests.box_families import (DM_DENSE_ORDER, ENTRIES, ERR_TOO_LARGE, LAYOUTS, MAX_SMEM, ONE_NEQ_PAD_MAX, REJECTED,
                                check_entry, dense_plan, edges, knob, layout, sides_flags, slack)


def _lib():
    from qpth_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libqpth_b200.so not built")
    return _lib


@pytest.fixture
def no_knob(monkeypatch):
    monkeypatch.delenv("QPB200_BOX_CLUSTER", raising=False)


# nz: every 7th up to 1000, plus the widths of the edges and their neighbours; neq: the padding steps, every value of
# the last two equality tiles one CTA or a replicated-M cluster can hold, the first distributed one, and the edges
GRID_NZ = sorted(set(range(1, 1001, 7)) | {121, 122, 128, 208, 209, 248, 249, 300, 416, 417, 534, 535, 876, 877,
                                          1000, 1089, 2000, 7008, 7009, 11008, 11009})
GRID_NEQ = [0, 1, 7, 8, 9, 64] + list(range(116, 129)) + [129, 136, 200, 249, 312, 352]
GRID_SIDES = ("lb", "ub", "both")


def _walk(L):
    """{layout: first shape} and the (shape, plan) of every shape the planner takes"""
    lib = L.load()
    seen, plans = {}, []
    for nz in GRID_NZ:
        for neq in GRID_NEQ:
            if neq > nz:
                continue
            for sides in GRID_SIDES:
                p = L.BoxPlan()
                if lib.qpb200_box_plan_init(nz, neq, *(int(f) for f in sides_flags(sides)), ctypes.byref(p)) != 0:
                    continue
                seen.setdefault(layout(p), (nz, neq, sides))
                plans.append(((nz, neq, sides), p))
    return seen, plans


def test_entries_on_their_edges():
    """every entry lands on its layout, and every edge entry on its ok / cl_ctas / neq_pad / cl_slice / slack / dense
    ms_pad (check_entry asserts them); every layout has an edge entry"""
    _lib()
    with_edge = set()
    for name, ent in ENTRIES.items():
        with knob(ent["knob"]):
            p = check_entry(name)
        if ent["edge"]:
            with_edge.add(ent["layout"])
            if layout(p) != "dense":
                assert slack(p) >= 0, name
    assert with_edge == set(LAYOUTS)
    assert {e["layout"] for e in ENTRIES.values()} == set(LAYOUTS)
    assert len(edges()) >= 19


def test_rejected_shapes_are_too_large(no_knob):
    """one step past the widest cl8 slice and past the largest distributed M: no path takes them"""
    L = _lib()
    for nz, neq, sides in REJECTED:
        rc = L.load().qpb200_box_plan_init(nz, neq, *(int(f) for f in sides_flags(sides)), ctypes.byref(L.BoxPlan()))
        assert rc == ERR_TOO_LARGE, (nz, neq, sides, rc)


def test_every_planner_layout_has_an_entry(no_knob):
    """Walk qpb200_box_plan_init over the grid without the knob: every layout it returns has an entry in the table, and
    the walk reaches every layout of the table (so it cannot pass vacuously)."""
    seen, _ = _walk(_lib())
    missing = {k: v for k, v in seen.items() if k not in LAYOUTS}
    assert not missing, "layouts without an entry in tests/box_families.py (layout: first shape): %s" % missing
    assert set(seen) == set(LAYOUTS), sorted(set(LAYOUTS) - set(seen))


def test_one_cta_neq_pad_limits(no_knob):
    """For neq <= nz (A of full row rank, all the walk takes) shared memory binds before the one-row-per-thread limit:
    no one-CTA plan has neq_pad > 120, and at neq_pad 128 even nz = 121 or 128 misses 227 KB. For neq > nz the
    `neq_pad <= 128` term of plan.ok is the one that decides: (8, 128, lb) runs on one CTA at neq_pad 128, and
    (8, 136, lb) / (32, 136, lb) fit in 227 KB but are refused a CTA by that term alone."""
    L = _lib()
    _, plans = _walk(L)
    one = [(s, p.neq_pad) for s, p in plans if layout(p) == "one"]
    assert one and max(npad for _, npad in one) == ONE_NEQ_PAD_MAX
    for nz in (121, 128):
        for sides in GRID_SIDES:
            p = L.box_plan_for(nz, 128, *sides_flags(sides))
            assert p.ok == 0 and p.smem_bytes > MAX_SMEM, (nz, sides)
    for nz in (8, 64, 100):
        p = L.box_plan_for(nz, 128, True, False)
        assert p.ok == 1 and p.neq_pad == 128 and p.smem_bytes <= MAX_SMEM, nz
    for nz in (8, 32):
        p = L.box_plan_for(nz, 136, True, False)
        assert p.neq_pad == 136 and p.smem_bytes <= MAX_SMEM and p.ok == 0, nz


def test_dense_dm_switch_sits_between_384_and_392(no_knob):
    """neq_pad > 128: dense kernels up to dense order ms_pad 384, the distributed-M kernels from 392 on (wherever one
    of their clusters fits); the walk sees both sides of the switch"""
    L = _lib()
    _, plans = _walk(L)
    near = set()
    for (nz, neq, sides), p in plans:
        if p.neq_pad <= 128:
            continue
        rc, d = dense_plan(nz, p.nineq, neq)
        if rc != 0:
            assert p.cl_ctas, (nz, neq, sides)              # the dense path rejects it: only the dm kernels are left
            continue
        if d.ms_pad <= DM_DENSE_ORDER:
            assert layout(p) == "dense", (nz, neq, sides, d.ms_pad)
        elif layout(p) == "dense":                          # past the switch: dense only where no cluster fits
            with knob(8):
                q = L.BoxPlan()
                assert L.load().qpb200_box_plan_init(nz, neq, p.has_lb, p.has_ub, ctypes.byref(q)) == 0
            assert q.cl_ctas == 0, (nz, neq, sides, d.ms_pad)
        if d.ms_pad in (DM_DENSE_ORDER, DM_DENSE_ORDER + 8):
            near.add((d.ms_pad, layout(p)))
    assert (DM_DENSE_ORDER, "dense") in near and (DM_DENSE_ORDER + 8, "dm2") in near, near
