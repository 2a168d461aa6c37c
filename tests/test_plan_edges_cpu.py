"""The edge entries of tests/kernel_families.py stay on their edges, and the table covers every (setup, solve) kernel
pairing the planner can give a shape, without a GPU (plans only: nothing runs on a device).

A pairing that no entry has is a pair of kernels that no test below convergence runs together; a planner change that
creates one fails here until the table has an entry for it.

The table's pairings are those the current planner gives the table's shapes. Only the edge entries pin theirs
(check_edge). A planner change that moves a mid-range family onto a new pairing therefore counts that pairing as
covered, and the family keeps running in-process instead of in the child process; its flags in FAMILIES usually catch
such a move.
"""
import ctypes
import os

import pytest

from tests.kernel_families import FAMILIES, cases, dispatch, family_env, family_plan, slack


def _lib():
    from qpth_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libqpth_b200.so not built")
    return _lib


# nz, nineq: every 3rd / 4th value up to 260 (the product-form and round-1 shapes), then every 30th up to 1000;
# neq: the padding steps (0, 1, 8 | 9, 16 | 17) and the most equality tiles (128 | 129)
GRID_NZ = list(range(1, 261, 3)) + list(range(270, 1001, 30))
GRID_NINEQ = list(range(1, 261, 4)) + list(range(270, 1001, 30))
GRID_NEQ = [0, 1, 5, 8, 9, 16, 17, 40, 64, 100, 128, 129]


def _modes(p, L):
    """The plan of each mode of QPFunction from one qpb200_plan_init result, as _lib.plan_for derives them."""
    lat = L.Plan.from_buffer_copy(p)
    lat.pf_two = lat.pf_three = 0
    thr = L.Plan.from_buffer_copy(p)
    thr.pf_three = 1 if thr.pf3_ok else 0
    thr.pf_two = 1 if (thr.pf2_ok and not thr.pf_three) else 0
    return lat, thr


def _table_pairings():
    out = {}
    for fam, shape in cases(forward=True):
        with family_env(fam):
            out.setdefault(dispatch(family_plan(fam, shape)), []).append((fam, shape))
    return out


def test_edge_entries_on_their_edges():
    """Every edge entry lands on its pairing, slack, ms_pad, neq_pad and lglobal side (family_plan asserts them), and
    every edge kernel keeps a non-negative slack."""
    _lib()
    n = 0
    for fam, shape in cases(forward=True):
        if "edge" not in FAMILIES[fam]:
            continue
        with family_env(fam):
            p = family_plan(fam, shape)
        su, so = slack(p)
        assert su >= 0 and so >= 0, (fam, shape, su, so)
        n += 1
    assert n >= 20


def test_shapes_have_full_row_rank_equality_constraints():
    """neq <= nz - 4 for every shape: the default mode needs A to have full row rank, which random rows of an A with at
    least 4 more columns than rows have."""
    for fam, shape in cases(forward=True):
        nz, nineq, neq = shape
        assert neq <= nz - 4 or neq == 0, (fam, shape)


def test_every_planner_pairing_has_an_entry():
    """Walk qpb200_plan_init over a coarse shape grid in latency and throughput mode (the default settings, no
    development knob): every (setup, solve) pairing it dispatches to is the pairing of some entry of the table."""
    L = _lib()
    lib = L.load()
    table = _table_pairings()
    seen = {}
    for nz in GRID_NZ:
        for nineq in GRID_NINEQ:
            for neq in GRID_NEQ:
                if neq > nz - 4:
                    continue
                p = L.Plan()
                if lib.qpb200_plan_init(nz, nineq, neq, ctypes.byref(p)) != 0:
                    continue
                for q in _modes(p, L):
                    seen.setdefault(dispatch(q), (nz, nineq, neq))
    missing = {k: v for k, v in seen.items() if k not in table}
    assert not missing, "pairings without an entry in tests/kernel_families.py (pairing: first shape): %s" % missing
    # and the grid is fine enough to find every pairing that the table's shapes get with the default settings (a grid
    # that missed the rare ones, such as the global-scratch setup before the resident solve, would pass vacuously)
    default = set()
    for fam, (nz, nineq, neq) in cases(forward=True):
        p = L.Plan()
        assert lib.qpb200_plan_init(nz, nineq, neq, ctypes.byref(p)) == 0
        default.add(dispatch(_modes(p, L)[1 if FAMILIES[fam]["two"] else 0]))
    assert default <= set(seen), sorted(default - set(seen))
