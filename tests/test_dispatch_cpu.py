"""The kernel table of the library (choose_kernel in qpth_b200/csrc/qp_kernels.cu, which every entry point switches on,
exported as qpb200_plan_kernels) agrees with the independent statement of it in tests/kernel_families.py: `dispatch`
for the setup, forward and backward / solve_kkt kernels, `reg_dispatch` for the regularised entry points, and `slack`
for the plan field that gives each launch its dynamic shared memory. The per-family and edge tests rely on that
statement to know which kernels they run.

Walks qpb200_plan_init and qpb200_plan_init_reg over a thinned copy of the grid of tests/test_plan_edges_cpu.py plus the
table's own shapes, under the planner knobs, crossed with the flags a caller may set after plan_init (pf_two, pf_three,
coop: also where their *_ok is clear). Plans only: nothing runs on a device."""
import ctypes
import itertools
import os

import pytest

from tests.kernel_families import KMAX_SMEM, PER_CTA, cases, dispatch, reg_dispatch, slack
from tests.test_plan_edges_cpu import GRID_NEQ, GRID_NINEQ, GRID_NZ

# QPB200_K_* (include/qpth_b200.h) in order; the setup and the solve entry points each have their own "tiny"
KERNELS = (None, "tiny", "setup_pf192", "setup_pf", "setup_fast", "setup_smem", "setup_global", "tiny", "pf192",
           "pf_two", "pf_global512", "pf_global256", "pf_res512", "pf_res", "coop", "fast", "generic_smem",
           "generic_global")
ENTRIES = ("setup", "forward", "kkt", "reg", "kkt_reg")      # QPB200_ENTRY_*
# the limit slack() measures a kernel's shared memory against (KMAX_SMEM for the others), and the non-256 CTA sizes
LIMIT = {"setup_pf192": PER_CTA[3], "pf192": PER_CTA[3], "pf_two": PER_CTA[2], "coop": 232448 // 2 - 1024 - 64}
THREADS = {"tiny": 32, "setup_pf192": 192, "pf192": 192, "pf_global512": 512, "pf_res512": 512}
KNOBS = ({}, {"QPB200_PF": "0"}, {"QPB200_NT512": "2"}, {"QPB200_SETUP_PF": "0"}, {"QPB200_SETUP_PF": "1"})


def _lib():
    from qpth_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libqpth_b200.so not built")
    return _lib


def _shapes():
    grid = itertools.product(GRID_NZ[::5], GRID_NINEQ[::5], GRID_NEQ[::2])
    return sorted(set(grid) | {tuple(s) for _, s in cases(forward=True)})


def expected(plan, L):
    """[(kernel, CTA size, shared-memory bytes)] per entry point, from dispatch, reg_dispatch and slack."""
    def row(name, sl):
        return (name, THREADS.get(name, 256), LIMIT.get(name, KMAX_SMEM) - sl)
    setup, solve = dispatch(plan)
    su, so = slack(plan)
    kkt = "pf_res" if solve == "pf_res512" else solve         # the resident 512-thread build is a forward only
    p256 = L.Plan.from_buffer_copy(plan)                        # solve_kkt_reg: the solve_kkt rules at 256 threads
    p256.pf_three, p256.pf_threads = 0, 256
    kkt_reg = dispatch(p256)[1]
    reg = reg_dispatch(plan)
    if reg is not None:
        assert reg == solve, (reg, solve)                       # (so its shared memory is the forward's)
    return [row(setup, su), row(solve, so), row(kkt, so), row(reg, so) if reg else (None, 0, 0),
            row(kkt_reg, slack(p256)[1])]


def test_plan_kernels_matches_the_restatement(monkeypatch):
    L = _lib()
    lib = L.load()
    out = (ctypes.c_int64 * (3 * len(ENTRIES)))()
    seen, done, n = {e: set() for e in ENTRIES}, set(), 0
    for knobs in KNOBS:
        for k in ("QPB200_PF", "QPB200_NT512", "QPB200_SETUP_PF"):
            monkeypatch.delenv(k, raising=False)
        for k, v in knobs.items():
            monkeypatch.setenv(k, v)
        for nz, nineq, neq in _shapes():
            for init in (lib.qpb200_plan_init, lib.qpb200_plan_init_reg):
                p = L.Plan()
                if init(nz, nineq, neq, ctypes.byref(p)) != 0:
                    continue
                for two, three, coop in itertools.product((0, 1), repeat=3):
                    q = L.Plan.from_buffer_copy(p)
                    q.pf_two, q.pf_three, q.coop = two, three, coop
                    key = bytes(q)
                    if key in done:
                        continue
                    done.add(key)
                    assert lib.qpb200_plan_kernels(ctypes.byref(q), out) == 0
                    got = [(KERNELS[out[3 * i]], out[3 * i + 1], out[3 * i + 2]) for i in range(len(ENTRIES))]
                    want = expected(q, L)
                    assert got == want, ((nz, nineq, neq), knobs, init.__name__, (two, three, coop), got, want)
                    for e, g in zip(ENTRIES, got):
                        seen[e].add(g[0])
                    n += 1
    assert n > 10000, n
    # every kernel of each entry point was reached (a grid that missed one would check it vacuously)
    solve = set(KERNELS[7:])
    assert seen["setup"] == set(KERNELS[1:7]), seen["setup"]
    assert seen["forward"] == solve, solve - seen["forward"]
    assert seen["kkt"] == solve - {"pf_res512"}, seen["kkt"]
    assert seen["reg"] == {None, "pf_global256", "pf_res", "generic_global"}, seen["reg"]
    assert seen["kkt_reg"] == solve - {"pf192", "pf_global512", "pf_res512"}, seen["kkt_reg"]


def test_plan_kernels_rejects_null():
    L = _lib()
    lib = L.load()
    out = (ctypes.c_int64 * 15)()
    assert lib.qpb200_plan_kernels(None, out) == 1
    assert lib.qpb200_plan_kernels(ctypes.byref(L.Plan()), None) == 1
