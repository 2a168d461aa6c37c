"""One table of the dense-Q box-QP shapes (csrc/qp_boxq.cu, BoxQPFunction(dense_Q=True)) at the edges of their plan,
with the benchmark's shapes and the first shapes past the plan.

The dense-Q kernels have one layout: one CTA of 256 threads per QP, the bordered staircase of order
nz_pad + neq_pad and every vector in shared memory (qpb200_boxq_plan.ok). Past it, BoxQPFunction runs the dense
kernels on the dense equivalent (`dense` entries).

Each entry has a shape (nz, neq, sides), the inputs passed un-batched (`shared`), the problem generator (`gen`:
"random" is tests.boxq_util.random_boxq, "bench" the problems of scripts/bench_box_dense.py) and what
qpb200_boxq_plan_init must report for it (`edge`): ok, order, neq_pad, and `max_slack`, the most bytes the CTA's
dynamic shared memory may leave under 227 KB. `past` names the dimensions one more of which makes the plan not ok
("nz": one more variable, "neq": one more equality row). check_entry asserts all of it before anything runs, so a
planner change cannot move an entry off its edge without failing.

The edges, as qpb200_boxq_plan_init reports them (slack in bytes):
  (192, 0, both) order 192, 128 B: the widest nz with both bounds;  (200, 0, lb) / (200, 0, ub) order 200, 3264 B
  (192, 1, lb) / (192, 1, ub) order 200, 2496 B and (184, 1, both) order 192, 192 B: tests/test_boxq_cpu.LARGEST
  (144, 32, both), (97, 71, lb) (odd nz, 1 padding equality row), (112, 60, ub): order 176, 0 B
  (84, 83, lb) order 176, 320 B and (88, 80, both) order 168, 4224 B: the most equality rows with neq <= nz
  (64, 8, both) and (64, 9, both): neq_pad 8 (no padding row) and 16 (7 padding rows with -1 on the diagonal)
Shared memory binds before the 256 rows of the sweeps everywhere: the first shape past each edge has order <= 256.

Every shape has neq <= nz: random rows of A then have full row rank, which M = A H^-1 A' needs.
"""
import ctypes

MAX_SMEM = 232448                # kBoxMaxSmem: 227 KB of dynamic shared memory per CTA
MAX_ORDER = 256                  # kBoxNT: the sweeps own one row per thread


def _e(shape, shared=(), gen="random", past=(), **edge):
    return dict(shape=shape, shared=tuple(shared), gen=gen, past=tuple(past), edge=edge)


ENTRIES = {
    # the widest nz
    "widest_both": _e((192, 0, "both"), ok=1, order=192, neq_pad=0, max_slack=128, past=("nz", "neq")),
    "widest_lb": _e((200, 0, "lb"), ok=1, order=200, neq_pad=0, max_slack=3264, past=("nz", "neq")),
    "widest_ub": _e((200, 0, "ub"), ok=1, order=200, neq_pad=0, max_slack=3264, past=("nz", "neq")),
    # tests/test_boxq_cpu.LARGEST: the largest shape per bound pattern with one equality row
    "largest_lb": _e((192, 1, "lb"), ok=1, order=200, neq_pad=8, max_slack=2496, past=("nz",)),
    "largest_ub": _e((192, 1, "ub"), ok=1, order=200, neq_pad=8, max_slack=2496, past=("nz",)),
    "largest_both": _e((184, 1, "both"), ok=1, order=192, neq_pad=8, max_slack=192, past=("nz", "neq")),
    # every byte of shared memory
    "full_both": _e((144, 32, "both"), ok=1, order=176, neq_pad=32, max_slack=0, past=("nz", "neq")),
    "full_odd_lb": _e((97, 71, "lb"), ok=1, order=176, neq_pad=72, max_slack=0, past=("nz", "neq")),
    "full_ub": _e((112, 60, "ub"), ok=1, order=176, neq_pad=64, max_slack=0, past=("nz", "neq")),
    # the most equality rows with neq <= nz
    "most_eq_lb": _e((84, 83, "lb"), ok=1, order=176, neq_pad=88, max_slack=320, past=("neq",)),
    "most_eq_both": _e((88, 80, "both"), ok=1, order=168, neq_pad=80, max_slack=4224, past=("nz", "neq")),
    # the equality tile boundary: no padding row, 7 padding rows
    "tile_8": _e((64, 8, "both"), ok=1, order=72, neq_pad=8),
    "tile_9": _e((64, 9, "both"), ok=1, order=80, neq_pad=16),
    # tiny
    "tiny_1_0": _e((1, 0, "both"), ok=1, order=8, neq_pad=0),
    "tiny_1_1": _e((1, 1, "lb"), ok=1, order=16, neq_pad=8),
    "tiny_8_1": _e((8, 1, "ub"), ok=1, order=16, neq_pad=8),
    # the benchmark's shapes (scripts/bench_box_dense.py), with its sharing and its problems
    "bench_portfolio": _e((100, 1, "both"), shared=("A", "b", "lb", "ub"), gen="bench", ok=1, order=112, neq_pad=8),
    "bench_mpc": _e((80, 0, "both"), shared=("Q", "lb", "ub"), gen="bench", ok=1, order=80, neq_pad=0),
    "bench_lb_64_40": _e((64, 40, "lb"), shared=("A", "b", "lb"), gen="bench", ok=1, order=104, neq_pad=40),
    "bench_largest": _e((184, 1, "both"), shared=("A", "b", "lb", "ub"), gen="bench", ok=1, order=192, neq_pad=8),
    # one step past an edge: the dense kernels on the dense equivalent
    "dense_193": _e((193, 0, "both"), ok=0, order=200, neq_pad=0),
    "dense_185": _e((185, 1, "both"), ok=0, order=200, neq_pad=8),
    "dense_145": _e((145, 32, "both"), ok=0, order=184, neq_pad=32),
}


def kernel_entries():
    """the entries the dense-Q kernels run"""
    return [k for k, v in ENTRIES.items() if v["edge"]["ok"]]


def edges():
    """the kernel entries at an edge of the plan (not the tile, tiny or benchmark entries)"""
    return [k for k, v in ENTRIES.items() if v["past"]]


def dense_entries():
    return [k for k, v in ENTRIES.items() if not v["edge"]["ok"]]


def sides_flags(sides):
    return sides != "ub", sides != "lb"


def plan_init(nz, neq, sides):
    """qpb200_boxq_plan_init, uncached: (rc, plan)"""
    from qpth_b200 import _lib
    p = _lib.BoxQPlan()
    hl, hu = sides_flags(sides)
    return _lib.load().qpb200_boxq_plan_init(nz, neq, int(hl), int(hu), ctypes.byref(p)), p


def next_shape(shape, dim):
    nz, neq, sides = shape
    return (nz + 1, neq, sides) if dim == "nz" else (nz, neq + 1, sides)


def check_entry(name):
    """The plan of entry `name`: asserts ok, order, neq_pad and the slack it reports, and that one more variable or
    equality row (`past`) is not ok because shared memory runs out (at order <= 256). Returns the plan."""
    ent = ENTRIES[name]
    nz, neq, sides = ent["shape"]
    assert neq <= nz, name
    rc, p = plan_init(nz, neq, sides)
    assert rc == 0, (name, rc)
    for k, v in ent["edge"].items():
        if k == "max_slack":
            assert 0 <= MAX_SMEM - p.smem_bytes <= v, (name, MAX_SMEM - p.smem_bytes, v)
        else:
            assert getattr(p, k) == v, (name, k, getattr(p, k), v)
    for dim in ent["past"]:
        rc, q = plan_init(*next_shape(ent["shape"], dim))
        assert rc == 0 and q.ok == 0, (name, dim)
        assert q.order <= MAX_ORDER and q.smem_bytes > MAX_SMEM, (name, dim, q.order, q.smem_bytes)
    return p


def problem(name, B, seed):
    """A problem dict of entry `name` (tests.boxq_util layout: Q, p, A, b, lb, ub, dl), B in the batch; the inputs in
    `shared` un-batched."""
    from tests.boxq_util import random_boxq
    ent = ENTRIES[name]
    nz, neq, sides = ent["shape"]
    if ent["gen"] == "random":
        return random_boxq(seed, B, nz, neq, sides, ent["shared"])
    return bench_problem(nz, sides, neq, ent["shared"], B, seed)


def bench_problem(n, sides, e, shared, B, seed):
    """The problems of scripts/bench_box_dense.py: Q = F F' / k + 0.05 I of rank n / 4 + 1 plus the ridge, lb = 0,
    ub = 1; one equality row is sum(z) = 1 (the long-only portfolio), more are random rows through an interior point."""
    import numpy as np
    rs = np.random.RandomState(seed)
    nq = 1 if "Q" in shared else B
    F = rs.randn(nq, n, n // 4 + 1)
    Q = np.einsum("bik,bjk->bij", F, F) / F.shape[-1] + 0.05 * np.eye(n)
    hl, hu = sides_flags(sides)
    lb = np.zeros(n) if hl else None
    ub = np.ones(n) if hu else None
    A = np.ones((e, n)) if e == 1 else rs.randn(e, n)
    z0 = 0.05 + 0.5 * rs.rand(n) / max(1, n // 20)
    b = A @ z0 if e else np.zeros(0)
    if e == 1:
        b = np.ones(1)
    bx = dict(Q=Q[0] if "Q" in shared else Q, p=rs.randn(B, n), A=A if e else np.zeros(0), b=b, lb=lb, ub=ub,
              dl=rs.randn(B, n))
    for k in ("A", "b", "lb", "ub"):        # the benchmark shares these; batch the ones this entry does not
        if k not in shared and bx[k] is not None and np.asarray(bx[k]).size:
            bx[k] = np.broadcast_to(bx[k], (B,) + np.shape(bx[k])).copy()
    return bx
