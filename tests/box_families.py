"""One table of the box-QP layouts the planner can pick (csrc/qp_box.cu), with the shapes at the edges of each plan.

Layouts: `one` (k_box_*<OneCta>, one CTA per QP), `cl2` / `cl4` / `cl8` (k_box_*<Cluster>, a cluster of C CTAs per
QP, M replicated), `dm2` / `dm4` / `dm8` (k_box_*_dm, M distributed over the cluster, neq_pad > 128) and `dense` (no
box kernel: BoxQPFunction runs the dense kernels on the dense equivalent).

Each entry has a shape (nz, neq, sides), the QPB200_BOX_CLUSTER value it runs under (None: the planner's own choice)
and, for edge entries, what makes it an edge: the expected ok / cl_ctas / neq_pad / cl_slice, the dense plan's ms_pad
(the dense / distributed-M switch), and `max_slack`, the most bytes that may be left under 227 KB by the CTA's dynamic
shared memory (smem_bytes for `one`, cl_smem_bytes for a cluster). check_entry asserts them before anything runs, so a
planner change cannot move an entry off its edge without failing. The non-edge entries are the mid-range shapes of
tests/test_gpu_box*.py.

The edges, as qpb200_box_plan_init reports them (slack in bytes):
  one   (121, 117, both) neq_pad 120, 128 B left: the most equality rows one CTA holds for neq <= nz (15 tiles; there
        shared memory binds before the `neq_pad <= 128` term of plan.ok, which decides only for neq > nz, e.g.
        (8, 136, lb)); (128, 120, lb) 1088 B; (876, 0, both) the widest nz, 384 B
  cl2   (877, 0, both) one CTA misses by 384 B; (122, 117, both) one CTA misses by 1.7 KB; (534, 64, lb) 0 B
  cl4   (208, 128, both) neq_pad 128 (16 tiles, one substitution row per thread), 0 B
  cl8   (416, 128, both) 0 B (one more variable and no box kernel fits); (7008, 0, both) slice 876, 128 B (the widest);
        (11008, 0, lb) slice 1376, 512 B; forced onto (9, 3, both) and (5, 1, both): ranks 5-7 hold no variables
  dm2   (249, 129, lb) dense order 392, just past kDmDenseOrder; (300, 232, lb) 960 B
  dm4   (1089, 264, lb) 0 B: one more equality row takes dm8
  dm8   (1000, 352, lb) 0 B, 44 block rows over 8 ranks (6 or 5 each); (2000, 312, lb) slice 250, 0 B
  dense (248, 129, lb) dense order 384; (417, 128, both) past the largest cl8 slice
Past the edges qpb200_box_plan_init returns QPB200_ERR_TOO_LARGE: REJECTED.

Every shape has neq <= nz: random rows of A then have full row rank, which M = A H^-1 A' needs.
"""
import contextlib
import ctypes
import os

MAX_SMEM = 232448                # kBoxMaxSmem: 227 KB of dynamic shared memory per CTA
DM_DENSE_ORDER = 384             # kDmDenseOrder: neq_pad > 128 runs the distributed-M kernels past this dense ms_pad
ONE_NEQ_PAD_MAX = 120            # the most equality rows (padded) one CTA holds for neq <= nz: shared memory binds
                                 # before the 128-row limit
LAYOUTS = ("one", "cl2", "cl4", "cl8", "dm2", "dm4", "dm8", "dense")
ERR_TOO_LARGE = 4


def _e(layout, shape, knob=None, **edge):
    return dict(layout=layout, shape=shape, knob=knob, edge=edge or None)


ENTRIES = {
    # one CTA per QP
    "one_mid_lb": _e("one", (64, 40, "lb")),
    "one_mid_both": _e("one", (31, 13, "both")),
    "one_mid_ub": _e("one", (20, 0, "ub")),
    "one_full": _e("one", (121, 117, "both"), ok=1, cl_ctas=0, neq_pad=120, max_slack=128),
    "one_neq120": _e("one", (128, 120, "lb"), ok=1, cl_ctas=0, neq_pad=120, max_slack=1088),
    "one_wide": _e("one", (876, 0, "both"), ok=1, cl_ctas=0, neq_pad=0, max_slack=384),
    # a cluster per QP, M replicated in every CTA
    "cl2_mid_forced": _e("cl2", (31, 13, "both"), knob=2),
    "cl2_mid": _e("cl2", (1000, 8, "both")),
    "cl2_mid_lb": _e("cl2", (1500, 3, "lb")),
    "cl2_past_one_wide": _e("cl2", (877, 0, "both"), ok=0, cl_ctas=2, neq_pad=0, cl_slice=439),
    "cl2_past_one_neq": _e("cl2", (122, 117, "both"), ok=0, cl_ctas=2, neq_pad=120, cl_slice=61, max_slack=14976),
    "cl2_full": _e("cl2", (534, 64, "lb"), ok=0, cl_ctas=2, neq_pad=64, cl_slice=267, max_slack=0),
    "cl4_mid_forced": _e("cl4", (31, 13, "both"), knob=4),
    "cl4_mid": _e("cl4", (600, 64, "both")),
    "cl4_mid_480": _e("cl4", (480, 64, "both")),
    "cl4_mid_lb": _e("cl4", (450, 100, "lb")),
    "cl4_full": _e("cl4", (208, 128, "both"), ok=0, cl_ctas=4, neq_pad=128, cl_slice=52, max_slack=0),
    "cl8_mid_forced": _e("cl8", (31, 13, "both"), knob=8),
    "cl8_mid": _e("cl8", (6000, 1, "both")),
    "cl8_mid_box": _e("cl8", (5000, 0, "both")),
    "cl8_full": _e("cl8", (416, 128, "both"), ok=0, cl_ctas=8, neq_pad=128, cl_slice=52, max_slack=0),
    "cl8_widest": _e("cl8", (7008, 0, "both"), ok=0, cl_ctas=8, neq_pad=0, cl_slice=876, max_slack=128),
    "cl8_widest_lb": _e("cl8", (11008, 0, "lb"), ok=0, cl_ctas=8, neq_pad=0, cl_slice=1376, max_slack=512),
    "cl8_empty_9": _e("cl8", (9, 3, "both"), knob=8, ok=1, cl_ctas=8, neq_pad=8, cl_slice=2),
    "cl8_empty_5": _e("cl8", (5, 1, "both"), knob=8, ok=1, cl_ctas=8, neq_pad=8, cl_slice=1),
    # M distributed over the cluster
    "dm2_mid_forced": _e("dm2", (150, 130, "ub"), knob=2),
    "dm2_boundary": _e("dm2", (249, 129, "lb"), ok=0, cl_ctas=2, neq_pad=136, cl_slice=125, dense_ms_pad=392),
    "dm2_full": _e("dm2", (300, 232, "lb"), ok=0, cl_ctas=2, neq_pad=232, cl_slice=150, max_slack=960),
    "dm4_mid_forced": _e("dm4", (160, 136, "both"), knob=4),
    "dm4_mid": _e("dm4", (600, 249, "lb")),
    "dm4_sudoku": _e("dm4", (729, 249, "lb")),
    "dm4_full": _e("dm4", (1089, 264, "lb"), ok=0, cl_ctas=4, neq_pad=264, cl_slice=273, max_slack=0),
    "dm8_mid_forced": _e("dm8", (200, 180, "lb"), knob=8),
    "dm8_full": _e("dm8", (1000, 352, "lb"), ok=0, cl_ctas=8, neq_pad=352, cl_slice=125, max_slack=0),
    "dm8_slice": _e("dm8", (2000, 312, "lb"), ok=0, cl_ctas=8, neq_pad=312, cl_slice=250, max_slack=0),
    # no box kernel: the dense kernels on the dense equivalent
    "dense_mid": _e("dense", (150, 130, "ub")),
    "dense_boundary": _e("dense", (248, 129, "lb"), ok=0, cl_ctas=0, neq_pad=136, dense_ms_pad=384),
    "dense_past_cl8": _e("dense", (417, 128, "both"), ok=0, cl_ctas=0, neq_pad=128),
}

REJECTED = [(7009, 0, "both"), (1000, 353, "lb")]


def edges():
    """names of the edge entries"""
    return [k for k, v in ENTRIES.items() if v["edge"]]


def sides_flags(sides):
    return sides != "ub", sides != "lb"


@contextlib.contextmanager
def knob(C):
    """QPB200_BOX_CLUSTER=C for the block (unset for None)"""
    old = os.environ.get("QPB200_BOX_CLUSTER")
    if C is None:
        os.environ.pop("QPB200_BOX_CLUSTER", None)
    else:
        os.environ["QPB200_BOX_CLUSTER"] = str(C)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("QPB200_BOX_CLUSTER", None)
        else:
            os.environ["QPB200_BOX_CLUSTER"] = old


def layout(plan):
    """the layout a box plan runs (the branches of box_launch and BoxQPFunction)"""
    if plan.cl_ctas:
        return ("dm%d" if plan.neq_pad > 128 else "cl%d") % plan.cl_ctas
    return "one" if plan.ok else "dense"


def slack(plan):
    """bytes left under 227 KB by one CTA of the layout; None for `dense`"""
    lay = layout(plan)
    if lay == "dense":
        return None
    return MAX_SMEM - (plan.smem_bytes if lay == "one" else plan.cl_smem_bytes)


def dense_plan(nz, nineq, neq):
    """(rc, plan) of qpb200_plan_init for the dense equivalent"""
    from qpth_b200 import _lib
    d = _lib.Plan()
    return _lib.load().qpb200_plan_init(nz, nineq, neq, ctypes.byref(d)), d


def check_entry(name):
    """The plan of entry `name` under its knob (call inside `knob(entry["knob"])`): asserts its layout and, for an edge
    entry, every value that makes it an edge. Returns the plan."""
    from qpth_b200 import _lib
    ent = ENTRIES[name]
    nz, neq, sides = ent["shape"]
    assert os.environ.get("QPB200_BOX_CLUSTER") == (None if ent["knob"] is None else str(ent["knob"])), name
    p = _lib.box_plan_for(nz, neq, *sides_flags(sides))
    assert layout(p) == ent["layout"], (name, layout(p))
    assert neq <= nz, name
    for k, v in (ent["edge"] or {}).items():
        if k == "max_slack":
            assert 0 <= slack(p) <= v, (name, slack(p), v)
        elif k == "dense_ms_pad":
            rc, d = dense_plan(nz, p.nineq, neq)
            assert rc == 0 and d.ms_pad == v, (name, rc, d.ms_pad)
        else:
            assert getattr(p, k) == v, (name, k, getattr(p, k), v)
    return p
