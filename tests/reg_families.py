"""The kernel families of QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) and their seeded problems, shared by the GPU tests of
tests/test_gpu_reg_families.py and the plan pins of tests/test_reg_refine_cpu.py.

Each family: the plan flags of `_lib.plan_for_ir` that identify it, and one SPD-Q, one low-rank-Q and one LP case
(pc.spd / pc.lowrank / pc.lp at the family's shapes). Every test asserts the flags before it solves, so a planner change
cannot move a case silently to another family. Across a family's shapes there is an odd nz, and an nineq and (where the
family has equality rows) an neq that are not multiples of 8. (nineq of pc.lowrank / pc.lp is nrand + 2 nz.)
"""
from oracle import psd_cases as pc

FAMILIES = {
    # the smallest product-form plans (ms_pad <= 32)
    "pf_small": dict(flags=dict(pf=1, pf_global=0, tiny=0), max_ms_pad=32, cases=dict(
        spd=lambda s: pc.spd(s, nz=13, nineq=19, neq=3),
        lowrank=lambda s: pc.lowrank(s, nz=9, nrand=3, rank=2, neq=2),
        lp=lambda s: pc.lp(s, nz=7, nrand=5, neq=0))),
    # product-form kernels with W, chol(Q) and the factor in shared memory
    "pf_resident": dict(flags=dict(pf=1, pf_global=0, smem_resident=1, tiny=0), cases=dict(
        spd=lambda s: pc.spd(s, nz=41, nineq=35, neq=6),
        lowrank=lambda s: pc.lowrank(s, nz=31, nrand=13, rank=4, neq=3),
        lp=lambda s: pc.lp(s, nz=45, nrand=13, neq=5))),
    # product-form kernels reading W and chol(Q) from global memory (L2)
    "pf_l2": dict(flags=dict(pf=1, pf_global=1, tiny=0), cases=dict(
        spd=lambda s: pc.spd(s, nz=61, nineq=157, neq=5),
        lowrank=lambda s: pc.lowrank(s, nz=99, nrand=1, rank=5, neq=0),
        lp=lambda s: pc.lp(s, nz=50, nrand=70, neq=10))),
    # the generic global-scratch kernels (k_forward / k_solve_kkt with kReg)
    "global_scratch": dict(flags=dict(pf=0, smem_resident=0, tiny=0), cases=dict(
        spd=lambda s: pc.spd(s, nz=121, nineq=257, neq=3),
        lowrank=lambda s: pc.lowrank(s, nz=119, nrand=3, rank=8, neq=5),
        lp=lambda s: pc.lp(s, nz=100, nrand=60, neq=10))),
}

CASES = [(fam, kind) for fam in FAMILIES for kind in ("spd", "lowrank", "lp")]


def ids(cs):
    return ["%s-%s" % c for c in cs]


def problem(fam, kind, seed):
    return FAMILIES[fam]["cases"][kind](seed)


def family_plan(fam, case):
    """The IR_UNOPT plan of a case, asserted to belong to family `fam`."""
    from qpth_b200 import _lib
    Q, p, G, h, A, b = case
    plan = _lib.plan_for_ir(Q.shape[0], G.shape[0], A.shape[0])
    f = FAMILIES[fam]
    for k, v in f["flags"].items():
        assert getattr(plan, k) == v, (fam, k, getattr(plan, k), v)
    if "max_ms_pad" in f:
        assert plan.ms_pad <= f["max_ms_pad"], (fam, plan.ms_pad)
    return plan
