"""The kernel families of QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) and their seeded problems, shared by the GPU tests of
tests/test_gpu_reg_families.py and the plan pins of tests/test_reg_refine_cpu.py.

Each family: the plan flags of `_lib.plan_for_ir` that identify it, and one SPD-Q, one low-rank-Q and one LP case
(pc.spd / pc.lowrank / pc.lp at the family's shapes); the edge entries at the end pin their (setup, solve) pairing and
edge as well, and have an SPD and (where the shape takes one) an LP case. Every test asserts the flags before it solves, so a planner change
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



def wellcond(seed, nz, nineq, neq):
    """One QP of tests/kernel_families.wellcond_qp_batch (cond(Q) <= 9 at every nz): the SPD case of the edge entries."""
    from tests.kernel_families import wellcond_qp_batch
    pr = wellcond_qp_batch(1, nz, nineq, neq, seed=seed)
    return tuple(pr[k][0] for k in ("Q", "p", "G", "h", "A", "b"))


# Shapes at the edges of tests/kernel_families.py whose IR_UNOPT plan is not that of a family above: a (setup, solve)
# pairing (kernel_families.dispatch) the families do not have, or a kernel at its last bytes, largest order or most
# equality rows. SPD cases (wellcond), and an LP where nineq = nrand + 2 nz fits the shape.
FAMILIES.update({
    # the resident build at 0 B of slack (ms_pad 168, neq 17)
    "edge_pf_res_full": dict(flags=dict(pf=1, pf_global=0, tiny=0), pair=("setup_pf", "pf_res"), slack=0, cases=dict(
        spd=lambda s: wellcond(s, 39, 144, 17),
        lp=lambda s: pc.lp(s, nz=39, nrand=66, neq=17))),
    # the resident build at its largest order (ms_pad 200)
    "edge_pf_res_order": dict(flags=dict(pf=1, pf_global=0, tiny=0), pair=("setup_pf", "pf_res"), ms_pad=200, cases=dict(
        spd=lambda s: wellcond(s, 4, 193, 0),
        lp=lambda s: pc.lp(s, nz=4, nrand=185, neq=0))),
    # the global-scratch setup writing the staircase for the resident solve (360 B left)
    "edge_gs_pf_res": dict(flags=dict(pf=1, pf_global=0, tiny=0), pair=("setup_global", "pf_res"), slack=360,
                           cases=dict(spd=lambda s: wellcond(s, 213, 8, 0))),
    # k_setup_fast before the resident solve with 64 equality rows
    "edge_sf_pf_res": dict(flags=dict(pf=1, pf_global=0, tiny=0), pair=("setup_fast", "pf_res"), neq_pad=64,
                           cases=dict(spd=lambda s: wellcond(s, 97, 9, 64))),
    # the L2 build with 129 equality rows (17 equality tiles): after the global-scratch setup with 72 B left, and after
    # k_setup_pf at ms_pad 200
    "edge_l2_full": dict(flags=dict(pf=1, pf_global=1, tiny=0), pair=("setup_global", "pf_global256"), slack=72,
                         neq_pad=136, cases=dict(spd=lambda s: wellcond(s, 430, 41, 129))),
    "edge_l2_order": dict(flags=dict(pf=1, pf_global=1, tiny=0), pair=("setup_pf", "pf_global256"), ms_pad=200,
                          neq_pad=136, cases=dict(spd=lambda s: wellcond(s, 208, 57, 129))),
    # the L2 build at the widest nz of the table (strided x passes over 256 threads, nz = 1000)
    "edge_l2_wide": dict(flags=dict(pf=1, pf_global=1, tiny=0), pair=("setup_global", "pf_global256"), neq_pad=104,
                         cases=dict(spd=lambda s: wellcond(s, 1000, 9, 100))),
    # the generic global-scratch kReg kernels at order 1056 with 129 equality rows (368 B left). backward_only: one model
    # solve of the forward takes ~8 s at this order (the trajectory test would spend ~10 minutes in the model); the kReg
    # forward of this kernel runs at order 272 (global_scratch above) and its default-mode forward at this shape
    # (tests/test_gpu_trajectory.py, edge_generic_full). With nineq = 920 >> nz the refinement contracts by only ~1e-2
    # per step here: the model's own error against the dense solve is 4.8e-3 / 3.4e-5 / 2.1e-7 / 1.3e-9 at IR_STEPS
    # 0 / 1 / 2 / 3, and the backward test's bounds (10 x that error) follow it
    "edge_generic_full": dict(flags=dict(pf=0, smem_resident=0, tiny=0), pair=("setup_global", "generic_global"),
                              slack=368, ms_pad=1056, neq_pad=136, backward_only=True,
                              cases=dict(spd=lambda s: wellcond(s, 133, 920, 129))),
})

CASES = [(fam, kind) for fam in FAMILIES for kind in FAMILIES[fam]["cases"]]


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
    if "pair" in f:
        from tests.kernel_families import dispatch, slack
        assert dispatch(plan) == f["pair"], (fam, dispatch(plan), f["pair"])
        assert 0 <= slack(plan)[1] <= f.get("slack", slack(plan)[1]), (fam, slack(plan), f.get("slack"))
        for k in ("ms_pad", "neq_pad"):
            assert getattr(plan, k) == f.get(k, getattr(plan, k)), (fam, k, getattr(plan, k))
    return plan
