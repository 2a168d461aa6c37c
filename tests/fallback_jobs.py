"""Job list shared by tests/test_gpu_zz_fallback_families.py (parent: compares) and tests/gpu_child.py (child: solves).

The jobs exercise kernel configurations that were added to the suite after the round's last GPU session. They run in ONE
child process so that a fault or a hang in a configuration that has never run on hardware cannot take the rest of the GPU
suite (or the CUDA context of the pytest process) with it: the child is killed after a timeout, jobs that finished
before keep their results, the others fail with the reason."""

# round-1 families under QPB200_PF=0, against the goldens of the real reference
PF0_GOLDEN = ["band_smem", "band_smem_eq", "band_setup", "band_setup_eq", "c4"]

# orders above 256 (no product-form kernel, nothing fits shared memory): global-scratch family, against the oracle
BEYOND_SMEM = {
    "order_260": dict(nBatch=3, nz=120, nineq=260, neq=0, seed=41),
    "order_300": dict(nBatch=3, nz=260, nineq=300, neq=0, seed=43),
    "order_312_eq": dict(nBatch=2, nz=300, nineq=300, neq=10, seed=44),
}

# Product-form configurations that no golden / sweep shape reaches (found by enumerating plan_init over a shape grid):
# (nBatch, nz, nineq, neq, seed) -> (pf_global, pf_threads, setup_pf, setup_fast, pf2_ok, pf3_ok)
PF_OFF_GOLDEN = {
    "wide_nz_eq":     ((3, 181, 49, 8, 51),  (1, 256, 1, 0, 1, 1)),   # nz > 128: W / chol(Q) from L2 at ONE QP per SM, 256 threads
    "wide_nz":        ((3, 235, 34, 0, 52),  (1, 256, 0, 0, 1, 1)),   # nz > 208: generic global-scratch setup writing the staircase
    "wide_nz_small":  ((3, 230, 20, 4, 58),  (1, 256, 0, 0, 1, 1)),
    "tall_resident":  ((3, 60, 130, 4, 54),  (0, 256, 1, 0, 0, 0)),   # order 144 > 128 with everything in shared memory
    "tall_512_eq":    ((3, 124, 190, 8, 55), (1, 512, 1, 0, 0, 0)),   # 512-thread build with equality columns
    "tall_512":       ((3, 100, 150, 0, 59), (1, 512, 1, 0, 0, 0)),
    "wide_512":       ((3, 211, 130, 0, 56), (1, 512, 0, 0, 0, 0)),   # 512-thread solve after the generic setup
    "mid_two_per_sm": ((3, 151, 100, 8, 57), (1, 256, 1, 0, 1, 0)),   # order 112: two per SM possible, three not
    "nz_above_cta":   ((3, 300, 40, 0, 60),  (1, 256, 0, 0, 1, 1)),   # nz > threads per CTA (256 and 192): strided x passes
    "nz_400_eq":      ((2, 400, 60, 8, 61),  (1, 256, 0, 0, 1, 0)),
}


# equality-only QPs (nineq == 0: qpth_b200/eqonly.py, an extension of the reference's surface) against the closed form
EQ_ONLY = {
    "eq_tiny": dict(B=5, nz=12, neq=5, shared=False, seed=71),          # one warp per system
    "eq_c2_sized": dict(B=4, nz=100, neq=30, shared=False, seed=72),    # product-form kernels
    "eq_shared": dict(B=6, nz=40, neq=10, shared=True, seed=73),        # un-batched Q and A: gradients are batch means
}


def eq_only_problem(B, nz, neq, shared, seed):
    import numpy as np
    rs = np.random.RandomState(seed)
    L = rs.randn(nz, nz) if shared else rs.randn(B, nz, nz)
    Q = L @ np.swapaxes(L, -1, -2) + 0.1 * np.eye(nz)
    A = rs.randn(neq, nz) if shared else rs.randn(B, neq, nz)
    return dict(Q=Q, p=rs.randn(B, nz), A=A, b=rs.randn(B, neq), dl=rs.randn(B, nz))


def jobs():
    """[(job name, kind, payload, env, mode)] in execution order."""
    out = []
    for name in PF0_GOLDEN:
        out.append(("pf0_" + name, "golden", name, {"QPB200_PF": "0"}, None))
    for name, cfg in BEYOND_SMEM.items():
        out.append(("big_" + name, "random", cfg, {}, None))
    for name, ((B, nz, nineq, neq, seed), _) in sorted(PF_OFF_GOLDEN.items()):
        cfg = dict(nBatch=B, nz=nz, nineq=nineq, neq=neq, seed=seed)
        for mode in ("latency", "throughput"):
            out.append(("pf_%s_%s" % (name, mode), "random", cfg, {}, mode))
    for name, cfg in EQ_ONLY.items():
        out.append((name, "eq_only", cfg, {}, None))
    return out


# Per-family tests (tests/kernel_families.py): the families with dispatch branches that had never run before them.
KKT_B = 3
KKT_VARIANTS = [(shared, reg) for shared in (False, True) for reg in (0.0, 1e-7)]
TRAJ_B = 2
TRAJ_RUNS = [(it, eps) for eps in (1e-12, 1e-6) for it in (1, 2, 3, 5, 20)]
# the edge entries (up to order 1056, where one model solve takes seconds): eps = 1e-12 only (the 1e-6 runs repeat its
# first iterations) and no un-batched variant (the index arithmetic of a shared system is that of the mid-range shapes)
TRAJ_RUNS_EDGE = [(it, 1e-12) for it in (1, 2, 3, 5, 20)]


def traj_runs(fam):
    from tests.kernel_families import FAMILIES
    return TRAJ_RUNS_EDGE if "edge" in FAMILIES[fam] else TRAJ_RUNS


def traj_unbatched(fam, shape):
    """[False] plus, for the first shape of a family that is not an edge entry, True (Q, G, A, h, b shared)."""
    from tests.kernel_families import FAMILIES
    f = FAMILIES[fam]
    return [False] + ([True] if shape == f["shapes"][0] and "edge" not in f else [])


def kkt_job_name(fam, shape, shared, reg):
    return "kkt_%s_%dx%dx%d_%s_%s" % ((fam,) + tuple(shape) + ("shared" if shared else "batched", "reg" if reg else "plain"))


def bwd_job_name(fam, shape):
    return "bwd_%s_%dx%dx%d" % ((fam,) + tuple(shape))


def traj_job_name(fam, shape, unbatched, it, eps):
    return "traj_%s_%dx%dx%d_%s_it%d_eps%g" % ((fam,) + tuple(shape) + ("unbatched" if unbatched else "batched", it, eps))


def family_kkt_jobs():
    from tests.kernel_families import cases
    return [(kkt_job_name(fam, s, shared, reg), "call",
             ("kkt_on_gpu", dict(fam=fam, shape=s, B=KKT_B, shared=shared, reg=reg)), {}, None)
            for fam, s in cases(child=True) for shared, reg in KKT_VARIANTS]


def family_backward_jobs():
    from tests.kernel_families import cases
    return [(bwd_job_name(fam, s), "call", ("backward_on_gpu", dict(fam=fam, shape=s)), {}, None)
            for fam, s in cases(child=True)]


def family_trajectory_jobs():
    from tests.kernel_families import cases
    out = []
    for fam, s in cases(child=True, forward=True):
        for u in traj_unbatched(fam, s):
            for it, eps in traj_runs(fam):
                out.append((traj_job_name(fam, s, u, it, eps), "call",
                            ("trajectory_on_gpu", dict(fam=fam, shape=s, B=TRAJ_B, unbatched=u, maxIter=it, eps=eps)),
                            {}, None))
    return out
