"""One table of the kernel families the planner can pick, and the GPU runs the per-family tests share.

Each family: development knobs (env), the `two=` argument of `_lib.plan_for` (throughput mode), the plan flags that
identify it, and shapes (nz, nineq, neq). Every test asserts the flags before it solves, so a planner change cannot
move a case silently to another family. Across a family's shapes there is an odd nz, an nineq and (where the family
takes equality constraints) an neq that are not multiples of 8.

`child`: families with dispatch branches that had never run before these tests (the 192- and 512-thread solve_kkt
builds, the regularised solve on a 512-thread plan, the resident 512-thread forward, the edge entries below). Their GPU
work runs in the child process of tests/gpu_child.py, so that a fault there fails only their own tests.

The `edge_*` entries sit at the edges of the planner: a kernel's last bytes of shared memory, its widest nz, the most
equality rows (neq_pad 136: 17 equality tiles), the largest order, the (setup, solve) pairings that only such shapes
reach, and the two sides of the staging of chol(Q) in the L2 product-form backward (`lglobal`). Their shapes were found
by walking qpb200_plan_init over a shape grid; `edge` pins what makes each one an edge (check_edge), so a planner change
cannot move it off. They use `gen="wellcond"` (wellcond_qp_batch): at random_qp_batch's conditioning (cond(Q) ~ 1e8 at
nz = 670) the tests' bounds would measure rounding instead of the kernels.
"""
import contextlib
import ctypes
import os

import numpy as np

FAMILIES = {
    "tiny": dict(env={}, two=False, flags=dict(tiny=1, threads=32),
                 shapes=[(24, 19, 5), (31, 21, 0), (17, 13, 3)]),
    "pf_one_setup_fast": dict(env={}, two=False,
                              flags=dict(tiny=0, pf=1, pf_global=0, pf_threads=256, setup_pf=0, setup_fast=1, pf_two=0,
                                         pf_three=0),
                              shapes=[(100, 100, 0), (99, 93, 3)]),
    "pf_one_setup_pf": dict(env={}, two=False,
                            flags=dict(tiny=0, pf=1, pf_global=0, pf_threads=256, setup_pf=1, pf_two=0, pf_three=0),
                            shapes=[(50, 50, 10), (45, 61, 3)]),
    "pf_one_setup_pf_env": dict(env={"QPB200_SETUP_PF": "1"}, two=False,
                                flags=dict(tiny=0, pf=1, pf_global=0, pf_threads=256, setup_pf=1, setup_fast=1, pf_two=0,
                                           pf_three=0),
                                shapes=[(100, 100, 0), (99, 93, 3)]),
    "pf_two": dict(env={"QPB200_MAXQPS": "2"}, two=True, flags=dict(tiny=0, pf=1, pf_two=1, pf_three=0),
                   shapes=[(100, 100, 0), (77, 90, 5), (151, 100, 8)]),
    "pf_three": dict(env={}, two=True, flags=dict(tiny=0, pf=1, pf_global=0, pf_two=0, pf_three=1), child=True,
                     shapes=[(100, 100, 0), (50, 50, 10), (108, 90, 0), (63, 85, 3)]),
    "pf_global_256": dict(env={}, two=False,
                          flags=dict(tiny=0, pf=1, pf_global=1, pf_threads=256, pf_two=0, pf_three=0),
                          shapes=[(181, 49, 8), (183, 45, 3)]),
    "pf_global_512": dict(env={}, two=False, flags=dict(tiny=0, pf=1, pf_global=1, pf_threads=512, pf_two=0, pf_three=0),
                          child=True, shapes=[(200, 200, 0), (124, 190, 8), (127, 187, 5)]),
    "pf_resident_512": dict(env={"QPB200_NT512": "2"}, two=False,
                            flags=dict(tiny=0, pf=1, pf_global=0, pf_threads=512, pf_two=0, pf_three=0),
                            child=True, forward_only=True, shapes=[(100, 100, 0), (61, 93, 5)]),
    "r1_fast": dict(env={"QPB200_PF": "0", "QPB200_COOP": "0"}, two=False, flags=dict(tiny=0, pf=0, fast=1, coop=0),
                    shapes=[(100, 100, 0), (87, 70, 3)]),
    "r1_coop": dict(env={"QPB200_PF": "0", "QPB200_COOP": "1"}, two=False, flags=dict(tiny=0, pf=0, fast=1, coop=1),
                    shapes=[(100, 100, 0), (87, 70, 3)]),
    "r1_generic_smem": dict(env={"QPB200_PF": "0"}, two=False,
                            flags=dict(tiny=0, pf=0, fast=0, setup_fast=0, smem_resident=1),
                            shapes=[(20, 120, 0), (24, 116, 4), (21, 115, 3)]),
    "r1_fast_generic_setup": dict(env={"QPB200_PF": "0"}, two=False,
                                  flags=dict(tiny=0, pf=0, fast=1, setup_fast=0, smem_resident=1),
                                  shapes=[(150, 20, 0), (151, 21, 3)]),
    "global_scratch": dict(env={}, two=False, flags=dict(tiny=0, pf=0, smem_resident=0),
                           shapes=[(120, 260, 0), (121, 257, 3)]),
}


def _edge(two, pair, shapes, **edge):
    return dict(env={}, two=two, flags=dict(tiny=int(pair[1] == "tiny")), child=True, gen="wellcond", shapes=shapes,
                edge=dict(pair=pair, **edge))


FAMILIES.update({
    # pairings that only these shapes reach
    "edge_gs_pf_res": _edge(False, ("setup_global", "pf_res"), [(213, 8, 0)], slack=360),
    "edge_sf_pf192": _edge(True, ("setup_fast", "pf192"), [(97, 9, 64)], neq_pad=64),
    "edge_sf_pf_two": _edge(True, ("setup_fast", "pf_two"), [(73, 49, 64), (65, 73, 40)], ms_pad=120),
    "edge_spf_pf192": _edge(True, ("setup_pf", "pf192"), [(193, 17, 64)], slack=936),
    # resident product form: every byte of kMaxSmem, and the largest order
    "edge_pf_res_full": _edge(False, ("setup_pf", "pf_res"), [(39, 144, 17)], slack=0, ms_pad=168),
    "edge_pf_res_order": _edge(False, ("setup_pf", "pf_res"), [(4, 193, 0)], ms_pad=200),
    # the 512-thread L2 build: 72 B left with 17 equality tiles, the widest nz, ms_pad 200 after k_setup_pf
    "edge_512_full": _edge(False, ("setup_global", "pf_global512"), [(670, 17, 129)], slack=72, neq_pad=136),
    "edge_512_wide": _edge(False, ("setup_global", "pf_global512"), [(880, 1, 128)], slack=824),
    "edge_512_order": _edge(False, ("setup_pf", "pf_global512"), [(208, 57, 129)], ms_pad=200, neq_pad=136),
    # the 256-thread L2 build (the 512-thread one does not fit): 72 B left with 17 equality tiles, and nz = 1000
    "edge_256_full": _edge(False, ("setup_global", "pf_global256"), [(430, 41, 129)], slack=72, neq_pad=136),
    "edge_256_wide": _edge(False, ("setup_global", "pf_global256"), [(1000, 9, 100)], slack=2112, neq_pad=104),
    # throughput mode: the widest nz (strided x passes at nz = 740 over 256 threads and nz = 480 over 192), and the
    # fullest two- / three-per-SM slots
    "edge_two_wide": _edge(True, ("setup_global", "pf_two"), [(740, 1, 0)], slack=808),
    "edge_192_wide": _edge(True, ("setup_global", "pf192"), [(480, 1, 0)], slack=2024),
    "edge_two_full": _edge(True, ("setup_global", "pf_two"), [(610, 9, 40)], slack=248),
    "edge_192_full": _edge(True, ("setup_global", "pf192"), [(390, 1, 40)], slack=0),
    # generic global-scratch solve: 368 B left, order 1056, 17 equality tiles
    "edge_generic_full": _edge(False, ("setup_global", "generic_global"), [(133, 920, 129)], slack=368, ms_pad=1056,
                               neq_pad=136),
    # one warp per QP: the fullest setup (nz = 29) and solve (nz = 32)
    "edge_tiny_full": _edge(False, ("tiny", "tiny"), [(29, 8, 17), (32, 8, 17)], ms_pad=32, neq_pad=24),
    # the L2 backward / solve_kkt on either side of L_elems <= pf_elems(ms_pad / 8): chol(Q) staged in the dead S region
    # (nz = 119 / 143) or read from global memory (nz = 120 / 144), for the 256- and the 512-thread build
    "edge_lg256_staged": _edge(False, ("setup_pf", "pf_global256"), [(119, 97, 5)], lglobal=False, ms_pad=112),
    "edge_lg256_global": _edge(False, ("setup_pf", "pf_global256"), [(120, 97, 5)], lglobal=True, ms_pad=112),
    "edge_lg512_staged": _edge(False, ("setup_pf", "pf_global512"), [(143, 121, 5)], lglobal=False, ms_pad=136),
    "edge_lg512_global": _edge(False, ("setup_pf", "pf_global512"), [(144, 121, 5)], lglobal=True, ms_pad=136),
})


# ------------------------------------------------------------------------------------------------------------------
# Which kernels a plan runs, and how close it sits to the planner's limits.

KMAX_SMEM = 232448 - 1024        # kMaxSmem (qp_kernels.cu): dynamic shared memory of one CTA per SM
SM_SMEM = 233472                 # shared memory of an SM that co-resident CTAs split, 1 KB of it reserved per CTA
PER_CTA = {2: SM_SMEM // 2 - 1024, 3: SM_SMEM // 3 - 1024}     # the planner's limits of the two- / three-per-SM CTAs


def dispatch(plan):
    """(setup kernel, solve kernel) that `plan` runs: a restatement of the setup and forward rules of choose_kernel in
    qpth_b200/csrc/qp_kernels.cu (qpb200_plan_kernels), written independently of it. The three solve entry points take
    the same branch, except that a resident product-form plan at 512 threads ("pf_res512") runs only the forward at 512
    threads and the backward / solve_kkt at 256 ("pf_res").

    setup: "tiny" k_setup<true, true>, "setup_pf192" the 192-thread k_setup_pf (qpb200_alt192_setup), "setup_pf"
    k_setup_pf<2>, "setup_fast" k_setup_fast, "setup_smem" k_setup<true>, "setup_global" k_setup<false>.
    solve: "tiny", "pf192" / "pf_two" the three- / two-per-SM product-form kernels, "pf_global512" / "pf_global256" the
    W/L-from-L2 builds, "pf_res512" / "pf_res" the resident builds, "coop", "fast" the round-1 shared-memory kernels,
    "generic_smem" / "generic_global" k_forward / k_solve_kkt with the factor in shared / global memory."""
    p = plan
    if p.tiny:
        return "tiny", "tiny"
    if p.pf and p.pf_three and p.pf3_ok and p.setup_pf_smem_bytes <= p.pf3_smem_bytes:
        setup = "setup_pf192"
    elif p.pf and p.setup_pf:
        setup = "setup_pf"
    elif p.setup_fast:
        setup = "setup_fast"
    elif p.smem_resident:
        setup = "setup_smem"
    else:
        setup = "setup_global"
    if p.pf:
        if p.pf_three and p.pf3_ok:
            solve = "pf192"
        elif p.pf_two and p.pf2_ok:
            solve = "pf_two"
        elif p.pf_global:
            solve = "pf_global512" if p.pf_threads == 512 else "pf_global256"
        else:
            solve = "pf_res512" if p.pf_threads == 512 else "pf_res"
    elif p.fast and p.coop and p.coop_ok:
        solve = "coop"
    elif p.fast:
        solve = "fast"
    else:
        solve = "generic_smem" if p.smem_resident else "generic_global"
    return setup, solve


def reg_dispatch(plan):
    """The solve kernel of the regularised forward / backward (qpb200_forward_reg, qpb200_backward_reg_duals,
    qpb200_jvp_reg), or None where they return QPB200_ERR_TOO_LARGE: the generic global-scratch kernels for a plan that
    is neither tiny, product form nor resident, else the one-QP-per-SM, 256-thread product-form kernels only."""
    p = plan
    if not p.tiny and not p.pf and not p.smem_resident:
        return "generic_global"
    if p.tiny or not p.pf or p.pf_two or p.pf_three or p.pf_threads != 256:
        return None
    return "pf_global256" if p.pf_global else "pf_res"


def slack(plan):
    """(setup, solve) bytes of shared memory left under the limit that the planner applies to each kernel: kMaxSmem for
    one CTA per SM, PER_CTA for the several-per-SM product-form kernels (and the 192-thread setup that shares their slot)."""
    setup, solve = dispatch(plan)
    if setup == "setup_pf192":
        su = PER_CTA[3] - plan.setup_pf_smem_bytes
    elif setup == "setup_pf":
        su = KMAX_SMEM - plan.setup_pf_smem_bytes
    else:
        su = KMAX_SMEM - plan.setup_smem_bytes
    if solve == "pf192":
        so = PER_CTA[3] - plan.pf3_smem_bytes
    elif solve == "pf_two":
        so = PER_CTA[2] - plan.pf2_smem_bytes
    elif solve.startswith("pf"):
        so = KMAX_SMEM - plan.pf_smem_bytes
    elif solve == "coop":
        so = 232448 // 2 - 1024 - 64 - plan.coop_smem_bytes      # coop_ok in plan_init_impl
    else:
        so = KMAX_SMEM - plan.solve_smem_bytes
    return su, so


def lglobal(plan):
    """The branch of the W/L-from-L2 product-form backward and solve_kkt (`C.lglobal` of f_make_ctx in qp_solve.cuh):
    True when chol(Q) (L_elems) does not fit the dead S region (pf_elems(ms_pad / 8), which is K_elems of such a plan), so
    the packed-L substitutions read it from global memory; False when it is staged there."""
    return plan.L_elems > plan.K_elems


def check_edge(fam, shape, plan):
    """Assert the entry's `edge`: the dispatched pair, and where given the largest solve / setup slack in bytes, ms_pad,
    neq_pad and the lglobal side."""
    e = FAMILIES[fam].get("edge")
    if e is None:
        return
    su, so = slack(plan)
    got = dict(pair=dispatch(plan), ms_pad=plan.ms_pad, neq_pad=plan.neq_pad, lglobal=lglobal(plan))
    for k in ("pair", "ms_pad", "neq_pad", "lglobal"):
        if k in e:
            assert got[k] == e[k], (fam, shape, k, got[k], e[k])
    if "slack" in e:
        assert 0 <= so <= e["slack"], (fam, shape, "solve slack", so, e["slack"])
    if "setup_slack" in e:
        assert 0 <= su <= e["setup_slack"], (fam, shape, "setup slack", su, e["setup_slack"])


def cases(*, child=None, forward=False):
    """[(family, shape)] of the families whose `child` entry equals `child` (None: all); backward / KKT tests leave
    out the forward-only families."""
    out = []
    for fam, f in FAMILIES.items():
        if child is not None and bool(f.get("child")) != child:
            continue
        if f.get("forward_only") and not forward:
            continue
        out += [(fam, s) for s in f["shapes"]]
    return out


def ids(cs):
    return ["%s-%dx%dx%d" % ((fam,) + tuple(s)) for fam, s in cs]


@contextlib.contextmanager
def family_env(fam):
    """The family's knobs in os.environ (plan_init and plan_for read them) and its MODE for QPFunction."""
    from qpth_b200 import qp as qpmod
    env = FAMILIES[fam]["env"]
    saved = {k: os.environ.get(k) for k in env}
    saved_mode = qpmod.MODE
    os.environ.update(env)
    qpmod.MODE = "throughput" if FAMILIES[fam]["two"] else "latency"
    try:
        yield
    finally:
        qpmod.MODE = saved_mode
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def family_plan(fam, shape):
    """The family's plan for `shape` (call inside family_env); asserts the flags that identify the family."""
    from qpth_b200 import _lib
    plan = _lib.plan_for(*shape, two=FAMILIES[fam]["two"])
    got = {k: getattr(plan, k) for k in FAMILIES[fam]["flags"]}
    assert got == FAMILIES[fam]["flags"], (fam, shape, got)
    check_edge(fam, shape, plan)
    return plan


# ------------------------------------------------------------------------------------------------------------------
# Inputs: seeded from the family and the shape, so the parent test and the child process build the same data.

def seed_for(fam, shape, salt):
    return (sum(map(ord, fam)) * 7919 + shape[0] * 131 + shape[1] * 17 + shape[2] + salt) % (2 ** 31)


def wellcond_qp_batch(nBatch, nz, nineq, neq=0, seed=0):
    """random_qp_batch's keys with cond(Q) <= 9 at every nz: Q = M M^T / nz + 0.5 I (M ~ N(0, 1)), G and A ~ N(0, 1/nz),
    h = G z0 + s0 with s0 ~ U(0.1, 1), b = A z0; p, z0 and dl ~ N(0, 1)."""
    rs = np.random.RandomState(seed)
    M = rs.randn(nBatch, nz, nz)
    Q = np.matmul(M, M.transpose(0, 2, 1)) / nz + 0.5 * np.eye(nz)
    G = rs.randn(nBatch, nineq, nz) / np.sqrt(nz)
    A = rs.randn(nBatch, neq, nz) / np.sqrt(nz)
    z0 = rs.randn(nBatch, nz)
    s0 = rs.uniform(0.1, 1.0, (nBatch, nineq))
    h = np.matmul(G, z0[:, :, None])[:, :, 0] + s0
    b = np.matmul(A, z0[:, :, None])[:, :, 0]
    return dict(Q=Q, p=rs.randn(nBatch, nz), G=G, h=h, A=A, b=b, dl=rs.randn(nBatch, nz))


def qp_batch(fam, B, shape, seed):
    """The family's generator (`gen`: random_qp_batch by default, "wellcond": wellcond_qp_batch) at the shape."""
    from qpth_b200.problems import random_qp_batch
    gen = wellcond_qp_batch if FAMILIES[fam].get("gen") == "wellcond" else random_qp_batch
    return gen(B, *shape, seed=seed)


def kkt_inputs(fam, shape, B, shared):
    """One batch of stand-alone KKT systems: the family's generator's matrices (one system if `shared`), d = 10^U(-8, 8),
    random right-hand sides."""
    nz, nineq, neq = shape
    pr = qp_batch(fam, 1 if shared else B, shape, seed_for(fam, shape, 1))
    rs = np.random.RandomState(seed_for(fam, shape, 2))
    return dict(Q=pr["Q"], G=pr["G"], A=pr["A"], d=10.0 ** rs.uniform(-8, 8, (B, nineq)), rx=rs.randn(B, nz),
                rs=rs.randn(B, nineq), rz=rs.randn(B, nineq), ry=rs.randn(B, neq))


def kkt_on_gpu(fam, shape, B, shared, reg, dev="cuda:0", Q=None, fill_L=None):
    """pre_factor_kkt[_reg] + solve_kkt[_reg] through the C ABI with the family's plan: batched systems (sF = 1) or one
    system for the whole batch (nsys = 1, sF = 0). Returns dx, ds, dz, dy (B rows each) and the SPD flags. Q: this Q
    in place of the generator's. fill_L: the packed L buffer is filled with this value first and returned as "L"."""
    import torch
    from qpth_b200 import _lib
    lib = _lib.load()
    nz, nineq, neq = shape
    x = kkt_inputs(fam, shape, B, shared)
    with family_env(fam):
        plan = family_plan(fam, shape)
    nsys = 1 if shared else B
    f64 = dict(dtype=torch.float64, device=dev)
    tt = lambda a: torch.tensor(np.ascontiguousarray(a), **f64)
    P = lambda t: ctypes.c_void_p(t.data_ptr()) if (t is not None and t.numel() > 0) else None
    Q, G, A = tt(x["Q"] if Q is None else Q), tt(x["G"]), (tt(x["A"]) if neq else None)
    L = torch.empty(nsys * plan.L_elems, **f64) if fill_L is None else torch.full((nsys * plan.L_elems,), fill_L, **f64)
    W = torch.empty(nsys * plan.W_elems, **f64)
    K = torch.empty(nsys * plan.K_elems, **f64)
    spd = torch.zeros(nsys, dtype=torch.int32, device=dev)
    nscr = max(nsys * plan.setup_scratch_elems, B * plan.solve_scratch_elems)
    scr = torch.empty(nscr, **f64) if nscr > 0 else None
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    sQ, sG, sA = (0, 0, 0) if shared else (nz * nz, nineq * nz, neq * nz)
    if reg > 0:
        _lib.check(lib.qpb200_pre_factor_kkt_reg(ctypes.byref(plan), nsys, P(Q), sQ, P(G), sG, P(A), sA, float(reg),
                                                 P(L), P(W), P(K), P(spd), P(scr), st))
    else:
        _lib.check(lib.qpb200_pre_factor_kkt(ctypes.byref(plan), nsys, P(Q), sQ, P(G), sG, P(A), sA,
                                             P(L), P(W), P(K), P(spd), P(scr), st))
    d, rx, rs, rz = (tt(x[k]) for k in ("d", "rx", "rs", "rz"))
    ry = tt(x["ry"]) if neq else None
    dx, ds, dz = torch.empty(B, nz, **f64), torch.empty(B, nineq, **f64), torch.empty(B, nineq, **f64)
    dy = torch.empty(B, neq, **f64) if neq else None
    sF = 0 if shared else 1
    if reg > 0:
        _lib.check(lib.qpb200_solve_kkt_reg(ctypes.byref(plan), B, P(d), P(rx), P(rs), P(rz), P(ry), float(reg),
                                            P(L), P(W), P(K), sF, P(dx), P(ds), P(dz), P(dy), P(scr), st))
    else:
        _lib.check(lib.qpb200_solve_kkt(ctypes.byref(plan), B, P(d), P(rx), P(rs), P(rz), P(ry),
                                        P(L), P(W), P(K), sF, P(dx), P(ds), P(dz), P(dy), P(scr), st))
    torch.cuda.synchronize()
    out = dict(dx=dx.cpu().numpy(), ds=ds.cpu().numpy(), dz=dz.cpu().numpy(), spd=spd.cpu().numpy())
    if neq:
        out["dy"] = dy.cpu().numpy()
    if fill_L is not None:
        out["L"] = L.cpu().numpy()
    return out


def trajectory_problem(fam, shape, B, unbatched):
    """The family's generator at the shape; `unbatched`: Q, G, A, h and b of the first QP shared by the batch (sF = 0,
    sh = 0), p batched (the classification-layer pattern, with equality constraints where the shape has them)."""
    pr = qp_batch(fam, B, shape, seed_for(fam, shape, 3))
    if unbatched:
        pr = dict(pr)
        for k in ("Q", "G", "A", "h", "b"):
            pr[k] = pr[k][0]
    return pr


def trajectory_on_gpu(fam, shape, B, unbatched, maxIter, eps, dev="cuda:0"):
    """QPFunction forward with the family's plan and qp.TRACE on: the returned iterate, iteration counts, best_resid
    and the per-iteration trace rows."""
    import torch
    from qpth_b200 import QPFunction, qp as qpmod
    pr = trajectory_problem(fam, shape, B, unbatched)
    e = torch.Tensor().to(dev).double()
    t = {k: (torch.tensor(pr[k], dtype=torch.float64, device=dev) if np.asarray(pr[k]).size else e)
         for k in ("Q", "p", "G", "h", "A", "b")}
    saved = qpmod.TRACE
    qpmod.TRACE = True
    try:
        with family_env(fam):
            family_plan(fam, shape)
            f = QPFunction(verbose=-1, eps=eps, maxIter=maxIter)
            z = f(t["Q"], t["p"], t["G"], t["h"], t["A"], t["b"])
    finally:
        qpmod.TRACE = saved
    st = f.last_solve()
    out = dict(zhat=z.cpu().numpy(), lam=st.lam.cpu().numpy(), slacks=st.slacks.cpu().numpy(),
               iters=st.iters.cpu().numpy(), best_resid=st.best_resid.cpu().numpy(), trace=st.trace.cpu().numpy())
    if st.nus is not None:
        out["nus"] = st.nus.cpu().numpy()
    return out


# ------------------------------------------------------------------------------------------------------------------
# Backward at a chosen point (tests/test_gpu_backward_families.py).

BWD_B = 4
GRAD_NAMES = ("dQ", "dp", "dG", "dh", "dA", "db")


def backward_point(shape, B, seed, fam=None):
    """The family's generator at the shape (random_qp_batch without a family) and a random primal-dual point: z, nu ~
    N(0, 1), lam, s ~ U(0.1, 10), so that d = lam / s is well conditioned and qpth's 1e-8 clamps do nothing."""
    from qpth_b200.problems import random_qp_batch
    nz, nineq, neq = shape
    pr = qp_batch(fam, B, shape, seed) if fam is not None else random_qp_batch(B, nz, nineq, neq, seed=seed)
    rs = np.random.RandomState(seed + 1)
    pr.update(z=rs.randn(B, nz), nu=rs.randn(B, neq), lam=rs.uniform(0.1, 10, (B, nineq)),
              s=rs.uniform(0.1, 10, (B, nineq)))
    return pr


def solution_backward(pr, batched, plan=None, dev="cuda:0"):
    """QPSolutionFunction + backward(dl) at the point of `pr`. batched: {name: bool} for Q, p, G, h, A, b (un-batched
    inputs take QP 0's value). plan: run pre_factor_kkt and the backward on this plan (a several-QPs-per-SM one) instead
    of the library default. Returns {gradient name: array or None}."""
    import torch
    from qpth_b200 import _lib
    from qpth_b200.solution import QPSolutionFunction
    neq = pr["A"].shape[1]
    t = {}
    for k in ("Q", "p", "G", "h", "A", "b"):
        v = pr[k] if batched[k] else pr[k][0]
        t[k] = torch.tensor(v, dtype=torch.float64, device=dev, requires_grad=True) if (neq or k not in "Ab") \
            else torch.Tensor().to(dev).double()
    sol = [torch.tensor(pr[k], dtype=torch.float64, device=dev) for k in ("z", "lam", "s")]
    nu = torch.tensor(pr["nu"], dtype=torch.float64, device=dev) if neq else torch.Tensor().to(dev).double()
    saved = _lib.plan_for
    if plan is not None:
        _lib.plan_for = lambda *a, **k: plan
    try:
        z = QPSolutionFunction()(t["Q"], t["p"], t["G"], t["h"], t["A"], t["b"], sol[0], sol[1], sol[2], nu)
        z.backward(torch.tensor(pr["dl"], dtype=torch.float64, device=dev))
    finally:
        _lib.plan_for = saved
    return {n: (t[k].grad.cpu().numpy() if t[k].grad is not None else None) for n, k in zip(GRAD_NAMES, "QpGhAb")}


def backward_on_gpu(fam, shape, B=BWD_B):
    """The family's backward at its chosen point (seed_for(..., 4)), every input batched: the gradients it returns."""
    pr = backward_point(shape, B, seed_for(fam, shape, 4), fam)
    with family_env(fam):
        plan = family_plan(fam, shape)
        got = solution_backward(pr, {k: True for k in "QpGhAb"}, plan)
    return {k: v for k, v in got.items() if v is not None}


# ------------------------------------------------------------------------------------------------------------------
# Only the lower triangle of Q is read (tests/test_gpu_q_lower_triangle.py, tests/test_q_lower_triangle_cpu.py).

# the symmetric matrix twice (the control: a difference there is nondeterminism, not the poison), then the strictly upper
# triangle set to NaN and to finite garbage
VARIANTS = ("sym", "sym_again", "nan", "garbage")
L_FILL = 0.375                   # the packed L buffer's contents before pre_factor_kkt, the same in every run


def sym_lower(Q):
    """The symmetric matrix of Q's lower triangle, tril(Q) + tril(Q, -1)^T: what the kernels solve with."""
    Q = np.asarray(Q)
    return np.tril(Q) + np.swapaxes(np.tril(Q, -1), -1, -2)


def poison(Q, how, rs):
    """Q with its strictly upper triangle replaced: NaN, or -1e3 times the transposed lower triangle plus N(0, 1) noise
    (finite and unrelated to the lower triangle: what fmin / fmax or a comparison would hide from NaN)."""
    Q = np.asarray(Q)
    upper = np.triu(np.ones(Q.shape[-2:], dtype=bool), 1)
    bad = np.full(Q.shape, np.nan) if how == "nan" else -1e3 * np.swapaxes(Q, -1, -2) + rs.randn(*Q.shape)
    return np.where(upper, bad, Q)


def q_variants(Q, seed):
    """{variant: Q} of VARIANTS, built from sym_lower(Q)."""
    Qs = sym_lower(Q)
    rs = np.random.RandomState(seed)
    return dict(sym=Qs, sym_again=Qs.copy(), nan=poison(Qs, "nan", rs), garbage=poison(Qs, "garbage", rs))


def adjoints(pr, seed):
    """Random adjoints of z, lam and nu for a problem dict with batched p, h, b."""
    rs = np.random.RandomState(seed)
    B = np.shape(pr["p"])[0]
    return {k: rs.randn(B, np.shape(pr[i])[-1] if np.size(pr[i]) else 0) for k, i in (("z", "p"), ("lam", "h"), ("nu", "b"))}


def leaf(x, dev, grad):
    """An array or tensor as a new fp64 leaf tensor on `dev` (a device tensor is copied as it is, every byte of it)."""
    import torch
    x = x if torch.is_tensor(x) else torch.tensor(np.asarray(x))
    return x.detach().to(device=dev, dtype=torch.float64).clone().requires_grad_(grad)


def qp_outputs(pr, adj, kkt_solver=None, backward=True, dev="cuda:0"):
    """QPFunction(duals=True, check_Q_spd=True) on `pr` with qp.TRACE on and deferred checks off, then a backward with
    the adjoints `adj` on z, lam and nu: z, lam, slacks, nu, iters, best_resid, the trace and every gradient."""
    import torch
    from qpth_b200 import KKTSolvers, QPFunction, qp as qpmod
    e = torch.Tensor().to(dev).double()
    t = {k: leaf(pr[k], dev, backward) for k in ("Q", "p", "G", "h", "A", "b")}
    t = {k: (v if v.numel() else e) for k, v in t.items()}
    saved = qpmod.TRACE, qpmod.LAZY_CHECKS
    qpmod.TRACE, qpmod.LAZY_CHECKS = True, False
    try:
        f = QPFunction(verbose=-1, check_Q_spd=True, kkt_solver=kkt_solver or KKTSolvers.LU_PARTIAL, duals=True)
        z, lam, nu = f(*(t[k] for k in ("Q", "p", "G", "h", "A", "b")))
        if backward:
            outs = [(z, "z"), (lam, "lam")] + ([(nu, "nu")] if nu.numel() else [])
            sum((o * torch.tensor(adj[k], dtype=torch.float64, device=dev)).sum() for o, k in outs).backward()
    finally:
        qpmod.TRACE, qpmod.LAZY_CHECKS = saved
    st = f.last_solve()
    out = dict(z=z.detach().cpu().numpy(), lam=lam.detach().cpu().numpy(), nu=nu.detach().cpu().numpy(),
               slacks=st.slacks.cpu().numpy(), iters=st.iters.cpu().numpy(), best_resid=st.best_resid.cpu().numpy(),
               trace=st.trace.cpu().numpy())
    out.update({"d" + k: v.grad.cpu().numpy() for k, v in t.items() if v.grad is not None})
    return out


def lower_triangle_runs(fam, shape, B=2):
    """Every VARIANT of Q on the family's plan: QPFunction's forward and backward with duals, with Q, G, A, h, b batched
    (nsys = B) and un-batched (nsys = 1), and pre_factor_kkt + solve_kkt at reg 0 and 1e-7 with the packed L buffer.
    Keys "<run>__<variant>__<output>"."""
    fwd_only = FAMILIES[fam].get("forward_only", False)
    out = {}
    for unbatched in (False, True):
        pr = trajectory_problem(fam, shape, B, unbatched)
        adj = adjoints(pr, seed_for(fam, shape, 5))
        with family_env(fam):
            family_plan(fam, shape)
            for v, Q in q_variants(pr["Q"], seed_for(fam, shape, 6)).items():
                r = qp_outputs(dict(pr, Q=Q), adj, backward=not fwd_only)
                out.update({"%s__%s__%s" % ("qp_unbatched" if unbatched else "qp_batched", v, k): a for k, a in r.items()})
    if not fwd_only:
        x = kkt_inputs(fam, shape, B, False)
        for reg in (0.0, 1e-7):
            for v, Q in q_variants(x["Q"], seed_for(fam, shape, 7)).items():
                r = kkt_on_gpu(fam, shape, B, False, reg, Q=Q, fill_L=L_FILL)
                out.update({"%s__%s__%s" % ("kkt_reg" if reg else "kkt", v, k): a for k, a in r.items()})
    return out


def compare_variants(rec):
    """Group `rec` ("<run>__<variant>__<output>") by run, and assert every variant bit-identical to "sym", output by
    output (NaN only where the trace has rows past a QP's last iteration). Returns the runs compared."""
    runs = sorted({k.split("__")[0] for k in rec})
    for run in runs:
        outs = sorted({k.split("__")[2] for k in rec if k.startswith(run + "__")})
        for o in outs:
            ref = rec["%s__sym__%s" % (run, o)]
            if o != "trace":
                assert np.isfinite(ref).all(), (run, o)
            for v in VARIANTS[1:]:
                got = rec["%s__%s__%s" % (run, v, o)]
                assert got.shape == ref.shape and np.array_equal(got, ref, equal_nan=(o == "trace")), \
                    (run, v, o, np.nanmax(np.abs(got - ref)) if got.shape == ref.shape else got.shape)
    return runs


def eq_outputs(pr, adj, tan, kkt_solver, dev="cuda:0"):
    """The equality-only path (Q, p, A, b; no inequality rows) of QPFunction(duals=True, check_Q_spd=True): z*, nu, the
    gradients of <adj_z, z> + <adj_nu, nu>, and the JVP (dz, dnu) along the tangents `tan` of Q, p, A and b."""
    import torch
    import torch.autograd.forward_ad as fwAD
    from qpth_b200 import QPFunction
    t = {k: leaf(v, dev, True) for k, v in pr.items() if k in ("Q", "p", "A", "b")}
    e = torch.Tensor().to(dev).double()
    f = QPFunction(verbose=-1, check_Q_spd=True, kkt_solver=kkt_solver, duals=True)
    z, lam, nu = f(t["Q"], t["p"], e, e, t["A"], t["b"])
    assert lam.shape == (z.shape[0], 0)
    T = lambda a: torch.tensor(a, dtype=torch.float64, device=dev)
    ((z * T(adj["z"])).sum() + (nu * T(adj["nu"])).sum()).backward()
    out = dict(z=z.detach().cpu().numpy(), nu=nu.detach().cpu().numpy(), **{"d" + k: v.grad.cpu().numpy() for k, v in t.items()})
    with fwAD.dual_level():
        zd, _, nud = f(*(fwAD.make_dual(t[k].detach(), T(tan[k])) if k in t else e for k in ("Q", "p", "G", "h", "A", "b")))
        out["jvp_z"] = fwAD.unpack_dual(zd).tangent.cpu().numpy()
        out["jvp_nu"] = fwAD.unpack_dual(nud).tangent.cpu().numpy()
    return out
