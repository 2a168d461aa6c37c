"""One table of the kernel families the planner can pick, and the GPU runs the per-family tests share.

Each family: development knobs (env), the `two=` argument of `_lib.plan_for` (throughput mode), the plan flags that
identify it, and shapes (nz, nineq, neq). Every test asserts the flags before it solves, so a planner change cannot
move a case silently to another family. Across a family's shapes there is an odd nz, an nineq and (where the family
takes equality constraints) an neq that are not multiples of 8.

`child`: families with dispatch branches that had never run before these tests (the 192- and 512-thread solve_kkt
builds, the regularised solve on a 512-thread plan, the resident 512-thread forward). Their GPU work runs in the child
process of tests/gpu_child.py, so that a fault there fails only their own tests.
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
    return plan


# ------------------------------------------------------------------------------------------------------------------
# Inputs: seeded from the family and the shape, so the parent test and the child process build the same data.

def seed_for(fam, shape, salt):
    return (sum(map(ord, fam)) * 7919 + shape[0] * 131 + shape[1] * 17 + shape[2] + salt) % (2 ** 31)


def kkt_inputs(fam, shape, B, shared):
    """One batch of stand-alone KKT systems: random_qp_batch matrices (one system if `shared`), d = 10^U(-8, 8), random
    right-hand sides."""
    from qpth_b200.problems import random_qp_batch
    nz, nineq, neq = shape
    pr = random_qp_batch(1 if shared else B, nz, nineq, neq, seed=seed_for(fam, shape, 1))
    rs = np.random.RandomState(seed_for(fam, shape, 2))
    return dict(Q=pr["Q"], G=pr["G"], A=pr["A"], d=10.0 ** rs.uniform(-8, 8, (B, nineq)), rx=rs.randn(B, nz),
                rs=rs.randn(B, nineq), rz=rs.randn(B, nineq), ry=rs.randn(B, neq))


def kkt_on_gpu(fam, shape, B, shared, reg, dev="cuda:0"):
    """pre_factor_kkt[_reg] + solve_kkt[_reg] through the C ABI with the family's plan: batched systems (sF = 1) or one
    system for the whole batch (nsys = 1, sF = 0). Returns dx, ds, dz, dy (B rows each) and the SPD flags."""
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
    Q, G, A = tt(x["Q"]), tt(x["G"]), (tt(x["A"]) if neq else None)
    L = torch.empty(nsys * plan.L_elems, **f64)
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
    return out


def trajectory_problem(fam, shape, B, unbatched):
    """random_qp_batch at the shape; `unbatched`: Q, G, A, h and b of the first QP shared by the batch (sF = 0, sh = 0),
    p batched (the classification-layer pattern, with equality constraints where the shape has them)."""
    from qpth_b200.problems import random_qp_batch
    pr = random_qp_batch(B, *shape, seed=seed_for(fam, shape, 3))
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
