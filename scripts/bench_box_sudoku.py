"""BoxQPFunction with neq_pad > 128 (the distributed-M cluster kernels): one JSON line on stdout.

    python scripts/bench_box_sudoku.py [--steps 3] [--pairs 3] [--quick]

Cases, fwd+bwd per step (CUDA events, median of `pairs` windows of `steps` steps), each with QPs/s and the mean Newton
iteration count:
- the 9x9 OptNet sudoku layer (nz = 729, neq = 249, z >= 0, q = 0.1, p = -puzzle, A and b shared) at B = 1, 64 and
  256, against QPFunction on the dense equivalent (order 992), with the largest per-QP relative difference of z* and of
  every gradient;
- the same layer with an upper bound z <= 1 at B = 256 (the dense kernels reject it);
- random shapes on both sides of the dense order past which the plan picks these kernels (kDmDenseOrder in
  csrc/qp_box.cu), B = 256, timed on both paths; below it the kernels are forced with QPB200_BOX_CLUSTER.
The line carries the GPU name and power limit. Nothing is written to the tree. --quick: B = 64 for the threshold cases.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402

from scripts.bench_box import gpu_info                  # noqa: E402
from scripts.bench_box_wide import _rel, _timed         # noqa: E402

KEYS = ("q", "p", "A", "b", "lb", "ub")


def _sudoku_inputs(dev, B, both):
    from oracle.box_sudoku_cases import puzzles, sudoku_matrix
    A = sudoku_matrix(3)
    n = A.shape[1]
    P, _ = puzzles(100 + B, B)
    f64 = dict(dtype=torch.float64, device=dev)
    ins = dict(q=torch.full((n,), 0.1, **f64), p=torch.tensor(-P, **f64), A=torch.tensor(A, **f64),
               b=torch.ones(A.shape[0], **f64), lb=torch.zeros(n, **f64), ub=torch.ones(n, **f64) if both else None)
    return ins, torch.tensor(np.random.RandomState(B).randn(B, n), **f64)


def _random_inputs(dev, B, nz, neq, seed):
    rs = np.random.RandomState(seed)
    f64 = dict(dtype=torch.float64, device=dev)
    A = rs.randn(neq, nz)
    z0 = 0.05 + rs.rand(nz)
    ins = dict(q=torch.tensor(0.1 + rs.rand(nz), **f64), p=torch.tensor(2.0 * rs.randn(B, nz), **f64),
               A=torch.tensor(A, **f64), b=torch.tensor(A @ z0, **f64), lb=torch.tensor(-rs.rand(nz), **f64), ub=None)
    return ins, torch.tensor(rs.randn(B, nz), **f64)


def _force(nz, neq, has_ub):
    """the smallest cluster size the knob can force on this shape"""
    from qpth_b200 import _lib
    for C in (2, 4, 8):
        os.environ["QPB200_BOX_CLUSTER"] = str(C)
        if _lib.box_plan_for(nz, neq, True, has_ub).cl_ctas == C:
            return C
    del os.environ["QPB200_BOX_CLUSTER"]
    raise RuntimeError("no cluster holds (%d, %d)" % (nz, neq))


def run_case(name, ins, dl, steps, pairs, dense, forced=False):
    from qpth_b200 import BoxQPFunction, QPFunction, _lib
    from qpth_b200.box import dense_equivalent
    B, nz = dl.shape
    neq = ins["A"].shape[0]
    has_ub = ins["ub"] is not None
    for v in ins.values():
        if v is not None:
            v.requires_grad_(True)
    if forced:
        _force(nz, neq, has_ub)
    else:
        os.environ.pop("QPB200_BOX_CLUSTER", None)
    plan = _lib.box_plan_for(nz, neq, True, has_ub)
    dp = _lib.Plan()
    _lib.load().qpb200_plan_init(nz, plan.nineq, neq, __import__("ctypes").byref(dp))
    fb = BoxQPFunction(verbose=-1, check_Q_spd=False)

    def box_once():
        for v in ins.values():
            if v is not None:
                v.grad = None
        z = fb(*(ins[k] for k in KEYS))
        z.backward(dl)
        return z
    mb, wb = _timed(box_once, steps, pairs)
    z = box_once().detach()
    out = {"case": name, "shape": {"B": B, "nz": nz, "neq": neq, "bounds": "both" if has_ub else "lb",
                                   "dense_order": dp.ms_pad},
           "plan": {"cl_ctas": plan.cl_ctas, "cl_slice": plan.cl_slice, "cl_smem_bytes": plan.cl_smem_bytes,
                    "forced": forced},
           "box": {"ms_per_step": mb, "QPs_per_s": B / (mb * 1e-3), "windows_ms": wb,
                   "mean_newton_iters": float(fb.last_solve().iters.double().mean())}}
    os.environ.pop("QPB200_BOX_CLUSTER", None)
    if not dense:
        out["dense"] = "not run: the dense kernels reject this shape"
        return out
    Q, G, h = dense_equivalent(ins["q"].detach(), ins["lb"].detach(), None if not has_ub else ins["ub"].detach())
    dn = dict(Q=Q, p=ins["p"].detach().clone(), G=G, h=h, A=ins["A"].detach().clone(), b=ins["b"].detach().clone())
    for t in dn.values():
        t.requires_grad_(True)
    fd = QPFunction(verbose=-1, check_Q_spd=False)

    def dense_once():
        for v in dn.values():
            v.grad = None
        zz = fd(dn["Q"], dn["p"], dn["G"], dn["h"], dn["A"], dn["b"])
        zz.backward(dl)
        return zz
    md, wd = _timed(dense_once, steps, pairs)
    zd = dense_once().detach()
    if forced:
        _force(nz, neq, has_ub)
    box_once()
    os.environ.pop("QPB200_BOX_CLUSTER", None)
    out["dense"] = {"ms_per_step": md, "QPs_per_s": B / (md * 1e-3), "windows_ms": wd,
                    "mean_newton_iters": float(fd.last_solve().iters.double().mean())}
    out["speedup_vs_dense"] = md / mb
    out["max_rel_diff_box_vs_dense"] = {
        "z": _rel(z, zd, 0.0), "dq": _rel(ins["q"].grad, torch.diagonal(dn["Q"].grad)),
        "dp": _rel(ins["p"].grad, dn["p"].grad), "dA": _rel(ins["A"].grad, dn["A"].grad),
        "db": _rel(ins["b"].grad, dn["b"].grad), "dlb": _rel(ins["lb"].grad, -dn["h"].grad[:nz])}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_box_sudoku: no CUDA device (a timing needs the GPU)")
    dev = torch.device("cuda:0")
    s, p = args.steps, args.pairs
    cases = []
    for B in (1, 64, 256):
        cases.append(run_case("sudoku9", *_sudoku_inputs(dev, B, False), s, p, dense=True))
    cases.append(run_case("sudoku9 0 <= z <= 1", *_sudoku_inputs(dev, 256, True), s, p, dense=False))
    Bt = 64 if args.quick else 256
    for nz, neq in ((200, 180), (300, 200), (400, 200), (600, 249)):
        from qpth_b200 import _lib
        os.environ.pop("QPB200_BOX_CLUSTER", None)
        chosen = _lib.box_plan_for(nz, neq, True, False).cl_ctas != 0
        cases.append(run_case("threshold", *_random_inputs(dev, Bt, nz, neq, nz + neq), s, p, dense=True,
                              forced=not chosen))
    line = {"cases": cases,
            "api": "BoxQPFunction(verbose=-1, check_Q_spd=False), fwd+bwd per step; q, A, b, lb, ub shared, p batched",
            "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
