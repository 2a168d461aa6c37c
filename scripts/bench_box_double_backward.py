"""The cost of second order through BoxQPFunction: forward + create_graph backward + one Hessian-vector product in p and
q (Q), against forward + backward alone and against a central-difference HVP (two more forward + backward). One JSON
line per workload on stdout.

    python scripts/bench_box_double_backward.py [--steps 20] [--pairs 5]

Workloads (loss 1/2 ||z||^2 + <w, z>; A, b and the bounds shared by the batch, as a learned layer has them):
  sudoku4        the 4x4 OptNet sudoku layer: B = 1024, nz = 64, neq = 40, lb only, q batched (one CTA per QP)
  sudoku9        the 9x9 sudoku layer: B = 64, nz = 729, neq = 249, lb only (the distributed-M cluster kernels)
  proj_cl2       a projection on a two-CTA cluster: B = 64, nz = 1000, neq = 8, both sides
  portfolio      the dense-Q portfolio: B = 1024, nz = 100, neq = 1, both sides, Q batched
  portfolio_Qsh  the same with Q shared (its second-order gradient is k_ggrad_sum's batch sum)
The three arms solve the same problems and alternate in one process (`pairs` rounds of `steps`-step windows, CUDA
events, median window). The new kernels are timed in a separate torch.profiler run (CUDA activities); their algorithmic
bytes come from the shape formulas below and are reported as a share of the H100 SXM's 3.35 TB/s. Each line carries the
GPU name and power limit. Nothing is written to the tree.
"""
import argparse
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402

from scripts.bench_duals import gpu_info   # noqa: E402

PEAK = 3.35e12
# name: (B, nz, neq, sides, dense_Q, q shared)
SHAPES = {"sudoku4": (1024, 64, 40, "lb", False, False), "sudoku9": (64, 729, 249, "lb", False, False),
          "proj_cl2": (64, 1000, 8, "both", False, False), "portfolio": (1024, 100, 1, "both", True, False),
          "portfolio_Qsh": (1024, 100, 1, "both", True, True)}
KERNELS = ("k_box_ggrad_rhs", "k_boxq_ggrad_rhs", "k_box_ggrad_out", "k_box_ggrad_sum_vec", "k_ggrad_sum")


def kernel_bytes(B, n, e, m, dense_Q, q_shared):
    """Algorithmic bytes per launch for the HVP in q (Q) and p (wq, wp the only cotangents, dq and dp the only
    gradients): the rhs kernel reads wq (n, or n^2 for a dense Q; once in all when shared), vx, vlam, ulam, lam, s and
    vnu and writes cz, clam, cnu, c_s; k_box_ggrad_out reads z, vx, ux, wx and writes dp and, q batched, dq (n or n^2);
    a shared q is summed by k_box_ggrad_sum_vec (diagonal) or k_ggrad_sum (dense), reading z, vx, ux, wx of every QP."""
    wq = n * n if dense_Q else n
    mats = wq if q_shared else B * wq
    vec = B * ((n + 4 * m + e) + (n + 2 * m + e))
    res = {"k_boxq_ggrad_rhs" if dense_Q else "k_box_ggrad_rhs": 8 * (mats + vec),
           "k_box_ggrad_out": 8 * B * (4 * n + n + (0 if q_shared else wq))}
    if q_shared:
        res["k_ggrad_sum" if dense_Q else "k_box_ggrad_sum_vec"] = 8 * (4 * B * n + wq)
    return res


def problem(B, n, e, sides, dense_Q, q_shared, dev):
    rs = np.random.RandomState(5)
    f64 = dict(dtype=torch.float64, device=dev)
    if dense_Q:
        F = rs.randn(1 if q_shared else B, n, n)
        q = F @ F.transpose(0, 2, 1) / n + 0.1 * np.eye(n)
    else:
        q = rs.uniform(0.5, 2.0, (1 if q_shared else B, n))
    A = rs.randn(e, n) / np.sqrt(n)
    z0 = rs.uniform(0.1, 0.4, n)
    ins = dict(q=torch.tensor(q[0] if q_shared else q, **f64), p=torch.tensor(rs.randn(B, n), **f64),
               A=torch.tensor(A, **f64), b=torch.tensor(A @ z0, **f64),
               lb=torch.zeros(n, **f64) if sides != "ub" else None,
               ub=torch.full((n,), 0.5, **f64) if sides != "lb" else None)
    w = torch.tensor(rs.randn(B, n), **f64)
    vp = torch.tensor(rs.randn(B, n), **f64)
    vq = torch.tensor(rs.randn(*ins["q"].shape), **f64)
    if dense_Q:
        vq = 0.5 * (vq + vq.transpose(-1, -2))
    return ins, w, vp, vq


def arms(ins, w, vp, vq, dense_Q):
    from qpth_b200 import BoxQPFunction
    f = BoxQPFunction(verbose=-1, check_Q_spd=False, dense_Q=dense_Q)

    def fwd_bwd(dq=None, dp=None, create=False):
        x = dict(ins)
        if dq is not None:
            x["q"], x["p"] = x["q"] + dq, x["p"] + dp
        q, p = x["q"].clone().requires_grad_(True), x["p"].clone().requires_grad_(True)
        z = f(q, p, x["A"], x["b"], x["lb"], x["ub"])
        loss = 0.5 * (z ** 2).sum() + (w * z).sum()
        return (q, p) + tuple(torch.autograd.grad(loss, (q, p), create_graph=create))

    def base():
        fwd_bwd()

    def hvp():
        q, p, gq, gp = fwd_bwd(create=True)
        torch.autograd.grad((gq * vq).sum() + (gp * vp).sum(), (q, p))

    def central(h=1e-5):
        fwd_bwd()
        a = fwd_bwd(h * vq, h * vp)
        b = fwd_bwd(-h * vq, -h * vp)
        return [(x - y) / (2 * h) for x, y in zip(a[2:], b[2:])]
    return dict(fwd_bwd=base, fwd_bwd_hvp=hvp, central_difference_hvp=central)


def time_arms(fns, steps, pairs):
    def window(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / steps
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(pairs):
        for k, fn in fns.items():
            res[k].append(window(fn))
    return res


def kernel_times(fns, reps=10):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fns["fwd_bwd_hvp"]()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if re.search(r"\b%s(\(|<|E|$)" % k, ev.key):
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total")
                out[k] = t / max(ev.count, 1) / 1e3       # ms per launch
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_box_double_backward: needs a CUDA device")
    dev = "cuda:0"
    name, power = gpu_info()
    for wl, (B, n, e, sides, dense_Q, q_shared) in SHAPES.items():
        if args.only and wl not in args.only.split(","):
            continue
        ins, w, vp, vq = problem(B, n, e, sides, dense_Q, q_shared, dev)
        fns = arms(ins, w, vp, vq, dense_Q)
        t = time_arms(fns, args.steps, args.pairs)
        med = {k: float(np.median(v)) for k, v in t.items()}
        kt = kernel_times(fns)
        m = n * ((sides != "ub") + (sides != "lb"))
        kb = kernel_bytes(B, n, e, m, dense_Q, q_shared)
        kern = {k: dict(ms=kt.get(k), bytes=kb[k], share_of_3_35_TBps=(kb[k] / (kt[k] * 1e-3) / PEAK if kt.get(k) else None))
                for k in kb}
        print(json.dumps(dict(workload=wl, B=B, nz=n, neq=e, sides=sides, dense_Q=dense_Q, q_shared=q_shared, gpu=name,
                              power_limit=power, steps=args.steps, pairs=args.pairs, ms=med,
                              hvp_over_fwd_bwd=med["fwd_bwd_hvp"] / med["fwd_bwd"],
                              central_over_fwd_bwd=med["central_difference_hvp"] / med["fwd_bwd"],
                              windows=t, kernels=kern)), flush=True)


if __name__ == "__main__":
    main()
