"""The cost of second order through QPFunction: forward + create_graph backward + one Hessian-vector product in p and Q,
against forward + backward alone and against a central-difference HVP (two more forward + backward). One JSON line per
workload on stdout.

    python scripts/bench_double_backward.py [--steps 20] [--pairs 5]

Workloads: C2 (B = 128, nz = nineq = 100, no equality rows) and C3 (B = 1024, nz = nineq = 50, neq = 10), every input
batched, and C2 with Q and G shared by the batch (C2_shared_QG: the second-order gradient of Q is the batch sum of
k_ggrad_sum), loss 1/2 ||z||^2 + <w, z>. The three arms solve the same problems and alternate in one process (`pairs` rounds
of `steps`-step windows, CUDA events, median window). The new kernels are timed in a separate torch.profiler run
(CUDA activities); each one's algorithmic bytes come from the shape formulas below and are reported as a share of the
H100 SXM's 3.35 TB/s. Each line carries the GPU name and power limit. Nothing is written to the tree.
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
SHAPES = {"C2": (128, 100, 100, 0, ()), "C3": (1024, 50, 50, 10, ()), "C2_shared_QG": (128, 100, 100, 0, ("Q", "G"))}
KERNELS = ("k_ggrad_rhs", "k_ggrad_out", "k_ggrad_sum")


def kernel_bytes(B, n, m, e, shared):
    """Algorithmic bytes per launch for the HVP in Q and p (wQ, wp the only cotangents, dQ and dp the only gradients):
    k_ggrad_rhs reads wQ (n^2) and G (m n) once per QP (once in all when shared), vx, vlam (twice), vnu, ulam, lam, s,
    and writes cz, clam, cnu, c_s; k_ggrad_out reads z, vx, ux, wx and writes dQ (n^2, when Q is batched) and dp (n);
    k_ggrad_sum (Q shared) reads wx, z, ux, vx of every QP and writes dQ once."""
    mats = (0 if "Q" in shared else B) * n * n + (0 if "G" in shared else B) * m * n
    mats += (n * n if "Q" in shared else 0) + (m * n if "G" in shared else 0)
    rhs = 8 * (mats + B * ((n + 5 * m + e) + (n + 2 * m + e)))
    out = B * 8 * (4 * n + (0 if "Q" in shared else n * n) + n)
    res = {"k_ggrad_rhs": rhs, "k_ggrad_out": out}
    if "Q" in shared:
        res["k_ggrad_sum"] = 8 * (4 * B * n + n * n)
    return res


def problem(B, n, m, e, shared, dev):
    from qpth_b200.problems import random_qp_batch
    pr = random_qp_batch(B, n, m, e, seed=5)
    f64 = dict(dtype=torch.float64, device=dev)
    ins = {k: torch.tensor(pr[k], **f64) for k in ("Q", "p", "G", "h", "A", "b")}
    if e == 0:
        ins["A"], ins["b"] = torch.Tensor().to(dev).double(), torch.Tensor().to(dev).double()
    rs = np.random.RandomState(7)
    w = torch.tensor(rs.randn(B, n), **f64)
    vp = torch.tensor(rs.randn(B, n), **f64)
    vQ = torch.tensor(rs.randn(B, n, n), **f64)
    for k in shared:
        ins[k] = ins[k][0].contiguous()
    if "Q" in shared:
        vQ = vQ[0]
    return ins, w, vp, 0.5 * (vQ + vQ.transpose(-1, -2))


def arms(ins, w, vp, vQ):
    from qpth_b200 import QPFunction
    f = QPFunction(verbose=-1, check_Q_spd=False)
    names = ("Q", "p", "G", "h", "A", "b")

    def fwd_bwd(dQ=None, dp=None, create=False):
        x = dict(ins)
        if dQ is not None:
            x["Q"], x["p"] = x["Q"] + dQ, x["p"] + dp
        Q, p = x["Q"].clone().requires_grad_(True), x["p"].clone().requires_grad_(True)
        z = f(Q, p, *(x[k] for k in names[2:]))
        loss = 0.5 * (z ** 2).sum() + (w * z).sum()
        return (Q, p) + tuple(torch.autograd.grad(loss, (Q, p), create_graph=create))

    def base():
        fwd_bwd()

    def hvp():
        Q, p, gQ, gp = fwd_bwd(create=True)
        torch.autograd.grad((gQ * vQ).sum() + (gp * vp).sum(), (Q, p))

    def central(h=1e-5):
        fwd_bwd()
        a = fwd_bwd(h * vQ, h * vp)
        b = fwd_bwd(-h * vQ, -h * vp)
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
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_double_backward: needs a CUDA device")
    dev = "cuda:0"
    name, power = gpu_info()
    for wl, (B, n, m, e, shared) in SHAPES.items():
        ins, w, vp, vQ = problem(B, n, m, e, shared, dev)
        fns = arms(ins, w, vp, vQ)
        t = time_arms(fns, args.steps, args.pairs)
        med = {k: float(np.median(v)) for k, v in t.items()}
        kt = kernel_times(fns)
        kb = kernel_bytes(B, n, m, e, shared)
        kern = {k: dict(ms=kt.get(k), bytes=kb[k], share_of_3_35_TBps=(kb[k] / (kt[k] * 1e-3) / PEAK if kt.get(k) else None))
                for k in kb}
        print(json.dumps(dict(workload=wl, B=B, nz=n, nineq=m, neq=e, shared=list(shared), gpu=name, power_limit=power,
                              steps=args.steps, pairs=args.pairs,
                              ms=med, hvp_over_fwd_bwd=med["fwd_bwd_hvp"] / med["fwd_bwd"],
                              central_over_fwd_bwd=med["central_difference_hvp"] / med["fwd_bwd"],
                              windows=t, kernels=kern)), flush=True)


if __name__ == "__main__":
    main()
