"""The cost of the dual outputs: fwd+bwd with duals=False (loss on z) against duals=True (loss on z, lam and nu), one JSON
line per workload on stdout.

    python scripts/bench_duals.py [--steps 50] [--pairs 7]

Workloads: C2 (QPFunction, B = 128, nz = nineq = 100, no equality rows), the box sudoku layer (BoxQPFunction, nz = 64,
neq = 40, lb only, B = 1024) and a cluster box shape (BoxQPFunction, nz = 1000, neq = 8, both sides, B = 128: two CTAs
per QP). The two variants solve the same problems and alternate in one process (`pairs` pairs of `steps`-step windows,
CUDA events, median window), so both see the same clocks and neighbours. check_Q_spd=False and verbose=-1: no call reads
a flag back to the host, so the device and not the host's scheduling sets the window. The duals=True backward reads one
extra (B, nineq + neq) adjoint. Each line carries the GPU name and power limit. Nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
    except Exception:     # noqa: BLE001 - the name from torch, the power limit unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def workloads(dev):
    from qpth_b200 import BoxQPFunction, QPFunction
    from qpth_b200.problems import random_qp_batch
    f64 = dict(dtype=torch.float64, device=dev)
    pr = random_qp_batch(128, 100, 100, 0, seed=2)
    c2 = {k: torch.tensor(pr[k], **f64) for k in ("Q", "p", "G", "h")}
    e = torch.Tensor().to(dev).double()

    def qp(duals):
        f = QPFunction(verbose=-1, check_Q_spd=False, duals=duals)
        return lambda x: f(x["Q"], x["p"], x["G"], x["h"], e, e)

    rs = np.random.RandomState(31)
    A_ = rs.randn(40, 64)
    sud = {"q": torch.full((64,), 0.1, **f64), "p": torch.tensor(-rs.rand(1024, 64), **f64),
           "A": torch.tensor(A_, **f64), "b": torch.tensor(A_ @ (rs.rand(64) + 0.1), **f64), "lb": torch.zeros(64, **f64)}
    A2 = rs.randn(8, 1000)
    z0 = 0.05 + 0.4 * rs.rand(1000)
    clu = {"q": torch.tensor(0.1 + rs.rand(128, 1000), **f64), "p": torch.tensor(2 * rs.randn(128, 1000), **f64),
           "A": torch.tensor(A2, **f64), "b": torch.tensor(A2 @ z0, **f64), "lb": torch.tensor(-rs.rand(128, 1000), **f64),
           "ub": torch.tensor(rs.rand(128, 1000) + 0.5, **f64)}

    def box(duals):
        f = BoxQPFunction(verbose=-1, check_Q_spd=False, duals=duals)
        return lambda x: f(x["q"], x["p"], x["A"], x["b"], x["lb"], x.get("ub"))

    return [("c2_128x100x100", c2, qp), ("box_sudoku_1024x64x40_lb", sud, box), ("box_cluster_128x1000x8_both", clu, box)]


def measure(name, ins, make, steps, pairs, dev):
    from qpth_b200 import _lib
    for t in ins.values():
        t.requires_grad_(True)
    f0, f1 = make(False), make(True)
    z = f0(ins)
    _, lam, nu = f1(ins)
    rs = np.random.RandomState(5)
    gz, gl, gn = (torch.tensor(rs.randn(*t.shape), dtype=torch.float64, device=dev) for t in (z, lam, nu))

    def once(duals):
        for t in ins.values():
            t.grad = None
        if duals:
            z, lam, nu = f1(ins)
            ((z * gz).sum() + (lam * gl).sum() + (nu * gn).sum()).backward()
        else:
            (f0(ins) * gz).sum().backward()

    def window(duals):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            once(duals)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    for d in (False, True):                     # warm-up: modules, plans, allocator
        for _ in range(3):
            once(d)
    torch.cuda.synchronize()
    t0, t1 = [], []
    for _ in range(pairs):
        t0.append(window(False))
        t1.append(window(True))
    plan = None
    if "q" in ins:
        p = _lib.box_plan_for(ins["q"].shape[-1], ins["A"].shape[-2], True, "ub" in ins)
        plan = dict(ok=p.ok, cl_ctas=p.cl_ctas)
    return dict(workload=name, ms_duals_false=float(np.median(t0)), ms_duals_true=float(np.median(t1)),
                ratio=float(np.median(t1) / np.median(t0)), windows_false=t0, windows_true=t1, box_plan=plan)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--pairs", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_duals: no CUDA device (there is no CPU fallback)")
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    for wl, ins, make in workloads(dev):
        rec = measure(wl, ins, make, a.steps, a.pairs, dev)
        rec.update(gpu=name, power_limit=power, steps=a.steps, pairs=a.pairs)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
