"""Cost of QPFunction(kkt_solver=KKTSolvers.IR_UNOPT) on the generic global-scratch kernels (orders the product-form
kernels do not take): fwd+bwd per step (CUDA events) and mean Newton iterations, for
  * the LP of oracle/psd_large_cases.lp280 (nz = 100, both bounds, 60 random rows, neq = 10: order 280) at B = 128 and
    1024, IR_UNOPT with IR_STEPS = 0 and 1 against the default mode on the Q = 1e-6 I workaround, alternated;
  * the order-664 LP of psd_large_cases.lp664 at B = 64;
  * the 9x9 sudoku LP relaxation (Q = 0, z >= 0, the 249 independent sudoku rows: order 992) at B = 1 and 64.
Each line also gives the largest relative difference of z* from the IR_STEPS = 1 run of the same seeded batch.
Prints one JSON line per workload, with the device name and power limit. Writes nothing."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import psd_large_cases as lc  # noqa: E402
from qpth_b200 import KKTSolvers, QPFunction, kkt  # noqa: E402


def _dev(a):
    return torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda", requires_grad=True)


def batch(cases, qeps=0.0):
    ins = [np.stack([c[k] for c in cases]) for k in range(6)]
    ins[0] = ins[0] + qeps * np.eye(ins[0].shape[-1])
    return [_dev(a) for a in ins]


def time_step(ins, steps, warmup=1, **opts):
    f = QPFunction(verbose=-1, check_Q_spd=False, **opts)
    dl = torch.randn(ins[1].shape[0], ins[0].shape[-1], dtype=torch.float64, device="cuda",
                     generator=torch.Generator(device="cuda").manual_seed(0))

    def one():
        for t in ins:
            t.grad = None
        z = f(*ins)
        z.backward(dl)
        return z
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        z = one()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, float(f.last_solve().iters.double().mean()), z.detach()


def run(name, cases, steps, rounds, res, default=True):
    """IR_UNOPT with IR_STEPS = 0 and 1 and (default) the default mode on Q + 1e-6 I, alternated for `rounds` rounds."""
    reg, shifted = batch(cases), batch(cases, 1e-6) if default else None
    for _ in range(rounds):
        out = {}
        for s in (1, 0):
            kkt.IR_STEPS = s
            out[s] = time_step(reg, steps, kkt_solver=KKTSolvers.IR_UNOPT)
        if default:
            out["d"] = time_step(shifted, steps)
        ref = out[1][2]
        for k, label in ((0, "IR_UNOPT steps=0"), (1, "IR_UNOPT steps=1"), ("d", "default, Q + 1e-6 I")):
            if k not in out:
                continue
            ms, it, z = out[k]
            dz = float((z - ref).abs().max() / ref.abs().max().clamp(min=1e-8))
            res.append(dict(workload="%s %s" % (name, label), ms_per_step=round(ms, 3), mean_iters=round(it, 2),
                            rel_dz_vs_steps1=float("%.3g" % dz)))
    kkt.IR_STEPS = 1


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = []
    run("LP order 280 B=128", [lc.lp280(s) for s in range(128)], 5, 2, res)
    run("LP order 280 B=1024", [lc.lp280(s) for s in range(1024)], 3, 2, res)
    run("LP order 664 B=64", [lc.lp664(s) for s in range(64)], 3, 1, res)
    run("sudoku9 LP order 992 B=1", lc.sudoku9_lp(0, B=1), 3, 1, res, default=False)
    run("sudoku9 LP order 992 B=64", lc.sudoku9_lp(0, B=64), 2, 1, res, default=False)
    for r in res:
        r["gpu"] = gpu
        print(json.dumps(r))


if __name__ == "__main__":
    main()
