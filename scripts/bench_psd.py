"""Cost of QPFunction(kkt_solver=KKTSolvers.IR_UNOPT), the regularised mode: fwd+bwd per step (CUDA events) and mean
Newton iterations, for
  * C2 (nz = nineq = 100, neq = 0, B = 128) in IR_UNOPT with IR_STEPS = 0 and 1, against the default mode;
  * the LP of oracle/psd_cases.lp (nz = 50, 170 rows, neq = 10) at B = 1024;
  * the 4x4 sudoku layer: IR_UNOPT with the full 64-row A against the default mode with the reduced 40-row A.
Prints one JSON line per workload, with the device name and power limit. Writes nothing."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import psd_cases as pc  # noqa: E402
from qpth_b200 import KKTSolvers, QPFunction, kkt  # noqa: E402
from qpth_b200.problems import random_qp_batch  # noqa: E402


def _dev(a):
    return torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda", requires_grad=True)


def time_step(ins, steps=20, warmup=3, **opts):
    f = QPFunction(verbose=-1, check_Q_spd=False, **opts)
    dl = torch.randn(ins[1].shape[0] if ins[1].dim() == 2 else 1, ins[0].shape[-1], dtype=torch.float64, device="cuda")

    def one():
        for t in ins:
            t.grad = None
        z = f(*ins)
        z.backward(dl.expand_as(z))
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        one()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, float(f.last_solve().iters.double().mean())


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = []
    pr = random_qp_batch(128, 100, 100, 0, seed=0)
    e = torch.empty(0, dtype=torch.float64, device="cuda")
    c2 = [_dev(pr[k]) for k in ("Q", "p", "G", "h")] + [e, e]
    for _ in range(2):                                   # alternate the variants: two rounds
        res.append(("C2 default", *time_step(c2)))
        for s in (0, 1):
            kkt.IR_STEPS = s
            res.append(("C2 IR_UNOPT steps=%d" % s, *time_step(c2, kkt_solver=KKTSolvers.IR_UNOPT)))
    kkt.IR_STEPS = 1
    cases = [pc.lp(s) for s in range(1024)]
    lp = [_dev(np.stack([c[k] for c in cases])) for k in range(6)]
    for s in (0, 1):
        kkt.IR_STEPS = s
        res.append(("LP B=1024 IR_UNOPT steps=%d" % s, *time_step(lp, steps=5, kkt_solver=KKTSolvers.IR_UNOPT)))
    kkt.IR_STEPS = 1
    B = 256
    Q, _, G, h, A, b = pc.sudoku4(0)
    p = np.stack([pc.sudoku4(s)[1] for s in range(B)])
    full = [_dev(Q), _dev(p), _dev(G), _dev(h), _dev(A), _dev(b)]
    # the reduced A: 40 independent rows of the full one (the notebook's layer has a rank-40, 40-row A)
    _, _, piv = __import__("scipy.linalg", fromlist=["qr"]).qr(A.T, pivoting=True)
    Ar = A[np.sort(piv[:40])]
    red = [_dev(Q), _dev(p), _dev(G), _dev(h), _dev(Ar), _dev(np.ones(40))]
    for _ in range(2):
        res.append(("sudoku4 B=256 default, 40-row A", *time_step(red)))
        res.append(("sudoku4 B=256 IR_UNOPT, full 64-row A", *time_step(full, kkt_solver=KKTSolvers.IR_UNOPT)))
    for name, ms, it in res:
        print(json.dumps(dict(workload=name, ms_per_step=round(ms, 3), mean_iters=round(it, 2), gpu=gpu)))


if __name__ == "__main__":
    main()
