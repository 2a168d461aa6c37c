"""BoxQPFunction against QPFunction at the OptNet sudoku shape: one JSON line on stdout.

    python scripts/bench_box.py [--batch 1024] [--steps 10] [--pairs 3]

Both solve the same problems (BoxQPFunction on q, lb; QPFunction on the dense equivalent Q = diag(q), G = -I, h = -lb),
fwd+bwd per step, alternating in one process so that both see the same clocks and neighbours. The line carries the GPU
name and power limit, ms per step, QPs/s and mean Newton iterations of each path, and the largest per-QP relative
difference of z* and of every gradient between them. Nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402


def run_box(dev, B=1024, nz=64, neq=40, steps=10, pairs=3):
    """The OptNet sudoku shape (example-sudoku.ipynb:305-323): q = 0.1 (Q = 0.1 I), lb = 0 (G = -I, h = 0), a shared A and
    b, batched p; fwd+bwd of BoxQPFunction against QPFunction on the dense equivalent, alternating in the same call
    (`pairs` pairs of `steps`-step windows, CUDA events, median window). B = 1024 fills the GPU several times over."""
    from qpth_b200 import BoxQPFunction, QPFunction
    rs = np.random.RandomState(31)
    A_ = rs.randn(neq, nz)
    z0 = rs.rand(nz) + 0.1
    f64 = dict(dtype=torch.float64, device=dev)
    box = {"q": torch.full((nz,), 0.1, **f64), "p": torch.tensor(-rs.rand(B, nz), **f64),
           "A": torch.tensor(A_, **f64), "b": torch.tensor(A_ @ z0, **f64), "lb": torch.zeros(nz, **f64)}
    dense = {"Q": 0.1 * torch.eye(nz, **f64), "p": box["p"].clone(), "G": -torch.eye(nz, **f64),
             "h": torch.zeros(nz, **f64), "A": box["A"].clone(), "b": box["b"].clone()}
    for t in list(box.values()) + list(dense.values()):
        t.requires_grad_(True)
    dl = torch.tensor(rs.randn(B, nz), **f64)
    fb, fd = BoxQPFunction(verbose=-1, check_Q_spd=False), QPFunction(verbose=-1, check_Q_spd=False)

    def run_box_once():
        for v in box.values():
            v.grad = None
        z = fb(box["q"], box["p"], box["A"], box["b"], box["lb"], None)
        z.backward(dl)
        return z

    def run_dense_once():
        for v in dense.values():
            v.grad = None
        z = fd(dense["Q"], dense["p"], dense["G"], dense["h"], dense["A"], dense["b"])
        z.backward(dl)
        return z

    def window(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps
    for _ in range(3):
        run_box_once(); run_dense_once()
    torch.cuda.synchronize()
    tb, td = [], []
    for _ in range(pairs):
        tb.append(window(run_box_once))
        td.append(window(run_dense_once))
    zb, zd = run_box_once().detach(), run_dense_once().detach()
    itb = float(fb.last_solve().iters.double().mean())
    itd = float(fd.last_solve().iters.double().mean())

    def rel(a, b, floor=1e-4):
        """max per-QP relative l2 difference; the denominator is floored at `floor` x the batch maximum, as in
        tests/parity.py (a QP at a vertex has dz*/dp = 0 and both paths return clamp noise there)"""
        a = a.reshape(a.shape[0], -1) if a.dim() > 1 else a.reshape(1, -1)
        b = b.reshape(b.shape[0], -1) if b.dim() > 1 else b.reshape(1, -1)
        nb = b.norm(dim=1)
        return float(((a - b).norm(dim=1) / torch.maximum(nb, floor * nb.max()).clamp_min(1e-300)).max())
    diffs = {"z": rel(zb, zd, 0.0), "dq": rel(box["q"].grad, torch.diagonal(dense["Q"].grad)), "dp": rel(box["p"].grad, dense["p"].grad),
             "dA": rel(box["A"].grad, dense["A"].grad), "db": rel(box["b"].grad, dense["b"].grad),
             "dlb": rel(box["lb"].grad, -dense["h"].grad)}
    mb, md = float(np.median(tb)), float(np.median(td))
    return {"shape": {"B": B, "nz": nz, "neq": neq, "bounds": "lb = 0", "shared": "q, A, b, lb", "batched": "p"},
            "box": {"ms_per_step": mb, "QPs_per_s": B / (mb * 1e-3), "mean_newton_iters": itb, "windows_ms": tb},
            "dense": {"ms_per_step": md, "QPs_per_s": B / (md * 1e-3), "mean_newton_iters": itd, "windows_ms": td},
            "speedup": md / mb, "max_rel_diff_box_vs_dense": diffs,
            "api": "BoxQPFunction(verbose=-1, check_Q_spd=False) vs QPFunction on Q = 0.1 I, G = -I, h = 0; fwd+bwd per step"}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_box: no CUDA device (a timing needs the GPU)")
    dev = torch.device("cuda:0")
    line = run_box(dev, B=args.batch, steps=args.steps, pairs=args.pairs)
    line["gpu"] = gpu_info()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
