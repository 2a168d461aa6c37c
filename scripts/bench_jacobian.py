"""The cost of a full Jacobian of (z*, lam, nu) with respect to (p, h, b): the kernel (qpb200_jacobian), the
column-by-column path (one qpb200_jvp per column, an un-batched unit tangent) and what a user does without either, nz
torch.autograd.grad calls on z.sum(0) with retain_graph=True (dz/dp only). One JSON line per shape on stdout.

    python scripts/bench_jacobian.py [--steps 5] [--pairs 5]

Each path is timed as forward + Jacobian per step with CUDA events, the three paths alternating in `pairs` windows of
`steps` steps, median window. The kernel alone is timed on the solved state of the last forward. Achieved rates use the
shape formulas below (fp64 operations and algorithmic bytes of the kernel); the line carries the GPU name and power
limit, and the largest per-QP relative difference between the kernel and the column-by-column path. Nothing is written
to the tree.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402

from scripts.bench_duals import gpu_info   # noqa: E402

# name, B, nz, nineq, neq, Q and G shared
SHAPES = [("c2", 128, 100, 100, 0, False), ("c3", 1024, 50, 50, 10, False), ("c4", 64, 200, 200, 0, True),
          ("tiny", 4096, 10, 5, 0, False), ("uncovered_201", 64, 201, 201, 0, True)]


def kernel_work(B, nz, nineq, neq):
    """(fp64 flops, bytes) of qpb200_jacobian with every row and column: S = W W' (ms^2 nz), its Cholesky (ms^3 / 3), and
    per column the L solve (nz^2, p columns), W U (2 ms nz, p columns), the S solve (2 ms^2), W' Y (2 ms nz) and the
    L' solve (nz^2); bytes: W and L read once, lam and s, J written."""
    ms = neq + nineq
    nc = nz + ms
    per = ms * ms * nz + ms ** 3 / 3 + nz * (nz * nz + 2 * ms * nz) + nc * (2 * ms * ms + 2 * ms * nz + nz * nz)
    byt = 8 * (ms * nz + nz * (nz + 1) / 2 + 2 * nineq + (nz + ms) * nc)
    return B * per, B * byt


def problem(B, nz, nineq, neq, shared, dev):
    from qpth_b200.problems import random_qp_batch
    pr = random_qp_batch(B, nz, nineq, neq, seed=3)
    t = {k: torch.tensor(pr[k], dtype=torch.float64, device=dev) for k in ("Q", "p", "G", "h", "A", "b")}
    if shared:
        t["Q"], t["G"] = t["Q"][0].contiguous(), t["G"][0].contiguous()
        if neq:
            t["A"] = t["A"][0].contiguous()
    if not neq:
        t["A"] = t["b"] = torch.Tensor().to(dev).double()
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jacobian: no CUDA device")
    from qpth_b200 import QPFunction
    from qpth_b200.qp import _jacobian_columns, _jacobian_kernel, jacobian_covered
    dev = torch.device("cuda:0")
    info = gpu_info()
    for name, B, nz, nineq, neq, shared in SHAPES:
        t = problem(B, nz, nineq, neq, shared, dev)
        f = QPFunction(verbose=-1, check_Q_spd=False)
        args6 = [t[k] for k in ("Q", "p", "G", "h", "A", "b")]
        wrt = ("p", "h", "b") if neq else ("p", "h")
        rows = cols = 7 if neq else 3
        R = nz + nineq + neq

        def step_path(path):
            if path == "autograd":
                p = t["p"].clone().requires_grad_(True)
                z = f(t["Q"], p, *args6[2:])
                s = z.sum(0)
                return [torch.autograd.grad(s[j], p, retain_graph=True)[0] for j in range(nz)]
            f(*args6)
            st = f.last_solve()
            J = torch.empty(B, R, R, dtype=torch.float64, device=dev)
            if path == "kernel":
                _jacobian_kernel(st, rows, cols, J)
            else:
                _jacobian_columns(st, rows, cols, J)
            return J

        covered = jacobian_covered(_lib_plan(f, args6))
        paths = (["kernel"] if covered else []) + ["columns", "autograd"]
        for pth in paths:                                    # warm-up
            step_path(pth)
        torch.cuda.synchronize()
        times = {pth: [] for pth in paths}
        for _ in range(args.pairs):
            for pth in paths:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step_path(pth)
                e1.record()
                torch.cuda.synchronize()
                times[pth].append(e0.elapsed_time(e1) / args.steps)
        out = dict(shape=name, B=B, nz=nz, nineq=nineq, neq=neq, shared_QG=shared, covered=covered, gpu=info)
        out.update({"fwd_jac_ms_" + pth: float(np.median(v)) for pth, v in times.items()})
        f(*args6)
        st = f.last_solve()
        Jc = torch.empty(B, R, R, dtype=torch.float64, device=dev)
        _jacobian_columns(st, rows, cols, Jc)
        if covered:
            J = torch.empty_like(Jc)
            _jacobian_kernel(st, rows, cols, J)
            n_k = 20
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n_k):
                _jacobian_kernel(st, rows, cols, J)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n_k
            fl, by = kernel_work(B, nz, nineq, neq)
            num = (J - Jc).abs().amax(dim=(1, 2))
            den = Jc.abs().amax(dim=(1, 2))
            out.update(kernel_ms=ms, kernel_gflops=fl / ms / 1e6, kernel_gbps=by / ms / 1e6,
                       max_rel_kernel_vs_columns=float((num / den).max()))
        print(json.dumps(out), flush=True)


def _lib_plan(f, args6):
    f(*args6)
    return f.last_solve().plan


if __name__ == "__main__":
    main()
