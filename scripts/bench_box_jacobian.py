"""The cost of a full BoxQPFunction Jacobian of (z*, lam, nu) with respect to (p, lb, ub, b): the kernel
(qpb200_box_jacobian, diagonal q; qpb200_boxq_jacobian, dense Q), the column-by-column path (one qpb200_box_jvp /
qpb200_boxq_jvp per column, an un-batched unit tangent) and what a user does without either, nz torch.autograd.grad calls on z.sum(0) with
retain_graph=True (dz/dp only). One JSON line per shape on stdout.

    python scripts/bench_box_jacobian.py [--steps 3] [--pairs 3]

Each path is timed as forward + Jacobian per step with CUDA events, the paths alternating in `pairs` windows of `steps`
steps, median window. The kernel alone is timed on the solved state of the last forward. Achieved rates use the shape
formulas of kernel_work / boxq_kernel_work (fp64 operations and algorithmic bytes); the line carries the GPU name and power limit, and the
largest per-QP relative difference between the kernel and the column path. Nothing is written to the tree.

Shapes: the OptNet sudoku layer of bench_box.py (one CTA per QP in the forward), a projection wide enough for a
two-CTA cluster forward (Jacobian with respect to p only: J is 1.5 GB there, so writing it may bound the kernel), and
the portfolio and MPC shapes of bench_box_dense.py (dense Q: qpb200_boxq_jacobian).
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402

from scripts.bench_duals import gpu_info   # noqa: E402

# name, B, nz, neq, sides, dense Q, wrt
SHAPES = [("sudoku_64_40", 1024, 64, 40, "lb", False, None), ("cluster_1000_8", 64, 1000, 8, "both", False, ("p",)),
          ("portfolio", 1024, 100, 1, "both", True, None), ("mpc", 1024, 80, 0, "both", True, None)]


def kernel_work(B, nz, neq, nlb, nub, R, C, p_blocks, b_cols):
    """(fp64 flops, bytes) of qpb200_box_jacobian: M = A H^-1 A' (neq^2 nz, lower half), its Cholesky (neq^3 / 3), per
    p column A H^-1 E (2 neq nz), the M solve (2 neq^2) and A'Y (2 neq nz), per b column the M solve and A'Y; bytes: A,
    q, lam and s read once, J written."""
    per = neq * neq * nz + neq ** 3 / 3 + p_blocks * (4 * neq * nz + 2 * neq * neq) + b_cols * (2 * neq * neq + 2 * neq * nz)
    byt = 8 * (neq * nz + nz + 2 * (nlb + nub) + R * C)
    return B * per, B * byt


def boxq_kernel_work(B, nz, neq, nlb, nub, R, C, p_blocks, b_cols):
    """(fp64 flops, bytes) of qpb200_boxq_jacobian: the bordered factor of order N = nz_pad + neq_pad (N^3 / 3) and per
    solved column the forward sweep, diagonal and backward sweep (2 N^2); bytes: Q, A, lam and s read once, J written."""
    N = (nz + 7) // 8 * 8 + (neq + 7) // 8 * 8
    per = N ** 3 / 3 + (p_blocks + b_cols) * 2 * N * N
    byt = 8 * (nz * nz + neq * nz + 2 * (nlb + nub) + R * C)
    return B * per, B * byt


def problem(name, B, nz, neq, sides, dense_Q, dev):
    """The inputs of bench_box.py (sudoku), bench_box_wide.py (projection) and bench_box_dense.py (portfolio, MPC)."""
    f64 = dict(dtype=torch.float64, device=dev)
    T = lambda a: None if a is None else torch.tensor(a, **f64)
    if dense_Q:
        from scripts.bench_box_dense import SHAPES as DSHAPES, problem as dproblem
        (shared,) = [s[4] for s in DSHAPES if s[0] == name]
        d, _ = dproblem(nz, sides, neq, shared, B, 5)
        return [T(d["Q"]), T(d["p"]), T(d["A"]), T(d["b"]), T(d["lb"]), T(d["ub"])]
    rs = np.random.RandomState(31)
    if name.startswith("sudoku"):
        A = rs.randn(neq, nz)
        z0 = rs.rand(nz) + 0.1
        return [torch.full((nz,), 0.1, **f64), T(-rs.rand(B, nz)), T(A), T(A @ z0), torch.zeros(nz, **f64), None]
    A = rs.randn(neq, nz)
    z0 = 0.05 + 0.4 * rs.rand(nz)
    return [T(0.1 + rs.rand(nz)), T(2.0 * rs.randn(B, nz)), T(A), T(A @ z0), T(-rs.rand(nz)), T(0.5 + rs.rand(nz))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_box_jacobian: no CUDA device")
    from qpth_b200 import BoxQPFunction
    from qpth_b200.box import BOX_JAC_WRT, _box_jacobian_columns, _box_jacobian_kernel, box_jacobian_covered
    dev = torch.device("cuda:0")
    info = gpu_info()
    for name, B, nz, neq, sides, dense_Q, wrt in SHAPES:
        ins = problem(name, B, nz, neq, sides, dense_Q, dev)
        f = BoxQPFunction(verbose=-1, check_Q_spd=False, dense_Q=dense_Q)
        nlb, nub = (nz if sides != "ub" else 0), (nz if sides != "lb" else 0)
        names = wrt or tuple(k for k, w in zip(BOX_JAC_WRT, (nz, nlb, nub, neq)) if w)
        rows = 7 if neq else 3
        cols = sum(1 << BOX_JAC_WRT.index(k) for k in names)
        R = nz + nlb + nub + neq
        C = sum(neq if k == "b" else nz for k in names)
        f(*ins)
        st = f.last_solve()
        covered = st.dense is None and box_jacobian_covered(st.plan, dense_Q)

        def step_path(path):
            if path == "autograd":
                p = ins[1].clone().requires_grad_(True)
                z = f(ins[0], p, *ins[2:])
                s = z.sum(0)
                return [torch.autograd.grad(s[j], p, retain_graph=True)[0] for j in range(nz)]
            f(*ins)
            J = torch.empty(B, R, C, dtype=torch.float64, device=dev)
            (_box_jacobian_kernel if path == "kernel" else _box_jacobian_columns)(f.last_solve(), rows, cols, J)
            return J

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
        out = dict(shape=name, B=B, nz=nz, neq=neq, sides=sides, dense_Q=dense_Q, wrt=list(names), columns=C,
                   covered=covered, gpu=info)
        out.update({"fwd_jac_ms_" + pth: float(np.median(v)) for pth, v in times.items()})
        if covered:
            f(*ins)
            st = f.last_solve()
            Jc = torch.empty(B, R, C, dtype=torch.float64, device=dev)
            _box_jacobian_columns(st, rows, cols, Jc)
            J = torch.empty_like(Jc)
            _box_jacobian_kernel(st, rows, cols, J)
            n_k = 10
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n_k):
                _box_jacobian_kernel(st, rows, cols, J)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n_k
            p_blocks = ((nz + 7) // 8) * 8 if (cols & 7) else 0
            b_cols = ((neq + 7) // 8) * 8 if (cols & 8) else 0
            fl, by = (boxq_kernel_work if dense_Q else kernel_work)(B, nz, neq, nlb, nub, R, C, p_blocks, b_cols)
            num = (J - Jc).abs().amax(dim=(1, 2))
            den = Jc.abs().amax(dim=(1, 2))
            out.update(kernel_ms=ms, kernel_gflops=fl / ms / 1e6, kernel_gbps=by / ms / 1e6,
                       max_rel_kernel_vs_columns=float((num / den).max()))
            del J, Jc
        print(json.dumps(out), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
