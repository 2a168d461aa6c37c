"""BoxQPFunction on shapes beyond one CTA (the thread block cluster kernels): one JSON line on stdout.

    python scripts/bench_box_wide.py [--steps 5] [--pairs 3]

Cases, fwd+bwd per step (CUDA events, median of `pairs` windows of `steps` steps):
- the capped-simplex projection (q = 1, p = -v, 1'z = k, 0 <= z <= 1) at nz = 2000, B = 256 and at nz = 6000, B = 1 and
  B = 256, with the largest distance of z* to the closed form (oracle/projections.py) and the Newton iteration counts;
- nz = 600, neq = 64, both bounds, B = 256;
- nz = 480, neq = 64, both bounds, B = 256, against QPFunction on the dense equivalent (the largest of these shapes the
  dense kernels still take: with both bounds they stop near nz = 500, so the cases above have no dense counterpart),
  with the largest per-QP relative difference of z* and of every gradient.
The line carries the GPU name and power limit. Nothing is written to the tree.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402

from scripts.bench_box import gpu_info   # noqa: E402


def _timed(fn, steps, pairs):
    def window():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ws = [window() for _ in range(pairs)]
    return float(np.median(ws)), ws


def _rel(a, b, floor=1e-4):
    a = a.reshape(a.shape[0], -1) if a.dim() > 1 else a.reshape(1, -1)
    b = b.reshape(b.shape[0], -1) if b.dim() > 1 else b.reshape(1, -1)
    nb = b.norm(dim=1)
    return float(((a - b).norm(dim=1) / torch.maximum(nb, floor * nb.max()).clamp_min(1e-300)).max())


def _box_inputs(dev, B, nz, neq, seed, simplex):
    rs = np.random.RandomState(seed)
    f64 = dict(dtype=torch.float64, device=dev)
    if simplex:
        v = 3.0 * rs.randn(B, nz) / np.sqrt(np.log(nz))
        ins = dict(q=torch.ones(nz, **f64), p=torch.tensor(-v, **f64), A=torch.ones(1, nz, **f64),
                   b=torch.full((1,), 0.1 * nz, **f64), lb=torch.zeros(nz, **f64), ub=torch.ones(nz, **f64))
    else:
        z0 = 0.05 + 0.4 * rs.rand(nz)
        A = rs.randn(neq, nz)
        ins = dict(q=torch.tensor(0.1 + rs.rand(nz), **f64), p=torch.tensor(2.0 * rs.randn(B, nz), **f64),
                   A=torch.tensor(A, **f64), b=torch.tensor(A @ z0, **f64), lb=torch.tensor(-rs.rand(nz), **f64),
                   ub=torch.tensor(0.5 + rs.rand(nz), **f64))
    for t in ins.values():
        t.requires_grad_(True)
    return ins, torch.tensor(rs.randn(B, nz), **f64)


def run_case(dev, B, nz, neq, simplex, steps, pairs, dense=False):
    from qpth_b200 import BoxQPFunction, QPFunction, _lib
    from qpth_b200.box import dense_equivalent
    ins, dl = _box_inputs(dev, B, nz, neq, 7 + nz + B, simplex)
    plan = _lib.box_plan_for(nz, neq, True, True)
    fb = BoxQPFunction(verbose=-1, check_Q_spd=False)
    keys = ("q", "p", "A", "b", "lb", "ub")

    def box_once():
        for v in ins.values():
            v.grad = None
        z = fb(*(ins[k] for k in keys))
        z.backward(dl)
        return z
    mb, wb = _timed(box_once, steps, pairs)
    z = box_once().detach()
    out = {"shape": {"B": B, "nz": nz, "neq": neq, "bounds": "both", "problem": "capped simplex" if simplex else "random"},
           "plan": {"ok": plan.ok, "cl_ctas": plan.cl_ctas, "cl_slice": plan.cl_slice,
                    "cl_smem_bytes": plan.cl_smem_bytes},
           "box": {"ms_per_step": mb, "QPs_per_s": B / (mb * 1e-3), "windows_ms": wb,
                   "mean_newton_iters": float(fb.last_solve().iters.double().mean())}}
    if simplex:
        from oracle.projections import project_capped_simplex
        p = ins["p"].detach().cpu().numpy()
        zc = np.stack([project_capped_simplex(np.ones(nz), p[i], 0.1 * nz, np.zeros(nz), np.ones(nz))[0]
                       for i in range(B)])
        out["max_abs_diff_z_vs_closed_form"] = float(np.abs(z.cpu().numpy() - zc).max())
    if dense:
        Q, G, h = dense_equivalent(ins["q"].detach(), ins["lb"].detach(), ins["ub"].detach())
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
        box_once()
        out["dense"] = {"ms_per_step": md, "QPs_per_s": B / (md * 1e-3), "windows_ms": wd,
                        "mean_newton_iters": float(fd.last_solve().iters.double().mean())}
        out["speedup"] = md / mb
        out["max_rel_diff_box_vs_dense"] = {
            "z": _rel(z, zd, 0.0), "dq": _rel(ins["q"].grad, torch.diagonal(dn["Q"].grad)),
            "dp": _rel(ins["p"].grad, dn["p"].grad), "dA": _rel(ins["A"].grad, dn["A"].grad),
            "db": _rel(ins["b"].grad, dn["b"].grad), "dlb": _rel(ins["lb"].grad, -dn["h"].grad[:nz]),
            "dub": _rel(ins["ub"].grad, dn["h"].grad[nz:])}
    else:
        out["dense"] = "not run: the dense kernels reject this shape"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_box_wide: no CUDA device (a timing needs the GPU)")
    dev = torch.device("cuda:0")
    s, p = args.steps, args.pairs
    line = {"cases": [run_case(dev, 256, 2000, 1, True, s, p), run_case(dev, 256, 600, 64, False, s, p),
                      run_case(dev, 256, 480, 64, False, s, p, dense=True), run_case(dev, 1, 6000, 1, True, s, p),
                      run_case(dev, 256, 6000, 1, True, s, p)],
            "api": "BoxQPFunction(verbose=-1, check_Q_spd=False), fwd+bwd per step; q, A, b, lb, ub shared, p batched",
            "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
