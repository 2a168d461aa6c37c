"""BoxQPFunction(dense_Q=True) against QPFunction on the dense equivalent: one JSON line on stdout.

    python scripts/bench_box_dense.py [--batch 1024] [--steps 10] [--pairs 3]

Both solve the same problems (BoxQPFunction(dense_Q=True) on Q, lb, ub; QPFunction on Q, G = [-I; I], h = [-lb; ub]),
fwd+bwd per step, alternating in one process so that both see the same clocks and neighbours. Per shape the line
carries ms per step, QPs/s and mean Newton iterations of each path and the largest per-QP relative difference of z* and
of every gradient between them; the GPU name and power limit are on the line. Nothing is written to the tree.
Shapes (nz, bounds, neq): the portfolio (100, both, 1; batched Q and p), an MPC-like (80, both, 0; shared Q, batched
p), (64, lb, 40) and the largest shape the plan covers with both bounds (184, both, 1).
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np   # noqa: E402
import torch         # noqa: E402

from bench_box import gpu_info   # noqa: E402

SHAPES = [("portfolio", 100, "both", 1, ("A", "b", "lb", "ub")),
          ("mpc", 80, "both", 0, ("Q", "lb", "ub")),
          ("lb_64_40", 64, "lb", 40, ("A", "b", "lb")),
          ("largest_both", 184, "both", 1, ("A", "b", "lb", "ub"))]


def problem(n, sides, e, shared, B, seed):
    rs = np.random.RandomState(seed)
    nq = 1 if "Q" in shared else B
    F = rs.randn(nq, n, n // 4 + 1)
    Q = np.einsum("bik,bjk->bij", F, F) / F.shape[-1] + 0.05 * np.eye(n)
    lb = np.zeros(n) if sides in ("lb", "both") else None
    ub = np.ones(n) if sides in ("ub", "both") else None
    A = np.ones((e, n)) if e == 1 else rs.randn(e, n)
    z0 = 0.05 + 0.5 * rs.rand(n) / max(1, n // 20)
    b = A @ z0 if e else np.zeros(0)
    if e == 1:
        b = np.ones(1)
    d = dict(Q=Q[0] if "Q" in shared else Q, p=rs.randn(B, n), A=A if e else np.zeros(0), b=b, lb=lb, ub=ub)
    return d, rs.randn(B, n)


def run_shape(dev, name, n, sides, e, shared, B, steps, pairs):
    from qpth_b200 import BoxQPFunction, QPFunction
    from qpth_b200.box import dense_equivalent
    bx, dl = problem(n, sides, e, shared, B, 7 + n + e)
    t = {k: (None if v is None else torch.tensor(v, dtype=torch.float64, device=dev)) for k, v in bx.items()}
    dlt = torch.tensor(dl, dtype=torch.float64, device=dev)
    keys = ("Q", "p", "A", "b", "lb", "ub")
    fb = BoxQPFunction(verbose=-1, check_Q_spd=False, dense_Q=True)
    fd = QPFunction(verbose=-1, check_Q_spd=False)
    Q, G, h = dense_equivalent(t["Q"], t["lb"], t["ub"], dense_Q=True)
    dense_in = dict(Q=Q, p=t["p"], G=G, h=h, A=t["A"], b=t["b"])

    def step_box():
        ins = {k: (None if v is None else v.detach().clone().requires_grad_(v.numel() > 0)) for k, v in t.items()}
        z = fb(*(ins[k] for k in keys))
        z.backward(dlt)
        return z, {k: ins[k].grad for k in keys if ins[k] is not None and ins[k].grad is not None}

    def step_dense():
        ins = {k: v.detach().clone().requires_grad_(v.numel() > 0) for k, v in dense_in.items()}
        z = fd(*(ins[k] for k in ("Q", "p", "G", "h", "A", "b")))
        z.backward(dlt)
        return z, ins

    def window(fn):
        s, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for _ in range(steps):
            fn()
        e_.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e_) / steps

    for _ in range(2):
        step_box(); step_dense()
    tb, td = [], []
    for _ in range(pairs):
        tb.append(window(step_box))
        td.append(window(step_dense))
    zb, gb = step_box()
    itb = float(fb.last_solve().iters.float().mean())
    zd, ind = step_dense()
    itd = float(fd.last_solve().iters.float().mean())

    def rel(a, b):
        a = a.detach().reshape(a.shape[0] if a.dim() > 1 else 1, -1)
        b = b.detach().reshape(a.shape)
        nb = b.norm(dim=1)
        den = torch.maximum(nb, 1e-4 * nb.max()).clamp_min(1e-300)
        return float(((a - b).norm(dim=1) / den).max())

    nlb = n if t["lb"] is not None else 0
    gd = dict(Q=ind["Q"].grad, p=ind["p"].grad, A=ind["A"].grad if e else None, b=ind["b"].grad if e else None)
    dh = ind["h"].grad
    if dh.dim() == 2 and t["lb"] is not None and t["lb"].dim() == 1:
        dh = dh.mean(0)
    if t["lb"] is not None:
        gd["lb"] = -dh[..., :nlb]
    if t["ub"] is not None:
        gd["ub"] = dh[..., nlb:]
    diffs = {"z": rel(zb, zd)}
    for k, g in gb.items():
        if gd.get(k) is not None:
            diffs["d" + k] = rel(g, gd[k])
    mb, md = float(np.median(tb)), float(np.median(td))
    return {"shape": name, "nz": n, "bounds": sides, "neq": e, "batch": B, "shared": list(shared),
            "box_dense_Q": {"ms_per_step": mb, "QPs_per_s": B / (mb * 1e-3), "mean_newton_iters": itb},
            "qpfunction": {"ms_per_step": md, "QPs_per_s": B / (md * 1e-3), "mean_newton_iters": itd},
            "speedup": md / mb, "max_rel_diff": diffs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_box_dense: no CUDA device (a timing needs the GPU)")
    dev = torch.device("cuda:0")
    rows = [run_shape(dev, *s, B=args.batch, steps=args.steps, pairs=args.pairs) for s in SHAPES]
    print(json.dumps({"gpu": gpu_info(), "api": "BoxQPFunction(dense_Q=True) vs QPFunction on the dense equivalent; "
                      "fwd+bwd per step, median of alternating windows", "shapes": rows}))


if __name__ == "__main__":
    main()
