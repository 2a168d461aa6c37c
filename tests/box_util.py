"""Helpers of the box-QP tests: load a BOX_CASES fixture, run BoxQPFunction / QPFunction on a box problem."""
import os

import numpy as np

from oracle.box_cases import BOX_CASES, dense_problem
from oracle.cases import checksum

BOX_KEYS = ("q", "p", "A", "b", "lb", "ub")
GRAD_KEYS = ("dq", "dp", "dA", "db", "dlb", "dub")


def load_box_case(name, golden_dir):
    bx = BOX_CASES[name]()
    gold = dict(np.load(os.path.join(golden_dir, name + ".npz")))
    cs = checksum(dense_problem(bx))
    assert abs(cs - float(gold["input_checksum"])) <= 1e-9 * abs(cs), "golden inputs no longer reproduce from the seed"
    return bx, gold


def run_box(bx, dev="cuda:0", requires=True, **opts):
    import torch
    from qpth_b200 import BoxQPFunction
    t = {}
    for k in BOX_KEYS:
        v = bx[k]
        if v is None:
            t[k] = None
        elif np.asarray(v).size == 0:
            t[k] = torch.Tensor().to(dev).double()
        else:
            t[k] = torch.tensor(np.asarray(v), dtype=torch.float64, device=dev, requires_grad=requires)
    f = BoxQPFunction(**dict(dict(verbose=-1), **opts))
    z = f(*(t[k] for k in BOX_KEYS))
    st = f.last_solve()
    out = dict(zhat=z.detach().cpu().numpy(), lam=st.lam.cpu().numpy(), slacks=st.slacks.cpu().numpy(),
               nus=None if st.nus is None else st.nus.cpu().numpy(), iters=st.iters.cpu().numpy(),
               best_resid=st.best_resid.cpu().numpy(), trace=None if st.trace is None else st.trace.cpu().numpy())
    if requires and bx.get("dl") is not None:
        z.backward(torch.tensor(np.asarray(bx["dl"]).reshape(z.shape), dtype=torch.float64, device=dev))
        out["grads"] = {g: (None if (t[k] is None or t[k].grad is None) else t[k].grad.cpu().numpy())
                        for g, k in zip(GRAD_KEYS, BOX_KEYS)}
    return out


def random_box(seed, B, n, e, sides, shared=(), q_scale=1.0):
    """sides: "lb", "ub" or "both"; shared: names of inputs passed un-batched."""
    rs = np.random.RandomState(seed)
    lb = -rs.rand(B, n) if sides in ("lb", "both") else None
    ub = rs.rand(B, n) + (0.5 if sides == "both" else 0.0) if sides in ("ub", "both") else None
    bx = dict(q=q_scale * (0.1 + rs.rand(B, n)), p=2.0 * rs.randn(B, n), A=rs.randn(B, e, n), lb=lb, ub=ub,
              dl=rs.randn(B, n))
    # a point strictly inside every QP's box: lb in [-1, 0], ub in [0, 1] (one side) or [0.5, 1.5] (both)
    z0 = {"both": 0.05 + 0.4 * rs.rand(n), "lb": 0.05 + rs.rand(n), "ub": -0.05 - rs.rand(n)}[sides]
    for k in shared:
        if bx.get(k) is not None:
            bx[k] = bx[k][0]
    b = bx["A"] @ z0
    bx["b"] = b if (b.ndim == 2 or "b" in shared) else np.tile(b, (B, 1))
    if e == 0:
        bx["A"] = np.zeros((0,))
        bx["b"] = np.zeros((0,))
    return bx
