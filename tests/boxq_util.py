"""Helpers of the dense-Q box-QP tests: load a BOXQ_CASES fixture, build random problems, run
BoxQPFunction(dense_Q=True) and QPFunction on the dense equivalent."""
import os

import numpy as np

from oracle.boxq_cases import BOXQ_CASES, dense_problem, map_dense_grads
from oracle.cases import checksum

KEYS = ("Q", "p", "A", "b", "lb", "ub")
GRAD_KEYS = ("dQ", "dp", "dA", "db", "dlb", "dub")


def load_boxq_case(name, golden_dir):
    bx = BOXQ_CASES[name]()
    gold = dict(np.load(os.path.join(golden_dir, name + ".npz")))
    cs = checksum(dense_problem(bx))
    assert abs(cs - float(gold["input_checksum"])) <= 1e-9 * abs(cs), "golden inputs no longer reproduce from the seed"
    return bx, gold


def random_boxq(seed, B, n, e, sides, shared=(), cond_decades=2.0):
    """sides: "lb", "ub" or "both"; shared: names of inputs passed un-batched (Q among them)."""
    rs = np.random.RandomState(seed)
    Q = np.empty((B, n, n))
    for i in range(B):
        U, _ = np.linalg.qr(rs.randn(n, n))
        Q[i] = (U * (10.0 ** (-cond_decades * rs.rand(n)) + 0.05)) @ U.T
        Q[i] = 0.5 * (Q[i] + Q[i].T)
    lb = -rs.rand(B, n) if sides in ("lb", "both") else None
    ub = rs.rand(B, n) + (0.5 if sides == "both" else 0.0) if sides in ("ub", "both") else None
    bx = dict(Q=Q, p=2.0 * rs.randn(B, n), A=rs.randn(B, e, n), lb=lb, ub=ub, dl=rs.randn(B, n))
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


def _tensors(bx, dev, requires):
    import torch
    t = {}
    for k in KEYS:
        v = bx[k]
        if v is None:
            t[k] = None
        elif np.asarray(v).size == 0:
            t[k] = torch.Tensor().to(dev).double()
        else:
            t[k] = torch.tensor(np.asarray(v), dtype=torch.float64, device=dev, requires_grad=requires)
    return t


def run_boxq(bx, dev="cuda:0", requires=True, **opts):
    import torch
    from qpth_b200 import BoxQPFunction
    t = _tensors(bx, dev, requires)
    f = BoxQPFunction(**dict(dict(verbose=-1, dense_Q=True), **opts))
    z = f(*(t[k] for k in KEYS))
    st = f.last_solve()
    out = dict(zhat=z.detach().cpu().numpy(), lam=st.lam.cpu().numpy(), slacks=st.slacks.cpu().numpy(),
               nus=None if st.nus is None else st.nus.cpu().numpy(), iters=st.iters.cpu().numpy(),
               best_resid=st.best_resid.cpu().numpy(), trace=None if st.trace is None else st.trace.cpu().numpy(),
               dense=st.dense is not None)
    if requires and bx.get("dl") is not None:
        z.backward(torch.tensor(np.asarray(bx["dl"]).reshape(z.shape), dtype=torch.float64, device=dev))
        out["grads"] = {g: (None if (t[k] is None or t[k].grad is None) else t[k].grad.cpu().numpy())
                        for g, k in zip(GRAD_KEYS, KEYS)}
    return out


def run_dense(bx, dev="cuda:0", **opts):
    """QPFunction on the dense equivalent (Q, G = [-I; I], h = [-lb; ub]); gradients mapped to the box inputs."""
    import torch
    from qpth_b200 import QPFunction
    from qpth_b200.box import dense_equivalent
    t = {k: (None if bx[k] is None else torch.tensor(np.asarray(bx[k]), dtype=torch.float64, device=dev)) for k in KEYS}
    Q, G, h = dense_equivalent(t["Q"], t["lb"], t["ub"], dense_Q=True)
    ins = dict(Q=Q, p=t["p"], G=G, h=h, A=t["A"], b=t["b"])
    for v in ins.values():
        if v.numel():
            v.requires_grad_(True)
    f = QPFunction(**dict(dict(verbose=-1), **opts))
    z = f(*(ins[k] for k in ("Q", "p", "G", "h", "A", "b")))
    z.backward(torch.tensor(np.asarray(bx["dl"]), dtype=torch.float64, device=dev))
    g = tuple(None if (v.grad is None) else v.grad.cpu().numpy() for v in ins.values())
    st = f.last_solve()
    return dict(zhat=z.detach().cpu().numpy(), iters=st.iters.cpu().numpy(), grads=map_dense_grads(g, bx))


def batched(bx, B):
    """Every input of a problem dict with a leading batch dimension (numpy), for the model."""
    n = np.asarray(bx["p"]).shape[-1]
    out = {}
    for k, nd in (("Q", 3), ("p", 2), ("lb", 2), ("ub", 2)):
        v = bx[k]
        out[k] = None if v is None else (np.asarray(v) if np.asarray(v).ndim == nd else np.broadcast_to(v, (B,) + np.shape(v)))
    A = np.asarray(bx["A"])
    if A.ndim >= 2 and A.shape[-2] > 0:
        out["A"] = A if A.ndim == 3 else np.broadcast_to(A, (B,) + A.shape)
        bb = np.asarray(bx["b"])
        out["b"] = bb if bb.ndim == 2 else np.broadcast_to(bb, (B,) + bb.shape)
    else:
        out["A"], out["b"] = np.zeros((B, 0, n)), np.zeros((B, 0))
    return out
