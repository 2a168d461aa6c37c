"""Child process of tests/test_gpu_boxq_edges.py: the first forward, backward, qpb200_boxq_jvp and qpb200_boxq_solve_kkt
of every entry of tests/boxq_families.py on cuda:0 (the `dense` entries: forward and backward on the dense kernels).
Most of these shapes sit on the last bytes of shared memory or at the widest nz, where a layout error would fault; in a
child process such a fault fails only their own tests instead of ending the suite. Each entry's plan is asserted
(check_entry) before it runs. Writes <out_dir>/<entry>.npz (or .err), and each entry's name to <out_dir>/progress.txt
as it starts. Also holds the ctypes calls of the entry points that the tests share.
Usage: python -m tests.boxq_edges_child <out_dir>"""
import ctypes
import os
import sys
import traceback

import numpy as np

DEV = "cuda:0"


def spd(rs, B, n, cond_decades=2.0):
    """B random SPD matrices U diag(10^-U(0, c) + 0.05) U'"""
    Q = np.empty((B, n, n))
    for i in range(B):
        U, _ = np.linalg.qr(rs.randn(n, n))
        Q[i] = (U * (10.0 ** (-cond_decades * rs.rand(n)) + 0.05)) @ U.T
        Q[i] = 0.5 * (Q[i] + Q[i].T)
    return Q


def kkt_inputs(plan, B, seed, lo=-8.0, hi=8.0):
    """(Q, A, d, rx, rs, rz, ry) of B random KKT systems of a dense-Q plan, d = 10^U(lo, hi)"""
    rs = np.random.RandomState(seed)
    n, e, m = plan.nz, plan.neq, plan.nineq
    return (spd(rs, B, n), rs.randn(B, e, n), 10.0 ** rs.uniform(lo, hi, (B, m)), rs.randn(B, n), rs.randn(B, m),
            rs.randn(B, m), rs.randn(B, e))


def point(plan, B, seed, wide=False):
    """A point at which to differentiate: dense SPD Q, A, z, nu, lam and s ~ U(0.1, 10) (wide: 10^U(-12, 0), so that
    d = clamp(lam) / clamp(s) spans [1e-8, 1e8] and the clamp at 1e-8 binds), and adjoints dl, glam, gnu."""
    rs = np.random.RandomState(seed)
    n, e, m = plan.nz, plan.neq, plan.nineq
    pt = dict(Q=spd(rs, B, n), A=rs.randn(B, e, n) / np.sqrt(n), z=rs.randn(B, n), nu=rs.randn(B, e))
    if wide:
        pt.update(lam=10.0 ** rs.uniform(-12, 0, (B, m)), s=10.0 ** rs.uniform(-12, 0, (B, m)))
    else:
        pt.update(lam=rs.uniform(0.1, 10, (B, m)), s=rs.uniform(0.1, 10, (B, m)))
    pt.update(dl=rs.randn(B, n), glam=rs.randn(B, m), gnu=rs.randn(B, e))
    return pt


def _T(a):
    import torch
    return torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)


def _P(t):
    return ctypes.c_void_p(t.data_ptr()) if (t is not None and t.numel()) else ctypes.c_void_p(0)


def run_kkt(plan, ins):
    """one qpb200_boxq_solve_kkt on cuda:0: [dx, ds, dz, dy] as numpy arrays"""
    import torch
    from qpth_b200 import _lib
    B = ins[0].shape[0]
    n, e, m = plan.nz, plan.neq, plan.nineq
    t = [_T(v) for v in ins]
    out = [torch.empty(B, k, dtype=torch.float64, device=DEV) for k in (n, m, m, e)]
    _lib.check(_lib.load().qpb200_boxq_solve_kkt(ctypes.byref(plan), B, _P(t[0]), n * n, _P(t[1]), e * n,
                                                 *(_P(v) for v in t[2:]), *(_P(o) for o in out), ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


GRAD_NAMES = ("dx", "dlam", "dnu", "dQ", "dp", "dlb", "dub", "dA", "db")


def run_backward(plan, pt, dl, glam, gnu):
    """qpb200_boxq_backward_duals at the point with adjoints (dl, glam, gnu; None: NULL), every gradient batched: dict
    of GRAD_NAMES (None where the QP has no such input)"""
    import torch
    from qpth_b200 import _lib
    B, n = pt["z"].shape
    e, m = plan.neq, plan.nineq
    ins = {k: _T(pt[k]) for k in ("Q", "A", "z", "nu", "lam", "s")}
    f64 = dict(dtype=torch.float64, device=DEV)
    outs = dict(zip(GRAD_NAMES, (torch.empty(B, *s, **f64) for s in ((n,), (m,), (e,), (n, n), (n,), (n,), (n,),
                                                                       (e, n), (e,)))))
    if not plan.has_lb:
        outs["dlb"] = None
    if not plan.has_ub:
        outs["dub"] = None
    if not e:
        outs.update(dnu=None, dA=None, db=None)
    adj = [None if a is None else _T(a) for a in (dl, glam, gnu)]       # (kept alive until the kernels have run)
    grads = []
    for k in ("dQ", "dp", "dlb", "dub", "dA", "db"):
        grads += [_P(outs[k]), 0]
    _lib.check(_lib.load().qpb200_boxq_backward_duals(
        ctypes.byref(plan), B, _P(ins["Q"]), n * n, _P(ins["A"]), e * n, *(_P(a) for a in adj), _P(ins["z"]),
        _P(ins["lam"]), _P(ins["s"]), _P(ins["nu"]), *grads, _P(outs["dx"]), _P(outs["dlam"]), _P(outs["dnu"]),
        ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    return {k: (None if v is None else v.cpu().numpy()) for k, v in outs.items()}


TANGENTS = ("Q", "p", "A", "b", "lb", "ub")


def run_jvp(plan, pt, tan):
    """qpb200_boxq_jvp at the point: (dz, dlam, dnu). tan: dict of TANGENTS, each None (NULL), batched (B, ...) or
    un-batched (stride 0)."""
    import torch
    from qpth_b200 import _lib
    B, n = pt["z"].shape
    e, m = plan.neq, plan.nineq
    ins = {k: _T(pt[k]) for k in ("Q", "A", "z", "nu", "lam", "s")}
    per = dict(Q=n * n, p=n, A=e * n, b=e, lb=n, ub=n)
    nd = dict(Q=3, p=2, A=3, b=2, lb=2, ub=2)
    tt = {k: (None if tan.get(k) is None else _T(tan[k])) for k in TANGENTS}
    args = []
    for k in TANGENTS:
        args += [_P(tt[k]), per[k] if (tt[k] is not None and tt[k].dim() == nd[k]) else 0]
    f64 = dict(dtype=torch.float64, device=DEV)
    rhs = torch.empty(B * (n + m + e), **f64)
    dz, dlam, dnu = torch.empty(B, n, **f64), torch.empty(B, m, **f64), torch.empty(B, e, **f64)
    _lib.check(_lib.load().qpb200_boxq_jvp(ctypes.byref(plan), B, _P(ins["Q"]), n * n, _P(ins["A"]), e * n, *args,
                                           _P(ins["z"]), _P(ins["lam"]), _P(ins["s"]), _P(ins["nu"]), _P(rhs), _P(dz),
                                           _P(dlam), _P(dnu), ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    return dz.cpu().numpy(), dlam.cpu().numpy(), dnu.cpu().numpy()


def tangents(plan, B, seed):
    """every tangent batched, dQ not symmetric; None for the inputs the QP does not have"""
    rs = np.random.RandomState(seed)
    n, e = plan.nz, plan.neq
    return dict(Q=rs.randn(B, n, n), p=rs.randn(B, n), A=rs.randn(B, e, n) if e else None,
                b=rs.randn(B, e) if e else None, lb=rs.randn(B, n) if plan.has_lb else None,
                ub=rs.randn(B, n) if plan.has_ub else None)


def main(out_dir):
    from tests.boxq_families import ENTRIES, check_entry, problem
    from tests.boxq_util import run_boxq
    for k, name in enumerate(ENTRIES):
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        try:
            plan = check_entry(name)
            out = run_boxq(problem(name, 2, 400 + k))
            rec = {kk: np.asarray(v) for kk, v in out.items() if kk not in ("grads", "trace") and v is not None}
            rec.update({"grad_" + kk: np.asarray(v) for kk, v in out["grads"].items() if v is not None})
            if plan.ok:
                pt = point(plan, 2, 3)
                rec["jvp_dz"] = run_jvp(plan, pt, tangents(plan, 2, 4))[0]
                rec["kkt_dx"] = run_kkt(plan, kkt_inputs(plan, 2, 5))[0]
            np.savez(os.path.join(out_dir, name + ".npz"), **rec)
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next entry still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


if __name__ == "__main__":
    main(sys.argv[1])
