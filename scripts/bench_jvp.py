"""The cost of forward mode: forward + JVP (torch.autograd.forward_ad, a tangent on every input) against forward +
backward (a loss on z, lam and nu), both with duals=True, and the right-hand-side kernel alone. One JSON line per
workload on stdout.

    python scripts/bench_jvp.py [--steps 50] [--pairs 7]

Workloads: C2 (QPFunction, B = 128, nz = nineq = 100, no equality rows, batched tangents of Q, p, G, h) and the box
sudoku layer of scripts/bench_duals.py (BoxQPFunction, nz = 64, neq = 40, lb only, B = 1024, batched tangents of every
input, dA included). The two variants solve the same problems and alternate in one process (`pairs` pairs of
`steps`-step windows, CUDA events, median window). The right-hand-side kernel is timed as qpb200_jvp (or
qpb200_box_jvp) minus the backward-with-duals call it makes, both on the solved state, and its achieved bandwidth is
the algorithmic bytes (tangents read once, z / lam / nu, the right-hand side written) over that time, against the
H100 SXM's 3.35 TB/s. Each line carries the GPU name and power limit. Nothing is written to the tree.
"""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402
import torch         # noqa: E402
import torch.autograd.forward_ad as fwAD   # noqa: E402

from scripts.bench_duals import gpu_info   # noqa: E402

PEAK = 3.35e12


def workloads(dev):
    from qpth_b200 import BoxQPFunction, QPFunction
    from qpth_b200.problems import random_qp_batch
    f64 = dict(dtype=torch.float64, device=dev)
    pr = random_qp_batch(128, 100, 100, 0, seed=2)
    c2 = {k: torch.tensor(pr[k], **f64) for k in ("Q", "p", "G", "h")}
    e = torch.Tensor().to(dev).double()
    fq = QPFunction(verbose=-1, check_Q_spd=False, duals=True)
    rs = np.random.RandomState(31)
    A_ = rs.randn(40, 64)
    sud = {"q": torch.full((1024, 64), 0.1, **f64), "p": torch.tensor(-rs.rand(1024, 64), **f64),
           "A": torch.tensor(A_, **f64).expand(1024, 40, 64).contiguous(),
           "b": torch.tensor(A_ @ (rs.rand(64) + 0.1), **f64).expand(1024, 40).contiguous(),
           "lb": torch.zeros(1024, 64, **f64)}
    fb = BoxQPFunction(verbose=-1, check_Q_spd=False, duals=True)
    return [("c2_128x100x100", c2, lambda x: fq(x["Q"], x["p"], x["G"], x["h"], e, e), fq),
            ("box_sudoku_1024x64x40_lb", sud, lambda x: fb(x["q"], x["p"], x["A"], x["b"], x["lb"], None), fb)]


def rhs_kernel(f, ins, tan, steps):
    """(ms of the right-hand-side kernel, algorithmic bytes) from the solved state of f's last forward."""
    from qpth_b200 import _lib
    from qpth_b200.qp import _ptr, _stream
    lib = _lib.load()
    st = f.last_solve()
    plan, B = st.plan, st.nBatch
    f64 = dict(dtype=torch.float64, device=st.zhat.device)
    box = hasattr(st, "q")
    nz, m, e = plan.nz, plan.nineq, plan.neq
    rhs = torch.empty(B * (nz + m + e), **f64)
    dz, dlam = torch.empty(B, nz, **f64), torch.empty(B, m, **f64)
    dnu = torch.empty(B, e, **f64) if e else None
    names = ("q", "p", "A", "b", "lb", "ub") if box else ("Q", "p", "G", "h", "A", "b")
    t = [tan.get(k) for k in names]
    per = [x[0].numel() if x is not None else 0 for x in t]
    args = []
    for x, s in zip(t, per):
        args += [_ptr(x), s]
    nbytes = sum(x.numel() * 8 for x in t if x is not None) + 8 * B * (2 * (nz + m + e))
    if box:
        jvp = lambda: lib.qpb200_box_jvp(ctypes.byref(plan), B, _ptr(st.q), st.sq, _ptr(st.A), st.sA, *args,
                                         _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(rhs),
                                         _ptr(dz), _ptr(dlam), _ptr(dnu), _stream())
        rx, rz, ry = rhs[:B * nz], rhs[B * nz:B * (nz + m)], rhs[B * (nz + m):]
        bwd = lambda: lib.qpb200_box_backward_duals(ctypes.byref(plan), B, _ptr(st.q), st.sq, _ptr(st.A), st.sA,
                                                    _ptr(rx), _ptr(rz), _ptr(ry), _ptr(st.zhat), _ptr(st.lam),
                                                    _ptr(st.slacks), _ptr(st.nus), *([None, 0] * 6), _ptr(dz),
                                                    _ptr(dlam), _ptr(dnu), _stream())
    else:
        sF = 1 if st.nsys > 1 else 0
        jvp = lambda: lib.qpb200_jvp(ctypes.byref(plan), B, *args, _ptr(st.zhat), _ptr(st.lam), _ptr(st.slacks),
                                     _ptr(st.nus), _ptr(st.L), _ptr(st.W), _ptr(st.K), sF, _ptr(rhs), _ptr(dz),
                                     _ptr(dlam), _ptr(dnu), _ptr(st.scratch), _stream())
        rx, rz = rhs[:B * nz], rhs[B * nz:B * (nz + m)]
        bwd = lambda: lib.qpb200_backward_duals(ctypes.byref(plan), B, _ptr(rx), _ptr(rz), None, _ptr(st.zhat),
                                                _ptr(st.lam), _ptr(st.slacks), _ptr(st.nus), _ptr(st.L), _ptr(st.W),
                                                _ptr(st.K), sF, *([None, 0] * 6), _ptr(dz), _ptr(dlam), _ptr(dnu),
                                                _ptr(st.scratch), _stream())

    def window(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            _lib.check(fn())
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    window(jvp), window(bwd)
    tj, tb = [], []
    for _ in range(5):
        tj.append(window(jvp))
        tb.append(window(bwd))
    return float(np.median(tj)) - float(np.median(tb)), float(np.median(tj)), float(np.median(tb)), nbytes


def measure(name, ins, fwd, f, steps, pairs, dev):
    rs = np.random.RandomState(5)
    tan = {k: torch.tensor(rs.randn(*v.shape), dtype=torch.float64, device=dev) for k, v in ins.items()}
    x = {k: v.clone().requires_grad_(True) for k, v in ins.items()}
    outs = fwd(x)
    adj = [torch.tensor(rs.randn(*o.shape), dtype=torch.float64, device=dev) for o in outs]

    def once(jvp):
        if jvp:
            with fwAD.dual_level():
                outs = fwd({k: fwAD.make_dual(v, tan[k]) for k, v in ins.items()})
                [fwAD.unpack_dual(o).tangent for o in outs]
        else:
            for v in x.values():
                v.grad = None
            sum((o * a).sum() for o, a in zip(fwd(x), adj)).backward()

    def window(jvp):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            once(jvp)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    for j in (False, True):
        for _ in range(3):
            once(j)
    torch.cuda.synchronize()
    tb, tj = [], []
    for _ in range(pairs):
        tb.append(window(False))
        tj.append(window(True))
    fwd(ins)                                             # the solved state rhs_kernel reads
    rhs_ms, jvp_ms, bwd_ms, nbytes = rhs_kernel(f, ins, tan, steps)
    return dict(workload=name, ms_fwd_bwd=float(np.median(tb)), ms_fwd_jvp=float(np.median(tj)),
                ratio=float(np.median(tj) / np.median(tb)), windows_fwd_bwd=tb, windows_fwd_jvp=tj,
                ms_jvp_call=jvp_ms, ms_solve_call=bwd_ms, ms_rhs_kernel=rhs_ms, rhs_bytes=nbytes,
                rhs_bytes_per_s=nbytes / (rhs_ms * 1e-3) if rhs_ms > 0 else None,
                rhs_fraction_of_3_35_TBps=(nbytes / (rhs_ms * 1e-3)) / PEAK if rhs_ms > 0 else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--pairs", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jvp: no CUDA device (there is no CPU fallback)")
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    for wl, ins, fwd, f in workloads(dev):
        rec = measure(wl, ins, fwd, f, a.steps, a.pairs, dev)
        rec.update(gpu=name, power_limit=power, steps=a.steps, pairs=a.pairs)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
