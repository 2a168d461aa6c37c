"""Child process of tests/test_gpu_box_edges.py: the first forward, backward and qpb200_box_solve_kkt of every edge entry
of tests/box_families.py on cuda:0. Several sit on the last byte of shared memory, where a layout error would fault; in
a child process such a fault fails only their own tests instead of ending the suite. Each entry's plan is asserted
(check_entry) before it runs. Writes <out_dir>/<entry>.npz (or .err), and each entry's name to
<out_dir>/progress.txt as it starts.  Usage: python -m tests.box_edges_child <out_dir>"""
import ctypes
import os
import sys
import traceback

import numpy as np


def kkt_inputs(plan, B, seed, lo=-8.0, hi=8.0):
    """(q, A, d, rx, rs, rz, ry) of B random KKT systems of a box plan, d = 10^U(lo, hi)"""
    rs = np.random.RandomState(seed)
    n, e, m = plan.nz, plan.neq, plan.nineq
    return (0.1 + rs.rand(B, n), rs.randn(B, e, n), 10.0 ** rs.uniform(lo, hi, (B, m)), rs.randn(B, n), rs.randn(B, m),
            rs.randn(B, m), rs.randn(B, e))


def run_kkt(plan, ins):
    """one qpb200_box_solve_kkt on cuda:0: (dx, ds, dz, dy) as numpy arrays"""
    import torch
    from qpth_b200 import _lib
    B = ins[0].shape[0]
    n, e, m = plan.nz, plan.neq, plan.nineq
    t = [torch.tensor(v, dtype=torch.float64, device="cuda:0").contiguous() for v in ins]
    out = [torch.empty(B, k, dtype=torch.float64, device="cuda:0") for k in (n, m, m, e)]

    def ptr(v):
        return ctypes.c_void_p(v.data_ptr()) if v.numel() else ctypes.c_void_p(0)
    _lib.check(_lib.load().qpb200_box_solve_kkt(ctypes.byref(plan), B, ptr(t[0]), n, ptr(t[1]), e * n,
                                                *(ptr(v) for v in t[2:]), *(ptr(o) for o in out), ctypes.c_void_p(0)))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def main(out_dir):
    from tests.box_families import ENTRIES, check_entry, edges, knob, layout
    from tests.box_util import random_box, run_box
    for k, name in enumerate(edges()):
        ent = ENTRIES[name]
        n, e, sides = ent["shape"]
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        try:
            with knob(ent["knob"]):
                plan = check_entry(name)
                out = run_box(random_box(400 + k, 2, n, e, sides))
                rec = {kk: np.asarray(v) for kk, v in out.items() if kk not in ("grads", "trace") and v is not None}
                rec.update({"grad_" + kk: np.asarray(v) for kk, v in out["grads"].items() if v is not None})
                if layout(plan) != "dense":
                    rec["kkt_dx"] = run_kkt(plan, kkt_inputs(plan, 2, 3))[0]
            np.savez(os.path.join(out_dir, name + ".npz"), **rec)
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next entry still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


if __name__ == "__main__":
    main(sys.argv[1])
