"""Child process of tests/test_gpu_box_cluster.py: the first runs of the box-QP cluster kernels (forward, backward, KKT
solve) on cuda:0 for every cluster size, so that a fault in them is reported as a failed test instead of ending the
suite. Writes <out_dir>/<job>.npz (or .err).  Usage: python -m tests.box_cluster_child <out_dir>"""
import ctypes
import os
import sys
import traceback

import numpy as np


def jobs():
    from tests.box_util import random_box
    for C in (2, 4, 8):
        yield "forced_%d" % C, str(C), random_box(11, 3, 31, 13, "both")
    yield "wide", None, random_box(12, 2, 600, 64, "both")


def _kkt(n, e, C):
    """one qpb200_box_solve_kkt on the plan the knob gives"""
    import torch
    from qpth_b200 import _lib
    plan = _lib.box_plan_for(n, e, True, True)
    assert plan.cl_ctas == C, (plan.cl_ctas, C)
    rs = np.random.RandomState(3)
    B, m = 2, plan.nineq
    ins = [torch.tensor(v, dtype=torch.float64, device="cuda:0").contiguous()
           for v in (0.1 + rs.rand(B, n), rs.randn(B, e, n), 0.5 + rs.rand(B, m), rs.randn(B, n), rs.randn(B, m),
                     rs.randn(B, m), rs.randn(B, e))]
    out = [torch.empty(B, k, dtype=torch.float64, device="cuda:0") for k in (n, m, m, e)]

    def ptr(t):
        return ctypes.c_void_p(t.data_ptr())
    _lib.check(_lib.load().qpb200_box_solve_kkt(ctypes.byref(plan), B, ptr(ins[0]), n, ptr(ins[1]), e * n,
                                                *(ptr(v) for v in ins[2:]), *(ptr(o) for o in out), ctypes.c_void_p(0)))
    return out[0].cpu().numpy()


def main(out_dir):
    from tests.box_util import run_box
    for name, knob, bx in jobs():
        try:
            if knob is None:
                os.environ.pop("QPB200_BOX_CLUSTER", None)
            else:
                os.environ["QPB200_BOX_CLUSTER"] = knob
            out = run_box(bx)
            rec = {k: np.asarray(v) for k, v in out.items() if k not in ("grads", "trace") and v is not None}
            rec.update({"grad_" + k: np.asarray(v) for k, v in out["grads"].items() if v is not None})
            if knob is not None:
                rec["kkt_dx"] = _kkt(31, 13, int(knob))
            np.savez(os.path.join(out_dir, name + ".npz"), **rec)
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


if __name__ == "__main__":
    main(sys.argv[1])
