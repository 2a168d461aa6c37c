"""Child process of tests/test_gpu_box_dm.py: the first runs of the distributed-M box kernels (forward, backward, KKT
solve) on cuda:0 for every cluster size, so that a fault in them is reported as a failed test instead of ending the
suite. Writes <out_dir>/<job>.npz (or .err).  Usage: python -m tests.box_dm_child <out_dir>"""
import os
import sys
import traceback

import numpy as np


def jobs():
    from oracle.box_sudoku_cases import sudoku9_problem
    from tests.box_util import random_box
    for C in (2, 4, 8):
        yield "forced_%d" % C, str(C), random_box(21, 2, 160, 136, "both")
    yield "sudoku9", None, sudoku9_problem()


def main(out_dir):
    from tests.box_cluster_child import _kkt
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
                rec["kkt_dx"] = _kkt(160, 136, int(knob))
            np.savez(os.path.join(out_dir, name + ".npz"), **rec)
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


if __name__ == "__main__":
    main(sys.argv[1])
