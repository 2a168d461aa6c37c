"""Child process of tests/test_gpu_boxq.py: the first runs of the dense-Q box kernels (forward, backward) on cuda:0, so
that a fault in them is reported as a failed test instead of ending the suite. Writes <out_dir>/<job>.npz (or .err).
Usage: python -m tests.boxq_child <out_dir>"""
import os
import sys
import traceback

import numpy as np


def jobs():
    from tests.boxq_util import random_boxq
    yield "portfolio", ("golden", "boxq_portfolio")
    for sides in ("lb", "ub", "both"):
        for e in (0, 13):
            yield "first_%s_%d" % (sides, e), ("random", random_boxq(11, 3, 21, e, sides))


def main(out_dir):
    from tests.boxq_util import load_boxq_case, run_boxq
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    for name, (kind, payload) in jobs():
        try:
            bx = load_boxq_case(payload, golden)[0] if kind == "golden" else payload
            out = run_boxq(bx)
            rec = {k: np.asarray(v) for k, v in out.items() if k not in ("grads", "trace") and v is not None}
            rec.update({"grad_" + k: np.asarray(v) for k, v in out["grads"].items() if v is not None})
            np.savez(os.path.join(out_dir, name + ".npz"), **rec)
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


if __name__ == "__main__":
    main(sys.argv[1])
