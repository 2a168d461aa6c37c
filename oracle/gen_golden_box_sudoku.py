"""Generate tests/golden/box_sudoku9*.npz by running the REAL reference on the dense equivalents of
`oracle.box_sudoku_cases.SUDOKU_BOX_CASES` (where the reference checkout is present):  python -m oracle.gen_golden_box_sudoku

Stored as gen_golden_box_wide.py stores box_wide: z*, lam, slacks, nus, the diagonal of dQ (dq), dp, dh, db, dA as the
projection dA @ v with v_k = cos(k + 1), and the reference's own sensitivity to a 1e-15 perturbation (sens_*)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_runner                             # noqa: E402
from oracle.box_cases import dense_problem                # noqa: E402
from oracle.box_sudoku_cases import SUDOKU_BOX_CASES      # noqa: E402
from oracle.cases import checksum, proj                   # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
KEYS = ("zhat", "dq", "dp", "dh", "db", "dA_proj")


def _outputs(prob):
    r = ref_runner.run_reference(prob)
    return r, dict(zhat=r["zhat"], dq=np.diagonal(r["dQ"], axis1=-2, axis2=-1).copy(), dp=r["dp"], dh=r["dh"],
                   db=r["db"], dA_proj=r["dA"] @ proj(r["dA"].shape[-1]))


def main():
    for name, build in SUDOKU_BOX_CASES.items():
        prob = dense_problem(build())
        _, out = _outputs(prob)
        d = ref_runner.run_reference_duals(prob)
        out.update(input_checksum=checksum(prob), lam=d["lam"], slacks=d["slacks"], nus=d["nus"])
        rs = np.random.RandomState(12345)
        pp = dict(prob)
        for k in ("Q", "p", "G", "h", "A", "b"):
            v = np.asarray(prob[k], dtype=np.float64)
            pp[k] = v * (1.0 + 1e-15 * rs.randn(*v.shape)) if v.size else v
        pp["Q"] = 0.5 * (pp["Q"] + np.swapaxes(pp["Q"], -1, -2))
        _, alt = _outputs(pp)
        for k in KEYS:
            a, b = np.atleast_2d(alt[k]), np.atleast_2d(out[k])
            nb = np.linalg.norm(b, axis=1)
            out["sens_" + k] = float((np.linalg.norm(a - b, axis=1) / np.maximum(nb, 1e-4 * nb.max())).max())
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path), "bytes", {k: out["sens_" + k] for k in KEYS})


if __name__ == "__main__":
    main()
