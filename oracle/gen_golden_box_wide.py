"""Generate tests/golden/box_wide*.npz by running the REAL reference on the dense equivalents of
`oracle.box_wide_cases.WIDE_BOX_CASES` (where the reference checkout is present):  python -m oracle.gen_golden_box_wide

At these sizes the reference's dense gradients are mostly structural zeros (dQ off its diagonal, dG), so a fixture keeps
only what the box gradients are made of: the diagonal of dQ (dq), dp, dh, db, and dA as the projection dA @ v with
v_k = cos(k + 1) (dA_proj), next to z*, lam, slacks and nus."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_runner                             # noqa: E402
from oracle.box_cases import dense_problem                # noqa: E402
from oracle.box_wide_cases import WIDE_BOX_CASES          # noqa: E402
from oracle.cases import checksum, proj                   # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def main():
    for name, build in WIDE_BOX_CASES.items():
        prob = dense_problem(build())
        r = ref_runner.run_reference(prob)
        d = ref_runner.run_reference_duals(prob)
        out = dict(input_checksum=checksum(prob), zhat=r["zhat"], lam=d["lam"], slacks=d["slacks"], nus=d["nus"],
                   dq=np.diagonal(r["dQ"], axis1=-2, axis2=-1).copy(), dp=r["dp"], dh=r["dh"], db=r["db"],
                   dA_proj=r["dA"] @ proj(r["dA"].shape[-1]))
        # The reference's OWN reproducibility, as gen_golden.py records it for the sweep cases: every input entry
        # perturbed by 1e-15 relative (seeded); sens_<key> is the largest relative change of that output (per row
        # norm, as tests/parity.py measures errors).
        rs = np.random.RandomState(12345)
        pp = dict(prob)
        for k in ("Q", "p", "G", "h", "A", "b"):
            v = np.asarray(prob[k], dtype=np.float64)
            pp[k] = v * (1.0 + 1e-15 * rs.randn(*v.shape)) if v.size else v
        pp["Q"] = 0.5 * (pp["Q"] + np.swapaxes(pp["Q"], -1, -2))
        r2 = ref_runner.run_reference(pp)
        alt = dict(zhat=r2["zhat"], dq=np.diagonal(r2["dQ"], axis1=-2, axis2=-1), dp=r2["dp"], dh=r2["dh"],
                   db=r2["db"], dA_proj=r2["dA"] @ proj(r2["dA"].shape[-1]))
        for k, v in alt.items():
            a, b = np.atleast_2d(v), np.atleast_2d(out[k])
            nb = np.linalg.norm(b, axis=1)
            out["sens_" + k] = float((np.linalg.norm(a - b, axis=1) / np.maximum(nb, 1e-4 * nb.max())).max())
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
