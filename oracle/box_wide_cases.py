"""Golden-case recipes of box QPs too large for one CTA's shared memory: the thread block cluster kernels of
csrc/qp_box.cu solve them (TEST INFRASTRUCTURE ONLY). Kept apart from `oracle.box_cases.BOX_CASES`, whose golden test
asserts that the one-CTA kernels cover every case. Fixtures: tests/golden/<name>.npz, written by
`python -m oracle.gen_golden_box_wide` from the real reference on the dense equivalent (`box_cases.dense_problem`)."""
import numpy as np

from oracle.box_cases import _box


def wide_problem():
    """nz = 600, neq = 64, both sides (lb in [-1, 0], ub in [0.5, 1.5], q in [0.2, 1.2]), batched A, B = 2."""
    rs = np.random.RandomState(45)
    n = 600
    return _box(45, B=2, n=n, e=64, lb=-rs.rand(n), ub=0.5 + rs.rand(n), q=0.2 + rs.rand(n))


WIDE_BOX_CASES = {
    "box_wide": wide_problem,
}
