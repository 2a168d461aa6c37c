"""Generate the box-QP fixtures tests/golden/box_*.npz by running the REAL reference on the dense equivalents of
`oracle.box_cases.BOX_CASES` (where the reference checkout is present):  python -m oracle.gen_golden_box"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.box_cases import BOX_CASES, dense_problem     # noqa: E402
from oracle.gen_golden import save                        # noqa: E402


def main():
    for name, build in BOX_CASES.items():
        if name.startswith("box_"):
            save(name, dense_problem(build()))


if __name__ == "__main__":
    main()
