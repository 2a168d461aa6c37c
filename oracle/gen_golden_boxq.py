"""Generate the dense-Q box-QP fixtures tests/golden/boxq_*.npz by running the REAL reference on the dense equivalents
of `oracle.boxq_cases.BOXQ_CASES` (where the reference checkout is present):  python -m oracle.gen_golden_boxq"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.boxq_cases import BOXQ_CASES, dense_problem     # noqa: E402
from oracle.gen_golden import save                          # noqa: E402


def main():
    for name, build in BOXQ_CASES.items():
        save(name, dense_problem(build()))


if __name__ == "__main__":
    main()
