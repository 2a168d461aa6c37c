"""qpth_b200 — H100-native batched differentiable QP layer (drop-in for qpth.qp.QPFunction)."""
from .qp import KKTSolvers, QPFunction, QPSolvers   # noqa: F401
from .solution import QPSolutionFunction, cvxpy_forward   # noqa: F401
from .box import BoxQPFunction   # noqa: F401

__version__ = "0.1.0"


def install_as_qpth():
    """Make `from qpth.qp import QPFunction, QPSolvers` resolve to this package.

    For callers (OptNet layers) that import the reference by name and should not be edited.
    """
    import sys
    import types
    from . import qp as _qp, util as _util
    pkg = types.ModuleType("qpth")
    pkg.qp = _qp
    pkg.util = _util
    pkg.__path__ = []
    sys.modules["qpth"] = pkg
    sys.modules["qpth.qp"] = _qp
    sys.modules["qpth.util"] = _util
    return pkg
