"""Local memory of the box-QP kernels (BoxQPFunction, with a diagonal or a dense Q).

The forward, backward and KKT kernels of every layout are instances of one set of templates (csrc/qp_box_loop.cuh), so
a change to the shared loop or to one family's phases can move another family's register allocation. This compiles
both box units as build.py does, with `-Xptxas -v`, and checks that no kernel has a larger stack frame or more spill
bytes than recorded below (nvcc 12.9, sm_90a). A spill there lands on a Newton iteration's critical path. About 20 s;
skipped where nvcc is missing."""
import os
import re
import subprocess
import tempfile

import pytest

from tests.test_local_memory_cpu import _nvcc, parse_ptxas

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# kernel (a pattern of its mangled name) -> (stack frame, spill stores, spill loads) in bytes, at most
LIMITS = {
    r"k_box_forwardINS_6OneCta": (208, 60, 68),
    r"k_box_forwardINS_7Cluster": (368, 0, 0),
    r"k_box_forward_dm": (400, 0, 0),
    r"k_box_forwardINS_6DenseQ": (144, 128, 324),
    r"k_box_backwardINS_6OneCta": (168, 0, 0),
    r"k_box_backwardINS_7Cluster": (368, 0, 0),
    r"k_box_backward_dm": (400, 0, 0),
    r"k_box_backwardINS_6DenseQ": (0, 0, 0),
    r"k_box_kktINS_6OneCta": (168, 0, 0),
    r"k_box_kktINS_7Cluster": (368, 0, 0),
    r"k_box_kkt_dm": (400, 0, 0),
    r"k_box_kktINS_6DenseQ": (0, 0, 0),
}


@pytest.fixture(scope="module")
def report():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    from qpth_b200 import build
    units = [u for u in build.UNITS if u[0] in ("qp_box.cu", "qp_boxq.cu")]
    assert len(units) == 2, build.UNITS
    rep = {}
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        for src, defs, tag in units:
            cmd = ([nvcc] + build.GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
                   + defs + ["-c", "-o", os.path.join(tmp, tag + ".o"), os.path.join(ROOT, "qpth_b200", "csrc", src)])
            procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
        for pr in procs:
            _, err = pr.communicate()
            assert pr.returncode == 0, err[-4000:]
            rep.update(parse_ptxas(err))
    assert rep
    return rep


@pytest.mark.parametrize("kernel", sorted(LIMITS))
def test_box_kernel_local_memory(report, kernel):
    found = {k: v for k, v in report.items() if re.search(kernel, k)}
    assert len(found) == 1, "%r matches %s" % (kernel, sorted(k for k in report if "k_box" in k))
    (entry, funcs), = found.items()
    assert funcs and funcs[0][0] == entry
    stack, st, ld = LIMITS[kernel]
    assert funcs[0][1] <= stack and funcs[0][2] <= st and funcs[0][3] <= ld, \
        "%s: (stack, spill stores, spill loads) = %s, at most %s" % (entry, funcs[0][1:], LIMITS[kernel])


def test_every_box_kernel_has_a_limit(report):
    kernels = [k for k in report if re.search(r"k_box_(forward|backward|kkt)", k)]
    assert len(kernels) == len(LIMITS), sorted(kernels)
