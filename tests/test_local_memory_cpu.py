"""Local memory of the three-per-SM kernels (the 192-thread build that throughput mode runs).

Three QPs per SM leave 28 KB of L1 per SM (the rest is the shared-memory carveout), so local memory there goes to L2,
and a spill reload or a register restore after a call sits on the critical path of a Newton-iteration phase. This
compiles the 192-thread unit with `-Xptxas -v` and checks what ptxas reports for each kernel and for the subroutines it
compiled under it: the backward and solve_kkt kernels use no local memory at all; in the forward kernel the block
substitutions (run three times per Newton iteration, 13 block steps each) and the block reductions use none, and the
stack frame stays at most 96 B (368 B before the substitutions stopped carrying their next P row across the step
barrier and the reductions took their values in registers). About 10 s; skipped where nvcc is missing."""
import os
import re
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "qpth_b200", "csrc", "qp_alt.cu")


def _nvcc():
    from qpth_b200 import build
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


def parse_ptxas(text):
    """ptxas -v output -> {entry (mangled): [(function, stack, spill stores, spill loads), ...]}. The first tuple is
    the entry itself; the others are the subroutines ptxas compiled for it."""
    out, entry, fn = {}, None, None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
            out[entry] = []
            continue
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and entry is not None and fn is not None:
            out[entry].append((fn, int(m.group(1)), int(m.group(2)), int(m.group(3))))
            fn = None
    return out


@pytest.fixture(scope="module")
def report():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-DQPB_NT=192", "-DQPB_ALT_CTAS=3", "-c", "-o", os.path.join(tmp, "alt192.o"), SRC],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    rep = parse_ptxas(r.stderr)
    assert rep, r.stderr[-4000:]
    return rep


def _entries(rep, pattern):
    found = {k: v for k, v in rep.items() if re.search(pattern, k)}
    assert found, "no kernel matches %r among %s" % (pattern, sorted(rep))
    return found


def _local_memory(funcs):
    return [f for f in funcs if f[1] or f[2] or f[3]]


def test_parse_ptxas():
    text = ("ptxas info    : Compiling entry function '_Z1kv' for 'sm_90a'\n"
            "ptxas info    : Function properties for _Z1kv\n"
            "    8 bytes stack frame, 0 bytes spill stores, 4 bytes spill loads\n"
            "ptxas info    : Function properties for _Z1fv\n"
            "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    assert parse_ptxas(text) == {"_Z1kv": [("_Z1kv", 8, 0, 4), ("_Z1fv", 0, 0, 0)]}


@pytest.mark.parametrize("kernel", [
    r"k_kkt_fastILb1ELb1ELb1ELi3ELb0E",              # k_kkt_fast<true, ...>: the backward
    r"k_kkt_fastILb0ELb1ELb1ELi3ELb0E",              # k_kkt_fast<false, ...>: solve_kkt
])
def test_three_per_sm_kkt_kernels_have_no_local_memory(report, kernel):
    for entry, funcs in _entries(report, kernel).items():
        assert funcs and funcs[0][0] == entry
        assert _local_memory(funcs) == [], "%s: (function, stack, spill stores, spill loads)" % entry


def test_three_per_sm_forward_local_memory(report):
    for entry, funcs in _entries(report, r"k_forward_fastILb1ELb1ELi3ELb0E").items():
        assert funcs and funcs[0][0] == entry
        assert funcs[0][1] <= 96, funcs[0]
        names = [f[0] for f in funcs]
        for sub in ("pf_fwd", "pf_bwd", "f_reduce"):
            assert any(sub in nm for nm in names), (sub, names)       # (still compiled as subroutines)
        hot = [f for f in _local_memory(funcs) if any(sub in f[0] for sub in ("pf_fwd", "pf_bwd", "pf_diag", "f_reduce"))]
        assert hot == [], hot
