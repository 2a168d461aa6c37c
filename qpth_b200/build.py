"""Build libqpth_b200.so in-tree with nvcc for sm_90a, H100 (`python -m qpth_b200.build`)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
import glob  # noqa: E402

DEPS = sorted(glob.glob(os.path.join(HERE, "csrc", "*"))) + [os.path.join(os.path.dirname(HERE), "include", "qpth_b200.h"),
                                                            os.path.abspath(__file__)]     # (a flag change rebuilds)
OUT = os.path.join(HERE, "libqpth_b200.so")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(d) <= t for d in DEPS)


# (source, extra defines, object suffix): the 256-thread build of every kernel + the 192- and 512-thread builds of the
# product-form solve kernels (three QPs per SM; large orders) + the 128-thread box-QP kernels (BoxQPFunction)
UNITS = [("qp_kernels.cu", [], "main"),
         ("qp_alt.cu", ["-DQPB_NT=192", "-DQPB_ALT_CTAS=3"], "alt192"),
         ("qp_alt.cu", ["-DQPB_NT=512", "-DQPB_ALT_CTAS=1"], "alt512"),
         ("qp_box.cu", ["-DQPB_NT=128"], "box")]


def build(force=False, verbose=False, extra=(), out=None):
    """Compile the translation units in parallel and link them into one shared library."""
    out = out or OUT
    if not force and out == OUT and up_to_date():
        return out
    import hashlib
    import tempfile
    objdir = os.path.join(tempfile.gettempdir(), "qpth_b200_obj_" + hashlib.sha1(out.encode()).hexdigest()[:10])
    os.makedirs(objdir, exist_ok=True)
    base = [nvcc_path()] + GENCODE + ["-O3", "-lineinfo", "-std=c++17",
                             "-Xcompiler", "-fPIC"] + list(extra)
    if verbose:
        base.insert(1, "-Xptxas=-v")
    procs, objs = [], []
    for src, defs, tag in UNITS:
        obj = os.path.join(objdir, tag + ".o")
        cmd = base + defs + ["-c", "-o", obj, os.path.join(HERE, "csrc", src)]
        if verbose:
            print(" ".join(cmd))
        procs.append((cmd, subprocess.Popen(cmd)))
        objs.append(obj)
    for cmd, pr in procs:
        if pr.wait() != 0:
            raise subprocess.CalledProcessError(pr.returncode, cmd)
    subprocess.check_call([nvcc_path()] + GENCODE + ["-shared", "-o", out] + objs)
    return out


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print("built", OUT)
