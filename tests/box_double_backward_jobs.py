"""GPU jobs of tests/test_gpu_box_double_backward.py, run in one child process with a timeout (qpb200_box_double_backward
and qpb200_boxq_double_backward are new to the device). Each job writes <name>.npz, or <name>.err with its traceback;
progress.txt lists the jobs started.

- `entry` / `boxq`: a box-family (dense-Q family) entry at the point of tests/box_jacobian_jobs.point, in three sharings
  (every input batched; q and A shared; p, b, lb, ub shared): the first backward's solve v and the double backward of
  random cotangents, and the JVP with the cotangents as tangents (w / B for a shared input).
- `dense`: a family entry no box kernel runs, through BoxQPFunction under create_graph (the dense fallback).
- `hess`: the p-Hessian of a scalar of z(p) by torch.autograd.functional.hessian over a batch.
- `jtj`: on a strictly complementary batch, the p-Hessian of 1/2 ||z||^2 and J'J from f.jacobian().
- `cd`: central differences of the first-order gradients along directions of q, p, A, b, lb, ub, the first order
  with and without create_graph, and gradgradcheck on a small shape.
- `roundtrip`: fp32 and CPU inputs.
"""
import os
import sys
import traceback

import numpy as np
import torch

from tests.box_jacobian_jobs import point, state

DEV = "cuda:0"
ENTRY_NAMES = ("one_mid_lb", "one_mid_both", "one_mid_ub", "one_full", "one_neq120", "one_wide", "cl2_mid_forced",
               "cl2_mid", "cl2_mid_lb", "cl2_past_one_wide", "cl2_past_one_neq", "cl2_full", "cl4_mid_forced",
               "cl4_mid", "cl4_mid_480", "cl4_mid_lb", "cl4_full", "cl8_mid_forced", "cl8_mid", "cl8_mid_box",
               "cl8_full", "cl8_widest", "cl8_widest_lb", "cl8_empty_9", "cl8_empty_5", "dm2_mid_forced",
               "dm2_boundary", "dm2_full", "dm4_mid_forced", "dm4_mid", "dm4_sudoku", "dm4_full", "dm8_mid_forced",
               "dm8_full", "dm8_slice")
DENSE_NAMES = ("dense_mid", "dense_boundary")
SHARINGS = {"batched": (), "shared_qA": ("q", "A"), "shared_pbs": ("p", "b", "lb", "ub")}
NAMES = ("q", "p", "A", "b", "lb", "ub")


def _T(a):
    return torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=DEV)


def _c(t):
    return np.zeros(0) if t is None else t.detach().cpu().numpy()


def omegas(plan, shared, seed, dense_Q=False, B=3):
    """random cotangents {name: array or None}, un-batched for the names in `shared`"""
    rs = np.random.RandomState(seed)
    n, e = plan.nz, plan.neq
    shp = dict(q=(n, n) if dense_Q else (n,), p=(n,), A=(e, n), b=(e,), lb=(n,), ub=(n,))
    absent = dict(A=e == 0, b=e == 0, lb=not plan.has_lb, ub=not plan.has_ub)
    return {k: None if absent.get(k) else rs.randn(*(shp[k] if k in shared else (B,) + shp[k])) for k in NAMES}


def point_job(plan, dense_Q):
    from qpth_b200 import box
    pt = point(plan, 11, dense_Q)
    e = plan.neq
    out = dict(q=pt["q"], A=pt["A"], z=pt["z"], nu=pt["nu"], lam=pt["lam"], s=pt["s"], dl=pt["dl"],
               glam=pt["glam"], gnu=pt["gnu"])
    for tag, shared in SHARINGS.items():
        st = state(plan, pt, "q" in shared, dense_Q)
        flags = tuple(k in shared for k in NAMES)
        om = omegas(plan, shared, 17, dense_Q)
        _, v = box.solve_box_backward(st, _T(pt["dl"]), flags, (False,) * 6, _T(pt["glam"]),
                                      _T(pt["gnu"]) if e else None, keep=True)
        res = box.solve_box_double_backward(st, v, [None if om[k] is None else _T(om[k]) for k in NAMES], flags,
                                            (True,) * 6)
        B = st.nBatch
        # w / B divided on the device, as solve_box_double_backward divides it
        jv = box.solve_box_jvp(st, [None if om[k] is None else (_T(om[k]) / B if k in shared else _T(om[k]))
                                    for k in NAMES])
        torch.cuda.synchronize()
        for k, x in zip(("vx", "vlam", "vnu"), v):
            out[tag + "_" + k] = _c(x)
        for k, x in zip(("gz", "glam", "gnu") + NAMES, res):
            out[tag + "_" + k] = _c(x)
        for k, x in zip(("jz", "jlam", "jnu"), jv):
            out[tag + "_" + k] = _c(x)
        for k in NAMES:
            out[tag + "_om_" + k] = np.zeros(0) if om[k] is None else om[k]
    return out


def entry_job(name):
    from tests.box_families import ENTRIES, check_entry, knob
    with knob(ENTRIES[name]["knob"]):
        return point_job(check_entry(name), False)


def boxq_entry_job(name):
    from tests.boxq_families import check_entry
    return point_job(check_entry(name), True)


def _problem(n, e, sides, seed, dense_Q=False, B=3):
    from tests.box_jacobian_jobs import _problem as pr
    return pr(n, e, sides, seed, dense_Q, B)


def _leaves(pr, e, dtype=torch.float64, device=DEV):
    T = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=dtype, device=device).requires_grad_(True)
    E = torch.empty(0, dtype=dtype, device=device)
    return dict(q=T(pr["q"]), p=T(pr["p"]), A=T(pr["A"]) if e else E, b=T(pr["b"]) if e else E,
                lb=None if pr["lb"] is None else T(pr["lb"]), ub=None if pr["ub"] is None else T(pr["ub"]))


def _second_order(f, L, gz, glam, gnu, om):
    """g1 = grad(<gz, z> + <glam, lam> + <gnu, nu>) under create_graph, then grad(sum <om, g1>)"""
    z, lam, nu = f(*(L[k] for k in NAMES))
    loss = (gz * z).sum() + (glam * lam).sum() + ((gnu * nu).sum() if gnu is not None else 0.0)
    keys = [k for k in NAMES if L[k] is not None and L[k].numel() > 0]
    g1 = torch.autograd.grad(loss, [L[k] for k in keys], create_graph=True)
    phi = sum((om[k] * g).sum() for k, g in zip(keys, g1))
    g2 = torch.autograd.grad(phi, [L[k] for k in keys])
    return z, lam, nu, keys, g1, g2


def dense_job(name):
    """The dense fallback under create_graph, with its returned point for the model."""
    from qpth_b200 import box
    from tests.box_families import ENTRIES, check_entry, knob
    ent = ENTRIES[name]
    n, e, sides = ent["shape"]
    with knob(ent["knob"]):
        check_entry(name)
        pr = _problem(n, e, sides, 5)
        pr["b"] = pr["b"][0]
        L = _leaves(pr, e)
        rs = np.random.RandomState(3)
        m = n * (int(pr["lb"] is not None) + int(pr["ub"] is not None))
        gz, glam, gnu = _T(rs.randn(3, n)), _T(rs.randn(3, m)), _T(rs.randn(3, e))
        om = {k: _T(rs.randn(*L[k].shape)) for k in NAMES if L[k] is not None and L[k].numel() > 0}
        f = box.BoxQPFunction(duals=True, verbose=-1)
        z, lam, nu, keys, g1, g2 = _second_order(f, L, gz, glam, gnu, om)
        st = f.last_solve()
        out = dict(dense=st.dense is not None, z=_c(st.zhat), lam=_c(st.lam), s=_c(st.slacks), nu=_c(st.nus),
                   gz=_c(gz), glam=_c(glam), gnu=_c(gnu), keys=np.array(keys))
        for k in NAMES:
            out["in_" + k] = np.zeros(0) if pr[k] is None else np.asarray(pr[k])
        for k, g in zip(keys, g2):
            out["om_" + k], out["g2_" + k] = _c(om[k]), _c(g)
        return out


def hess_job():
    """p-Hessian (B n x B n) of a scalar of z(p) on a one-CTA shape."""
    from qpth_b200 import box
    pr = _problem(31, 13, "both", 8)
    f = box.BoxQPFunction(verbose=-1)
    q, A, b, lb, ub = _T(pr["q"]), _T(pr["A"]), _T(pr["b"]), _T(pr["lb"]), _T(pr["ub"])
    c = _T(np.random.RandomState(2).randn(3, 31))
    H = torch.autograd.functional.hessian(lambda p: (0.5 * f(q, p, A, b, lb, ub) ** 2 + c * f(q, p, A, b, lb, ub)).sum(),
                                          _T(pr["p"]))
    return dict(H=_c(H))


def jtj_job(n, e, sides):
    """On a strictly complementary batch: the p-Hessian of 1/2 ||z||^2 per QP and J'J from jacobian()."""
    from qpth_b200 import box
    from tests.dual_models import complementary_box
    prs = [complementary_box(7 + i, n, e, sides) for i in range(2)]
    st = {k: None if prs[0][k] is None else _T(np.stack([p[k] for p in prs])) for k in ("q", "p", "A", "b", "lb", "ub")}
    f = box.BoxQPFunction(verbose=-1)
    H = torch.autograd.functional.hessian(
        lambda p: 0.5 * (f(st["q"], p, st["A"], st["b"], st["lb"], st["ub"]) ** 2).sum(), st["p"])
    J = f.jacobian(wrt="p")["p"]
    return dict(H=_c(H), JtJ=_c(torch.matmul(J.transpose(1, 2), J)))


def cd_job():
    """Central differences of <w, first-order gradients> along directions of every input, against create_graph; the
    first order under create_graph bit-identical to first order without it; gradgradcheck on a small shape."""
    from qpth_b200 import box
    from tests.dual_models import complementary_box
    prs = [complementary_box(21 + i, 9, 3, "both") for i in range(2)]
    base = {k: np.stack([p[k] for p in prs]) for k in NAMES}
    rs = np.random.RandomState(5)
    tan = {k: rs.randn(*base[k].shape) for k in NAMES}
    w = {k: _T(rs.randn(*base[k].shape)) for k in NAMES}
    cz = _T(rs.randn(2, 9))
    f = box.BoxQPFunction(verbose=-1, eps=1e-15)

    def grads(vals, create):
        L = {k: _T(v).requires_grad_(True) for k, v in vals.items()}
        z = f(*(L[k] for k in NAMES))
        g = torch.autograd.grad(0.5 * (z ** 2).sum() + (cz * z).sum(), [L[k] for k in NAMES], create_graph=create)
        return L, g

    L, g1 = grads(base, True)
    phi = sum((w[k] * g).sum() for k, g in zip(NAMES, g1))
    g2 = torch.autograd.grad(phi, [L[k] for k in NAMES])
    an = float(sum((g * _T(tan[k])).sum() for k, g in zip(NAMES, g2)))
    _, g0 = grads(base, False)
    same = all(torch.equal(a.detach(), b_) for a, b_ in zip(g1, g0))
    h = 1e-6
    ph = lambda sgn: float(sum((w[k] * g).sum() for k, g in zip(
        NAMES, grads({k: base[k] + sgn * h * tan[k] for k in NAMES}, False)[1])))
    fd = (ph(1) - ph(-1)) / (2 * h)
    pr = complementary_box(31, 6, 2, "both")
    ins = tuple(_T(pr[k]).requires_grad_(k in ("q", "p", "b", "ub")) for k in NAMES)
    ok = torch.autograd.gradgradcheck(lambda *a: box.BoxQPFunction(verbose=-1, eps=1e-15)(*a), ins, atol=1e-5,
                                      rtol=1e-4, raise_exception=False)
    return dict(an=an, fd=fd, same=same, gradgradcheck=ok)


def roundtrip_job():
    """fp32 CUDA and fp64 CPU inputs: dtype and device of the second-order gradients, against fp64 CUDA."""
    from qpth_b200 import box
    pr = _problem(12, 3, "both", 9)
    pr["b"] = pr["b"][0]
    rs = np.random.RandomState(4)
    gz, glam, gnu, om = rs.randn(3, 12), rs.randn(3, 24), rs.randn(3, 3), {k: None for k in NAMES}
    out = {}
    for tag, dt, dev in (("f64", torch.float64, DEV), ("f32", torch.float32, DEV), ("cpu", torch.float64, "cpu")):
        L = _leaves(pr, 3, dt, dev)
        T = lambda a: torch.tensor(a, dtype=dt, device=dev)
        om = {k: T(np.random.RandomState(6).randn(*L[k].shape)) for k in NAMES}
        f = box.BoxQPFunction(duals=True, verbose=-1)
        _, _, _, keys, _, g2 = _second_order(f, L, T(gz), T(glam), T(gnu), om)
        out[tag] = np.concatenate([g.double().cpu().numpy().ravel() for g in g2])
        out[tag + "_meta"] = np.array([str(g2[0].dtype), g2[0].device.type])
    return out


def jobs():
    from tests.boxq_families import kernel_entries
    out = [("entry_" + nm, entry_job, (nm,)) for nm in ENTRY_NAMES]
    out += [("boxq_" + nm, boxq_entry_job, (nm,)) for nm in kernel_entries()]
    out += [("dense_" + nm, dense_job, (nm,)) for nm in DENSE_NAMES]
    out += [("hess", hess_job, ()), ("jtj_9_3_both", jtj_job, (9, 3, "both")), ("jtj_10_2_lb", jtj_job, (10, 2, "lb")),
            ("cd", cd_job, ()), ("roundtrip", roundtrip_job, ())]
    return out


def main(out_dir):
    for name, fn, args in jobs():
        with open(os.path.join(out_dir, "progress.txt"), "a") as fh:
            fh.write(name + "\n")
        try:
            np.savez(os.path.join(out_dir, name + ".npz"), **fn(*args))
        except BaseException:      # noqa: BLE001 - recorded for the parent, the next job still runs
            with open(os.path.join(out_dir, name + ".err"), "w") as fh:
                fh.write(traceback.format_exc())


def run_child(out_dir, timeout_s=1200):
    """main() in a child process; returns "" or why it did not finish."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        r = subprocess.run([sys.executable, "-m", "tests.box_double_backward_jobs", out_dir], cwd=root,
                           timeout=timeout_s, capture_output=True, text=True)
        if r.returncode != 0:
            return "child exited with %d: %s" % (r.returncode, (r.stderr or "")[-2000:])
    except subprocess.TimeoutExpired:
        prog = os.path.join(out_dir, "progress.txt")
        last = open(prog).read().split()[-1:] if os.path.exists(prog) else []
        return "child killed after %d s, last job started: %s" % (timeout_s, last)
    return ""


if __name__ == "__main__":
    main(sys.argv[1])
