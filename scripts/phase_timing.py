"""Cycle accounting of k_forward_fast (needs a -DQPB_TIMING build: QPB200_TIMING_LIB or libqpth_b200_timing.so).

Reports (1) per-CTA wall times of one launch (globaltimer at entry/exit, SM, Newton iterations): how the kernel's
duration decomposes into launch + slowest QP + tail, and (2) the thread-0 phase slots of the SLOWEST QP of the batch,
which by construction sum to that CTA's duration.

    python scripts/phase_timing.py [B n m e [QP]]
QP: report the phase slots of this QP instead of the slowest one. At a batch above the SM count QPFunction runs the
throughput-mode plan (three or two QPs per SM); a QP from the middle of such a batch shares its SM with other QPs for
its whole life, while the slowest QP of the batch may finish alone in the tail."""
import sys, os, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from qpth_b200 import _lib
_lib.LIB_PATH = os.environ.get("QPB200_TIMING_LIB") or os.path.join(os.path.dirname(_lib.LIB_PATH), "libqpth_b200_timing.so")
from qpth_b200 import QPFunction
from qpth_b200.problems import random_qp_batch
B, n, m, e = [int(x) for x in (sys.argv[1:5] if len(sys.argv) > 4 else (128, 100, 100, 0))]
target = int(sys.argv[5]) if len(sys.argv) > 5 else None
lib = _lib.load()
pr = random_qp_batch(B, n, m, e, seed=0)
dev = "cuda:0"
t = {k: (torch.tensor(v, dtype=torch.float64, device=dev) if v.size else torch.Tensor().to(dev).double()) for k, v in pr.items() if k != "dl"}
f = QPFunction(verbose=-1, check_Q_spd=False)
from qpth_b200 import qp as _qp
two = _qp.MODE == "throughput" or (_qp.MODE == "auto" and B > _lib.sm_count(0))     # QPFunction's choice
plan = _lib.plan_for(n, m, e, two=two)
print("card: %s; mode %s: pf_three=%d pf_two=%d" % (torch.cuda.get_device_name(0), _qp.MODE, plan.pf_three, plan.pf_two))
print("plan: fast=%d coop=%d pf=%d pf_global=%d" % (plan.fast, plan.coop, plan.pf, plan.pf_global))
# the three-per-SM forward is the 192-thread build (qp_alt.cu), which keeps its own slots
pre = "qpb200_alt192_" if (plan.pf and plan.pf_three) else "qpb200_"
debug_timing, debug_cta = getattr(lib, pre + "debug_timing"), getattr(lib, pre + "debug_cta")
for fn in (debug_timing, debug_cta):
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int]
f(t["Q"], t["p"], t["G"], t["h"], t["A"], t["b"]); torch.cuda.synchronize()
iters = f.last_solve().iters.cpu().numpy()
slow = int(np.argmax(iters)) if target is None else target
debug_timing(None, 2 + slow)
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
f(t["Q"], t["p"], t["G"], t["h"], t["A"], t["b"]); torch.cuda.synchronize()
nq = min(B, 8192)
cta = (ctypes.c_longlong * (4 * nq))()
debug_cta(cta, nq)
c = np.array(cta[:]).reshape(nq, 4)
t0 = c[:, 0].min()
dur = (c[:, 1] - c[:, 0]) / 1e3
print("per-CTA (one forward launch of %d QPs): first entry -> last exit %.1f us; CTA duration min/mean/max %.1f/%.1f/%.1f us; last CTA entry at +%.1f us; iters min/mean/max %d/%.1f/%d"
      % (nq, (c[:, 1].max() - t0) / 1e3, dur.min(), dur.mean(), dur.max(), (c[:, 0].max() - t0) / 1e3, c[:, 2].min(), c[:, 2].mean(), c[:, 2].max()))
per_it = dur / (c[:, 2] + 1)
print("us per (iteration + 1): min %.2f mean %.2f max %.2f; SMs used %d; reported QP %d: %d iterations, %.1f us" % (per_it.min(), per_it.mean(), per_it.max(), len(set(c[:, 3].tolist())), slow, c[slow, 2], dur[slow]))
if slow < nq:                            # co-residency of the reported QP: other CTAs on its SM, time-weighted over its life
    same = (c[:, 3] == c[slow, 3]) & (np.arange(nq) != slow)
    ov = np.clip(np.minimum(c[same, 1], c[slow, 1]) - np.maximum(c[same, 0], c[slow, 0]), 0, None).sum()
    print("QP %d: SM %d, on average %.2f other CTAs of this launch resident beside it" % (slow, c[slow, 3], ov / max(1, c[slow, 1] - c[slow, 0])))
buf = (ctypes.c_longlong * 128)()
debug_timing(buf, 0)
it = int(c[slow, 2])
names = {0: "make_ctx (TMA staging)", 1: "load vectors", 2: "whiten (+ first K issue)", 3: "loop misc/update (prev)", 4: "matvec_cols (r~x, iteration 0)", 5: "matvec_rows2 + tri_norm2", 6: "residual elementwise", 8: "reduce_sum4",
         9: "best/exit/aug build", 10: "factor_and_solve tail", 11: "aff step, sigma, rhs", 12: "trsv_fwd (cor)", 13: "trsv_bwd (cor)", 14: "issue_K + combine", 15: "alpha, update, matvec_cols2 (dx~, next r~x)", 16: "exit: unwhiten + outputs",
         24: "chol: diag tile k+1 update", 26: "chol: (chain) F_k+1 / end of step", 32: "chol exit", 33: "trsv_bwd (aff)",
         40: "[warp1] gap", 42: "[warp1] named barrier wait", 44: "[warp1] step barrier wait"}
tot = sum(buf[i] for i in range(40)) + sum(buf[i] for i in range(80, 128))   # thread 0 owns slots 0..39 and 80..127 (per-step Cholesky slots); 40..79 are warp 1's
print("QP %d: thread-0 slots sum to %d cycles = %.1f us @1.965 GHz (CTA duration by globaltimer: %.1f us); per iteration %.0f cycles" % (slow, tot, tot / 1965.0, dur[slow], tot / (it + 1)))
chol_steps = sum(buf[i] for i in range(80, 128))
print("   per-step Cholesky slots of the chain warp (80..127, table below): %d cyc %5.1f%%   per-iter %7.0f" % (chol_steps, 100.0 * chol_steps / tot, chol_steps / (it + 1)))
for i in list(range(48)):
    if buf[i]:
        print("%2d %-34s %9d cyc  %5.1f%%   per-iter %7.0f" % (i, names.get(i, "?"), buf[i], 100.0 * buf[i] / tot, buf[i] / (it + 1)))
nf = it + 1
print("per Cholesky step k (cycles per factorization): S_k[w1]  U_k[w1] | s_k[w0]  F_k+1[w0]  wait[w0]")
for k in range(13):
    print("%2d  %6.0f %6.0f | %6.0f %6.0f %6.0f" % (k, buf[64 + k] / nf, buf[48 + k] / nf, buf[96 + k] / nf, buf[80 + k] / nf, buf[112 + k] / nf))
