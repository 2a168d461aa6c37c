"""pre_factor_kkt in throughput mode: k_setup_pf at 192 threads, three per SM (the plan of `plan_for(..., two=True)`).
L L^T = Q (+ eps I), W = [A; G] L^-T against a dense solve, and the K template (Schur complement of the equality block,
equality columns in product form) against its definition, on a shape with equality constraints, on the regularised
variant, and on a shape whose chol(Q) staircase is larger than W's (nz > ms_pad: W rows in two register chunks)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import pdipm_oracle as orc
from qpth_b200.problems import random_qp_batch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _prefactor(plan, pr, B, n, m, e, reg=None):
    from qpth_b200 import _lib
    lib = _lib.load()
    tt = lambda a: torch.tensor(a, dtype=torch.float64, device=DEV).contiguous()
    Q, G = tt(pr["Q"]), tt(pr["G"])
    A = tt(pr["A"]) if e else None
    L = torch.full((B, plan.L_elems), float("nan"), dtype=torch.float64, device=DEV)
    W = torch.full((B, plan.ms, plan.ldw), float("nan"), dtype=torch.float64, device=DEV)
    K = torch.full((B, plan.K_elems), float("nan"), dtype=torch.float64, device=DEV)
    spd = torch.full((B,), 7, dtype=torch.int32, device=DEV)
    P = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if reg is None:
        rc = lib.qpb200_pre_factor_kkt(ctypes.byref(plan), B, P(Q), n * n, P(G), m * n, P(A), e * n,
                                       P(L), P(W), P(K), P(spd), None, st)
    else:
        rc = lib.qpb200_pre_factor_kkt_reg(ctypes.byref(plan), B, P(Q), n * n, P(G), m * n, P(A), e * n, reg,
                                           P(L), P(W), P(K), P(spd), None, st)
    _lib.check(rc)
    torch.cuda.synchronize()
    Kf = K.cpu().numpy()
    Kn = np.zeros((B, plan.ms_pad, plan.ms_pad))
    for r in range(plan.ms_pad):        # staircase: element (r, c) at (32 i + 64) i + (r % 8)(8 i + 12) + c, i = r // 8
        i = r // 8
        off = (32 * i + 64) * i + (r % 8) * (8 * i + 12)
        Kn[:, r, :8 * i + 8] = Kf[:, off:off + 8 * i + 8]
    return L.cpu().numpy(), W.cpu().numpy(), Kn, spd.cpu().numpy()


@pytest.mark.parametrize("shape", [(64, 50, 50, 10), (16, 100, 100, 0), (16, 108, 90, 0)])
@pytest.mark.parametrize("reg", [None, 1e-4])
def test_throughput_setup_matches_definition(shape, reg):
    from qpth_b200 import _lib
    B, n, m, e = shape
    plan = _lib.plan_for(n, m, e, two=True)
    assert plan.pf_three == 1 and plan.setup_pf_smem_bytes <= plan.pf3_smem_bytes    # the 192-thread setup runs
    pr = random_qp_batch(B, n, m, e, seed=11)
    Lp, Wp, Kn, spd = _prefactor(plan, pr, B, n, m, e, reg)
    assert (spd == 0).all()
    eps = 0.0 if reg is None else reg
    ep, ms = plan.neq_pad, plan.ms
    tri = np.tril_indices(n)
    for i in range(B):
        Qi = pr["Q"][i] + eps * np.eye(n)
        Ln = np.zeros((n, n)); Ln[tri] = Lp[i][:n * (n + 1) // 2]       # packed lower, row by row
        assert np.abs(Ln @ Ln.T - Qi).max() < 1e-10 * np.abs(Qi).max()
        X = np.vstack([pr["A"][i], pr["G"][i]]) if e else pr["G"][i]
        Wref = np.linalg.solve(Ln, X.T).T
        Wall = np.zeros((ms, n)); Wall[:e] = Wref[:e]; Wall[ep:] = Wref[e:]
        assert np.abs(Wp[i][:, :n] - Wall).max() < 1e-8 * np.abs(Wref).max()
        assert (Wp[i][:, n:] == 0.0).all() and (Wp[i][e:ep] == 0.0).all()
        # S template: W W^T, + eps on the real equality rows, 1 on the dummy rows; its first ep columns in product form
        S = Wall @ Wall.T
        S[np.arange(e), np.arange(e)] += eps
        S[np.arange(e, ep), np.arange(e, ep)] += 1.0
        if ep == 0:
            assert np.abs(np.tril(Kn[i][:ms, :ms]) - np.tril(S)).max() < 1e-8 * np.abs(S).max()
            continue
        L11 = np.linalg.cholesky(S[:ep, :ep])
        L21 = np.linalg.solve(L11, S[ep:, :ep].T).T
        R = S[ep:, ep:] - L21 @ L21.T
        assert np.abs(np.tril(Kn[i][ep:ms, ep:ms]) - np.tril(R)).max() < 1e-8 * np.abs(R).max()
        F = orc.Factors(pr["Q"][i:i + 1], pr["G"][i:i + 1], pr["A"][i:i + 1])
        if reg is None:
            assert np.abs(np.tril(Kn[i][ep:ms, ep:ms]) - np.tril(F.R[0])).max() < 1e-8 * np.abs(F.R[0]).max()
        Lfull = np.vstack([L11, L21])
        for k in range(ep // 8):
            T = np.linalg.inv(Lfull[8 * k:8 * k + 8, 8 * k:8 * k + 8])
            assert np.abs(np.tril(Kn[i][8 * k:8 * k + 8, 8 * k:8 * k + 8]) - np.tril(T)).max() < 1e-8 * np.abs(T).max()
            Pref = Lfull[8 * k + 8:, 8 * k:8 * k + 8] @ T
            assert np.abs(Kn[i][8 * k + 8:ms, 8 * k:8 * k + 8] - Pref).max() < 1e-8 * max(1.0, np.abs(Pref).max())


def test_throughput_setup_flags_non_spd():
    from qpth_b200 import _lib
    B, n, m, e = 4, 100, 100, 0
    plan = _lib.plan_for(n, m, e, two=True)
    pr = random_qp_batch(B, n, m, e, seed=3)
    pr["Q"] = pr["Q"].copy()
    pr["Q"][2] = -np.eye(n)
    _, _, _, spd = _prefactor(plan, pr, B, n, m, e)
    assert spd.tolist() == [0, 0, 1, 0]
