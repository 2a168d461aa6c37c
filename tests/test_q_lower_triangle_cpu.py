"""Only the lower triangle of Q is read: the host logic of the equality-only path (qpth_b200/eqonly.py) on the CPU.

The two stand-alone KKT solves are replaced by a dense numpy solve that, like the kernels, reads only the lower triangle of
Q and regularises as they do (Q + eps I, D + eps I, -eps I on both constraint blocks). With the strictly upper triangle
of Q set to NaN, or to finite values unrelated to the lower one, z*, nu, every gradient of a backward with adjoints on z
and nu, and a forward-mode JVP must equal, bit for bit, those of the symmetric matrix tril(Q) + tril(Q, -1)^T, for both
KKT solvers: LU_PARTIAL (one solve) and IR_UNOPT (a regularised solve refined against the matrix the factor saw)."""
import numpy as np
import pytest
import torch

from tests.kernel_families import eq_outputs, poison, sym_lower


class LowerFactor:
    """Stand-in for qpth_b200.kkt._Factored that reads only the lower triangle of Q:
    [Q~ 0 G' A'; 0 D~ I 0; G I -eps I 0; A 0 0 -eps I] [dx ds dz dy] = -[rx rs rz ry], Q~ = sym_lower(Q) + eps I,
    D~ = D + eps I (eps = 0: the plain system)."""

    def __init__(self, Q, G, A, reg):
        self.reg = float(reg)
        self.Q = sym_lower(Q.detach().cpu().numpy()) + self.reg * np.eye(Q.shape[-1])
        self.G, self.A = (t.detach().cpu().numpy() for t in (G, A))
        self.spd = torch.tensor([int(np.linalg.eigvalsh(q).min() <= 0) for q in self.Q])

    def solve(self, d, rx, rs, rz, ry):
        d, rx, rs, rz, ry = (t.detach().cpu().numpy() for t in (d, rx, rs, rz, ry))
        B, m, n = self.G.shape
        e, eps = self.A.shape[1], self.reg
        out = []
        for i in range(B):
            K = np.zeros((n + 2 * m + e,) * 2)
            K[:n, :n] = self.Q[i]; K[:n, n + m:n + 2 * m] = self.G[i].T; K[:n, n + 2 * m:] = self.A[i].T
            K[n:n + m, n:n + m] = np.diag(d[i] + eps); K[n:n + m, n + m:n + 2 * m] = np.eye(m)
            K[n + m:n + 2 * m, :n] = self.G[i]; K[n + m:n + 2 * m, n:n + m] = np.eye(m)
            K[n + m:n + 2 * m, n + m:n + 2 * m] = -eps * np.eye(m)
            K[n + 2 * m:, :n] = self.A[i]; K[n + 2 * m:, n + 2 * m:] = -eps * np.eye(e)
            out.append(np.linalg.solve(K, -np.concatenate([rx[i], rs[i], rz[i], ry[i]])))
        s = torch.tensor(np.stack(out))
        return s[:, :n], s[:, n:n + m], s[:, n + m:n + 2 * m], s[:, n + 2 * m:]


@pytest.fixture
def on_cpu(monkeypatch):
    from qpth_b200 import eqonly
    monkeypatch.setattr(eqonly, "_factor", LowerFactor)
    monkeypatch.setattr(eqonly, "_target_device", lambda Q_: torch.device("cpu"))
    return eqonly


def _problem(shared, seed=5, B=3, nz=11, neq=4):
    rs = np.random.RandomState(seed)
    L = rs.randn(nz, nz) if shared else rs.randn(B, nz, nz)
    Q = sym_lower(L @ np.swapaxes(L, -1, -2) + 0.5 * np.eye(nz))
    A = rs.randn(neq, nz) if shared else rs.randn(B, neq, nz)
    pr = dict(Q=Q, p=rs.randn(B, nz), A=A, b=rs.randn(B, neq))
    adj = dict(z=rs.randn(B, nz), nu=rs.randn(B, neq))
    tan = {k: rs.randn(*np.shape(v)) for k, v in pr.items()}       # dQ in full and asymmetric: it enters as sym(dQ)
    return pr, adj, tan, rs


@pytest.mark.parametrize("shared", [False, True], ids=["batched_Q", "shared_Q"])
@pytest.mark.parametrize("how", ["nan", "garbage"])
@pytest.mark.parametrize("solver", ["LU_PARTIAL", "IR_UNOPT"])
def test_equality_only_reads_only_the_lower_triangle(on_cpu, solver, how, shared):
    from qpth_b200 import KKTSolvers
    kkt_solver = getattr(KKTSolvers, solver)
    pr, adj, tan, rs = _problem(shared)
    ref = eq_outputs(pr, adj, tan, kkt_solver, dev="cpu")
    assert all(np.isfinite(v).all() for v in ref.values())
    got = eq_outputs(dict(pr, Q=poison(pr["Q"], how, rs)), adj, tan, kkt_solver, dev="cpu")
    assert set(got) == set(ref)
    for k in ref:
        assert np.array_equal(got[k], ref[k]), (k, np.abs(got[k] - ref[k]).max())


def test_the_stand_in_ignores_the_upper_triangle():
    """LowerFactor itself: the same solve, bit for bit, whatever lies above the diagonal."""
    pr, _, _, rs = _problem(False)
    B, nz = pr["p"].shape
    G = torch.zeros(B, 1, nz, dtype=torch.float64)
    A = torch.tensor(pr["A"])
    args = [torch.ones(B, 1, dtype=torch.float64), torch.tensor(pr["p"]), torch.zeros(B, 1, dtype=torch.float64),
            -torch.ones(B, 1, dtype=torch.float64), torch.tensor(pr["b"])]
    for reg in (0.0, 1e-7):
        a = LowerFactor(torch.tensor(pr["Q"]), G, A, reg).solve(*args)
        b = LowerFactor(torch.tensor(poison(pr["Q"], "nan", rs)), G, A, reg).solve(*args)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
