"""Index-level numpy model of the distributed-M factorization and substitutions of the box kernels k_box_*_dm
(qpth_b200/csrc/qp_box.cu) (TEST INFRASTRUCTURE ONLY), in the spirit of oracle/pf_model.py.

C ranks each hold the staircase block rows i = rank + C li of M in a local array at dm_boff(C, rank, li) (row stride
8 i + 12), and a panel of all 8 nts rows. The steps are the kernel's: F_k on the owner of block row k; S_k on every rank
for its own block rows below k (with the running right-hand side); panel rows copied from their owners; U_k on every
rank for its own tiles. The forward sweep reads b_k from its owner; the backward sweep sums per-rank partials in rank
order on the owner of each block, then every rank gathers w. tests/test_box_dm_cpu.py checks it against
numpy.linalg.solve, which separates "the ownership / offset arithmetic is wrong" from "the CUDA code has a bug"."""
import numpy as np

KPANLD = 12


def boff(C, rank, li):
    return 64 * rank * li + 32 * C * li * (li - 1) + 96 * li


def nblk(nts, C, rank):
    return (nts - rank + C - 1) // C if rank < nts else 0


def below(C, rank, k):
    """first own block row below block k"""
    return (k - rank) // C + 1 if k >= rank else 0


def stair_doubles(nts, C):
    """the largest local staircase of any rank (the kernel's per-CTA share of M)"""
    return max(boff(C, r, nblk(nts, C, r)) for r in range(C))


class Rank:
    def __init__(self, C, rank, nts):
        self.C, self.rank, self.nts = C, rank, nts
        self.nb = nblk(nts, C, rank)
        self.S = np.full(boff(C, rank, self.nb), np.nan)    # NaN: a read of an element never written shows up
        self.P = np.full((8 * nts, KPANLD), np.nan)
        self.b = np.full(8 * nts, np.nan)

    def at(self, r, c):
        """local index of element (r, c) of an own block row"""
        i = r >> 3
        assert i % self.C == self.rank and c <= 8 * i + 7, (r, c)
        return boff(self.C, self.rank, i // self.C) + (r & 7) * (8 * i + 12) + c

    def tile(self, i, j):
        return np.array([[self.S[self.at(8 * i + r, 8 * j + c)] for c in range(8)] for r in range(8)])

    def put(self, i, j, V):
        for r in range(8):
            for c in range(8):
                self.S[self.at(8 * i + r, 8 * j + c)] = V[r, c]

    def own(self, lo=0):
        return [self.rank + self.C * li for li in range(lo, self.nb)]


def distribute(M, C):
    """Ranks holding the lower block rows of M (order 8 nts) as dm_form leaves them."""
    nts = M.shape[0] // 8
    ranks = [Rank(C, r, nts) for r in range(C)]
    for R in ranks:
        for i in R.own():
            for j in range(i + 1):
                R.put(i, j, M[8 * i:8 * i + 8, 8 * j:8 * j + 8])
    return ranks


def chol(ranks, h):
    """dm_chol with h carried as the running right-hand side (every rank starts from the full h)."""
    C, nts = ranks[0].C, ranks[0].nts
    for R in ranks:
        R.b[:] = h
    for k in range(nts):
        own = ranks[k % C]
        D = own.tile(k, k)
        D = np.tril(D) + np.tril(D, -1).T
        T = np.linalg.inv(np.linalg.cholesky(D))
        for r in range(8):                                  # T_k published in the diagonal tile (lower part)
            for c in range(r + 1):
                own.S[own.at(8 * k + r, 8 * k + c)] = T[r, c]
        # --- cluster barrier: every rank copies T_k (upper part zero) and b_k from the owner
        Tk = np.tril(own.tile(k, k))
        bk = own.b[8 * k:8 * k + 8].copy()
        for R in ranks:
            for i in R.own(below(C, R.rank, k)):
                L = R.tile(i, k) @ Tk.T
                R.P[8 * i:8 * i + 8, :8] = L
                R.put(i, k, L @ Tk)
                R.b[8 * i:8 * i + 8] -= R.tile(i, k) @ bk
        if k + 1 == nts:
            break
        # --- cluster barrier: panel rows of the other ranks, then the own trailing tiles
        for R in ranks:
            last = R.rank + C * (R.nb - 1) if R.nb else k
            for j in range(k + 1, last + 1):
                if j % C != R.rank:
                    R.P[8 * j:8 * j + 8, :8] = ranks[j % C].P[8 * j:8 * j + 8, :8]
            for i in R.own(below(C, R.rank, k)):
                Li = R.P[8 * i:8 * i + 8, :8]
                for j in range(k + 1, i + 1):
                    R.put(i, j, R.tile(i, j) - Li @ R.P[8 * j:8 * j + 8, :8].T)


def fwd(ranks, h):
    """dm_fwd with an existing factor (b_k read from its owner after each barrier)."""
    C, nts = ranks[0].C, ranks[0].nts
    for R in ranks:
        R.b[:] = h
    for k in range(nts - 1):
        bk = ranks[k % C].b[8 * k:8 * k + 8].copy()
        for R in ranks:
            for i in R.own(below(C, R.rank, k)):
                R.b[8 * i:8 * i + 8] -= R.tile(i, k) @ bk


def diag_and_bwd(ranks):
    """dm_diag (local) and dm_bwd: returns w as every rank gathers it (they must agree)."""
    C, nts = ranks[0].C, ranks[0].nts
    n = 8 * nts
    cv = [np.full(n, np.nan) for _ in ranks]
    for R in ranks:
        for i in R.own():
            T = np.tril(R.tile(i, i))
            cv[R.rank][8 * i:8 * i + 8] = T.T @ (T @ R.b[8 * i:8 * i + 8])
    part = [np.zeros(n) for _ in ranks]
    wpub = [np.full(n, np.nan) for _ in ranks]
    for i in range(nts - 1, -1, -1):
        o = i % C
        s = cv[o][8 * i:8 * i + 8].copy()
        for r in range(C):                                   # rank order
            s = s - part[r][8 * i:8 * i + 8]
        wpub[o][8 * i:8 * i + 8] = s
        R = ranks[o]
        for t in range(8 * i):
            part[o][t] += sum(R.S[R.at(8 * i + rr, t)] * s[rr] for rr in range(8))
    ws = [np.concatenate([wpub[(t // 8) % C][t:t + 1] for t in range(n)]) for _ in ranks]
    return ws[0]


def solve(M, h, C, refactor_rhs=None):
    """Factor M over C ranks carrying h, solve M w = h; with refactor_rhs, also solve with the existing factor (the
    corrector's path). Returns w (and w2)."""
    ranks = distribute(M, C)
    chol(ranks, h)
    w = diag_and_bwd(ranks)
    if refactor_rhs is None:
        return w
    fwd(ranks, refactor_rhs)
    return w, diag_and_bwd(ranks)
