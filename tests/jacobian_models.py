"""Numpy models of the Jacobians of (z, lam, nu) with respect to (p, h, b) (TEST INFRASTRUCTURE ONLY).

dense_jacobian: the negated inverse of the backward's system, from np.linalg.solve of
    K = [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0],   D = clamp(lam, 1e-8) / clamp(s, 1e-8)
with identity right-hand sides: R = K^-1 and, from the JVP's right-hand side (rx = dp, rz = -dh, ry = -db),
    J_.,p = -R_.,x      J_.,h = R_.,lam      J_.,b = R_.,nu.
blocked_jacobian: the arithmetic of qpb200_jacobian (csrc/qp_jac.cu) step by step from W = [A; 0; G] L^-T (equality
rows padded to a multiple of 8 with zero rows) and L = chol(Q): S = W W' + diag(0, 1, 1/d) identity-padded to a
multiple of 8, its product-form factor (T_k = L_kk^-1, P_ik = L_ik T_k), and per 8-column block
    p block j:  U = L^-1 E_j by 8x8 block forward substitution, Y = S^-1 (W U)
    w block c:  U = 0, Y = S^-1 E_c
    J_w = -Y,   J_z = -L^-T (U - W' Y),
S^-1 applied as the forward sweep Y_i -= P_ik Y_k, the diagonal Y_k = T_k' T_k Y_k and the backward sweep
Y_k -= P_ik' Y_i. Both return rows [z; lam; nu] and columns [p, h, b].
"""
import numpy as np


def clamped_d(lam, s):
    return np.maximum(lam, 1e-8) / np.maximum(s, 1e-8)


def dense_jacobian(Q, G, A, lam, s):
    n, m = Q.shape[0], G.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    N = n + 2 * m + e
    K = np.zeros((N, N))
    K[:n, :n] = Q
    K[:n, n + m:n + 2 * m] = G.T
    K[n:n + m, n:n + m] = np.diag(clamped_d(lam, s))
    K[n:n + m, n + m:n + 2 * m] = np.eye(m)
    K[n + m:n + 2 * m, :n] = G
    K[n + m:n + 2 * m, n:n + m] = np.eye(m)
    if e:
        K[:n, n + 2 * m:] = A.T
        K[n + 2 * m:, :n] = A
    R = np.linalg.solve(K, np.eye(N))
    rows = np.concatenate([np.arange(n), n + m + np.arange(m), n + 2 * m + np.arange(e)])
    return np.concatenate([-R[rows][:, :n], R[rows][:, n + m:n + 2 * m], R[rows][:, n + 2 * m:]], axis=1)


def factors(Q, G, A):
    """(L, W) as qpb200_pre_factor_kkt stores them: chol(Q) and [A; 0; G] L^-T with neq_pad - neq zero rows."""
    n = Q.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    ep = (e + 7) // 8 * 8
    L = np.linalg.cholesky(Q)
    C = np.zeros((ep + G.shape[0], n))
    if e:
        C[:e] = A
    C[ep:] = G
    return L, np.linalg.solve(L, C.T).T


def _pad_identity(M, size):
    out = np.eye(size)
    out[:M.shape[0], :M.shape[1]] = M
    return out


def blocked_jacobian(L, W, lam, s, neq):
    n, ms = L.shape[0], W.shape[0]
    m, e = lam.shape[0], neq
    ep = ms - m
    msp, np_ = (ms + 7) // 8 * 8, (n + 7) // 8 * 8
    nts, ntz = msp // 8, np_ // 8
    Wp = np.zeros((msp, np_))
    Wp[:ms, :n] = W
    Lp = _pad_identity(L, np_)
    dg = np.ones(msp)
    dg[:e] = 0.0
    dg[ep:ms] = 1.0 / clamped_d(lam, s)
    S = Wp @ Wp.T + np.diag(dg)
    LS = np.linalg.cholesky(S)
    tile = lambda M, i, k: M[8 * i:8 * i + 8, 8 * k:8 * k + 8]
    T = [np.linalg.inv(tile(LS, k, k)) for k in range(nts)]
    P = {(i, k): tile(LS, i, k) @ T[k] for k in range(nts) for i in range(k + 1, nts)}
    TL = [np.linalg.inv(tile(Lp, k, k)) for k in range(ntz)]

    def s_solve(Y, kf):
        Y = Y.copy()
        for k in range(kf, nts - 1):
            for i in range(k + 1, nts):
                Y[8 * i:8 * i + 8] -= P[i, k] @ Y[8 * k:8 * k + 8]
        for k in range(kf, nts):
            Y[8 * k:8 * k + 8] = T[k].T @ (T[k] @ Y[8 * k:8 * k + 8])
        for i in range(nts - 1, 0, -1):
            for k in range(i):
                Y[8 * k:8 * k + 8] -= P[i, k].T @ Y[8 * i:8 * i + 8]
        return Y

    def l_solve(jb):
        U = np.zeros((np_, 8))
        for i in range(jb, ntz):
            c = np.eye(8) if i == jb else np.zeros((8, 8))
            for k in range(jb, i):
                c = c - tile(Lp, i, k) @ U[8 * k:8 * k + 8]
            U[8 * i:8 * i + 8] = TL[i] @ c
        return U

    def lt_solve(U):
        U = U.copy()
        for i in range(ntz - 1, -1, -1):
            c = U[8 * i:8 * i + 8]
            for k in range(i + 1, ntz):
                c = c - tile(Lp, k, i).T @ U[8 * k:8 * k + 8]
            U[8 * i:8 * i + 8] = TL[i].T @ c
        return U

    Jz = np.zeros((np_, np_ + msp))
    Jw = np.zeros((msp, np_ + msp))
    for jb in range(ntz):
        U = l_solve(jb)
        Y = s_solve(Wp @ U, 0)
        Jw[:, 8 * jb:8 * jb + 8] = -Y
        Jz[:, 8 * jb:8 * jb + 8] = -lt_solve(U - Wp.T @ Y)
    for c in range(nts):
        Y = s_solve(np.eye(msp)[:, 8 * c:8 * c + 8], c)
        Jw[:, np_ + 8 * c:np_ + 8 * c + 8] = -Y
        Jz[:, np_ + 8 * c:np_ + 8 * c + 8] = -lt_solve(-Wp.T @ Y)
    rows = [Jz[:n], Jw[ep:ms], Jw[:e]]
    J = np.concatenate(rows, axis=0)
    return np.concatenate([J[:, :n], J[:, np_ + ep:np_ + ms], J[:, np_:np_ + e]], axis=1)


def split(J, n, m, e):
    """{(row name, column name): block} of a full [z; lam; nu] x [p, h, b] Jacobian."""
    rs = dict(z=(0, n), lam=(n, n + m), nu=(n + m, n + m + e))
    cs = dict(p=(0, n), h=(n, n + m), b=(n + m, n + m + e))
    return {(r, c): J[r0:r1, c0:c1] for r, (r0, r1) in rs.items() for c, (c0, c1) in cs.items()}


def symmetry_residuals(J, n, m, e):
    """Max abs of the identities J_z,p = J_z,p', J_lam,h = J_lam,h', J_z,h = -J_lam,p', J_z,b = -J_nu,p',
    J_lam,b = J_nu,h'."""
    B = split(J, n, m, e)
    res = [B["z", "p"] - B["z", "p"].T, B["lam", "h"] - B["lam", "h"].T, B["z", "h"] + B["lam", "p"].T,
           B["z", "b"] + B["nu", "p"].T, B["lam", "b"] - B["nu", "h"].T]
    return max(float(np.abs(r).max()) if r.size else 0.0 for r in res)
