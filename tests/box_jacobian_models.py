"""Numpy models of BoxQPFunction's Jacobians of (z, lam, nu) with respect to (p, lb, ub, b) (TEST INFRASTRUCTURE ONLY).

dense_box_jacobian: tests/jacobian_models.dense_jacobian on the dense equivalent (Q = diag(q) or Q, G = [-I; I] of the
    sides given, h = [-lb; ub]) with the h columns mapped to J_lb = -J_h[:, :nlb] and J_ub = J_h[:, nlb:].
blocked_box_jacobian: the arithmetic of qpb200_box_jacobian (csrc/qp_jac.cu, diagonal q) step by step: H^-1 with
    H = q + d_lb + d_ub, M = A H^-1 A' identity-padded to a multiple of 8, its product-form factor (T_k = L_kk^-1,
    P_ik = L_ik T_k), and per 8-column block
        p block j:  Y = M^-1 (A H^-1 E_j),  z = -H^-1 (E_j - A'Y),  nu = -Y
        b block c:  Y = M^-1 E_c (forward sweep from block c),  z = H^-1 A'Y,  nu = -Y
    with the lb / ub columns the p columns scaled by -d_lb_j / -d_ub_j and the lam rows d_lb o (rz_lb - z),
    d_ub o (rz_ub + z) (rz_lb = e_j in lb column j, rz_ub = -e_j in ub column j).
Both return rows [z; lam; nu] and columns [p, lb, ub, b] (the sides given; b only when neq > 0).
diagonal_box_jacobian: a diagonal q and no equality rows, one long-double KKT block per variable (the reference at
    widths whose dense model is too large to form).
"""
import numpy as np

from tests import jacobian_models as jm


def dense_G(n, nlb, has_ub):
    return np.concatenate(([-np.eye(n)] if nlb else []) + ([np.eye(n)] if has_ub else []), 0)


def dense_box_jacobian(Q, A, lam, s, nlb, has_ub):
    """Q: (n, n) (np.diag(q) for a diagonal q)."""
    n, m = Q.shape[0], lam.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    Jd = jm.dense_jacobian(Q, dense_G(n, nlb, has_ub), A if e else None, lam, s)
    cols = [Jd[:, :n]] + ([-Jd[:, n:n + nlb]] if nlb else []) + ([Jd[:, n + nlb:n + m]] if has_ub else [])
    return np.concatenate(cols + ([Jd[:, n + m:]] if e else []), axis=1)


def _pf(M):
    """The product-form factor of M (order a multiple of 8): (T, P) with T_k = L_kk^-1, P_ik = L_ik T_k."""
    L = np.linalg.cholesky(M)
    nts = M.shape[0] // 8
    tile = lambda i, k: L[8 * i:8 * i + 8, 8 * k:8 * k + 8]
    T = [np.linalg.inv(tile(k, k)) for k in range(nts)]
    return T, {(i, k): tile(i, k) @ T[k] for k in range(nts) for i in range(k + 1, nts)}


def _pf_solve(T, P, Y, kf):
    """jac_ssolve: forward sweep from block kf, the diagonal T_k' T_k, backward sweep."""
    nts = len(T)
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


def blocked_box_jacobian(q, A, lam, s, nlb, has_ub):
    n, m = q.shape[0], lam.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    ep, np_ = (e + 7) // 8 * 8, (n + 7) // 8 * 8
    d = jm.clamped_d(lam, s)
    dlb = d[:nlb] if nlb else np.zeros(n)
    dub = d[nlb:] if has_ub else np.zeros(n)
    hv = np.zeros(np_)
    hv[:n] = 1.0 / (q + dlb + dub)
    Ap = np.zeros((ep, np_))
    if e:
        Ap[:e, :n] = A
    M = Ap @ np.diag(hv) @ Ap.T
    M[e:, e:] = np.eye(ep - e)
    T, P = _pf(M) if ep else ([], {})
    Zp, Np = np.zeros((np_, np_)), np.zeros((ep, np_))      # -z and -nu of the p columns, block by block
    for jb in range(np_ // 8):
        E = np.eye(np_)[:, 8 * jb:8 * jb + 8]
        Y = _pf_solve(T, P, Ap @ (hv[:, None] * E), 0)
        Zp[:, 8 * jb:8 * jb + 8] = hv[:, None] * (E - Ap.T @ Y)
        Np[:, 8 * jb:8 * jb + 8] = Y
    Zb, Nb = np.zeros((np_, ep)), np.zeros((ep, ep))
    for c in range(ep // 8):
        Y = _pf_solve(T, P, np.eye(ep)[:, 8 * c:8 * c + 8], c)
        Zb[:, 8 * c:8 * c + 8] = hv[:, None] * (-Ap.T @ Y)
        Nb[:, 8 * c:8 * c + 8] = Y

    return _assemble(Zp, Np, Zb, Nb, n, e, dlb, dub, nlb, has_ub)


def _assemble(Zp, Np, Zb, Nb, n, e, dlb, dub, nlb, has_ub):
    """box_jac_store over every block: rows [z; lam; nu] and columns [p, lb, ub, b] from U = -z, Y = -nu of the p
    solves (Zp, Np) and the b solves (Zb, Nb)."""
    def column_block(U, Y, kind, ncol):
        sc = np.ones(ncol) if kind == 0 else -(dlb if kind == 1 else dub)[:ncol]
        z = -U[:n, :ncol] * sc
        rz_lb = np.eye(n) if kind == 1 else np.zeros((n, ncol))
        rz_ub = -np.eye(n) if kind == 2 else np.zeros((n, ncol))
        lam_rows = ([dlb[:, None] * (rz_lb - z)] if nlb else []) + ([dub[:, None] * (rz_ub + z)] if has_ub else [])
        return np.concatenate([z] + lam_rows + [-Y[:e, :ncol] * sc], axis=0)

    cols = [column_block(Zp, Np, 0, n)]
    cols += [column_block(Zp, Np, 1, n)] if nlb else []
    cols += [column_block(Zp, Np, 2, n)] if has_ub else []
    cols += [column_block(Zb, Nb, 0, e)] if e else []
    return np.concatenate(cols, axis=1)


def bordered_box_jacobian(Q, A, lam, s, nlb, has_ub):
    """The arithmetic of qpb200_boxq_jacobian (csrc/qp_boxq.cu, dense Q): K = [H A'; A 0] = L diag(I, -I) L' with
    oracle/boxq_model.py's L11, L21, L22 placed on the padded order N = nz_pad + neq_pad (identity padding), its
    product-form tiles, and per 8-column block the forward sweep from the block of the unit rows, T_k' T_k with the
    block rows past nz_pad negated, the backward sweep: X = K^-1 E_j for a p block, -K^-1 E_(nz_pad + c) for a b block,
    U = X's z rows, Y = its nu rows."""
    from oracle.boxq_model import _SysQ
    n, m = Q.shape[0], lam.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    ep, np_ = (e + 7) // 8 * 8, (n + 7) // 8 * 8
    N = np_ + ep
    d = jm.clamped_d(lam, s)
    var = np.concatenate(([np.arange(n)] if nlb else []) + ([np.arange(n)] if has_ub else []))
    sgn = np.concatenate(([-np.ones(n)] if nlb else []) + ([np.ones(n)] if has_ub else []))
    sys_ = _SysQ(Q, A if e else np.zeros((0, n)), var, sgn, d)
    L = np.eye(N)
    L[:n, :n] = sys_.L11
    if e:
        L[np_:np_ + e, :n] = sys_.L21
        L[np_:np_ + e, np_:np_ + e] = sys_.L22
    nts = N // 8
    tile = lambda i, k: L[8 * i:8 * i + 8, 8 * k:8 * k + 8]
    T = [np.linalg.inv(tile(k, k)) for k in range(nts)]
    P = {(i, k): tile(i, k) @ T[k] for k in range(nts) for i in range(k + 1, nts)}
    kneg = np_ // 8

    def solve(Y, kf):
        Y = Y.copy()
        for k in range(kf, nts - 1):
            for i in range(k + 1, nts):
                Y[8 * i:8 * i + 8] -= P[i, k] @ Y[8 * k:8 * k + 8]
        for k in range(kf, nts):
            Y[8 * k:8 * k + 8] = (-1 if k >= kneg else 1) * T[k].T @ (T[k] @ Y[8 * k:8 * k + 8])
        for i in range(nts - 1, 0, -1):
            for k in range(i):
                Y[8 * k:8 * k + 8] -= P[i, k].T @ Y[8 * i:8 * i + 8]
        return Y

    I = np.eye(N)
    Xp = np.concatenate([solve(I[:, 8 * t:8 * t + 8], t) for t in range(np_ // 8)], axis=1)
    Xb = np.concatenate([solve(-I[:, np_ + 8 * c:np_ + 8 * c + 8], kneg + c) for c in range(ep // 8)], axis=1) \
        if ep else np.zeros((N, 0))
    dlb = d[:nlb] if nlb else np.zeros(n)
    dub = d[nlb:] if has_ub else np.zeros(n)
    return _assemble(Xp[:np_], Xp[np_:], Xb[:np_], Xb[np_:], n, e, dlb, dub, nlb, has_ub)


def dense_box_jacobian_refined(Q, A, lam, s, nlb, has_ub, steps=3):
    """dense_box_jacobian with iterative refinement of K^-1, the residual I - K X evaluated in np.longdouble: the
    reference for d spread over many decades, where one fp64 solve of the order-(n + 2m + e) system loses digits."""
    n, m = Q.shape[0], lam.shape[0]
    e = 0 if (A is None or A.size == 0) else A.shape[0]
    G = dense_G(n, nlb, has_ub)
    Nk = n + 2 * m + e
    K = np.zeros((Nk, Nk))
    K[:n, :n] = Q
    K[:n, n + m:n + 2 * m] = G.T
    K[n:n + m, n:n + m] = np.diag(jm.clamped_d(lam, s))
    K[n:n + m, n + m:n + 2 * m] = np.eye(m)
    K[n + m:n + 2 * m, :n] = G
    K[n + m:n + 2 * m, n:n + m] = np.eye(m)
    if e:
        K[:n, n + 2 * m:] = A.T
        K[n + 2 * m:, :n] = A
    R = np.linalg.solve(K, np.eye(Nk))
    Kl = K.astype(np.longdouble)
    for _ in range(steps):
        res = (np.eye(Nk, dtype=np.longdouble) - Kl @ R.astype(np.longdouble)).astype(np.float64)
        R = R + np.linalg.solve(K, res)
    rows = np.concatenate([np.arange(n), n + m + np.arange(m), n + 2 * m + np.arange(e)])
    Jd = np.concatenate([-R[rows][:, :n], R[rows][:, n + m:n + 2 * m], R[rows][:, n + 2 * m:]], axis=1)
    cols = [Jd[:, :n]] + ([-Jd[:, n:n + nlb]] if nlb else []) + ([Jd[:, n + nlb:n + m]] if has_ub else [])
    return np.concatenate(cols + ([Jd[:, n + m:]] if e else []), axis=1)


def diagonal_box_jacobian(q, lam, s, nlb, has_ub):
    """dense_box_jacobian of a diagonal q without equality rows, from one KKT block per variable: with A empty the
    backward's system decouples into [q_j 0 g'; 0 D_j I; g I 0] over (z_j, the slacks and the duals of its sides),
    g = -1 for lb and +1 for ub. Each block (order 3 or 5) is inverted by Gauss-Jordan elimination in np.longdouble
    (pivots q_j, d, then the negative definite -(g g' / q_j + D_j^-1): no pivoting needed), and J is assembled from them:
    rows [z; lam], columns [p, lb, ub] of the sides given. The reference for widths whose dense model is too large."""
    n = q.shape[0]
    sides = ([-1.0] if nlb else []) + ([1.0] if has_ub else [])
    k = len(sides)
    d = jm.clamped_d(lam, s).astype(np.longdouble).reshape(k, n).T            # (n, k): d of variable j's sides
    o = 1 + 2 * k
    K = np.zeros((n, o, o), dtype=np.longdouble)
    K[:, 0, 0] = q
    for a, g in enumerate(sides):
        K[:, 0, 1 + k + a] = K[:, 1 + k + a, 0] = g
        K[:, 1 + a, 1 + a] = d[:, a]
        K[:, 1 + a, 1 + k + a] = K[:, 1 + k + a, 1 + a] = 1.0
    R = np.broadcast_to(np.eye(o, dtype=np.longdouble), (n, o, o)).copy()
    for c in range(o):
        piv = K[:, c, c].copy()
        K[:, c] /= piv[:, None]
        R[:, c] /= piv[:, None]
        for r in range(o):
            if r != c:
                f = K[:, r, c].copy()
                K[:, r] -= f[:, None] * K[:, c]
                R[:, r] -= f[:, None] * R[:, c]
    R = R.astype(np.float64)
    m = k * n
    J = np.zeros((n + m, n * (1 + k)))
    j = np.arange(n)
    rows = [j] + [n + a * n + j for a in range(k)]                             # z_j, then lam_j of each side
    for ri, r in enumerate(rows):
        slot = 0 if ri == 0 else 1 + k + (ri - 1)
        J[r, j] = -R[:, slot, 0]                                               # p: -R_.,x
        for a, g in enumerate(sides):                                          # h: R_.,(G x + s) of that side,
            J[r, n + a * n + j] = g * R[:, slot, 1 + k + a]                    # lb = -h, ub = h
    return J


def split(J, n, m, e, nlb, has_ub):
    """{(row name, column name): block} of a full [z; lam; nu] x [p, lb, ub, b] Jacobian."""
    rs = dict(z=(0, n), lam=(n, n + m), nu=(n + m, n + m + e))
    names = ["p"] + (["lb"] if nlb else []) + (["ub"] if has_ub else []) + (["b"] if e else [])
    cs, c0 = {}, 0
    for nm in names:
        w = e if nm == "b" else n
        cs[nm], c0 = (c0, c0 + w), c0 + w
    return {(r, c): J[r0:r1, c0:c1] for r, (r0, r1) in rs.items() for c, (c0, c1) in cs.items()}


def identity_residuals(J, n, m, e, nlb, has_ub, d):
    """Max abs of J_z,p = J_z,p', J_z,b = -J_nu,p', J_nu,b = J_nu,b', J_z,lb = -J_z,p diag(d_lb),
    J_z,ub = -J_z,p diag(d_ub); d: the clamped D."""
    B = split(J, n, m, e, nlb, has_ub)
    zp = B["z", "p"]
    res = [zp - zp.T]
    if e:
        res += [B["z", "b"] + B["nu", "p"].T, B["nu", "b"] - B["nu", "b"].T]
    if nlb:
        res.append(B["z", "lb"] + zp * d[:n][None, :])
    if has_ub:
        res.append(B["z", "ub"] + zp * d[nlb:][None, :])
    return max(float(np.abs(r).max()) for r in res)
