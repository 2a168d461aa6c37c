// qp_jac.cuh - the warp-level block steps of the Jacobian kernels (k_jacobian and k_box_jacobian in qp_jac.cu,
// k_boxq_jacobian in qp_boxq.cu): 8 right-hand-side columns per warp, buffers row-major with row stride 8. Every step is
// an 8x8 by 8x8 product, two mma.m8n8k4.f64, and a warp sweeps its block with __syncwarp only. Lane (g, q) =
// (lane >> 2, lane & 3) holds A[g][q], B[q][g] and C[g][2q..2q+1] of mma.m8n8k4 (dmma884). Include after qp_pf.cuh.
#pragma once

namespace {

using namespace qpb::pf;
using qpb::dmma884;

// Y = W U (ms_pad x 8; rows >= ms zero), W rows of stride ldw, columns < n read
__device__ __noinline__ void jac_wu(const double* __restrict__ Wg, int ldw, int n, int ms, int nts, int np,
                                   const double* U, double* Y) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
#pragma unroll 1
    for (int i = 0; i < nts; ++i) {
        const int r = 8 * i + g;
        const bool ok = r < ms;
        const double* Wr = Wg + (int64_t)(ok ? r : 0) * ldw;
        double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;       // two accumulator chains
#pragma unroll 4
        for (int k = 0; k < np; k += 8) {
            const double a0 = (ok && k + q < n) ? Wr[k + q] : 0.0, a1 = (ok && k + q + 4 < n) ? Wr[k + q + 4] : 0.0;
            dmma884(c0, c1, a0, U[(k + q) * 8 + g]);
            dmma884(e0, e1, a1, U[(k + q + 4) * 8 + g]);
        }
        *reinterpret_cast<double2*>(Y + r * 8 + 2 * q) = make_double2(c0 + e0, c1 + e1);
    }
    __syncwarp();
}

// U -= W' Y (nz_pad x 8)
__device__ __noinline__ void jac_u_minus_wty(const double* __restrict__ Wg, int ldw, int n, int ms, int ntz, int msp,
                                            const double* Y, double* U) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
#pragma unroll 1
    for (int i = 0; i < ntz; ++i) {
        const int cidx = 8 * i + g;                          // A[g][q] = W[k + q][cidx]
        const bool ok = cidx < n;
        double2 cv = *reinterpret_cast<const double2*>(U + cidx * 8 + 2 * q);
        double e0 = 0.0, e1 = 0.0;
#pragma unroll 4
        for (int k = 0; k < msp; k += 8) {
            const double a0 = (ok && k + q < ms) ? Wg[(int64_t)(k + q) * ldw + cidx] : 0.0;
            const double a1 = (ok && k + q + 4 < ms) ? Wg[(int64_t)(k + q + 4) * ldw + cidx] : 0.0;
            dmma884(cv.x, cv.y, -a0, Y[(k + q) * 8 + g]);
            dmma884(e0, e1, -a1, Y[(k + q + 4) * 8 + g]);
        }
        *reinterpret_cast<double2*>(U + cidx * 8 + 2 * q) = make_double2(cv.x + e0, cv.y + e1);
    }
    __syncwarp();
}

// Y = S^-1 Y with the product-form factor at M (T_k on the diagonal tiles, P_ik below): Y's block rows < kf are zero.
//     forward  Y_i -= P_ik Y_k (k ascending),  diagonal  Y_k = T_k' T_k Y_k,  backward  Y_k -= P_ik' Y_i (i descending)
// kFlip: M holds the factor of a bordered matrix L diag(I, -I) L' whose -I starts at block row kneg; the diagonal step
// negates those block rows, so Y = L^-T diag(I, -I) L^-1 Y.
template <bool kFlip>
__device__ __forceinline__ void jac_ssolve_t(const double* M, int nts, int kf, int kneg, double* Y) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
#pragma unroll 1
    for (int k = kf; k < nts - 1; ++k) {
        const int k0 = 8 * k;
        const double b0 = Y[(k0 + q) * 8 + g], b1 = Y[(k0 + q + 4) * 8 + g];
#pragma unroll 2
        for (int i = k + 1; i < nts; ++i) {
            const double* Pr = M + pf_rowoff(8 * i + g) + k0;
            double2* cp = reinterpret_cast<double2*>(Y + (8 * i + g) * 8 + 2 * q);
            double2 cv = *cp;
            dmma884(cv.x, cv.y, -Pr[q], b0);
            dmma884(cv.x, cv.y, -Pr[q + 4], b1);
            *cp = cv;
        }
        __syncwarp();
    }
#pragma unroll 1
    for (int k = kf; k < nts; ++k) {
        const int k0 = 8 * k;
        const double* Tg = M + pf_rowoff(k0 + g) + k0;       // row g of T_k (entries above the diagonal are not T)
        double z0 = 0.0, z1 = 0.0;
        dmma884(z0, z1, (q <= g) ? Tg[q] : 0.0, Y[(k0 + q) * 8 + g]);
        dmma884(z0, z1, (q + 4 <= g) ? Tg[q + 4] : 0.0, Y[(k0 + q + 4) * 8 + g]);
        __syncwarp();
        *reinterpret_cast<double2*>(Y + (k0 + g) * 8 + 2 * q) = make_double2(z0, z1);
        __syncwarp();
        const double t0 = (g <= q) ? M[pf_rowoff(k0 + q) + k0 + g] : 0.0;          // T'[g][q] = T[q][g]
        const double t1 = (g <= q + 4) ? M[pf_rowoff(k0 + q + 4) + k0 + g] : 0.0;
        double c0 = 0.0, c1 = 0.0;
        dmma884(c0, c1, t0, Y[(k0 + q) * 8 + g]);
        dmma884(c0, c1, t1, Y[(k0 + q + 4) * 8 + g]);
        __syncwarp();
        if (kFlip && k >= kneg) { c0 = -c0; c1 = -c1; }     // diag(I, -I) of a bordered factor L diag(I, -I) L'
        *reinterpret_cast<double2*>(Y + (k0 + g) * 8 + 2 * q) = make_double2(c0, c1);
    }
    __syncwarp();
#pragma unroll 1
    for (int i = nts - 1; i > 0; --i) {
        const int i0 = 8 * i;
        const double b0 = Y[(i0 + q) * 8 + g], b1 = Y[(i0 + q + 4) * 8 + g];
        const double* P0 = M + pf_rowoff(i0 + q) + g;        // A[g][q] = P_ik[q][g]
        const double* P1 = M + pf_rowoff(i0 + q + 4) + g;
#pragma unroll 2
        for (int k = 0; k < i; ++k) {
            double2* cp = reinterpret_cast<double2*>(Y + (8 * k + g) * 8 + 2 * q);
            double2 cv = *cp;
            dmma884(cv.x, cv.y, -P0[8 * k], b0);
            dmma884(cv.x, cv.y, -P1[8 * k], b1);
            *cp = cv;
        }
        __syncwarp();
    }
}


// the symmetric positive definite factor (k_jacobian, k_box_jacobian)
__device__ __noinline__ void jac_ssolve(const double* M, int nts, int kf, double* Y) { jac_ssolve_t<false>(M, nts, kf, 0, Y); }

// the bordered factor L diag(I, -I) L' of qp_boxq.cu, -I from block row kneg (k_boxq_jacobian)
__device__ __noinline__ void jac_ssolve_bordered(const double* M, int nts, int kf, int kneg, double* Y) {
    jac_ssolve_t<true>(M, nts, kf, kneg, Y);
}

// ---- the box Jacobians (qpb200_box_jacobian, qpb200_boxq_jacobian) -------------------------------------------------
// Row offsets of the z, lam, nu blocks and column offsets of the p, lb, ub, b blocks in one QP's R x C block of J
struct BOut {
    int R, C;
    int rz, rl, rn, cp, clb, cub, cb;
};

// J columns col0 + c (c < ncol) from a solved block (U = -z, Y = -nu of a p or b column, rows j0 + c the block's
// unit rows): kind 0 the p (or b) columns themselves, kind 1 / 2 the lb / ub columns of variables j0 + c, which are
// the p columns scaled by s = -d_lb_j / -d_ub_j. The lam rows are d_lb o (rz_lb - z) and d_ub o (rz_ub + z), with
// rz_lb = e_j in lb column j and rz_ub = -e_j in ub column j (zero otherwise).
__device__ __forceinline__ void box_jac_store(double* Jq, const BOut& O, int n, int nlb, int m, int e, const double* dv,
                                              const double* U, const double* Y, int kind, int col0, int j0, int ncol) {
    const int c = threadIdx.x & 7;                       // every idx a lane visits has idx & 7 == lane & 7
    if (c >= ncol) return;
    const int lane = threadIdx.x & 31, j = j0 + c;
    const double s = (kind == 0) ? 1.0 : -dv[(kind == 2 ? nlb : 0) + j];
    if (O.rz >= 0)
#pragma unroll 1
        for (int idx = lane; idx < 8 * n; idx += 32)
            Jq[(int64_t)(O.rz + (idx >> 3)) * O.C + col0 + c] = -s * U[idx];
    if (O.rl >= 0)
#pragma unroll 1
        for (int idx = lane; idx < 8 * m; idx += 32) {
            const int i = idx >> 3, lb = i < nlb, v = lb ? i : i - nlb;
            const double z = -s * U[v * 8 + c];
            const double v0 = lb ? (((kind == 1 && v == j) ? 1.0 : 0.0) - z) : (((kind == 2 && v == j) ? -1.0 : 0.0) + z);
            Jq[(int64_t)(O.rl + i) * O.C + col0 + c] = dv[i] * v0;
        }
    if (O.rn >= 0)
#pragma unroll 1
        for (int idx = lane; idx < 8 * e; idx += 32)
            Jq[(int64_t)(O.rn + (idx >> 3)) * O.C + col0 + c] = -s * Y[idx];
}

}  // namespace
