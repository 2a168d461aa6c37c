// qp_jac.cu - Jacobians of (z*, lam, nu) with respect to (p, h, b) at a returned point (qpb200_jacobian), and of box QPs
// with respect to (p, lb, ub, b) (qpb200_box_jacobian, below k_jacobian).
//
// The Jacobian is the negated inverse of the backward's symmetric system K = [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0],
// D = clamp(lam, 1e-8) / clamp(s, 1e-8). In the whitened form of DESIGN section 3, with V = W L^-1 (L = chol(Q),
// W = [A; 0; G] L^-T, equality rows first) and S = W W' + diag(0 on the equality rows, 1 on their padding, 1/d):
//     J_z,p = -L^-T L^-1 + V' S^-1 V      J_w,p = -S^-1 V      J_z,c = V' S^-1 E_c      J_w,c = -S^-1 E_c
// w = [nu; lam] in the row order of S, c a column of w (b columns: the equality rows, h columns: the inequality rows).
// Every 8-column block of right-hand sides is carried through the same steps:
//     p block j:  U = L^-1 E_j (block forward substitution with L), Y = S^-1 (W U)
//     w block c:  U = 0,                                             Y = S^-1 E_c
// and then J_w = -Y, J_z = -L^-T (U - W' Y).
//
// One CTA of 256 threads per QP. It forms S = W W' + diag from Wfac (DMMA, as k_setup_pf forms K) in the staircase of
// qp_pf.cuh, factors it once with pf_chol, and then each warp owns whole 8-column blocks: every substitution step is an
// 8x8 by 8x8 product, two mma.m8n8k4.f64, and a warp sweeps its block with __syncwarp only. L (packed lower) and W are
// read from global memory (L2); S's factor and each warp's two column buffers (nz_pad x 8 and ms_pad x 8) live in shared
// memory, and the number of warps that hold a block is what the shared memory left after the factor takes (jac_dims).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/qpth_b200.h"
#ifndef QPB_NT
#define QPB_NT 256
#endif
// the device functions of the headers have external linkage (host stubs): give this build its own namespace
#define qpb qpb_jac
#include "qp_pf.cuh"
#include "qp_jac.cuh"

extern "C" int qpb200_internal_set_smem(const void* kernel, size_t bytes);   // (qp_kernels.cu) the kernels' smem limits
extern "C" void qpb200_internal_cuda_error(int err, const char* what);     // (qp_kernels.cu) qpb200_last_cuda_error

namespace {

using namespace qpb::pf;
using qpb::dmma884;

constexpr int64_t kJacMaxSmem = 232448 - 1024;   // 227 KB opt-in limit per CTA on sm_90, minus static smem slack

// ---- shapes and shared-memory layout (doubles; every offset a multiple of 8) ----------------------------------------
struct JDims {
    int n, m, e, ep, ms, msp, nts, np, ntz;   // nz, nineq, neq, neq_pad, ms, ms_pad, ms_pad / 8, nz_pad, nz_pad / 8
    int ldw;
    int64_t lp;                               // doubles per system of Lfac
    int pan, tab, aug, blk, per;              // S at 0; panel scratch, tile table, pf_chol's running vector, buffers
    int nblk;                                 // column blocks in flight (warps holding buffers), 0: not covered
    int64_t smem;                             // dynamic shared memory, bytes
};

JDims jac_dims(const qpb200_plan* p) {
    JDims D{};
    D.n = p->nz; D.m = p->nineq; D.e = p->neq; D.ep = p->neq_pad; D.ms = p->ms; D.msp = p->ms_pad;
    D.nts = D.msp >> 3; D.np = (D.n + 7) & ~7; D.ntz = D.np >> 3;
    D.ldw = p->ldw; D.lp = p->L_elems;
    D.pan = pf_elems(D.nts);
    D.tab = D.pan + (8 * D.nts + 8) * kPanLd;
    D.aug = D.tab + ((pf_tab_doubles(D.nts) + 7) & ~7);
    D.blk = D.aug + 8 * D.nts;
    D.per = 8 * (D.np + D.msp);
    const int64_t left = kJacMaxSmem - 8 * (int64_t)D.blk;
    int64_t nb = left > 0 ? left / (8 * (int64_t)D.per) : 0;
    if (nb > kNT / 32) nb = kNT / 32;
    D.nblk = (D.m >= 1) ? (int)nb : 0;
    D.smem = D.nblk ? 8 * ((int64_t)D.blk + (int64_t)D.nblk * D.per) : 0;
    return D;
}

// Output placement: row offsets of the z, lam, nu blocks and column offsets of the p, h, b blocks in one QP's R x C
// block of J (-1: not requested)
struct JOut {
    int R, C;
    int rz, rl, rn, cp, ch, cb;
};

// ---- warp-level block steps (8 right-hand-side columns, buffers row-major with row stride 8) -------------------------
// Lane (g, q) = (lane >> 2, lane & 3) holds A[g][q], B[q][g] and C[g][2q..2q+1] of mma.m8n8k4 (dmma884).

// U = L^-1 E_j: block forward substitution with the packed lower L (rows >= n: identity), U's rows < 8 jb are zero.
__device__ __noinline__ void jac_lsolve(const double* __restrict__ Lg, int n, int ntz, int jb, double* U) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    for (int i = lane; i < 8 * jb * 8; i += 32) U[i] = 0.0;
#pragma unroll 1
    for (int i = jb; i < ntz; ++i) {
        const int r = 8 * i + g;
        double c0 = (i == jb && g == 2 * q) ? 1.0 : 0.0, c1 = (i == jb && g == 2 * q + 1) ? 1.0 : 0.0;
        const double* Lr = Lg + ((int64_t)r * (r + 1)) / 2;
#pragma unroll 2
        for (int k = jb; k < i; ++k) {
            const double a0 = (r < n) ? Lr[8 * k + q] : 0.0, a1 = (r < n) ? Lr[8 * k + q + 4] : 0.0;
            dmma884(c0, c1, -a0, U[(8 * k + q) * 8 + g]);
            dmma884(c0, c1, -a1, U[(8 * k + q + 4) * 8 + g]);
        }
        *reinterpret_cast<double2*>(U + r * 8 + 2 * q) = make_double2(c0, c1);
        __syncwarp();
        // L_ii x = c, column lane & 7 (every lane computes it; lanes < 8 store)
        const int c = lane & 7, i0 = 8 * i;
        double x[8];
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
            const int row = i0 + rr;
            double s = U[row * 8 + c];
            if (row < n) {
                const double* Lrr = Lg + ((int64_t)row * (row + 1)) / 2 + i0;
#pragma unroll
                for (int j = 0; j < rr; ++j) s = fma(-Lrr[j], x[j], s);
                s /= Lrr[rr];
            }
            x[rr] = s;
        }
        __syncwarp();
        if (lane < 8) {
#pragma unroll
            for (int rr = 0; rr < 8; ++rr) U[(i0 + rr) * 8 + c] = x[rr];
        }
        __syncwarp();
    }
}

// X = L^-T X in place (block backward substitution with the transpose of the packed lower L; rows >= n: identity)
__device__ __noinline__ void jac_ltsolve(const double* __restrict__ Lg, int n, int ntz, double* U) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
#pragma unroll 1
    for (int i = ntz - 1; i >= 0; --i) {
        const int i0 = 8 * i;
        double2 cv = *reinterpret_cast<const double2*>(U + (i0 + g) * 8 + 2 * q);
        const bool col = i0 + g < n;
#pragma unroll 2
        for (int k = i + 1; k < ntz; ++k) {
            const int r0 = 8 * k + q, r1 = r0 + 4;          // A[g][q] = L[r][i0 + g]
            const double a0 = (col && r0 < n) ? Lg[((int64_t)r0 * (r0 + 1)) / 2 + i0 + g] : 0.0;
            const double a1 = (col && r1 < n) ? Lg[((int64_t)r1 * (r1 + 1)) / 2 + i0 + g] : 0.0;
            dmma884(cv.x, cv.y, -a0, U[r0 * 8 + g]);
            dmma884(cv.x, cv.y, -a1, U[r1 * 8 + g]);
        }
        *reinterpret_cast<double2*>(U + (i0 + g) * 8 + 2 * q) = cv;
        __syncwarp();
        // L_ii' x = c, rows from the bottom up
        const int c = lane & 7;
        double x[8];
#pragma unroll
        for (int rr = 7; rr >= 0; --rr) {
            const int row = i0 + rr;
            double s = U[row * 8 + c];
            if (row < n) {
#pragma unroll
                for (int j = rr + 1; j < 8; ++j)
                    if (i0 + j < n) s = fma(-Lg[((int64_t)(i0 + j) * (i0 + j + 1)) / 2 + row], x[j], s);
                s /= Lg[((int64_t)row * (row + 1)) / 2 + row];
            }
            x[rr] = s;
        }
        __syncwarp();
        if (lane < 8) {
#pragma unroll
            for (int rr = 0; rr < 8; ++rr) U[(i0 + rr) * 8 + c] = x[rr];
        }
        __syncwarp();
    }
}

// J rows [row0, row0 + cnt) <- -B[src0 + ..] (8 columns at column col0, the first ncol of them valid)
__device__ __forceinline__ void jac_store(double* Jq, const JOut& O, int row0, int cnt, const double* B, int src0,
                                          int col0, int ncol) {
    const int lane = threadIdx.x & 31;
    for (int idx = lane; idx < 8 * cnt; idx += 32) {
        const int r = idx >> 3, c = idx & 7;
        if (c < ncol) Jq[(int64_t)(row0 + r) * O.C + col0 + c] = -B[(src0 + r) * 8 + c];
    }
}

__global__ void __launch_bounds__(kNT, 1)
k_jacobian(JDims D, JOut O, const double* __restrict__ lam, const double* __restrict__ slk,
           const double* __restrict__ Lfac, const double* __restrict__ Wfac, int sF, double* __restrict__ J) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, q = lane & 3;
    const int64_t qp = blockIdx.x, sys = sF ? qp : 0;
    const int n = D.n, e = D.e, ep = D.ep, ms = D.ms, nts = D.nts;
    const double* Lg = Lfac + sys * D.lp;
    const double* Wg = Wfac + sys * (int64_t)ms * D.ldw;
    const double* lq = lam + qp * D.m;
    const double* sq = slk + qp * D.m;
    double* M = qsm;
    // ---- 1. S = W W' + diag(0 on the equality rows, 1 on their padding and past ms, 1/d) -> staircase (lower tiles)
    {
        const int T2 = nts * (nts + 1) / 2;
#pragma unroll 1
        for (int t = warp; t < T2; t += kNT / 32) {
            int ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while (ti * (ti + 1) / 2 > t) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
            const int tj = t - ti * (ti + 1) / 2;
            const int ra = 8 * ti + g, rb = 8 * tj + g;
            const bool oka = ra < ms, okb = rb < ms;
            const double* pa = Wg + (int64_t)(oka ? ra : 0) * D.ldw;
            const double* pb = Wg + (int64_t)(okb ? rb : 0) * D.ldw;
            double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;   // two accumulator chains
#pragma unroll 4
            for (int kk = 0; kk < D.np; kk += 8) {
                const bool k0 = kk + q < n, k1 = kk + q + 4 < n;
                dmma884(c0, c1, (oka && k0) ? pa[kk + q] : 0.0, (okb && k0) ? pb[kk + q] : 0.0);
                dmma884(e0, e1, (oka && k1) ? pa[kk + q + 4] : 0.0, (okb && k1) ? pb[kk + q + 4] : 0.0);
            }
            const int rr = 8 * ti + g, cc = 8 * tj + 2 * q;
            double v0 = c0 + e0, v1 = c1 + e1;
            if (rr == cc || rr == cc + 1) {
                double dg = 1.0;                             // equality padding rows, rows past ms
                if (rr < e) dg = 0.0;
                else if (rr >= ep && rr < ms)
                    dg = fmax(sq[rr - ep], 1e-8) / fmax(lq[rr - ep], 1e-8);   // 1 / d, the backward's clamps
                if (rr == cc) v0 += dg; else v1 += dg;
            }
            *reinterpret_cast<double2*>(M + pf_rowoff(rr) + cc) = make_double2(v0, v1);
        }
    }
    for (int i = tid; i < 8 * nts; i += kNT) qsm[D.aug + i] = 0.0;
    pf_build_tab(D.tab, nts);
    __syncthreads();
    // ---- 2. S = L_S L_S' in product form
    pf_chol(0, nts, 0, D.aug, D.pan, D.tab);
    __syncthreads();
    // ---- 3. column blocks: p blocks, then the b (equality) and h (inequality) tiles of w, one warp per block
    if (warp >= D.nblk) return;
    double* U = qsm + D.blk + (int64_t)warp * D.per;
    double* Y = U + 8 * D.np;
    const int npb = (O.cp >= 0) ? D.ntz : 0;
    const int ebeg = (O.cb >= 0) ? 0 : (ep >> 3), eend = (O.ch >= 0) ? nts : (ep >> 3);
    const int nblocks = npb + (eend - ebeg);
    double* Jq = J + qp * (int64_t)O.R * O.C;
#pragma unroll 1
    for (int t = warp; t < nblocks; t += D.nblk) {
        int kf = 0, col0 = 0, ncol = 0;
        if (t < npb) {                                       // p block t: U = L^-1 E_t, Y = W U
            jac_lsolve(Lg, n, D.ntz, t, U);
            jac_wu(Wg, D.ldw, n, ms, nts, D.np, U, Y);
            col0 = O.cp + 8 * t;
            ncol = min(8, n - 8 * t);
        } else {                                             // w tile c: U = 0, Y = E_c
            const int c = ebeg + (t - npb);
            for (int i = lane; i < 8 * D.np; i += 32) U[i] = 0.0;
            for (int i = lane; i < 8 * D.msp; i += 32) Y[i] = ((i >> 3) == 8 * c + (i & 7)) ? 1.0 : 0.0;
            kf = c;
            if (8 * c < ep) { col0 = O.cb + 8 * c; ncol = min(8, e - 8 * c); }
            else { col0 = O.ch + 8 * c - ep; ncol = min(8, ms - 8 * c); }
            __syncwarp();
        }
        jac_ssolve(M, nts, kf, Y);
        if (O.rn >= 0) jac_store(Jq, O, O.rn, e, Y, 0, col0, ncol);
        if (O.rl >= 0) jac_store(Jq, O, O.rl, D.m, Y, ep, col0, ncol);
        if (O.rz >= 0) {
            jac_u_minus_wty(Wg, D.ldw, n, ms, D.ntz, D.msp, Y, U);
            jac_ltsolve(Lg, n, D.ntz, U);
            jac_store(Jq, O, O.rz, n, U, 0, col0, ncol);
        }
        __syncwarp();
    }
}

// ---- BoxQPFunction, diagonal Q (qpb200_box_jacobian) -----------------------------------------------------------------
// With Q = diag(q) and G = [-I; I] the inequality block is eliminated as in the box kernels: H = q + d_lb + d_ub
// (diagonal), M = A H^-1 A' (order neq), and with K_b = [H A'; A 0]
//     p block j:  U = H^-1 E_j, Y = M^-1 (A U),   z = -H^-1 (E_j - A'Y),   nu = -Y
//     b block c:  Y = M^-1 E_c,                     z =  H^-1 A'Y,           nu = -Y
// i.e. the steps of k_jacobian with W = A and L = H^(1/2), whose triangular solves become a diagonal scaling. The lb and
// ub columns are the p columns scaled by -d_lb_j / -d_ub_j, and the lam rows d_lb o (rz_lb - z), d_ub o (rz_ub + z), so
// they are written from the p blocks' solves (box_jac_store). One CTA of 256 threads per QP; A (row stride nz) is read
// from global memory (L2); M's staircase, H^-1, d and the warps' column buffers (nz_pad x 8 and neq_pad x 8) live in
// shared memory. It does not use the forward's layout: any box plan whose buffers fit is covered.
struct BDims {
    int n, m, e, ep, nlb, nts, np, ntz;       // nz, nineq, neq, neq_pad, nz if lb given else 0, neq_pad / 8, nz_pad, / 8
    int pan, tab, aug, hv, dv, blk, per;      // M at 0; panel, tile table, pf_chol's vector, H^-1, d, buffers
    int nblk;                                 // column blocks in flight, 0: not covered
    int64_t smem;                             // dynamic shared memory, bytes
};

BDims box_jac_dims(const qpb200_box_plan* p) {
    BDims D{};
    D.n = p->nz; D.m = p->nineq; D.e = p->neq; D.ep = p->neq_pad; D.nlb = p->has_lb ? p->nz : 0;
    D.nts = D.ep >> 3; D.np = (D.n + 7) & ~7; D.ntz = D.np >> 3;
    D.pan = pf_elems(D.nts);
    D.tab = D.pan + (8 * D.nts + 8) * kPanLd;
    D.aug = D.tab + ((pf_tab_doubles(D.nts) + 7) & ~7);
    D.hv = D.aug + 8 * D.nts;
    D.dv = D.hv + D.np;
    D.blk = D.dv + ((D.m + 7) & ~7);
    D.per = 8 * (D.np + D.ep);
    const int64_t left = kJacMaxSmem - 8 * (int64_t)D.blk;
    int64_t nb = left > 0 ? left / (8 * (int64_t)D.per) : 0;
    if (nb > kNT / 32) nb = kNT / 32;
    D.nblk = (int)nb;
    D.smem = D.nblk ? 8 * ((int64_t)D.blk + (int64_t)D.nblk * D.per) : 0;
    return D;
}

__global__ void __launch_bounds__(kNT, 1)
k_box_jacobian(BDims D, BOut O, const double* __restrict__ q, int64_t sq, const double* __restrict__ A, int64_t sA,
               const double* __restrict__ lam, const double* __restrict__ slk, double* __restrict__ J) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, q4 = lane & 3;
    const int64_t qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, nts = D.nts, np = D.np;
    const double* qv = q + qp * sq;
    const double* Ag = (e > 0) ? A + qp * sA : nullptr;
    double* hv = qsm + D.hv;
    double* dv = qsm + D.dv;
    // ---- 1. d = clamp(lam, 1e-8) / clamp(s, 1e-8) as the backward forms it, H^-1 (0 past nz)
    for (int i = tid; i < m; i += kNT) dv[i] = fmax(lam[qp * m + i], 1e-8) / fmax(slk[qp * m + i], 1e-8);
    __syncthreads();
    for (int j = tid; j < np; j += kNT) {
        double h = 0.0;
        if (j < n) {
            h = qv[j];
            if (D.nlb) h += dv[j];
            if (m > D.nlb) h += dv[D.nlb + j];
            h = 1.0 / h;
        }
        hv[j] = h;
    }
    __syncthreads();
    // ---- 2. M = A H^-1 A' (identity past neq) -> staircase (lower tiles), M = L_M L_M' in product form
    if (e > 0) {
        const int T2 = nts * (nts + 1) / 2;
#pragma unroll 1
        for (int t = warp; t < T2; t += kNT / 32) {
            int ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while (ti * (ti + 1) / 2 > t) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
            const int tj = t - ti * (ti + 1) / 2;
            const int ra = 8 * ti + g, rb = 8 * tj + g;
            const bool oka = ra < e, okb = rb < e;
            const double* pa = Ag + (int64_t)(oka ? ra : 0) * n;
            const double* pb = Ag + (int64_t)(okb ? rb : 0) * n;
            double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;   // two accumulator chains
#pragma unroll 4
            for (int kk = 0; kk < np; kk += 8) {
                const bool k0 = kk + q4 < n, k1 = kk + q4 + 4 < n;
                dmma884(c0, c1, (oka && k0) ? pa[kk + q4] * hv[kk + q4] : 0.0, (okb && k0) ? pb[kk + q4] : 0.0);
                dmma884(e0, e1, (oka && k1) ? pa[kk + q4 + 4] * hv[kk + q4 + 4] : 0.0, (okb && k1) ? pb[kk + q4 + 4] : 0.0);
            }
            const int rr = 8 * ti + g, cc = 8 * tj + 2 * q4;
            double v0 = c0 + e0, v1 = c1 + e1;
            if (rr >= e) {                                   // padding rows: identity
                if (rr == cc) v0 = 1.0;
                if (rr == cc + 1) v1 = 1.0;
            }
            *reinterpret_cast<double2*>(qsm + pf_rowoff(rr) + cc) = make_double2(v0, v1);
        }
        for (int i = tid; i < 8 * nts; i += kNT) qsm[D.aug + i] = 0.0;
        pf_build_tab(D.tab, nts);
        __syncthreads();
        pf_chol(0, nts, 0, D.aug, D.pan, D.tab);
        __syncthreads();
    }
    // ---- 3. column blocks: p blocks (which also give the lb and ub columns), then the b tiles, one warp per block
    if (warp >= D.nblk) return;
    double* U = qsm + D.blk + (int64_t)warp * D.per;
    double* Y = U + 8 * np;
    const int npb = (O.cp >= 0 || O.clb >= 0 || O.cub >= 0) ? D.ntz : 0;
    const int nblocks = npb + ((O.cb >= 0) ? nts : 0);
    double* Jq = J + qp * (int64_t)O.R * O.C;
#pragma unroll 1
    for (int t = warp; t < nblocks; t += D.nblk) {
        const bool pblk = t < npb;
        const int j0 = 8 * (pblk ? t : t - npb);
        if (pblk) {                                          // Y = A H^-1 E_t, then U = E_t
            for (int i = lane; i < 8 * np; i += 32) U[i] = ((i >> 3) == j0 + (i & 7)) ? hv[i >> 3] : 0.0;
            __syncwarp();
            jac_wu(Ag, n, n, e, nts, np, U, Y);
            for (int i = lane; i < 8 * np; i += 32) U[i] = ((i >> 3) == j0 + (i & 7)) ? 1.0 : 0.0;
        } else {                                             // U = 0, Y = E_c
            for (int i = lane; i < 8 * np; i += 32) U[i] = 0.0;
            for (int i = lane; i < 8 * D.ep; i += 32) Y[i] = ((i >> 3) == j0 + (i & 7)) ? 1.0 : 0.0;
        }
        __syncwarp();
        jac_ssolve(qsm, nts, pblk ? 0 : (j0 >> 3), Y);
        jac_u_minus_wty(Ag, n, n, e, D.ntz, D.ep, Y, U);
        for (int i = lane; i < 8 * np; i += 32) U[i] *= hv[i >> 3];
        __syncwarp();
        // a p block: its p, lb and ub columns (kind 0, 1, 2); a b tile: its b columns
#pragma unroll 1
        for (int kind = 0; kind < (pblk ? 3 : 1); ++kind) {
            const int c0 = pblk ? (kind == 0 ? O.cp : (kind == 1 ? O.clb : O.cub)) : O.cb;
            if (c0 >= 0) box_jac_store(Jq, O, D.n, D.nlb, D.m, D.e, dv, U, Y, kind, c0 + j0, j0, min(8, (pblk ? n : e) - j0));
        }
        __syncwarp();
    }
}

}  // namespace

extern "C" {

int qpb200_jacobian_smem(const qpb200_plan* plan, int64_t* smem_bytes) {
    if (!plan || !smem_bytes) return QPB200_ERR_BAD_ARG;
    if (plan->nz <= 0 || plan->nineq < 0 || plan->neq < 0 || plan->ms_pad <= 0) return QPB200_ERR_BAD_ARG;
    *smem_bytes = jac_dims(plan).smem;
    return QPB200_OK;
}

int qpb200_jacobian(const qpb200_plan* plan, int nbatch, int rows, int cols, const double* lam, const double* slacks,
                    const double* Lfac, const double* Wfac, int sF, double* J, void* stream) {
    if (!plan || !lam || !slacks || !Lfac || !Wfac || !J || nbatch < 1) return QPB200_ERR_BAD_ARG;
    if (rows <= 0 || cols <= 0 || (rows & ~7) || (cols & ~7) || (sF != 0 && sF != 1)) return QPB200_ERR_BAD_ARG;
    if (plan->nz <= 0 || plan->nineq < 0 || plan->neq < 0 || plan->ms_pad <= 0) return QPB200_ERR_BAD_ARG;
    if (plan->neq == 0 && ((rows & 4) || (cols & 4))) return QPB200_ERR_BAD_ARG;
    const JDims D = jac_dims(plan);
    if (D.nblk < 1) return QPB200_ERR_TOO_LARGE;
    JOut O;
    int off = 0;
    O.rz = (rows & 1) ? off : -1; off += (rows & 1) ? D.n : 0;
    O.rl = (rows & 2) ? off : -1; off += (rows & 2) ? D.m : 0;
    O.rn = (rows & 4) ? off : -1; off += (rows & 4) ? D.e : 0;
    O.R = off; off = 0;
    O.cp = (cols & 1) ? off : -1; off += (cols & 1) ? D.n : 0;
    O.ch = (cols & 2) ? off : -1; off += (cols & 2) ? D.m : 0;
    O.cb = (cols & 4) ? off : -1; off += (cols & 4) ? D.e : 0;
    O.C = off;
    int rc = qpb200_internal_set_smem((const void*)k_jacobian, (size_t)D.smem);
    if (rc) return rc;
    k_jacobian<<<nbatch, kNT, (size_t)D.smem, (cudaStream_t)stream>>>(D, O, lam, slacks, Lfac, Wfac, sF, J);
    const cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, "k_jacobian"); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}

int qpb200_box_jacobian_smem(const qpb200_box_plan* plan, int64_t* smem_bytes) {
    if (!plan || !smem_bytes) return QPB200_ERR_BAD_ARG;
    if (plan->nz <= 0 || plan->neq < 0 || plan->neq_pad != ((plan->neq + 7) & ~7) ||
        plan->nineq != (plan->has_lb + plan->has_ub) * plan->nz || plan->nineq <= 0)
        return QPB200_ERR_BAD_ARG;
    *smem_bytes = box_jac_dims(plan).smem;
    return QPB200_OK;
}

int qpb200_box_jacobian(const qpb200_box_plan* plan, int nbatch, int rows, int cols, const double* q, int64_t sq,
                        const double* A, int64_t sA, const double* lam, const double* slacks, double* J, void* stream) {
    int64_t smem = 0;
    int rc = qpb200_box_jacobian_smem(plan, &smem);
    if (rc) return rc;
    if (!q || !lam || !slacks || !J || nbatch < 1 || sq < 0 || sA < 0) return QPB200_ERR_BAD_ARG;
    if (rows <= 0 || cols <= 0 || (rows & ~7) || (cols & ~15)) return QPB200_ERR_BAD_ARG;
    if (plan->neq == 0 && ((rows & 4) || (cols & 8))) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && !A) return QPB200_ERR_BAD_ARG;
    if (((cols & 2) && !plan->has_lb) || ((cols & 4) && !plan->has_ub)) return QPB200_ERR_BAD_ARG;
    if (smem == 0) return QPB200_ERR_TOO_LARGE;
    const BDims D = box_jac_dims(plan);
    BOut O;
    int off = 0;
    O.rz = (rows & 1) ? off : -1; off += (rows & 1) ? D.n : 0;
    O.rl = (rows & 2) ? off : -1; off += (rows & 2) ? D.m : 0;
    O.rn = (rows & 4) ? off : -1; off += (rows & 4) ? D.e : 0;
    O.R = off; off = 0;
    O.cp = (cols & 1) ? off : -1; off += (cols & 1) ? D.n : 0;
    O.clb = (cols & 2) ? off : -1; off += (cols & 2) ? D.n : 0;
    O.cub = (cols & 4) ? off : -1; off += (cols & 4) ? D.n : 0;
    O.cb = (cols & 8) ? off : -1; off += (cols & 8) ? D.e : 0;
    O.C = off;
    rc = qpb200_internal_set_smem((const void*)k_box_jacobian, (size_t)D.smem);
    if (rc) return rc;
    k_box_jacobian<<<nbatch, kNT, (size_t)D.smem, (cudaStream_t)stream>>>(D, O, q, sq, A, sA, lam, slacks, J);
    const cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, "k_box_jacobian"); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}

}  // extern "C"
