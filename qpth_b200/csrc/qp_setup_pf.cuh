// k_setup_pf: pre_factor_kkt (batch.py:375-429) on the product-form machinery, sized to share an SM. Included by
// qp_kernels.cu (kNT = 256: two per SM, latency mode and large shapes) and by qp_alt.cu (kNT = 192: three per SM next to
// the three-per-SM forward / backward CTAs, throughput mode).
//   1. lower triangle of Q -> staircase in shared memory; pf_chol factors it IN PRODUCT FORM (T_k, P_ik). The panel
//      warps emit the plain factor's off-diagonal tiles L_ik to global memory as they appear; the pivot-chain warp only
//      parks the strictly lower part of each L_kk in the unused upper triangle of its diagonal tile, and every thread
//      emits the diagonal blocks of L (true diagonal = 1 / diagonal of T_k) after the factorization;
//   2. W = [A; 0; G] L^-T on every warp, one 8-row tile per warp with the tile in registers (pf_w_rowtile);
//   3. K = W W^T (DMMA, operands re-read from L2: W was written by this CTA) into the staircase that held chol(Q);
//   4. equality block: the first neq_pad columns of K factored in product form by the same pf_chol (kend), K -> global.
// Shared memory: staircase of order max(nz_pad, ms_pad) + panel scratch + vector + tile table: 60.9 KB at C2 (three per
// SM fit next to the 76,240 B forward CTAs; k_setup_fast holds Q and W side by side: 181 KB, one per SM), 194 KB at
// nz = nineq = 200 (where the only other setup kernel works from global scratch on one CTA).
#pragma once
#include "qp_common.cuh"
#include "qp_pf.cuh"

namespace {
namespace fk {
struct PLayout { int SQ, pan, aug, tab, total; };
__host__ __device__ inline PLayout setup_pf_layout(const KDims& D) {
    PLayout L;
    const int np = (D.n + 7) & ~7;
    const int ord = np > D.msp ? np : D.msp;
    const int nts = ord >> 3;
    L.SQ = 0;
    L.pan = qpb::pf::pf_elems(nts) - 8 * qpb::pf::kPanLd;   // (its first 8 rows are never touched: overlap the staircase)
    L.aug = L.pan + (ord + 8) * qpb::pf::kPanLd;
    L.tab = L.aug + ord;
    L.total = L.tab + ((qpb::pf::pf_tab_doubles(nts) + 1) & ~1);
    return L;
}

constexpr int kWRegT = 13;      // block columns of a W row tile held in registers at a time (all of them up to nz = 104)

// Rows 8 rt .. 8 rt + 7 of W = [A; 0; G] L^-T, i.e. the forward substitution L W_r^T = X_r^T of one 8-row tile X_r, by
// one warp with the tile in registers. The accumulator fragment of a DMMA 8x8x4 (lane (g, q): columns 2q, 2q+1 of row g)
// also serves as its A operand when the k index is permuted: one DMMA takes the even columns, the other the odd ones,
// and the B fragment (lane (g, q): B[q][g]) becomes the 16-byte pair P_ik[g][2q .. 2q+1] of the staircase. Per block
// column k: y_k = x_k T_k^T -> W, and x_i -= x_k P_ik^T for i > k (running right-hand side). Block columns beyond the
// first kWRegT are done kWRegT at a time; the finished columns k of the earlier chunks enter as x_i -= y_k L_ik^T with
// y_k re-read from W (this lane's own stores) and L_ik from the plain factor in global memory.
__device__ __forceinline__ void pf_w_rowtile(const KDims& D, const double* SQ, const double* Ag, const double* Gg,
                                             const double* Lg, double* Wg, int rt) {
    using namespace qpb::pf;
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int n = D.n, ntq = (n + 7) >> 3;
    const int wrow = 8 * rt + g;                            // this lane's row of W
    const bool live = wrow < D.ms;
    const double* src = nullptr;
    if (wrow < D.e) src = Ag + (int64_t)wrow * n;
    else if (wrow >= D.ep && live) src = Gg + (int64_t)(wrow - D.ep) * n;
    double* wr = Wg + (int64_t)(live ? wrow : 0) * D.ldw;
#pragma unroll 1
    for (int c0 = 0; c0 < ntq; c0 += kWRegT) {
        double x0[kWRegT], x1[kWRegT];                       // columns 8 (c0 + j) + 2q, + 1
#pragma unroll
        for (int j = 0; j < kWRegT; ++j) {
            const int c = 8 * (c0 + j) + 2 * q;
            x0[j] = (src != nullptr && c < n) ? src[c] : 0.0;
            x1[j] = (src != nullptr && c + 1 < n) ? src[c + 1] : 0.0;
        }
#pragma unroll 1
        for (int k = 0; k < c0; ++k) {                       // earlier chunks: x_i -= y_k L_ik^T
            const int c = 8 * k + 2 * q;
            const double y0 = (live && c < n) ? wr[c] : 0.0, y1 = (live && c + 1 < n) ? wr[c + 1] : 0.0;
            int gk = g;
            asm volatile("" : "+r"(gk));                     // (recompute the 13 row addresses per k instead of spilling them)
#pragma unroll
            for (int i = 0; i < kWRegT; ++i) {
                const int R = 8 * (c0 + i) + gk;
                const double* lr = Lg + ((int64_t)R * (R + 1)) / 2 + c;
                const double l0 = (R < n) ? lr[0] : 0.0, l1 = (R < n) ? lr[1] : 0.0;
                dmma884(x0[i], x1[i], -y0, l0);
                dmma884(x0[i], x1[i], -y1, l1);
            }
        }
#pragma unroll
        for (int j = 0; j < kWRegT; ++j) {
            const int k = c0 + j, k0 = 8 * k;
            if (k < ntq) {                                   // (warp-uniform)
#pragma unroll
                for (int i = j + 1; i < kWRegT; ++i) {      // running right-hand side, block k+1 first
                    if (c0 + i < ntq) {
                        const double2 p = *reinterpret_cast<const double2*>(SQ + pf_rowoff(8 * (c0 + i) + g) + k0 + 2 * q);
                        dmma884(x0[i], x1[i], -x0[j], p.x);
                        dmma884(x0[i], x1[i], -x1[j], p.y);
                    }
                }
                // y_k = x_k T_k^T (T_k: lower triangle of the diagonal tile; its upper triangle holds the parked L_kk)
                const double2 t = *reinterpret_cast<const double2*>(SQ + pf_rowoff(k0 + g) + k0 + 2 * q);
                double d0 = 0.0, d1 = 0.0;
                dmma884(d0, d1, x0[j], (2 * q <= g) ? t.x : 0.0);
                dmma884(d0, d1, x1[j], (2 * q + 1 <= g) ? t.y : 0.0);
                if (live) {
                    if (k0 + 2 * q < n) wr[k0 + 2 * q] = d0;
                    if (k0 + 2 * q + 1 < n) wr[k0 + 2 * q + 1] = d1;
                }
            }
        }
    }
    if (live && q == 0)
        for (int c = n; c < D.ldw; ++c) wr[c] = 0.0;        // (padding columns of the W layout)
}
}  // namespace fk

template <int kMinCtas>
__global__ void __launch_bounds__(qpb::fast::kNT, kMinCtas)
k_setup_pf(KDims D, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ G, int64_t sG,
           const double* __restrict__ A, int64_t sA, double* __restrict__ Lfac, double* __restrict__ Wfac,
           double* __restrict__ Kfac, int* __restrict__ spd_flag) {
    using namespace fk;
    using namespace qpb::pf;
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, q = lane & 3;
    const int sys = blockIdx.x;
    const int n = D.n, e = D.e, ep = D.ep, ms = D.ms, msp = D.msp;
    const PLayout PL = setup_pf_layout(D);
    const int np = (n + 7) & ~7, ntq = np >> 3, nts = msp >> 3;
    const int ntsq = (np > msp ? np : msp) >> 3;
    const double* Qg = Q + (int64_t)sys * sQ;
    const double* Gg = G + (int64_t)sys * sG;
    const double* Ag = (e > 0) ? (A + (int64_t)sys * sA) : nullptr;
    double* Lg = Lfac + (int64_t)sys * D.lp;
    double* Wg = Wfac + (int64_t)sys * ms * D.ldw;
    double* Kg = Kfac + (int64_t)sys * pf_elems(nts);
    double* SQ = qsm + PL.SQ;
    __shared__ int s_flag;
    if (tid == 0) s_flag = 0;
#ifdef QPB_TIMING
    if (threadIdx.x == 0) { for (int i = 0; i < 128; ++i) s_tim[i] = 0; s_tim[128] = clock64(); s_tim2 = s_tim[128]; }
    __syncthreads();
#endif
    // ---- 1. Q (lower triangle, identity padded, + eps I in the regularised variant) -> staircase. Bound by the latency
    // of the loads of Q: a warp takes four rows of one block row at a time, 16 loads in flight per lane.
    for (int r0 = 4 * warp; r0 < np; r0 += 4 * (kNT / 32)) {
        const int len = 8 * (r0 >> 3) + 8;
        for (int cb = 0; cb < len; cb += 128) {
            double v[4][4];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    const int r = r0 + a, c = cb + 32 * b + lane;
                    v[a][b] = (r == c) ? 1.0 : 0.0;
                    if (r < n && c < n && c < len) v[a][b] = Qg[(int64_t)r * n + c] + ((r == c) ? D.reg : 0.0);
                }
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    const int c = cb + 32 * b + lane;
                    if (c < len) SQ[pf_rowoff(r0 + a) + c] = v[a][b];
                }
        }
    }
    for (int i = tid; i < (ntsq << 3); i += kNT) qsm[PL.aug + i] = 0.0;
    pf_build_tab(PL.tab, ntsq);
    __syncthreads();
    QPB_TICK(34);   // staging
    pf_chol_setup(PL.SQ, ntq, 0, ntq, PL.aug, PL.pan, PL.tab, Lg, n);
    QPB_TICK(35);   // chol(Q)
    // SPD check (qp.py:81-85): every reciprocal pivot (diagonal of the T_k) must be a positive finite number. The same
    // pass emits the diagonal blocks of L: row i's strictly lower entries from where the chain warp parked them.
    for (int i = tid; i < n; i += kNT) {
        const double ri = SQ[pf_rowoff(i) + i];
        if (!(ri > 0.0) || isinf(ri)) s_flag = 1;
        const int k0 = i & ~7, r = i & 7;
        const double* parked = SQ + pf_rowoff(k0 + 7 - r) + k0 + 8 - r;
        double* row = Lg + ((int64_t)i * (i + 1)) / 2 + k0;
        for (int c = 0; c < r; ++c) row[c] = parked[c];
        row[r] = 1.0 / ri;
    }
    if (tid == 0 && (D.lp > n * (n + 1) / 2)) Lg[D.lp - 1] = 0.0;
    // ---- 2. W = [A; 0; G] L^-T, one row tile per warp (reads the T_k, P_ik and the off-diagonal L_ik emitted before the
    // last barrier of pf_chol_setup)
    for (int rt = warp; rt < nts; rt += kNT / 32) pf_w_rowtile(D, SQ, Ag, Gg, Lg, Wg, rt);
    __syncthreads();                                         // W is in global memory (visible to the block), chol(Q) is dead
    QPB_TICK(37);   // W
    if (tid == 0) spd_flag[sys] = s_flag;
    // ---- 3. K = W W^T -> staircase (lower tiles), unit diagonal on dummy / pad rows, + eps on the real equality rows
    {
        const int T2 = nts * (nts + 1) / 2;
        for (int t = warp; t < T2; t += kNT / 32) {
            int ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while (ti * (ti + 1) / 2 > t) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
            const int tj = t - ti * (ti + 1) / 2;
            const int ra = 8 * ti + g, rb = 8 * tj + g;
            const double* pa = Wg + (int64_t)(ra < ms ? ra : 0) * D.ldw + q;
            const double* pb = Wg + (int64_t)(rb < ms ? rb : 0) * D.ldw + q;
            const bool oka = ra < ms, okb = rb < ms;
            double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;   // two accumulator chains
            // W comes back from L2 (written by this CTA in step 2): 28 loads in flight per lane, then their 14 DMMAs
#pragma unroll 1
            for (int kk0 = 0; kk0 < np; kk0 += 56) {
                double x0[7], y0[7], x1[7], y1[7];
#pragma unroll
                for (int u = 0; u < 7; ++u) {
                    const int kk = kk0 + 8 * u;
                    x0[u] = (oka && kk + q < n) ? pa[kk] : 0.0;
                    y0[u] = (okb && kk + q < n) ? pb[kk] : 0.0;
                    x1[u] = (oka && kk + 4 + q < n) ? pa[kk + 4] : 0.0;
                    y1[u] = (okb && kk + 4 + q < n) ? pb[kk + 4] : 0.0;
                }
#pragma unroll
                for (int u = 0; u < 7; ++u) {
                    if (kk0 + 8 * u < np) {                  // (warp-uniform)
                        dmma884(c0, c1, x0[u], y0[u]);
                        dmma884(e0, e1, x1[u], y1[u]);
                    }
                }
            }
            const int rr = 8 * ti + g, cc = 8 * tj + 2 * q;
            double v0 = c0 + e0, v1 = c1 + e1;
            if (rr == cc && ((rr >= e && rr < ep) || rr >= ms)) v0 += 1.0;
            if (rr == cc + 1 && ((rr >= e && rr < ep) || rr >= ms)) v1 += 1.0;
            if (rr == cc && rr < e) v0 += D.reg;
            if (rr == cc + 1 && rr < e) v1 += D.reg;
            *reinterpret_cast<double2*>(SQ + pf_rowoff(rr) + cc) = make_double2(v0, v1);
        }
    }
    __syncthreads();
    QPB_TICK(39);   // K = W W^T
    // ---- 4. equality block in product form (columns [0, ep)), then K -> global
    if (ep > 0) pf_chol_setup(PL.SQ, nts, 0, ep >> 3, PL.aug, PL.pan, PL.tab, nullptr, 0);
    __syncthreads();
    QPB_TICK(45);   // equality block
    for (int i = tid; i < pf_elems(nts); i += kNT) Kg[i] = SQ[i];
    QPB_TICK(46);   // write K
#ifdef QPB_TIMING
    if (tid == 0 && sys == 0) for (int i = 0; i < 128; ++i) g_tim[i] = s_tim[i];
#endif
}

}  // namespace
