// The shared-memory solve kernels (k_forward_fast, k_kkt_fast) and their layout / context helpers. Included by
// qp_kernels.cu (kNT = 256) and by qp_alt.cu (kNT = 192: three QPs per SM; kNT = 512: large problems).
#pragma once
#include "qp_common.cuh"
#include "qp_fast.cuh"
#include "qp_pf.cuh"

using namespace qpb;

namespace {

// =============================================================================================
// FAST PATH (shared-memory resident, padded to 8, compact code): k_forward_fast / k_kkt_fast
// =============================================================================================
namespace fk {
using namespace qpb::fast;
// (F_DINV, the reciprocal diagonal of the pre-factored equality block, is LAST: the product-form layouts do not have it)
enum FVec { F_PT = 0, F_XT, F_RXT, F_S, F_V, F_RV, F_HW, F_W, F_DSA, F_DS, F_D, F_BXT, F_BS, F_BV, F_HB,
            F_DINVL, F_AUG, F_T0, F_T1, F_DINV, F_COUNT };

constexpr int kFastRed = 4 * qpb::fast::kFastStride;   // reduction scratch of the fast kernels (block_reduce<4>, up to 16 warps)
struct FLayout {              // offsets in doubles into the dynamic shared array
    int W, LS, Lp, vec, red, bar, tab, pan;
    int vl;
};
__host__ __device__ inline int fast_vl(int n, int msp) { return ((n > msp ? n : msp) + 7) & ~7; }
// coop = W and packed L are NOT staged (they are read from global memory, qp_fast.cuh). Without pf the packed L
// visits the S workspace twice (whitening at entry, un-whitening at exit), so Lp aliases LS; with pf the two packed-L
// substitutions read L straight from global memory and nothing is staged.
// pf = product-form factor in the staircase layout (qp_pf.cuh): S shrinks to pf_elems, plus the panel scratch.
__host__ __device__ inline int s_doubles(const KDims& D, bool pf) {
    return pf ? qpb::pf::pf_elems(D.msp >> 3) : D.msp * D.lds;
}
__host__ __device__ inline FLayout fast_layout(const KDims& D, bool coop, bool pf = false) {
    FLayout L;
    L.vl = fast_vl(D.n, D.msp);
    L.W = 0;
    L.LS = coop ? 0 : L.W + D.ms * D.ldw;
    // panel scratch of pf_chol: rows 8 .. msp-1 and 8 private rows; its (never touched) first 8 rows overlap the end of S
    const int s_end = L.LS + s_doubles(D, pf);
    L.pan = s_end - 8 * qpb::pf::kPanLd;
    const int after_s = pf ? L.pan + (D.msp + 8) * qpb::pf::kPanLd : s_end;
    L.Lp = coop ? L.LS : after_s;
    L.vec = coop ? after_s : L.Lp + D.lp;
    L.red = L.vec + (pf ? F_COUNT - 1 : F_COUNT) * L.vl;
    L.bar = L.red + kFastRed;
    L.tab = L.bar + 2;                                       // tile table: round-1 Cholesky (kTabDoubles) / pf_build_tab
    return L;
}
__host__ __device__ inline size_t fast_smem_doubles(const KDims& D, bool coop, bool pf = false) {
    const FLayout L = fast_layout(D, coop, pf);
    return (size_t)L.tab + (pf ? qpb::pf::pf_tab_doubles(D.msp >> 3) : kTabDoubles);
}

struct FCtx {
    FLayout L;
    const double* Kg;
    const double* Wg;     // co-resident mode: W and packed L in global memory
    const double* Lg;
    uint32_t kphase;
    uint32_t lphase;      // parity of the next completion on bar[0] (W/L staging)
    uint32_t kbytes;      // size of the K template (square or staircase layout)
    bool kpending;
    bool lglobal;         // W/L-from-global product-form kernels: chol(Q) does not fit the (dead) S region it would visit,
                          // so the two packed-L substitutions read it from global memory
};
#define FV(i) (C.L.vec + (i) * C.L.vl)

__device__ __noinline__ void f_issue_K_impl(int LS, const double* Kg, int bar_off, uint32_t bytes) {
    QPB_SMEM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(qsm + bar_off);
    fence_proxy_async();
    mbar_expect_tx(bar + 1, bytes);
    bulk_issue_thread(qsm + LS, Kg, bytes, bar + 1);
}
// Call with all threads AFTER a block barrier that retired every reader of the previous factor.
__device__ __forceinline__ void f_issue_K(const KDims& D, FCtx& C) {
    if (threadIdx.x == 0) f_issue_K_impl(C.L.LS, C.Kg, C.L.bar, C.kbytes);
    C.kpending = true;
}
__device__ __forceinline__ void f_wait_K(FCtx& C) {
    QPB_SMEM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(qsm + C.L.bar);
    mbar_wait(bar + 1, C.kphase);
    C.kphase ^= 1u;
    C.kpending = false;
}

// Co-resident mode: bring the packed L into the (currently dead) S workspace. Call with all threads after a block
// barrier that retired every reader of the workspace and with no K copy in flight; returns when L has landed.
__device__ __forceinline__ void f_stage_L(const KDims& D, FCtx& C) {
    QPB_SMEM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(qsm + C.L.bar);
    if (threadIdx.x == 0) {
        fence_proxy_async();
        mbar_expect_tx(bar, (uint32_t)(D.lp * 8));
        bulk_issue_thread(qsm + C.L.Lp, C.Lg, (uint32_t)(D.lp * 8), bar);
    }
    mbar_wait(bar, C.lphase);
    C.lphase ^= 1u;
}

// Stage W and packed L with TMA, start the first K copy, build the tile table.
// kCoop: only L is staged (into the S workspace, for the whitening of the caller's first vector); the caller issues
// the first K copy itself once it is done with L (f_issue_K after a block barrier).
// kStageL (W/L-from-global product-form kernels): stage chol(Q) in the dead S region for the two packed-L substitutions
// instead of reading it from global memory inside them. Measured (r2o/r2z, B = 8192): the backward kernel, whose one
// iteration makes the substitutions a large share, gains 24 %; the forward kernel LOSES 2 % (the first K copy can no
// longer overlap the whitening) - so only the backward / solve_kkt kernel stages.
template <bool kCoop, bool kPF = false, bool kStageL = false>
__device__ __forceinline__ FCtx f_make_ctx(const KDims& D, int qp, const double* Lfac, const double* Wfac,
                                           const double* Kfac, int sF) {
    QPB_SMEM;
    FCtx C;
    C.L = fast_layout(D, kCoop, kPF);
    const int64_t sys = sF ? qp : 0;
    C.kbytes = (uint32_t)(s_doubles(D, kPF) * 8);
    C.Lg = Lfac + sys * (int64_t)D.lp;
    C.Wg = Wfac + sys * (int64_t)D.ms * D.ldw;
    C.Kg = Kfac + sys * (int64_t)s_doubles(D, kPF);
    C.kphase = 0;
    C.lphase = 0;
    C.kpending = false;
    const int tid = threadIdx.x;
    uint64_t* bar = reinterpret_cast<uint64_t*>(qsm + C.L.bar);
    if (tid == 0) {
        mbar_init(bar, 1);
        mbar_init(bar + 1, 1);
    }
    if (!kPF) build_tile_table(reinterpret_cast<uint16_t*>(qsm + C.L.tab), (D.msp - D.ep) >> 3, tid);
    else qpb::pf::pf_build_tab(C.L.tab, D.msp >> 3);
    __syncthreads();
    C.lglobal = kCoop && kPF && (!kStageL || D.lp > s_doubles(D, true));
    if (kCoop && kPF && C.lglobal) {
        f_issue_K(D, C);                                         // nothing is staged: L is read from global memory
        _Pragma("unroll 1") for (int i = tid; i < D.n; i += kNT) qsm[FV(F_DINVL) + i] = 1.0 / C.Lg[(i * (i + 1)) / 2 + i];
        return C;
    }
    if (kCoop) {
        f_stage_L(D, C);
    } else {
        if (tid == 0) {
            const uint32_t wb = (uint32_t)(D.ms * D.ldw * 8), lb = (uint32_t)(D.lp * 8);
            mbar_expect_tx(bar, wb + lb);
            bulk_issue_thread(qsm + C.L.W, C.Wg, wb, bar);
            bulk_issue_thread(qsm + C.L.Lp, C.Lg, lb, bar);
        }
        f_issue_K(D, C);
        mbar_wait(bar, 0);
    }
    // reciprocal diagonals of L (packed) and of the pre-factored equality block
    _Pragma("unroll 1") for (int i = tid; i < D.n; i += kNT) qsm[FV(F_DINVL) + i] = 1.0 / qsm[C.L.Lp + (i * (i + 1)) / 2 + i];
    return C;
}

// x~ = L^-1 x and x = L^-T x~ with the packed L in shared memory (staged into the dead S region in the W/L-from-global
// kernels: 13 block steps with a global load on each step's critical path were 6.7 % of the warp samples of the
// co-resident capture), or straight from global memory when it does not fit there
__device__ __forceinline__ void f_whiten_x(const KDims& D, const FCtx& C, int b, int u) {
    QPB_SMEM;
    if (C.lglobal) trsv_fwd(C.Lg, PackedIdx{}, D.n, 0, D.n, qsm + FV(F_DINVL), qsm + b, qsm + u, (int)threadIdx.x, kNT);
    else f_whiten(C.L.Lp, D.n, FV(F_DINVL), b, u);
}
__device__ __forceinline__ void f_unwhiten_x(const KDims& D, const FCtx& C, int u, int w) {
    QPB_SMEM;
    if (C.lglobal) trsv_bwd(C.Lg, PackedIdx{}, D.n, qsm + FV(F_DINVL), qsm + u, qsm + w, (int)threadIdx.x, kNT);
    else f_unwhiten(C.L.Lp, D.n, FV(F_DINVL), u, w);
}

// mat-vec dispatch: shared-memory resident W / L, or the global-memory passes of the co-resident mode
template <bool kCoop>
__device__ __forceinline__ void mv_rows1(const KDims& D, const FCtx& C, int x1, int y1) {
    if (kCoop) g_matvec_rows1(C.Wg, D.ldw, D.ms, D.n, x1, y1);
    else f_matvec_rows1(C.L.W, D.ldw, D.ms, D.n, x1, y1);
}
template <bool kCoop>
__device__ __forceinline__ void mv_rows2(const KDims& D, const FCtx& C, int x1, int x2, int y1, int y2) {
    if (kCoop) g_matvec_rows2(C.Wg, D.ldw, D.ms, D.n, x1, x2, y1, y2);
    else f_matvec_rows2(C.L.W, D.ldw, D.ms, D.n, x1, x2, y1, y2);
}
// One pass over W for the end of a Newton iteration (v, s already updated; ends with a block barrier):
//   dx~ = -r~x - W^T dv,   x~ += alpha dx~,   r~x = x~ + W^T v + p~   (the next iteration's residual).
// p0 .. p3: partial-sum scratch of the shared-memory pass.
template <bool kCoop>
__device__ __forceinline__ void mv_cols2(const KDims& D, const FCtx& C, int dv, int v, int p0, int p1, int p2, int p3,
                                         int xt, int rxt, int pt, double alpha) {
    if (kCoop) g_matvec_cols2(C.Wg, D.ldw, D.ms, D.n, dv, v, xt, rxt, pt, alpha);
    else f_matvec_cols2(C.L.W, D.ldw, D.ms, D.n, dv, v, p0, p1, p2, p3, xt, rxt, pt, alpha);
}
template <bool kCoop>
__device__ __forceinline__ void mv_cols(const KDims& D, const FCtx& C, int v, int p0, int p1, int out, int a, double sa,
                                        int b, double sgn) {
    if (kCoop) g_matvec_cols(C.Wg, D.ldw, D.ms, D.n, v, out, a, sa, b, sgn);
    else f_matvec_cols(C.L.W, D.ldw, D.ms, D.n, v, p0, p1, out, a, sa, b, sgn);
}

// factor_kkt + first half of solve_kkt: F_AUG = -h_full (pad entries 0), F_D = d  ->  F_W = -S^-1 h_full
__device__ __forceinline__ void f_factor_and_solve(const KDims& D, FCtx& C) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    f_wait_K(C);
    _Pragma("unroll 1") for (int i = D.ep + tid; i < D.ms; i += kNT) qsm[C.L.LS + i * D.lds + i] += 1.0 / qsm[FV(F_D) + i];
    __syncthreads();
    if (D.ep > 0) {
        f_trsv_fwd(C.L.LS, D.lds, D.msp, 0, D.ep, FV(F_AUG), FV(F_T0));
        _Pragma("unroll 1") for (int i = tid; i < D.ep; i += kNT) qsm[FV(F_AUG) + i] = qsm[FV(F_T0) + i];
        __syncthreads();
    }
    f_chol(C.L.LS, D.lds, D.msp, D.ep, FV(F_AUG), C.L.tab);
    QPB_TICK(32);   // (chol internals are 20..27)
    f_trsv_bwd(C.L.LS, D.lds, D.msp, FV(F_AUG), FV(F_W));
    QPB_TICK(33);   // backward substitution
}

// The same with the product-form factor (qp_pf.cuh): F_AUG = -h_full, F_D = d  ->  F_W = -S^-1 h_full; F_T0 scratch.
// kReg: F_D holds d + eps and the inequality diagonal gets 1 / (d + eps) + eps (the regularised system; the eps of the
// equality rows is already in K, pre_factor_kkt_reg).
template <bool kReg = false>
__device__ __forceinline__ void f_factor_and_solve_pf(const KDims& D, FCtx& C) {
    QPB_SMEM;
    using namespace qpb::pf;
    const int tid = threadIdx.x;
    f_wait_K(C);
    _Pragma("unroll 1") for (int i = D.ep + tid; i < D.ms; i += kNT)
        qsm[C.L.LS + pf_rowoff(i) + i] += kReg ? 1.0 / qsm[FV(F_D) + i] + D.reg : 1.0 / qsm[FV(F_D) + i];
    __syncthreads();
    if (D.ep > 0) pf_fwd(C.L.LS, D.msp, 0, D.ep >> 3, FV(F_AUG));
    pf_chol(C.L.LS, D.msp >> 3, D.ep >> 3, FV(F_AUG), C.L.pan, C.L.tab);
    QPB_TICK(32);
    pf_diag(C.L.LS, D.msp, FV(F_AUG), FV(F_T0), FV(F_AUG));
    pf_bwd(C.L.LS, D.msp, FV(F_AUG), FV(F_W));
    QPB_TICK(33);
}

__device__ __forceinline__ double f_step_fix(double v) { return (isinf(v) && v > 0.0) ? 1.0 : v; }

// ---- regularised mode (kReg: QPFunction with kkt_solver=IR_UNOPT) ---------------------------------------------------
// The factors are those of pre_factor_kkt_reg: L = chol(Q + eps I), K with eps on the equality rows. Every KKT solve
// uses the regularised system [Q+eI 0 G' A'; 0 D+eI I 0; G I -eI 0; A 0 0 -eI], while the residuals are those of the
// true problem, so the Newton loop converges to the exact KKT point of a Q that is only positive semidefinite.

// r~x -= eps L^-1 L^-T x~: the whitened dual residual of the true problem (L^-1 (Qx + p + G'z + A'y)) from the one of
// Q + eps I that the W pass produces. t0, t1: scratch. Ends with a block barrier.
__device__ __forceinline__ void f_true_rx(const KDims& D, const FCtx& C, int xt, int rxt, int t0, int t1) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    _Pragma("unroll 1") for (int i = tid; i < D.n; i += kNT) qsm[t1 + i] = qsm[xt + i];
    __syncthreads();
    f_unwhiten_x(D, C, t1, t0);                              // t0 = x = L^-T x~
    f_whiten_x(D, C, t0, t1);                                // t1 = L^-1 x
    _Pragma("unroll 1") for (int i = tid; i < D.n; i += kNT) qsm[rxt + i] = fma(-D.reg, qsm[t1 + i], qsm[rxt + i]);
    __syncthreads();
}

// One refinement step, with the factor still in the S workspace, of a solution of the regularised system: dv = [dy; dz],
// ds, and dx~ = -base + ntx - W^T dv kept implicit. With K = K~ - Delta, the true residual of d = d0 + c1 + .. + ck is
// -Delta ck = (-eps dx, -eps ds, eps dz, eps dy) of the LAST correction ck (of the solution d0 itself in the first step);
// the next correction solves the regularised system with it and is added in place (ntx += eps L^-1 dx).
// Between the steps of one solve c, e, f carry that correction: c = -eps L^-1 dx, e = eps ds, f = [dy; dz]; the first
// step (first = true) reads the solution instead. F_D holds d + eps. a, b: scratch slots. Ends with a block barrier.
template <bool kCoop>
__device__ __forceinline__ void f_refine(const KDims& D, const FCtx& C, int base, int ntx, int dv, int ds, int a, int b,
                                         int c, int e, int f, bool first) {
    QPB_SMEM;
    const int tid = threadIdx.x, dd = FV(F_D);
    if (first) mv_cols<kCoop>(D, C, dv, e, f, a, base, -1.0, ntx, -1.0);   // a = dx~ of the solution
    else mv_cols<kCoop>(D, C, f, a, b, a, c, -1.0, -1, -1.0);             // a = dx~ of the correction: eps L^-1 dx - W^T f
    f_unwhiten_x(D, C, a, b);                                // b = dx
    f_whiten_x(D, C, b, c);                                  // c = L^-1 dx
    _Pragma("unroll 1") for (int i = tid; i < D.n; i += kNT) {
        const double r = D.reg * qsm[c + i];
        qsm[c + i] = -r;                                     // whitened x residual  L^-1 (-eps dx)
        qsm[ntx + i] += r;
    }
    __syncthreads();
    const int wt = first ? e : b;                            // W t (e holds eps ds of the correction after the first)
    mv_rows1<kCoop>(D, C, c, wt);
    __syncthreads();
    // reduced right-hand side -(W t - [r_y; r_z] + [0; r_s / (d + eps)])  (the elimination of solve_kkt)
    if (first) {
        _Pragma("unroll 1") for (int i = tid; i < D.msp; i += kNT) {
            double hf = 0.0;
            if (i < D.ms) {
                hf = fma(-D.reg, qsm[dv + i], qsm[e + i]);
                if (i >= D.ep) hf -= D.reg * qsm[ds + i] / qsm[dd + i];
            }
            qsm[a + i] = -hf;
        }
    } else {
        _Pragma("unroll 1") for (int i = tid; i < D.msp; i += kNT) {
            double hf = 0.0;
            if (i < D.ms) {
                hf = fma(-D.reg, qsm[f + i], qsm[b + i]);
                if (i >= D.ep) hf -= qsm[e + i] / qsm[dd + i];
            }
            qsm[a + i] = -hf;
        }
    }
    __syncthreads();
    qpb::pf::pf_solve(C.L.LS, D.msp, a, b, f);              // f = correction of [dy; dz]
    if (first) {
        _Pragma("unroll 1") for (int i = tid; i < D.ms; i += kNT) {
            const double wi = qsm[f + i];
            if (i >= D.ep) {
                const double dsc = (D.reg * qsm[ds + i] - wi) / qsm[dd + i];
                qsm[ds + i] += dsc;
                qsm[e + i] = D.reg * dsc;
            }
            qsm[dv + i] += wi;
        }
    } else {
        _Pragma("unroll 1") for (int i = tid; i < D.ms; i += kNT) {
            const double wi = qsm[f + i];
            if (i >= D.ep) {
                const double dsc = (qsm[e + i] - wi) / qsm[dd + i];
                qsm[ds + i] += dsc;
                qsm[e + i] = D.reg * dsc;
            }
            qsm[dv + i] += wi;
        }
    }
    __syncthreads();
}

}  // namespace fk

// kCoop: co-resident mode (two CTAs per SM; W and L read from global memory, see qp_fast.cuh).
// kPF: product-form factor in the staircase layout (qp_pf.cuh); with kCoop it is the "large problem" kernel: factor
// and vectors in shared memory, W and L read from global memory (L2-resident when the system is shared), ONE CTA per SM.
// kMinCtas (with kCoop && kPF): the same kernel compiled for 2 (256 threads, 128 registers) or 3 (192 threads, 112
// registers: qp_alt.cu) CTAs per SM: <= 76.8 KB of shared memory per QP at C2, so the QPs of an SM fill each other's
// pivot-chain bubbles.
// kReg (with kPF, kMinCtas = 0): the regularised mode (fk::f_true_rx, fk::f_refine); D.reg = eps, ir_steps refinement
// steps of the initial point and of each iteration's combined direction (a trailing parameter: KDims keeps its layout).
template <bool kCoop, bool kPF = false, int kMinCtas = 0, bool kReg = false>
__global__ void __launch_bounds__(qpb::fast::kNT, kMinCtas ? kMinCtas : ((kCoop && !kPF) ? 2 : 1))
k_forward_fast(KDims D, const double* __restrict__ p, int64_t sp, const double* __restrict__ h, int64_t sh,
               const double* __restrict__ b, int64_t sb, const double* __restrict__ Lfac,
               const double* __restrict__ Wfac, const double* __restrict__ Kfac, int sF, double eps,
               double stall_tol, double best_tie, int notImprovedLim, int maxIter,
               double* __restrict__ zhat, double* __restrict__ lam, double* __restrict__ slacks,
               double* __restrict__ nus, int* __restrict__ iters_out, double* __restrict__ resid_out,
               double* __restrict__ trace, int ir_steps = 0) {
    using namespace fk;
    QPB_SMEM;
    const int tid = threadIdx.x;
    const int qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, ms = D.ms, msp = D.msp;
#ifdef QPB_TIMING
    if (threadIdx.x == 0) {
        for (int i = 0; i < 128; ++i) s_tim[i] = 0;
        s_tim[128] = clock64(); s_tim2 = s_tim[128];
        if (qp < 8192) { g_cta[4 * qp] = gtimer(); g_cta[4 * qp + 3] = smid(); }
    }
    __syncthreads();
#endif
    FCtx C = f_make_ctx<kCoop, kPF>(D, qp, Lfac, Wfac, Kfac, sF);
    QPB_TICK(0);
    const int pt = FV(F_PT), xt = FV(F_XT), rxt = FV(F_RXT), s = FV(F_S), v = FV(F_V), rv = FV(F_RV),
              hW = FV(F_HW), w = FV(F_W), dsa = FV(F_DSA), ds = FV(F_DS), d = FV(F_D), hb = FV(F_HB),
              aug = FV(F_AUG), t0 = FV(F_T0), t1 = FV(F_T1);

    const double* pg = p + (int64_t)qp * sp;
    const double* hg = h + (int64_t)qp * sh;
    const double* bg = (e > 0) ? (b + (int64_t)qp * sb) : nullptr;
    _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[t1 + i] = pg[i];
    _Pragma("unroll 1") for (int i = tid; i < msp; i += kNT) {
        double val = 0.0;
        if (i < e) val = bg[i];
        else if (i >= ep && i < ms) val = hg[i - ep];
        qsm[hb + i] = val;
        qsm[d + i] = kReg ? 1.0 + D.reg : 1.0;
        qsm[s + i] = 0.0;
        qsm[v + i] = 0.0;
        qsm[aug + i] = 0.0;
        qsm[w + i] = 0.0;
    }
    __syncthreads();
    QPB_TICK(1);
    f_whiten_x(D, C, t1, pt);                              // p~ = L^-1 p
    if (kCoop && !C.lglobal) {                                  // L leaves the S workspace: the first K copy may land
        __syncthreads();
        f_issue_K(D, C);
    }
    QPB_TICK(2);

    // ---- initial point: solve_kkt(p, 0, -h, -b) with d = 1   (batch.py:61-67)
    mv_rows1<kCoop>(D, C, pt, hW);
    __syncthreads();
    _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) qsm[aug + i] = -(qsm[hW + i] + qsm[hb + i]);
    __syncthreads();
    if (kPF) f_factor_and_solve_pf<kReg>(D, C); else f_factor_and_solve(D, C);
    const bool refine = kReg && ir_steps > 0;
    if (kReg) {
        // s = -w / (1 + eps); rv accumulates the x part of the refinement (x~ = -p~ + rv - W^T w)
        _Pragma("unroll 1") for (int i = ep + tid; i < ms; i += kNT) qsm[s + i] = -qsm[w + i] / qsm[d + i];
        _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[rv + i] = 0.0;
        __syncthreads();
        _Pragma("unroll 1") for (int k = 0; k < ir_steps; ++k) f_refine<kCoop>(D, C, pt, rv, w, s, t1, t0, aug, hW, dsa, k == 0);
    }
    f_issue_K(D, C);
    mv_cols<kCoop>(D, C, w, t0, t1, xt, pt, -1.0, refine ? rv : -1, -1.0);   // x~ = -p~ - W^T w
    {
        double mn[2] = {INFINITY, INFINITY};
        _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) {
            const double wi = qsm[w + i];
            qsm[v + i] = wi;
            if (i >= ep) {
                const double si = kReg ? qsm[s + i] : -wi;
                qsm[s + i] = si;
                mn[0] = fmin(mn[0], si);
                mn[1] = fmin(mn[1], wi);
            }
        }
        f_reduce_min2(mn, C.L.red);
        _Pragma("unroll 1") for (int i = ep + tid; i < ms; i += kNT) {               // slacks and duals >= 1 (batch.py:77-87)
            if (mn[0] < 0.0) qsm[s + i] -= mn[0] - 1.0;
            if (mn[1] < 0.0) qsm[v + i] -= mn[1] - 1.0;
        }
        __syncthreads();
    }

    double best = 0.0;
    int nNot = 0, iters_run = 0;
    const double dm = (double)m;
    for (int it = 0; it < maxIter; ++it) {
        iters_run = it + 1;
        // ---- residuals (batch.py:94-107)
        QPB_TICK(3);
        // r~x = x~ + p~ + W^T [y;z]: here at the initial point; later iterations get it from the previous one's mv_cols2
        if (it == 0) mv_cols<kCoop>(D, C, v, t0, t1, rxt, xt, 1.0, pt, 1.0);
        if (kReg) f_true_rx(D, C, xt, rxt, t0, t1);
        QPB_TICK(4);
        double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // |ry|^2, |rz|^2, |L r~x|^2, s.z
        mv_rows2<kCoop>(D, C, xt, rxt, rv, hW);                      // W x~ , W r~x
        // chol(Q) pass in the same phase as the W row pass (it needs r~x only): their load latencies overlap
        acc[2] = kCoop ? g_tri_norm2(C.Lg, n, rxt) : f_tri_norm2(C.L.Lp, n, rxt);
        __syncthreads();
        QPB_TICK(5);
        _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) {
            const double r = qsm[rv + i] - qsm[hb + i] + ((i >= ep) ? qsm[s + i] : 0.0);
            qsm[rv + i] = r;
            if (i < ep) acc[0] = fma(r, r, acc[0]);
            else { acc[1] = fma(r, r, acc[1]); acc[3] = fma(qsm[s + i], qsm[v + i], acc[3]); }
        }
        QPB_TICK(6);
        f_reduce_sum4(acc, C.L.red);
        QPB_TICK(8);
        const double mu = fabs(acc[3] / dm);
        const double resid = sqrt(acc[1]) + sqrt(acc[0]) + sqrt(acc[2]) + dm * mu;
        if (trace != nullptr && tid == 0) {                     // what verbose=1 prints (batch.py:115-117)
            double* tr = trace + ((int64_t)qp * maxIter + it) * 4;
            tr[0] = sqrt(acc[1]) + sqrt(acc[0]); tr[1] = sqrt(acc[2]); tr[2] = mu; tr[3] = resid;
        }
        // ---- best-iterate tracking and exit tests (batch.py:118-143), per QP (see k_forward)
        const bool improved = (it == 0) || (resid < best);
        if (improved) { best = resid; nNot = 0; } else { ++nNot; }
        if (improved || resid < best_tie * best) {
            _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[FV(F_BXT) + i] = qsm[xt + i];
            _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) { qsm[FV(F_BS) + i] = qsm[s + i]; qsm[FV(F_BV) + i] = qsm[v + i]; }
        }
        if ((nNot == notImprovedLim && best < stall_tol) || best < eps || mu > 1e32) break;
        if (!(resid == resid) || isinf(resid)) break;
        // ---- factor_kkt with d = z/s and the affine right-hand side (batch.py:109-113,150)
        _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) {
            double hfull = qsm[hW + i] - qsm[rv + i];
            if (i >= ep) {
                const double di = kReg ? qsm[v + i] / qsm[s + i] + D.reg : qsm[v + i] / qsm[s + i];
                qsm[d + i] = di;
                hfull += qsm[v + i] / di;
            }
            qsm[aug + i] = -hfull;
        }
        __syncthreads();
        QPB_TICK(9);
        if (kPF) f_factor_and_solve_pf<kReg>(D, C); else f_factor_and_solve(D, C);   // w = [dy_aff; dz_aff]
        QPB_TICK(10);
        // ---- affine step length and sigma (batch.py:160-168)
        double mn[2] = {INFINITY, INFINITY};
        _Pragma("unroll 1") for (int i = ep + tid; i < ms; i += kNT) {
            const double dz = qsm[w + i];
            const double dsi = (-qsm[v + i] - dz) / qsm[d + i];
            qsm[dsa + i] = dsi;
            mn[0] = fmin(mn[0], step_candidate(qsm[v + i], dz));
            mn[1] = fmin(mn[1], step_candidate(qsm[s + i], dsi));
        }
        f_reduce_min2(mn, C.L.red);
        {
            const double alpha = fmin(fmin(f_step_fix(mn[0]), f_step_fix(mn[1])), 1.0);
            double sm[2] = {0.0, 0.0};
            _Pragma("unroll 1") for (int i = ep + tid; i < ms; i += kNT) {
                sm[0] = fma(qsm[s + i] + alpha * qsm[dsa + i], qsm[v + i] + alpha * qsm[w + i], sm[0]);
                sm[1] = fma(qsm[s + i], qsm[v + i], sm[1]);
            }
            f_reduce_sum2(sm, C.L.red);
            const double sr = sm[0] / sm[1];
            const double sig = sr * sr * sr;
            // ---- corrector right-hand side (batch.py:170-181)
            _Pragma("unroll 1") for (int i = tid; i < msp; i += kNT) {
                double rhs = 0.0;
                if (i >= ep && i < ms) {
                    const double rsc = (-mu * sig + qsm[dsa + i] * qsm[w + i]) / qsm[s + i];
                    qsm[ds + i] = rsc;
                    rhs = -(rsc / qsm[d + i]);
                }
                qsm[t1 + i] = rhs;
            }
            __syncthreads();
        }
        QPB_TICK(11);
        int wc = t1;                                             // where [dy_cor; dz_cor] lands
        if (kPF) {
            qpb::pf::pf_solve(C.L.LS, msp, t1, t0, hW);         // (hW is dead until the combined direction below)
            wc = hW;
            QPB_TICK(12);
        } else {
            f_trsv_fwd(C.L.LS, D.lds, msp, 0, msp, t1, t0);
            QPB_TICK(12);
            f_trsv_bwd(C.L.LS, D.lds, msp, t0, t1);              // t1 = [dy_cor; dz_cor]
        }
        QPB_TICK(13);
        if (!refine) f_issue_K(D, C);                            // next factor_kkt's K copy overlaps the rest
        // ---- combined direction, step length, update (batch.py:185-203)
        mn[0] = INFINITY; mn[1] = INFINITY;
        _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) {
            const double wci = qsm[wc + i];
            const double dv = qsm[w + i] + wci;
            qsm[w + i] = dv;
            if (i >= ep) {
                const double dsc = (-qsm[ds + i] - wci) / qsm[d + i];
                const double dsi = qsm[dsa + i] + dsc;
                qsm[ds + i] = dsi;
                mn[0] = fmin(mn[0], step_candidate(qsm[v + i], dv));
                mn[1] = fmin(mn[1], step_candidate(qsm[s + i], dsi));
            }
        }
        if (refine) {
            // The refinement is linear in the right-hand side, so refining the combined direction equals refining the
            // affine and the corrector direction one by one; sigma above comes from the unrefined affine direction.
            _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[rv + i] = 0.0;
            __syncthreads();
            _Pragma("unroll 1") for (int k = 0; k < ir_steps; ++k) f_refine<kCoop>(D, C, rxt, rv, w, ds, t1, t0, aug, hW, dsa, k == 0);
            f_issue_K(D, C);
            mn[0] = INFINITY; mn[1] = INFINITY;
            _Pragma("unroll 1") for (int i = ep + tid; i < ms; i += kNT) {
                mn[0] = fmin(mn[0], step_candidate(qsm[v + i], qsm[w + i]));
                mn[1] = fmin(mn[1], step_candidate(qsm[s + i], qsm[ds + i]));
            }
            _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[rxt + i] -= qsm[rv + i];   // dx~ = -(r~x - rv) - W^T dv
        }
        QPB_TICK(14);
        // the step length does not depend on dx~: v and s move first, then one pass over W gives dx~, x~ and the next
        // iteration's r~x (none after the last iteration: nothing reads x~ then)
        f_reduce_min2(mn, C.L.red);
        const double alpha = fmin(0.999 * fmin(f_step_fix(mn[0]), f_step_fix(mn[1])), 1.0);
        _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) {
            qsm[v + i] = fma(alpha, qsm[w + i], qsm[v + i]);
            if (i >= ep) qsm[s + i] = fma(alpha, qsm[ds + i], qsm[s + i]);
        }
        __syncthreads();
        if (it + 1 < maxIter) mv_cols2<kCoop>(D, C, w, v, t0, t1, hW, dsa, xt, rxt, pt, alpha);   // (t0, t1, hW, dsa dead)
        QPB_TICK(15);
    }

    // ---- outputs: x = L^-T x~_best, y, z, s of the returned iterate (batch.py:205-207)
    __syncthreads();
    QPB_TICK(16);
    if (kCoop && !C.lglobal) {                                   // the S workspace is dead: L comes back for x = L^-T x~
        if (C.kpending) f_wait_K(C);
        __syncthreads();
        f_stage_L(D, C);
    }
    f_unwhiten_x(D, C, FV(F_BXT), t0);
    if (C.kpending) f_wait_K(C);                                 // drain the in-flight copy before exit
    _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) zhat[(int64_t)qp * n + i] = qsm[t0 + i];
    _Pragma("unroll 1") for (int i = tid; i < m; i += kNT) {
        lam[(int64_t)qp * m + i] = qsm[FV(F_BV) + ep + i];
        slacks[(int64_t)qp * m + i] = qsm[FV(F_BS) + ep + i];
    }
    if (e > 0 && nus != nullptr)
        _Pragma("unroll 1") for (int i = tid; i < e; i += kNT) nus[(int64_t)qp * e + i] = qsm[FV(F_BV) + i];
    if (tid == 0) {
        iters_out[qp] = iters_run;
        resid_out[qp] = best;          // the minimum over the iterations, as the reference reports (batch.py:126-142)
    }
#ifdef QPB_TIMING
    QPB_TICK(16);
    if (tid == 0 && qp == g_tim_target) for (int i = 0; i < 128; ++i) g_tim[i] = s_tim[i];
    if (tid == 0 && qp < 8192) { g_cta[4 * qp + 1] = gtimer(); g_cta[4 * qp + 2] = iters_run; }
#endif
}

// kReg (with kBackward, kPF, kMinCtas = 0): the backward pass of the regularised mode, d + eps and ir_steps refinement
// steps (fk::f_refine). chol(Q) is then read from global memory in the W/L-from-global build: the refinement needs it
// while the factor occupies the S workspace.
template <bool kBackward, bool kCoop, bool kPF = false, int kMinCtas = 0, bool kReg = false>
__global__ void __launch_bounds__(qpb::fast::kNT, kMinCtas ? kMinCtas : ((kCoop && !kPF) ? 2 : 1))
k_kkt_fast(KDims D, const double* __restrict__ d_in, const double* __restrict__ rx_in,
           const double* __restrict__ rs_in, const double* __restrict__ rz_in,
           const double* __restrict__ ry_in, const double* __restrict__ zhat,
           const double* __restrict__ lam, const double* __restrict__ slacks,
           const double* __restrict__ nus, const double* __restrict__ Lfac,
           const double* __restrict__ Wfac, const double* __restrict__ Kfac, int sF,
           double* __restrict__ dx_out, double* __restrict__ ds_out, double* __restrict__ dz_out,
           double* __restrict__ dy_out, BwdOut O, int ir_steps = 0) {
    using namespace fk;
    QPB_SMEM;
    const int tid = threadIdx.x;
    const int qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, ms = D.ms, msp = D.msp;
    FCtx C = f_make_ctx<kCoop, kPF, !kReg>(D, qp, Lfac, Wfac, Kfac, sF);
    const int t = FV(F_PT), d = FV(F_D), hW = FV(F_HW), aug = FV(F_AUG), w = FV(F_W), t0 = FV(F_T0),
              t1 = FV(F_T1), rsv = FV(F_S), c2 = FV(F_RV), dxt = FV(F_RXT), dxo = FV(F_XT);
    _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[t1 + i] = rx_in[(int64_t)qp * n + i];
    _Pragma("unroll 1") for (int i = tid; i < msp; i += kNT) {
        double di = 1.0, extra = 0.0, rsi = 0.0;
        if (i >= ep && i < ms) {
            const int j = i - ep;
            if (kBackward) {
                di = fmax(lam[(int64_t)qp * m + j], 1e-8) / fmax(slacks[(int64_t)qp * m + j], 1e-8);   // qp.py:148
                if (kReg) di += D.reg;
            } else {
                // regularised variant (D.reg > 0, batch.py:244-310): d~ = d + eps in the complementarity row, and the slot
                // holds 1 / (1/d~ + eps) because factor_kkt adds the RECIPROCAL of this slot to the diagonal of S
                const double dt = d_in[(int64_t)qp * m + j] + D.reg;
                di = (D.reg > 0.0) ? 1.0 / (1.0 / dt + D.reg) : dt;
                rsi = rs_in[(int64_t)qp * m + j];
                extra = rsi / dt - rz_in[(int64_t)qp * m + j];
            }
        } else if (!kBackward && i < e) {
            extra = -ry_in[(int64_t)qp * e + i];
        }
        qsm[d + i] = di;
        qsm[rsv + i] = rsi;
        qsm[hW + i] = extra;
        qsm[aug + i] = 0.0;
    }
    // backward: the adjoints of the duals (either may be NULL) are rz = dl/dlam and ry = dl/dnu, with rs = 0. A loop of
    // its own, over each thread's own rows: inside the one above the load cost the 256-thread coop build spills.
    if (kBackward && (rz_in != nullptr || ry_in != nullptr)) {
        _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) {
            if (i >= ep) {
                if (rz_in != nullptr) qsm[hW + i] = -rz_in[(int64_t)qp * m + i - ep];
            } else if (i < e && ry_in != nullptr) {
                qsm[hW + i] = -ry_in[(int64_t)qp * e + i];
            }
        }
    }
    if (kReg) {                                                  // x part of the refinement (dx~ = -t + it - W^T w)
        _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[FV(F_DSA) + i] = 0.0;
    }
    __syncthreads();
    f_whiten_x(D, C, t1, t);                               // t = L^-1 rx
    if (kCoop && !C.lglobal) {
        __syncthreads();
        f_issue_K(D, C);
    }
    mv_rows1<kCoop>(D, C, t, c2);
    __syncthreads();
    _Pragma("unroll 1") for (int i = tid; i < ms; i += kNT) qsm[aug + i] = -(qsm[c2 + i] + qsm[hW + i]);
    __syncthreads();
    if (kPF) f_factor_and_solve_pf<kReg>(D, C); else f_factor_and_solve(D, C);   // w = [dy; dz]
    const int ntx = FV(F_DSA), dsr = FV(F_DS);
    if (kReg) {
        _Pragma("unroll 1") for (int i = ep + tid; i < ms; i += kNT) qsm[dsr + i] = -qsm[w + i] / qsm[d + i];   // ds (rs = 0)
        __syncthreads();
        _Pragma("unroll 1") for (int k = 0; k < ir_steps; ++k) f_refine<kCoop>(D, C, t, ntx, w, dsr, aug, t0, t1, hW, c2, k == 0);
    }
    mv_cols<kCoop>(D, C, w, t0, t1, dxt, t, -1.0, kReg ? ntx : -1, -1.0);
    if (kCoop && !C.lglobal) f_stage_L(D, C);                   // (mv_cols ended with a block barrier; no K copy in flight)
    f_unwhiten_x(D, C, dxt, dxo);                          // dx = L^-T dx~
    _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) dx_out[(int64_t)qp * n + i] = qsm[dxo + i];
    _Pragma("unroll 1") for (int i = tid; i < m; i += kNT) {
        dz_out[(int64_t)qp * m + i] = qsm[w + ep + i];
        if (!kBackward) ds_out[(int64_t)qp * m + i] = (-qsm[rsv + ep + i] - qsm[w + ep + i]) / (d_in[(int64_t)qp * m + i] + D.reg);
    }
    if (e > 0 && dy_out != nullptr)
        _Pragma("unroll 1") for (int i = tid; i < e; i += kNT) dy_out[(int64_t)qp * e + i] = qsm[w + i];
    if (!kBackward) return;

    // ---- gradients for batched inputs (qp.py:157-176); 128-bit coalesced stores
    const int zs = FV(F_BXT), ls = FV(F_BV);
    _Pragma("unroll 1") for (int i = tid; i < n; i += kNT) qsm[zs + i] = zhat[(int64_t)qp * n + i];
    _Pragma("unroll 1") for (int i = tid; i < m; i += kNT) qsm[ls + ep + i] = lam[(int64_t)qp * m + i];
    _Pragma("unroll 1") for (int i = tid; i < e; i += kNT) qsm[ls + i] = nus[(int64_t)qp * e + i];
    __syncthreads();
    if (O.dp && !O.mp) for (int i = tid; i < n; i += kNT) O.dp[(int64_t)qp * n + i] = qsm[dxo + i];
    if (O.dh && !O.mh) for (int i = tid; i < m; i += kNT) O.dh[(int64_t)qp * m + i] = -qsm[w + ep + i];
    if (O.db && !O.mb && e > 0) for (int i = tid; i < e; i += kNT) O.db[(int64_t)qp * e + i] = -qsm[w + i];
    const bool even = (n & 1) == 0;
    if (O.dQ && !O.mQ) {
        double* o = O.dQ + (int64_t)qp * n * n;
        if (even) {
            const int n2 = n >> 1;
            _Pragma("unroll 1") for (int i = tid; i < n * n2; i += kNT) {
                const int r = i / n2, c = (i - r * n2) * 2;
                const double dr = qsm[dxo + r], zr = qsm[zs + r];
                reinterpret_cast<double2*>(o)[i] = make_double2(0.5 * (dr * qsm[zs + c] + zr * qsm[dxo + c]),
                                                                0.5 * (dr * qsm[zs + c + 1] + zr * qsm[dxo + c + 1]));
            }
        } else {
            _Pragma("unroll 1") for (int i = tid; i < n * n; i += kNT) {
                const int r = i / n, c = i - r * n;
                o[i] = 0.5 * (qsm[dxo + r] * qsm[zs + c] + qsm[zs + r] * qsm[dxo + c]);
            }
        }
    }
    if (O.dG && !O.mG) {
        double* o = O.dG + (int64_t)qp * m * n;
        if (even) {
            const int n2 = n >> 1;
            _Pragma("unroll 1") for (int i = tid; i < m * n2; i += kNT) {
                const int r = i / n2, c = (i - r * n2) * 2;
                const double wr = qsm[w + ep + r], lr = qsm[ls + ep + r];
                reinterpret_cast<double2*>(o)[i] = make_double2(wr * qsm[zs + c] + lr * qsm[dxo + c],
                                                                wr * qsm[zs + c + 1] + lr * qsm[dxo + c + 1]);
            }
        } else {
            _Pragma("unroll 1") for (int i = tid; i < m * n; i += kNT) {
                const int r = i / n, c = i - r * n;
                o[i] = qsm[w + ep + r] * qsm[zs + c] + qsm[ls + ep + r] * qsm[dxo + c];
            }
        }
    }
    if (O.dA && !O.mA && e > 0) {
        double* o = O.dA + (int64_t)qp * e * n;
        _Pragma("unroll 1") for (int i = tid; i < e * n; i += kNT) {
            const int r = i / n, c = i - r * n;
            o[i] = qsm[w + r] * qsm[zs + c] + qsm[ls + r] * qsm[dxo + c];
        }
    }
}



}  // namespace
