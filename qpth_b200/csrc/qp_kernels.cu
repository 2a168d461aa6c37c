// qpth_b200 — sm_90a kernels + C ABI for the batched differentiable QP hot path.
//
// Mapping to the reference (locuslab/qpth @ 528e9f6, citations relative to /root/reference):
//   k_setup*    <- pre_factor_kkt            qpth/solvers/pdipm/batch.py:375-429  (+ SPD check qp.py:81-85)
//   k_forward*  <- forward (PDIPM loop)      qpth/solvers/pdipm/batch.py:47-207   (+ get_step :210-213)
//   k_kkt_fast<true> / k_solve_kkt<..,true>  <- QPFunctionFn.backward     qpth/qp.py:128-182
//   k_kkt_fast<false> / k_solve_kkt          <- factor_kkt + solve_kkt    qpth/solvers/pdipm/batch.py:435-470, 349-372
// Kernel families (chosen by qpb200_plan_init, see include/qpth_b200.h): product form (qp_solve.cuh + qp_pf.cuh; the
// default wherever the reduced system has order <= 256), round-1 shared-memory kernels (QPB200_PF=0), generic kernels
// below (one warp per QP for tiny shapes; global scratch for shapes nothing else fits).
//
// Formulation (DESIGN.md): with Q = L L^T the variables are whitened, x~ = L^T x, so
//   W = [A; G] L^-T            (rows 0..ep-1: equality rows, zero-padded to a multiple of 8; then G rows)
//   S = W W^T + diag(0, 1/d)   (the reduced KKT matrix of solve_kkt; R = G Q^-1 G^T is its lower-right block)
//   K = block-Cholesky template of S: columns [0,ep) factored once (L11, L21), the trailing block holds
//       R - L21 L21^T; each factor_kkt call copies K, adds 1/d on the diagonal and finishes the Cholesky.
// One CTA solves one QP; the whole Newton loop runs inside k_forward with no host round trips.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "../../include/qpth_b200.h"
#include "qp_device.cuh"
#include "qp_fast.cuh"
#include "qp_pf.cuh"

using namespace qpb;

namespace {

constexpr int kThreads = 256;
constexpr int kTinyThreads = 32;        // tiny problems: one warp per QP (generic shared-memory kernels, 32-thread CTAs)
constexpr int kTinyCtasPerSm = 16;
constexpr int kTinyMax = 32;            // nz and ms_pad up to this size take the one-warp-per-QP path
constexpr int kMaxSmem = 232448 - 1024;   // 227 KB opt-in limit per CTA on sm_90, minus static smem slack

}  // namespace
#include "qp_common.cuh"
namespace {

// Reduced KKT solve with the current factor (solve_kkt, batch.py:349-372), whitened:
//   aug (in: -h_full restricted to the S system, already forward-substituted) -> w = S^-1 (-h_full)
// is done by the callers through chol_partial/trsv; this helper finishes dxt = -t - W^T w.
__device__ __forceinline__ void finish_dxt(const double* W, int ldw, int ms, int n, const double* w,
                                           const double* t, double* dxt, double* part, int vl,
                                           int tid, int nt) {
    const int G = matvec_cols_partial(W, ldw, ms, n, w, part, vl, tid, nt);
    __syncthreads();
    for (int c = tid; c < n; c += nt) {
        double s = 0.0;
        for (int g = 0; g < G; ++g) s += part[g * vl + c];
        dxt[c] = -t[c] - s;
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// k_setup: pre_factor_kkt. One CTA per (Q,G,A) system.
// ---------------------------------------------------------------------------------------------
// kTiny: the same kernel launched with ONE WARP per system (plan->tiny: nz, ms <= 32), up to 16 systems per SM; every
// __syncthreads() is then a single-warp barrier and the rows-per-thread loops make one pass.
template <bool kSmem, bool kTiny = false>
__global__ void __launch_bounds__(kTiny ? kTinyThreads : kThreads, kTiny ? kTinyCtasPerSm : 1)
k_setup(KDims D, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ G, int64_t sG,
        const double* __restrict__ A, int64_t sA, double* __restrict__ Lfac,
        double* __restrict__ Wfac, double* __restrict__ Kfac, int* __restrict__ spd_flag,
        double* __restrict__ gscratch, int64_t scratch_per_sys, int pf) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int sys = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, ms = D.ms;
    const int ldn = ld_for(n), ldk = ld_for(ms);
    const int regA = max(n * ldn, ms * ldk);
    double* base = kSmem ? smem : (gscratch + (int64_t)sys * scratch_per_sys);
    double* RA = base;                 // Q -> L, later K
    double* RB = base + regA;          // [Apad; G] -> W   (ms x ldn)
    double* dinv = kSmem ? (smem + regA + ms * ldn) : smem;   // max(n, ms) doubles
    __shared__ int s_flag;
    if (tid == 0) s_flag = 0;

    const double* Qg = Q + (int64_t)sys * sQ;
    const double* Gg = G + (int64_t)sys * sG;
    const double* Ag = (e > 0) ? (A + (int64_t)sys * sA) : nullptr;
    copy_matrix(RA, ldn, Qg, n, n, n, tid, nt);
    if (e > 0) copy_matrix(RB, ldn, Ag, n, e, n, tid, nt);
    for (int i = tid; i < (ep - e) * n; i += nt) {   // identity-padded equality rows: W row = 0
        const int r = e + i / n, c = i % n;
        RB[r * ldn + c] = 0.0;
    }
    copy_matrix(RB + ep * ldn, ldn, Gg, n, m, n, tid, nt);
    __syncthreads();
    if (D.reg > 0.0) {                                       // Q~ = Q + eps I (solve_kkt_ir, batch.py:247-249)
        for (int i = tid; i < n; i += nt) RA[i * ldn + i] += D.reg;
        __syncthreads();
    }

    // [Q; Apad; G] -> [L; W]: Cholesky of Q with the constraint rows riding along (W = [A;G] L^-T)
    chol_partial(RA, ldn, n, 0, n, RB, ldn, ms, dinv, &s_flag, tid, nt);

    double* Lg = Lfac + (int64_t)sys * D.lp;                 // packed lower
    double* Wg = Wfac + (int64_t)sys * ms * D.ldw;           // row stride ldw (= the SMEM layout)
    // msp rows, row stride lds (= the SMEM layout), or the staircase of the product-form kernels (qp_pf.cuh)
    double* Kg = Kfac + (int64_t)sys * (pf ? qpb::pf::pf_elems(D.msp >> 3) : D.msp * D.lds);
    for (int i = tid; i < n * n; i += nt) {
        const int r = i / n, c = i - r * n;
        if (c <= r) Lg[(r * (r + 1)) / 2 + c] = RA[r * ldn + c];
    }
    if (tid == 0 && (D.lp > n * (n + 1) / 2)) Lg[D.lp - 1] = 0.0;
    for (int i = tid; i < ms * D.ldw; i += nt) {
        const int r = i / D.ldw, c = i - r * D.ldw;
        Wg[i] = (c < n) ? RB[r * ldn + c] : 0.0;
    }
    if (tid == 0) spd_flag[sys] = s_flag;
    __syncthreads();

    // K = W W^T (lower 8x8 tiles, DMMA), dummy equality rows get a unit diagonal
    {
        const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
        const int g = lane >> 2, q = lane & 3;
        const int nts = (ms + 7) >> 3;
        const int T = nts * (nts + 1) / 2;
        for (int t = warp; t < T; t += nw) {
            int ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while (ti * (ti + 1) / 2 > t) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
            const int tj = t - ti * (ti + 1) / 2;
            const int rr = 8 * ti + g, br = 8 * tj + g;
            const bool rok = rr < ms, bok = br < ms;
            const double* pa = RB + (rok ? rr : 0) * ldn;
            const double* pb = RB + (bok ? br : 0) * ldn;
            double c0 = 0.0, c1 = 0.0;
            for (int kk = 0; kk < n; kk += 4) {                 // warp-uniform trip count (mma.sync)
                const int k = kk + q;
                const double a = (rok && k < n) ? pa[k] : 0.0, b = (bok && k < n) ? pb[k] : 0.0;
                dmma884(c0, c1, a, b);
            }
            const int cc = 8 * tj + 2 * q;
            // dummy equality rows: unit diagonal; real ones: + eps in the regularised variant (A Q~^-1 A^T + eps I)
            if (rok && cc < ms) RA[rr * ldk + cc] = c0 + ((rr == cc && rr >= e && rr < ep) ? 1.0 : ((rr == cc && rr < e) ? D.reg : 0.0));
            if (rok && cc + 1 < ms) RA[rr * ldk + cc + 1] = c1 + ((rr == cc + 1 && rr >= e && rr < ep) ? 1.0 : ((rr == cc + 1 && rr < e) ? D.reg : 0.0));
        }
    }
    __syncthreads();
    if (ep > 0) chol_partial(RA, ldk, ms, 0, ep, nullptr, 0, 0, dinv, nullptr, tid, nt);
    for (int i = tid; i < ms * ldk; i += nt) {                  // clean upper triangle (DMMA tiles spill into it)
        const int r = i / ldk, c = i - r * ldk;
        if (c > r) RA[i] = 0.0;
    }
    __syncthreads();
    // storage convention: the diagonal of the pre-factored equality columns holds 1 / L_cc
    for (int i = tid; i < ep; i += nt) RA[i * ldk + i] = 1.0 / RA[i * ldk + i];
    __syncthreads();
    if (pf) {                                                   // equality columns -> product form, K -> staircase
        qpb::pf::pf_convert_cols(RA, ldk, ms, ep >> 3, tid, nt);
        qpb::pf::pf_write_staircase(Kg, RA, ldk, ms, D.msp, tid, nt);
        return;
    }
    for (int i = tid; i < D.msp * D.lds; i += nt) {             // msp rows: identity-padded to a multiple of 8
        const int r = i / D.lds, c = i - r * D.lds;
        Kg[i] = (r < ms) ? ((c < ms) ? RA[r * ldk + c] : 0.0) : (r == c ? 1.0 : 0.0);
    }
}

// ---------------------------------------------------------------------------------------------
// Shared pieces of k_forward / k_backward / k_solve_kkt
// ---------------------------------------------------------------------------------------------
struct Ctx {
    const double* W;    // ms x ldw   (shared memory, or the factor storage itself in global mode)
    double* LS;         // rows_s x lds: S workspace
    const double* Lp;   // packed lower chol(Q)
    double* vec;        // vector slots
    double* red;        // reduction scratch
    uint64_t* bar;      // [0]: W + L staged, [1]: K -> LS copies       (shared-memory mode only)
    const double* Kg;   // K template in global memory (row stride lds)
    uint32_t kphase;    // parity of the next K copy completion
    bool kpending;
};

// K -> LS: one TMA bulk copy per factor_kkt call, issued as soon as the previous factor is dead so that it
// overlaps the step-length / residual work of the Newton iteration. Call with all threads, after a barrier.
template <bool kSmem>
__device__ __forceinline__ void issue_K(const KDims& D, Ctx& C, int tid) {
    if (kSmem) {
        if (tid < 32) {
            fence_proxy_async();
            if (tid == 0) mbar_expect_tx(C.bar + 1, (uint32_t)(D.ms * D.lds * 8));
            __syncwarp();
            bulk_issue_warp(C.LS, C.Kg, (uint32_t)(D.ms * D.lds * 8), C.bar + 1, tid);
        }
    }
    C.kpending = true;
}
template <bool kSmem>
__device__ __forceinline__ void wait_K(const KDims& D, Ctx& C, int tid, int nt) {
    if (kSmem) {
        mbar_wait(C.bar + 1, C.kphase);
        C.kphase ^= 1u;
    } else {
        copy_K(C.LS, C.Kg, D.ms * D.lds, tid, nt);
        __syncthreads();
    }
    C.kpending = false;
}

template <bool kSmem>
__device__ __forceinline__ Ctx make_ctx(const KDims& D, double* smem, double* gscratch,
                                        int64_t scratch_per_qp, int qp, const double* Lfac,
                                        const double* Wfac, const double* Kfac, int sF) {
    Ctx c;
    const int64_t sys = sF ? qp : 0;
    const double* Lg = Lfac + sys * (int64_t)D.lp;
    const double* Wg = Wfac + sys * (int64_t)D.ms * D.ldw;
    c.Kg = Kfac + sys * (int64_t)D.msp * D.lds;
    c.kphase = 0;
    c.kpending = false;
    const int tid = threadIdx.x;
    if (kSmem) {
        double* W = smem;
        c.LS = W + D.ms * D.ldw;
        double* Lp = c.LS + D.rows_s * D.lds;
        c.vec = Lp + D.lp;
        c.red = c.vec + (size_t)V_COUNT * D.vl;
        c.bar = reinterpret_cast<uint64_t*>(c.red + kRedDoubles);
        c.W = W;
        c.Lp = Lp;
        if (tid == 0) {
            mbar_init(c.bar, 1);
            mbar_init(c.bar + 1, 1);
        }
        __syncthreads();
        if (tid < 32) {
            const uint32_t wb = (uint32_t)(D.ms * D.ldw * 8), lb = (uint32_t)(D.lp * 8);
            if (tid == 0) mbar_expect_tx(c.bar, wb + lb);
            __syncwarp();
            bulk_issue_warp(W, Wg, wb, c.bar, tid);
            bulk_issue_warp(Lp, Lg, lb, c.bar, tid);
        }
        issue_K<kSmem>(D, c, tid);
        mbar_wait(c.bar, 0);
    } else {
        c.W = Wg;
        c.Lp = Lg;
        c.LS = gscratch + (int64_t)qp * scratch_per_qp;
        c.vec = smem;
        c.red = c.vec + (size_t)V_COUNT * D.vl;
        c.bar = nullptr;
        c.kpending = true;
    }
    return c;
}

#define VEC(i) (C.vec + (size_t)(i) * D.vl)

// factor_kkt + the forward half of solve_kkt: on entry V_AUG holds -h_full (length ms) and V_D holds d.
// On exit V_W holds w = -S^-1 h_full. Destroys V_AUG, V_T0.
// kReg: V_D holds d + eps and the inequality diagonal gets 1 / (d + eps) + eps (the regularised system of the kReg
// kernels; the eps of the equality rows is already in K, pre_factor_kkt_reg).
template <bool kSmem, bool kReg = false>
__device__ __forceinline__ void factor_and_solve(const KDims& D, Ctx& C, int tid, int nt) {
    double* aug = VEC(V_AUG);
    wait_K<kSmem>(D, C, tid, nt);
    for (int i = D.ep + tid; i < D.ms; i += nt)
        C.LS[i * D.lds + i] += kReg ? 1.0 / VEC(V_D)[i] + D.reg : 1.0 / VEC(V_D)[i];
    __syncthreads();
    const FullIdx at{D.lds};
    if (D.ep > 0) {
        // equality block: forward-substitute the first ep entries with the pre-factored L11 / L21
        trsv_fwd(C.LS, at, D.ms, 0, D.ep, VEC(V_DINV), aug, VEC(V_T0), tid, nt);
        for (int i = tid; i < D.ep; i += nt) aug[i] = VEC(V_T0)[i];
        __syncthreads();
    }
    chol_partial(C.LS, D.lds, D.ms, D.ep, D.ms, aug, 0, 1, VEC(V_DINV), nullptr, tid, nt);
    trsv_bwd(C.LS, at, D.ms, VEC(V_DINV), aug, VEC(V_W), tid, nt);
}

// Solve with the factor already in LS: rhs in V_T1 (destroyed) -> result in `out`.
__device__ __forceinline__ void solve_with_factor(const KDims& D, const Ctx& C, double* out, int tid,
                                                  int nt) {
    const FullIdx at{D.lds};
    trsv_fwd(C.LS, at, D.ms, 0, D.ms, VEC(V_DINV), VEC(V_T1), VEC(V_T0), tid, nt);
    trsv_bwd(C.LS, at, D.ms, VEC(V_DINV), VEC(V_T0), out, tid, nt);
}

// x~ = L^-1 x: V_T1 (destroyed) -> dst.  x = L^-T x~: u (destroyed) -> out.
__device__ __forceinline__ void whiten(const KDims& D, const Ctx& C, double* dst, int tid, int nt) {
    trsv_fwd(C.Lp, PackedIdx{}, D.n, 0, D.n, VEC(V_DINVL), VEC(V_T1), dst, tid, nt);
}
__device__ __forceinline__ void unwhiten(const KDims& D, const Ctx& C, double* u, double* out, int tid,
                                         int nt) {
    trsv_bwd(C.Lp, PackedIdx{}, D.n, VEC(V_DINVL), u, out, tid, nt);
}
// common prologue: reciprocal diagonals of L and of the pre-factored equality block
__device__ __forceinline__ void load_dinvs(const KDims& D, const Ctx& C, int tid, int nt) {
    for (int i = tid; i < D.n; i += nt) VEC(V_DINVL)[i] = 1.0 / C.Lp[(i * (i + 1)) / 2 + i];
    for (int i = tid; i < D.ep; i += nt) VEC(V_DINV)[i] = C.Kg[(int64_t)i * D.lds + i];   // K stores 1/L_cc there
}

// ---- regularised mode (kReg: QPFunction with kkt_solver=IR_UNOPT) on the generic kernels ------------------------------
// The arithmetic of fk::f_true_rx / fk::f_refine (qp_solve.cuh) with the generic building blocks: the factors are those
// of pre_factor_kkt_reg (L = chol(Q + eps I), K with eps on the equality rows), every KKT solve uses the regularised
// system [Q+eI 0 G' A'; 0 D+eI I 0; G I -eI 0; A 0 0 -eI], and the residuals are those of the true problem.

// r~x -= eps L^-1 L^-T x~: the whitened dual residual of the true problem from the one of Q + eps I. Destroys V_T0,
// V_T1. Ends with a block barrier.
__device__ __forceinline__ void true_rx(const KDims& D, const Ctx& C, const double* xt, double* rxt, int tid, int nt) {
    double* t0 = VEC(V_T0);
    for (int i = tid; i < D.n; i += nt) t0[i] = xt[i];
    __syncthreads();
    unwhiten(D, C, t0, VEC(V_T1), tid, nt);                    // T1 = x = L^-T x~
    whiten(D, C, t0, tid, nt);                                  // T0 = L^-1 x
    for (int i = tid; i < D.n; i += nt) rxt[i] = fma(-D.reg, t0[i], rxt[i]);
    __syncthreads();
}

// One refinement step, with the factor still in the S workspace, of a solution of the regularised system: dv = [dy; dz],
// ds, and dx~ = -base + ntx - W^T dv kept implicit. With K = K~ - Delta, the true residual of d = d0 + c1 + .. + ck is
// -Delta ck = (-eps dx, -eps ds, eps dz, eps dy) of the LAST correction ck (of the solution d0 itself in the first step);
// the next correction solves the regularised system with it and is added in place (ntx += eps L^-1 dx).
// Between the steps of one solve c, e, f carry that correction: c = -eps L^-1 dx, e = eps ds, f = [dy; dz]; the first
// step (first = true) reads the solution instead. V_D holds d + eps. a: scratch slot; destroys V_T0, V_T1, V_PART.
// Ends with a block barrier.
__device__ __forceinline__ void refine(const KDims& D, const Ctx& C, const double* base, double* ntx, double* dv,
                                       double* ds, double* a, double* c, double* e, double* f, bool first, int tid,
                                       int nt) {
    const double* dd = VEC(V_D);
    double* t1 = VEC(V_T1); double* part = VEC(V_PART);
    const int G = matvec_cols_partial(C.W, D.ldw, D.ms, D.n, first ? dv : f, part, D.vl, tid, nt);
    __syncthreads();
    if (first) {
        for (int i = tid; i < D.n; i += nt) {
            double s = 0.0;
            for (int g = 0; g < G; ++g) s += part[g * D.vl + i];
            a[i] = ntx[i] - base[i] - s;                        // dx~ of the solution
        }
    } else {
        for (int i = tid; i < D.n; i += nt) {
            double s = 0.0;
            for (int g = 0; g < G; ++g) s += part[g * D.vl + i];
            a[i] = -c[i] - s;                                   // dx~ of the correction: eps L^-1 dx - W^T f
        }
    }
    __syncthreads();
    unwhiten(D, C, a, t1, tid, nt);                             // T1 = dx
    whiten(D, C, c, tid, nt);                                   // c = L^-1 dx
    for (int i = tid; i < D.n; i += nt) {
        const double r = D.reg * c[i];
        c[i] = -r;                                              // whitened x residual  L^-1 (-eps dx)
        ntx[i] += r;
    }
    __syncthreads();
    double* wt = first ? e : a;                                 // W t (e holds eps ds of the correction after the first)
    matvec_rows<false>(C.W, D.ldw, D.ms, D.n, c, nullptr, wt, nullptr, tid, nt);
    __syncthreads();
    // reduced right-hand side -(W t - [r_y; r_z] + [0; r_s / (d + eps)])  (the elimination of solve_kkt)
    if (first) {
        for (int i = tid; i < D.ms; i += nt) {
            double hf = fma(-D.reg, dv[i], e[i]);
            if (i >= D.ep) hf -= D.reg * ds[i] / dd[i];
            t1[i] = -hf;
        }
    } else {
        for (int i = tid; i < D.ms; i += nt) {
            double hf = fma(-D.reg, f[i], a[i]);
            if (i >= D.ep) hf -= e[i] / dd[i];
            t1[i] = -hf;
        }
    }
    __syncthreads();
    solve_with_factor(D, C, f, tid, nt);                        // f = correction of [dy; dz]
    if (first) {
        for (int i = tid; i < D.ms; i += nt) {
            const double wi = f[i];
            if (i >= D.ep) {
                const double dsc = (D.reg * ds[i] - wi) / dd[i];
                ds[i] += dsc;
                e[i] = D.reg * dsc;
            }
            dv[i] += wi;
        }
    } else {
        for (int i = tid; i < D.ms; i += nt) {
            const double wi = f[i];
            if (i >= D.ep) {
                const double dsc = (e[i] - wi) / dd[i];
                ds[i] += dsc;
                e[i] = D.reg * dsc;
            }
            dv[i] += wi;
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// k_forward: the PDIPM loop (batch.py:47-207), per-QP semantics.
// ---------------------------------------------------------------------------------------------
// kReg (with !kSmem, !kTiny: the global-scratch build): the regularised mode (true_rx, refine); D.reg = eps, ir_steps
// refinement steps of the initial point and of each iteration's combined direction (a trailing parameter: KDims keeps
// its layout).
template <bool kSmem, bool kTiny = false, bool kReg = false>
__global__ void __launch_bounds__(kTiny ? kTinyThreads : kThreads, kTiny ? kTinyCtasPerSm : 1)
k_forward(KDims D, const double* __restrict__ p, int64_t sp, const double* __restrict__ h,
          int64_t sh, const double* __restrict__ b, int64_t sb, const double* __restrict__ Lfac,
          const double* __restrict__ Wfac, const double* __restrict__ Kfac, int sF, double eps,
          double stall_tol, double best_tie, int notImprovedLim, int maxIter, double* __restrict__ zhat, double* __restrict__ lam,
          double* __restrict__ slacks, double* __restrict__ nus, int* __restrict__ iters_out,
          double* __restrict__ resid_out, double* __restrict__ trace, double* __restrict__ gscratch,
          int64_t scratch_per_qp, int ir_steps = 0) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, ms = D.ms;
    Ctx C = make_ctx<kSmem>(D, smem, gscratch, scratch_per_qp, qp, Lfac, Wfac, Kfac, sF);

    double* pt = VEC(V_PT); double* xt = VEC(V_XT); double* rxt = VEC(V_RXT);
    double* s = VEC(V_S); double* v = VEC(V_V); double* rv = VEC(V_RV); double* hW = VEC(V_HW);
    double* c2 = VEC(V_C2); double* w = VEC(V_W); double* wc = VEC(V_WC); double* dsa = VEC(V_DSA);
    double* ds = VEC(V_DS); double* dxt = VEC(V_DXT); double* d = VEC(V_D); double* hb = VEC(V_HB);
    double* aug = VEC(V_AUG); double* t1 = VEC(V_T1); double* part = VEC(V_PART);

    // ---- load per-QP vectors; hb = [b; 0; h]
    const double* pg = p + (int64_t)qp * sp;
    const double* hg = h + (int64_t)qp * sh;
    const double* bg = (e > 0) ? (b + (int64_t)qp * sb) : nullptr;
    for (int i = tid; i < n; i += nt) t1[i] = pg[i];
    for (int i = tid; i < ms; i += nt) {
        double val = 0.0;
        if (i < e) val = bg[i];
        else if (i >= ep) val = hg[i - ep];
        hb[i] = val;
        d[i] = kReg ? 1.0 + D.reg : 1.0;
        s[i] = 0.0;
    }
    load_dinvs(D, C, tid, nt);
    __syncthreads();
    whiten(D, C, pt, tid, nt);                                  // p~ = L^-1 p

    // ---- initial point: solve_kkt(p, 0, -h, -b) with d = 1   (batch.py:61-67)
    matvec_rows<false>(C.W, D.ldw, ms, n, pt, nullptr, hW, nullptr, tid, nt);
    __syncthreads();
    for (int i = tid; i < ms; i += nt) aug[i] = -(hW[i] + hb[i]);
    __syncthreads();
    factor_and_solve<kSmem, kReg>(D, C, tid, nt);
    const bool refine_on = kReg && ir_steps > 0;
    if (kReg) {
        // s = -w / (1 + eps); rv accumulates the x part of the refinement (x~ = -p~ + rv - W^T w)
        for (int i = ep + tid; i < ms; i += nt) s[i] = -w[i] / d[i];
        for (int i = tid; i < n; i += nt) rv[i] = 0.0;
        __syncthreads();
        for (int k = 0; k < ir_steps; ++k) refine(D, C, pt, rv, w, s, aug, hW, c2, dsa, k == 0, tid, nt);
        for (int i = tid; i < n; i += nt) hW[i] = pt[i] - rv[i];   // (read after finish_dxt's first barrier)
    }
    issue_K<kSmem>(D, C, tid);
    finish_dxt(C.W, D.ldw, ms, n, w, kReg ? hW : pt, xt, part, D.vl, tid, nt);   // x~ = -p~ - W^T w
    {
        double mn[2] = {INFINITY, INFINITY};
        for (int i = ep + tid; i < ms; i += nt) {
            v[i] = w[i];
            if (kReg) {
                mn[0] = fmin(mn[0], s[i]);
            } else {
                s[i] = -w[i];
                mn[0] = fmin(mn[0], -w[i]);
            }
            mn[1] = fmin(mn[1], w[i]);
        }
        for (int i = tid; i < ep; i += nt) v[i] = w[i];
        block_reduce<2, true>(mn, C.red, tid, nt);
        // make slacks and inequality duals >= 1 (batch.py:77-87)
        for (int i = ep + tid; i < ms; i += nt) {
            if (mn[0] < 0.0) s[i] -= mn[0] - 1.0;
            if (mn[1] < 0.0) v[i] -= mn[1] - 1.0;
        }
        __syncthreads();
    }

    double best = 0.0;
    int nNot = 0, it = 0, iters_run = 0;
    const double dm = (double)m;
    for (it = 0; it < maxIter; ++it) {
        iters_run = it + 1;
        // ---- residuals (batch.py:94-107)
        {
            const int G = matvec_cols_partial(C.W, D.ldw, ms, n, v, part, D.vl, tid, nt);
            __syncthreads();
            for (int c = tid; c < n; c += nt) {
                double sum = 0.0;
                for (int g = 0; g < G; ++g) sum += part[g * D.vl + c];
                rxt[c] = xt[c] + pt[c] + sum;                   // L^-1 (Qx + p + G^T z + A^T y)
            }
            __syncthreads();
        }
        if (kReg) true_rx(D, C, xt, rxt, tid, nt);
        matvec_rows<true>(C.W, D.ldw, ms, n, xt, rxt, c2, hW, tid, nt);
        __syncthreads();
        double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // |ry|^2, |rz|^2, |L r~x|^2, s.z
        for (int i = tid; i < ms; i += nt) {
            const double r = c2[i] - hb[i] + ((i >= ep) ? s[i] : 0.0);   // [Ax - b; Gx + s - h]
            rv[i] = r;
            if (i < ep) acc[0] = fma(r, r, acc[0]);
            else { acc[1] = fma(r, r, acc[1]); acc[3] = fma(s[i], v[i], acc[3]); }
        }
        acc[2] = tri_norm2_partial(C.Lp, n, rxt, tid, nt);      // || L r~x ||^2 = ||Qx + p + G^T z + A^T y||^2
        block_reduce<4, false>(acc, C.red, tid, nt);
        const double mu = fabs(acc[3] / dm);
        const double resid = sqrt(acc[1]) + sqrt(acc[0]) + sqrt(acc[2]) + dm * mu;
        if (trace != nullptr && tid == 0) {                     // what verbose=1 prints (batch.py:115-117)
            double* tr = trace + ((int64_t)qp * maxIter + it) * 4;
            tr[0] = sqrt(acc[1]) + sqrt(acc[0]); tr[1] = sqrt(acc[2]); tr[2] = mu; tr[3] = resid;
        }
        // ---- best-iterate tracking and exit tests (batch.py:118-143), per QP
        const bool improved = (it == 0) || (resid < best);      // strict, as the reference (NaN never improves)
        if (improved) { best = resid; nNot = 0; } else { ++nNot; }
        // Returned iterate: the reference keeps argmin resids. At the rounding floor consecutive iterates tie
        // to within noise while mu keeps shrinking 1000x per step; among iterates within best_tie of the
        // minimum the LATEST is kept, so the backward pass's 1e-8 clamps (qp.py:148) see converged duals.
        if (improved || resid < best_tie * best) {
            for (int i = tid; i < n; i += nt) VEC(V_BXT)[i] = xt[i];
            for (int i = tid; i < ms; i += nt) { VEC(V_BS)[i] = s[i]; VEC(V_BV)[i] = v[i]; }
        }
        // batch.py:140 per QP; the not-improved rule only fires once the QP is in its converged regime
        // (best < stall_tol): in a batch the reference keeps iterating while any other QP improves.
        if ((nNot == notImprovedLim && best < stall_tol) || best < eps || mu > 1e32) break;
        if (!(resid == resid) || isinf(resid)) break;           // every later iterate is NaN too
        // ---- factor_kkt with d = z/s and the affine right-hand side (batch.py:109-113,150)
        for (int i = tid; i < ms; i += nt) {
            double hfull = hW[i] - rv[i];
            if (i >= ep) {
                const double di = kReg ? v[i] / s[i] + D.reg : v[i] / s[i];
                d[i] = di;
                hfull += v[i] / di;                             // rs/d with rs = z
            }
            aug[i] = -hfull;
        }
        __syncthreads();
        factor_and_solve<kSmem, kReg>(D, C, tid, nt);                // w = [dy_aff; dz_aff]
        // ---- affine step length and sigma (batch.py:160-168)
        double mn[2] = {INFINITY, INFINITY};
        for (int i = ep + tid; i < ms; i += nt) {
            const double dz = w[i];
            const double dsi = (-v[i] - dz) / d[i];
            dsa[i] = dsi;
            mn[0] = fmin(mn[0], step_candidate(v[i], dz));
            mn[1] = fmin(mn[1], step_candidate(s[i], dsi));
        }
        block_reduce<2, true>(mn, C.red, tid, nt);
        {
            const double stz = isinf(mn[0]) && mn[0] > 0 ? 1.0 : mn[0];
            const double sts = isinf(mn[1]) && mn[1] > 0 ? 1.0 : mn[1];
            const double alpha = fmin(fmin(stz, sts), 1.0);
            double sm[2] = {0.0, 0.0};
            for (int i = ep + tid; i < ms; i += nt) {
                sm[0] = fma(s[i] + alpha * dsa[i], v[i] + alpha * w[i], sm[0]);
                sm[1] = fma(s[i], v[i], sm[1]);
            }
            block_reduce<2, false>(sm, C.red, tid, nt);
            const double sr = sm[0] / sm[1];
            const double sig = sr * sr * sr;
            // ---- corrector (batch.py:170-181): rx = rz = ry = 0, rs = (-mu*sig + ds_aff*dz_aff)/s
            for (int i = tid; i < ms; i += nt) {
                double rhs = 0.0;
                if (i >= ep) {
                    const double rsc = (-mu * sig + dsa[i] * w[i]) / s[i];
                    ds[i] = rsc;                                 // keep rs_c for ds_cor below
                    rhs = -(rsc / d[i]);
                }
                t1[i] = rhs;
            }
            __syncthreads();
        }
        solve_with_factor(D, C, wc, tid, nt);                        // wc = [dy_cor; dz_cor]
        if (!refine_on) issue_K<kSmem>(D, C, tid);              // next factor_kkt's copy of K overlaps the rest
        // ---- combined direction, step length, update (batch.py:185-203)
        mn[0] = INFINITY; mn[1] = INFINITY;
        for (int i = tid; i < ms; i += nt) {
            const double dv = w[i] + wc[i];
            w[i] = dv;
            if (i >= ep) {
                const double dsc = (-ds[i] - wc[i]) / d[i];
                const double dsi = dsa[i] + dsc;
                ds[i] = dsi;
                mn[0] = fmin(mn[0], step_candidate(v[i], dv));
                mn[1] = fmin(mn[1], step_candidate(s[i], dsi));
            }
        }
        if (refine_on) for (int i = tid; i < n; i += nt) rv[i] = 0.0;
        __syncthreads();
        if (refine_on) {
            // The refinement is linear in the right-hand side, so refining the combined direction equals refining the
            // affine and the corrector direction one by one; sigma above comes from the unrefined affine direction.
            for (int k = 0; k < ir_steps; ++k) refine(D, C, rxt, rv, w, ds, aug, hW, c2, wc, k == 0, tid, nt);
            issue_K<kSmem>(D, C, tid);
            mn[0] = INFINITY; mn[1] = INFINITY;
            for (int i = ep + tid; i < ms; i += nt) {
                mn[0] = fmin(mn[0], step_candidate(v[i], w[i]));
                mn[1] = fmin(mn[1], step_candidate(s[i], ds[i]));
            }
            for (int i = tid; i < n; i += nt) rxt[i] -= rv[i];   // dx~ = -(r~x - rv) - W^T dv (read after a barrier)
        }
        finish_dxt(C.W, D.ldw, ms, n, w, rxt, dxt, part, D.vl, tid, nt);   // dx~ = -r~x - W^T dv
        block_reduce<2, true>(mn, C.red, tid, nt);
        {
            const double stz = isinf(mn[0]) && mn[0] > 0 ? 1.0 : mn[0];
            const double sts = isinf(mn[1]) && mn[1] > 0 ? 1.0 : mn[1];
            const double alpha = fmin(0.999 * fmin(stz, sts), 1.0);
            for (int i = tid; i < n; i += nt) xt[i] = fma(alpha, dxt[i], xt[i]);
            for (int i = tid; i < ms; i += nt) {
                v[i] = fma(alpha, w[i], v[i]);
                if (i >= ep) s[i] = fma(alpha, ds[i], s[i]);
            }
        }
        __syncthreads();
    }

    // ---- outputs: x = L^-T x~_best, y, z, s of the best iterate (batch.py:205-207)
    __syncthreads();
    unwhiten(D, C, VEC(V_BXT), VEC(V_T0), tid, nt);
    if (kSmem && C.kpending) wait_K<kSmem>(D, C, tid, nt);      // drain the in-flight copy before exit
    for (int i = tid; i < n; i += nt) zhat[(int64_t)qp * n + i] = VEC(V_T0)[i];
    for (int i = tid; i < m; i += nt) {
        lam[(int64_t)qp * m + i] = VEC(V_BV)[ep + i];
        slacks[(int64_t)qp * m + i] = VEC(V_BS)[ep + i];
    }
    if (e > 0 && nus != nullptr)
        for (int i = tid; i < e; i += nt) nus[(int64_t)qp * e + i] = VEC(V_BV)[i];
    if (tid == 0) {
        iters_out[qp] = iters_run;
        resid_out[qp] = best;          // the minimum over the iterations, as the reference reports (batch.py:126-142)
    }
}

// ---------------------------------------------------------------------------------------------
// k_solve_kkt: factor_kkt + solve_kkt for caller-supplied d and right-hand sides.
// kBackward: the backward pass of QPFunction (qp.py:128-182): d from clamped lam/slacks, rx = dl,
// other right-hand sides zero, fused gradient outer products for batched inputs.
// kReg (with kBackward, !kSmem, !kTiny: the global-scratch build): the backward pass of the regularised mode, d + eps and
// ir_steps refinement steps (refine).
// ---------------------------------------------------------------------------------------------

template <bool kSmem, bool kBackward, bool kTiny = false, bool kReg = false>
__global__ void __launch_bounds__(kTiny ? kTinyThreads : kThreads, kTiny ? kTinyCtasPerSm : 1)
k_solve_kkt(KDims D, const double* __restrict__ d_in, const double* __restrict__ rx_in,
            const double* __restrict__ rs_in, const double* __restrict__ rz_in,
            const double* __restrict__ ry_in, const double* __restrict__ zhat,
            const double* __restrict__ lam, const double* __restrict__ slacks,
            const double* __restrict__ nus, const double* __restrict__ Lfac,
            const double* __restrict__ Wfac, const double* __restrict__ Kfac, int sF,
            double* __restrict__ dx_out, double* __restrict__ ds_out, double* __restrict__ dz_out,
            double* __restrict__ dy_out, BwdOut O, double* __restrict__ gscratch,
            int64_t scratch_per_qp, int ir_steps = 0) {
    extern __shared__ __align__(16) double smem[];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, ms = D.ms;
    Ctx C = make_ctx<kSmem>(D, smem, gscratch, scratch_per_qp, qp, Lfac, Wfac, Kfac, sF);
    double* t = VEC(V_PT); double* d = VEC(V_D); double* hW = VEC(V_HW); double* aug = VEC(V_AUG);
    double* w = VEC(V_W); double* t1 = VEC(V_T1); double* dxt = VEC(V_DXT); double* part = VEC(V_PART);
    double* rsv = VEC(V_S);

    for (int i = tid; i < n; i += nt) t1[i] = rx_in[(int64_t)qp * n + i];
    for (int i = tid; i < ms; i += nt) {
        double di = 1.0, extra = 0.0, rsi = 0.0;
        if (i >= ep) {
            const int j = i - ep;
            if (kBackward) {
                di = fmax(lam[(int64_t)qp * m + j], 1e-8) / fmax(slacks[(int64_t)qp * m + j], 1e-8);   // qp.py:148
                if (kReg) di += D.reg;
                if (rz_in != nullptr) extra = -rz_in[(int64_t)qp * m + j];   // dl/dlam (rs = 0)
            } else {
                // regularised variant (D.reg > 0, batch.py:244-310): d~ = d + eps in the complementarity row, and the slot
                // holds 1 / (1/d~ + eps) because factor_kkt adds the RECIPROCAL of this slot to the diagonal of S
                const double dt = d_in[(int64_t)qp * m + j] + D.reg;
                di = (D.reg > 0.0) ? 1.0 / (1.0 / dt + D.reg) : dt;
                rsi = rs_in[(int64_t)qp * m + j];
                extra = rsi / dt - rz_in[(int64_t)qp * m + j];
            }
        } else if (i < e && (!kBackward || ry_in != nullptr)) {     // (backward: dl/dnu)
            extra = -ry_in[(int64_t)qp * e + i];
        }
        d[i] = di;
        rsv[i] = rsi;
        hW[i] = extra;                                          // [-ry; rs/d - rz]
    }
    load_dinvs(D, C, tid, nt);
    __syncthreads();
    whiten(D, C, t, tid, nt);                                   // t = L^-1 rx
    matvec_rows<false>(C.W, D.ldw, ms, n, t, nullptr, VEC(V_C2), nullptr, tid, nt);
    __syncthreads();
    for (int i = tid; i < ms; i += nt) aug[i] = -(VEC(V_C2)[i] + hW[i]);
    __syncthreads();
    factor_and_solve<kSmem, kReg>(D, C, tid, nt);                    // w = [dy; dz]
    if (kReg) {
        double* ntx = VEC(V_DSA); double* dsr = VEC(V_DS);     // x part of the refinement (dx~ = -t + ntx - W^T w), ds
        for (int i = ep + tid; i < ms; i += nt) dsr[i] = -w[i] / d[i];   // (rs = 0)
        for (int i = tid; i < n; i += nt) ntx[i] = 0.0;
        __syncthreads();
        for (int k = 0; k < ir_steps; ++k) refine(D, C, t, ntx, w, dsr, aug, hW, VEC(V_C2), VEC(V_WC), k == 0, tid, nt);
        for (int i = tid; i < n; i += nt) t[i] -= ntx[i];       // (read after finish_dxt's first barrier)
    }
    finish_dxt(C.W, D.ldw, ms, n, w, t, dxt, part, D.vl, tid, nt);
    unwhiten(D, C, dxt, VEC(V_XT), tid, nt);                    // dx = L^-T dx~
    const double* dx = VEC(V_XT);
    for (int i = tid; i < n; i += nt) dx_out[(int64_t)qp * n + i] = dx[i];
    for (int i = tid; i < m; i += nt) {
        dz_out[(int64_t)qp * m + i] = w[ep + i];
        if (!kBackward) ds_out[(int64_t)qp * m + i] = (-rsv[ep + i] - w[ep + i]) / (d_in[(int64_t)qp * m + i] + D.reg);
    }
    if (e > 0 && dy_out != nullptr)
        for (int i = tid; i < e; i += nt) dy_out[(int64_t)qp * e + i] = w[i];
    if (!kBackward) return;

    // ---- gradients for batched inputs (qp.py:157-176); mean-reduced ones are done by k_mean_*
    double* zs = VEC(V_BXT); double* ls = VEC(V_BV);
    for (int i = tid; i < n; i += nt) zs[i] = zhat[(int64_t)qp * n + i];
    for (int i = tid; i < m; i += nt) ls[ep + i] = lam[(int64_t)qp * m + i];
    for (int i = tid; i < e; i += nt) ls[i] = nus[(int64_t)qp * e + i];
    __syncthreads();
    if (O.dp && !O.mp) for (int i = tid; i < n; i += nt) O.dp[(int64_t)qp * n + i] = dx[i];
    if (O.dh && !O.mh) for (int i = tid; i < m; i += nt) O.dh[(int64_t)qp * m + i] = -w[ep + i];
    if (O.db && !O.mb && e > 0) for (int i = tid; i < e; i += nt) O.db[(int64_t)qp * e + i] = -w[i];
    if (O.dQ && !O.mQ) {
        double* o = O.dQ + (int64_t)qp * n * n;
        for (int i = tid; i < n * n; i += nt) {
            const int r = i / n, c = i - r * n;
            o[i] = 0.5 * (dx[r] * zs[c] + zs[r] * dx[c]);
        }
    }
    if (O.dG && !O.mG) {
        double* o = O.dG + (int64_t)qp * m * n;
        for (int i = tid; i < m * n; i += nt) {
            const int r = i / n, c = i - r * n;
            o[i] = w[ep + r] * zs[c] + ls[ep + r] * dx[c];
        }
    }
    if (O.dA && !O.mA && e > 0) {
        double* o = O.dA + (int64_t)qp * e * n;
        for (int i = tid; i < e * n; i += nt) {
            const int r = i / n, c = i - r * n;
            o[i] = w[r] * zs[c] + ls[r] * dx[c];
        }
    }
}

// Batch-mean gradients for un-batched inputs (qp.py:159-177):
//   out[r][c] = scale / B * sum_b (u_b[r] x_b[c] + y_b[r] v_b[c])     i.e.  scale / B * (U^T X + Y^T V),
// a (rows x B)(B x cols) product computed straight from the per-QP vectors (no B x rows x cols round trip).
// One CTA per 32 x 64 output tile: the batch is walked in chunks of 16 QPs staged in shared memory with loads that are
// contiguous in the vector index, every thread owns a 2 x 4 register tile (8 outputs, 16 FMAs per staged b).
constexpr int kMoR = 32, kMoC = 64, kMoB = 16;
__global__ void __launch_bounds__(256)
k_mean_outer(int B, int rows, int cols, const double* __restrict__ u, const double* __restrict__ x,
             const double* __restrict__ y, const double* __restrict__ v, double scale, double* __restrict__ out) {
    __shared__ double su[kMoB][kMoR], sy[kMoB][kMoR], sx[kMoB][kMoC], sv[kMoB][kMoC];
    const int tid = threadIdx.x;
    const int r0 = blockIdx.y * kMoR, c0 = blockIdx.x * kMoC;
    const int tr = (tid >> 4) * 2, tc = (tid & 15) * 4;           // 16 x 16 threads, 2 x 4 outputs each
    double acc[2][4] = {{0.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0}};
    for (int b0 = 0; b0 < B; b0 += kMoB) {
        for (int i = tid; i < kMoB * kMoR; i += 256) {
            const int bb = i / kMoR, rr = i - bb * kMoR;
            const bool ok = (b0 + bb < B) && (r0 + rr < rows);
            su[bb][rr] = ok ? u[(int64_t)(b0 + bb) * rows + r0 + rr] : 0.0;
            sy[bb][rr] = ok ? y[(int64_t)(b0 + bb) * rows + r0 + rr] : 0.0;
        }
        for (int i = tid; i < kMoB * kMoC; i += 256) {
            const int bb = i / kMoC, cc = i - bb * kMoC;
            const bool ok = (b0 + bb < B) && (c0 + cc < cols);
            sx[bb][cc] = ok ? x[(int64_t)(b0 + bb) * cols + c0 + cc] : 0.0;
            sv[bb][cc] = ok ? v[(int64_t)(b0 + bb) * cols + c0 + cc] : 0.0;
        }
        __syncthreads();
#pragma unroll 4
        for (int bb = 0; bb < kMoB; ++bb) {
            const double u0 = su[bb][tr], u1 = su[bb][tr + 1], y0 = sy[bb][tr], y1 = sy[bb][tr + 1];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double xj = sx[bb][tc + j], vj = sv[bb][tc + j];
                acc[0][j] = fma(u0, xj, fma(y0, vj, acc[0][j]));
                acc[1][j] = fma(u1, xj, fma(y1, vj, acc[1][j]));
            }
        }
        __syncthreads();
    }
    const double sc = scale / (double)B;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (r0 + tr + i < rows && c0 + tc + j < cols) out[(int64_t)(r0 + tr + i) * cols + c0 + tc + j] = acc[i][j] * sc;
}
__global__ void k_mean_vec(int B, int len, const double* __restrict__ u, double scale,
                           double* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= len) return;
    double s = 0.0;
    for (int bidx = 0; bidx < B; ++bidx) s += u[(int64_t)bidx * len + idx];
    out[idx] = s * scale / (double)B;
}


}  // namespace
#include "qp_solve.cuh"
namespace {
// ---------------------------------------------------------------------------------------------
// k_setup_fast: pre_factor_kkt (batch.py:375-429) with the fast building blocks.
//   1. chol(Q) with the pipelined f_chol (Q identity-padded to a multiple of 8),
//   2. T = L_kk^-1 for every diagonal block (warps in parallel),
//   3. W = [A; 0; G] L^-T: every 8-row tile independently inside one warp (left-looking, DMMA), no barriers,
//   4. K = W W^T (DMMA), unit diagonal on dummy / pad rows, partial Cholesky of the equality columns.
// ---------------------------------------------------------------------------------------------
namespace fk {
struct SLayout { int QA, WA, aug, tab, np, ldq, total; };
__host__ __device__ inline SLayout setup_layout(const KDims& D) {
    SLayout L;
    L.np = (D.n + 7) & ~7;
    L.ldq = ld_for(L.np);
    const int qa = L.np * L.ldq, ka = D.msp * D.lds;
    L.QA = 0;
    L.WA = qa > ka ? qa : ka;
    L.aug = L.WA + D.msp * L.ldq;
    L.tab = L.aug + (((L.np > D.msp ? L.np : D.msp) + 7) & ~7);
    L.total = L.tab + kTabDoubles;
    return L;
}
}  // namespace fk

__global__ void __launch_bounds__(kThreads, 1)
k_setup_fast(KDims D, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ G, int64_t sG,
             const double* __restrict__ A, int64_t sA, double* __restrict__ Lfac, double* __restrict__ Wfac,
             double* __restrict__ Kfac, int* __restrict__ spd_flag, int pf) {
    using namespace fk;
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sys = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, ms = D.ms, msp = D.msp;
    const SLayout S = setup_layout(D);
    const int np = S.np, ldq = S.ldq;
#ifdef QPB_TIMING
    if (threadIdx.x == 0) { for (int i = 0; i < 128; ++i) s_tim[i] = 0; s_tim[128] = clock64(); s_tim2 = s_tim[128]; }
    __syncthreads();
#endif
    __shared__ int s_flag;
    if (tid == 0) s_flag = 0;
    const double* Qg = Q + (int64_t)sys * sQ;
    const double* Gg = G + (int64_t)sys * sG;
    const double* Ag = (e > 0) ? (A + (int64_t)sys * sA) : nullptr;
    // ---- stage Q (identity padded) and [A; 0; G; 0] (zero padded): one TMA bulk copy per matrix row (the rows are
    // contiguous in HBM but padded in shared memory), padding written by the threads meanwhile.
    __shared__ __align__(8) uint64_t s_bar;
    const bool tma_rows = ((n & 1) == 0) && ((reinterpret_cast<uintptr_t>(Qg) & 15) == 0) &&
                          ((reinterpret_cast<uintptr_t>(Gg) & 15) == 0) && (e == 0 || (reinterpret_cast<uintptr_t>(Ag) & 15) == 0);
    if (tma_rows) {
        if (tid == 0) mbar_init(&s_bar, 1);
        __syncthreads();
        if (tid < 32) {
            const uint32_t rowb = (uint32_t)(n * 8);
            if (tid == 0) mbar_expect_tx(&s_bar, rowb * (uint32_t)(n + e + m));
            __syncwarp();
            for (int r = tid; r < n; r += 32) bulk_g2s(qsm + S.QA + r * ldq, Qg + (int64_t)r * n, rowb, &s_bar);
            for (int r = tid; r < e; r += 32) bulk_g2s(qsm + S.WA + r * ldq, Ag + (int64_t)r * n, rowb, &s_bar);
            for (int r = tid; r < m; r += 32) bulk_g2s(qsm + S.WA + (ep + r) * ldq, Gg + (int64_t)r * n, rowb, &s_bar);
        }
        for (int r = warp; r < np; r += kThreads / 32)
            for (int c = lane; c < ldq; c += 32)
                if (r >= n || c >= n) qsm[S.QA + r * ldq + c] = (r == c) ? 1.0 : 0.0;
        for (int r = warp; r < msp; r += kThreads / 32) {
            const bool real = (r < e) || (r >= ep && r < ms);
            for (int c = lane; c < ldq; c += 32)
                if (!real || c >= n) qsm[S.WA + r * ldq + c] = 0.0;
        }
        mbar_wait(&s_bar, 0);
    } else {
        for (int r = warp; r < np; r += kThreads / 32)
            for (int c = lane; c < ldq; c += 32)
                qsm[S.QA + r * ldq + c] = (r < n && c < n) ? Qg[(int64_t)r * n + c] : ((r == c && r >= n) ? 1.0 : 0.0);
        for (int r = warp; r < msp; r += kThreads / 32) {
            const double* src = nullptr;
            if (r < e) src = Ag + (int64_t)r * n;
            else if (r >= ep && r < ms) src = Gg + (int64_t)(r - ep) * n;
            for (int c = lane; c < ldq; c += 32) qsm[S.WA + r * ldq + c] = (src != nullptr && c < n) ? src[c] : 0.0;
        }
    }
    for (int i = tid; i < np; i += kThreads) qsm[S.aug + i] = 0.0;
    build_tile_table(reinterpret_cast<uint16_t*>(qsm + S.tab), np >> 3, tid);
    __syncthreads();
    if (D.reg > 0.0) {                                       // Q~ = Q + eps I (solve_kkt_ir, batch.py:247-249)
        for (int i = tid; i < n; i += kThreads) qsm[S.QA + i * ldq + i] += D.reg;
        __syncthreads();
    }
    QPB_TICK(34);   // staging
    // ---- 1. Q = L L^T
    f_chol(S.QA, ldq, np, 0, S.aug, S.tab);
    QPB_TICK(35);   // chol(Q)
    for (int i = tid; i < n; i += kThreads) {
        const double ri = qsm[S.QA + i * ldq + i];                   // reciprocal of L_ii; NaN/inf if a pivot failed
        if (!(ri > 0.0) || isinf(ri)) s_flag = 1;
    }
    // ---- 2. inverted diagonal blocks
    for (int blk = warp; blk < (np >> 3); blk += kThreads / 32) f_invert8(S.QA + (8 * blk) * ldq + 8 * blk, ldq);
    __syncthreads();
    QPB_TICK(36);   // T blocks
    // ---- 3. W = rows * L^-T, one warp per 8-row tile
    for (int rt = warp; rt < (msp >> 3); rt += kThreads / 32) f_rows_times_LinvT(S.QA, ldq, np, S.WA, ldq, rt);
    __syncthreads();
    QPB_TICK(37);   // W
    // ---- outputs L (packed lower, true diagonal) and W (compact ms x ldw)
    double* Lg = Lfac + (int64_t)sys * D.lp;
    double* Wg = Wfac + (int64_t)sys * ms * D.ldw;
    double* Kg = Kfac + (int64_t)sys * s_doubles(D, pf != 0);
    for (int r = warp; r < n; r += kThreads / 32)
        for (int c = lane; c < r; c += 32) Lg[(r * (r + 1)) / 2 + c] = qsm[S.QA + r * ldq + c];
    for (int r = tid; r < n; r += kThreads) Lg[(r * (r + 1)) / 2 + r] = 1.0 / qsm[S.QA + r * ldq + r];   // true diagonal
    if (tid == 0 && (D.lp > n * (n + 1) / 2)) Lg[D.lp - 1] = 0.0;
    for (int r = warp; r < ms; r += kThreads / 32)
        for (int c = lane; c < D.ldw; c += 32) Wg[r * D.ldw + c] = (c < n) ? qsm[S.WA + r * ldq + c] : 0.0;
    if (tid == 0) spd_flag[sys] = s_flag;
    __syncthreads();
    QPB_TICK(38);   // write L, W
    // ---- 4. K = W W^T (lower tiles), into the Q area with leading dimension lds
    {
        const int g = lane >> 2, q = lane & 3;
        const int nts = msp >> 3;
        const int T = nts * (nts + 1) / 2;
        const int lds = D.lds;
        for (int i = tid; i < msp * lds; i += kThreads) qsm[S.QA + i] = 0.0;      // (also clears the upper triangle)
        __syncthreads();
        for (int t = warp; t < T; t += kThreads / 32) {
            int ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while (ti * (ti + 1) / 2 > t) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
            const int tj = t - ti * (ti + 1) / 2;
            const double* pa = qsm + S.WA + (8 * ti + g) * ldq + q;
            const double* pb = qsm + S.WA + (8 * tj + g) * ldq + q;
            double c0 = 0.0, c1 = 0.0, d0 = 0.0, d1 = 0.0;                         // two accumulator chains
            for (int kk = 0; kk < np; kk += 8) {
                dmma884(c0, c1, pa[kk], pb[kk]);
                dmma884(d0, d1, pa[kk + 4], pb[kk + 4]);
            }
            const int rr = 8 * ti + g, cc = 8 * tj + 2 * q;
            double v0 = c0 + d0, v1 = c1 + d1;
            // dummy equality rows and pad rows: unit diagonal
            if (rr == cc && ((rr >= e && rr < ep) || rr >= ms)) v0 += 1.0;
            if (rr == cc + 1 && ((rr >= e && rr < ep) || rr >= ms)) v1 += 1.0;
            if (rr == cc && rr < e) v0 += D.reg;             // regularised variant: A Q~^-1 A^T + eps I
            if (rr == cc + 1 && rr < e) v1 += D.reg;
            if (cc <= rr) qsm[S.QA + rr * lds + cc] = v0;
            if (cc + 1 <= rr) qsm[S.QA + rr * lds + cc + 1] = v1;
        }
    }
    __syncthreads();
    QPB_TICK(39);   // K = W W^T
    if (ep > 0) {
        double* RA = qsm + S.QA;
        chol_partial(RA, D.lds, ms, 0, ep, nullptr, 0, 0, qsm + S.aug, nullptr, tid, kThreads);
        for (int i = tid; i < ms * D.lds; i += kThreads) {                         // DMMA tiles spill into the upper triangle
            const int r = i / D.lds, c = i - r * D.lds;
            if (c > r) RA[i] = 0.0;
        }
        __syncthreads();
        for (int i = tid; i < ep; i += kThreads) RA[i * D.lds + i] = 1.0 / RA[i * D.lds + i];   // reciprocal-diagonal convention
        __syncthreads();
    }
    QPB_TICK(45);   // partial chol of the equality block
    if (pf) {                                                   // equality columns -> product form, K -> staircase
        qpb::pf::pf_convert_cols(qsm + S.QA, D.lds, msp, ep >> 3, tid, kThreads);
        qpb::pf::pf_write_staircase(Kg, qsm + S.QA, D.lds, msp, msp, tid, kThreads);
    } else
    for (int i = tid; i < msp * D.lds; i += kThreads) Kg[i] = qsm[S.QA + i];
    QPB_TICK(46);   // write K
#ifdef QPB_TIMING
    if (tid == 0 && sys == 0) for (int i = 0; i < 128; ++i) g_tim[i] = s_tim[i];
#endif
}

}  // namespace
#include "qp_setup_pf.cuh"
namespace {

// ---------------------------------------------------------------------------------------------
// OptNet parameterisation either side of the path (example-cls-layer.ipynb:125-129; SURVEY 8f.3):
//   construct:  Q = tril(L) tril(L)^T + eps I,   h = G z0 + s0           (shared parameters: one system per batch)
//   chain:      dL = tril((dQ + dQ^T) tril(L)),  dG = dG_qp + dh z0^T,  dz0 = G^T dh,  ds0 = dh
// One launch each (n, m <= a few hundred: one thread per output element, rows of L / G read coalesced), instead of the
// eight torch kernels and their (n x n) temporaries on either side of every QPFunction call.
// ---------------------------------------------------------------------------------------------
__global__ void k_optnet_construct(int n, int m, const double* __restrict__ L, const double* __restrict__ G,
                                   const double* __restrict__ z0, const double* __restrict__ s0, double eps,
                                   double* __restrict__ Q, double* __restrict__ h) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < n * n) {
        const int r = idx / n, c = idx - r * n;
        const int kmax = r < c ? r : c;
        double acc = (r == c) ? eps : 0.0;
        for (int k = 0; k <= kmax; ++k) acc = fma(L[r * n + k], L[c * n + k], acc);
        Q[idx] = acc;
    } else if (idx < n * n + m) {
        const int i = idx - n * n;
        double acc = s0[i];
        for (int k = 0; k < n; ++k) acc = fma(G[i * n + k], z0[k], acc);
        h[i] = acc;
    }
}
__global__ void k_optnet_chain(int n, int m, const double* __restrict__ L, const double* __restrict__ G,
                               const double* __restrict__ z0, const double* __restrict__ dQ,
                               const double* __restrict__ dGq, const double* __restrict__ dh, double* __restrict__ dL,
                               double* __restrict__ dG, double* __restrict__ dz0, double* __restrict__ ds0) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < n * n) {
        const int r = idx / n, c = idx - r * n;
        double acc = 0.0;
        if (c <= r)                                          // dL[r][c] = sum_{k >= c} (dQ[r][k] + dQ[k][r]) L[k][c]
            for (int k = c; k < n; ++k) acc = fma(dQ[r * n + k] + dQ[k * n + r], L[k * n + c], acc);
        dL[idx] = acc;
    } else if (idx < n * n + m * n) {
        const int j = idx - n * n, i = j / n, c = j - i * n;
        dG[j] = dGq[j] + dh[i] * z0[c];
    } else if (idx < n * n + m * n + n) {
        const int c = idx - n * n - m * n;
        double acc = 0.0;
        for (int i = 0; i < m; ++i) acc = fma(G[i * n + c], dh[i], acc);
        dz0[c] = acc;
    } else if (idx < n * n + m * n + n + m) {
        const int i = idx - n * n - m * n - n;
        ds0[i] = dh[i];
    }
}

// fp64 FMA issue-rate probe: 8 independent DFMA chains per thread (roofline denominator for bench.py)
__global__ void k_dfma_probe(int iters, double* out) {
    double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5,
           a6 = a0 + 6, a7 = a0 + 7;
    const double m = 1.0000001, c = 1e-9;
    for (int i = 0; i < iters; ++i) {
        a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
        a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));
}

// ---------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------
thread_local char g_cuda_err[256] = "";

int cuda_fail(cudaError_t err, const char* what) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s", what, cudaGetErrorString(err));
    return QPB200_ERR_CUDA;
}
#define CK(call)                                          \
    do {                                                  \
        cudaError_t _e = (call);                          \
        if (_e != cudaSuccess) return cuda_fail(_e, #call); \
    } while (0)

KDims dims_of(const qpb200_plan* p) {
    KDims D;
    D.n = p->nz; D.m = p->nineq; D.e = p->neq; D.ep = p->neq_pad; D.ms = p->ms; D.msp = p->ms_pad;
    D.ldw = p->ldw; D.lds = p->lds; D.rows_s = p->rows_s; D.vl = p->vl;
    D.lp = (int)p->L_elems;
    D.reg = 0.0;
    return D;
}

// cudaFuncSetAttribute is not free (and may serialise with the driver): raise the dynamic shared-memory
// limit of a kernel only when it has to grow. Keyed by (device, kernel).
// The table is shared by every host thread that calls into the library (ctypes releases the GIL: the autograd engine
// thread runs backward while user threads run forward, one thread per GPU in multi-device processes), hence the lock.
struct SmemSet { const void* fn; int dev; size_t bytes; };
SmemSet g_smem_set[64];
int g_smem_n = 0;
std::mutex g_smem_mu;

template <typename K>
int set_smem(K kernel, size_t bytes) {
    int dev = 0;
    CK(cudaGetDevice(&dev));
    const void* fn = reinterpret_cast<const void*>(kernel);
    std::lock_guard<std::mutex> lock(g_smem_mu);
    for (int i = 0; i < g_smem_n; ++i)
        if (g_smem_set[i].fn == fn && g_smem_set[i].dev == dev) {
            if (g_smem_set[i].bytes >= bytes) return QPB200_OK;
            CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
            g_smem_set[i].bytes = bytes;
            return QPB200_OK;
        }
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    if (g_smem_n < 64) g_smem_set[g_smem_n++] = SmemSet{fn, dev, bytes};
    return QPB200_OK;
}

}  // namespace

// ---- the 192- and 512-thread builds of the product-form solve kernels (qp_alt.cu) ----------------------------------
extern "C" {
#define QPB_ALT_DECL(NT)                                                                                                  \
    int qpb200_alt##NT##_forward(const qpb200_plan*, size_t, int, const double*, int64_t, const double*, int64_t,          \
                                 const double*, int64_t, const double*, const double*, const double*, int, double, double, \
                                 double, int, int, double*, double*, double*, double*, int*, double*, double*, void*);     \
    int qpb200_alt##NT##_solve_kkt(const qpb200_plan*, size_t, int, const double*, const double*, const double*,           \
                                   const double*, const double*, const double*, const double*, const double*, int,         \
                                   double*, double*, double*, double*, void*);                                             \
    int qpb200_alt##NT##_backward(const qpb200_plan*, size_t, int, const double*, const double*, const double*,            \
                                  const double*, const double*, const double*, const double*, const double*,              \
                                  const double*, const double*, int, double*, int, double*, int, double*, int, double*,    \
                                  int, double*, int, double*, int, double*, double*, double*, void*);
QPB_ALT_DECL(192)
QPB_ALT_DECL(512)
int qpb200_alt192_setup(const qpb200_plan*, size_t, int, const double*, int64_t, const double*, int64_t, const double*,
                        int64_t, double, double*, double*, double*, int*, void*);
int qpb200_alt512_forward_res(const qpb200_plan*, size_t, int, const double*, int64_t, const double*, int64_t,
                              const double*, int64_t, const double*, const double*, const double*, int, double, double,
                              double, int, int, double*, double*, double*, double*, int*, double*, double*, void*);
#undef QPB_ALT_DECL
void qpb200_internal_cuda_error(int err, const char* what) { cuda_fail((cudaError_t)err, what); }
}

extern "C" {

int qpb200_version(void) { return 100; }

const char* qpb200_error_string(int code) {
    switch (code) {
        case QPB200_OK: return "ok";
        case QPB200_ERR_BAD_ARG: return "bad argument";
        case QPB200_ERR_NO_CONSTRAINTS: return "neq == 0 and nineq == 0";
        case QPB200_ERR_CUDA: return "CUDA runtime error";
        case QPB200_ERR_TOO_LARGE: return "problem too large";
        default: return "unknown error";
    }
}

const char* qpb200_last_cuda_error(void) { return g_cuda_err; }

// allow_tiny = false: the plan of the regularised mode, whose kernels exist in the product-form family only
static int plan_init_impl(int nz, int nineq, int neq, qpb200_plan* plan, bool allow_tiny) {
    if (plan == nullptr || nz <= 0 || nineq < 0 || neq < 0) return QPB200_ERR_BAD_ARG;
    if (nineq == 0 && neq == 0) return QPB200_ERR_NO_CONSTRAINTS;
    if (nz > 4096 || nineq > 4096 || neq > 4096) return QPB200_ERR_TOO_LARGE;
    memset(plan, 0, sizeof(*plan));
    plan->nz = nz; plan->nineq = nineq; plan->neq = neq;
    plan->neq_pad = (neq + 7) & ~7;
    plan->ms = plan->neq_pad + nineq;
    plan->ms_pad = (plan->ms + 7) & ~7;
    const int ms = plan->ms, msp = plan->ms_pad;
    plan->ldw = ld_for(nz);
    plan->lds = ld_for(msp);
    plan->rows_s = msp;
    plan->vl = (((nz > msp ? nz : msp) + 8) + 7) & ~7;
    plan->threads = kThreads;
    plan->L_elems = (((int64_t)nz * (nz + 1)) / 2 + 1) & ~(int64_t)1;   // packed lower, even count
    plan->W_elems = (int64_t)ms * plan->ldw;
    plan->K_elems = (int64_t)msp * plan->lds;
    const int ldn = ld_for(nz), ldk = ld_for(ms);
    const int64_t regA = (int64_t)nz * ldn > (int64_t)ms * ldk ? (int64_t)nz * ldn : (int64_t)ms * ldk;
    const int64_t setup_mat = regA + (int64_t)ms * ldn;
    const int64_t setup_vec = (nz > ms ? nz : ms) + 8;
    const int64_t solve_mat_s = (int64_t)ms * plan->ldw + (int64_t)plan->rows_s * plan->lds + plan->L_elems;
    const int64_t solve_mat = (int64_t)plan->rows_s * plan->lds;     // global mode: only the S workspace
    const int64_t solve_vec = (int64_t)solve_vec_doubles(plan->vl);
    KDims D = dims_of(plan);
    const int64_t fast_doubles = (int64_t)fk::fast_smem_doubles(D, false);
    const int64_t coop_doubles = (int64_t)fk::fast_smem_doubles(D, true);
    const bool setup_fits = (setup_mat + setup_vec) * 8 <= kMaxSmem;
    const bool fast_ok = setup_fits && fast_doubles * 8 <= kMaxSmem && nineq <= 8 * kCholMaxTiles && (msp - plan->neq_pad) / 8 >= 1 && msp <= 224;
    const bool fits = setup_fits && (solve_mat_s + solve_vec) * 8 <= kMaxSmem;
    const fk::SLayout SL = fk::setup_layout(D);
    const bool setup_fast_ok = fast_ok && nz <= 8 * kCholMaxTiles && (int64_t)SL.total * 8 <= kMaxSmem;
    // tiny problems (the sizes of the reference's own tests and prof scripts, test.py:99-187 nz = 10): a 256-thread
    // CTA per QP is 8 warps synchronising over a handful of rows; one warp per QP and 16 QPs per SM instead
    const bool tiny = allow_tiny && fits && nz <= kTinyMax && msp <= kTinyMax;
    plan->tiny = tiny ? 1 : 0;
    plan->pf = 0; plan->pf_global = 0; plan->pf_smem_bytes = 0; plan->pf2_ok = 0; plan->pf2_smem_bytes = 0; plan->pf_two = 0; plan->pf3_ok = 0; plan->pf3_smem_bytes = 0; plan->pf_three = 0; plan->pf_threads = 256; plan->setup_pf = 0; plan->setup_pf_smem_bytes = 0;
    if (tiny) {
        plan->fast = 0; plan->setup_fast = 0; plan->smem_resident = 1; plan->threads = kTinyThreads;
        plan->setup_smem_bytes = (setup_mat + setup_vec) * 8;
        plan->solve_smem_bytes = (solve_mat_s + solve_vec) * 8;
        plan->setup_scratch_elems = 0; plan->solve_scratch_elems = 0;
        plan->coop_smem_bytes = 0; plan->coop_ok = 0; plan->coop = 0;
        return QPB200_OK;
    }
    plan->fast = fast_ok ? 1 : 0;
    plan->setup_fast = setup_fast_ok ? 1 : 0;
    // co-resident mode: two CTAs per SM (each needs its share of the 227 KB plus the 1 KB the hardware reserves per
    // CTA), the packed L must fit the S workspace it visits, W rows must be 16-byte aligned (ld is even by construction)
    plan->coop_smem_bytes = coop_doubles * 8;
    plan->coop_ok = (fast_ok && coop_doubles * 8 <= (232448 / 2 - 1024 - 64) && plan->L_elems <= (int64_t)msp * plan->lds) ? 1 : 0;
    // opt-in only (QPB200_COOP): the co-resident kernels lost in A/B runs (the 128-register cap spills the
    // register-resident Cholesky, L2 passes cost 3x the shared-memory ones)
    plan->coop = 0;
    plan->smem_resident = (fast_ok || fits) ? 1 : 0;
    if (setup_fits && (fast_ok || fits)) {
        plan->setup_smem_bytes = setup_fast_ok ? (int64_t)SL.total * 8 : (setup_mat + setup_vec) * 8;
        plan->solve_smem_bytes = fast_ok ? fast_doubles * 8 : (solve_mat_s + solve_vec) * 8;
        plan->setup_scratch_elems = 0;
        plan->solve_scratch_elems = 0;
    } else {
        plan->setup_smem_bytes = setup_vec * 8;
        plan->solve_smem_bytes = solve_vec * 8;
        if (plan->solve_smem_bytes > kMaxSmem) return QPB200_ERR_TOO_LARGE;
        plan->setup_scratch_elems = setup_mat;
        plan->solve_scratch_elems = solve_mat;
    }
    // product-form kernels (qp_pf.cuh): factor in the staircase layout; W and chol(Q) in shared memory when they fit
    // next to it, else read from global memory ("large problem" kernel, e.g. nz = nineq = 200). One row per thread in the
    // substitutions: order <= 256.
    {
        const int64_t pf_res = (int64_t)fk::fast_smem_doubles(D, false, true) * 8;
        const int64_t pf_glb = (int64_t)fk::fast_smem_doubles(D, true, true) * 8;
        const bool shape_ok = msp <= kThreads && (msp - plan->neq_pad) / 8 >= 1;
        const bool res_ok = shape_ok && pf_res <= kMaxSmem, glb_ok = shape_ok && pf_glb <= kMaxSmem;
        // wherever they fit: never slower than the round-1 kernels in A/B runs at C2, C3 and C4
        const char* env = getenv("QPB200_PF");               // development / A-B knob: "0" never, "1" wherever possible,
        const bool want = !(env != nullptr && env[0] == '0'); // "2" = "1" + two QPs per SM (W, L from L2) where that fits
        // co-residency: every CTA also costs the 1 KB the hardware reserves, out of 228 KB per SM
        const bool two_ok = glb_ok && 2 * (pf_glb + 1024) <= 233472;
        const bool three_ok = glb_ok && 3 * (pf_glb + 1024) <= 233472 && msp <= 192;   // 192-thread CTAs: one row per thread
        const bool want_two = env != nullptr && env[0] == '2';
        const bool use = want && (res_ok || glb_ok);
        if (use) {
            plan->pf = 1;
            plan->pf_global = res_ok ? 0 : 1;
            plan->pf_smem_bytes = res_ok ? pf_res : pf_glb;
            plan->pf2_ok = two_ok ? 1 : 0;
            plan->pf2_smem_bytes = two_ok ? pf_glb : 0;
            plan->pf_two = (two_ok && want_two) ? 1 : 0;
            plan->pf3_ok = three_ok ? 1 : 0;
            plan->pf3_smem_bytes = three_ok ? pf_glb : 0;
            plan->pf_three = (three_ok && env != nullptr && env[0] == '3') ? 1 : 0;
            // large orders (nz = nineq = 200): 15 update warps instead of 7 (the factorization is update-bound there)
            const char* e512 = getenv("QPB200_NT512");
            plan->pf_threads = (plan->pf_global && msp > 128 && !(e512 != nullptr && e512[0] == '0')) ? 512 : 256;
            // experiment knob: "2" = also the RESIDENT forward kernel at 512 threads (backward / solve_kkt stay at 256)
            if (!plan->pf_global && e512 != nullptr && e512[0] == '2') plan->pf_threads = 512;
            // the 512-thread build keeps a wider reduction scratch (16 warps): its layout ends 64 doubles later
            if (plan->pf_threads == 512) {
                plan->pf_smem_bytes += 512;
                if (plan->pf_smem_bytes > kMaxSmem) { plan->pf_threads = 256; plan->pf_smem_bytes -= 512; }
            }
            plan->K_elems = (int64_t)qpb::pf::pf_elems(msp >> 3);
            plan->solve_scratch_elems = 0;                   // the factor lives in shared memory: no per-QP global workspace
            // pre_factor_kkt on the same machinery (k_setup_pf) whenever its shared memory fits. In throughput mode
            // (pf_three) pre_factor_impl runs its 192-thread build wherever it fits the three-per-SM slot; the choice
            // below is the latency-mode one: the 256-thread build is faster than the global-scratch setup at
            // nz = nineq = 200, but a lone CTA of it is slower than k_setup_fast at C2 - so it is the default only where
            // there is no fast setup or the problem is small (nz <= 64: it wins at C3)
            const int64_t spf = (int64_t)fk::setup_pf_layout(D).total * 8;
            const char* esp = getenv("QPB200_SETUP_PF");     // development / A-B knob: "0" never, "1" wherever it fits
            const bool want_spf = (esp != nullptr) ? (esp[0] == '1') : (!setup_fast_ok || nz <= 64);
            // (room for one more row tile of [A; G]: the shapes this choice has been measured on. Beyond them, e.g.
            // nz = 211, latency mode keeps the generic setup.)
            const bool spf_fits = spf + 64 * (int64_t)(((nz + 7) & ~7) + 4) <= kMaxSmem;
            plan->setup_pf = (spf_fits && want_spf) ? 1 : 0;
            plan->setup_pf_smem_bytes = spf;
            if (plan->setup_pf) plan->setup_scratch_elems = 0;
        }
    }
    return QPB200_OK;
}

int qpb200_plan_init(int nz, int nineq, int neq, qpb200_plan* plan) {
    return plan_init_impl(nz, nineq, neq, plan, true);
}

int qpb200_plan_init_reg(int nz, int nineq, int neq, qpb200_plan* plan) {
    const int rc = plan_init_impl(nz, nineq, neq, plan, false);
    if (rc != QPB200_OK) return rc;
    if (!plan->pf) return QPB200_ERR_TOO_LARGE;            // order ms_pad > 256, or no inequality rows
    if (plan->pf_threads == 512) plan->pf_smem_bytes -= 512;
    plan->pf_threads = 256;                                // one QP per SM, 256 threads: the only regularised build
    plan->pf2_ok = 0; plan->pf_two = 0; plan->pf2_smem_bytes = 0;
    plan->pf3_ok = 0; plan->pf_three = 0; plan->pf3_smem_bytes = 0;
    return QPB200_OK;
}

static int pre_factor_impl(const qpb200_plan* plan, int nsys, const double* Q, int64_t sQ,
                           const double* G, int64_t sG, const double* A, int64_t sA, double* Lfac,
                           double* Wfac, double* Kfac, int* spd_flag, double* scratch, void* stream, double reg);
int qpb200_pre_factor_kkt(const qpb200_plan* plan, int nsys, const double* Q, int64_t sQ,
                          const double* G, int64_t sG, const double* A, int64_t sA, double* Lfac,
                          double* Wfac, double* Kfac, int* spd_flag, double* scratch, void* stream) {
    return pre_factor_impl(plan, nsys, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac, spd_flag, scratch, stream, 0.0);
}
int qpb200_pre_factor_kkt_reg(const qpb200_plan* plan, int nsys, const double* Q, int64_t sQ,
                              const double* G, int64_t sG, const double* A, int64_t sA, double reg_eps, double* Lfac,
                              double* Wfac, double* Kfac, int* spd_flag, double* scratch, void* stream) {
    if (!(reg_eps >= 0.0)) return QPB200_ERR_BAD_ARG;
    return pre_factor_impl(plan, nsys, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac, spd_flag, scratch, stream, reg_eps);
}
static int pre_factor_impl(const qpb200_plan* plan, int nsys, const double* Q, int64_t sQ,
                           const double* G, int64_t sG, const double* A, int64_t sA, double* Lfac,
                           double* Wfac, double* Kfac, int* spd_flag, double* scratch, void* stream, double reg) {
    if (!plan || nsys <= 0 || !Q || !Lfac || !Wfac || !Kfac || !spd_flag) return QPB200_ERR_BAD_ARG;
    if (plan->nineq > 0 && !G) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && !A) return QPB200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = dims_of(plan);
    D.reg = reg;
    if (plan->tiny) {
        int rc = set_smem(k_setup<true, true>, plan->setup_smem_bytes);
        if (rc) return rc;
        k_setup<true, true><<<nsys, kTinyThreads, plan->setup_smem_bytes, st>>>(D, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac,
                                                                                 spd_flag, nullptr, 0, 0);
    } else if (plan->pf && plan->pf_three && plan->pf3_ok && plan->setup_pf_smem_bytes <= plan->pf3_smem_bytes) {
        // throughput mode: the setup CTA fits a three-per-SM slot like the forward / backward CTAs around it
        return qpb200_alt192_setup(plan, (size_t)plan->setup_pf_smem_bytes, nsys, Q, sQ, G, sG, A, sA, reg, Lfac, Wfac, Kfac,
                                   spd_flag, stream);
    } else if (plan->pf && plan->setup_pf) {
        int rc = set_smem(k_setup_pf<2>, plan->setup_pf_smem_bytes);
        if (rc) return rc;
        k_setup_pf<2><<<nsys, kThreads, plan->setup_pf_smem_bytes, st>>>(D, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac, spd_flag);
    } else if (plan->setup_fast) {
        int rc = set_smem(k_setup_fast, plan->setup_smem_bytes);
        if (rc) return rc;
        k_setup_fast<<<nsys, kThreads, plan->setup_smem_bytes, st>>>(D, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac, spd_flag, plan->pf);
    } else if (plan->smem_resident) {
        int rc = set_smem(k_setup<true>, plan->setup_smem_bytes);
        if (rc) return rc;
        k_setup<true><<<nsys, kThreads, plan->setup_smem_bytes, st>>>(D, Q, sQ, G, sG, A, sA, Lfac, Wfac,
                                                                    Kfac, spd_flag, nullptr, 0, plan->pf);
    } else {
        if (!scratch) return QPB200_ERR_BAD_ARG;
        int rc = set_smem(k_setup<false>, plan->setup_smem_bytes);
        if (rc) return rc;
        k_setup<false><<<nsys, kThreads, plan->setup_smem_bytes, st>>>(
            D, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac, spd_flag, scratch, plan->setup_scratch_elems, plan->pf);
    }
    CK(cudaGetLastError());
    return QPB200_OK;
}

int qpb200_forward(const qpb200_plan* plan, int nbatch, const double* p, int64_t sp, const double* h,
                   int64_t sh, const double* b, int64_t sb, const double* Lfac, const double* Wfac,
                   const double* Kfac, int sF, double eps, double stall_tol, double best_tie,
                   int notImprovedLim, int maxIter, double* zhat, double* lam, double* slacks, double* nus, int* iters,
                   double* best_resid, double* trace, double* scratch, void* stream) {
    if (!plan || nbatch <= 0 || !p || !Lfac || !Wfac || !Kfac || !zhat || !lam || !slacks || !iters ||
        !best_resid)
        return QPB200_ERR_BAD_ARG;
    if (plan->nineq > 0 && !h) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!b || !nus)) return QPB200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = dims_of(plan);
#define QPB_LAUNCH_FWD(KS, SCR, SCRN)                                                                   \
    do {                                                                                                \
        int rc = set_smem(k_forward<KS>, plan->solve_smem_bytes);                                       \
        if (rc) return rc;                                                                              \
        k_forward<KS><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(                                \
            D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim,     \
            maxIter, zhat, lam, slacks, nus, iters, best_resid, trace, SCR, SCRN);                      \
    } while (0)
    if (plan->tiny) {
        int rc = set_smem(k_forward<true, true>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_forward<true, true><<<nbatch, kTinyThreads, plan->solve_smem_bytes, st>>>(
            D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam,
            slacks, nus, iters, best_resid, trace, nullptr, 0);
    } else if (plan->pf) {
#define QPB_LAUNCH_PF(KG, K2)                                                                           \
        do {                                                                                            \
            const size_t sb_ = K2 ? plan->pf2_smem_bytes : plan->pf_smem_bytes;                         \
            int rc = set_smem(k_forward_fast<KG, true, K2>, sb_);                                       \
            if (rc) return rc;                                                                          \
            k_forward_fast<KG, true, K2><<<nbatch, qpb::fast::kNT, sb_, st>>>(                                \
                D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, \
                maxIter, zhat, lam, slacks, nus, iters, best_resid, trace);                             \
        } while (0)
        if (plan->pf_three && plan->pf3_ok)
            return qpb200_alt192_forward(plan, (size_t)plan->pf3_smem_bytes, nbatch, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps,
                                         stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam, slacks, nus, iters, best_resid,
                                         trace, stream);
        else if (plan->pf_two && plan->pf2_ok) QPB_LAUNCH_PF(true, 2);
        else if (plan->pf_global && plan->pf_threads == 512)
            return qpb200_alt512_forward(plan, (size_t)plan->pf_smem_bytes, nbatch, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps,
                                         stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam, slacks, nus, iters, best_resid,
                                         trace, stream);
        else if (plan->pf_global) QPB_LAUNCH_PF(true, 0);
        else if (plan->pf_threads == 512)                    // resident (latency) kernel at 512 threads: 15 update warps
            return qpb200_alt512_forward_res(plan, (size_t)plan->pf_smem_bytes, nbatch, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF,
                                             eps, stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam, slacks, nus, iters,
                                             best_resid, trace, stream);
        else QPB_LAUNCH_PF(false, 0);
#undef QPB_LAUNCH_PF
    } else if (plan->fast && plan->coop && plan->coop_ok) {
        int rc = set_smem(k_forward_fast<true>, plan->coop_smem_bytes);
        if (rc) return rc;
        k_forward_fast<true><<<nbatch, kThreads, plan->coop_smem_bytes, st>>>(
            D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter,
            zhat, lam, slacks, nus, iters, best_resid, trace);
    } else if (plan->fast) {
        int rc = set_smem(k_forward_fast<false>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_forward_fast<false><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(
            D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter,
            zhat, lam, slacks, nus, iters, best_resid, trace);
    } else if (plan->smem_resident) {
        QPB_LAUNCH_FWD(true, nullptr, 0);
    } else {
        if (!scratch) return QPB200_ERR_BAD_ARG;
        QPB_LAUNCH_FWD(false, scratch, plan->solve_scratch_elems);
    }
#undef QPB_LAUNCH_FWD
    CK(cudaGetLastError());
    return QPB200_OK;
}

static int solve_kkt_impl(const qpb200_plan* plan, int nbatch, const double* d, const double* rx,
                          const double* rs, const double* rz, const double* ry, const double* Lfac,
                          const double* Wfac, const double* Kfac, int sF, double* dx, double* ds,
                          double* dz, double* dy, double* scratch, void* stream, double reg);
int qpb200_solve_kkt(const qpb200_plan* plan, int nbatch, const double* d, const double* rx,
                     const double* rs, const double* rz, const double* ry, const double* Lfac,
                     const double* Wfac, const double* Kfac, int sF, double* dx, double* ds,
                     double* dz, double* dy, double* scratch, void* stream) {
    return solve_kkt_impl(plan, nbatch, d, rx, rs, rz, ry, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, scratch, stream, 0.0);
}
int qpb200_solve_kkt_reg(const qpb200_plan* plan, int nbatch, const double* d, const double* rx,
                         const double* rs, const double* rz, const double* ry, double reg_eps, const double* Lfac,
                         const double* Wfac, const double* Kfac, int sF, double* dx, double* ds,
                         double* dz, double* dy, double* scratch, void* stream) {
    if (!plan || !(reg_eps >= 0.0)) return QPB200_ERR_BAD_ARG;
    qpb200_plan p256 = *plan;            // the regularised variant exists in the 256-thread builds only
    p256.pf_three = 0;
    p256.pf_threads = 256;
    return solve_kkt_impl(&p256, nbatch, d, rx, rs, rz, ry, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, scratch, stream, reg_eps);
}
static int solve_kkt_impl(const qpb200_plan* plan, int nbatch, const double* d, const double* rx,
                          const double* rs, const double* rz, const double* ry, const double* Lfac,
                          const double* Wfac, const double* Kfac, int sF, double* dx, double* ds,
                          double* dz, double* dy, double* scratch, void* stream, double reg) {
    if (!plan || nbatch <= 0 || !d || !rx || !rs || !rz || !Lfac || !Wfac || !Kfac || !dx || !ds || !dz)
        return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!ry || !dy)) return QPB200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = dims_of(plan);
    D.reg = reg;
    BwdOut O;
    memset(&O, 0, sizeof(O));
#define QPB_LAUNCH_KKT(KS, SCR, SCRN)                                                                   \
    do {                                                                                                \
        int rc = set_smem(k_solve_kkt<KS, false>, plan->solve_smem_bytes);                              \
        if (rc) return rc;                                                                              \
        k_solve_kkt<KS, false><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(                       \
            D, d, rx, rs, rz, ry, nullptr, nullptr, nullptr, nullptr, Lfac, Wfac, Kfac, sF, dx, ds, dz, \
            dy, O, SCR, SCRN);                                                                          \
    } while (0)
    if (plan->tiny) {
        int rc = set_smem(k_solve_kkt<true, false, true>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_solve_kkt<true, false, true><<<nbatch, kTinyThreads, plan->solve_smem_bytes, st>>>(
            D, d, rx, rs, rz, ry, nullptr, nullptr, nullptr, nullptr, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, O, nullptr, 0);
    } else if (plan->pf) {
#define QPB_LAUNCH_PF(KG, K2)                                                                           \
        do {                                                                                            \
            const size_t sb_ = K2 ? plan->pf2_smem_bytes : plan->pf_smem_bytes;                         \
            int rc = set_smem(k_kkt_fast<false, KG, true, K2>, sb_);                                    \
            if (rc) return rc;                                                                          \
            k_kkt_fast<false, KG, true, K2><<<nbatch, qpb::fast::kNT, sb_, st>>>(                             \
                D, d, rx, rs, rz, ry, nullptr, nullptr, nullptr, nullptr, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, O); \
        } while (0)
        if (plan->pf_three && plan->pf3_ok)
            return qpb200_alt192_solve_kkt(plan, (size_t)plan->pf3_smem_bytes, nbatch, d, rx, rs, rz, ry, Lfac, Wfac, Kfac, sF, dx, ds,
                                           dz, dy, stream);
        else if (plan->pf_two && plan->pf2_ok) QPB_LAUNCH_PF(true, 2);
        else if (plan->pf_global && plan->pf_threads == 512)
            return qpb200_alt512_solve_kkt(plan, (size_t)plan->pf_smem_bytes, nbatch, d, rx, rs, rz, ry, Lfac, Wfac, Kfac, sF, dx, ds,
                                           dz, dy, stream);
        else if (plan->pf_global) QPB_LAUNCH_PF(true, 0);
        else QPB_LAUNCH_PF(false, 0);
#undef QPB_LAUNCH_PF
    } else if (plan->fast && plan->coop && plan->coop_ok) {
        int rc = set_smem(k_kkt_fast<false, true>, plan->coop_smem_bytes);
        if (rc) return rc;
        k_kkt_fast<false, true><<<nbatch, kThreads, plan->coop_smem_bytes, st>>>(
            D, d, rx, rs, rz, ry, nullptr, nullptr, nullptr, nullptr, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, O);
    } else if (plan->fast) {
        int rc = set_smem(k_kkt_fast<false, false>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_kkt_fast<false, false><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(
            D, d, rx, rs, rz, ry, nullptr, nullptr, nullptr, nullptr, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, O);
    } else if (plan->smem_resident) {
        QPB_LAUNCH_KKT(true, nullptr, 0);
    } else {
        if (!scratch) return QPB200_ERR_BAD_ARG;
        QPB_LAUNCH_KKT(false, scratch, plan->solve_scratch_elems);
    }
#undef QPB_LAUNCH_KKT
    CK(cudaGetLastError());
    return QPB200_OK;
}

static int launch_means(int nbatch, int n, int m, int e, const double* zhat, const double* lam, const double* nus,
                        double* dQ, int mean_Q, double* dp, int mean_p, double* dG, int mean_G, double* dh, int mean_h,
                        double* dA, int mean_A, double* db, int mean_b, const double* dxv, const double* dlamv,
                        const double* dnuv, cudaStream_t st);
int qpb200_backward(const qpb200_plan* plan, int nbatch, const double* dl_dzhat, const double* zhat,
                    const double* lam, const double* slacks, const double* nus, const double* Lfac,
                    const double* Wfac, const double* Kfac, int sF, double* dQ, int mean_Q, double* dp,
                    int mean_p, double* dG, int mean_G, double* dh, int mean_h, double* dA, int mean_A,
                    double* db, int mean_b, double* dxv, double* dlamv, double* dnuv, double* scratch,
                    void* stream) {
    return qpb200_backward_duals(plan, nbatch, dl_dzhat, nullptr, nullptr, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF,
                                 dQ, mean_Q, dp, mean_p, dG, mean_G, dh, mean_h, dA, mean_A, db, mean_b, dxv, dlamv, dnuv,
                                 scratch, stream);
}

// dl_dlam / dl_dnu (either may be NULL: zero) go into the rz / ry slots of the backward solve:
//   [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dlam dnu] = -[dl_dzhat; 0; dl_dlam; dl_dnu]
static int check_dual_adjoints(const qpb200_plan* plan, const double* dl_dnu) {
    return (dl_dnu != nullptr && plan->neq == 0) ? QPB200_ERR_BAD_ARG : QPB200_OK;
}

int qpb200_backward_duals(const qpb200_plan* plan, int nbatch, const double* dl_dzhat, const double* dl_dlam,
                          const double* dl_dnu, const double* zhat, const double* lam, const double* slacks,
                          const double* nus, const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                          double* dQ, int mean_Q, double* dp, int mean_p, double* dG, int mean_G, double* dh, int mean_h,
                          double* dA, int mean_A, double* db, int mean_b, double* dxv, double* dlamv, double* dnuv,
                          double* scratch, void* stream) {
    if (!plan || nbatch <= 0 || !dl_dzhat || !zhat || !lam || !slacks || !Lfac || !Wfac || !Kfac ||
        !dxv || !dlamv)
        return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!nus || !dnuv)) return QPB200_ERR_BAD_ARG;
    if (check_dual_adjoints(plan, dl_dnu)) return QPB200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = dims_of(plan);
    const int n = plan->nz, m = plan->nineq, e = plan->neq;
    BwdOut O;
    O.dQ = dQ; O.dp = dp; O.dG = dG; O.dh = dh; O.dA = dA; O.db = db;
    O.mQ = mean_Q; O.mp = mean_p; O.mG = mean_G; O.mh = mean_h; O.mA = mean_A; O.mb = mean_b;
#define QPB_LAUNCH_BWD(KS, SCR, SCRN)                                                                   \
    do {                                                                                                \
        int rc = set_smem(k_solve_kkt<KS, true>, plan->solve_smem_bytes);                               \
        if (rc) return rc;                                                                              \
        k_solve_kkt<KS, true><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(                        \
            D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac,  \
            sF, dxv, nullptr, dlamv, dnuv, O, SCR, SCRN);                                               \
    } while (0)
    if (plan->tiny) {
        int rc = set_smem(k_solve_kkt<true, true, true>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_solve_kkt<true, true, true><<<nbatch, kTinyThreads, plan->solve_smem_bytes, st>>>(
            D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv, nullptr,
            dlamv, dnuv, O, nullptr, 0);
    } else if (plan->pf) {
#define QPB_LAUNCH_PF(KG, K2)                                                                           \
        do {                                                                                            \
            const size_t sb_ = K2 ? plan->pf2_smem_bytes : plan->pf_smem_bytes;                         \
            int rc = set_smem(k_kkt_fast<true, KG, true, K2>, sb_);                                     \
            if (rc) return rc;                                                                          \
            k_kkt_fast<true, KG, true, K2><<<nbatch, qpb::fast::kNT, sb_, st>>>(                              \
                D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv, \
                nullptr, dlamv, dnuv, O);                                                               \
        } while (0)
        if (plan->pf_three && plan->pf3_ok) {
            int rc = qpb200_alt192_backward(plan, (size_t)plan->pf3_smem_bytes, nbatch, dl_dzhat, dl_dlam, dl_dnu, zhat, lam,
                                            slacks, nus, Lfac, Wfac, Kfac, sF, dQ, mean_Q, dp, mean_p, dG, mean_G, dh,
                                            mean_h, dA, mean_A, db, mean_b, dxv, dlamv, dnuv, stream);
            if (rc) return rc;
        } else if (plan->pf_two && plan->pf2_ok) QPB_LAUNCH_PF(true, 2);
        else if (plan->pf_global && plan->pf_threads == 512) {
            int rc = qpb200_alt512_backward(plan, (size_t)plan->pf_smem_bytes, nbatch, dl_dzhat, dl_dlam, dl_dnu, zhat, lam,
                                            slacks, nus, Lfac, Wfac, Kfac, sF, dQ, mean_Q, dp, mean_p, dG, mean_G, dh,
                                            mean_h, dA, mean_A, db, mean_b, dxv, dlamv, dnuv, stream);
            if (rc) return rc;
        } else if (plan->pf_global) QPB_LAUNCH_PF(true, 0);
        else QPB_LAUNCH_PF(false, 0);
#undef QPB_LAUNCH_PF
    } else if (plan->fast && plan->coop && plan->coop_ok) {
        int rc = set_smem(k_kkt_fast<true, true>, plan->coop_smem_bytes);
        if (rc) return rc;
        k_kkt_fast<true, true><<<nbatch, kThreads, plan->coop_smem_bytes, st>>>(
            D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv,
            nullptr, dlamv, dnuv, O);
    } else if (plan->fast) {
        int rc = set_smem(k_kkt_fast<true, false>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_kkt_fast<true, false><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(
            D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv,
            nullptr, dlamv, dnuv, O);
    } else if (plan->smem_resident) {
        QPB_LAUNCH_BWD(true, nullptr, 0);
    } else {
        if (!scratch) return QPB200_ERR_BAD_ARG;
        QPB_LAUNCH_BWD(false, scratch, plan->solve_scratch_elems);
    }
#undef QPB_LAUNCH_BWD
    CK(cudaGetLastError());
    return launch_means(nbatch, n, m, e, zhat, lam, nus, dQ, mean_Q, dp, mean_p, dG, mean_G, dh, mean_h, dA, mean_A, db,
                        mean_b, dxv, dlamv, dnuv, st);
}

// Batch-mean gradients of the un-batched inputs (qp.py:159-177) from the per-QP dx, dlam, dnu of a backward kernel.
static int launch_means(int nbatch, int n, int m, int e, const double* zhat, const double* lam, const double* nus,
                        double* dQ, int mean_Q, double* dp, int mean_p, double* dG, int mean_G, double* dh, int mean_h,
                        double* dA, int mean_A, double* db, int mean_b, const double* dxv, const double* dlamv,
                        const double* dnuv, cudaStream_t st) {
    const int TB = 256;
    if (dQ && mean_Q)
        k_mean_outer<<<dim3((n + kMoC - 1) / kMoC, (n + kMoR - 1) / kMoR), 256, 0, st>>>(nbatch, n, n, dxv, zhat, zhat, dxv, 0.5, dQ);
    if (dp && mean_p) k_mean_vec<<<(n + TB - 1) / TB, TB, 0, st>>>(nbatch, n, dxv, 1.0, dp);
    if (dG && mean_G)
        k_mean_outer<<<dim3((n + kMoC - 1) / kMoC, (m + kMoR - 1) / kMoR), 256, 0, st>>>(nbatch, m, n, dlamv, zhat, lam, dxv, 1.0, dG);
    if (dh && mean_h) k_mean_vec<<<(m + TB - 1) / TB, TB, 0, st>>>(nbatch, m, dlamv, -1.0, dh);
    if (e > 0) {
        if (dA && mean_A)
            k_mean_outer<<<dim3((n + kMoC - 1) / kMoC, (e + kMoR - 1) / kMoR), 256, 0, st>>>(nbatch, e, n, dnuv, zhat, nus, dxv, 1.0, dA);
        if (db && mean_b) k_mean_vec<<<(e + TB - 1) / TB, TB, 0, st>>>(nbatch, e, dnuv, -1.0, db);
    }
    CK(cudaGetLastError());
    return QPB200_OK;
}

// ---- regularised mode (QPFunction kkt_solver=IR_UNOPT): the solve kernels with kReg ---------------------------------
// Two families: the product-form kernels (a plan from qpb200_plan_init_reg) and, for the larger shapes, the generic
// global-scratch kernels (a plan from qpb200_plan_init with tiny = pf = smem_resident = 0), which need `scratch`.
static bool reg_global_plan(const qpb200_plan* plan) { return !plan->tiny && !plan->pf && !plan->smem_resident; }

static int check_reg_plan(const qpb200_plan* plan, double reg_eps, int ir_steps, const double* scratch) {
    if (!(reg_eps >= 0.0) || ir_steps < 0 || ir_steps > 8) return QPB200_ERR_BAD_ARG;
    if (reg_global_plan(plan)) return scratch ? QPB200_OK : QPB200_ERR_BAD_ARG;
    if (plan->tiny || !plan->pf || plan->pf_two || plan->pf_three || plan->pf_threads != 256) return QPB200_ERR_TOO_LARGE;
    return QPB200_OK;
}

int qpb200_forward_reg(const qpb200_plan* plan, int nbatch, const double* p, int64_t sp, const double* h,
                       int64_t sh, const double* b, int64_t sb, const double* Lfac, const double* Wfac,
                       const double* Kfac, int sF, double eps, double stall_tol, double best_tie,
                       int notImprovedLim, int maxIter, double reg_eps, int ir_steps, double* zhat, double* lam,
                       double* slacks, double* nus, int* iters, double* best_resid, double* trace, double* scratch,
                       void* stream) {
    if (!plan || nbatch <= 0 || !p || !h || !Lfac || !Wfac || !Kfac || !zhat || !lam || !slacks || !iters || !best_resid)
        return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!b || !nus)) return QPB200_ERR_BAD_ARG;
    int rc = check_reg_plan(plan, reg_eps, ir_steps, scratch);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = dims_of(plan);
    D.reg = reg_eps;
    if (reg_global_plan(plan)) {
        rc = set_smem(k_forward<false, false, true>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_forward<false, false, true><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(
            D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam,
            slacks, nus, iters, best_resid, trace, scratch, plan->solve_scratch_elems, ir_steps);
        CK(cudaGetLastError());
        return QPB200_OK;
    }
    const size_t sb_ = (size_t)plan->pf_smem_bytes;
#define QPB_LAUNCH_REG(KG)                                                                                   \
    do {                                                                                                     \
        rc = set_smem(k_forward_fast<KG, true, 0, true>, sb_);                                               \
        if (rc) return rc;                                                                                   \
        k_forward_fast<KG, true, 0, true><<<nbatch, qpb::fast::kNT, sb_, st>>>(                              \
            D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter, \
            zhat, lam, slacks, nus, iters, best_resid, trace, ir_steps);                                     \
    } while (0)
    if (plan->pf_global) QPB_LAUNCH_REG(true);
    else QPB_LAUNCH_REG(false);
#undef QPB_LAUNCH_REG
    CK(cudaGetLastError());
    return QPB200_OK;
}

int qpb200_backward_reg(const qpb200_plan* plan, int nbatch, const double* dl_dzhat, const double* zhat,
                        const double* lam, const double* slacks, const double* nus, const double* Lfac,
                        const double* Wfac, const double* Kfac, int sF, double reg_eps, int ir_steps, double* dQ,
                        int mean_Q, double* dp, int mean_p, double* dG, int mean_G, double* dh, int mean_h, double* dA,
                        int mean_A, double* db, int mean_b, double* dxv, double* dlamv, double* dnuv, double* scratch,
                        void* stream) {
    return qpb200_backward_reg_duals(plan, nbatch, dl_dzhat, nullptr, nullptr, zhat, lam, slacks, nus, Lfac, Wfac, Kfac,
                                     sF, reg_eps, ir_steps, dQ, mean_Q, dp, mean_p, dG, mean_G, dh, mean_h, dA, mean_A, db,
                                     mean_b, dxv, dlamv, dnuv, scratch, stream);
}

int qpb200_backward_reg_duals(const qpb200_plan* plan, int nbatch, const double* dl_dzhat, const double* dl_dlam,
                              const double* dl_dnu, const double* zhat, const double* lam, const double* slacks,
                              const double* nus, const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                              double reg_eps, int ir_steps, double* dQ, int mean_Q, double* dp, int mean_p, double* dG,
                              int mean_G, double* dh, int mean_h, double* dA, int mean_A, double* db, int mean_b,
                              double* dxv, double* dlamv, double* dnuv, double* scratch, void* stream) {
    if (!plan || nbatch <= 0 || !dl_dzhat || !zhat || !lam || !slacks || !Lfac || !Wfac || !Kfac || !dxv || !dlamv)
        return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!nus || !dnuv)) return QPB200_ERR_BAD_ARG;
    if (check_dual_adjoints(plan, dl_dnu)) return QPB200_ERR_BAD_ARG;
    int rc = check_reg_plan(plan, reg_eps, ir_steps, scratch);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = dims_of(plan);
    D.reg = reg_eps;
    BwdOut O;
    O.dQ = dQ; O.dp = dp; O.dG = dG; O.dh = dh; O.dA = dA; O.db = db;
    O.mQ = mean_Q; O.mp = mean_p; O.mG = mean_G; O.mh = mean_h; O.mA = mean_A; O.mb = mean_b;
    if (reg_global_plan(plan)) {
        rc = set_smem(k_solve_kkt<false, true, false, true>, plan->solve_smem_bytes);
        if (rc) return rc;
        k_solve_kkt<false, true, false, true><<<nbatch, kThreads, plan->solve_smem_bytes, st>>>(
            D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv, nullptr,
            dlamv, dnuv, O, scratch, plan->solve_scratch_elems, ir_steps);
        CK(cudaGetLastError());
        return launch_means(nbatch, plan->nz, plan->nineq, plan->neq, zhat, lam, nus, dQ, mean_Q, dp, mean_p, dG, mean_G,
                            dh, mean_h, dA, mean_A, db, mean_b, dxv, dlamv, dnuv, st);
    }
    const size_t sb_ = (size_t)plan->pf_smem_bytes;
#define QPB_LAUNCH_REG(KG)                                                                                   \
    do {                                                                                                     \
        rc = set_smem(k_kkt_fast<true, KG, true, 0, true>, sb_);                                             \
        if (rc) return rc;                                                                                   \
        k_kkt_fast<true, KG, true, 0, true><<<nbatch, qpb::fast::kNT, sb_, st>>>(                            \
            D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv, \
            nullptr, dlamv, dnuv, O, ir_steps);                                                              \
    } while (0)
    if (plan->pf_global) QPB_LAUNCH_REG(true);
    else QPB_LAUNCH_REG(false);
#undef QPB_LAUNCH_REG
    CK(cudaGetLastError());
    return launch_means(nbatch, plan->nz, plan->nineq, plan->neq, zhat, lam, nus, dQ, mean_Q, dp, mean_p, dG, mean_G, dh,
                        mean_h, dA, mean_A, db, mean_b, dxv, dlamv, dnuv, st);
}

#ifdef QPB_TIMING
int qpb200_debug_timing(long long* host64, int reset) {
    if (reset) {                          // 1: clear the slots; 2 + qp: clear and export QP `qp`'s slots from now on
        long long z[128] = {0};
        CK(cudaMemcpyToSymbol(qpb::fast::g_tim, z, sizeof(z)));
        const int target = reset >= 2 ? reset - 2 : 0;
        CK(cudaMemcpyToSymbol(qpb::fast::g_tim_target, &target, sizeof(int)));
        return QPB200_OK;
    }
    CK(cudaMemcpyFromSymbol(host64, qpb::fast::g_tim, 128 * sizeof(long long)));
    return QPB200_OK;
}
int qpb200_debug_cta(long long* host64, int nqp) {    // {t0_ns, t1_ns, iters, smid} per QP of the last forward launch
    CK(cudaMemcpyFromSymbol(host64, qpb::fast::g_cta, (size_t)4 * nqp * sizeof(long long)));
    return QPB200_OK;
}
#endif

int qpb200_dfma_probe(int blocks, int threads, int iters, double* out, void* stream) {
    if (blocks <= 0 || threads <= 0 || iters <= 0 || !out) return QPB200_ERR_BAD_ARG;
    k_dfma_probe<<<blocks, threads, 0, (cudaStream_t)stream>>>(iters, out);
    CK(cudaGetLastError());
    return QPB200_OK;
}

// Device resources of one qpb200_qp_host call: released on every exit path.
namespace {
struct HostCallGuard {
    cudaStream_t st = nullptr;
    double* arena = nullptr;
    int* iarena = nullptr;
    ~HostCallGuard() {
        if (arena) cudaFree(arena);
        if (iarena) cudaFree(iarena);
        if (st) cudaStreamDestroy(st);
    }
};
}  // namespace

int qpb200_qp_host(int device, int nbatch, int nz, int nineq, int neq, const double* Q_host,
                   const double* p_host, const double* G_host, const double* h_host,
                   const double* A_host, const double* b_host, const double* dl_host, double eps,
                   int notImprovedLim, int maxIter, double* zhat_host, double* dQ_host,
                   double* dp_host, double* dG_host, double* dh_host, double* dA_host, double* db_host,
                   int* spd_flag_host) {
    qpb200_plan P;
    int rc = qpb200_plan_init(nz, nineq, neq, &P);
    if (rc) return rc;
    if (nbatch <= 0 || !Q_host || !p_host || !zhat_host) return QPB200_ERR_BAD_ARG;
    if (nineq <= 0 || !G_host || !h_host) return QPB200_ERR_BAD_ARG;      // (equality-only problems: not supported, as in QPFunction)
    if (neq > 0 && (!A_host || !b_host)) return QPB200_ERR_BAD_ARG;
    CK(cudaSetDevice(device));
    HostCallGuard R;
    CK(cudaStreamCreate(&R.st));
    cudaStream_t st = R.st;
    const int64_t B = nbatch, n = nz, m = nineq, e = neq;
    const bool bwd = dl_host != nullptr;
    // one arena: inputs | factors | outputs | work
    const int64_t nin = B * (n * n + n + m * n + m + e * n + e + (bwd ? n : 0));
    const int64_t nfac = B * (P.L_elems + P.W_elems + P.K_elems);
    const int64_t nout = B * (n + 2 * m + e) + B /*resid*/;
    const int64_t ngrad = bwd ? B * (n * n + n + m * n + m + e * n + e + n + m + e) : 0;
    const int64_t nscr = B * (P.solve_scratch_elems > P.setup_scratch_elems ? P.solve_scratch_elems
                                                                             : P.setup_scratch_elems);
    CK(cudaMalloc(&R.arena, (size_t)(nin + nfac + nout + ngrad + nscr + 8) * sizeof(double)));
    CK(cudaMalloc(&R.iarena, (size_t)(2 * B) * sizeof(int)));
    double* q = R.arena;
    double* dQm = q; q += B * n * n;
    double* dpv = q; q += B * n;
    double* dGm = q; q += B * m * n;
    double* dhv = q; q += B * m;
    double* dAm = q; q += B * e * n;
    double* dbv = q; q += B * e;
    double* ddl = q; q += bwd ? B * n : 0;
    double* Lf = q; q += B * P.L_elems;
    double* Wf = q; q += B * P.W_elems;
    double* Kf = q; q += B * P.K_elems;
    double* dz = q; q += B * n;
    double* dlam = q; q += B * m;
    double* dsl = q; q += B * m;
    double* dnu = q; q += B * e;
    double* dres = q; q += B;
    double *gQ = nullptr, *gp = nullptr, *gG = nullptr, *gh = nullptr, *gA = nullptr, *gb = nullptr,
           *wx = nullptr, *wl = nullptr, *wn = nullptr;
    if (bwd) {
        gQ = q; q += B * n * n; gp = q; q += B * n; gG = q; q += B * m * n; gh = q; q += B * m;
        gA = q; q += B * e * n; gb = q; q += B * e; wx = q; q += B * n; wl = q; q += B * m; wn = q; q += B * e;
    }
    double* scr = nscr ? q : nullptr;
    int* dflag = R.iarena;
    int* diters = R.iarena + B;
#define H2D(dst, src, cnt) if ((cnt) > 0) CK(cudaMemcpyAsync(dst, src, (size_t)(cnt) * sizeof(double), cudaMemcpyHostToDevice, st))
#define D2H(dst, src, cnt) if ((cnt) > 0 && (dst)) CK(cudaMemcpyAsync(dst, src, (size_t)(cnt) * sizeof(double), cudaMemcpyDeviceToHost, st))
    H2D(dQm, Q_host, B * n * n); H2D(dpv, p_host, B * n); H2D(dGm, G_host, B * m * n);
    H2D(dhv, h_host, B * m); H2D(dAm, A_host, B * e * n); H2D(dbv, b_host, B * e);
    if (bwd) H2D(ddl, dl_host, B * n);
    rc = qpb200_pre_factor_kkt(&P, nbatch, dQm, n * n, dGm, m * n, dAm, e * n, Lf, Wf, Kf, dflag, scr, st);
    if (!rc)
        rc = qpb200_forward(&P, nbatch, dpv, n, dhv, m, dbv, e, Lf, Wf, Kf, 1, eps, 1e-6, 1.5, notImprovedLim, maxIter,
                            dz, dlam, dsl, e > 0 ? dnu : nullptr, diters, dres, nullptr, scr, st);
    if (!rc && bwd)
        rc = qpb200_backward(&P, nbatch, ddl, dz, dlam, dsl, e > 0 ? dnu : nullptr, Lf, Wf, Kf, 1, gQ, 0, gp,
                             0, gG, 0, gh, 0, e > 0 ? gA : nullptr, 0, e > 0 ? gb : nullptr, 0, wx, wl,
                             e > 0 ? wn : nullptr, scr, st);
    if (!rc) {
        D2H(zhat_host, dz, B * n);
        if (bwd) {
            D2H(dQ_host, gQ, B * n * n); D2H(dp_host, gp, B * n); D2H(dG_host, gG, B * m * n);
            D2H(dh_host, gh, B * m); D2H(dA_host, gA, B * e * n); D2H(db_host, gb, B * e);
        }
        if (spd_flag_host)
            CK(cudaMemcpyAsync(spd_flag_host, dflag, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    // the stream is drained on every path before the guard frees what the queued work uses
    cudaError_t err = cudaStreamSynchronize(st);
    if (!rc && err != cudaSuccess) rc = cuda_fail(err, "cudaStreamSynchronize");
#undef H2D
#undef D2H
    return rc;
}

// Symmetric matrices (Q, and the gradient dQ = 1/2 (dx z^T + z dx^T), qp.py:157-158) cross PCIe as their lower
// triangle only: `band`-row strips, strip b = rows [b band, (b+1) band) x columns [0, (b+1) band) of every matrix of the
// batch, one strided 3-D copy per strip (cudaMemcpy3DAsync; the copy engine walks the pitch). 100 x 100, band 20:
// 60 % of the bytes. The strictly upper part of the destination (beyond the strips) is left untouched; none of the
// kernels reads it (Cholesky of Q works on the lower triangle). direction: 0 = host -> device, 1 = device -> host.
int qpb200_copy_lower(const double* src, double* dst, int nbatch, int n, int band, int direction, void* stream) {
    if (!src || !dst || nbatch <= 0 || n <= 0 || band <= 0) return QPB200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    for (int r0 = 0; r0 < n; r0 += band) {
        const int r1 = (r0 + band < n) ? r0 + band : n;
        cudaMemcpy3DParms p;
        memset(&p, 0, sizeof(p));
        p.srcPtr = make_cudaPitchedPtr((void*)src, (size_t)n * 8, (size_t)n * 8, (size_t)n);
        p.dstPtr = make_cudaPitchedPtr((void*)dst, (size_t)n * 8, (size_t)n * 8, (size_t)n);
        p.srcPos = make_cudaPos(0, (size_t)r0, 0);
        p.dstPos = make_cudaPos(0, (size_t)r0, 0);
        p.extent = make_cudaExtent((size_t)r1 * 8, (size_t)(r1 - r0), (size_t)nbatch);
        p.kind = direction ? cudaMemcpyDeviceToHost : cudaMemcpyHostToDevice;
        CK(cudaMemcpy3DAsync(&p, st));
    }
    return QPB200_OK;
}

int qpb200_optnet_construct(int nz, int nineq, const double* L, const double* G, const double* z0, const double* s0,
                            double eps, double* Q, double* h, void* stream) {
    if (nz <= 0 || nineq <= 0 || !L || !G || !z0 || !s0 || !Q || !h) return QPB200_ERR_BAD_ARG;
    const int total = nz * nz + nineq, TB = 128;
    k_optnet_construct<<<(total + TB - 1) / TB, TB, 0, (cudaStream_t)stream>>>(nz, nineq, L, G, z0, s0, eps, Q, h);
    CK(cudaGetLastError());
    return QPB200_OK;
}

int qpb200_optnet_chain(int nz, int nineq, const double* L, const double* G, const double* z0, const double* dQ,
                        const double* dG_qp, const double* dh, double* dL, double* dG, double* dz0, double* ds0,
                        void* stream) {
    if (nz <= 0 || nineq <= 0 || !L || !G || !z0 || !dQ || !dG_qp || !dh || !dL || !dG || !dz0 || !ds0) return QPB200_ERR_BAD_ARG;
    const int total = nz * nz + nineq * nz + nz + nineq, TB = 128;
    k_optnet_chain<<<(total + TB - 1) / TB, TB, 0, (cudaStream_t)stream>>>(nz, nineq, L, G, z0, dQ, dG_qp, dh, dL, dG, dz0, ds0);
    CK(cudaGetLastError());
    return QPB200_OK;
}

}  // extern "C"
