// qp_boxq.cu - BoxQPFunction(dense_Q=True): simple bounds with a DENSE Q (only its lower triangle is read),
//     min 1/2 z'Qz + p'z   s.t.   A z = b,   lb <= z <= ub,
// the dense equivalent being QPFunction's (Q, G = [-I; I] with the sides given, h = [-lb; ub]). The inequality block of
// the KKT system is eliminated as in qp_box.cu (r = rx + G'(D rz - rs), dz = D (G dx + rz) - rs, ds = (-rs - dz) / D),
// but H = Q + G'DG is now dense, so a Newton iteration factors the bordered, quasi-definite matrix
//     K = [H A'; A 0] = L diag(I, -I) L',   L = [L11 0; L21 L22],   L11 = chol(H), L21 = A L11^-T, L22 = chol(A H^-1 A'),
// of order N = nz_pad + neq_pad, ONCE, on the product-form staircase of qp_pf.cuh:
//   1. the staircase holds H's lower triangle (identity padding), A in the border rows and, in the trailing block,
//      zeros with -1 on the diagonal of the padding rows past neq;
//   2. pf_chol_setup over the first nz_pad / 8 block columns: L11 and L21 in product form, K22 - L21 L21' = -M left in
//      the trailing block;
//   3. the trailing block negated (M, identity padding);
//   4. pf_chol from block column nz_pad / 8: L22.
// A solve is pf_fwd (or the right-hand side carried through the factorization), pf_diag, the sign of the trailing
// entries flipped, and pf_bwd: dx and dy at once. The predictor and the corrector share the factor. Compared with
// QPFunction on the dense equivalent (order 2 nz + neq, a W of (2 nz + neq) x nz), the factorization is of order
// nz + neq and there is no W. oracle/boxq_model.py is the numpy model of exactly this arithmetic.
//
// Q is read from global memory (L2) once per Newton iteration: the pass that writes Q + diag(g) into the staircase also
// forms Q x for the dual residual. The forward's prologue factors Q itself once: the test of 'Q is not SPD.' (the
// initial point's Q + G'G can be SPD for an indefinite Q).
//
// One CTA of kQNT = 256 threads per QP; the sweeps own one row per thread, so N <= 256, and the whole working set
// (staircase, panel scratch, A, vectors) lives in shared memory (qpb200_boxq_plan.ok). Shapes past that take the dense
// path on the dense equivalent. The loop is this unit's own (the _dm kernels of qp_box.cu do the same): k_box_forward<F>
// is written over a diagonal H and an order-neq factor, and no existing kernel changes.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/qpth_b200.h"
#ifndef QPB_NT
#define QPB_NT 256
#endif
// the device functions of the headers have external linkage (host stubs): give this build its own namespace
#define qpb qpb_boxq
#include "qp_pf.cuh"
#include "qp_jvp.cuh"

extern "C" void qpb200_internal_cuda_error(int err, const char* what);   // (qp_kernels.cu) records the message, per thread
extern "C" int qpb200_internal_set_smem(const void* kernel, size_t bytes);   // (qp_kernels.cu) the kernels' smem limits
// (qp_kernels.cu) out = scale / B (U^T X + Y^T V) by k_mean_outer: the batch mean of dQ for an un-batched Q
extern "C" int qpb200_internal_mean_outer(int B, int rows, int cols, const double* u, const double* x, const double* y,
                                          const double* v, double scale, double* out, void* stream);
// (qp_box.cu) the batch means of dp, dlb, dub, dA, db from the backward's dx, dlam, dnu, as qpb200_box_backward_duals
extern "C" int qpb200_internal_box_means(int nbatch, int n, int m, int e, int nlb, const double* dxv,
                                         const double* dlamv, const double* dnuv, const double* zhat, const double* nus,
                                         double* dp, int mean_p, double* dlb, int mean_lb, double* dub, int mean_ub,
                                         double* dA, int mean_A, double* db, int mean_b, void* stream);

namespace {

using namespace qpb::pf;
constexpr int kQNT = qpb::fast::kNT;
constexpr int kQW = kQNT / 32;
constexpr int kQMaxSmem = 232448;          // H100: 227 KB of dynamic shared memory per CTA

// ---- shared-memory layout (doubles; every offset a multiple of 8) ---------------------------------------------------
struct QDims {
    int n, m, e, np, ep, N, nlb;   // nz, inequality rows (nlb lb rows then ub rows), neq, nz_pad, neq_pad, order, lb rows
    int lda;                       // row stride of A in shared memory
    int S, pan, tab, red, A;
    int p, x, rx, qx, dxa, dx, bx;                          // length np
    int h, s, z, d, rz, dsa, dza, ds, dz, bs, bz, rsc;      // length m
    int b, y, ry, dya, dy, by;                              // length ep
    int u, w, t;                                            // length N: right-hand side, solution, pf_diag scratch
    int total;
};

__host__ __device__ inline int r8(int v) { return (v + 7) & ~7; }

__host__ __device__ inline QDims boxq_dims(int n, int e, int has_lb, int has_ub) {
    QDims D;
    D.n = n; D.e = e; D.np = r8(n); D.ep = r8(e); D.N = D.np + D.ep;
    D.nlb = has_lb ? n : 0; D.m = (has_lb ? n : 0) + (has_ub ? n : 0);
    D.lda = n | 1;
    const int nts = D.N >> 3;
    int o = 0;
    D.S = o; o += r8(pf_elems(nts));
    D.pan = o; o += r8((8 * nts + 8) * kPanLd);
    D.tab = o; o += r8(pf_tab_doubles(nts));
    D.red = o; o += 4 * qpb::kRedStride;
    D.A = o; o += r8(e * D.lda);
    int* vn[] = {&D.p, &D.x, &D.rx, &D.qx, &D.dxa, &D.dx, &D.bx};
    for (int* v : vn) { *v = o; o += D.np; }
    const int mm = r8(D.m);
    int* vm[] = {&D.h, &D.s, &D.z, &D.d, &D.rz, &D.dsa, &D.dza, &D.ds, &D.dz, &D.bs, &D.bz, &D.rsc};
    for (int* v : vm) { *v = o; o += mm; }
    int* ve[] = {&D.b, &D.y, &D.ry, &D.dya, &D.dy, &D.by};
    for (int* v : ve) { *v = o; o += D.ep; }
    int* vN[] = {&D.u, &D.w, &D.t};
    for (int* v : vN) { *v = o; o += D.N; }
    D.total = o;
    return D;
}

// inequality row i is sign(i) * e_var(i)
__device__ __forceinline__ int bvar(const QDims& D, int i) { return i < D.nlb ? i : i - D.nlb; }
__device__ __forceinline__ double bsgn(const QDims& D, int i) { return i < D.nlb ? -1.0 : 1.0; }
__device__ __forceinline__ double gt_col(const QDims& D, const double* v, int j) {
    double a = 0.0;
    if (D.nlb) a -= v[j];
    if (D.m > D.nlb) a += v[D.nlb + j];
    return a;
}
__device__ __forceinline__ double box_step(double v, double dv) { return (dv > 0.0) ? INFINITY : (-v / dv); }
__device__ __forceinline__ double box_step_fix(double v) { return (isinf(v) && v > 0.0) ? 1.0 : v; }

// Stage A (e x n, row stride lda), b (zero past neq; nullptr: zero) and the tile table. Ends with a block barrier.
__device__ void boxq_stage(const QDims& D, const double* A, const double* b) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    for (int t = tid; t < D.e * D.n; t += kQNT) {
        const int i = t / D.n, j = t - i * D.n;
        qsm[D.A + i * D.lda + j] = A[t];
    }
    for (int i = tid; i < D.ep; i += kQNT) qsm[D.b + i] = (b != nullptr && i < D.e) ? b[i] : 0.0;
    pf_build_tab(D.tab, D.N >> 3);
    __syncthreads();
}

// The staircase of the Newton matrix, one warp per row. Rows < nz_pad: the lower triangle of Q (read from global memory,
// lower triangle only) plus g_j = G'DG on the diagonal when with_g, identity padding. With border (rows up to N): A in
// the border rows, zeros in the trailing block except -1 on the diagonal of the padding rows past neq. The entries of a
// diagonal tile above the diagonal are written as zeros. qx >= 0: Q x (x at D.x) into qsm[qx] in the same pass - the
// row pass gives the lower triangle's part, a column pass over the staircase (the strictly lower entries are Q's own)
// the rest. Ends with a block barrier.
__device__ __noinline__ void boxq_fill(const QDims& D, const double* __restrict__ Qg, bool with_g, bool border, int qx) {
    QPB_SMEM;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = D.n, np = D.np, e = D.e;
    const int rows = border ? D.N : np;
    for (int r = warp; r < rows; r += kQW) {
        const int len = 8 * (r >> 3) + 8;
        double* Sr = qsm + D.S + pf_rowoff(r);
        if (r < np) {
            double acc = 0.0;
            for (int c = lane; c < len; c += 32) {
                double v = (r == c) ? 1.0 : 0.0;
                if (r < n && c < n && c <= r) {
                    v = Qg[(int64_t)r * n + c];
                    if (qx >= 0) acc = fma(v, qsm[D.x + c], acc);
                    if (with_g && c == r)
                        v += (D.nlb ? qsm[D.d + r] : 0.0) + ((D.m > D.nlb) ? qsm[D.d + D.nlb + r] : 0.0);
                } else if (c != r) {
                    v = 0.0;
                }
                Sr[c] = v;
            }
            if (qx >= 0) {
                acc = qpb::warp_sum(acc);
                if (lane == 0) qsm[qx + r] = acc;
            }
        } else {
            const int i = r - np;
            for (int c = lane; c < len; c += 32) {
                double v;
                if (c < np) v = (i < e && c < n) ? qsm[D.A + i * D.lda + c] : 0.0;
                else v = (c == r && i >= e) ? -1.0 : 0.0;
                Sr[c] = v;
            }
        }
    }
    __syncthreads();
    if (qx >= 0) {
        for (int j = threadIdx.x; j < n; j += kQNT) {
            double s0 = 0.0, s1 = 0.0;
            int r = j + 1;
            for (; r + 1 < n; r += 2) {
                s0 = fma(qsm[D.S + pf_rowoff(r) + j], qsm[D.x + r], s0);
                s1 = fma(qsm[D.S + pf_rowoff(r + 1) + j], qsm[D.x + r + 1], s1);
            }
            if (r < n) s0 = fma(qsm[D.S + pf_rowoff(r) + j], qsm[D.x + r], s0);
            qsm[qx + j] += s0 + s1;
        }
        __syncthreads();
    }
}

// chol(Q) of the staircase boxq_fill(with_g = false, border = false) left: 1 where a pivot broke down
__device__ int boxq_spd_bad(const QDims& D) {
    QPB_SMEM;
    for (int i = threadIdx.x; i < D.N; i += kQNT) qsm[D.u + i] = 0.0;
    __syncthreads();
    pf_chol(D.S, D.np >> 3, 0, D.u, D.pan, D.tab);
    __syncthreads();
    int bad = 0;
    for (int i = threadIdx.x; i < D.n; i += kQNT) {
        const double ri = qsm[D.S + pf_rowoff(i) + i];       // 1 / L_ii
        bad |= !(ri > 0.0) || isinf(ri);
    }
    return __syncthreads_or(bad);
}

// The structured KKT solve with the staircase of the last boxq_fill (fresh: factored here, the right-hand side carried
// along) or its existing factor:  K [dx ds dz dy] = -[rx rs rz ry];  rs, rz, ry may be -1 (zero). Ends with a barrier.
__device__ __noinline__ void boxq_solve(const QDims& D, bool fresh, int rx, int rs, int rz, int ry, int dx, int ds,
                                        int dz, int dy) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const int n = D.n, m = D.m, e = D.e, np = D.np, N = D.N;
    const int nts = N >> 3, ntz = np >> 3;
    // u = -[r; ry],  r = rx + G'(D rz - rs)
    for (int j = tid; j < N; j += kQNT) {
        double a = 0.0;
        if (j < n) {
            a = qsm[rx + j];
            if (D.nlb) a -= ((rz >= 0) ? qsm[D.d + j] * qsm[rz + j] : 0.0) - ((rs >= 0) ? qsm[rs + j] : 0.0);
            if (m > D.nlb) {
                const int i = D.nlb + j;
                a += ((rz >= 0) ? qsm[D.d + i] * qsm[rz + i] : 0.0) - ((rs >= 0) ? qsm[rs + i] : 0.0);
            }
        } else if (j >= np && j - np < e && ry >= 0) {
            a = qsm[ry + j - np];
        }
        qsm[D.u + j] = -a;
    }
    __syncthreads();
    if (fresh) {
        if (e > 0) {
            pf_chol_setup(D.S, nts, 0, ntz, D.u, D.pan, D.tab, nullptr, 0);   // L11, L21; -M in the trailing block
            for (int t = tid; t < D.ep * D.ep; t += kQNT) {
                const int r = np + t / D.ep, c = np + t % D.ep;
                if (c <= r) qsm[D.S + pf_rowoff(r) + c] = -qsm[D.S + pf_rowoff(r) + c];
            }
            __syncthreads();
            pf_chol(D.S, nts, ntz, D.u, D.pan, D.tab);                        // L22
        } else {
            pf_chol(D.S, nts, 0, D.u, D.pan, D.tab);
        }
        __syncthreads();
    } else {
        pf_fwd(D.S, N, 0, nts - 1, D.u);
    }
    pf_diag(D.S, N, D.u, D.t, D.u);
    if (tid >= np && tid < N) qsm[D.u + tid] = -qsm[D.u + tid];   // diag(I, -I); pf_bwd's thread tid reads only u[tid]
    pf_bwd(D.S, N, D.u, D.w);
    for (int j = tid; j < n; j += kQNT) qsm[dx + j] = qsm[D.w + j];
    for (int i = tid; i < e; i += kQNT) qsm[dy + i] = qsm[D.w + np + i];
    __syncthreads();
    for (int i = tid; i < m; i += kQNT) {
        const double di = qsm[D.d + i];
        const double rsi = (rs >= 0) ? qsm[rs + i] : 0.0;
        const double dzi = di * (bsgn(D, i) * qsm[dx + bvar(D, i)] + ((rz >= 0) ? qsm[rz + i] : 0.0)) - rsi;
        qsm[dz + i] = dzi;
        qsm[ds + i] = (-rsi - dzi) / di;
    }
    __syncthreads();
}

// forward (batch.py:47-207): the loop, exits, trace and outputs of k_box_forward (qp_box.cu) with the bordered
// factorization. d = z / s is formed before the residuals, so that one pass over Q gives both Q x and the staircase.
__global__ void __launch_bounds__(kQNT, 2)
k_boxq_forward(QDims D, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ p, int64_t sp,
               const double* __restrict__ A, int64_t sA, const double* __restrict__ b, int64_t sb,
               const double* __restrict__ lb, int64_t slb, const double* __restrict__ ub, int64_t sub, double eps,
               double stall_tol, double best_tie, int notImprovedLim, int maxIter, double* __restrict__ zhat,
               double* __restrict__ lam, double* __restrict__ slacks, double* __restrict__ nus,
               int* __restrict__ iters_out, double* __restrict__ resid_out, double* __restrict__ trace,
               int* __restrict__ spd_flag) {
    QPB_SMEM;
    const int tid = threadIdx.x, qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep;
    const double* Qg = Q + (int64_t)qp * sQ;
    boxq_stage(D, A + (int64_t)qp * sA, (e > 0) ? b + (int64_t)qp * sb : nullptr);
    for (int j = tid; j < n; j += kQNT) qsm[D.p + j] = p[(int64_t)qp * sp + j];
    for (int i = tid; i < m; i += kQNT) {
        qsm[D.h + i] = (i < D.nlb) ? -lb[(int64_t)qp * slb + i] : ub[(int64_t)qp * sub + i - D.nlb];
        qsm[D.d + i] = 1.0;
        qsm[D.rz + i] = -qsm[D.h + i];
    }
    for (int i = tid; i < ep; i += kQNT) { qsm[D.ry + i] = -qsm[D.b + i]; qsm[D.y + i] = 0.0; }
    // ---- 'Q is not SPD.' (qp.py:81-85): chol(Q) itself
    boxq_fill(D, Qg, false, false, -1);
    {
        const int bad = boxq_spd_bad(D);
        if (tid == 0 && spd_flag != nullptr) spd_flag[qp] = bad;
    }

    // ---- initial point: solve_kkt(p, 0, -h, -b) with d = 1   (batch.py:61-67)
    boxq_fill(D, Qg, true, true, -1);
    boxq_solve(D, true, D.p, -1, D.rz, D.ry, D.x, D.s, D.z, D.y);
    {
        double mn[2] = {INFINITY, INFINITY};
        for (int i = tid; i < m; i += kQNT) { mn[0] = fmin(mn[0], qsm[D.s + i]); mn[1] = fmin(mn[1], qsm[D.z + i]); }
        qpb::block_reduce<2, true>(mn, qsm + D.red, tid, kQNT);
        for (int i = tid; i < m; i += kQNT) {                   // slacks and duals >= 1 (batch.py:77-87)
            if (mn[0] < 0.0) qsm[D.s + i] -= mn[0] - 1.0;
            if (mn[1] < 0.0) qsm[D.z + i] -= mn[1] - 1.0;
        }
        __syncthreads();
    }

    double best = 0.0;
    int nNot = 0, iters_run = 0;
    const double dm = (double)m;
    for (int it = 0; it < maxIter; ++it) {
        iters_run = it + 1;
        // ---- d = z/s; one pass over Q: the staircase of this iteration's Newton matrix and Q x
        for (int i = tid; i < m; i += kQNT) qsm[D.d + i] = qsm[D.z + i] / qsm[D.s + i];
        __syncthreads();
        boxq_fill(D, Qg, true, true, D.qx);
        // ---- residuals (batch.py:94-107)
        double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // |ry|^2, |rz|^2, |rx|^2, s.z
        for (int j = tid; j < n; j += kQNT) {
            double a = 0.0;
            for (int i = 0; i < e; ++i) a = fma(qsm[D.A + i * D.lda + j], qsm[D.y + i], a);
            const double r = qsm[D.qx + j] + qsm[D.p + j] + gt_col(D, qsm + D.z, j) + a;
            qsm[D.rx + j] = r;
            acc[2] = fma(r, r, acc[2]);
        }
        for (int i = tid; i < m; i += kQNT) {
            const double r = bsgn(D, i) * qsm[D.x + bvar(D, i)] + qsm[D.s + i] - qsm[D.h + i];
            qsm[D.rz + i] = r;
            acc[1] = fma(r, r, acc[1]);
            acc[3] = fma(qsm[D.s + i], qsm[D.z + i], acc[3]);
        }
        {   // ry = A x - b, one warp per row
            const int lane = tid & 31, warp = tid >> 5;
            for (int i = warp; i < ep; i += kQW) {
                double a = 0.0;
                if (i < e)
                    for (int k = lane; k < n; k += 32) a = fma(qsm[D.A + i * D.lda + k], qsm[D.x + k], a);
                a = qpb::warp_sum(a);
                const double r = (i < e) ? a - qsm[D.b + i] : 0.0;
                if (lane == 0) { qsm[D.ry + i] = r; acc[0] = fma(r, r, acc[0]); }
            }
        }
        qpb::block_reduce<4, false>(acc, qsm + D.red, tid, kQNT);
        const double mu = fabs(acc[3] / dm);
        const double resid = sqrt(acc[1]) + sqrt(acc[0]) + sqrt(acc[2]) + dm * mu;
        if (trace != nullptr && tid == 0) {                     // what verbose=1 prints (batch.py:115-117)
            double* tr = trace + ((int64_t)qp * maxIter + it) * 4;
            tr[0] = sqrt(acc[1]) + sqrt(acc[0]); tr[1] = sqrt(acc[2]); tr[2] = mu; tr[3] = resid;
        }
        // ---- best-iterate tracking and exit tests (batch.py:118-143), per QP
        const bool improved = (it == 0) || (resid < best);
        if (improved) { best = resid; nNot = 0; } else { ++nNot; }
        if (improved || resid < best_tie * best) {
            for (int j = tid; j < n; j += kQNT) qsm[D.bx + j] = qsm[D.x + j];
            for (int i = tid; i < m; i += kQNT) { qsm[D.bs + i] = qsm[D.s + i]; qsm[D.bz + i] = qsm[D.z + i]; }
            for (int i = tid; i < e; i += kQNT) qsm[D.by + i] = qsm[D.y + i];
        }
        if ((nNot == notImprovedLim && best < stall_tol) || best < eps || mu > 1e32) break;
        if (!(resid == resid) || isinf(resid)) break;
        // ---- the affine direction (batch.py:109-113,150) factors K
        boxq_solve(D, true, D.rx, D.z, D.rz, D.ry, D.dxa, D.dsa, D.dza, D.dya);
        // ---- affine step length and sigma (batch.py:160-168)
        double mn[2] = {INFINITY, INFINITY};
        for (int i = tid; i < m; i += kQNT) {
            mn[0] = fmin(mn[0], box_step(qsm[D.z + i], qsm[D.dza + i]));
            mn[1] = fmin(mn[1], box_step(qsm[D.s + i], qsm[D.dsa + i]));
        }
        qpb::block_reduce<2, true>(mn, qsm + D.red, tid, kQNT);
        {
            const double alpha = fmin(fmin(box_step_fix(mn[0]), box_step_fix(mn[1])), 1.0);
            double sm[2] = {0.0, 0.0};
            for (int i = tid; i < m; i += kQNT) {
                sm[0] = fma(qsm[D.s + i] + alpha * qsm[D.dsa + i], qsm[D.z + i] + alpha * qsm[D.dza + i], sm[0]);
                sm[1] = fma(qsm[D.s + i], qsm[D.z + i], sm[1]);
            }
            qpb::block_reduce<2, false>(sm, qsm + D.red, tid, kQNT);
            const double sr = sm[0] / sm[1];
            const double sig = sr * sr * sr;
            // ---- corrector right-hand side (batch.py:170-181): rs = (-mu sig + dsa dza) / s, rx = rz = ry = 0
            for (int i = tid; i < m; i += kQNT)
                qsm[D.rsc + i] = (-mu * sig + qsm[D.dsa + i] * qsm[D.dza + i]) / qsm[D.s + i];
            for (int j = tid; j < n; j += kQNT) qsm[D.rx + j] = 0.0;
            __syncthreads();
        }
        boxq_solve(D, false, D.rx, D.rsc, -1, -1, D.dx, D.ds, D.dz, D.dy);
        // ---- combined direction, step length, update (batch.py:185-203)
        mn[0] = INFINITY; mn[1] = INFINITY;
        for (int i = tid; i < m; i += kQNT) {
            const double dzi = qsm[D.dza + i] + qsm[D.dz + i], dsi = qsm[D.dsa + i] + qsm[D.ds + i];
            qsm[D.dz + i] = dzi;
            qsm[D.ds + i] = dsi;
            mn[0] = fmin(mn[0], box_step(qsm[D.z + i], dzi));
            mn[1] = fmin(mn[1], box_step(qsm[D.s + i], dsi));
        }
        qpb::block_reduce<2, true>(mn, qsm + D.red, tid, kQNT);
        const double alpha = fmin(0.999 * fmin(box_step_fix(mn[0]), box_step_fix(mn[1])), 1.0);
        for (int j = tid; j < n; j += kQNT) qsm[D.x + j] = fma(alpha, qsm[D.dxa + j] + qsm[D.dx + j], qsm[D.x + j]);
        for (int i = tid; i < m; i += kQNT) {
            qsm[D.s + i] = fma(alpha, qsm[D.ds + i], qsm[D.s + i]);
            qsm[D.z + i] = fma(alpha, qsm[D.dz + i], qsm[D.z + i]);
        }
        for (int i = tid; i < e; i += kQNT) qsm[D.y + i] = fma(alpha, qsm[D.dya + i] + qsm[D.dy + i], qsm[D.y + i]);
        __syncthreads();
    }
    __syncthreads();
    for (int j = tid; j < n; j += kQNT) zhat[(int64_t)qp * n + j] = qsm[D.bx + j];
    for (int i = tid; i < m; i += kQNT) {
        lam[(int64_t)qp * m + i] = qsm[D.bz + i];
        slacks[(int64_t)qp * m + i] = qsm[D.bs + i];
    }
    if (nus != nullptr)
        for (int i = tid; i < e; i += kQNT) nus[(int64_t)qp * e + i] = qsm[D.by + i];
    if (tid == 0) { iters_out[qp] = iters_run; resid_out[qp] = best; }
}

// QPFunctionFn.backward (qp.py:128-182) for the dense-Q box QP: d from the clamped duals (qp.py:148), one factor and one
// solve per QP, then dQ = 1/2 (dx z' + z dx'), dp = dx, dlb = dlam_lb, dub = -dlam_ub, dA = dnu z' + nu dx', db = -dnu.
// dxv, dlamv, dnuv always receive dx, dlam, dnu (the batch means read them); a gradient whose mean flag is set is
// skipped here. dl_dlam / dl_dnu (NULL: zero) are the adjoints of the returned duals, the rz / ry of the solve.
struct QGrads {
    double *dQ, *dp, *dlb, *dub, *dA, *db;
    int mQ, mp, mlb, mub, mA, mb;
};

__global__ void __launch_bounds__(kQNT, 2)
k_boxq_backward(QDims D, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ A, int64_t sA,
                const double* __restrict__ dl, const double* __restrict__ dl_dlam, const double* __restrict__ dl_dnu,
                const double* __restrict__ zhat, const double* __restrict__ lam, const double* __restrict__ slacks,
                const double* __restrict__ nus, QGrads O, double* __restrict__ dxv, double* __restrict__ dlamv,
                double* __restrict__ dnuv) {
    QPB_SMEM;
    const int tid = threadIdx.x, qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e;
    boxq_stage(D, A + (int64_t)qp * sA, nullptr);
    for (int j = tid; j < n; j += kQNT) {
        qsm[D.rx + j] = dl[(int64_t)qp * n + j];
        qsm[D.x + j] = zhat[(int64_t)qp * n + j];
    }
    for (int i = tid; i < m; i += kQNT) {
        const int64_t g = (int64_t)qp * m + i;
        qsm[D.d + i] = fmax(lam[g], 1e-8) / fmax(slacks[g], 1e-8);
        if (dl_dlam != nullptr) qsm[D.rz + i] = dl_dlam[g];
    }
    if (dl_dnu != nullptr)
        for (int i = tid; i < e; i += kQNT) qsm[D.ry + i] = dl_dnu[(int64_t)qp * e + i];
    __syncthreads();
    boxq_fill(D, Q + (int64_t)qp * sQ, true, true, -1);
    boxq_solve(D, true, D.rx, -1, dl_dlam != nullptr ? D.rz : -1, dl_dnu != nullptr ? D.ry : -1, D.dx, D.ds, D.dz,
               D.dy);
    for (int j = tid; j < n; j += kQNT) {
        const int64_t g = (int64_t)qp * n + j;
        const double dx = qsm[D.dx + j];
        dxv[g] = dx;
        if (O.dp && !O.mp) O.dp[g] = dx;
    }
    if (O.dQ && !O.mQ)
        for (int t = tid; t < n * n; t += kQNT) {
            const int i = t / n, j = t - i * n;
            O.dQ[(int64_t)qp * n * n + t] = 0.5 * fma(qsm[D.dx + i], qsm[D.x + j], qsm[D.x + i] * qsm[D.dx + j]);
        }
    for (int i = tid; i < m; i += kQNT) {
        const double dz = qsm[D.dz + i];
        dlamv[(int64_t)qp * m + i] = dz;
        if (i < D.nlb) { if (O.dlb && !O.mlb) O.dlb[(int64_t)qp * n + i] = dz; }
        else if (O.dub && !O.mub) O.dub[(int64_t)qp * n + i - D.nlb] = -dz;
    }
    for (int i = tid; i < e; i += kQNT) {
        dnuv[(int64_t)qp * e + i] = qsm[D.dy + i];
        if (O.db && !O.mb) O.db[(int64_t)qp * e + i] = -qsm[D.dy + i];
    }
    if (O.dA && !O.mA)
        for (int t = tid; t < e * n; t += kQNT) {
            const int i = t / n, j = t - i * n;
            O.dA[((int64_t)qp * e + i) * n + j] = fma(qsm[D.dy + i], qsm[D.x + j], nus[(int64_t)qp * e + i] * qsm[D.dx + j]);
        }
}

// qpb200_boxq_solve_kkt: the bordered factor and solve for caller-given d and right-hand sides (all vectors (B, len))
__global__ void __launch_bounds__(kQNT, 2)
k_boxq_kkt(QDims D, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ A, int64_t sA,
           const double* __restrict__ d, const double* __restrict__ rx, const double* __restrict__ rs,
           const double* __restrict__ rz, const double* __restrict__ ry, double* __restrict__ dx, double* __restrict__ ds,
           double* __restrict__ dz, double* __restrict__ dy) {
    QPB_SMEM;
    const int tid = threadIdx.x, qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e;
    boxq_stage(D, A + (int64_t)qp * sA, nullptr);
    for (int j = tid; j < n; j += kQNT) qsm[D.rx + j] = rx[(int64_t)qp * n + j];
    for (int i = tid; i < m; i += kQNT) {
        const int64_t g = (int64_t)qp * m + i;
        qsm[D.d + i] = d[g];
        qsm[D.rsc + i] = rs[g];
        qsm[D.rz + i] = rz[g];
    }
    for (int i = tid; i < e; i += kQNT) qsm[D.ry + i] = ry[(int64_t)qp * e + i];
    __syncthreads();
    boxq_fill(D, Q + (int64_t)qp * sQ, true, true, -1);
    boxq_solve(D, true, D.rx, D.rsc, D.rz, D.ry, D.dx, D.ds, D.dz, D.dy);
    for (int j = tid; j < n; j += kQNT) dx[(int64_t)qp * n + j] = qsm[D.dx + j];
    for (int i = tid; i < m; i += kQNT) {
        ds[(int64_t)qp * m + i] = qsm[D.ds + i];
        dz[(int64_t)qp * m + i] = qsm[D.dz + i];
    }
    if (dy != nullptr)
        for (int i = tid; i < e; i += kQNT) dy[(int64_t)qp * e + i] = qsm[D.dy + i];
}

// Forward mode (qpb200_boxq_jvp): the right-hand side of the JVP solve, one QP per CTA,
//   rx = sym(dQ) z + dp + dA' nu,   rz = [dlb; -dub] (lam's [lb rows; ub rows] layout),   ry = dA z - db,
// with qp_jvp.cuh::contract for both tangent matrices (one pass over each). Strides and NULL tangents as k_box_jvp_rhs.
inline size_t boxq_jvp_smem_bytes(int n, int e) { return (size_t)(2 * r8(n) + 2 * r8(e) + qpb::jvp::part_doubles(kQNT)) * 8; }
__global__ void __launch_bounds__(kQNT)
k_boxq_jvp_rhs(int n, int e, int nlb, int m, const double* __restrict__ dQ, int64_t sdQ, const double* __restrict__ dp,
               int64_t sdp, const double* __restrict__ dA, int64_t sdA, const double* __restrict__ db, int64_t sdb,
               const double* __restrict__ dlb, int64_t sdlb, const double* __restrict__ dub, int64_t sdub,
               const double* __restrict__ zhat, const double* __restrict__ nus, double* __restrict__ rx,
               double* __restrict__ rz, double* __restrict__ ry) {
    QPB_SMEM;
    const int64_t qp = blockIdx.x;
    const int tid = threadIdx.x;
    double* z = qsm;
    double* ax = z + r8(n);
    double* nu = ax + r8(n);
    double* ay = nu + r8(e);
    double* part = ay + r8(e);
    for (int i = tid; i < n; i += kQNT) {
        z[i] = zhat[qp * n + i];
        ax[i] = dp ? dp[qp * sdp + i] : 0.0;
    }
    for (int i = tid; i < e; i += kQNT) {
        nu[i] = nus[qp * e + i];
        ay[i] = db ? -db[qp * sdb + i] : 0.0;
    }
    __syncthreads();
    if (dQ)
        qpb::jvp::contract<kQNT>(dQ + qp * sdQ, n, n, z, z, part, [&](int r, double s) { ax[r] += 0.5 * s; },
                                 [&](int c, double s) { ax[c] += 0.5 * s; });
    if (dA && e > 0)
        qpb::jvp::contract<kQNT>(dA + qp * sdA, e, n, z, nu, part, [&](int r, double s) { ay[r] += s; },
                                 [&](int c, double s) { ax[c] += s; });
    __syncthreads();
    for (int i = tid; i < n; i += kQNT) {
        rx[qp * n + i] = ax[i];
        if (nlb) rz[qp * m + i] = dlb ? dlb[qp * sdlb + i] : 0.0;
        if (m > nlb) rz[qp * m + nlb + i] = dub ? -dub[qp * sdub + i] : 0.0;
    }
    for (int i = tid; i < e; i += kQNT) ry[qp * e + i] = ay[i];
}

int boxq_check_launch(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, what); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}

int boxq_plan_check(const qpb200_boxq_plan* P) {
    if (P == nullptr) return QPB200_ERR_BAD_ARG;
    if (!P->ok) return QPB200_ERR_TOO_LARGE;
    return QPB200_OK;
}

template <typename... KArgs, typename... Args>
int boxq_launch(const char* what, void (*kernel)(KArgs...), const qpb200_boxq_plan* plan, int nbatch, void* stream,
                Args... args) {
    const QDims D = boxq_dims(plan->nz, plan->neq, plan->has_lb, plan->has_ub);
    const size_t bytes = (size_t)D.total * 8;
    const int rc = qpb200_internal_set_smem((const void*)kernel, bytes);
    if (rc) return rc;
    kernel<<<nbatch, kQNT, bytes, (cudaStream_t)stream>>>(D, args...);
    return boxq_check_launch(what);
}

}  // namespace

extern "C" {

int qpb200_boxq_plan_init(int nz, int neq, int has_lb, int has_ub, qpb200_boxq_plan* plan) {
    if (plan == nullptr || nz <= 0 || neq < 0) return QPB200_ERR_BAD_ARG;
    if (!has_lb && !has_ub) return QPB200_ERR_NO_CONSTRAINTS;
    memset(plan, 0, sizeof(*plan));
    plan->nz = nz; plan->neq = neq; plan->neq_pad = r8(neq);
    plan->has_lb = has_lb ? 1 : 0; plan->has_ub = has_ub ? 1 : 0;
    plan->nineq = (plan->has_lb + plan->has_ub) * nz;
    plan->threads = kQNT;
    if (nz > 4096 || neq > 4096) return QPB200_OK;          // (ok = 0: far past one CTA; keeps the sizes in int range)
    plan->order = r8(nz) + r8(neq);
    const QDims D = boxq_dims(nz, neq, plan->has_lb, plan->has_ub);
    plan->smem_bytes = (int64_t)D.total * 8;
    plan->ok = (plan->order <= kQNT && plan->smem_bytes <= kQMaxSmem) ? 1 : 0;
    return QPB200_OK;
}

int qpb200_boxq_forward(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* p,
                        int64_t sp, const double* A, int64_t sA, const double* b, int64_t sb, const double* lb,
                        int64_t slb, const double* ub, int64_t sub, double eps, double stall_tol, double best_tie,
                        int notImprovedLim, int maxIter, double* zhat, double* lam, double* slacks, double* nus,
                        int* iters, double* best_resid, double* trace, int* spd_flag, void* stream) {
    int rc = boxq_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || maxIter < 1 || !Q || !p || !zhat || !lam || !slacks || !iters || !best_resid) return QPB200_ERR_BAD_ARG;
    if ((plan->has_lb && !lb) || (plan->has_ub && !ub) || (plan->neq > 0 && (!A || !b || !nus))) return QPB200_ERR_BAD_ARG;
    return boxq_launch("k_boxq_forward", k_boxq_forward, plan, nbatch, stream, Q, sQ, p, sp, A, sA, b, sb, lb, slb, ub,
                       sub, eps, stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam, slacks, nus, iters, best_resid,
                       trace, spd_flag);
}

int qpb200_boxq_backward_duals(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A,
                               int64_t sA, const double* dl_dzhat, const double* dl_dlam, const double* dl_dnu,
                               const double* zhat, const double* lam, const double* slacks, const double* nus,
                               double* dQ, int mean_Q, double* dp, int mean_p, double* dlb, int mean_lb, double* dub,
                               int mean_ub, double* dA, int mean_A, double* db, int mean_b, double* dxv,
                               double* dlamv, double* dnuv, void* stream) {
    int rc = boxq_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || !Q || !dl_dzhat || !zhat || !lam || !slacks || !dxv || !dlamv) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!A || !nus || !dnuv)) return QPB200_ERR_BAD_ARG;
    if (dl_dnu && plan->neq == 0) return QPB200_ERR_BAD_ARG;
    if ((dlb && !plan->has_lb) || (dub && !plan->has_ub)) return QPB200_ERR_BAD_ARG;
    const int n = plan->nz, m = plan->nineq, e = plan->neq, nlb = plan->has_lb ? n : 0;
    QGrads O;
    O.dQ = dQ; O.dp = dp; O.dlb = dlb; O.dub = dub; O.dA = e > 0 ? dA : nullptr; O.db = e > 0 ? db : nullptr;
    O.mQ = mean_Q; O.mp = mean_p; O.mlb = mean_lb; O.mub = mean_ub; O.mA = mean_A; O.mb = mean_b;
    rc = boxq_launch("k_boxq_backward", k_boxq_backward, plan, nbatch, stream, Q, sQ, A, sA, dl_dzhat, dl_dlam, dl_dnu,
                     zhat, lam, slacks, nus, O, dxv, dlamv, dnuv);
    if (rc) return rc;
    if (dQ && mean_Q) {
        rc = qpb200_internal_mean_outer(nbatch, n, n, dxv, zhat, zhat, dxv, 0.5, dQ, stream);
        if (rc) return rc;
    }
    return qpb200_internal_box_means(nbatch, n, m, e, nlb, dxv, dlamv, dnuv, zhat, nus, dp, mean_p, dlb, mean_lb, dub,
                                     mean_ub, e > 0 ? dA : nullptr, mean_A, e > 0 ? db : nullptr, mean_b, stream);
}

int qpb200_boxq_jvp(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A, int64_t sA,
                    const double* dQ, int64_t sdQ, const double* dp, int64_t sdp, const double* dA, int64_t sdA,
                    const double* db, int64_t sdb, const double* dlb, int64_t sdlb, const double* dub, int64_t sdub,
                    const double* zhat, const double* lam, const double* slacks, const double* nus, double* rhs,
                    double* dz, double* dlam, double* dnu, void* stream) {
    // every check of qpb200_boxq_backward_duals, before k_boxq_jvp_rhs is launched
    int rc = boxq_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || !Q || !zhat || !lam || !slacks || !rhs || !dz || !dlam) return QPB200_ERR_BAD_ARG;
    if (sdQ < 0 || sdp < 0 || sdA < 0 || sdb < 0 || sdlb < 0 || sdub < 0) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!A || !nus || !dnu)) return QPB200_ERR_BAD_ARG;
    if (plan->neq == 0 && (dA || db || dnu)) return QPB200_ERR_BAD_ARG;
    if ((dlb && !plan->has_lb) || (dub && !plan->has_ub)) return QPB200_ERR_BAD_ARG;
    const int n = plan->nz, m = plan->nineq, e = plan->neq, nlb = plan->has_lb ? n : 0;
    const size_t bytes = boxq_jvp_smem_bytes(n, e);
    rc = qpb200_internal_set_smem((const void*)k_boxq_jvp_rhs, bytes);
    if (rc) return rc;
    const int64_t B = nbatch;
    double* rx = rhs;
    double* rz = rx + B * n;
    double* ry = rz + B * m;
    k_boxq_jvp_rhs<<<nbatch, kQNT, bytes, (cudaStream_t)stream>>>(n, e, nlb, m, dQ, sdQ, dp, sdp, dA, sdA, db, sdb, dlb,
                                                                  sdlb, dub, sdub, zhat, nus, rx, rz, ry);
    rc = boxq_check_launch("k_boxq_jvp_rhs");
    if (rc) return rc;
    return qpb200_boxq_backward_duals(plan, nbatch, Q, sQ, A, sA, rx, (dlb || dub) ? rz : nullptr,
                                      (dA || db) ? ry : nullptr, zhat, lam, slacks, nus, nullptr, 0, nullptr, 0, nullptr,
                                      0, nullptr, 0, nullptr, 0, nullptr, 0, dz, dlam, dnu, stream);
}

int qpb200_boxq_solve_kkt(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A,
                          int64_t sA, const double* d, const double* rx, const double* rs, const double* rz,
                          const double* ry, double* dx, double* ds, double* dz, double* dy, void* stream) {
    int rc = boxq_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || !Q || !d || !rx || !rs || !rz || !dx || !ds || !dz) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!A || !ry || !dy)) return QPB200_ERR_BAD_ARG;
    return boxq_launch("k_boxq_kkt", k_boxq_kkt, plan, nbatch, stream, Q, sQ, A, sA, d, rx, rs, rz, ry, dx, ds, dz, dy);
}

}  // extern "C"
