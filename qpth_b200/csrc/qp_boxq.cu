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
// One CTA of kBoxNT = 256 threads per QP; the sweeps own one row per thread, so N <= 256, and the whole working set
// (staircase, panel scratch, A, vectors) lives in shared memory (qpb200_boxq_plan.ok). Shapes past that take the dense
// path on the dense equivalent. The Mehrotra loop, the backward and the KKT kernel are those of qp_box_loop.cuh, for the
// family DenseQ below.
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
#include "qp_box_loop.cuh"
#include "qp_jac.cuh"

extern "C" int qpb200_internal_set_smem(const void* kernel, size_t bytes);   // (qp_kernels.cu) the kernels' smem limits
// (qp_kernels.cu) out = scale / B (U^T X + Y^T V) by k_mean_outer: the batch mean of dQ for an un-batched Q
extern "C" int qpb200_internal_mean_outer(int B, int rows, int cols, const double* u, const double* x, const double* y,
                                          const double* v, double scale, double* out, void* stream);
// (qp_box.cu) the batch means of dp, dlb, dub, dA, db from the backward's dx, dlam, dnu, as qpb200_box_backward_duals
extern "C" int qpb200_internal_box_means(int nbatch, int n, int m, int e, int nlb, const double* dxv,
                                         const double* dlamv, const double* dnuv, const double* zhat, const double* nus,
                                         double* dp, int mean_p, double* dlb, int mean_lb, double* dub, int mean_ub,
                                         double* dA, int mean_A, double* db, int mean_b, void* stream);
// (qp_box.cu) the double backward's per-QP gradients and batch sums, as in qpb200_box_double_backward (dense: dQ)
extern "C" int qpb200_internal_box_ggrad_out(int nbatch, int n, int m, int e, int nlb, int dense, const double* zhat,
                                             const double* nus, const double* dxv, const double* dnuv,
                                             const double* gg_z, const double* gg_nu, const double* wx,
                                             const double* wl, const double* wn, const double* cs, double* dq,
                                             int sum_q, double* dp, int sum_p, double* dlb, int sum_lb, double* dub,
                                             int sum_ub, double* dA, int sum_A, double* db, int sum_b, void* stream);

namespace {

using namespace qpb::pf;

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

// Stage A (e x n, row stride lda), b (zero past neq; nullptr: zero) and the tile table. Ends with a block barrier.
__device__ void boxq_stage(const QDims& D, const double* A, const double* b) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    for (int t = tid; t < D.e * D.n; t += kBoxNT) {
        const int i = t / D.n, j = t - i * D.n;
        qsm[D.A + i * D.lda + j] = A[t];
    }
    for (int i = tid; i < D.ep; i += kBoxNT) qsm[D.b + i] = (b != nullptr && i < D.e) ? b[i] : 0.0;
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
    for (int r = warp; r < rows; r += kClW) {
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
        for (int j = threadIdx.x; j < n; j += kBoxNT) {
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
    for (int i = threadIdx.x; i < D.N; i += kBoxNT) qsm[D.u + i] = 0.0;
    __syncthreads();
    pf_chol(D.S, D.np >> 3, 0, D.u, D.pan, D.tab);
    __syncthreads();
    int bad = 0;
    for (int i = threadIdx.x; i < D.n; i += kBoxNT) {
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
    for (int j = tid; j < N; j += kBoxNT) {
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
            for (int t = tid; t < D.ep * D.ep; t += kBoxNT) {
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
    for (int j = tid; j < n; j += kBoxNT) qsm[dx + j] = qsm[D.w + j];
    for (int i = tid; i < e; i += kBoxNT) qsm[dy + i] = qsm[D.w + np + i];
    __syncthreads();
    for (int i = tid; i < m; i += kBoxNT) {
        const double di = qsm[D.d + i];
        const double rsi = (rs >= 0) ? qsm[rs + i] : 0.0;
        const double dzi = di * (bsgn(D, i) * qsm[dx + bvar(D, i)] + ((rz >= 0) ? qsm[rz + i] : 0.0)) - rsi;
        qsm[dz + i] = dzi;
        qsm[ds + i] = (-rsi - dzi) / di;
    }
    __syncthreads();
}

// One CTA per QP with a dense Q (read from global memory) and the bordered factorization. The phases take the layout
// by reference, so the family refers to the kernel parameter rather than copying it: a copy would put the whole family,
// Q's pointer included, in the stack frame.
struct DenseQ : BoxCta<QDims, const QDims&> {
    static constexpr int kMinFwd = 2, kMinBwd = 2, kMinKkt = 2;
    const double* Qg = nullptr;      // this QP's Q (stage)

    __device__ explicit DenseQ(const QDims& P) : BoxCta(P) {}
    __device__ void stage(const double* Q, const double* A, const double* b) {
        Qg = Q;
        boxq_stage(D, A, b);
    }
    // 'Q is not SPD.' (qp.py:81-85): chol(Q) itself
    __device__ int spd_bad() const {
        boxq_fill(D, Qg, false, false, -1);
        return boxq_spd_bad(D);
    }
    __device__ void form() const { boxq_fill(D, Qg, true, true, -1); }
    // one pass over Q: the staircase of this iteration's Newton matrix and Q x
    template <class G> __device__ void before_residuals(G form_d) const {
        form_d();
        boxq_fill(D, Qg, true, true, D.qx);
    }
    __device__ double qx_p(int j) const { QPB_SMEM; return qsm[D.qx + j] + qsm[D.p + j]; }
    template <class G> __device__ static void before_affine(G) {}
    __device__ void solve(bool fresh, int rx, int rs, int rz, int ry, int dx, int ds, int dz, int dy) const {
        boxq_solve(D, fresh, rx, rs, rz, ry, dx, ds, dz, dy);
    }
    // dQ = 1/2 (dx z' + z dx')
    __device__ void write_dq(double* dQ, int qp, const double* __restrict__ zhat) const {
        QPB_SMEM;
        const int n = D.n;
        const double* z = zhat + (int64_t)qp * n;
        for (int t = threadIdx.x; t < n * n; t += kBoxNT) {
            const int i = t / n, j = t - i * n;
            dQ[(int64_t)qp * n * n + t] = 0.5 * fma(qsm[D.dx + i], z[j], z[i] * qsm[D.dx + j]);
        }
    }
};

// Forward mode (qpb200_boxq_jvp): the right-hand side of the JVP solve, one QP per CTA,
//   rx = sym(dQ) z + dp + dA' nu,   rz = [dlb; -dub] (lam's [lb rows; ub rows] layout),   ry = dA z - db,
// with qp_jvp.cuh::contract for both tangent matrices (one pass over each). Strides and NULL tangents as k_box_jvp_rhs.
inline size_t boxq_jvp_smem_bytes(int n, int e) { return (size_t)(2 * r8(n) + 2 * r8(e) + qpb::jvp::part_doubles(kBoxNT)) * 8; }
__global__ void __launch_bounds__(kBoxNT)
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
    for (int i = tid; i < n; i += kBoxNT) {
        z[i] = zhat[qp * n + i];
        ax[i] = dp ? dp[qp * sdp + i] : 0.0;
    }
    for (int i = tid; i < e; i += kBoxNT) {
        nu[i] = nus[qp * e + i];
        ay[i] = db ? -db[qp * sdb + i] : 0.0;
    }
    __syncthreads();
    if (dQ)
        qpb::jvp::contract<kBoxNT>(dQ + qp * sdQ, n, n, z, z, part, [&](int r, double s) { ax[r] += 0.5 * s; },
                                 [&](int c, double s) { ax[c] += 0.5 * s; });
    if (dA && e > 0)
        qpb::jvp::contract<kBoxNT>(dA + qp * sdA, e, n, z, nu, part, [&](int r, double s) { ay[r] += s; },
                                 [&](int c, double s) { ax[c] += s; });
    __syncthreads();
    for (int i = tid; i < n; i += kBoxNT) {
        rx[qp * n + i] = ax[i];
        if (nlb) rz[qp * m + i] = dlb ? dlb[qp * sdlb + i] : 0.0;
        if (m > nlb) rz[qp * m + nlb + i] = dub ? -dub[qp * sdub + i] : 0.0;
    }
    for (int i = tid; i < e; i += kBoxNT) ry[qp * e + i] = ay[i];
}

// Double backward (qpb200_boxq_double_backward): k_box_ggrad_rhs (qp_box.cu) with the cotangent wQ of a dense Q,
//   cz = sym(wQ) vx + wA' vnu + c_s_lb - c_s_ub,   clam = c_lam,   cnu = wA vx,
// one jvp::contract pass over wQ (into the n accumulator of cz) and one over wA. Shared memory: vx and cz (n), vnu and
// cnu (e), the column partials: boxq_jvp_smem_bytes(n, e).
__global__ void __launch_bounds__(kBoxNT)
k_boxq_ggrad_rhs(int n, int e, int nlb, int m, const double* __restrict__ wQ, int64_t swQ, const double* __restrict__ wA,
                 int64_t swA, const double* __restrict__ dxv, const double* __restrict__ dlamv,
                 const double* __restrict__ dnuv, const double* __restrict__ ulam, const double* __restrict__ lam,
                 const double* __restrict__ slacks, double* __restrict__ cz, double* __restrict__ clam,
                 double* __restrict__ cnu, double* __restrict__ cs) {
    QPB_SMEM;
    const int64_t qp = blockIdx.x;
    const int tid = threadIdx.x;
    double* vx = qsm;
    double* az = vx + r8(n);
    double* vn = az + r8(n);
    double* an = vn + r8(e);
    double* part = an + r8(e);
    const int64_t o = qp * m;
    auto c_s = [&](int i) {                        // row i's c_s, and its c_lam into clam
        double cl, c;
        qpb::jvp::clamp_cotangents(lam[o + i], slacks[o + i], ulam[o + i], dlamv[o + i], cl, c);
        clam[o + i] = cl;
        cs[o + i] = c;
        return c;
    };
    for (int i = tid; i < n; i += kBoxNT) {
        vx[i] = dxv[qp * n + i];
        az[i] = (nlb ? c_s(i) : 0.0) - (m > nlb ? c_s(nlb + i) : 0.0);
    }
    for (int i = tid; i < e; i += kBoxNT) {
        vn[i] = dnuv[qp * e + i];
        an[i] = 0.0;
    }
    __syncthreads();
    if (wQ)
        qpb::jvp::contract<kBoxNT>(wQ + qp * swQ, n, n, vx, vx, part, [&](int r, double s) { az[r] += 0.5 * s; },
                                 [&](int c, double s) { az[c] += 0.5 * s; });
    if (wA && e > 0)
        qpb::jvp::contract<kBoxNT>(wA + qp * swA, e, n, vx, vn, part, [&](int r, double s) { an[r] += s; },
                                 [&](int c, double s) { az[c] += s; });
    __syncthreads();
    for (int i = tid; i < n; i += kBoxNT) cz[qp * n + i] = az[i];
    for (int i = tid; i < e; i += kBoxNT) cnu[qp * e + i] = an[i];
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
    kernel<<<nbatch, kBoxNT, bytes, (cudaStream_t)stream>>>(D, args...);
    return box_check_launch(what);
}

// ---- Jacobians of z*, lam, nu with respect to p, lb, ub, b (qpb200_boxq_jacobian) ----------------------------------
// At the returned point with the backward's clamped D, X = K^-1 for K = [H A'; A 0], H = Q + G'DG: p column j is
// -X e_j (z and nu rows), b column c is X e_(nz_pad + c), the lb / ub columns and the lam rows are scalings of them
// (box_jac_store). One CTA per QP builds K's staircase with boxq_fill, factors it as the forward does (pf_chol_setup,
// the trailing block negated, pf_chol: K = L diag(I, -I) L'), and then each warp sweeps whole 8-column blocks with
// jac_ssolve_bordered: the forward sweep from the block of the right-hand side's unit rows, T_k' T_k, the trailing block
// rows negated, the backward sweep. Shared memory: the staircase, panel, tile table, pf_chol's vector (N) and d; then
// the warps' N x 8 buffers, where A is staged for boxq_fill before the factorization (the staircase holds A after it).
struct BQDims {
    int aug, blk, per, nblk;       // pf_chol's vector, the buffers (A staged there first), doubles per buffer, buffers
    int64_t smem;                  // dynamic shared memory, bytes; 0: not covered
};

// the layout of k_boxq_jacobian: the QDims fields boxq_fill reads (S, pan, tab, d, A), and the buffers
BQDims boxq_jac_dims(const qpb200_boxq_plan* p, QDims& D) {
    D = QDims{};
    D.n = p->nz; D.e = p->neq; D.np = r8(D.n); D.ep = r8(D.e); D.N = D.np + D.ep;
    D.nlb = p->has_lb ? D.n : 0; D.m = (p->has_lb + p->has_ub) * D.n;
    D.lda = D.n | 1;
    const int nts = D.N >> 3;
    BQDims J{};
    int o = 0;
    D.S = o; o += r8(pf_elems(nts));
    D.pan = o; o += r8((8 * nts + 8) * kPanLd);
    D.tab = o; o += r8(pf_tab_doubles(nts));
    J.aug = o; o += D.N;
    D.d = o; o += r8(D.m);
    J.blk = D.A = o;
    J.per = 8 * D.N;
    const int64_t cap = kBoxMaxSmem / 8, a_end = (int64_t)J.blk + r8(D.e * D.lda);
    int64_t nb = (cap - J.blk) / J.per;
    if (nb > kBoxNT / 32) nb = kBoxNT / 32;
    if (D.N > kBoxNT || a_end > cap || nb < 1) nb = 0;     // the factorization's order bound of qpb200_boxq_plan.ok
    J.nblk = (int)nb;
    const int64_t end = (int64_t)J.blk + nb * J.per;
    J.smem = nb ? 8 * (end > a_end ? end : a_end) : 0;
    return J;
}

__global__ void __launch_bounds__(kBoxNT, 1)
k_boxq_jacobian(const __grid_constant__ QDims D, BQDims J, BOut O, const double* __restrict__ Q, int64_t sQ, const double* __restrict__ A,
                int64_t sA, const double* __restrict__ lam, const double* __restrict__ slk, double* __restrict__ Jg) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t qp = blockIdx.x;
    const int n = D.n, m = D.m, e = D.e, np = D.np, N = D.N, nts = N >> 3, ntz = np >> 3;
    // ---- 1. d = clamp(lam, 1e-8) / clamp(s, 1e-8), A staged, K's staircase, K = L diag(I, -I) L'
    for (int i = tid; i < m; i += kBoxNT) qsm[D.d + i] = fmax(lam[qp * m + i], 1e-8) / fmax(slk[qp * m + i], 1e-8);
    if (e > 0) {
        const double* Aq = A + qp * sA;
        for (int t = tid; t < e * n; t += kBoxNT) {
            const int i = t / n, j = t - i * n;
            qsm[D.A + i * D.lda + j] = Aq[t];
        }
    }
    for (int i = tid; i < N; i += kBoxNT) qsm[J.aug + i] = 0.0;
    pf_build_tab(D.tab, nts);
    __syncthreads();
    boxq_fill(D, Q + qp * sQ, true, true, -1);
    if (e > 0) {
        pf_chol_setup(D.S, nts, 0, ntz, J.aug, D.pan, D.tab, nullptr, 0);   // L11, L21; -M in the trailing block
        for (int t = tid; t < D.ep * D.ep; t += kBoxNT) {
            const int r = np + t / D.ep, c = np + t % D.ep;
            if (c <= r) qsm[D.S + pf_rowoff(r) + c] = -qsm[D.S + pf_rowoff(r) + c];
        }
        __syncthreads();
        pf_chol(D.S, nts, ntz, J.aug, D.pan, D.tab);                        // L22
    } else {
        pf_chol(D.S, nts, 0, J.aug, D.pan, D.tab);
    }
    __syncthreads();
    // ---- 2. column blocks: p blocks (which also give the lb and ub columns), then the b tiles, one warp per block
    if (warp >= J.nblk) return;
    double* X = qsm + J.blk + (int64_t)warp * J.per;
    const double* dv = qsm + D.d;
    const int npb = (O.cp >= 0 || O.clb >= 0 || O.cub >= 0) ? ntz : 0;
    const int nblocks = npb + ((O.cb >= 0) ? (D.ep >> 3) : 0);
    double* Jq = Jg + qp * (int64_t)O.R * O.C;
#pragma unroll 1
    for (int t = warp; t < nblocks; t += J.nblk) {
        const bool pblk = t < npb;
        const int j0 = 8 * (pblk ? t : t - npb), row0 = pblk ? j0 : np + j0;
        // X = K^-1 E (p) or -K^-1 E (b): then U = X's z rows and Y = its nu rows are -z and -nu of the column
        const double one = pblk ? 1.0 : -1.0;
        for (int i = lane; i < 8 * N; i += 32) X[i] = ((i >> 3) == row0 + (i & 7)) ? one : 0.0;
        __syncwarp();
        jac_ssolve_bordered(qsm + D.S, nts, row0 >> 3, ntz, X);
#pragma unroll 1
        for (int kind = 0; kind < (pblk ? 3 : 1); ++kind) {
            const int c0 = pblk ? (kind == 0 ? O.cp : (kind == 1 ? O.clb : O.cub)) : O.cb;
            if (c0 >= 0) box_jac_store(Jq, O, n, D.nlb, m, e, dv, X, X + 8 * np, kind, c0 + j0, j0, min(8, (pblk ? n : e) - j0));
        }
        __syncwarp();
    }
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
    plan->threads = kBoxNT;
    if (nz > 4096 || neq > 4096) return QPB200_OK;          // (ok = 0: far past one CTA; keeps the sizes in int range)
    plan->order = r8(nz) + r8(neq);
    const QDims D = boxq_dims(nz, neq, plan->has_lb, plan->has_ub);
    plan->smem_bytes = (int64_t)D.total * 8;
    plan->ok = (plan->order <= kBoxNT && plan->smem_bytes <= kBoxMaxSmem) ? 1 : 0;
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
    return boxq_launch("k_boxq_forward", k_box_forward<DenseQ>, plan, nbatch, stream, Q, sQ, p, sp, A, sA, b, sb, lb, slb, ub,
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
    BoxGrads O;
    O.dq = dQ; O.dp = dp; O.dlb = dlb; O.dub = dub; O.dA = e > 0 ? dA : nullptr; O.db = e > 0 ? db : nullptr;
    O.mq = mean_Q; O.mp = mean_p; O.mlb = mean_lb; O.mub = mean_ub; O.mA = mean_A; O.mb = mean_b;
    rc = boxq_launch("k_boxq_backward", k_box_backward<DenseQ>, plan, nbatch, stream, Q, sQ, A, sA, dl_dzhat, dl_dlam, dl_dnu,
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
    k_boxq_jvp_rhs<<<nbatch, kBoxNT, bytes, (cudaStream_t)stream>>>(n, e, nlb, m, dQ, sdQ, dp, sdp, dA, sdA, db, sdb, dlb,
                                                                  sdlb, dub, sdub, zhat, nus, rx, rz, ry);
    rc = box_check_launch("k_boxq_jvp_rhs");
    if (rc) return rc;
    return qpb200_boxq_backward_duals(plan, nbatch, Q, sQ, A, sA, rx, (dlb || dub) ? rz : nullptr,
                                      (dA || db) ? ry : nullptr, zhat, lam, slacks, nus, nullptr, 0, nullptr, 0, nullptr,
                                      0, nullptr, 0, nullptr, 0, nullptr, 0, dz, dlam, dnu, stream);
}

int qpb200_boxq_double_backward(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ,
                                const double* A, int64_t sA, const double* wQ, int64_t swQ, const double* wp,
                                int64_t swp, const double* wA, int64_t swA, const double* wb, int64_t swb,
                                const double* wlb, int64_t swlb, const double* wub, int64_t swub, const double* dxv,
                                const double* dlamv, const double* dnuv, const double* zhat, const double* lam,
                                const double* slacks, const double* nus, double* gg_z, double* gg_lam, double* gg_nu,
                                double* dQ, int sum_Q, double* dp, int sum_p, double* dlb, int sum_lb, double* dub,
                                int sum_ub, double* dA, int sum_A, double* db, int sum_b, double* work, void* stream) {
    // the checks beyond qpb200_boxq_jvp's, which that call runs before its first launch
    int rc = boxq_plan_check(plan);
    if (rc) return rc;
    if (!dxv || !dlamv || !work || (plan->neq > 0 && !dnuv)) return QPB200_ERR_BAD_ARG;
    if (plan->neq == 0 && (dA || db)) return QPB200_ERR_BAD_ARG;
    if ((dlb && !plan->has_lb) || (dub && !plan->has_ub)) return QPB200_ERR_BAD_ARG;
    const int n = plan->nz, m = plan->nineq, e = plan->neq, nlb = plan->has_lb ? n : 0;
    rc = qpb200_boxq_jvp(plan, nbatch, Q, sQ, A, sA, wQ, swQ, wp, swp, wA, swA, wb, swb, wlb, swlb, wub, swub, zhat, lam,
                         slacks, nus, work, gg_z, gg_lam, gg_nu, stream);
    if (rc) return rc;
    // work as in qpb200_box_double_backward
    const int64_t B = nbatch;
    double* cz = work;
    double* clam = cz + B * n;
    double* cnu = clam + B * m;
    double* cs = cnu + B * e;
    double* wx = cs + B * m;
    double* wl = wx + B * n;
    double* wn = wl + B * m;
    const size_t bytes = boxq_jvp_smem_bytes(n, e);
    rc = qpb200_internal_set_smem((const void*)k_boxq_ggrad_rhs, bytes);
    if (rc) return rc;
    k_boxq_ggrad_rhs<<<nbatch, kBoxNT, bytes, (cudaStream_t)stream>>>(n, e, nlb, m, wQ, swQ, wA, swA, dxv, dlamv, dnuv,
                                                                      gg_lam, lam, slacks, cz, clam, cnu, cs);
    rc = box_check_launch("k_boxq_ggrad_rhs");
    if (rc) return rc;
    rc = qpb200_boxq_backward_duals(plan, nbatch, Q, sQ, A, sA, cz, clam, (e > 0 && wA) ? cnu : nullptr, zhat, lam,
                                    slacks, nus, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0,
                                    wx, wl, e > 0 ? wn : nullptr, stream);
    if (rc) return rc;
    return qpb200_internal_box_ggrad_out(nbatch, n, m, e, nlb, 1, zhat, nus, dxv, dnuv, gg_z, gg_nu, wx, wl, wn, cs, dQ,
                                         sum_Q, dp, sum_p, dlb, sum_lb, dub, sum_ub, dA, sum_A, db, sum_b, stream);
}

int qpb200_boxq_solve_kkt(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A,
                          int64_t sA, const double* d, const double* rx, const double* rs, const double* rz,
                          const double* ry, double* dx, double* ds, double* dz, double* dy, void* stream) {
    int rc = boxq_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || !Q || !d || !rx || !rs || !rz || !dx || !ds || !dz) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!A || !ry || !dy)) return QPB200_ERR_BAD_ARG;
    return boxq_launch("k_boxq_kkt", k_box_kkt<DenseQ>, plan, nbatch, stream, Q, sQ, A, sA, d, rx, rs, rz, ry, dx, ds, dz, dy);
}


int qpb200_boxq_jacobian_smem(const qpb200_boxq_plan* plan, int64_t* smem_bytes) {
    if (!plan || !smem_bytes) return QPB200_ERR_BAD_ARG;
    if (plan->nz <= 0 || plan->neq < 0 || plan->neq_pad != r8(plan->neq) ||
        plan->nineq != (plan->has_lb + plan->has_ub) * plan->nz || plan->nineq <= 0)
        return QPB200_ERR_BAD_ARG;
    QDims D;
    *smem_bytes = boxq_jac_dims(plan, D).smem;
    return QPB200_OK;
}

int qpb200_boxq_jacobian(const qpb200_boxq_plan* plan, int nbatch, int rows, int cols, const double* Q, int64_t sQ,
                         const double* A, int64_t sA, const double* lam, const double* slacks, double* J, void* stream) {
    int64_t smem = 0;
    int rc = qpb200_boxq_jacobian_smem(plan, &smem);
    if (rc) return rc;
    if (!Q || !lam || !slacks || !J || nbatch < 1 || sQ < 0 || sA < 0) return QPB200_ERR_BAD_ARG;
    if (rows <= 0 || cols <= 0 || (rows & ~7) || (cols & ~15)) return QPB200_ERR_BAD_ARG;
    if (plan->neq == 0 && ((rows & 4) || (cols & 8))) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && !A) return QPB200_ERR_BAD_ARG;
    if (((cols & 2) && !plan->has_lb) || ((cols & 4) && !plan->has_ub)) return QPB200_ERR_BAD_ARG;
    if (smem == 0) return QPB200_ERR_TOO_LARGE;
    QDims D;
    const BQDims Jd = boxq_jac_dims(plan, D);
    const int n = D.n, m = D.m, e = D.e;
    BOut O;
    int off = 0;
    O.rz = (rows & 1) ? off : -1; off += (rows & 1) ? n : 0;
    O.rl = (rows & 2) ? off : -1; off += (rows & 2) ? m : 0;
    O.rn = (rows & 4) ? off : -1; off += (rows & 4) ? e : 0;
    O.R = off; off = 0;
    O.cp = (cols & 1) ? off : -1; off += (cols & 1) ? n : 0;
    O.clb = (cols & 2) ? off : -1; off += (cols & 2) ? n : 0;
    O.cub = (cols & 4) ? off : -1; off += (cols & 4) ? n : 0;
    O.cb = (cols & 8) ? off : -1; off += (cols & 8) ? e : 0;
    O.C = off;
    rc = qpb200_internal_set_smem((const void*)k_boxq_jacobian, (size_t)Jd.smem);
    if (rc) return rc;
    k_boxq_jacobian<<<nbatch, kBoxNT, (size_t)Jd.smem, (cudaStream_t)stream>>>(D, Jd, O, Q, sQ, A, sA, lam, slacks, J);
    return box_check_launch("k_boxq_jacobian");
}

}  // extern "C"
