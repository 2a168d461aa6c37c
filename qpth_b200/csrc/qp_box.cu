// qp_box.cu - the structured solver of BoxQPFunction: diagonal Q = diag(q), inequality rows G = [-I; I] (the sides
// given: "lb rows" then "ub rows", h = [-lb; ub]) and dense equality rows A z = b. The inequality block of the KKT
// system (batch.py:349-372) is eliminated in closed form:
//     H = q + G'DG (diagonal),  r = rx + G'(D rz - rs),  M = A H^-1 A'  (order neq, SPD for full-row-rank A),
//     M dy = ry - A H^-1 r,  dx = -H^-1 (r + A'dy),  dz = D (G dx + rz) - rs,  ds = (-rs - dz) / D,
// so a Newton iteration factors an order-neq matrix (no chol(Q), no W, no K template) and everything else is
// elementwise or one pass over A. M is factored by the product-form Cholesky of qp_pf.cuh (pf_chol on a staircase of
// order neq_pad) and solved with pf_fwd / pf_diag / pf_bwd; the predictor and the corrector share one factor.
// oracle/box_model.py is the numpy model of exactly this arithmetic.
//
// Three layouts run this solver, all with 128-thread CTAs:
//   one CTA per QP (family OneCta): A (neq x nz, row stride nz | 1), the factor of M and every vector live in shared
//            memory, within the 227 KB an H100 CTA may use, and neq_pad <= 128: the substitutions own one row per
//            thread (qpb200_box_plan.ok needs both). For neq <= nz (A of full row rank) shared memory binds first: the
//            most such a CTA holds is neq_pad 120 ((121, 117, both), 128 B left). For neq > nz the 128-row term is the
//            one that decides: (8, 136, lb) fits in 114 KB and is rejected by it alone.
//   a cluster per QP (family Cluster): past that, a thread block cluster of 2, 4 or 8 CTAs (qpb200_box_plan.cl_ctas),
//            each CTA holding a slice of the variables; M is summed and factored redundantly in every CTA.
//   distributed M (k_box_*_dm): past neq_pad = 128, M is distributed over the cluster as well and A is read from
//            global memory.
// BoxQPFunction runs the dense kernels on the dense equivalent only where none covers the shape. For the first two the
// Mehrotra loop (k_box_forward<F>), the backward and KKT kernels and the structured solve (box_solve<F>) are written
// once; a family supplies only what differs: its per-CTA context, its reductions, how A is staged, how M is formed and
// solved.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <utility>

#include "../../include/qpth_b200.h"
#ifndef QPB_NT
#define QPB_NT 128
#endif
// the device functions of the headers have external linkage (host stubs): give this build its own namespace
#define qpb qpb_box
#include "qp_pf.cuh"

extern "C" void qpb200_internal_cuda_error(int err, const char* what);   // (qp_kernels.cu) records the message, per thread

namespace {

using namespace qpb::pf;
namespace cg = cooperative_groups;
constexpr int kBoxNT = qpb::fast::kNT;
constexpr int kClW = kBoxNT / 32;          // warps per CTA: scalar partials are published per warp
constexpr int kBoxMaxSmem = 232448;        // H100: 227 KB of dynamic shared memory per CTA

// ---- shared-memory layout (doubles; every offset a multiple of 8, i.e. 64-byte aligned) ------------------------------
struct BoxDims {
    int n, m, e, ep, nlb;    // nz, inequality rows (nlb lb rows then ub rows), neq, neq_pad, nz if lb given else 0
    int lda;                 // row stride of A in shared memory (odd: the row-wise passes are bank-conflict free)
    // offsets
    int A, S, pan, tab, red;
    int q, p, x, rx, r, hinv, dxa, dx, bx;                   // length n
    int h, s, z, d, rz, dsa, dza, ds, dz, bs, bz, rsc;       // length m
    int b, y, ry, rhs, t, dya, dy, by;                       // length ep
    int total;               // doubles
};

__host__ __device__ inline int r8(int v) { return (v + 7) & ~7; }

// the n-, m- and ep-length vectors of D (counts set) from offset o; returns the end
__host__ __device__ inline int box_vectors(BoxDims& D, int o) {
    const int nn = r8(D.n), mm = r8(D.m), ee = D.ep;
    int* vn[] = {&D.q, &D.p, &D.x, &D.rx, &D.r, &D.hinv, &D.dxa, &D.dx, &D.bx};
    for (int* v : vn) { *v = o; o += nn; }
    int* vm[] = {&D.h, &D.s, &D.z, &D.d, &D.rz, &D.dsa, &D.dza, &D.ds, &D.dz, &D.bs, &D.bz, &D.rsc};
    for (int* v : vm) { *v = o; o += mm; }
    int* ve[] = {&D.b, &D.y, &D.ry, &D.rhs, &D.t, &D.dya, &D.dy, &D.by};
    for (int* v : ve) { *v = o; o += ee; }
    return o;
}

__host__ __device__ inline BoxDims box_dims(int n, int e, int has_lb, int has_ub) {
    BoxDims D;
    D.n = n; D.e = e; D.ep = r8(e); D.nlb = has_lb ? n : 0; D.m = (has_lb ? n : 0) + (has_ub ? n : 0);
    D.lda = n | 1;
    const int nts = D.ep >> 3;
    int o = 0;
    D.A = o; o += r8(e * D.lda);
    D.S = o; o += r8(pf_elems(nts));
    D.pan = o; o += (e > 0) ? r8((8 * nts + 8) * kPanLd) : 0;
    D.tab = o; o += r8(pf_tab_doubles(nts));
    D.red = o; o += 4 * qpb::kRedStride;
    D.total = box_vectors(D, o);
    return D;
}

// inequality row i is sign(i) * e_var(i)
__device__ __forceinline__ int bvar(const BoxDims& D, int i) { return i < D.nlb ? i : i - D.nlb; }
__device__ __forceinline__ double bsgn(const BoxDims& D, int i) { return i < D.nlb ? -1.0 : 1.0; }

// G'v of a length-m shared vector at column j (the lb row and/or the ub row of variable j)
__device__ __forceinline__ double gt_col(const BoxDims& D, const double* v, int j) {
    double a = 0.0;
    if (D.nlb) a -= v[j];
    if (D.m > D.nlb) a += v[D.nlb + j];
    return a;
}

__device__ __forceinline__ double box_step(double v, double dv) { return (dv > 0.0) ? INFINITY : (-v / dv); }
__device__ __forceinline__ double box_step_fix(double v) { return (isinf(v) && v > 0.0) ? 1.0 : v; }

// hinv = 1 / (q + G'DG) for the local variables and the d currently in shared memory (no barrier)
__device__ __forceinline__ void form_hinv(const BoxDims& D) {
    QPB_SMEM;
    for (int j = threadIdx.x; j < D.n; j += kBoxNT) {
        double hj = qsm[D.q + j];
        if (D.nlb) hj += qsm[D.d + j];
        if (D.m > D.nlb) hj += qsm[D.d + D.nlb + j];
        qsm[D.hinv + j] = 1.0 / hj;
    }
}

// row of entry t of a packed lower triangle (t = r (r + 1) / 2 + c)
__device__ __forceinline__ int tri_row(int t) {
    int r = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while ((r * (r + 1)) / 2 > t) --r;
    while (((r + 1) * (r + 2)) / 2 <= t) ++r;
    return r;
}

// (A H^-1 A')_rc over the n shared columns of rows ar, ac (lda apart in shared memory)
__device__ __forceinline__ double ahat(const double* ar, const double* ac, const double* hv, int n) {
    double s0 = 0.0, s1 = 0.0;
    int k = 0;
    for (; k + 1 < n; k += 2) {
        s0 = fma(ar[k] * hv[k], ac[k], s0);
        s1 = fma(ar[k + 1] * hv[k + 1], ac[k + 1], s1);
    }
    if (k < n) s0 = fma(ar[k] * hv[k], ac[k], s0);
    return s0 + s1;
}

// The factor of the staircase in D.S with the right-hand side D.rhs carried along (fresh), or its forward sweep with
// the existing factor; then pf_diag and the backward sweep into dy.
__device__ __forceinline__ void stair_solve(const BoxDims& D, bool fresh, int dy) {
    const int nts = D.ep >> 3;
    if (fresh) {
        pf_chol(D.S, nts, 0, D.rhs, D.pan, D.tab);
        __syncthreads();
    } else {
        pf_fwd(D.S, D.ep, 0, nts - 1, D.rhs);
    }
    pf_diag(D.S, D.ep, D.rhs, D.t, D.rhs);
    pf_bwd(D.S, D.ep, D.rhs, dy);
}

// ---- the families -------------------------------------------------------------------------------------------------------
// Each is the per-CTA context of one layout, built in the kernel from its parameter (F::Dims), and supplies:
//   qp(), j0() (first local variable), ng() / mg() (nz and inequality rows of the whole QP), grow(i) (global
//   inequality row of local row i), leader() (rank 0: writes the length-neq outputs, iters, best_resid, the trace and
//   spd_flag), a(i, j) (A at local column j), reduce_sum / reduce_min, any (the SPD test), stage, form (H^-1 and M),
//   ry_step (ry = A x - b, |ry|^2 into acc, and the reduction of acc), solve_mid (rhs = ry - A H^-1 r, factor or forward
//   sweep, pf_diag, backward sweep to dy) and sync() (the closing cluster barrier).

// One CTA per QP; j0 = 0 and leader() (rank 0) are compile-time facts.
struct OneCta {
    using Dims = BoxDims;
    static constexpr int kMinFwd = 3, kMinBwd = 4, kMinKkt = 0;     // CTAs per SM (0: no bound)
    BoxDims D;

    __device__ explicit OneCta(const BoxDims& P) : D(P) {}
    __device__ static int qp() { return blockIdx.x; }
    __host__ __device__ static constexpr int j0() { return 0; }
    __device__ int ng() const { return D.n; }
    __device__ int mg() const { return D.m; }
    __device__ static int64_t grow(int i) { return i; }
    __host__ __device__ static constexpr bool leader() { return true; }
    __device__ double a(int i, int j) const { QPB_SMEM; return qsm[D.A + i * D.lda + j]; }
    template <int N> __device__ void reduce_sum(double (&v)[N]) {
        QPB_SMEM;
        qpb::block_reduce<N, false>(v, qsm + D.red, threadIdx.x, kBoxNT);
    }
    template <int N> __device__ void reduce_min(double (&v)[N]) {
        QPB_SMEM;
        qpb::block_reduce<N, true>(v, qsm + D.red, threadIdx.x, kBoxNT);
    }
    __device__ static int any(int v) { return __syncthreads_or(v); }
    __device__ static void sync() {}

    // q, A, b (nullptr in the backward and KKT kernels) of this QP; the staircase tile table
    __device__ void stage(const double* q, const double* A, const double* b) const {
        QPB_SMEM;
        const int tid = threadIdx.x;
        for (int j = tid; j < D.n; j += kBoxNT) qsm[D.q + j] = q[j];
        for (int t = tid; t < D.e * D.n; t += kBoxNT) {
            const int i = t / D.n, j = t - i * D.n;
            qsm[D.A + i * D.lda + j] = A[t];
        }
        for (int i = tid; i < D.ep; i += kBoxNT) qsm[D.b + i] = (b != nullptr && i < D.e) ? b[i] : 0.0;
        if (D.e > 0) pf_build_tab(D.tab, D.ep >> 3);
        __syncthreads();
    }

    // H^-1; with A, M into the staircase (lower tiles, identity rows beyond neq). Ends with a block barrier.
    __device__ __noinline__ void form() const {
        QPB_SMEM;
        form_hinv(D);
        __syncthreads();
        if (D.e == 0) return;
        const int ep = D.ep, n = D.n, lda = D.lda;
        const int tot = (ep * (ep + 1)) / 2;
        for (int t = threadIdx.x; t < tot; t += kBoxNT) {
            const int r = tri_row(t), c = t - (r * (r + 1)) / 2;
            const double v = (r < D.e) ? ahat(qsm + D.A + r * lda, qsm + D.A + c * lda, qsm + D.hinv, n)
                                       : ((r == c) ? 1.0 : 0.0);
            qsm[D.S + pf_rowoff(r) + c] = v;
        }
        __syncthreads();
    }

    // ry = A x - b, one warp per row; |ry|^2 per warp before the block reduction
    __device__ void ry_step(double (&acc)[4]) {
        QPB_SMEM;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int i = warp; i < D.ep; i += kClW) {
            double a = 0.0;
            if (i < D.e)
                for (int k = lane; k < D.n; k += 32) a = fma(qsm[D.A + i * D.lda + k], qsm[D.x + k], a);
            a = qpb::warp_sum(a);
            const double r = (i < D.e) ? a - qsm[D.b + i] : 0.0;
            if (lane == 0) { qsm[D.ry + i] = r; acc[0] = fma(r, r, acc[0]); }
        }
        reduce_sum(acc);
    }

    __device__ void solve_mid(bool fresh, int ry, int dy) {
        QPB_SMEM;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const int n = D.n, e = D.e, ep = D.ep, lda = D.lda;
        // rhs = ry - A H^-1 r: one warp per row, lanes over the columns
        for (int i = warp; i < ep; i += kClW) {
            double a = 0.0;
            if (i < e)
                for (int k = lane; k < n; k += 32) a = fma(qsm[D.A + i * lda + k], qsm[D.r + k], a);
            a = qpb::warp_sum(a);
            if (lane == 0) qsm[D.rhs + i] = (i < e) ? (((ry >= 0) ? qsm[ry + i] : 0.0) - a) : 0.0;
        }
        __syncthreads();
        stair_solve(D, fresh, dy);
    }
};

// ---- one thread block cluster of C CTAs per QP ------------------------------------------------------------------------
// CTA `rank` owns the variables [rank * slice, rank * slice + nloc) (the last slice may be partial or empty). In its own
// shared memory it holds its entries of every length-nz vector and the lb / ub rows of those variables (local row order:
// lb rows, then ub rows), laid out as for slice variables so that every CTA has the same footprint; the length-neq_pad
// vectors are replicated. A reduction is combined in rank order (then warp order) from the partials every CTA publishes,
// so every CTA holds bit-identical sums and minima (see the invariant at k_box_forward).
//
// Publish buffers alternate: a CTA rewrites buffer (ph & 1) only after the cluster barrier of the reduction that
// followed its previous use, and every CTA finishes reading a buffer before it arrives at that barrier.
struct ClDims {
    BoxDims L;               // layout of one slice (L.n = slice); counts are set per CTA in cl_local
    int C, slice, ng, nlbg, mg;   // cluster size, variables per CTA, nz, lb rows, inequality rows (global)
    int Mp, pub, pb;         // partial M (e (e + 1) / 2 doubles), publish buffers (two of pb doubles: ep + 4 kClW)
    int total;               // doubles per CTA
};

// the variable slices of a cluster of C CTAs
__host__ __device__ inline void cl_slices(ClDims& X, int n, int has_lb, int has_ub, int C) {
    X.C = C; X.slice = (n + C - 1) / C; X.ng = n;
    X.nlbg = has_lb ? n : 0; X.mg = (has_lb ? n : 0) + (has_ub ? n : 0);
}

__host__ __device__ inline ClDims cl_dims(int n, int e, int has_lb, int has_ub, int C) {
    ClDims X;
    cl_slices(X, n, has_lb, has_ub, C);
    X.L = box_dims(X.slice, e, has_lb, has_ub);
    int o = X.L.total;
    X.Mp = o; o += r8((e * (e + 1)) / 2);
    X.pb = r8(X.L.ep + 4 * kClW);
    X.pub = o; o += 2 * X.pb;
    X.total = o;
    return X;
}

__device__ __forceinline__ int cl_buf(const ClDims& X, int ph) { return X.pub + (ph & 1) * X.pb; }

// this CTA's counts: nloc variables from j0
__device__ __forceinline__ BoxDims cl_local(const ClDims& X, int rank, int& j0) {
    BoxDims D = X.L;
    j0 = rank * X.slice;
    const int nloc = max(0, min(X.slice, X.ng - j0));
    D.n = nloc;
    D.nlb = X.nlbg ? nloc : 0;
    D.m = (X.nlbg ? nloc : 0) + (X.mg > X.nlbg ? nloc : 0);
    return D;
}
// global inequality row of local row i
__device__ __forceinline__ int64_t cl_grow(const ClDims& X, const BoxDims& D, int j0, int i) {
    return (i < D.nlb) ? (int64_t)(j0 + i) : (int64_t)(X.nlbg + j0 + i - D.nlb);
}

// Cluster-wide reduction of N scalars (sum or min) and, when vlen > 0, of the length-vlen vector the caller wrote to
// qsm[cl_buf(X, ph)] (vdst: where its sum goes). One cluster barrier; every thread returns with the combined scalars.
// Ends with a block barrier when vlen > 0.
template <int N, bool kMin>
__device__ __forceinline__ void cl_reduce(const ClDims& X, double (&v)[N], int& ph, int vlen, int vdst) {
    QPB_SMEM;
    cg::cluster_group cl = cg::this_cluster();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int buf = cl_buf(X, ph), sc = buf + X.L.ep;
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = kMin ? qpb::warp_min(v[k]) : qpb::warp_sum(v[k]);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) qsm[sc + k * kClW + warp] = v[k];
    }
    cl.sync();
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = kMin ? INFINITY : 0.0;
    for (int r = 0; r < X.C; ++r) {
        const double* rp = cl.map_shared_rank(qsm + sc, r);
#pragma unroll
        for (int k = 0; k < N; ++k)
#pragma unroll
            for (int w = 0; w < kClW; ++w) v[k] = kMin ? fmin(v[k], rp[k * kClW + w]) : v[k] + rp[k * kClW + w];
    }
    if (vlen > 0) {
        for (int i = tid; i < vlen; i += kBoxNT) {
            double s = 0.0;
            for (int r = 0; r < X.C; ++r) s += cl.map_shared_rank(qsm + buf, r)[i];
            qsm[vdst + i] = s;
        }
        __syncthreads();
    }
    ++ph;
}

// A cluster per QP: every CTA holds its columns of A, forms its partial A_r H_r^-1 A_r' (compact lower triangle, X.Mp),
// and sums the partials in rank order and factors M itself (same input, same code: bit-identical factor and dy, with no
// broadcast and no extra barrier). The partial M is rewritten by the next form only after the right-hand-side reduction
// of the solve that read it.
struct Cluster {
    using Dims = ClDims;
    static constexpr int kMinFwd = 1, kMinBwd = 1, kMinKkt = 1;
    ClDims X;
    BoxDims D;               // this CTA's slice
    int ph = 0;              // cluster reductions so far: selects the publish buffer

    __device__ explicit Cluster(const ClDims& P) : X(P) {
        int j0;
        D = cl_local(X, rank(), j0);
    }
    __device__ int qp() const { return blockIdx.x / X.C; }
    __device__ static int rank() { return (int)cg::this_cluster().block_rank(); }
    __device__ int j0() const { return rank() * X.slice; }
    __device__ int ng() const { return X.ng; }
    __device__ int mg() const { return X.mg; }
    __device__ int64_t grow(int i) const { return cl_grow(X, D, j0(), i); }
    __device__ static bool leader() { return rank() == 0; }
    template <int N> __device__ void reduce_sum(double (&v)[N]) { cl_reduce<N, false>(X, v, ph, 0, 0); }
    template <int N> __device__ void reduce_min(double (&v)[N]) { cl_reduce<N, true>(X, v, ph, 0, 0); }
    __device__ int any(int bad) {
        double v[1] = {bad ? 1.0 : 0.0};
        reduce_sum(v);
        return v[0] > 0.0;
    }
    // no CTA exits while another may still read its shared memory
    __device__ static void sync() { cg::this_cluster().sync(); }
    __device__ double a(int i, int j) const { QPB_SMEM; return qsm[D.A + i * D.lda + j]; }

    // q and this CTA's columns of A; b replicated (forward only); the staircase tile table
    __device__ void stage(const double* q, const double* A, const double* b) const {
        QPB_SMEM;
        const int tid = threadIdx.x, j0 = this->j0();
        for (int j = tid; j < D.n; j += kBoxNT) qsm[D.q + j] = q[j0 + j];
        for (int t = tid; t < D.e * D.n; t += kBoxNT) {
            const int i = t / D.n, j = t - i * D.n;
            qsm[D.A + i * D.lda + j] = A[(int64_t)i * X.ng + j0 + j];
        }
        for (int i = tid; i < D.ep; i += kBoxNT) qsm[D.b + i] = (b != nullptr && i < D.e) ? b[i] : 0.0;
        if (D.e > 0) pf_build_tab(D.tab, D.ep >> 3);
        __syncthreads();
    }

    // H^-1 and the partial M (rows < e) into X.Mp; summed by the next solve
    __device__ __noinline__ void form() const {
        QPB_SMEM;
        form_hinv(D);
        __syncthreads();
        if (D.e == 0) return;
        const int tot = (D.e * (D.e + 1)) / 2;
        for (int t = threadIdx.x; t < tot; t += kBoxNT) {
            const int r = tri_row(t), c = t - (r * (r + 1)) / 2;
            qsm[X.Mp + t] = ahat(qsm + D.A + r * D.lda, qsm + D.A + c * D.lda, qsm + D.hinv, D.n);
        }
    }

    // this CTA's partials of A v (rows < e, its columns) into the publish buffer of the next reduction, a warp per row
    __device__ void publish_av(int v) const {
        QPB_SMEM;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, buf = cl_buf(X, ph);
        for (int i = warp; i < D.e; i += kClW) {
            double a = 0.0;
            for (int k = lane; k < D.n; k += 32) a = fma(qsm[D.A + i * D.lda + k], qsm[v + k], a);
            a = qpb::warp_sum(a);
            if (lane == 0) qsm[buf + i] = a;
        }
    }

    // ry = A x - b: A x is reduced with the scalars, ry and |ry|^2 are formed redundantly after the cluster reduction
    __device__ void ry_step(double (&acc)[4]) {
        QPB_SMEM;
        const int e = D.e;
        publish_av(D.x);
        cl_reduce<4, false>(X, acc, ph, e, D.ry);
        for (int i = 0; i < e; ++i) {
            const double r = qsm[D.ry + i] - qsm[D.b + i];
            acc[0] = fma(r, r, acc[0]);
        }
        __syncthreads();                                     // every thread has read the sums of A x
        for (int i = threadIdx.x; i < D.ep; i += kBoxNT) qsm[D.ry + i] = (i < e) ? qsm[D.ry + i] - qsm[D.b + i] : 0.0;
    }

    // rhs = ry - sum_r A_r H_r^-1 r_r in one cluster barrier; fresh: the partial M of the last form is summed into the
    // staircase in the same barrier
    __device__ void solve_mid(bool fresh, int ry, int dy) {
        QPB_SMEM;
        cg::cluster_group cl = cg::this_cluster();
        const int e = D.e, buf = cl_buf(X, ph);
        publish_av(D.r);
        cl.sync();
        for (int i = threadIdx.x; i < D.ep; i += kBoxNT) {
            double a = 0.0;
            if (i < e)
                for (int k = 0; k < X.C; ++k) a += cl.map_shared_rank(qsm + buf, k)[i];
            qsm[D.rhs + i] = (i < e) ? (((ry >= 0) ? qsm[ry + i] : 0.0) - a) : 0.0;
        }
        ++ph;
        if (fresh) {
            const int tot = (D.ep * (D.ep + 1)) / 2;
            for (int t = threadIdx.x; t < tot; t += kBoxNT) {
                const int r = tri_row(t), c = t - (r * (r + 1)) / 2;
                double v = 0.0;
                if (r < e)
                    for (int k = 0; k < X.C; ++k) v += cl.map_shared_rank(qsm + X.Mp, k)[t];
                else
                    v = (r == c) ? 1.0 : 0.0;
                qsm[D.S + pf_rowoff(r) + c] = v;
            }
        }
        __syncthreads();
        stair_solve(D, fresh, dy);
    }
};

// ---- the solver, written once over the families ------------------------------------------------------------------------
// The structured KKT solve with the H / M of the last form:
//   K [dx ds dz dy] = -[rx rs rz ry];  rs, rz, ry may be -1 (zero). fresh: M was just formed and is factored here
// (with the right-hand side carried along), else the existing factor is reused. Ends with a block barrier.
template <class F>
__device__ __noinline__ void box_solve(F& f, bool fresh, int rx, int rs, int rz, int ry, int dx, int ds, int dz, int dy) {
    QPB_SMEM;
    const BoxDims& D = f.D;
    const int tid = threadIdx.x;
    const int n = D.n, m = D.m, e = D.e;
    // r = rx + G'(D rz - rs), kept as H^-1 r in D.r
    for (int j = tid; j < n; j += kBoxNT) {
        double a = qsm[rx + j];
        if (D.nlb) {
            const double t = ((rz >= 0) ? qsm[D.d + j] * qsm[rz + j] : 0.0) - ((rs >= 0) ? qsm[rs + j] : 0.0);
            a -= t;
        }
        if (m > D.nlb) {
            const int i = D.nlb + j;
            const double t = ((rz >= 0) ? qsm[D.d + i] * qsm[rz + i] : 0.0) - ((rs >= 0) ? qsm[rs + i] : 0.0);
            a += t;
        }
        qsm[D.r + j] = a * qsm[D.hinv + j];
    }
    __syncthreads();
    if (e > 0) f.solve_mid(fresh, ry, dy);
    // dx = -H^-1 r - H^-1 A'dy
    for (int j = tid; j < n; j += kBoxNT) {
        double a = 0.0;
        for (int i = 0; i < e; ++i) a = fma(f.a(i, j), qsm[dy + i], a);
        qsm[dx + j] = -qsm[D.r + j] - a * qsm[D.hinv + j];
    }
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

// forward (batch.py:47-207) with the structured solve; the loop of k_forward_fast (qp_solve.cuh). Every CTA writes its
// slice of zhat, lam and slacks; the leader nus, iters, best_resid, the trace rows and spd_flag. One CTA per QP: three
// CTAs per SM (at most 168 registers; about 48 KB of shared memory per QP at nz = 64, neq = 40): four (128 registers)
// spill.
//
// INVARIANT (Cluster, and the k_box_*_dm kernels, which repeat this loop): every CTA of a cluster executes the same
// sequence of cluster.sync() calls. Every reduction leaves bit-identical sums and minima in every CTA, and so does every
// solve (M is summed in rank order and factored redundantly, or dy is gathered from its owners), so y, mu, the residual
// and the step lengths are bit-identical too. Every branch that reaches a cluster barrier (the exit tests, NaN and mu > 1e32 exits, best-iterate
// tracking, notImprovedLim, e > 0, fresh) is decided from those values or from kernel arguments only; a CTA that branched
// on a value of its own would deadlock its cluster.
template <class F>
__global__ void __launch_bounds__(kBoxNT, F::kMinFwd)
k_box_forward(typename F::Dims P, const double* __restrict__ q, int64_t sq, const double* __restrict__ p, int64_t sp,
              const double* __restrict__ A, int64_t sA, const double* __restrict__ b, int64_t sb,
              const double* __restrict__ lb, int64_t slb, const double* __restrict__ ub, int64_t sub, double eps,
              double stall_tol, double best_tie, int notImprovedLim, int maxIter, double* __restrict__ zhat,
              double* __restrict__ lam, double* __restrict__ slacks, double* __restrict__ nus, int* __restrict__ iters_out,
              double* __restrict__ resid_out, double* __restrict__ trace, int* __restrict__ spd_flag) {
    QPB_SMEM;
    F f(P);
    const BoxDims& D = f.D;
    const int tid = threadIdx.x, qp = f.qp(), j0 = f.j0();
    const int n = D.n, m = D.m, e = D.e, ep = D.ep;
    f.stage(q + (int64_t)qp * sq, A + (int64_t)qp * sA, (e > 0) ? b + (int64_t)qp * sb : nullptr);
    {
        int bad = 0;
        for (int j = tid; j < n; j += kBoxNT) {
            qsm[D.p + j] = p[(int64_t)qp * sp + j0 + j];
            bad |= !(qsm[D.q + j] > 0.0);
        }
        bad = f.any(bad);
        if (f.leader() && tid == 0 && spd_flag != nullptr) spd_flag[qp] = bad;
    }
    for (int i = tid; i < m; i += kBoxNT) {
        qsm[D.h + i] = (i < D.nlb) ? -lb[(int64_t)qp * slb + j0 + i] : ub[(int64_t)qp * sub + j0 + i - D.nlb];
        qsm[D.d + i] = 1.0;
        qsm[D.rz + i] = -qsm[D.h + i];
    }
    for (int i = tid; i < ep; i += kBoxNT) { qsm[D.ry + i] = -qsm[D.b + i]; qsm[D.y + i] = 0.0; }
    __syncthreads();

    // ---- initial point: solve_kkt(p, 0, -h, -b) with d = 1   (batch.py:61-67)
    f.form();
    box_solve(f, true, D.p, -1, D.rz, D.ry, D.x, D.s, D.z, D.y);
    {
        double mn[2] = {INFINITY, INFINITY};
        for (int i = tid; i < m; i += kBoxNT) { mn[0] = fmin(mn[0], qsm[D.s + i]); mn[1] = fmin(mn[1], qsm[D.z + i]); }
        f.reduce_min(mn);
        for (int i = tid; i < m; i += kBoxNT) {                  // slacks and duals >= 1 (batch.py:77-87)
            if (mn[0] < 0.0) qsm[D.s + i] -= mn[0] - 1.0;
            if (mn[1] < 0.0) qsm[D.z + i] -= mn[1] - 1.0;
        }
        __syncthreads();
    }

    double best = 0.0;
    int nNot = 0, iters_run = 0;
    const double dm = (double)f.mg();
    for (int it = 0; it < maxIter; ++it) {
        iters_run = it + 1;
        // ---- residuals (batch.py:94-107)
        double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // |ry|^2, |rz|^2, |rx|^2, s.z
        for (int j = tid; j < n; j += kBoxNT) {
            double a = 0.0;
            for (int i = 0; i < e; ++i) a = fma(f.a(i, j), qsm[D.y + i], a);
            const double r = fma(qsm[D.q + j], qsm[D.x + j], qsm[D.p + j]) + gt_col(D, qsm + D.z, j) + a;
            qsm[D.rx + j] = r;
            acc[2] = fma(r, r, acc[2]);
        }
        for (int i = tid; i < m; i += kBoxNT) {
            const double r = bsgn(D, i) * qsm[D.x + bvar(D, i)] + qsm[D.s + i] - qsm[D.h + i];
            qsm[D.rz + i] = r;
            acc[1] = fma(r, r, acc[1]);
            acc[3] = fma(qsm[D.s + i], qsm[D.z + i], acc[3]);
        }
        f.ry_step(acc);
        const double mu = fabs(acc[3] / dm);
        const double resid = sqrt(acc[1]) + sqrt(acc[0]) + sqrt(acc[2]) + dm * mu;
        if (trace != nullptr && f.leader() && tid == 0) {       // what verbose=1 prints (batch.py:115-117)
            double* tr = trace + ((int64_t)qp * maxIter + it) * 4;
            tr[0] = sqrt(acc[1]) + sqrt(acc[0]); tr[1] = sqrt(acc[2]); tr[2] = mu; tr[3] = resid;
        }
        // ---- best-iterate tracking and exit tests (batch.py:118-143), per QP: cluster-wide values only
        const bool improved = (it == 0) || (resid < best);
        if (improved) { best = resid; nNot = 0; } else { ++nNot; }
        if (improved || resid < best_tie * best) {
            for (int j = tid; j < n; j += kBoxNT) qsm[D.bx + j] = qsm[D.x + j];
            for (int i = tid; i < m; i += kBoxNT) { qsm[D.bs + i] = qsm[D.s + i]; qsm[D.bz + i] = qsm[D.z + i]; }
            for (int i = tid; i < e; i += kBoxNT) qsm[D.by + i] = qsm[D.y + i];
        }
        if ((nNot == notImprovedLim && best < stall_tol) || best < eps || mu > 1e32) break;
        if (!(resid == resid) || isinf(resid)) break;
        // ---- d = z/s, H, M; the affine direction (batch.py:109-113,150) factors M
        for (int i = tid; i < m; i += kBoxNT) qsm[D.d + i] = qsm[D.z + i] / qsm[D.s + i];
        __syncthreads();
        f.form();
        box_solve(f, true, D.rx, D.z, D.rz, D.ry, D.dxa, D.dsa, D.dza, D.dya);
        // ---- affine step length and sigma (batch.py:160-168)
        double mn[2] = {INFINITY, INFINITY};
        for (int i = tid; i < m; i += kBoxNT) {
            mn[0] = fmin(mn[0], box_step(qsm[D.z + i], qsm[D.dza + i]));
            mn[1] = fmin(mn[1], box_step(qsm[D.s + i], qsm[D.dsa + i]));
        }
        f.reduce_min(mn);
        {
            const double alpha = fmin(fmin(box_step_fix(mn[0]), box_step_fix(mn[1])), 1.0);
            double sm[2] = {0.0, 0.0};
            for (int i = tid; i < m; i += kBoxNT) {
                sm[0] = fma(qsm[D.s + i] + alpha * qsm[D.dsa + i], qsm[D.z + i] + alpha * qsm[D.dza + i], sm[0]);
                sm[1] = fma(qsm[D.s + i], qsm[D.z + i], sm[1]);
            }
            f.reduce_sum(sm);
            const double sr = sm[0] / sm[1];
            const double sig = sr * sr * sr;
            // ---- corrector right-hand side (batch.py:170-181): rs = (-mu sig + dsa dza) / s, rx = rz = ry = 0
            for (int i = tid; i < m; i += kBoxNT)
                qsm[D.rsc + i] = (-mu * sig + qsm[D.dsa + i] * qsm[D.dza + i]) / qsm[D.s + i];
            for (int j = tid; j < n; j += kBoxNT) qsm[D.rx + j] = 0.0;
            __syncthreads();
        }
        box_solve(f, false, D.rx, D.rsc, -1, -1, D.dx, D.ds, D.dz, D.dy);
        // ---- combined direction, step length, update (batch.py:185-203)
        mn[0] = INFINITY; mn[1] = INFINITY;
        for (int i = tid; i < m; i += kBoxNT) {
            const double dzi = qsm[D.dza + i] + qsm[D.dz + i], dsi = qsm[D.dsa + i] + qsm[D.ds + i];
            qsm[D.dz + i] = dzi;
            qsm[D.ds + i] = dsi;
            mn[0] = fmin(mn[0], box_step(qsm[D.z + i], dzi));
            mn[1] = fmin(mn[1], box_step(qsm[D.s + i], dsi));
        }
        f.reduce_min(mn);
        const double alpha = fmin(0.999 * fmin(box_step_fix(mn[0]), box_step_fix(mn[1])), 1.0);
        for (int j = tid; j < n; j += kBoxNT) qsm[D.x + j] = fma(alpha, qsm[D.dxa + j] + qsm[D.dx + j], qsm[D.x + j]);
        for (int i = tid; i < m; i += kBoxNT) {
            qsm[D.s + i] = fma(alpha, qsm[D.ds + i], qsm[D.s + i]);
            qsm[D.z + i] = fma(alpha, qsm[D.dz + i], qsm[D.z + i]);
        }
        for (int i = tid; i < e; i += kBoxNT) qsm[D.y + i] = fma(alpha, qsm[D.dya + i] + qsm[D.dy + i], qsm[D.y + i]);
        __syncthreads();
    }
    __syncthreads();
    for (int j = tid; j < n; j += kBoxNT) zhat[(int64_t)qp * f.ng() + j0 + j] = qsm[D.bx + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * f.mg() + f.grow(i);
        lam[g] = qsm[D.bz + i];
        slacks[g] = qsm[D.bs + i];
    }
    if (f.leader()) {
        if (nus != nullptr)
            for (int i = tid; i < e; i += kBoxNT) nus[(int64_t)qp * e + i] = qsm[D.by + i];
        if (tid == 0) { iters_out[qp] = iters_run; resid_out[qp] = best; }
    }
    f.sync();
}

// QPFunctionFn.backward (qp.py:128-182) for the box QP: d from the clamped duals (qp.py:148), one factor of M and one
// solve per QP, then dq = dx o z, dp = dx, dlb = dlam_lb, dub = -dlam_ub, dA = dnu z' + nu dx', db = -dnu. dxv, dlamv
// and dnuv always receive dx, dlam, dnu (the batch means read them); a gradient whose mean flag is set is skipped here.
// Every CTA writes its slice of dx, dlam, dq, dp, dlb, dub and its columns of dA; the leader dnu and db. dl_dlam and dl_dnu
// (NULL: zero) are the adjoints of the returned duals: they are the rz and ry of the solve, which rz / ry are not otherwise.
struct BoxGrads {
    double *dq, *dp, *dlb, *dub, *dA, *db;
    int mq, mp, mlb, mub, mA, mb;
};

template <class F>
__global__ void __launch_bounds__(kBoxNT, F::kMinBwd)
k_box_backward(typename F::Dims P, const double* __restrict__ q, int64_t sq, const double* __restrict__ A, int64_t sA,
               const double* __restrict__ dl, const double* __restrict__ dl_dlam, const double* __restrict__ dl_dnu,
               const double* __restrict__ zhat, const double* __restrict__ lam,
               const double* __restrict__ slacks, const double* __restrict__ nus, BoxGrads O,
               double* __restrict__ dxv, double* __restrict__ dlamv, double* __restrict__ dnuv) {
    QPB_SMEM;
    F f(P);
    const BoxDims& D = f.D;
    const int tid = threadIdx.x, qp = f.qp(), j0 = f.j0();
    const int n = D.n, m = D.m, e = D.e, N = f.ng();
    f.stage(q + (int64_t)qp * sq, A + (int64_t)qp * sA, nullptr);
    for (int j = tid; j < n; j += kBoxNT) qsm[D.rx + j] = dl[(int64_t)qp * N + j0 + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * f.mg() + f.grow(i);
        qsm[D.d + i] = fmax(lam[g], 1e-8) / fmax(slacks[g], 1e-8);
        if (dl_dlam != nullptr) qsm[D.rz + i] = dl_dlam[g];
    }
    // every CTA loads all of dl_dnu: the right-hand side of M stays bit-identical across the cluster (see k_box_forward)
    if (dl_dnu != nullptr)
        for (int i = tid; i < e; i += kBoxNT) qsm[D.ry + i] = dl_dnu[(int64_t)qp * e + i];
    __syncthreads();
    f.form();
    box_solve(f, true, D.rx, -1, dl_dlam != nullptr ? D.rz : -1, dl_dnu != nullptr ? D.ry : -1, D.dx, D.ds, D.dz, D.dy);
    for (int j = tid; j < n; j += kBoxNT) {
        const int64_t g = (int64_t)qp * N + j0 + j;
        const double dx = qsm[D.dx + j], z = zhat[g];
        dxv[g] = dx;
        if (O.dq && !O.mq) O.dq[g] = dx * z;
        if (O.dp && !O.mp) O.dp[g] = dx;
    }
    for (int i = tid; i < m; i += kBoxNT) {
        const double dz = qsm[D.dz + i];
        dlamv[(int64_t)qp * f.mg() + f.grow(i)] = dz;
        if (i < D.nlb) { if (O.dlb && !O.mlb) O.dlb[(int64_t)qp * N + j0 + i] = dz; }
        else if (O.dub && !O.mub) O.dub[(int64_t)qp * N + j0 + i - D.nlb] = -dz;
    }
    if (f.leader())
        for (int i = tid; i < e; i += kBoxNT) {
            dnuv[(int64_t)qp * e + i] = qsm[D.dy + i];
            if (O.db && !O.mb) O.db[(int64_t)qp * e + i] = -qsm[D.dy + i];
        }
    if (O.dA && !O.mA)
        for (int t = tid; t < e * n; t += kBoxNT) {
            const int i = t / n, j = t - i * n;
            O.dA[((int64_t)qp * e + i) * N + j0 + j] = fma(qsm[D.dy + i], zhat[(int64_t)qp * N + j0 + j],
                                                           nus[(int64_t)qp * e + i] * qsm[D.dx + j]);
        }
    f.sync();
}

// qpb200_box_solve_kkt: the structured factor and solve for caller-given d and right-hand sides (all vectors (B, len))
template <class F>
__global__ void __launch_bounds__(kBoxNT, F::kMinKkt)
k_box_kkt(typename F::Dims P, const double* __restrict__ q, int64_t sq, const double* __restrict__ A, int64_t sA,
          const double* __restrict__ d, const double* __restrict__ rx, const double* __restrict__ rs,
          const double* __restrict__ rz, const double* __restrict__ ry, double* __restrict__ dx, double* __restrict__ ds,
          double* __restrict__ dz, double* __restrict__ dy) {
    QPB_SMEM;
    F f(P);
    const BoxDims& D = f.D;
    const int tid = threadIdx.x, qp = f.qp(), j0 = f.j0();
    const int n = D.n, m = D.m, e = D.e, N = f.ng();
    f.stage(q + (int64_t)qp * sq, A + (int64_t)qp * sA, nullptr);
    for (int j = tid; j < n; j += kBoxNT) qsm[D.rx + j] = rx[(int64_t)qp * N + j0 + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * f.mg() + f.grow(i);
        qsm[D.d + i] = d[g];
        qsm[D.rsc + i] = rs[g];
        qsm[D.rz + i] = rz[g];
    }
    for (int i = tid; i < e; i += kBoxNT) qsm[D.ry + i] = ry[(int64_t)qp * e + i];
    __syncthreads();
    f.form();
    box_solve(f, true, D.rx, D.rsc, D.rz, D.ry, D.dx, D.ds, D.dz, D.dy);
    for (int j = tid; j < n; j += kBoxNT) dx[(int64_t)qp * N + j0 + j] = qsm[D.dx + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * f.mg() + f.grow(i);
        ds[g] = qsm[D.ds + i];
        dz[g] = qsm[D.dz + i];
    }
    if (dy != nullptr && f.leader())
        for (int i = tid; i < e; i += kBoxNT) dy[(int64_t)qp * e + i] = qsm[D.dy + i];
    f.sync();
}

// ---- distributed-M kernels: neq_pad > 128 on a cluster ---------------------------------------------------------------
// Past neq_pad = 128 a full copy of M per CTA no longer fits (the staircase of order 256 alone is 272 KB). These kernels
// keep the variable slices, the reductions, the Mehrotra loop and the invariant of the cluster kernels above, but M is
// DISTRIBUTED: block row i of the staircase (8 rows, columns 0 .. 8i+7) lives on rank i mod C, which balances both the
// storage and the trailing-update work. A is read from global memory (a shared A stays in L2 for the whole batch).
//   form:     the full H^-1 is gathered from the slices; column chunks of A are staged through shared memory and every
//             CTA forms its own block rows, M_ij = sum_v A_iv h_v A_jv, with DMMA 8x8x4.
//   factor:   pf_chol's steps. F_k: the owner of block row k factors the diagonal tile and publishes T_k there. After a
//             cluster barrier, S_k: every CTA forms L_ik (into its panel rows) and P_ik for its own block rows and
//             sweeps its rows of the running right-hand side with b_k. After a second barrier, U_k: every CTA copies the
//             panel rows of the other ranks that its trailing tiles need and updates its own tiles.
//   sweeps:   forward (corrector): one barrier per block step, after which b_k is final on its owner. pf_diag: local.
//             Backward: one barrier per block step; each CTA adds P_ik' w_i of its own block rows into a partial, and
//             the owner of block k sums the partials in rank order. Then dy is gathered into every CTA.
// dy is computed once, by the owners of its blocks, and copied: every CTA holds it bit for bit, so everything derived
// from it is cluster-wide and the branch rule of the cluster kernels holds unchanged.
struct DmDims {
    ClDims X;                // slices and reductions; X.L.S: this CTA's block rows, X.L.pan: panel rows of all of M
    int nts;                 // block rows of M
    int hfull, Tk, cv, part, wpub, As;   // full H^-1, T_k and b_k, pf_diag output, backward partial, w blocks, A chunk
    int total;               // doubles per CTA (the rank with the largest share of M)
};
constexpr int kDmKC = 16;                // columns of A per staged chunk
constexpr int kDmLdA = kDmKC + 4;        // row stride of the chunk (== 4 mod 16: conflict-free DMMA fragment reads)
constexpr int kDmDenseOrder = 384;       // dense order ms_pad past which they are chosen (H100: parity at 384, 2.2x at 504)

// local offset of the li-th own block row (block i = rank + C li, 8 (8i + 12) doubles each) and own block-row count
__host__ __device__ inline int dm_boff(int C, int rank, int li) { return 64 * rank * li + 32 * C * li * (li - 1) + 96 * li; }
__host__ __device__ inline int dm_nblk(int nts, int C, int rank) { return rank < nts ? (nts - rank + C - 1) / C : 0; }
// first own block row below block k
__device__ __forceinline__ int dm_below(int C, int rank, int k) { return (k >= rank) ? (k - rank) / C + 1 : 0; }

__host__ __device__ inline DmDims dm_dims(int n, int e, int has_lb, int has_ub, int C) {
    DmDims Y;
    ClDims& X = Y.X;
    cl_slices(X, n, has_lb, has_ub, C);
    BoxDims& D = X.L;
    D.n = X.slice; D.e = e; D.ep = r8(e);
    D.nlb = has_lb ? X.slice : 0; D.m = (has_lb ? X.slice : 0) + (has_ub ? X.slice : 0);
    D.lda = 0; D.A = 0; D.tab = 0; D.red = 0;           // (A is not staged; no tile table, no block reductions)
    Y.nts = D.ep >> 3;
    int stair = 0;
    for (int r = 0; r < C; ++r) {
        const int s = dm_boff(C, r, dm_nblk(Y.nts, C, r));
        stair = s > stair ? s : stair;
    }
    int o = 0;
    D.S = o; o += r8(stair);
    D.pan = o; o += 8 * Y.nts * kPanLd;
    o = box_vectors(D, o);
    D.total = o;
    X.Mp = 0;
    X.pb = r8(D.ep + 4 * kClW);
    X.pub = o; o += 2 * X.pb;
    Y.hfull = o; o += r8(n) + kDmKC;                     // zero past n: the last chunk reads it
    Y.Tk = o; o += 72;                                   // T_k (64, upper part zero), then b_k (8)
    Y.cv = o; o += D.ep;
    Y.part = o; o += D.ep;
    Y.wpub = o; o += D.ep;
    Y.As = o; o += D.ep * kDmLdA;
    X.total = Y.total = o;
    return Y;
}

// hinv for this CTA's variables, the gathered full H^-1, and this CTA's block rows of M (identity rows beyond neq).
// One cluster barrier; ends with a block barrier.
__device__ __noinline__ void dm_form(const DmDims& Y, const BoxDims& D, int rank, const double* __restrict__ Ag) {
    QPB_SMEM;
    cg::cluster_group cl = cg::this_cluster();
    const ClDims& X = Y.X;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
    const int N = X.ng, e = D.e, C = X.C, nb = dm_nblk(Y.nts, C, rank);
    for (int j = tid; j < D.n; j += kBoxNT) {
        double hj = qsm[D.q + j];
        if (D.nlb) hj += qsm[D.d + j];
        if (D.m > D.nlb) hj += qsm[D.d + D.nlb + j];
        qsm[D.hinv + j] = 1.0 / hj;
    }
    cl.sync();                                           // every slice of H^-1 is published
    for (int v = tid; v < r8(N) + kDmKC; v += kBoxNT)
        qsm[Y.hfull + v] = (v < N) ? cl.map_shared_rank(qsm + D.hinv, v / X.slice)[v % X.slice] : 0.0;
    double* S = qsm + D.S;
    const double* As = qsm + Y.As;
    const double* hf = qsm + Y.hfull;
    for (int v0 = 0; v0 < N; v0 += kDmKC) {
        __syncthreads();                                 // the previous chunk is consumed (first: H^-1 is gathered)
        for (int t = tid; t < D.ep * kDmKC; t += kBoxNT) {
            const int r = t / kDmKC, c = t - r * kDmKC, v = v0 + c;
            qsm[Y.As + r * kDmLdA + c] = (r < e && v < N) ? Ag[(int64_t)r * N + v] : 0.0;
        }
        __syncthreads();
        // own tiles (i, j), j <= i, dealt round-robin over the warps (cnt is warp-uniform)
        int cnt = 0;
        for (int li = 0; li < nb; ++li) {
            const int i = rank + C * li;
            double* rowp = S + dm_boff(C, rank, li) + g * (8 * i + 12) + 2 * q;
            const double* ai = As + (8 * i + g) * kDmLdA + q;
            for (int j = 0; j <= i; ++j, ++cnt) {
                if ((cnt & (kClW - 1)) != warp) continue;
                double2 acc = (v0 == 0) ? make_double2(0.0, 0.0) : *reinterpret_cast<const double2*>(rowp + 8 * j);
                const double* aj = As + (8 * j + g) * kDmLdA + q;
#pragma unroll
                for (int kk = 0; kk < kDmKC; kk += 4) qpb::dmma884(acc.x, acc.y, ai[kk] * hf[v0 + kk + q], aj[kk]);
                *reinterpret_cast<double2*>(rowp + 8 * j) = acc;
            }
        }
    }
    __syncthreads();
    for (int t = tid; t < 8 * nb; t += kBoxNT) {
        const int li = t >> 3, i = rank + C * li, r = 8 * i + (t & 7);
        if (r >= e) S[dm_boff(C, rank, li) + (t & 7) * (8 * i + 12) + r] = 1.0;
    }
    __syncthreads();
}

// pf_chol over the cluster, with the running right-hand side b (offset; this CTA's block rows are meaningful) carried
// along. 2 nts - 1 cluster barriers; ends with a block barrier.
__device__ __noinline__ void dm_chol(const DmDims& Y, const BoxDims& D, int rank, int b) {
    QPB_SMEM;
    cg::cluster_group cl = cg::this_cluster();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, q = lane & 3;
    const int C = Y.X.C, nts = Y.nts, nb = dm_nblk(nts, C, rank);
    double* S = qsm + D.S;
    double* P = qsm + D.pan;
    double* Tk = qsm + Y.Tk;
#pragma unroll 1
    for (int k = 0; k < nts; ++k) {
        const int k0 = 8 * k, own = k % C, lk = k / C, ldk = 8 * k + 12;
        if (rank == own && warp == 0) {                  // F_k
            double* Mb = S + dm_boff(C, rank, lk) + k0;
            double Lk[36], Tc[8];
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int c = 0; c <= r; ++c) Lk[QPB_LIDX(r, c)] = Mb[r * ldk + c];
            __syncwarp();
            pf_factor8(Lk);
            pf_inv8_col(Lk, lane & 7, Tc);
            if (lane < 8) {
#pragma unroll
                for (int r = 0; r < 8; ++r)
                    if (r >= lane) Mb[r * ldk + lane] = Tc[r];
            }
        }
        cl.sync();                                       // T_k and b_k are final on their owner
        {
            const double* Mo = cl.map_shared_rank(S, own) + dm_boff(C, own, lk) + k0;
            for (int t = tid; t < 64; t += kBoxNT) {
                const int r = t >> 3, c = t & 7;
                Tk[t] = (c <= r) ? Mo[r * ldk + c] : 0.0;
            }
            if (tid < 8) Tk[64 + tid] = cl.map_shared_rank(qsm + b, own)[k0 + tid];
        }
        __syncthreads();
        const int lo = dm_below(C, rank, k);
        {                                                // S_k: one own block row per warp
            const double bT0 = Tk[g * 8 + q], bT1 = Tk[g * 8 + q + 4];      // T[g][q], T[g][q+4]
            const double bP0 = Tk[q * 8 + g], bP1 = Tk[(q + 4) * 8 + g];    // T[q][g], T[q+4][g]
#pragma unroll 1
            for (int li = lo + warp; li < nb; li += kClW) {
                const int i = rank + C * li;
                double* row = S + dm_boff(C, rank, li) + g * (8 * i + 12) + k0;
                const double a0 = row[q], a1 = row[q + 4];
                double d0 = 0.0, d1 = 0.0;
                qpb::dmma884(d0, d1, a0, bT0);
                qpb::dmma884(d0, d1, a1, bT1);
                double* pl = P + (8 * i + g) * kPanLd;
                *reinterpret_cast<double2*>(pl + 2 * q) = make_double2(d0, d1);
                __syncwarp();
                const double la0 = pl[q], la1 = pl[q + 4];
                double e0 = 0.0, e1 = 0.0;
                qpb::dmma884(e0, e1, la0, bP0);
                qpb::dmma884(e0, e1, la1, bP1);
                *reinterpret_cast<double2*>(row + 2 * q) = make_double2(e0, e1);
            }
        }
        __syncthreads();
        for (int t = 8 * lo + tid; t < 8 * nb; t += kBoxNT) {       // b_r -= P[r][k0 .. k0+7] . b_k, own rows below k
            const int li = t >> 3, i = rank + C * li, rr = t & 7;
            const double* pr = S + dm_boff(C, rank, li) + rr * (8 * i + 12) + k0;
            double s0 = qsm[b + 8 * i + rr], s1 = 0.0;
#pragma unroll
            for (int c = 0; c < 8; c += 2) { s0 = fma(-pr[c], Tk[64 + c], s0); s1 = fma(-pr[c + 1], Tk[65 + c], s1); }
            qsm[b + 8 * i + rr] = s0 + s1;
        }
        if (k + 1 == nts) break;
        cl.sync();                                       // every panel row of step k is written
        const int nj = (nb > 0) ? rank + C * (nb - 1) - k : 0;       // block rows k+1 .. this CTA's last one
        for (int t = tid; t < 64 * nj; t += kBoxNT) {
            const int j = k + 1 + (t >> 6), o = (8 * j + ((t >> 3) & 7)) * kPanLd + (t & 7);
            if (j % C != rank) P[o] = cl.map_shared_rank(P, j % C)[o];
        }
        __syncthreads();
        int cnt = 0;                                     // U_k: own tiles (i, j), k < j <= i, round-robin
#pragma unroll 1
        for (int li = lo; li < nb; ++li) {
            const int i = rank + C * li;
            double* rowp = S + dm_boff(C, rank, li) + g * (8 * i + 12) + 2 * q;
            const double la0 = P[(8 * i + g) * kPanLd + q], la1 = P[(8 * i + g) * kPanLd + q + 4];
#pragma unroll 1
            for (int j = k + 1; j <= i; ++j, ++cnt) {
                if ((cnt & (kClW - 1)) != warp) continue;
                double2 v = *reinterpret_cast<const double2*>(rowp + 8 * j);
                const double* pb = P + (8 * j + g) * kPanLd + q;
                qpb::dmma884(v.x, v.y, -la0, pb[0]);
                qpb::dmma884(v.x, v.y, -la1, pb[4]);
                *reinterpret_cast<double2*>(rowp + 8 * j) = v;
            }
        }
        __syncthreads();
    }
    __syncthreads();
}

// pf_fwd over the cluster with an existing factor: b_i -= P_ik b_k. nts - 1 cluster barriers; ends with a block barrier.
__device__ __noinline__ void dm_fwd(const DmDims& Y, const BoxDims& D, int rank, int b) {
    QPB_SMEM;
    cg::cluster_group cl = cg::this_cluster();
    const int tid = threadIdx.x, C = Y.X.C, nts = Y.nts, nb = dm_nblk(nts, C, rank);
    const double* S = qsm + D.S;
#pragma unroll 1
    for (int k = 0; k + 1 < nts; ++k) {
        cl.sync();                                       // b_k is final on its owner
        const double* bk = cl.map_shared_rank(qsm + b, k % C) + 8 * k;
        for (int t = 8 * dm_below(C, rank, k) + tid; t < 8 * nb; t += kBoxNT) {
            const int li = t >> 3, i = rank + C * li, rr = t & 7;
            const double* pr = S + dm_boff(C, rank, li) + rr * (8 * i + 12) + 8 * k;
            double s0 = qsm[b + 8 * i + rr], s1 = 0.0;
#pragma unroll
            for (int c = 0; c < 8; c += 2) { s0 = fma(-pr[c], bk[c], s0); s1 = fma(-pr[c + 1], bk[c + 1], s1); }
            qsm[b + 8 * i + rr] = s0 + s1;
        }
    }
    __syncthreads();
}

// pf_diag on this CTA's block rows: c_k = T_k^T (T_k b_k), with y a scratch vector. c != b (other CTAs may still read b).
// Ends with a block barrier.
__device__ __noinline__ void dm_diag(const DmDims& Y, const BoxDims& D, int rank, int b, int y, int c) {
    QPB_SMEM;
    const int tid = threadIdx.x, C = Y.X.C, nb = dm_nblk(Y.nts, C, rank);
    const double* S = qsm + D.S;
    for (int t = tid; t < 8 * nb; t += kBoxNT) {
        const int li = t >> 3, i = rank + C * li, r = t & 7, ld = 8 * i + 12;
        const double* Tr = S + dm_boff(C, rank, li) + r * ld + 8 * i;       // row r of T_k
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int cc = 0; cc < 8; cc += 2) {
            s0 = fma((cc <= r) ? Tr[cc] : 0.0, (cc <= r) ? qsm[b + 8 * i + cc] : 0.0, s0);
            s1 = fma((cc + 1 <= r) ? Tr[cc + 1] : 0.0, (cc + 1 <= r) ? qsm[b + 8 * i + cc + 1] : 0.0, s1);
        }
        qsm[y + 8 * i + r] = s0 + s1;
    }
    __syncthreads();
    for (int t = tid; t < 8 * nb; t += kBoxNT) {
        const int li = t >> 3, i = rank + C * li, r = t & 7, ld = 8 * i + 12;
        const double* Tc = S + dm_boff(C, rank, li) + 8 * i + r;            // column r of T_k: T[j][r] at Tc[j ld]
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            s0 = fma((j >= r) ? Tc[j * ld] : 0.0, (j >= r) ? qsm[y + 8 * i + j] : 0.0, s0);
            s1 = fma((j + 1 >= r) ? Tc[(j + 1) * ld] : 0.0, (j + 1 >= r) ? qsm[y + 8 * i + j + 1] : 0.0, s1);
        }
        qsm[c + 8 * i + r] = s0 + s1;
    }
    __syncthreads();
}

// pf_bwd over the cluster: w_k = c_k - sum_{i>k} P_ik' w_i, then w gathered into every CTA (offset w, length ep).
// nts + 1 cluster barriers; ends with a block barrier.
__device__ __noinline__ void dm_bwd(const DmDims& Y, const BoxDims& D, int rank, int c, int w) {
    QPB_SMEM;
    cg::cluster_group cl = cg::this_cluster();
    const int tid = threadIdx.x, C = Y.X.C, nts = Y.nts, ep = D.ep;
    const double* S = qsm + D.S;
    double* part = qsm + Y.part;
    double* wp = qsm + Y.wpub;
    for (int t = tid; t < ep; t += kBoxNT) part[t] = 0.0;
#pragma unroll 1
    for (int i = nts - 1; i >= 0; --i) {
        cl.sync();                                       // every partial holds the block rows below i
        if (rank == i % C) {                             // (CTA-uniform)
            const int i0 = 8 * i, ld = 8 * i + 12;
            if (tid < 8) {
                double s = qsm[c + i0 + tid];
                for (int r = 0; r < C; ++r) s -= cl.map_shared_rank(part, r)[i0 + tid];
                wp[i0 + tid] = s;
            }
            __syncthreads();
            const double* blk = S + dm_boff(C, rank, i / C);
            for (int t = tid; t < i0; t += kBoxNT) {
                double s0 = part[t], s1 = 0.0;
#pragma unroll
                for (int rr = 0; rr < 8; rr += 2) {
                    s0 = fma(blk[rr * ld + t], wp[i0 + rr], s0);
                    s1 = fma(blk[(rr + 1) * ld + t], wp[i0 + rr + 1], s1);
                }
                part[t] = s0 + s1;
            }
        }
    }
    cl.sync();                                           // every block of w is final on its owner
    for (int t = tid; t < ep; t += kBoxNT) qsm[w + t] = cl.map_shared_rank(wp, (t >> 3) % C)[t];
    __syncthreads();
}

// box_solve<Cluster> with M distributed (Ag: this QP's A in global memory). Ends with a block barrier.
__device__ __noinline__ void dm_solve(const DmDims& Y, const BoxDims& D, int rank, const double* __restrict__ Ag, int j0,
                                      int& ph, bool fresh, int rx, int rs, int rz, int ry, int dx, int ds, int dz, int dy) {
    QPB_SMEM;
    cg::cluster_group cl = cg::this_cluster();
    const ClDims& X = Y.X;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, N = X.ng;
    for (int j = tid; j < n; j += kBoxNT) {
        double a = qsm[rx + j];
        if (D.nlb) {
            const double t = ((rz >= 0) ? qsm[D.d + j] * qsm[rz + j] : 0.0) - ((rs >= 0) ? qsm[rs + j] : 0.0);
            a -= t;
        }
        if (m > D.nlb) {
            const int i = D.nlb + j;
            const double t = ((rz >= 0) ? qsm[D.d + i] * qsm[rz + i] : 0.0) - ((rs >= 0) ? qsm[rs + i] : 0.0);
            a += t;
        }
        qsm[D.r + j] = a * qsm[D.hinv + j];
    }
    __syncthreads();
    const int buf = cl_buf(X, ph);
    for (int i = warp; i < e; i += kClW) {
        double a = 0.0;
        for (int k = lane; k < n; k += 32) a = fma(Ag[(int64_t)i * N + j0 + k], qsm[D.r + k], a);
        a = qpb::warp_sum(a);
        if (lane == 0) qsm[buf + i] = a;
    }
    cl.sync();                                           // the partials of A H^-1 r are published
    for (int i = tid; i < ep; i += kBoxNT) {
        double a = 0.0;
        if (i < e)
            for (int k = 0; k < X.C; ++k) a += cl.map_shared_rank(qsm + buf, k)[i];
        qsm[D.rhs + i] = (i < e) ? (((ry >= 0) ? qsm[ry + i] : 0.0) - a) : 0.0;
    }
    ++ph;
    __syncthreads();
    if (fresh) dm_chol(Y, D, rank, D.rhs);
    else dm_fwd(Y, D, rank, D.rhs);
    dm_diag(Y, D, rank, D.rhs, D.t, Y.cv);
    dm_bwd(Y, D, rank, Y.cv, dy);
    for (int j = tid; j < n; j += kBoxNT) {
        double a = 0.0;
        for (int i = 0; i < e; ++i) a = fma(Ag[(int64_t)i * N + j0 + j], qsm[dy + i], a);
        qsm[dx + j] = -qsm[D.r + j] - a * qsm[D.hinv + j];
    }
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

// q (this CTA's slice) and b (replicated; forward only)
__device__ __forceinline__ void dm_stage(const BoxDims& D, int j0, const double* q, const double* b) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    for (int j = tid; j < D.n; j += kBoxNT) qsm[D.q + j] = q[j0 + j];
    for (int i = tid; i < D.ep; i += kBoxNT) qsm[D.b + i] = (b != nullptr && i < D.e) ? b[i] : 0.0;
    __syncthreads();
}

// k_box_forward<Cluster> with M distributed (outputs as there)
__global__ void __launch_bounds__(kBoxNT, 1)
k_box_forward_dm(DmDims Y, const double* __restrict__ q, int64_t sq, const double* __restrict__ p, int64_t sp,
                 const double* __restrict__ A, int64_t sA, const double* __restrict__ b, int64_t sb,
                 const double* __restrict__ lb, int64_t slb, const double* __restrict__ ub, int64_t sub, double eps,
                 double stall_tol, double best_tie, int notImprovedLim, int maxIter, double* __restrict__ zhat,
                 double* __restrict__ lam, double* __restrict__ slacks, double* __restrict__ nus,
                 int* __restrict__ iters_out, double* __restrict__ resid_out, double* __restrict__ trace,
                 int* __restrict__ spd_flag) {
    QPB_SMEM;
    const ClDims& X = Y.X;
    const int rank = (int)cg::this_cluster().block_rank();
    const int tid = threadIdx.x, qp = blockIdx.x / X.C;
    int j0, ph = 0;
    const BoxDims D = cl_local(X, rank, j0);
    const int n = D.n, m = D.m, e = D.e, ep = D.ep, N = X.ng;
    const double* Ag = A + (int64_t)qp * sA;
    dm_stage(D, j0, q + (int64_t)qp * sq, b + (int64_t)qp * sb);
    {
        double bad[1] = {0.0};
        for (int j = tid; j < n; j += kBoxNT) {
            qsm[D.p + j] = p[(int64_t)qp * sp + j0 + j];
            if (!(qsm[D.q + j] > 0.0)) bad[0] = 1.0;
        }
        cl_reduce<1, false>(X, bad, ph, 0, 0);
        if (rank == 0 && tid == 0 && spd_flag != nullptr) spd_flag[qp] = bad[0] > 0.0;
    }
    for (int i = tid; i < m; i += kBoxNT) {
        qsm[D.h + i] = (i < D.nlb) ? -lb[(int64_t)qp * slb + j0 + i] : ub[(int64_t)qp * sub + j0 + i - D.nlb];
        qsm[D.d + i] = 1.0;
        qsm[D.rz + i] = -qsm[D.h + i];
    }
    for (int i = tid; i < ep; i += kBoxNT) { qsm[D.ry + i] = -qsm[D.b + i]; qsm[D.y + i] = 0.0; }
    __syncthreads();

    // ---- initial point: solve_kkt(p, 0, -h, -b) with d = 1   (batch.py:61-67)
    dm_form(Y, D, rank, Ag);
    dm_solve(Y, D, rank, Ag, j0, ph, true, D.p, -1, D.rz, D.ry, D.x, D.s, D.z, D.y);
    {
        double mn[2] = {INFINITY, INFINITY};
        for (int i = tid; i < m; i += kBoxNT) { mn[0] = fmin(mn[0], qsm[D.s + i]); mn[1] = fmin(mn[1], qsm[D.z + i]); }
        cl_reduce<2, true>(X, mn, ph, 0, 0);
        for (int i = tid; i < m; i += kBoxNT) {                  // slacks and duals >= 1 (batch.py:77-87)
            if (mn[0] < 0.0) qsm[D.s + i] -= mn[0] - 1.0;
            if (mn[1] < 0.0) qsm[D.z + i] -= mn[1] - 1.0;
        }
        __syncthreads();
    }

    double best = 0.0;
    int nNot = 0, iters_run = 0;
    const double dm = (double)X.mg;
    for (int it = 0; it < maxIter; ++it) {
        iters_run = it + 1;
        // ---- residuals (batch.py:94-107): A x is reduced with the scalars, ry and |ry|^2 are formed redundantly
        double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // |ry|^2, |rz|^2, |rx|^2, s.z
        for (int j = tid; j < n; j += kBoxNT) {
            double a = 0.0;
            for (int i = 0; i < e; ++i) a = fma(Ag[(int64_t)i * N + j0 + j], qsm[D.y + i], a);
            const double r = fma(qsm[D.q + j], qsm[D.x + j], qsm[D.p + j]) + gt_col(D, qsm + D.z, j) + a;
            qsm[D.rx + j] = r;
            acc[2] = fma(r, r, acc[2]);
        }
        for (int i = tid; i < m; i += kBoxNT) {
            const double r = bsgn(D, i) * qsm[D.x + bvar(D, i)] + qsm[D.s + i] - qsm[D.h + i];
            qsm[D.rz + i] = r;
            acc[1] = fma(r, r, acc[1]);
            acc[3] = fma(qsm[D.s + i], qsm[D.z + i], acc[3]);
        }
        {
            const int lane = tid & 31, warp = tid >> 5, buf = cl_buf(X, ph);
            for (int i = warp; i < e; i += kClW) {
                double a = 0.0;
                for (int k = lane; k < n; k += 32) a = fma(Ag[(int64_t)i * N + j0 + k], qsm[D.x + k], a);
                a = qpb::warp_sum(a);
                if (lane == 0) qsm[buf + i] = a;
            }
        }
        cl_reduce<4, false>(X, acc, ph, e, D.ry);
        for (int i = 0; i < e; ++i) {
            const double r = qsm[D.ry + i] - qsm[D.b + i];
            acc[0] = fma(r, r, acc[0]);
        }
        __syncthreads();                                         // every thread has read the sums of A x
        for (int i = tid; i < ep; i += kBoxNT) qsm[D.ry + i] = (i < e) ? qsm[D.ry + i] - qsm[D.b + i] : 0.0;
        const double mu = fabs(acc[3] / dm);
        const double resid = sqrt(acc[1]) + sqrt(acc[0]) + sqrt(acc[2]) + dm * mu;
        if (trace != nullptr && rank == 0 && tid == 0) {          // what verbose=1 prints (batch.py:115-117)
            double* tr = trace + ((int64_t)qp * maxIter + it) * 4;
            tr[0] = sqrt(acc[1]) + sqrt(acc[0]); tr[1] = sqrt(acc[2]); tr[2] = mu; tr[3] = resid;
        }
        // ---- best-iterate tracking and exit tests (batch.py:118-143), per QP: cluster-wide values only
        const bool improved = (it == 0) || (resid < best);
        if (improved) { best = resid; nNot = 0; } else { ++nNot; }
        if (improved || resid < best_tie * best) {
            for (int j = tid; j < n; j += kBoxNT) qsm[D.bx + j] = qsm[D.x + j];
            for (int i = tid; i < m; i += kBoxNT) { qsm[D.bs + i] = qsm[D.s + i]; qsm[D.bz + i] = qsm[D.z + i]; }
            for (int i = tid; i < e; i += kBoxNT) qsm[D.by + i] = qsm[D.y + i];
        }
        if ((nNot == notImprovedLim && best < stall_tol) || best < eps || mu > 1e32) break;
        if (!(resid == resid) || isinf(resid)) break;
        // ---- d = z/s, H, M; the affine direction (batch.py:109-113,150) factors M
        for (int i = tid; i < m; i += kBoxNT) qsm[D.d + i] = qsm[D.z + i] / qsm[D.s + i];
        __syncthreads();
        dm_form(Y, D, rank, Ag);
        dm_solve(Y, D, rank, Ag, j0, ph, true, D.rx, D.z, D.rz, D.ry, D.dxa, D.dsa, D.dza, D.dya);
        // ---- affine step length and sigma (batch.py:160-168)
        double mn[2] = {INFINITY, INFINITY};
        for (int i = tid; i < m; i += kBoxNT) {
            mn[0] = fmin(mn[0], box_step(qsm[D.z + i], qsm[D.dza + i]));
            mn[1] = fmin(mn[1], box_step(qsm[D.s + i], qsm[D.dsa + i]));
        }
        cl_reduce<2, true>(X, mn, ph, 0, 0);
        {
            const double alpha = fmin(fmin(box_step_fix(mn[0]), box_step_fix(mn[1])), 1.0);
            double sm[2] = {0.0, 0.0};
            for (int i = tid; i < m; i += kBoxNT) {
                sm[0] = fma(qsm[D.s + i] + alpha * qsm[D.dsa + i], qsm[D.z + i] + alpha * qsm[D.dza + i], sm[0]);
                sm[1] = fma(qsm[D.s + i], qsm[D.z + i], sm[1]);
            }
            cl_reduce<2, false>(X, sm, ph, 0, 0);
            const double sr = sm[0] / sm[1];
            const double sig = sr * sr * sr;
            // ---- corrector right-hand side (batch.py:170-181): rs = (-mu sig + dsa dza) / s, rx = rz = ry = 0
            for (int i = tid; i < m; i += kBoxNT)
                qsm[D.rsc + i] = (-mu * sig + qsm[D.dsa + i] * qsm[D.dza + i]) / qsm[D.s + i];
            for (int j = tid; j < n; j += kBoxNT) qsm[D.rx + j] = 0.0;
            __syncthreads();
        }
        dm_solve(Y, D, rank, Ag, j0, ph, false, D.rx, D.rsc, -1, -1, D.dx, D.ds, D.dz, D.dy);
        // ---- combined direction, step length, update (batch.py:185-203)
        mn[0] = INFINITY; mn[1] = INFINITY;
        for (int i = tid; i < m; i += kBoxNT) {
            const double dzi = qsm[D.dza + i] + qsm[D.dz + i], dsi = qsm[D.dsa + i] + qsm[D.ds + i];
            qsm[D.dz + i] = dzi;
            qsm[D.ds + i] = dsi;
            mn[0] = fmin(mn[0], box_step(qsm[D.z + i], dzi));
            mn[1] = fmin(mn[1], box_step(qsm[D.s + i], dsi));
        }
        cl_reduce<2, true>(X, mn, ph, 0, 0);
        const double alpha = fmin(0.999 * fmin(box_step_fix(mn[0]), box_step_fix(mn[1])), 1.0);
        for (int j = tid; j < n; j += kBoxNT) qsm[D.x + j] = fma(alpha, qsm[D.dxa + j] + qsm[D.dx + j], qsm[D.x + j]);
        for (int i = tid; i < m; i += kBoxNT) {
            qsm[D.s + i] = fma(alpha, qsm[D.ds + i], qsm[D.s + i]);
            qsm[D.z + i] = fma(alpha, qsm[D.dz + i], qsm[D.z + i]);
        }
        for (int i = tid; i < e; i += kBoxNT) qsm[D.y + i] = fma(alpha, qsm[D.dya + i] + qsm[D.dy + i], qsm[D.y + i]);
        __syncthreads();
    }
    __syncthreads();
    for (int j = tid; j < n; j += kBoxNT) zhat[(int64_t)qp * N + j0 + j] = qsm[D.bx + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * X.mg + cl_grow(X, D, j0, i);
        lam[g] = qsm[D.bz + i];
        slacks[g] = qsm[D.bs + i];
    }
    if (rank == 0) {
        for (int i = tid; i < e; i += kBoxNT) nus[(int64_t)qp * e + i] = qsm[D.by + i];
        if (tid == 0) { iters_out[qp] = iters_run; resid_out[qp] = best; }
    }
    cg::this_cluster().sync();       // no CTA exits while another may still read its shared memory
}

// k_box_backward<Cluster> with M distributed
__global__ void __launch_bounds__(kBoxNT, 1)
k_box_backward_dm(DmDims Y, const double* __restrict__ q, int64_t sq, const double* __restrict__ A, int64_t sA,
                  const double* __restrict__ dl, const double* __restrict__ dl_dlam,
                  const double* __restrict__ dl_dnu, const double* __restrict__ zhat, const double* __restrict__ lam,
                  const double* __restrict__ slacks, const double* __restrict__ nus, BoxGrads O,
                  double* __restrict__ dxv, double* __restrict__ dlamv, double* __restrict__ dnuv) {
    QPB_SMEM;
    const ClDims& X = Y.X;
    const int rank = (int)cg::this_cluster().block_rank();
    const int tid = threadIdx.x, qp = blockIdx.x / X.C;
    int j0, ph = 0;
    const BoxDims D = cl_local(X, rank, j0);
    const int n = D.n, m = D.m, e = D.e, N = X.ng;
    const double* Ag = A + (int64_t)qp * sA;
    dm_stage(D, j0, q + (int64_t)qp * sq, nullptr);
    for (int j = tid; j < n; j += kBoxNT) qsm[D.rx + j] = dl[(int64_t)qp * N + j0 + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * X.mg + cl_grow(X, D, j0, i);
        qsm[D.d + i] = fmax(lam[g], 1e-8) / fmax(slacks[g], 1e-8);
        if (dl_dlam != nullptr) qsm[D.rz + i] = dl_dlam[g];
    }
    if (dl_dnu != nullptr)                                       // all of it in every CTA, as in k_box_backward
        for (int i = tid; i < e; i += kBoxNT) qsm[D.ry + i] = dl_dnu[(int64_t)qp * e + i];
    __syncthreads();
    dm_form(Y, D, rank, Ag);
    dm_solve(Y, D, rank, Ag, j0, ph, true, D.rx, -1, dl_dlam != nullptr ? D.rz : -1, dl_dnu != nullptr ? D.ry : -1,
             D.dx, D.ds, D.dz, D.dy);
    for (int j = tid; j < n; j += kBoxNT) {
        const int64_t g = (int64_t)qp * N + j0 + j;
        const double dx = qsm[D.dx + j], z = zhat[g];
        dxv[g] = dx;
        if (O.dq && !O.mq) O.dq[g] = dx * z;
        if (O.dp && !O.mp) O.dp[g] = dx;
    }
    for (int i = tid; i < m; i += kBoxNT) {
        const double dz = qsm[D.dz + i];
        dlamv[(int64_t)qp * X.mg + cl_grow(X, D, j0, i)] = dz;
        if (i < D.nlb) { if (O.dlb && !O.mlb) O.dlb[(int64_t)qp * N + j0 + i] = dz; }
        else if (O.dub && !O.mub) O.dub[(int64_t)qp * N + j0 + i - D.nlb] = -dz;
    }
    if (rank == 0)
        for (int i = tid; i < e; i += kBoxNT) {
            dnuv[(int64_t)qp * e + i] = qsm[D.dy + i];
            if (O.db && !O.mb) O.db[(int64_t)qp * e + i] = -qsm[D.dy + i];
        }
    if (O.dA && !O.mA)
        for (int t = tid; t < e * n; t += kBoxNT) {
            const int i = t / n, j = t - i * n;
            O.dA[((int64_t)qp * e + i) * N + j0 + j] = fma(qsm[D.dy + i], zhat[(int64_t)qp * N + j0 + j],
                                                           nus[(int64_t)qp * e + i] * qsm[D.dx + j]);
        }
    cg::this_cluster().sync();
}

// k_box_kkt<Cluster> with M distributed
__global__ void __launch_bounds__(kBoxNT, 1)
k_box_kkt_dm(DmDims Y, const double* __restrict__ q, int64_t sq, const double* __restrict__ A, int64_t sA,
             const double* __restrict__ d, const double* __restrict__ rx, const double* __restrict__ rs,
             const double* __restrict__ rz, const double* __restrict__ ry, double* __restrict__ dx,
             double* __restrict__ ds, double* __restrict__ dz, double* __restrict__ dy) {
    QPB_SMEM;
    const ClDims& X = Y.X;
    const int rank = (int)cg::this_cluster().block_rank();
    const int tid = threadIdx.x, qp = blockIdx.x / X.C;
    int j0, ph = 0;
    const BoxDims D = cl_local(X, rank, j0);
    const int n = D.n, m = D.m, e = D.e, N = X.ng;
    const double* Ag = A + (int64_t)qp * sA;
    dm_stage(D, j0, q + (int64_t)qp * sq, nullptr);
    for (int j = tid; j < n; j += kBoxNT) qsm[D.rx + j] = rx[(int64_t)qp * N + j0 + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * X.mg + cl_grow(X, D, j0, i);
        qsm[D.d + i] = d[g];
        qsm[D.rsc + i] = rs[g];
        qsm[D.rz + i] = rz[g];
    }
    for (int i = tid; i < e; i += kBoxNT) qsm[D.ry + i] = ry[(int64_t)qp * e + i];
    __syncthreads();
    dm_form(Y, D, rank, Ag);
    dm_solve(Y, D, rank, Ag, j0, ph, true, D.rx, D.rsc, D.rz, D.ry, D.dx, D.ds, D.dz, D.dy);
    for (int j = tid; j < n; j += kBoxNT) dx[(int64_t)qp * N + j0 + j] = qsm[D.dx + j];
    for (int i = tid; i < m; i += kBoxNT) {
        const int64_t g = (int64_t)qp * X.mg + cl_grow(X, D, j0, i);
        ds[g] = qsm[D.ds + i];
        dz[g] = qsm[D.dz + i];
    }
    if (rank == 0)
        for (int i = tid; i < e; i += kBoxNT) dy[(int64_t)qp * e + i] = qsm[D.dy + i];
    cg::this_cluster().sync();
}

// batch means of the gradients of un-batched inputs (qp.py:159-177)
// out[c] = scale / B * sum_b u[b * su + c] (* x[b * len + c] when x != null)
__global__ void k_box_mean_vec(int B, int len, const double* __restrict__ u, int64_t su, const double* __restrict__ x,
                               double scale, double* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= len) return;
    double s0 = 0.0, s1 = 0.0;
    int bb = 0;
    for (; bb + 1 < B; bb += 2) {
        s0 += x ? u[(int64_t)bb * su + c] * x[(int64_t)bb * len + c] : u[(int64_t)bb * su + c];
        s1 += x ? u[(int64_t)(bb + 1) * su + c] * x[(int64_t)(bb + 1) * len + c] : u[(int64_t)(bb + 1) * su + c];
    }
    if (bb < B) s0 += x ? u[(int64_t)bb * su + c] * x[(int64_t)bb * len + c] : u[(int64_t)bb * su + c];
    out[c] = (s0 + s1) * scale / (double)B;
}
// dA mean: out[r][c] = 1/B sum_b (dnu[b][r] z[b][c] + nu[b][r] dx[b][c]); one thread per entry, a block per 128 columns
__global__ void k_box_mean_outer(int B, int rows, int cols, const double* __restrict__ dnu, const double* __restrict__ z,
                                 const double* __restrict__ nu, const double* __restrict__ dx, double* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= cols) return;
    double s = 0.0;
    for (int bb = 0; bb < B; ++bb)
        s = fma(dnu[(int64_t)bb * rows + r], z[(int64_t)bb * cols + c], fma(nu[(int64_t)bb * rows + r], dx[(int64_t)bb * cols + c], s));
    out[(int64_t)r * cols + c] = s / (double)B;
}

std::mutex g_mu;
// cudaFuncAttributeMaxDynamicSharedMemorySize already set, per (kernel, device): its high-water mark
std::map<std::pair<const void*, int>, size_t> g_smem;

template <typename K>
int box_set_smem(K kernel, size_t bytes) {
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, "cudaGetDevice"); return QPB200_ERR_CUDA; }
    std::lock_guard<std::mutex> lock(g_mu);
    size_t& cur = g_smem[{(const void*)kernel, dev}];
    if (cur >= bytes) return QPB200_OK;
    err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, "cudaFuncSetAttribute"); return QPB200_ERR_CUDA; }
    cur = bytes;
    return QPB200_OK;
}
int box_check_launch(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, what); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}

int box_plan_check(const qpb200_box_plan* P) {
    if (P == nullptr) return QPB200_ERR_BAD_ARG;
    if (P->cl_ctas != 0 && P->cl_ctas != 2 && P->cl_ctas != 4 && P->cl_ctas != 8) return QPB200_ERR_BAD_ARG;
    if (!P->ok && !P->cl_ctas) return QPB200_ERR_TOO_LARGE;
    return QPB200_OK;
}

// Whether a cluster of C CTAs with `bytes` of shared memory each can be resident at all (cudaOccupancyMaxActiveClusters
// > 0), checked once per (kernel, C, bytes, device): QPB200_ERR_TOO_LARGE if not.
struct ClKey {
    const void* k; int C; size_t bytes; int dev;
    bool operator<(const ClKey& o) const {
        if (k != o.k) return k < o.k;
        if (C != o.C) return C < o.C;
        if (bytes != o.bytes) return bytes < o.bytes;
        return dev < o.dev;
    }
};
std::map<ClKey, bool> g_cl_ok;

template <typename K>
int cl_prepare(K kernel, int C, size_t bytes) {
    int rc = box_set_smem(kernel, bytes);
    if (rc) return rc;
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, "cudaGetDevice"); return QPB200_ERR_CUDA; }
    const ClKey key{(const void*)kernel, C, bytes, dev};
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_cl_ok.find(key);
    if (it == g_cl_ok.end()) {
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3(C); cfg.blockDim = dim3(kBoxNT); cfg.dynamicSmemBytes = bytes;
        cfg.attrs = at; cfg.numAttrs = 1;
        int nclusters = 0;
        err = cudaOccupancyMaxActiveClusters(&nclusters, (const void*)kernel, &cfg);
        if (err != cudaSuccess) {
            qpb200_internal_cuda_error((int)err, "cudaOccupancyMaxActiveClusters");
            return QPB200_ERR_CUDA;
        }
        it = g_cl_ok.emplace(key, nclusters > 0).first;
    }
    return it->second ? QPB200_OK : QPB200_ERR_TOO_LARGE;
}

template <typename... KArgs, typename... Args>
int cl_launch(const char* what, void (*kernel)(KArgs...), int C, int nbatch, size_t bytes, cudaStream_t st,
              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)nbatch * (unsigned)C); cfg.blockDim = dim3(kBoxNT); cfg.dynamicSmemBytes = bytes;
    cfg.stream = st; cfg.attrs = at; cfg.numAttrs = 1;
    const cudaError_t err = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, what); return QPB200_ERR_CUDA; }
    return box_check_launch(what);
}

// Launches the kernel for the layout the plan selects: k1 (k_box_*<OneCta>) with one CTA per QP, or a cluster per QP
// (cl_ctas): kc (k_box_*<Cluster>), or kd (k_box_*_dm) with M distributed past neq_pad = 128.
template <class K1, class KC, class KD, class... Args>
int box_launch(const char* what, const qpb200_box_plan* plan, int nbatch, void* stream, K1 k1, KC kc, KD kd,
               Args... args) {
    cudaStream_t st = (cudaStream_t)stream;
    auto run = [&](auto kernel, const auto& P) {
        const size_t bytes = (size_t)P.total * 8;
        if (!plan->cl_ctas) {
            const int rc = box_set_smem(kernel, bytes);
            if (rc) return rc;
            kernel<<<nbatch, kBoxNT, bytes, st>>>(P, args...);
            return box_check_launch(what);
        }
        const int rc = cl_prepare(kernel, plan->cl_ctas, bytes);
        if (rc) return rc;
        return cl_launch(what, kernel, plan->cl_ctas, nbatch, bytes, st, P, args...);
    };
    const int n = plan->nz, e = plan->neq, lb = plan->has_lb, ub = plan->has_ub, C = plan->cl_ctas;
    if (!C) return run(k1, box_dims(n, e, lb, ub));
    if (plan->neq_pad > kBoxNT) return run(kd, dm_dims(n, e, lb, ub, C));
    return run(kc, cl_dims(n, e, lb, ub, C));
}

}  // namespace

extern "C" {

int qpb200_box_plan_init(int nz, int neq, int has_lb, int has_ub, qpb200_box_plan* plan) {
    if (plan == nullptr || nz <= 0 || neq < 0) return QPB200_ERR_BAD_ARG;
    if (!has_lb && !has_ub) return QPB200_ERR_NO_CONSTRAINTS;
    // past every path: the dense kernels stop at 4096, and 8 CTAs of 227 KB hold fewer than 12000 variables
    if (nz > 16384 || neq > 4096) return QPB200_ERR_TOO_LARGE;
    memset(plan, 0, sizeof(*plan));
    plan->nz = nz; plan->neq = neq; plan->neq_pad = r8(neq);
    plan->has_lb = has_lb ? 1 : 0; plan->has_ub = has_ub ? 1 : 0;
    plan->nineq = (plan->has_lb + plan->has_ub) * nz;
    plan->threads = kBoxNT;
    const BoxDims D = box_dims(nz, neq, plan->has_lb, plan->has_ub);
    plan->smem_bytes = (int64_t)D.total * 8;
    plan->ok = (plan->neq_pad <= kBoxNT && plan->smem_bytes <= kBoxMaxSmem) ? 1 : 0;
    // A cluster of C CTAs, the smallest whose slice fits: the cluster kernels for shapes one CTA does not hold; past
    // neq_pad = 128 the distributed-M kernels, where the dense path rejects the shape or its order is past
    // kDmDenseOrder (below it the dense kernels are faster). QPB200_BOX_CLUSTER=C (development knob, C in {2, 4, 8})
    // forces them where that C fits.
    const bool distm = plan->neq_pad > kBoxNT;
    auto cl_for = [&](int C) -> ClDims {
        return distm ? dm_dims(nz, neq, plan->has_lb, plan->has_ub, C).X : cl_dims(nz, neq, plan->has_lb, plan->has_ub, C);
    };
    auto fits = [&](int C) { return (int64_t)cl_for(C).total * 8 <= kBoxMaxSmem; };
    auto wanted = [&]() {
        if (!distm) return !plan->ok;
        qpb200_plan dp;
        const int rc = qpb200_plan_init(nz, plan->nineq, neq, &dp);
        return rc == QPB200_ERR_TOO_LARGE || (rc == QPB200_OK && dp.ms_pad > kDmDenseOrder);
    };
    const char* env = getenv("QPB200_BOX_CLUSTER");
    const int forced = env ? atoi(env) : 0;
    int C = 0;
    if ((forced == 2 || forced == 4 || forced == 8) && fits(forced)) C = forced;
    else if (wanted())
        for (int c = 2; c <= 8 && !C; c *= 2)
            if (fits(c)) C = c;
    if (C) {
        const ClDims X = cl_for(C);
        plan->cl_ctas = C;
        plan->cl_slice = X.slice;
        plan->cl_smem_bytes = (int64_t)X.total * 8;
    }
    if (!plan->ok && !plan->cl_ctas) {          // only the dense kernels on the dense equivalent are left
        qpb200_plan dp;
        const int rc = qpb200_plan_init(nz, plan->nineq, neq, &dp);
        if (rc == QPB200_ERR_TOO_LARGE) return rc;
    }
    return QPB200_OK;
}

int qpb200_box_forward(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* p, int64_t sp,
                       const double* A, int64_t sA, const double* b, int64_t sb, const double* lb, int64_t slb,
                       const double* ub, int64_t sub, double eps, double stall_tol, double best_tie, int notImprovedLim,
                       int maxIter, double* zhat, double* lam, double* slacks, double* nus, int* iters,
                       double* best_resid, double* trace, int* spd_flag, void* stream) {
    int rc = box_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || maxIter < 1 || !q || !p || !zhat || !lam || !slacks || !iters || !best_resid) return QPB200_ERR_BAD_ARG;
    if ((plan->has_lb && !lb) || (plan->has_ub && !ub) || (plan->neq > 0 && (!A || !b || !nus))) return QPB200_ERR_BAD_ARG;
    return box_launch("k_box_forward", plan, nbatch, stream, k_box_forward<OneCta>, k_box_forward<Cluster>,
                      k_box_forward_dm, q, sq, p, sp, A, sA, b, sb, lb, slb, ub, sub, eps, stall_tol, best_tie,
                      notImprovedLim, maxIter, zhat, lam, slacks, nus, iters, best_resid, trace, spd_flag);
}

int qpb200_box_backward(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                        int64_t sA, const double* dl_dzhat, const double* zhat, const double* lam, const double* slacks,
                        const double* nus, double* dq, int mean_q, double* dp, int mean_p, double* dlb, int mean_lb,
                        double* dub, int mean_ub, double* dA, int mean_A, double* db, int mean_b, double* dxv,
                        double* dlamv, double* dnuv, void* stream) {
    return qpb200_box_backward_duals(plan, nbatch, q, sq, A, sA, dl_dzhat, nullptr, nullptr, zhat, lam, slacks, nus, dq,
                                     mean_q, dp, mean_p, dlb, mean_lb, dub, mean_ub, dA, mean_A, db, mean_b, dxv, dlamv,
                                     dnuv, stream);
}

int qpb200_box_backward_duals(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                              int64_t sA, const double* dl_dzhat, const double* dl_dlam, const double* dl_dnu,
                              const double* zhat, const double* lam, const double* slacks, const double* nus, double* dq,
                              int mean_q, double* dp, int mean_p, double* dlb, int mean_lb, double* dub, int mean_ub,
                              double* dA, int mean_A, double* db, int mean_b, double* dxv, double* dlamv, double* dnuv,
                              void* stream) {
    int rc = box_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || !q || !dl_dzhat || !zhat || !lam || !slacks || !dxv || !dlamv) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!A || !nus || !dnuv)) return QPB200_ERR_BAD_ARG;
    if (dl_dnu && plan->neq == 0) return QPB200_ERR_BAD_ARG;
    if ((dlb && !plan->has_lb) || (dub && !plan->has_ub)) return QPB200_ERR_BAD_ARG;
    const int n = plan->nz, m = plan->nineq, e = plan->neq, nlb = plan->has_lb ? n : 0;
    BoxGrads O;
    O.dq = dq; O.dp = dp; O.dlb = dlb; O.dub = dub; O.dA = e > 0 ? dA : nullptr; O.db = e > 0 ? db : nullptr;
    O.mq = mean_q; O.mp = mean_p; O.mlb = mean_lb; O.mub = mean_ub; O.mA = mean_A; O.mb = mean_b;
    rc = box_launch("k_box_backward", plan, nbatch, stream, k_box_backward<OneCta>, k_box_backward<Cluster>,
                    k_box_backward_dm, q, sq, A, sA, dl_dzhat, dl_dlam, dl_dnu, zhat, lam, slacks, nus, O, dxv, dlamv,
                    dnuv);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int TB = 128;
    if (dq && mean_q) k_box_mean_vec<<<(n + TB - 1) / TB, TB, 0, st>>>(nbatch, n, dxv, n, zhat, 1.0, dq);
    if (dp && mean_p) k_box_mean_vec<<<(n + TB - 1) / TB, TB, 0, st>>>(nbatch, n, dxv, n, nullptr, 1.0, dp);
    if (dlb && mean_lb) k_box_mean_vec<<<(n + TB - 1) / TB, TB, 0, st>>>(nbatch, n, dlamv, m, nullptr, 1.0, dlb);
    if (dub && mean_ub)
        k_box_mean_vec<<<(n + TB - 1) / TB, TB, 0, st>>>(nbatch, n, dlamv + nlb, m, nullptr, -1.0, dub);
    if (e > 0) {
        if (dA && mean_A) k_box_mean_outer<<<dim3((n + TB - 1) / TB, e), TB, 0, st>>>(nbatch, e, n, dnuv, zhat, nus, dxv, dA);
        if (db && mean_b) k_box_mean_vec<<<(e + TB - 1) / TB, TB, 0, st>>>(nbatch, e, dnuv, e, nullptr, -1.0, db);
    }
    return box_check_launch("k_box_mean");
}

int qpb200_box_solve_kkt(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                         int64_t sA, const double* d, const double* rx, const double* rs, const double* rz,
                         const double* ry, double* dx, double* ds, double* dz, double* dy, void* stream) {
    int rc = box_plan_check(plan);
    if (rc) return rc;
    if (nbatch <= 0 || !q || !d || !rx || !rs || !rz || !dx || !ds || !dz) return QPB200_ERR_BAD_ARG;
    if (plan->neq > 0 && (!A || !ry || !dy)) return QPB200_ERR_BAD_ARG;
    return box_launch("k_box_kkt", plan, nbatch, stream, k_box_kkt<OneCta>, k_box_kkt<Cluster>, k_box_kkt_dm, q, sq,
                      A, sA, d, rx, rs, rz, ry, dx, ds, dz, dy);
}

}  // extern "C"
