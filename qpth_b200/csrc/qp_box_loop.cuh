// The Mehrotra loop, backward and KKT kernels of BoxQPFunction, written once over a family F (a layout of the KKT solve
// with the bounds eliminated). Included by qp_box.cu (kNT = 128: diagonal Q, families OneCta and Cluster) and by
// qp_boxq.cu (kNT = 256: dense Q, family DenseQ); each unit sets its own QPB_NT and its own `qpb` namespace first.
//
// A family is the per-CTA context of one layout, built in the kernel from its parameter (F::Dims, __grid_constant__: a
// family may hold a reference to it without ptxas copying the parameter into local memory), with
//   D                     this CTA's layout: counts (n, m, e, ep, nlb: its local variables, inequality rows, neq,
//                         neq_pad, lb rows) and the shared-memory offsets of the vectors below;
//   kMinFwd / kMinBwd / kMinKkt   the CTAs per SM of each kernel's __launch_bounds__ (0: no bound);
//   qp(), j0() (first local variable), ng() / mg() (nz and inequality rows of the whole QP), grow(i) (global inequality
//   row of local row i), leader() (writes the length-neq outputs, iters, best_resid, the trace and spd_flag), a(i, j)
//   (A at local column j), reduce_sum / reduce_min (QP-wide, bit-identical in every CTA), sync() (the closing barrier);
// and the whole phases that differ between layouts:
//   stage(q, A, b)        q or Q, A, b (nullptr in the backward and KKT kernels) of this QP; ends with a block barrier;
//   spd_bad()             the QP-wide 'Q is not SPD.' flag;
//   form()                the Newton matrix for the d in shared memory;
//   before_residuals(form_d)   dense Q: d = z / s (form_d()) and the Newton matrix, formed with the Q x of the
//                         residual in one pass over Q;
//   qx_p(j)               (Q x + p)_j of the dual residual, rounded as the family has always rounded it;
//   ry_step(acc)          ry = A x - b and |ry|^2 into acc[0], then the reduction of acc;
//   before_affine(form_d)    the box families: d = z / s and the Newton matrix, only once the exit tests have passed
//                         (so the exiting iteration forms nothing);
//   solve(fresh, rx, rs, rz, ry, dx, ds, dz, dy)   K [dx ds dz dy] = -[rx rs rz ry] with the matrix of the last form
//                         (rs, rz, ry may be -1: zero); fresh: factor it here, else reuse the factor. Ends with a barrier;
//   write_dq(dq, qp, zhat)   the gradient of q (dq = dx o z) or of Q (dQ = 1/2 (dx z' + z dx')).
// The shared code never branches on the family.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/qpth_b200.h"
#include "qp_pf.cuh"

extern "C" void qpb200_internal_cuda_error(int err, const char* what);   // (qp_kernels.cu) records the message, per thread

namespace {

constexpr int kBoxNT = qpb::fast::kNT;
constexpr int kClW = kBoxNT / 32;          // warps per CTA
constexpr int kBoxMaxSmem = 232448;        // H100: 227 KB of dynamic shared memory per CTA

__host__ __device__ inline int r8(int v) { return (v + 7) & ~7; }

// inequality row i is sign(i) * e_var(i)
template <class Dims> __device__ __forceinline__ int bvar(const Dims& D, int i) { return i < D.nlb ? i : i - D.nlb; }
template <class Dims> __device__ __forceinline__ double bsgn(const Dims& D, int i) { return i < D.nlb ? -1.0 : 1.0; }

// G'v of a length-m shared vector at column j (the lb row and/or the ub row of variable j)
template <class Dims> __device__ __forceinline__ double gt_col(const Dims& D, const double* v, int j) {
    double a = 0.0;
    if (D.nlb) a -= v[j];
    if (D.m > D.nlb) a += v[D.nlb + j];
    return a;
}

__device__ __forceinline__ double box_step(double v, double dv) { return (dv > 0.0) ? INFINITY : (-v / dv); }
__device__ __forceinline__ double box_step_fix(double v) { return (isinf(v) && v > 0.0) ? 1.0 : v; }

int box_check_launch(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { qpb200_internal_cuda_error((int)err, what); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}

// What the one-CTA families (OneCta, DenseQ) share: A in shared memory, block reductions. Held: how the family holds
// the layout, a copy or a reference to the kernel parameter.
template <class Dims_, class Held = Dims_>
struct BoxCta {
    using Dims = Dims_;
    Held D;

    __device__ explicit BoxCta(const Dims& P) : D(P) {}
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
    __device__ static void sync() {}

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
};

// forward (batch.py:47-207); the loop of k_forward_fast (qp_solve.cuh). Every CTA writes its slice of zhat, lam and
// slacks; the leader nus, iters, best_resid, the trace rows and spd_flag.
//
// INVARIANT (Cluster, and the k_box_*_dm kernels of qp_box.cu, which repeat this loop): every CTA of a cluster executes
// the same sequence of cluster.sync() calls. Every reduction leaves bit-identical sums and minima in every CTA, and so
// does every solve (M is summed in rank order and factored redundantly, or dy is gathered from its owners), so y, mu,
// the residual and the step lengths are bit-identical too. Every branch that reaches a cluster barrier (the exit
// tests, NaN and mu > 1e32 exits, best-iterate tracking, notImprovedLim, e > 0, fresh) is decided from those values or
// from kernel arguments only; a CTA that branched on a value of its own would deadlock its cluster.
template <class F>
__global__ void __launch_bounds__(kBoxNT, F::kMinFwd)
k_box_forward(const __grid_constant__ typename F::Dims P, const double* __restrict__ q, int64_t sq,
              const double* __restrict__ p, int64_t sp, const double* __restrict__ A, int64_t sA,
              const double* __restrict__ b, int64_t sb, const double* __restrict__ lb, int64_t slb,
              const double* __restrict__ ub, int64_t sub, double eps, double stall_tol, double best_tie,
              int notImprovedLim, int maxIter, double* __restrict__ zhat, double* __restrict__ lam,
              double* __restrict__ slacks, double* __restrict__ nus, int* __restrict__ iters_out,
              double* __restrict__ resid_out, double* __restrict__ trace, int* __restrict__ spd_flag) {
    QPB_SMEM;
    F f(P);
    const auto& D = f.D;
    const int tid = threadIdx.x, qp = f.qp(), j0 = f.j0();
    const int n = D.n, m = D.m, e = D.e, ep = D.ep;
    f.stage(q + (int64_t)qp * sq, A + (int64_t)qp * sA, (e > 0) ? b + (int64_t)qp * sb : nullptr);
    for (int j = tid; j < n; j += kBoxNT) qsm[D.p + j] = p[(int64_t)qp * sp + j0 + j];
    for (int i = tid; i < m; i += kBoxNT) {
        qsm[D.h + i] = (i < D.nlb) ? -lb[(int64_t)qp * slb + j0 + i] : ub[(int64_t)qp * sub + j0 + i - D.nlb];
        qsm[D.d + i] = 1.0;
        qsm[D.rz + i] = -qsm[D.h + i];
    }
    for (int i = tid; i < ep; i += kBoxNT) { qsm[D.ry + i] = -qsm[D.b + i]; qsm[D.y + i] = 0.0; }
    {
        const int bad = f.spd_bad();
        if (f.leader() && tid == 0 && spd_flag != nullptr) spd_flag[qp] = bad;
    }
    __syncthreads();

    // ---- initial point: solve_kkt(p, 0, -h, -b) with d = 1   (batch.py:61-67)
    f.form();
    f.solve(true, D.p, -1, D.rz, D.ry, D.x, D.s, D.z, D.y);
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

    // d = z / s, for the Newton matrix of this iteration; ends with a block barrier
    auto form_d = [&]() {
        for (int i = tid; i < m; i += kBoxNT) qsm[D.d + i] = qsm[D.z + i] / qsm[D.s + i];
        __syncthreads();
    };
    double best = 0.0;
    int nNot = 0, iters_run = 0;
    const double dm = (double)f.mg();
    for (int it = 0; it < maxIter; ++it) {
        iters_run = it + 1;
        f.before_residuals(form_d);
        // ---- residuals (batch.py:94-107)
        double acc[4] = {0.0, 0.0, 0.0, 0.0};                   // |ry|^2, |rz|^2, |rx|^2, s.z
        for (int j = tid; j < n; j += kBoxNT) {
            double a = 0.0;
            for (int i = 0; i < e; ++i) a = fma(f.a(i, j), qsm[D.y + i], a);
            const double r = f.qx_p(j) + gt_col(D, qsm + D.z, j) + a;
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
        // ---- best-iterate tracking and exit tests (batch.py:118-143), per QP: QP-wide values only
        const bool improved = (it == 0) || (resid < best);
        if (improved) { best = resid; nNot = 0; } else { ++nNot; }
        if (improved || resid < best_tie * best) {
            for (int j = tid; j < n; j += kBoxNT) qsm[D.bx + j] = qsm[D.x + j];
            for (int i = tid; i < m; i += kBoxNT) { qsm[D.bs + i] = qsm[D.s + i]; qsm[D.bz + i] = qsm[D.z + i]; }
            for (int i = tid; i < e; i += kBoxNT) qsm[D.by + i] = qsm[D.y + i];
        }
        if ((nNot == notImprovedLim && best < stall_tol) || best < eps || mu > 1e32) break;
        if (!(resid == resid) || isinf(resid)) break;
        // ---- the affine direction (batch.py:109-113,150) factors the Newton matrix
        f.before_affine(form_d);
        f.solve(true, D.rx, D.z, D.rz, D.ry, D.dxa, D.dsa, D.dza, D.dya);
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
        f.solve(false, D.rx, D.rsc, -1, -1, D.dx, D.ds, D.dz, D.dy);
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

// QPFunctionFn.backward (qp.py:128-182) for the box QP: d from the clamped duals (qp.py:148), one factor and one solve
// per QP, then dq (f.write_dq), dp = dx, dlb = dlam_lb, dub = -dlam_ub, dA = dnu z' + nu dx', db = -dnu. dxv, dlamv and
// dnuv always receive dx, dlam, dnu (the batch means read them); a gradient whose mean flag is set is skipped here.
// Every CTA writes its slice of dx, dlam, dq, dp, dlb, dub and its columns of dA; the leader dnu and db. dl_dlam and
// dl_dnu (NULL: zero) are the adjoints of the returned duals: they are the rz and ry of the solve, which rz / ry are not
// otherwise.
struct BoxGrads {
    double *dq, *dp, *dlb, *dub, *dA, *db;   // dq: (B, nz) for a diagonal Q, dQ (B, nz, nz) for a dense one
    int mq, mp, mlb, mub, mA, mb;
};

template <class F>
__global__ void __launch_bounds__(kBoxNT, F::kMinBwd)
k_box_backward(const __grid_constant__ typename F::Dims P, const double* __restrict__ q, int64_t sq,
               const double* __restrict__ A, int64_t sA, const double* __restrict__ dl,
               const double* __restrict__ dl_dlam, const double* __restrict__ dl_dnu, const double* __restrict__ zhat,
               const double* __restrict__ lam, const double* __restrict__ slacks, const double* __restrict__ nus,
               BoxGrads O, double* __restrict__ dxv, double* __restrict__ dlamv, double* __restrict__ dnuv) {
    QPB_SMEM;
    F f(P);
    const auto& D = f.D;
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
    f.solve(true, D.rx, -1, dl_dlam != nullptr ? D.rz : -1, dl_dnu != nullptr ? D.ry : -1, D.dx, D.ds, D.dz, D.dy);
    for (int j = tid; j < n; j += kBoxNT) {
        const int64_t g = (int64_t)qp * N + j0 + j;
        const double dx = qsm[D.dx + j];
        dxv[g] = dx;
        if (O.dp && !O.mp) O.dp[g] = dx;
    }
    if (O.dq && !O.mq) f.write_dq(O.dq, qp, zhat);
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

// qpb200_box_solve_kkt / qpb200_boxq_solve_kkt: the factor and solve for caller-given d and right-hand sides (all
// vectors (B, len))
template <class F>
__global__ void __launch_bounds__(kBoxNT, F::kMinKkt)
k_box_kkt(const __grid_constant__ typename F::Dims P, const double* __restrict__ q, int64_t sq,
          const double* __restrict__ A, int64_t sA, const double* __restrict__ d, const double* __restrict__ rx,
          const double* __restrict__ rs, const double* __restrict__ rz, const double* __restrict__ ry,
          double* __restrict__ dx, double* __restrict__ ds, double* __restrict__ dz, double* __restrict__ dy) {
    QPB_SMEM;
    F f(P);
    const auto& D = f.D;
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
    f.solve(true, D.rx, D.rsc, D.rz, D.ry, D.dx, D.ds, D.dz, D.dy);
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

}  // namespace
