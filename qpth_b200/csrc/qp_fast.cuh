// Fast path of the per-QP solve: everything in shared memory, compact code.
//
// Why a second set of routines next to qp_device.cuh: the first version inlined and fully unrolled every
// building block at every call site and ended up with ~20k SASS instructions (317 KB) per kernel, far
// beyond the instruction caches (ncu: 12-45 % "no_inst" stalls).  Here every building block is a
// __noinline__ function that exists once, shared-memory objects are addressed as OFFSETS (in doubles) into
// the one dynamic shared array so the compiler still emits LDS/STS, and the reduced KKT system is padded to
// a multiple of 8 (identity rows) so no block is ever partial.
//
// Reference functions implemented (qpth/solvers/pdipm/batch.py): factor_kkt :435-470 -> f_chol,
// solve_kkt :349-372 -> f_trsv_* + f_matvec_*, forward :47-207 -> k_forward_fast (qp_kernels.cu).
#pragma once
#include "qp_device.cuh"

namespace qpb {
namespace fast {

#define QPB_SMEM extern __shared__ __align__(16) double qsm[]

// Optional cycle accounting (build with -DQPB_TIMING): thread 0 of block 0 accumulates clock64() deltas per
// phase into g_tim[]; read back with qpb200_debug_timing(). Compiled out of the product build.
#ifdef QPB_TIMING
// per-CTA record of k_forward_fast: {globaltimer at entry, at exit (ns), Newton iterations, SM id}
__device__ long long g_cta[4 * 8192];
__device__ int g_tim_target = 0;          // which QP's phase slots are exported (qpb200_debug_timing(., 2 + qp))
__device__ __forceinline__ long long gtimer() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ int smid() { int r; asm volatile("mov.u32 %0, %smid;" : "=r"(r)); return r; }
__device__ long long g_tim[128];
// accumulators live in (static) shared memory so that a tick costs ~40 cycles, not a global round trip
__shared__ long long s_tim[129];
#define QPB_TICK(i)                                                         \
    do {                                                                    \
        if (threadIdx.x == 0) {                                             \
            const long long _t = clock64();                                 \
            s_tim[i] += _t - s_tim[128];                                    \
            s_tim[128] = _t;                                                \
        }                                                                   \
    } while (0)
// second clock on thread 32 (warp 1, an update warp): slots 40.., own time base in s_tim2
__shared__ long long s_tim2;
#define QPB_TICK1(i)                                                        \
    do {                                                                    \
        if (threadIdx.x == 32) {                                            \
            const long long _t = clock64();                                 \
            s_tim[i] += _t - s_tim2;                                        \
            s_tim2 = _t;                                                    \
        }                                                                   \
    } while (0)
#else
#define QPB_TICK(i) do {} while (0)
#define QPB_TICK1(i) do {} while (0)
#endif

#ifndef QPB_NT
#define QPB_NT 256       // CTA size of the solve kernels; qp_alt.cu builds the product-form ones at 192 and 512 threads as well
#endif
constexpr int kNT = QPB_NT;

// ---- 8x8 diagonal block helpers (always full blocks here) -------------------------------------------
// Storage convention of a factored diagonal block: strictly-lower part = L, DIAGONAL = 1 / L_cc.
// (Nothing downstream needs L_cc itself; every use is a multiplication by its reciprocal.)

// Load the lower triangle (incl. diagonal) of the 8x8 block at Mb with 128-bit loads (20 LDS.128).
__device__ __forceinline__ void f_load_lower8(const double* Mb, int ld, double (&Lk)[36]) {
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c <= r; c += 2) {
            const double2 v = *reinterpret_cast<const double2*>(Mb + r * ld + c);
            Lk[QPB_LIDX(r, c)] = v.x;
            if (c + 1 <= r) Lk[QPB_LIDX(r, c + 1)] = v.y;
        }
}

// 1/sqrt(x) for the pivots: MUFU seed (~23 bits) + one third-order step; 4 dependent fp64 ops after the MUFU
// instead of the library rsqrt()'s 5 + special-case branch.
// Negative / zero pivots give NaN, which is what the callers want to propagate.
__device__ __forceinline__ double f_rsqrt(double x) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    const double t = x * y;
    const double e = fma(-t, y, 1.0);
    const double p = fma(0.375, e, 0.5);
    const double ye = y * e;
    return fma(ye, p, y);
}

// In-register factorization of an 8x8 block (lower triangle in Lk): on exit strictly lower = L, diagonal = 1/L_cc.
__device__ __forceinline__ void f_factor8_regs(double (&Lk)[36]) {
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const double ri = f_rsqrt(Lk[QPB_LIDX(c, c)]);
        Lk[QPB_LIDX(c, c)] = ri;
#pragma unroll
        for (int r = c + 1; r < 8; ++r) Lk[QPB_LIDX(r, c)] *= ri;
#pragma unroll
        for (int r = c + 1; r < 8; ++r)
#pragma unroll
            for (int cc = c + 1; cc <= r; ++cc)
                Lk[QPB_LIDX(r, cc)] = fma(-Lk[QPB_LIDX(r, c)], Lk[QPB_LIDX(cc, c)], Lk[QPB_LIDX(r, cc)]);
    }
}
__device__ __forceinline__ void f_store_lower8(double* Mb, int ld, const double (&Lk)[36]) {
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c <= r; c += 2)      // the odd tail writes one element of the (unused) upper part
            *reinterpret_cast<double2*>(Mb + r * ld + c) =
                make_double2(Lk[QPB_LIDX(r, c)], (c + 1 <= r) ? Lk[QPB_LIDX(r, c + 1)] : 0.0);
}

// a <- a * L_kk^-T by substitution (Lk: strictly lower = L, diagonal = reciprocal).
__device__ __forceinline__ void f_row_solve8(double (&a)[8], const double (&Lk)[36]) {
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        a[c] *= Lk[QPB_LIDX(c, c)];
#pragma unroll
        for (int c2 = c + 1; c2 < 8; ++c2) a[c2] = fma(-a[c], Lk[QPB_LIDX(c2, c)], a[c2]);
    }
}

__device__ __forceinline__ void f_ld8(const double* p, double (&a)[8]) {
    const double2 v0 = *reinterpret_cast<const double2*>(p), v1 = *reinterpret_cast<const double2*>(p + 2),
                  v2 = *reinterpret_cast<const double2*>(p + 4), v3 = *reinterpret_cast<const double2*>(p + 6);
    a[0] = v0.x; a[1] = v0.y; a[2] = v1.x; a[3] = v1.y; a[4] = v2.x; a[5] = v2.y; a[6] = v3.x; a[7] = v3.y;
}
__device__ __forceinline__ void f_st8(double* p, const double (&a)[8]) {
    *reinterpret_cast<double2*>(p) = make_double2(a[0], a[1]);
    *reinterpret_cast<double2*>(p + 2) = make_double2(a[2], a[3]);
    *reinterpret_cast<double2*>(p + 4) = make_double2(a[4], a[5]);
    *reinterpret_cast<double2*>(p + 6) = make_double2(a[6], a[7]);
}

// ---- Cholesky: register-resident off-diagonal tiles, warp 0 runs the critical chain one panel ahead -----
// n multiple of 8, (n - c0)/8 <= 13, blockDim.x == 256. aug (offset) = right-hand side (length n) carried
// along so that L^-1 aug falls out of the factorization. Diagonal blocks end up in the convention above.
//
// Tasks of panel k:  F_k  factor diagonal block k                         (needs tile (k,k) final)
//                    s_k  solve the 8 panel rows of block k+1             (needs F_k)
//                    u_k  update diagonal tile k+1 with those rows        (needs s_k)      } critical chain,
//                    S_k  solve all other panel rows + the aug row        (needs F_k)        all on warp 0
//                    U_k  rest of the trailing update with panel k        (needs s_k, S_k)
// One step = [warp 0: s_k, u_k, F_{k+1}] in parallel with [warps 1..7: S_k, then U_k]; warp 0 signals s_k through
// named barrier 1 (bar.arrive, never waits), one __syncthreads per step. Warp 4 shares its scheduler with warp 0
// and takes no DMMA work, so the rsqrt/DFMA chain of F runs uncontended.
__device__ __forceinline__ void named_bar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Role 1 (warp 0): the critical chain  F_0, then per step  s_k -> signal -> u_k -> F_{k+1}.
__device__ __noinline__ void f_chol_chain(int A, int ld, int n, int c0) {
    QPB_SMEM;
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    const int nts = (n - c0) >> 3;
    double* M = qsm + A;
    double Lk[36];                                           // the current diagonal block stays in registers
    // k = -1 is the prologue step (F_0 only): ONE instance of the unrolled 8x8 factorization in the code.
    for (int k = -1; k < nts; ++k) {
        const int k0 = c0 + 8 * k;
        if (k >= 0 && k + 1 < nts) {
            // ---- s_k: the 8 panel rows of block k+1 (lanes 0..7), L_kk still in registers from F_k
            if (lane < 8) {
                double a[8];
                double* rowp = M + (k0 + 8 + lane) * ld + k0;
                f_ld8(rowp, a);
                f_row_solve8(a, Lk);
                f_st8(rowp, a);
            }
            __syncwarp();
            named_bar_arrive(1, kNT);
            QPB_TICK(96 + k);   // s_k, per step
            // ---- u_k: diagonal tile k+1 (lives in shared memory)
            double* pd = M + (k0 + 8 + g) * ld + k0 + 8 + 2 * q;
            const double* pr = M + (k0 + 8 + g) * ld + k0 + q;
            double2 cv = *reinterpret_cast<const double2*>(pd);
            const double a0 = pr[0], a1 = pr[4];
            dmma884(cv.x, cv.y, -a0, a0);
            dmma884(cv.x, cv.y, -a1, a1);
            *reinterpret_cast<double2*>(pd) = cv;
            __syncwarp();
            QPB_TICK(24);
        }
        if (k + 1 < nts) {
            f_load_lower8(M + (k0 + 8) * ld + k0 + 8, ld, Lk);
            __syncwarp();                                                             // all lanes have read the tile
            f_factor8_regs(Lk);                                                       // F_{k+1}
            if (lane == 0) f_store_lower8(M + (k0 + 8) * ld + k0 + 8, ld, Lk);
            if (k >= 0) QPB_TICK(80 + k);   // F_{k+1}, per step
        }
        QPB_TICK(26);
        __syncthreads();
        if (k >= 0) QPB_TICK(112 + k);      // chain warp waiting for the update warps, per step
    }
}

// Role 2 (warps 1..7): per step  S_k (all other panel rows + the aug row), wait for s_k, then U_k.
// Update warps 1,2,3,5,6,7 own the off-diagonal tiles as DMMA accumulators in registers; warp 4 shares its
// scheduler (and fp64 pipe) with the chain warp, so it only carries the right-hand side along.
__device__ __noinline__ void f_chol_update(int A, int ld, int n, int c0, int aug, int tabo) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, q = lane & 3;
    const int nts = (n - c0) >> 3;
    const int noff = (nts * (nts - 1)) / 2;
    const uint16_t* tab = reinterpret_cast<const uint16_t*>(qsm + tabo);
    double* M = qsm + A;
    const int uw = (warp == 4) ? -1 : (warp < 4 ? warp - 1 : warp - 2);
    double C[kCholMaxOff][2];
    // per slot only the packed tile id (ti << 8 | tj, -1: empty) lives in a register; fragment offsets are two IMADs
    // away. (Arrays of precomputed offsets pushed this function into local memory: 26 STL + 4 LDL per tile pair.)
    int tt_of[kCholMaxOff];
    const int gq = (c0 + g) * ld + q;
    if (uw >= 0) {
#pragma unroll
        for (int s = 0; s < kCholMaxOff; ++s) {
            const int idx = s * 6 + uw;
            const bool ok = idx < noff;
            const int tt = ok ? tab[idx] : 0;
            tt_of[s] = ok ? tt : -1;
            const double2 v = ok ? *reinterpret_cast<const double2*>(M + gq + q + 8 * (tt >> 8) * ld + c0 + 8 * (tt & 255))
                                 : make_double2(0.0, 0.0);
            C[s][0] = v.x; C[s][1] = v.y;
        }
    }
    __syncthreads();
    for (int k = 0; k < nts; ++k) {
        const int k0 = c0 + 8 * k;
        const bool last = (k + 1 >= nts);
        QPB_TICK1(40);
        // ---- S_k: all other rows below (i >= k0 + 16) and the aug row: row <- row * L_kk^-T
        {
            const int t = tid - 32;
            const int nrows = n - k0 - 16;                  // may be <= 0 near the end
            const int naug = nrows > 0 ? nrows : 0;
            if (t <= naug) {
                double Ls[36], a[8];
                double* rowp = (t < naug) ? (M + (k0 + 16 + t) * ld + k0) : (qsm + aug + k0);
                f_ld8(rowp, a);
                f_load_lower8(M + k0 * ld + k0, ld, Ls);
                f_row_solve8(a, Ls);
                f_st8(rowp, a);
            }
        }
        QPB_TICK1(64 + k);      // S_k, per step
        if (!last) {
            named_bar_sync(1, kNT);                         // all panel rows (incl. the chain warp's) are in place
            QPB_TICK1(42);
            if (uw >= 0) {
                // tiles come column by column, so the active ones (tj > k) are a suffix of this warp's slots;
                // two tiles at a time: 4 independent DMMAs keep the pipe busy
#pragma unroll
                for (int s = kCholMaxOff - 1; s >= 0; s -= 2) {
                    const int s1 = s, s2 = (s - 1 >= 0) ? s - 1 : 0;
                    const int t1 = tt_of[s1], t2 = tt_of[s2];
                    const bool act1 = (t1 & 255) > k && t1 >= 0;               // warp-uniform
                    const bool act2 = (s - 1 >= 0) && (t2 & 255) > k && t2 >= 0;
                    if (!act1 && !act2) continue;
                    const double* pa1 = M + gq + 8 * (t1 >> 8) * ld + k0;
                    const double* pb1 = M + gq + 8 * (t1 & 255) * ld + k0;
                    const double* pa2 = M + gq + 8 * (t2 >> 8) * ld + k0;
                    const double* pb2 = M + gq + 8 * (t2 & 255) * ld + k0;
                    double a10 = 0, a11 = 0, b10 = 0, b11 = 0, a20 = 0, a21 = 0, b20 = 0, b21 = 0;
                    if (act1) { a10 = pa1[0]; a11 = pa1[4]; b10 = pb1[0]; b11 = pb1[4]; }
                    if (act2) { a20 = pa2[0]; a21 = pa2[4]; b20 = pb2[0]; b21 = pb2[4]; }
                    if (act1) dmma884(C[s1][0], C[s1][1], -a10, b10);
                    if (act2) dmma884(C[s2][0], C[s2][1], -a20, b20);
                    if (act1) dmma884(C[s1][0], C[s1][1], -a11, b11);
                    if (act2) dmma884(C[s2][0], C[s2][1], -a21, b21);
                    if (act1 && (t1 & 255) == k + 1)           // this tile belongs to the next panel: publish it
                        *reinterpret_cast<double2*>(M + gq + q + 8 * (t1 >> 8) * ld + c0 + 8 * (k + 1)) = make_double2(C[s1][0], C[s1][1]);
                    if (act2 && (t2 & 255) == k + 1)
                        *reinterpret_cast<double2*>(M + gq + q + 8 * (t2 >> 8) * ld + c0 + 8 * (k + 1)) = make_double2(C[s2][0], C[s2][1]);
                }
                // diagonal tiles s > k+1 are updated in place in shared memory, spread over the update warps
                for (int s = k + 2 + uw; s < nts; s += 6) {
                    double* pd = M + (c0 + 8 * s + g) * ld + c0 + 8 * s + 2 * q;
                    const double* pr = M + (c0 + 8 * s + g) * ld + k0 + q;
                    double2 cv = *reinterpret_cast<const double2*>(pd);
                    const double a0 = pr[0], a1 = pr[4];
                    dmma884(cv.x, cv.y, -a0, a0);
                    dmma884(cv.x, cv.y, -a1, a1);
                    *reinterpret_cast<double2*>(pd) = cv;
                }
            } else {                                        // warp 4: right-hand side, aug[j] -= P[j][:] . y
                double y[8];
                f_ld8(qsm + aug + k0, y);
                for (int j = k0 + 8 + lane; j < n; j += 32) {
                    double pr[8];
                    f_ld8(M + j * ld + k0, pr);
                    double acc0 = qsm[aug + j], acc1 = 0.0;
#pragma unroll
                    for (int c = 0; c < 8; c += 2) { acc0 = fma(-pr[c], y[c], acc0); acc1 = fma(-pr[c + 1], y[c + 1], acc1); }
                    qsm[aug + j] = acc0 + acc1;
                }
            }
        }
        QPB_TICK1(48 + k);      // U_k, per step
        __syncthreads();
        QPB_TICK1(44);
    }
}

// n multiple of 8, (n - c0)/8 <= 13, blockDim.x == 256. aug (offset) = right-hand side (length n) carried along so
// that L^-1 aug falls out of the factorization. Two roles with separate register allocations.
__device__ __forceinline__ void f_chol(int A, int ld, int n, int c0, int aug, int tabo) {
    if (threadIdx.x < 32) f_chol_chain(A, ld, n, c0);
    else f_chol_update(A, ld, n, c0, aug, tabo);
}

// ---- triangular solves by substitution on 8-blocks (n multiple of 8) --------------------------------------
// Forward over blocks [kbeg, kend): u[k] = solution entries; b[i >= kend] updated. b destroyed. b != u.
__device__ __noinline__ void f_trsv_fwd(int A, int ld, int n, int kbeg, int kend, int b, int u) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const double* M = qsm + A;
    for (int k0 = kbeg; k0 < kend; k0 += 8) {
        const int nbelow = n - k0 - 8;
        if (tid < nbelow || tid == 0) {
            double Lk[36], y[8], row[8];
            const bool has = tid < nbelow;
            f_ld8(qsm + b + k0, y);
            if (has) f_ld8(M + (k0 + 8 + tid) * ld + k0, row);
            f_load_lower8(M + k0 * ld + k0, ld, Lk);
            double acc0 = has ? qsm[b + k0 + 8 + tid] : 0.0, acc1 = 0.0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                y[c] *= Lk[QPB_LIDX(c, c)];
#pragma unroll
                for (int c2 = c + 1; c2 < 8; ++c2) y[c2] = fma(-y[c], Lk[QPB_LIDX(c2, c)], y[c2]);
                if (has) { if (c & 1) acc1 = fma(-row[c], y[c], acc1); else acc0 = fma(-row[c], y[c], acc0); }
            }
            if (tid == 0) f_st8(qsm + u + k0, y);
            if (has) qsm[b + k0 + 8 + tid] = acc0 + acc1;
        }
        __syncthreads();
    }
}

// Backward: L^T w = u over all blocks. u destroyed. u != w.
__device__ __noinline__ void f_trsv_bwd(int A, int ld, int n, int u, int w) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const double* M = qsm + A;
    for (int k0 = n - 8; k0 >= 0; k0 -= 8) {
        if (tid < k0 || tid == 0) {
            double Lk[36], y[8];
            const bool has = tid < k0;
            f_ld8(qsm + u + k0, y);
            double col[8];
            if (has) {
#pragma unroll
                for (int c = 0; c < 8; ++c) col[c] = M[(k0 + c) * ld + tid];
            }
            f_load_lower8(M + k0 * ld + k0, ld, Lk);
            double acc0 = has ? qsm[u + tid] : 0.0, acc1 = 0.0;
#pragma unroll
            for (int c = 7; c >= 0; --c) {
                y[c] *= Lk[QPB_LIDX(c, c)];
#pragma unroll
                for (int c2 = 0; c2 < c; ++c2) y[c2] = fma(-y[c], Lk[QPB_LIDX(c, c2)], y[c2]);
                if (has) { if (c & 1) acc1 = fma(-col[c], y[c], acc1); else acc0 = fma(-col[c], y[c], acc0); }
            }
            if (tid == 0) f_st8(qsm + w + k0, y);
            if (has) qsm[u + tid] = acc0 + acc1;
        }
        __syncthreads();
    }
}

// Invert a factored 8x8 diagonal block (strictly lower = L, diagonal = 1/L_cc): T = L_kk^-1. T's strictly
// lower part is written TRANSPOSED into the (unused) upper triangle of the block; its diagonal is the
// reciprocal diagonal already there. One lane does the work (pre_factor_kkt only; off the Newton loop).
__device__ __noinline__ void f_invert8(int Mb_off, int ld) {
    QPB_SMEM;
    double* Mb = qsm + Mb_off;
    if ((threadIdx.x & 31) == 0) {
        double Lk[36], T[36];
        f_load_lower8(Mb, ld, Lk);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            T[QPB_LIDX(c, c)] = Lk[QPB_LIDX(c, c)];
#pragma unroll
            for (int r = c + 1; r < 8; ++r) {
                double sacc = 0.0;
#pragma unroll
                for (int j = c; j < r; ++j) sacc = fma(Lk[QPB_LIDX(r, j)], T[QPB_LIDX(j, c)], sacc);
                T[QPB_LIDX(r, c)] = -Lk[QPB_LIDX(r, r)] * sacc;
            }
        }
#pragma unroll
        for (int r = 1; r < 8; ++r)
#pragma unroll
            for (int c = 0; c < r; ++c) Mb[c * ld + r] = T[QPB_LIDX(r, c)];
    }
    __syncwarp();
}

// W row tile `rt` (8 rows) <- rows * L^-T for the factored n x n matrix at A (n multiple of 8, diagonal blocks
// in the reciprocal-diagonal convention with T^T in their upper triangles). Left-looking over column tiles,
// all inside ONE warp: no block-level synchronisation, row tiles are independent of each other.
__device__ __noinline__ void f_rows_times_LinvT(int A, int ld, int n, int Wm, int ldw, int rt) {
    QPB_SMEM;
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const double* M = qsm + A;
    double* Wp = qsm + Wm + (8 * rt + g) * ldw;              // this lane's row of the tile
    const int nct = n >> 3;
    for (int j = 0; j < nct; ++j) {
        double2 cv = *reinterpret_cast<const double2*>(Wp + 8 * j + 2 * q);
        const double* pb = M + (8 * j + g) * ld + q;         // rows of block j of L, panel columns follow
        for (int i = 0; i < j; ++i) {
            const double a0 = Wp[8 * i + q], a1 = Wp[8 * i + 4 + q];
            const double b0 = pb[8 * i], b1 = pb[8 * i + 4];
            dmma884(cv.x, cv.y, -a0, b0);
            dmma884(cv.x, cv.y, -a1, b1);
        }
        *reinterpret_cast<double2*>(Wp + 8 * j + 2 * q) = cv;
        __syncwarp();
        // tile <- tile * T_jj^T   (B[k][nn] = T[nn][k]; T lower: reciprocal diagonal, strictly lower part stored transposed)
        const double a0 = Wp[8 * j + q], a1 = Wp[8 * j + 4 + q];
        const double* Tb = M + (8 * j) * ld + 8 * j;
        const int c0 = q, c1 = 4 + q;
        const double b0 = (c0 < g) ? Tb[c0 * ld + g] : (c0 == g ? Tb[g * ld + g] : 0.0);
        const double b1 = (c1 < g) ? Tb[c1 * ld + g] : (c1 == g ? Tb[g * ld + g] : 0.0);
        double d0 = 0.0, d1 = 0.0;
        dmma884(d0, d1, a0, b0);
        dmma884(d0, d1, a1, b1);
        __syncwarp();
        *reinterpret_cast<double2*>(Wp + 8 * j + 2 * q) = make_double2(d0, d1);
        __syncwarp();
    }
}

// ---- packed-L substitution (x~ = L^-1 x, x = L^-T x~): twice per kernel, off the hot loop ----------------
__device__ __noinline__ void f_whiten(int Lp, int n, int dinvL, int b, int u) {
    QPB_SMEM;
    trsv_fwd(qsm + Lp, PackedIdx{}, n, 0, n, qsm + dinvL, qsm + b, qsm + u, (int)threadIdx.x, kNT);
}
__device__ __noinline__ void f_unwhiten(int Lp, int n, int dinvL, int u, int w) {
    QPB_SMEM;
    trsv_bwd(qsm + Lp, PackedIdx{}, n, qsm + dinvL, qsm + u, qsm + w, (int)threadIdx.x, kNT);
}

// ---- mat-vecs with W (rows x cols, ld) ---------------------------------------------------------------------
// CODE SIZE is a first-class constraint in this file: the Newton loop runs ~150 KB of SASS once per iteration in
// the first version, against a 32 KB L1.5 instruction cache, and ncu/clock64 accounting showed every cold phase
// costing ~0.5 cycle per byte of code it touches (a 16-26 KB single-warp routine: 15-20k cycles for ~1000
// executed instructions). Loops below are therefore rolled (unroll 1-2) and long expansions (fp64 divide, sqrt,
// reductions) are shared subroutines.
//
// y1 = W x1 (, y2 = W x2): 2 lanes per row, 128 rows per pass; lane h of a pair takes the 16-byte column pairs
// 4k + 2h, so a quarter-warp's LDS.128 hits 8 distinct 16-byte bank groups for any ld % 8 == 4.
template <bool kTwo>
__device__ __forceinline__ void f_matvec_rows_impl(int W, int ld, int rows, int cols, int x1, int x2, int y1, int y2) {
    QPB_SMEM;
    const int tid = threadIdx.x, h = tid & 1;
    for (int rb = 0; rb < rows; rb += kNT / 2) {
        const int r = rb + (tid >> 1);
        const bool ok = r < rows;
        const double* a = qsm + W + (ok ? r : 0) * ld + 2 * h;
        double s1a = 0.0, s1b = 0.0, s2a = 0.0, s2b = 0.0;
#pragma unroll 2
        for (int c = 2 * h; c < cols; c += 4, a += 4) {
            const double2 w = *reinterpret_cast<const double2*>(a);
            const double2 u = *reinterpret_cast<const double2*>(qsm + x1 + c);
            const bool hi = c + 1 < cols;                     // odd cols: neither W[r][cols] nor x[cols] is ours
            const double wy = hi ? w.y : 0.0;
            s1a = fma(w.x, u.x, s1a); s1b = fma(wy, hi ? u.y : 0.0, s1b);
            if (kTwo) {
                const double2 v = *reinterpret_cast<const double2*>(qsm + x2 + c);
                s2a = fma(w.x, v.x, s2a); s2b = fma(wy, hi ? v.y : 0.0, s2b);
            }
        }
        double s1 = s1a + s1b, s2 = s2a + s2b;
        __syncwarp();                                        // converged warp -> the shuffles take their fast path
        s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
        if (kTwo) s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
        if (ok && h == 0) {
            qsm[y1 + r] = s1;
            if (kTwo) qsm[y2 + r] = s2;
        }
    }
}
__device__ __noinline__ void f_matvec_rows2(int W, int ld, int rows, int cols, int x1, int x2, int y1, int y2) {
    f_matvec_rows_impl<true>(W, ld, rows, cols, x1, x2, y1, y2);
}
__device__ __noinline__ void f_matvec_rows1(int W, int ld, int rows, int cols, int x1, int y1) {
    f_matvec_rows_impl<false>(W, ld, rows, cols, x1, 0, y1, 0);
}
// out[c] = a[c] + sgn * (W^T v)[c] (+ b[c] if b >= 0). Two row groups, partial sums in p0/p1.
__device__ __noinline__ void f_matvec_cols(int W, int ld, int rows, int cols, int v, int p0, int p1, int out,
                                           int a, double sa, int b, double sgn) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const int half = kNT / 2;
    const int gidx = tid / half, c = tid - gidx * half;
    const int chunk = (rows + 1) >> 1;
    for (int c0 = 0; c0 < cols; c0 += half) {
        const int cc = c0 + c;
        if (cc < cols) {
            const int r0 = gidx * chunk, r1 = min(rows, r0 + chunk);
            const double* Wp = qsm + W + cc;
            double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
            int r = r0;
#pragma unroll 1
            for (; r + 3 < r1; r += 4) {
                s0 = fma(Wp[(r + 0) * ld], qsm[v + r + 0], s0);
                s1 = fma(Wp[(r + 1) * ld], qsm[v + r + 1], s1);
                s2 = fma(Wp[(r + 2) * ld], qsm[v + r + 2], s2);
                s3 = fma(Wp[(r + 3) * ld], qsm[v + r + 3], s3);
            }
#pragma unroll 1
            for (; r < r1; ++r) s0 = fma(Wp[r * ld], qsm[v + r], s0);
            qsm[(gidx ? p1 : p0) + cc] = (s0 + s1) + (s2 + s3);
        }
    }
    __syncthreads();
    for (int cc = tid; cc < cols; cc += kNT) {
        double r = sa * qsm[a + cc] + sgn * (qsm[p0 + cc] + qsm[p1 + cc]);
        if (b >= 0) r += qsm[b + cc];
        qsm[out + cc] = r;
    }
    __syncthreads();
}

// End of a Newton iteration, column c: dx~ = -r~x - (W^T dv)_c, x~ += alpha dx~, r~x = x~ + (W^T v)_c + p~
// (each with the rounding of the separate passes it replaces).
__device__ __forceinline__ void f_cols2_out(int c, double wdv, double wv, int xt, int rxt, int pt, double alpha) {
    QPB_SMEM;
    const double dx = -qsm[rxt + c] - wdv;
    const double x = fma(alpha, dx, qsm[xt + c]);
    qsm[xt + c] = x;
    qsm[rxt + c] = (x + wv) + qsm[pt + c];
}
// W^T dv and W^T v side by side (each W element read once) with the row split and summation order of
// f_matvec_cols; partial sums in p0/p1 (dv) and p2/p3 (v). Ends with a block barrier.
__device__ __noinline__ void f_matvec_cols2(int W, int ld, int rows, int cols, int dv, int v, int p0, int p1, int p2,
                                            int p3, int xt, int rxt, int pt, double alpha) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const int half = kNT / 2;
    const int gidx = tid / half, c = tid - gidx * half;
    const int chunk = (rows + 1) >> 1;
    for (int c0 = 0; c0 < cols; c0 += half) {
        const int cc = c0 + c;
        if (cc < cols) {
            const int r0 = gidx * chunk, r1 = min(rows, r0 + chunk);
            const double* Wp = qsm + W + cc;
            double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, u0 = 0.0, u1 = 0.0, u2 = 0.0, u3 = 0.0;
            int r = r0;
#pragma unroll 1
            for (; r + 3 < r1; r += 4) {
                const double w0 = Wp[(r + 0) * ld], w1 = Wp[(r + 1) * ld], w2 = Wp[(r + 2) * ld], w3 = Wp[(r + 3) * ld];
                s0 = fma(w0, qsm[dv + r + 0], s0); u0 = fma(w0, qsm[v + r + 0], u0);
                s1 = fma(w1, qsm[dv + r + 1], s1); u1 = fma(w1, qsm[v + r + 1], u1);
                s2 = fma(w2, qsm[dv + r + 2], s2); u2 = fma(w2, qsm[v + r + 2], u2);
                s3 = fma(w3, qsm[dv + r + 3], s3); u3 = fma(w3, qsm[v + r + 3], u3);
            }
#pragma unroll 1
            for (; r < r1; ++r) {
                const double w0 = Wp[r * ld];
                s0 = fma(w0, qsm[dv + r], s0); u0 = fma(w0, qsm[v + r], u0);
            }
            qsm[(gidx ? p1 : p0) + cc] = (s0 + s1) + (s2 + s3);
            qsm[(gidx ? p3 : p2) + cc] = (u0 + u1) + (u2 + u3);
        }
    }
    __syncthreads();
    for (int cc = tid; cc < cols; cc += kNT)
        f_cols2_out(cc, qsm[p0 + cc] + qsm[p1 + cc], qsm[p2 + cc] + qsm[p3 + cc], xt, rxt, pt, alpha);
    __syncthreads();
}

// || L x ||^2 partial sums (packed lower L in shared memory): 4 lanes per row, rows paired (r, n-1-r) so that every
// lane group streams n + 1 entries. Returns this thread's partial (lane l == 0 of a group); sum over the block after.
__device__ __noinline__ double f_tri_norm2(int Lp, int n, int x) {
    QPB_SMEM;
    const int tid = threadIdx.x, q4 = tid >> 2, l = tid & 3;
    double acc = 0.0;
    const int npairs = (n + 1) >> 1;
    for (int pb = 0; pb < npairs; pb += kNT / 4) {           // warp-uniform trip count
        const int pi = pb + q4;
        const bool act = pi < npairs;
        const int ra = act ? pi : 0, rb = n - 1 - ra;
        const double* La = qsm + Lp + (ra * (ra + 1)) / 2;
        const double* Lb = qsm + Lp + (rb * (rb + 1)) / 2;
        double sa = 0.0, sb = 0.0;
        if (act) {
#pragma unroll 2
            for (int c = l; c <= ra; c += 4) sa = fma(La[c], qsm[x + c], sa);
            if (rb != ra) {
#pragma unroll 2
                for (int c = l; c <= rb; c += 4) sb = fma(Lb[c], qsm[x + c], sb);
            }
        }
        __syncwarp();                                        // (the row loops above diverge)
        sa += __shfl_xor_sync(0xffffffffu, sa, 1); sb += __shfl_xor_sync(0xffffffffu, sb, 1);
        sa += __shfl_xor_sync(0xffffffffu, sa, 2); sb += __shfl_xor_sync(0xffffffffu, sb, 2);
        if (l == 0) acc = fma(sa, sa, fma(sb, sb, acc));
    }
    return acc;
}

// ---- co-resident mode (two CTAs per SM): W and packed L stay in GLOBAL memory ---------------------------------
// Shared memory per CTA then holds only the S workspace and the vectors (107 KB at C2), so two QPs share an SM and
// each one's latency chains (Cholesky pivots, substitutions, reductions) run in the other's bubbles. The passes over
// W (80 KB) and L (40 KB) become L2 reads: every element is used once per pass, so staging it in shared memory would
// buy nothing; what matters is the number of loads in flight, hence the register batches below (one L2 round trip
// per batch). The factors were written by the previous launch and are read-only here: ld.global.nc.
__device__ __forceinline__ double2 ldg2(const double* p) { return __ldg(reinterpret_cast<const double2*>(p)); }

// y1 = W x1 (, y2 = W x2). 8 lanes per row (lane j: 16-byte column pairs 2j + 16k), kNT/8 rows per pass, two passes
// (14 loads) in flight per thread. Row groups are numbered from the LAST warp, so a partial last pass (rows 96-99 at
// C2 with 192 threads) falls to the highest warps: warp 0 already carries the partial pass of g_tri_norm2, which
// shares this phase in the forward kernel.
template <bool kTwo>
__device__ __forceinline__ void g_matvec_rows_impl(const double* __restrict__ Wg, int ld, int rows, int cols, int x1,
                                                   int x2, int y1, int y2) {
    QPB_SMEM;
    constexpr int kRG = kNT / 8;                             // row groups per pass (8 lanes per row)
    const int tid = threadIdx.x, j = tid & 7, rg = kRG - 1 - (tid >> 3);
#pragma unroll 1
    for (int rb = 0; rb < rows; rb += 2 * kRG) {             // warp-uniform trip count
        const int r0 = rb + rg, r1 = r0 + kRG;
        const bool ok0 = r0 < rows, ok1 = r1 < rows;
        const double* p0 = Wg + (size_t)(ok0 ? r0 : 0) * ld;
        const double* p1 = Wg + (size_t)(ok1 ? r1 : 0) * ld;
        double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;       // row r0: (x1, x2); row r1: (x1, x2)
#pragma unroll 1
        for (int cb = 2 * j; cb < cols; cb += 112) {
            double2 w0[7], w1[7];
#pragma unroll
            for (int k = 0; k < 7; ++k) {
                const int c = cb + 16 * k;
                const bool in = c < cols;
                w0[k] = in ? ldg2(p0 + c) : make_double2(0.0, 0.0);
                w1[k] = in ? ldg2(p1 + c) : make_double2(0.0, 0.0);
            }
#pragma unroll
            for (int k = 0; k < 7; ++k) {
                const int c = cb + 16 * k;
                if (c < cols) {
                    const bool hi = c + 1 < cols;             // odd cols: neither W[r][cols] nor x[cols] is ours
                    double2 u = *reinterpret_cast<const double2*>(qsm + x1 + c);
                    if (!hi) u.y = 0.0;
                    const double wy0 = hi ? w0[k].y : 0.0, wy1 = hi ? w1[k].y : 0.0;
                    a0 = fma(w0[k].x, u.x, a0); a0 = fma(wy0, u.y, a0);
                    b0 = fma(w1[k].x, u.x, b0); b0 = fma(wy1, u.y, b0);
                    if (kTwo) {
                        double2 v = *reinterpret_cast<const double2*>(qsm + x2 + c);
                        if (!hi) v.y = 0.0;
                        a1 = fma(w0[k].x, v.x, a1); a1 = fma(wy0, v.y, a1);
                        b1 = fma(w1[k].x, v.x, b1); b1 = fma(wy1, v.y, b1);
                    }
                }
            }
        }
        __syncwarp();                                        // converged warp -> the shuffles take their fast path
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            a0 += __shfl_xor_sync(0xffffffffu, a0, o);
            b0 += __shfl_xor_sync(0xffffffffu, b0, o);
            if (kTwo) {
                a1 += __shfl_xor_sync(0xffffffffu, a1, o);
                b1 += __shfl_xor_sync(0xffffffffu, b1, o);
            }
        }
        if (j == 0) {
            if (ok0) { qsm[y1 + r0] = a0; if (kTwo) qsm[y2 + r0] = a1; }
            if (ok1) { qsm[y1 + r1] = b0; if (kTwo) qsm[y2 + r1] = b1; }
        }
    }
}
__device__ __noinline__ void g_matvec_rows2(const double* __restrict__ Wg, int ld, int rows, int cols, int x1, int x2,
                                            int y1, int y2) {
    g_matvec_rows_impl<true>(Wg, ld, rows, cols, x1, x2, y1, y2);
}
__device__ __noinline__ void g_matvec_rows1(const double* __restrict__ Wg, int ld, int rows, int cols, int x1, int y1) {
    g_matvec_rows_impl<false>(Wg, ld, rows, cols, x1, 0, y1, 0);
}

// out[c] = sa * a[c] + sgn * (W^T v)[c] (+ b[c] if b >= 0). A warp owns 16 columns: lane = (row group g, column pair
// cq), a warp-wide load touches 4 rows x 128 contiguous bytes; the four row groups are summed with two shuffles.
// Ends with a block barrier (out is complete for every thread).
__device__ __noinline__ void g_matvec_cols(const double* __restrict__ Wg, int ld, int rows, int cols, int v, int out,
                                           int a, double sa, int b, double sgn) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 3, cq = lane & 7;
#pragma unroll 1
    for (int c0 = 0; c0 < cols; c0 += 16 * (kNT / 32)) {     // warp-uniform trip count
        const int c = c0 + 16 * warp + 2 * cq;
        const bool okc = c < cols;
        const double* pc = Wg + (okc ? c : 0);
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 1
        for (int rb = g; rb < rows; rb += 4 * 13) {
            double2 w[13];
#pragma unroll
            for (int k = 0; k < 13; ++k) {
                const int r = rb + 4 * k;
                w[k] = (r < rows) ? ldg2(pc + (size_t)r * ld) : make_double2(0.0, 0.0);
            }
#pragma unroll
            for (int k = 0; k < 13; ++k) {
                const int r = rb + 4 * k;
                if (r < rows) {
                    const double vr = qsm[v + r];
                    s0 = fma(w[k].x, vr, s0);
                    s1 = fma(w[k].y, vr, s1);
                }
            }
        }
        __syncwarp();
        s0 += __shfl_xor_sync(0xffffffffu, s0, 8);  s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
        s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        if (g == 0 && okc) {
            double r0 = sa * qsm[a + c] + sgn * s0;
            if (b >= 0) r0 += qsm[b + c];
            qsm[out + c] = r0;
            if (c + 1 < cols) {
                double r1 = sa * qsm[a + c + 1] + sgn * s1;
                if (b >= 0) r1 += qsm[b + c + 1];
                qsm[out + c + 1] = r1;
            }
        }
    }
    __syncthreads();
}

// W^T dv and W^T v side by side, each W element loaded once, with the lane/row pairing and shuffle tree of
// g_matvec_cols; the owning lane finishes its columns with f_cols2_out. Ends with a block barrier.
__device__ __noinline__ void g_matvec_cols2(const double* __restrict__ Wg, int ld, int rows, int cols, int dv, int v,
                                            int xt, int rxt, int pt, double alpha) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 3, cq = lane & 7;
#pragma unroll 1
    for (int c0 = 0; c0 < cols; c0 += 16 * (kNT / 32)) {     // warp-uniform trip count
        const int c = c0 + 16 * warp + 2 * cq;
        const bool okc = c < cols;
        const double* pc = Wg + (okc ? c : 0);
        double s0 = 0.0, s1 = 0.0, u0 = 0.0, u1 = 0.0;       // W^T dv, W^T v
#pragma unroll 1
        for (int rb = g; rb < rows; rb += 4 * 13) {
            double2 w[13];
#pragma unroll
            for (int k = 0; k < 13; ++k) {
                const int r = rb + 4 * k;
                w[k] = (r < rows) ? ldg2(pc + (size_t)r * ld) : make_double2(0.0, 0.0);
            }
#pragma unroll
            for (int k = 0; k < 13; ++k) {
                const int r = rb + 4 * k;
                if (r < rows) {
                    const double dr = qsm[dv + r], vr = qsm[v + r];
                    s0 = fma(w[k].x, dr, s0);
                    s1 = fma(w[k].y, dr, s1);
                    u0 = fma(w[k].x, vr, u0);
                    u1 = fma(w[k].y, vr, u1);
                }
            }
        }
        __syncwarp();
        s0 += __shfl_xor_sync(0xffffffffu, s0, 8);  s1 += __shfl_xor_sync(0xffffffffu, s1, 8);
        u0 += __shfl_xor_sync(0xffffffffu, u0, 8);  u1 += __shfl_xor_sync(0xffffffffu, u1, 8);
        s0 += __shfl_xor_sync(0xffffffffu, s0, 16); s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        u0 += __shfl_xor_sync(0xffffffffu, u0, 16); u1 += __shfl_xor_sync(0xffffffffu, u1, 16);
        if (g == 0 && okc) {
            f_cols2_out(c, s0, u0, xt, rxt, pt, alpha);
            if (c + 1 < cols) f_cols2_out(c + 1, s1, u1, xt, rxt, pt, alpha);
        }
    }
    __syncthreads();
}

// || L x ||^2 partial sums with the packed lower L in global memory: same lane/row pairing as f_tri_norm2.
__device__ __noinline__ double g_tri_norm2(const double* __restrict__ Lg, int n, int x) {
    QPB_SMEM;
    const int tid = threadIdx.x, q4 = tid >> 2, l = tid & 3;
    double acc = 0.0;
    const int npairs = (n + 1) >> 1;
    for (int pb = 0; pb < npairs; pb += kNT / 4) {           // warp-uniform trip count
        const int pi = pb + q4;
        const bool act = pi < npairs;
        const int ra = act ? pi : 0, rb = n - 1 - ra;
        const double* La = Lg + (ra * (ra + 1)) / 2;
        const double* Lb = Lg + (rb * (rb + 1)) / 2;
        double sa = 0.0, sb = 0.0;
        if (act) {
#pragma unroll 1
            for (int cb = l; cb <= rb; cb += 4 * 13) {       // row rb >= row ra: one loop covers both
                double wa[13], wb[13];
#pragma unroll
                for (int k = 0; k < 13; ++k) {
                    const int c = cb + 4 * k;
                    wb[k] = (c <= rb) ? __ldg(Lb + c) : 0.0;
                    wa[k] = (c <= ra && rb != ra) ? __ldg(La + c) : 0.0;
                }
#pragma unroll
                for (int k = 0; k < 13; ++k) {
                    const int c = cb + 4 * k;
                    if (c <= rb) {
                        const double xc = qsm[x + c];
                        sb = fma(wb[k], xc, sb);
                        sa = fma(wa[k], xc, sa);
                    }
                }
            }
        }
        __syncwarp();                                        // (the row loops above diverge)
        sa += __shfl_xor_sync(0xffffffffu, sa, 1); sb += __shfl_xor_sync(0xffffffffu, sb, 1);
        sa += __shfl_xor_sync(0xffffffffu, sa, 2); sb += __shfl_xor_sync(0xffffffffu, sb, 2);
        if (l == 0) acc = fma(sa, sa, fma(sb, sb, acc));
    }
    return acc;
}

constexpr int kFastStride = (kNT / 32 <= 8) ? 8 : 16;       // per-value stride of the fast kernels' reduction scratch
__device__ __noinline__ void f_reduce_sum4(double (&v)[4], int red) {
    QPB_SMEM;
    block_reduce<4, false, kFastStride>(v, qsm + red, (int)threadIdx.x, kNT);
}
__device__ __noinline__ void f_reduce_sum2(double (&v)[2], int red) {
    QPB_SMEM;
    block_reduce<2, false, kFastStride>(v, qsm + red, (int)threadIdx.x, kNT);
}
__device__ __noinline__ void f_reduce_min2(double (&v)[2], int red) {
    QPB_SMEM;
    block_reduce<2, true, kFastStride>(v, qsm + red, (int)threadIdx.x, kNT);
}

}  // namespace fast
}  // namespace qpb
