// Device-side building blocks of the per-QP interior-point solve (sm_90a, fp64).
//
// One CTA owns one QP.  All matrices the Newton loop touches are dense, row-major,
// and live in shared memory (or, for shapes that do not fit 227 KB, in an L2-resident
// global scratch — same code, different pointers).  Leading dimensions are chosen
// with ld % 8 == 4 so that the "4 lanes x 4 consecutive doubles per row" access
// pattern used by the DMMA fragments and the row mat-vecs is bank-conflict free.
//
// Reference functions these pieces implement (qpth/solvers/pdipm/batch.py):
//   chol_partial  <- factor_kkt :435-470 (Cholesky of R + D^-1 instead of pivoted LU;
//                    also pre_factor_kkt's factorizations :375-429)
//   trsv_fwd/bwd  <- the lu_solve calls of solve_kkt :349-372
//   matvec_*      <- the bmm mat-vecs of forward :94-101 and solve_kkt :355-364
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace qpb {

#define QPB_LIDX(r, c) (((r) * ((r) + 1)) / 2 + (c))

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

// Both reductions start with __syncwarp(): they are called after loops whose trip count differs between lanes
// (for (i = tid; i < ms; ...)). Without it the compiler cannot prove convergence and the shuffles go through their
// divergent-warp fallback (BRA.DIV -> WARPSYNC.COLLECTIVE per shuffle), several times slower.
__device__ __forceinline__ double warp_sum(double v) {
    __syncwarp();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// min that propagates nothing special: callers only feed non-NaN candidates or +inf
__device__ __forceinline__ double warp_min(double v) {
    __syncwarp();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}


// ---- matrix accessors: full row-major with leading dimension, or packed lower triangle
struct FullIdx {
    int ld;
    __device__ __forceinline__ int operator()(int r, int c) const { return r * ld + c; }
};
struct PackedIdx {
    __device__ __forceinline__ int operator()(int r, int c) const { return (r * (r + 1)) / 2 + c; }
};

// ---- mbarrier + 1-D TMA bulk copy (global -> shared), the sm_90 async-proxy path (SASS: UBLKCP)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
// order prior generic-proxy accesses to shared memory before subsequent async-proxy (TMA) writes
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
// bytes must be a multiple of 16; src and dst 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// Issue a contiguous copy as 16 KB chunks from ONE thread (rolled loop). The barrier must already have been armed
// (mbar_expect_tx) with the total byte count of everything that will land on it. (cp.async.bulk takes uniform
// operands: issued per lane, every call site became a serialised elect loop and ~2 KB of SASS.)
__device__ __forceinline__ void bulk_issue_thread(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    const uint32_t chunk = 16384;
#pragma unroll 1
    for (uint32_t off = 0; off < bytes; off += chunk) {
        const uint32_t nb = (bytes - off < chunk) ? (bytes - off) : chunk;
        bulk_g2s((char*)dst_smem + off, (const char*)src_gmem + off, nb, bar);
    }
}
// (lane-parallel variant, kept for the generic kernels)
__device__ __forceinline__ void bulk_issue_warp(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                                uint64_t* bar, int lane) {
    const uint32_t chunk = 16384;
    for (uint32_t off = (uint32_t)lane * chunk; off < bytes; off += 32u * chunk) {
        const uint32_t nb = (bytes - off < chunk) ? (bytes - off) : chunk;
        bulk_g2s((char*)dst_smem + off, (const char*)src_gmem + off, nb, bar);
    }
}

// || L x ||^2 contributions for the packed lower factor L (n x n): each warp owns rows, returns this
// thread's partial (only lane 0 of each warp carries a value; sum over the block afterwards).
__device__ __forceinline__ double tri_norm2_partial(const double* Lp, int n, const double* x, int tid, int nt) {
    const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    double acc = 0.0;
    for (int r = warp; r < n; r += nw) {
        const double* Lr = Lp + (r * (r + 1)) / 2;
        double s0 = 0.0, s1 = 0.0;
        int c = lane;
        for (; c + 32 <= r; c += 64) {
            s0 = fma(Lr[c], x[c], s0);
            s1 = fma(Lr[c + 32], x[c + 32], s1);
        }
        if (c <= r) s0 = fma(Lr[c], x[c], s0);
        const double s = warp_sum(s0 + s1);
        if (lane == 0) acc = fma(s, s, acc);
    }
    return acc;
}

// Block-wide reductions of N values. `red` is shared scratch of >= N * kRedStride doubles (up to 16 warps).
constexpr int kRedStride = 16;
// Every thread returns with the reduced values. Two barriers per call.
template <int N, bool kMin, int kStride = kRedStride>
__device__ __forceinline__ void block_reduce(double (&v)[N], double* red, int tid, int nt) {
    const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = kMin ? warp_min(v[k]) : warp_sum(v[k]);
    __syncthreads();                                         // protect scratch from the previous call's readers
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) red[k * kStride + warp] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        double a = kMin ? INFINITY : 0.0;
        for (int w = 0; w < nw; ++w) a = kMin ? fmin(a, red[k * kStride + w]) : a + red[k * kStride + w];
        v[k] = a;
    }
}

// dst[r*ldd + c] = src[r*lds + c]   (rows x cols), warp per row, coalesced.
__device__ __forceinline__ void copy_matrix(double* dst, int ldd, const double* src, int64_t lds,
                                            int rows, int cols, int tid, int nt) {
    const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    for (int r = warp; r < rows; r += nw) {
        const double* s = src + (int64_t)r * lds;
        double* d = dst + r * ldd;
        for (int c = lane; c < cols; c += 32) d[c] = s[c];
    }
}

// y1 = A x1, y2 = A x2 (A rows x cols, row-major). 4 lanes per row. kTwo=false ignores x2/y2.
// Optional epilogue is left to the caller (results land in y1/y2).
template <bool kTwo>
__device__ __forceinline__ void matvec_rows(const double* A, int ld, int rows, int cols,
                                            const double* x1, const double* x2, double* y1,
                                            double* y2, int tid, int nt) {
    const int q = tid >> 2, l = tid & 3, nq = nt >> 2;
    for (int rb = 0; rb < rows; rb += nq) {
        const int r = rb + q;
        const bool ok = r < rows;
        const double* a = A + (ok ? r : 0) * ld;
        double s1a = 0.0, s1b = 0.0, s2a = 0.0, s2b = 0.0;
        int c = l;
        for (; c + 4 < cols; c += 8) {
            const double a0 = ok ? a[c] : 0.0, a1 = ok ? a[c + 4] : 0.0;
            s1a = fma(a0, x1[c], s1a);
            s1b = fma(a1, x1[c + 4], s1b);
            if (kTwo) {
                s2a = fma(a0, x2[c], s2a);
                s2b = fma(a1, x2[c + 4], s2b);
            }
        }
        if (c < cols) {
            const double a0 = ok ? a[c] : 0.0;
            s1a = fma(a0, x1[c], s1a);
            if (kTwo) s2a = fma(a0, x2[c], s2a);
        }
        double s1 = s1a + s1b, s2 = s2a + s2b;
        s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
        s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
        if (kTwo) {
            s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
            s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
        }
        if (ok && l == 0) {
            y1[r] = s1;
            if (kTwo) y2[r] = s2;
        }
    }
}

// part[g*vl + c] = sum over row-chunk g of A[r][c] * v[r]; caller sums the G chunks after a barrier.
// Returns G (number of chunks). Thread per column, rows split over G thread groups.
__device__ __forceinline__ int matvec_cols_partial(const double* A, int ld, int rows, int cols,
                                                   const double* v, double* part, int vl, int tid,
                                                   int nt) {
    const int cg = (cols + 31) & ~31;
    int G = nt / cg;
    if (G < 1) G = 1;
    if (G > 4) G = 4;
    const int chunk = (rows + G - 1) / G;
    for (int idx = tid; idx < G * cg; idx += nt) {
        const int g = idx / cg, c = idx - g * cg;
        if (c >= cols) continue;
        const int r0 = g * chunk, r1 = min(rows, r0 + chunk);
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int r = r0;
        for (; r + 3 < r1; r += 4) {
            s0 = fma(A[(r + 0) * ld + c], v[r + 0], s0);
            s1 = fma(A[(r + 1) * ld + c], v[r + 1], s1);
            s2 = fma(A[(r + 2) * ld + c], v[r + 2], s2);
            s3 = fma(A[(r + 3) * ld + c], v[r + 3], s3);
        }
        for (; r < r1; ++r) s0 = fma(A[r * ld + c], v[r], s0);
        part[g * vl + c] = (s0 + s1) + (s2 + s3);
    }
    return G;
}

// Blocked right-looking Cholesky of columns [c0, c1) of the nsq x nsq lower matrix A (ld),
// trailing updates applied to the whole remaining square and to the nx "extra" rows X (ldx)
// that ride along below it (right-hand sides fused into the factorization, or the G/A rows
// in pre_factor_kkt).  dinv[k] receives 1 / L[k][k].  c0 must be a multiple of 8.
// flag (may be null): set to 1 if a pivot is not > 0.
__device__ __forceinline__ void chol_partial(double* A, int ld, int nsq, int c0, int c1, double* X,
                                             int ldx, int nx, double* dinv, int* flag, int tid,
                                             int nt) {
    const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    for (int k0 = c0; k0 < c1; k0 += 8) {
        const int nb = min(8, c1 - k0);
        const int nsr = nsq - k0;      // square rows at/below the diagonal block
        const int nrows = nsr + nx;
        if (tid < nrows) {
            // ---- diagonal block, factored redundantly in registers by every row-owning thread
            double Lk[36], rinv[8];
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int c = 0; c <= r; ++c)
                    Lk[QPB_LIDX(r, c)] = (r < nb && c < nb) ? A[(k0 + r) * ld + k0 + c]
                                                             : (r == c ? 1.0 : 0.0);
            bool bad = false;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const double piv = Lk[QPB_LIDX(c, c)];
                bad = bad || !(piv > 0.0);
                const double ri = rsqrt(piv);
                rinv[c] = ri;
                Lk[QPB_LIDX(c, c)] = piv * ri;
#pragma unroll
                for (int r = c + 1; r < 8; ++r) Lk[QPB_LIDX(r, c)] *= ri;
#pragma unroll
                for (int r = c + 1; r < 8; ++r)
#pragma unroll
                    for (int cc = c + 1; cc <= r; ++cc)
                        Lk[QPB_LIDX(r, cc)] = fma(-Lk[QPB_LIDX(r, c)], Lk[QPB_LIDX(cc, c)],
                                                  Lk[QPB_LIDX(r, cc)]);
            }
            if (tid == 0) {
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < nb) dinv[k0 + c] = rinv[c];
                if (flag != nullptr && bad) *flag = 1;
            }
            // ---- own row(s) of the panel: a <- a * Lkk^-T  (diag rows reproduce L's own rows)
            for (int t = tid; t < nrows; t += nt) {
                double* rowp = (t < nsr) ? (A + (k0 + t) * ld + k0) : (X + (t - nsr) * ldx + k0);
                double a[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) a[c] = (c < nb) ? rowp[c] : 0.0;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    a[c] *= rinv[c];
#pragma unroll
                    for (int c2 = c + 1; c2 < 8; ++c2)
                        a[c2] = fma(-a[c], Lk[QPB_LIDX(c2, c)], a[c2]);
                }
                const int cmax = (t < nb) ? t : (nb - 1);   // diag rows: lower part only
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c <= cmax) rowp[c] = a[c];
            }
        }
        __syncthreads();
        // ---- trailing update with DMMA 8x8x4 tiles: C -= P_rows * P_cols^T
        const int r0 = k0 + 8;
        if (nb == 8 && r0 < nsq) {
            const int nts = (nsq - r0 + 7) >> 3;
            const int tri = nts * (nts + 1) / 2;
            const int ntr = (nx + 7) >> 3;
            const int T = tri + ntr * nts;
            const int g = lane >> 2, q = lane & 3;
            for (int t = warp; t < T; t += nw) {
                int ti, tj, rbase, rbound, ldr;
                double* rptr;
                if (t < tri) {
                    ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
                    while (ti * (ti + 1) / 2 > t) --ti;
                    while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
                    tj = t - ti * (ti + 1) / 2;
                    rptr = A; ldr = ld; rbase = r0 + 8 * ti; rbound = nsq;
                } else {
                    const int t2 = t - tri;
                    ti = t2 / nts; tj = t2 - ti * nts;
                    rptr = X; ldr = ldx; rbase = 8 * ti; rbound = nx;
                }
                const int cb = r0 + 8 * tj;
                const int rr = rbase + g, br = cb + g;
                const bool rok = rr < rbound, bok = br < nsq;
                const double* pa = rptr + (rok ? rr : 0) * ldr + k0 + q;
                const double* pb = A + (bok ? br : 0) * ld + k0 + q;
                const double a0 = rok ? pa[0] : 0.0, a1 = rok ? pa[4] : 0.0;
                const double b0 = bok ? pb[0] : 0.0, b1 = bok ? pb[4] : 0.0;
                double* pc = rptr + (rok ? rr : 0) * ldr + cb + 2 * q;
                const bool k0ok = rok && (cb + 2 * q < nsq), k1ok = rok && (cb + 2 * q + 1 < nsq);
                double cc0 = k0ok ? pc[0] : 0.0, cc1 = k1ok ? pc[1] : 0.0;
                dmma884(cc0, cc1, -a0, b0);
                dmma884(cc0, cc1, -a1, b1);
                if (k0ok) pc[0] = cc0;
                if (k1ok) pc[1] = cc1;
            }
        }
        __syncthreads();
    }
}

// Tile table of the register-resident Cholesky f_chol (qp_fast.cuh).
constexpr int kCholMaxTiles = 13;       // tile rows supported by f_chol (order <= 104)
constexpr int kCholMaxOff = 13;         // off-diagonal tiles per update warp of f_chol (6 update warps)

// tab[idx] = (ti << 8) | tj for the off-diagonal tiles (ti > tj) enumerated column by column.
// The table holds 96 entries (kTabDoubles): orders above 13 tile rows must not write it.
__device__ __forceinline__ void build_tile_table(uint16_t* tab, int nts, int tid) {
    if (nts > kCholMaxTiles) return;
    if (tid < nts - 1) {
        const int tj = tid;
        const int base = tj * (nts - 1) - (tj * (tj - 1)) / 2;
        for (int ti = tj + 1; ti < nts; ++ti) tab[base + ti - tj - 1] = (uint16_t)((ti << 8) | tj);
    }
}

// Forward substitution over diagonal blocks [kbeg, kend) of the lower factor A (n x n):
// on exit u[k] (kbeg <= k < kend) = solution entries, b[i] (i >= kend) = updated right-hand side.
// b is destroyed. b and u must not alias. kbeg multiple of 8.
template <typename Idx>
__device__ __forceinline__ void trsv_fwd(const double* A, Idx at, int n, int kbeg, int kend,
                                         const double* dinv, double* b, double* u, int tid, int nt) {
    for (int k0 = kbeg; k0 < kend; k0 += 8) {
        const int nb = min(8, kend - k0);
        const int nrows = n - k0;
        if (tid < nrows) {
            double Lk[36], y[8];
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int c = 0; c < r; ++c)
                    Lk[QPB_LIDX(r, c)] = (r < nb) ? A[at(k0 + r, k0 + c)] : 0.0;
#pragma unroll
            for (int c = 0; c < 8; ++c) y[c] = (c < nb) ? b[k0 + c] : 0.0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                y[c] *= (c < nb) ? dinv[k0 + c] : 1.0;
#pragma unroll
                for (int c2 = c + 1; c2 < 8; ++c2) y[c2] = fma(-y[c], Lk[QPB_LIDX(c2, c)], y[c2]);
            }
            if (tid == 0) {
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < nb) u[k0 + c] = y[c];
            }
            for (int t = tid + nb; t < nrows; t += nt) {
                const double* rowp = A + at(k0 + t, k0);
                double s = b[k0 + t];
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < nb) s = fma(-rowp[c], y[c], s);
                b[k0 + t] = s;
            }
        }
        __syncthreads();
    }
}

// Back substitution L^T w = u over all diagonal blocks of the n x n lower factor A.
// u is destroyed; w receives the solution. u and w must not alias.
template <typename Idx>
__device__ __forceinline__ void trsv_bwd(const double* A, Idx at, int n, const double* dinv,
                                         double* u, double* w, int tid, int nt) {
    const int nblk = (n + 7) >> 3;
    for (int kb = nblk - 1; kb >= 0; --kb) {
        const int k0 = kb * 8;
        const int nb = min(8, n - k0);
        if (tid < k0 || tid == 0) {
            double Lk[36], y[8];
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int c = 0; c < r; ++c)
                    Lk[QPB_LIDX(r, c)] = (r < nb) ? A[at(k0 + r, k0 + c)] : 0.0;
#pragma unroll
            for (int c = 0; c < 8; ++c) y[c] = (c < nb) ? u[k0 + c] : 0.0;
#pragma unroll
            for (int c = 7; c >= 0; --c) {
                y[c] *= (c < nb) ? dinv[k0 + c] : 1.0;
#pragma unroll
                for (int c2 = 0; c2 < c; ++c2) y[c2] = fma(-y[c], Lk[QPB_LIDX(c, c2)], y[c2]);
            }
            if (tid == 0) {
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < nb) w[k0 + c] = y[c];
            }
            for (int i = tid; i < k0; i += nt) {
                double s = u[i];
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < nb) s = fma(-A[at(k0 + c, i)], y[c], s);
                u[i] = s;
            }
        }
        __syncthreads();
    }
}

}  // namespace qpb
