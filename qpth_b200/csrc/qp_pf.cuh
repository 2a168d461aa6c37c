// Product-form factorization of the reduced KKT matrix S (factor_kkt, qpth/solvers/pdipm/batch.py:435-470) and the
// chain-free substitutions that go with it (the lu_solve calls of solve_kkt, batch.py:349-372).
//
// Why: round-1/2 accounting of k_forward_fast put the three 13-step substitutions of
// a Newton iteration at 27 % of it and the factorization at 43 %: every substitution step redid an 8-deep dependent
// chain in every thread and re-read the 8x8 diagonal block 256 times; every factorization step solved the panel rows
// by the same chain. Here the factor is produced DIRECTLY in product form, one 8x8 tile at a time on the fp64 tensor
// pipe:
//     F_k:  S_kk = L_kk L_kk^T  and  T_k = L_kk^-1           (chain warp, registers; T_k is published in the diagonal tile)
//     S_k:  L_ik = A_ik T_k^T   (2 DMMA)  -> panel scratch    P_ik = L_ik T_k  (2 DMMA) -> in place of A_ik
//     U_k:  C_ij -= L_ik L_jk^T (2 DMMA)                      trailing tiles, operands from the panel scratch
// and a solve never sees L again:
//     L y = h    :  b_i -= P_ik b_k (running right-hand side),  y_k = T_k b_k
//     L^T w = y  :  w_k = T_k^T y_k - sum_{i>k} P_ik^T w_i
// i.e. one 8-term dot product per row and block step, no dependent chain inside a step, and the diagonal block is
// never re-read. The matrix is stored as a STAIRCASE (block row i keeps columns 0 .. 8i+7, row stride 8i+12): half the
// shared memory of the square workspace (49.9 KB instead of 89.9 KB at order 104, 172.8 KB at order 200 - which is
// what lets the nz = nineq = 200 problems of the cls-layer config keep their factor in shared memory at all).
#pragma once
#include "qp_fast.cuh"

namespace qpb {
namespace pf {
using namespace qpb::fast;

// ---- staircase layout -------------------------------------------------------------------------------------------
// element (r, c), c <= 8 (r >> 3) + 7, lives at pf_rowoff(r) + c; the row stride of block row i is 8 i + 12
// (== 4 mod 8: the DMMA fragment pattern "4 rows x 4 consecutive doubles per half-warp" stays bank-conflict free).
__host__ __device__ __forceinline__ int pf_rowoff(int r) {
    const int i = r >> 3;
    return (32 * i + 64) * i + (r & 7) * (8 * i + 12);
}
__host__ __device__ __forceinline__ int pf_elems(int nts) { return (32 * nts + 64) * nts; }
constexpr int kPanLd = 12;              // row stride of the panel scratch (8 used)

// In-register factorization of an 8x8 SPD block (lower triangle in Lk, every lane holds all of it): on exit strictly
// lower = L, diagonal = 1 / L_cc. A non-positive pivot gives NaN/inf everywhere below it.
__device__ __forceinline__ void pf_factor8(double (&Lk)[36]) {
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
// Column c = lane & 7 of T = L^-1 from the factored block (every lane holds Lk; the lane dependence is in predicates
// only, so the eight columns are computed side by side instead of one lane doing all 112 operations):
//   T[c][c] = 1/L_cc,  T[r][c] = -(sum_{j=c}^{r-1} L[r][j] T[j][c]) / L_rr  (r > c),  0 above the diagonal.
__device__ __forceinline__ void pf_inv8_col(const double (&Lk)[36], int c, double (&Tc)[8]) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        double sacc = 0.0;
#pragma unroll
        for (int j = 0; j < r; ++j) sacc = fma((j >= c) ? Lk[QPB_LIDX(r, j)] : 0.0, (j >= c) ? Tc[j] : 0.0, sacc);
        const double dr = Lk[QPB_LIDX(r, r)];
        Tc[r] = (r < c) ? 0.0 : ((r == c) ? dr : -dr * sacc);
    }
}

// lower triangle (incl. diagonal) of the 8x8 tile whose row r starts at M + rowoff(r0 + r) + c0
__device__ __forceinline__ void pf_load_lower8(const double* M, int r0, int c0, double (&Lk)[36]) {
    const int i = r0 >> 3, ldi = 8 * i + 12;
    const double* Mb = M + (32 * i + 64) * i + c0;
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c <= r; c += 2) {
            const double2 v = *reinterpret_cast<const double2*>(Mb + r * ldi + c);
            Lk[QPB_LIDX(r, c)] = v.x;
            if (c + 1 <= r) Lk[QPB_LIDX(r, c + 1)] = v.y;
        }
}
__device__ __forceinline__ void pf_store_lower8(double* M, int r0, int c0, const double (&Lk)[36]) {
    const int i = r0 >> 3, ldi = 8 * i + 12;
    double* Mb = M + (32 * i + 64) * i + c0;
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c <= r; c += 2)      // the odd tail writes one element of the (unused) upper part of the tile
            *reinterpret_cast<double2*>(Mb + r * ldi + c) =
                make_double2(Lk[QPB_LIDX(r, c)], (c + 1 <= r) ? Lk[QPB_LIDX(r, c + 1)] : 0.0);
}

// ---- tile table of the trailing updates -----------------------------------------------------------------------------
// The trailing tiles of step k are (i, j), k < j <= i < nts. In MIRRORED coordinates j' = nts-1-j, i' = nts-1-i they are
// the leading triangle i' <= j' <= nts-2-k, so with the tiles enumerated as t' = j'(j'+1)/2 + i' the active ones of ANY
// step of ANY order are the prefix [0, (nts-1-k)(nts-k)/2) of ONE table, whose last element is the chain warp's tile
// (k+1, k+1). tab[t'] = (j' << 8) | i'. (The first version walked the triangle with while-loops: 8 % of all the
// instructions of the three-per-SM forward kernel.)
__host__ __device__ __forceinline__ int pf_tab_doubles(int nts) { return ((nts * (nts + 1)) / 2 + 3) >> 2; }
__device__ __forceinline__ void pf_build_tab(int tabo, int nts) {
    QPB_SMEM;
    uint16_t* tab = reinterpret_cast<uint16_t*>(qsm + tabo);
    for (int jp = threadIdx.x; jp < nts; jp += kNT)
        for (int ip = 0; ip <= jp; ++ip) tab[(jp * (jp + 1)) / 2 + ip] = (uint16_t)((jp << 8) | ip);
}

// ---- the factorization --------------------------------------------------------------------------------------------
// Staircase matrix at offset S (order 8 nts), block columns < kb0 already in product form (the pre-factored equality
// block of pre_factor_kkt, batch.py:402-424) with their contribution already subtracted from the trailing block.
// aug (offset): right-hand side carried along as a RUNNING right-hand side b (the caller has already swept the block
// columns < kb0 over it with pf_fwd): on exit aug = b with  y_k = T_k b_k  still to be applied (pf_diag).
// pan (offset): panel scratch, (8 nts + 8) rows x kPanLd.
// Roles: warp 0 = the pivot chain (F_k, the tile below it, the next diagonal tile, F_k+1), warps 1.. = panel + trailing
// update. Named barrier 1: T_k published (chain arrives, update warps wait); named barrier 2: panel complete (chain
// arrives, update warps wait); one __syncthreads per step. blockDim.x == kNT.
// kSetup (pre_factor_kkt, k_setup_pf): stop after block column kend - 1 (the trailing block keeps the Schur complement)
// and, when Lg != nullptr, emit the plain factor L (rows < ln; packed lower) to global memory: the update warps store
// the off-diagonal tiles L_ik as they appear, the chain warp parks the strictly lower part of each L_kk in the strict
// upper triangle of its diagonal tile (pf_park_lower8), which k_setup_pf copies out after the factorization. The chain
// warp thus issues 16 shared stores per step instead of 36 global stores and 8 divisions on the critical path.
// Row r of L_kk (r entries) goes to tile row 7 - r, columns 8 - r .. 7 (r free slots); 16-byte stores where aligned.
__device__ __forceinline__ void pf_park_lower8(double* M, int k, const double (&Lk)[36]) {
    double* Mb = M + (32 * k + 64) * k + 8 * k;
    const int ldk = 8 * k + 12;
#pragma unroll
    for (int r = 1; r < 8; ++r) {
        double* d = Mb + (7 - r) * ldk + 8 - r;
        if (r & 1) d[0] = Lk[QPB_LIDX(r, 0)];
#pragma unroll
        for (int c = r & 1; c + 1 < r; c += 2)
            *reinterpret_cast<double2*>(d + c) = make_double2(Lk[QPB_LIDX(r, c)], Lk[QPB_LIDX(r, c + 1)]);
    }
}
template <bool kSetup>
__device__ __noinline__ void pf_chol_chain_t(int S, int nts, int kb0, int kend, int pan, double* Lg, int ln) {
    QPB_SMEM;
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    double* M = qsm + S;
    double* P = qsm + pan;
    double Lk[36], Tc[8];                                   // Tc: column (lane & 7) of T_k
    pf_load_lower8(M, 8 * kb0, 8 * kb0, Lk);
    __syncwarp();
    pf_factor8(Lk);
    pf_inv8_col(Lk, lane & 7, Tc);
    if (kSetup && Lg != nullptr) pf_park_lower8(M, kb0, Lk);
#pragma unroll 1
    for (int k = kb0; k < (kSetup ? kend : nts); ++k) {
        const int k0 = 8 * k;
        const bool more = k + 1 < nts;
        const int rn = pf_rowoff(k0 + 8 + g);               // this lane's row of block k+1 (only used if `more`)
        double a0 = 0.0, a1 = 0.0;
        if (more) { a0 = M[rn + k0 + q]; a1 = M[rn + k0 + q + 4]; }   // A_{k+1,k} BEFORE its owner overwrites it with P
        if (lane < 8) {                                      // publish T_k in the diagonal tile: lane c stores column c
            const int ldk = 8 * k + 12;
            double* Tb = M + (32 * k + 64) * k + k0 + lane;
#pragma unroll
            for (int r = 0; r < 8; ++r)
                if (r >= lane) Tb[r * ldk] = Tc[r];
        }
        __syncwarp();
        named_bar_arrive(1, kNT);
        if (k < 16) QPB_TICK(96 + k);   // publish T_k
        if (more) {
            // L_{k+1,k} = A T_k^T : B[kk][nn] = T[nn][kk]
            const int rk = pf_rowoff(k0 + g) + k0;
            const double bT0 = (q <= g) ? M[rk + q] : 0.0, bT1 = (q + 4 <= g) ? M[rk + q + 4] : 0.0;
            double d0 = 0.0, d1 = 0.0;
            dmma884(d0, d1, a0, bT0);
            dmma884(d0, d1, a1, bT1);
            *reinterpret_cast<double2*>(P + (k0 + 8 + g) * kPanLd + 2 * q) = make_double2(d0, d1);
            __syncwarp();
            named_bar_arrive(2, kNT);                        // the panel rows of block k+1 are in the scratch
            const double la0 = P[(k0 + 8 + g) * kPanLd + q], la1 = P[(k0 + 8 + g) * kPanLd + q + 4];
            // diagonal tile k+1 -= L L^T
            double2 cv = *reinterpret_cast<const double2*>(M + rn + k0 + 8 + 2 * q);
            dmma884(cv.x, cv.y, -la0, la0);
            dmma884(cv.x, cv.y, -la1, la1);
            *reinterpret_cast<double2*>(M + rn + k0 + 8 + 2 * q) = cv;
            __syncwarp();
            QPB_TICK(24);               // tile below + next diagonal tile
            if (!kSetup || k + 1 < kend) {
                pf_load_lower8(M, k0 + 8, k0 + 8, Lk);
                __syncwarp();
                pf_factor8(Lk);                              // F_{k+1}
                pf_inv8_col(Lk, lane & 7, Tc);               // T_{k+1}
                if (kSetup && Lg != nullptr) pf_park_lower8(M, k + 1, Lk);
            }
            if (k < 16) QPB_TICK(80 + k);   // F_{k+1}
        } else {
            named_bar_arrive(2, kNT);
        }
        __syncthreads();
        if (k < 16) QPB_TICK(112 + k);      // chain warp waiting for the update warps
    }
}

__device__ __forceinline__ void pf_chol_chain(int S, int nts, int kb0, int pan) {
    pf_chol_chain_t<false>(S, nts, kb0, nts, pan, nullptr, 0);
}

template <bool kSetup>
__device__ __noinline__ void pf_chol_update_t(int S, int nts, int kb0, int kend, int aug, int pan, int tabo, double* Lg, int ln) {
    QPB_SMEM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, q = lane & 3;
    const int uw = warp - 1, nuw = kNT / 32 - 1;
    double* M = qsm + S;
    double* P = qsm + pan;
#pragma unroll 1
    for (int k = kb0; k < (kSetup ? kend : nts); ++k) {
        const int k0 = 8 * k;
        QPB_TICK1(40);
        named_bar_sync(1, kNT);                              // T_k is in the diagonal tile
        QPB_TICK1(42);
        {
            const int rg = pf_rowoff(k0 + g) + k0, rq = pf_rowoff(k0 + q) + k0 + g;
            const int ld4 = 4 * (8 * k + 12);
            const double bT0 = (q <= g) ? M[rg + q] : 0.0, bT1 = (q + 4 <= g) ? M[rg + q + 4] : 0.0;   // T[g][q], T[g][q+4]
            const double bP0 = (g <= q) ? M[rq] : 0.0, bP1 = (g <= q + 4) ? M[rq + ld4] : 0.0;        // T[q][g], T[q+4][g]
            // ---- S_k: panel tiles (i, k), i > k, dealt round-robin
#pragma unroll 1
            for (int i = k + 1 + uw; i < nts; i += nuw) {
                const int r = 8 * i + g;
                double* row = M + pf_rowoff(r) + k0;
                const double a0 = row[q], a1 = row[q + 4];
                double d0 = 0.0, d1 = 0.0;
                dmma884(d0, d1, a0, bT0);
                dmma884(d0, d1, a1, bT1);
                if (kSetup && Lg != nullptr && r < ln) {     // the plain factor, packed lower (columns k0 + 2q, + 1 < r)
                    double* lrow = Lg + ((int64_t)r * (r + 1)) / 2 + k0 + 2 * q;
                    lrow[0] = d0; lrow[1] = d1;
                }
                // rows of block k+1 belong to the chain warp in the shared scratch: keep a private copy past its end
                double* pl = P + ((i == k + 1) ? (8 * nts + g) : r) * kPanLd;
                *reinterpret_cast<double2*>(pl + 2 * q) = make_double2(d0, d1);
                __syncwarp();
                const double la0 = pl[q], la1 = pl[q + 4];
                double e0 = 0.0, e1 = 0.0;
                dmma884(e0, e1, la0, bP0);
                dmma884(e0, e1, la1, bP1);
                *reinterpret_cast<double2*>(row + 2 * q) = make_double2(e0, e1);
            }
        }
        if (k < 16) QPB_TICK1(64 + k);      // S_k
        named_bar_sync(2, kNT);                               // every panel row of this step is in the scratch (the chain warp's too), every P_ik in place
        QPB_TICK1(43);                      // waiting for the panel
        // running right-hand side: b_r -= P[r][k0 .. k0+7] . b_k, one row per thread (no shuffles: under this warp-role
        // branch they take their divergent fallback)
#pragma unroll 1
        for (int r = k0 + 8 + (tid - 32); r < 8 * nts; r += kNT - 32) {
            double pr[8], y[8];
            f_ld8(M + pf_rowoff(r) + k0, pr);
            f_ld8(qsm + aug + k0, y);
            double s0 = qsm[aug + r], s1 = 0.0;
#pragma unroll
            for (int c = 0; c < 8; c += 2) { s0 = fma(-pr[c], y[c], s0); s1 = fma(-pr[c + 1], y[c + 1], s1); }
            qsm[aug + r] = s0 + s1;
        }
        QPB_TICK1(45);                      // right-hand side rows
        // ---- U_k: trailing tiles (i, j), k < j <= i, except the chain warp's (k+1, k+1) (= the last entry of the table
        // prefix), dealt round-robin, four tiles (= four independent DMMA chains) in flight per warp
        {
            const uint16_t* tab = reinterpret_cast<const uint16_t*>(qsm + tabo);
            const int nact = ((nts - 1 - k) * (nts - k)) / 2 - 1;
            // a warp takes FOUR CONSECUTIVE table entries at a time: they mostly lie in one tile column, whose panel
            // fragment (the B operand) is then loaded once
#pragma unroll 1
            for (int t0 = 4 * uw; t0 < nact; t0 += 4 * nuw) {
                int ti[4], tj[4];
                bool ok[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    ok[u] = t0 + u < nact;
                    const int e = tab[ok[u] ? t0 + u : t0];
                    ti[u] = nts - 1 - (e & 255);
                    tj[u] = nts - 1 - (e >> 8);
                }
                double2 v[4];
                double a0[4], a1[4], b0[4], b1[4];
                double* cp[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    cp[u] = M + pf_rowoff(8 * ti[u] + g) + 8 * tj[u] + 2 * q;
                    const double* pa = P + (8 * ti[u] + g) * kPanLd + q;
                    v[u] = *reinterpret_cast<const double2*>(cp[u]);
                    a0[u] = pa[0]; a1[u] = pa[4];
                    if (u == 0 || tj[u] != tj[u - 1]) {      // (warp-uniform)
                        const double* pb = P + (8 * tj[u] + g) * kPanLd + q;
                        b0[u] = pb[0]; b1[u] = pb[4];
                    } else {
                        b0[u] = b0[u - 1]; b1[u] = b1[u - 1];
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (ok[u]) dmma884(v[u].x, v[u].y, -a0[u], b0[u]);
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (ok[u]) dmma884(v[u].x, v[u].y, -a1[u], b1[u]);
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (ok[u]) *reinterpret_cast<double2*>(cp[u]) = v[u];
            }
        }
        if (k < 16) QPB_TICK1(48 + k);      // U_k (+ right-hand side rows)
        __syncthreads();
        QPB_TICK1(44);
    }
}

__device__ __forceinline__ void pf_chol_update(int S, int nts, int kb0, int aug, int pan, int tabo) {
    pf_chol_update_t<false>(S, nts, kb0, nts, aug, pan, tabo, nullptr, 0);
}

// tabo: the tile table of pf_build_tab (any order >= nts)
__device__ __forceinline__ void pf_chol(int S, int nts, int kb0, int aug, int pan, int tabo) {
    if (threadIdx.x < 32) pf_chol_chain(S, nts, kb0, pan);
    else pf_chol_update(S, nts, kb0, aug, pan, tabo);
}
// pre_factor_kkt flavour: block columns [kb0, kend) only, optional emission of the plain factor (see pf_chol_chain_t)
__device__ __forceinline__ void pf_chol_setup(int S, int nts, int kb0, int kend, int aug, int pan, int tabo, double* Lg, int ln) {
    if (threadIdx.x < 32) pf_chol_chain_t<true>(S, nts, kb0, kend, pan, Lg, ln);
    else pf_chol_update_t<true>(S, nts, kb0, kend, aug, pan, tabo, Lg, ln);
}

// ---- substitutions (order n = 8 nts <= kNT: thread tid owns entry tid) ----------------------------------------------
// Running right-hand side over block columns [kb, ke):  b_i -= P_ik b_k  for every row below block k. In place.
// Ends with a block barrier; afterwards b holds the running right-hand side of ALL rows.
// Every block step ends with a block barrier. Measured slower on H100 at C2: synchronising only the row-owning warps on
// a named barrier, and one warp running the whole sweep (four rows per lane, __syncwarp between steps) at about 1.8x
// the cycles per sweep in the latency-mode kernel; prefetching that warp's next P rows into registers spilled in the
// three-per-SM build and was slower still.
__device__ __noinline__ void pf_fwd(int S, int n, int kb, int ke, int b) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const double* M = qsm + S;
    const bool mine = tid < n;
    {
        const int ro = pf_rowoff(mine ? tid : 0);
        double acc = mine ? qsm[b + tid] : 0.0;
        double row[8];
        if (mine && tid >= 8 * kb + 8 && kb < ke) f_ld8(M + ro + 8 * kb, row);
#pragma unroll 1
        for (int k = kb; k < ke; ++k) {
            const int k0 = 8 * k;
            if (mine && tid >= k0 + 8) {
                double y[8];
                f_ld8(qsm + b + k0, y);
                double s1 = row[1] * y[1];
                acc = fma(-row[0], y[0], acc); s1 = fma(row[3], y[3], s1);
                acc = fma(-row[2], y[2], acc); s1 = fma(row[5], y[5], s1);
                acc = fma(-row[4], y[4], acc); s1 = fma(row[7], y[7], s1);
                acc = fma(-row[6], y[6], acc);
                acc -= s1;
                if (tid < k0 + 16) qsm[b + tid] = acc;           // block k+1 becomes final
                else if (k + 1 < ke) f_ld8(M + ro + k0 + 8, row);  // next step's P row (static data: no hazard)
            }
            __syncthreads();
        }
        if (mine && tid >= 8 * ke + 8 && kb < ke) qsm[b + tid] = acc;   // rows not yet published (partial sweeps only)
    }
    __syncthreads();
}

// c_k = T_k^T (T_k b_k) for every block. y: scratch vector. c may alias b (not y). Ends with a block barrier.
__device__ __noinline__ void pf_diag(int S, int n, int b, int y, int c) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const double* M = qsm + S;
    const bool mine = tid < n;
    const int k0 = tid & ~7, r = tid & 7;
    if (mine) {
        double t[8], bb[8];
        f_ld8(M + pf_rowoff(tid) + k0, t);                   // row r of T_k (entries c > r are not T: masked)
        f_ld8(qsm + b + k0, bb);
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int cc = 0; cc < 8; cc += 2) {
            s0 = fma((cc <= r) ? t[cc] : 0.0, (cc <= r) ? bb[cc] : 0.0, s0);
            s1 = fma((cc + 1 <= r) ? t[cc + 1] : 0.0, (cc + 1 <= r) ? bb[cc + 1] : 0.0, s1);
        }
        qsm[y + tid] = s0 + s1;
    }
    __syncwarp();                                            // a block's 8 threads sit in one warp
    if (mine) {
        const int i = k0 >> 3, ldi = 8 * i + 12;
        const double* Tc = M + (32 * i + 64) * i + k0 + r;   // column r of T_k: T[j][r] at Tc[j * ldi], j >= r
        double yy[8];
        f_ld8(qsm + y + k0, yy);
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            s0 = fma((j >= r) ? Tc[j * ldi] : 0.0, (j >= r) ? yy[j] : 0.0, s0);
            s1 = fma((j + 1 >= r) ? Tc[(j + 1) * ldi] : 0.0, (j + 1 >= r) ? yy[j + 1] : 0.0, s1);
        }
        qsm[c + tid] = s0 + s1;
    }
    __syncthreads();
}

// w_k = c_k - sum_{i > k} P_ik^T w_i. c is only read. c != w. Ends with a block barrier.
__device__ __noinline__ void pf_bwd(int S, int n, int c, int w) {
    QPB_SMEM;
    const int tid = threadIdx.x;
    const double* M = qsm + S;
    const int nts = n >> 3;
    {
        double acc = (tid < n) ? qsm[c + tid] : 0.0;
        if (tid >= n - 8 && tid < n) qsm[w + tid] = acc;
        double col[8];
        {
            const int i = nts - 1, ldi = 8 * i + 12;
            const double* Pc = M + (32 * i + 64) * i + tid;
            if (tid < 8 * i) {
#pragma unroll
                for (int r = 0; r < 8; ++r) col[r] = Pc[r * ldi];
            }
        }
        __syncthreads();
#pragma unroll 1
        for (int i = nts - 1; i > 0; --i) {
            const int i0 = 8 * i;
            if (tid < i0) {
                double y[8];
                f_ld8(qsm + w + i0, y);
                double s1 = col[1] * y[1];
                acc = fma(-col[0], y[0], acc); s1 = fma(col[3], y[3], s1);
                acc = fma(-col[2], y[2], acc); s1 = fma(col[5], y[5], s1);
                acc = fma(-col[4], y[4], acc); s1 = fma(col[7], y[7], s1);
                acc = fma(-col[6], y[6], acc);
                acc -= s1;
                if (tid >= i0 - 8) qsm[w + tid] = acc;           // block i-1 becomes final
                else {
                    const int im = i - 1, ldm = 8 * im + 12;
                    const double* Pc = M + (32 * im + 64) * im + tid;
#pragma unroll
                    for (int r = 0; r < 8; ++r) col[r] = Pc[r * ldm];
                }
            }
            __syncthreads();
        }
    }
    __syncthreads();
}

// Full solve with a product-form factor: rhs (destroyed) -> out. y: scratch. rhs, y, out distinct.
__device__ __forceinline__ void pf_solve(int S, int n, int rhs, int y, int out) {
    pf_fwd(S, n, 0, (n >> 3) - 1, rhs);
    pf_diag(S, n, rhs, y, rhs);
    pf_bwd(S, n, rhs, out);
}

// ---- pre_factor_kkt side: equality columns of the K template into product form, K into the staircase ----------------
// RA: row-major matrix (leading dimension ld), rows [0, rows): columns [0, 8 kb0) hold a partial Cholesky factor in the
// reciprocal-diagonal convention (diagonal blocks: strictly lower = L, diagonal = 1/L_cc). Rewrites those columns as
// T_k (diagonal tiles, lower incl. diagonal) and P_ik = L_ik T_k (below). Generic pointers, any block size; ends with a
// block barrier. Off the hot path (once per system).
__device__ __forceinline__ void pf_convert_cols(double* RA, int ld, int rows, int kb0, int tid, int nt) {
    if (kb0 <= 0) return;
    // (i) T_k: thread (k, c) computes column c of T_k in registers; all of them write after a barrier
    double Tc[8];
    const bool tk = tid < 8 * kb0;
    const int tk0 = tid & ~7, tc = tid & 7;
    if (tk) {
        const double* Mb = RA + tk0 * ld + tk0;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            double sacc = 0.0;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (j < r && j >= tc) sacc = fma(Mb[r * ld + j], Tc[j], sacc);
            const double dr = Mb[r * ld + r];
            Tc[r] = (r < tc) ? 0.0 : ((r == tc) ? dr : -dr * sacc);
        }
    }
    __syncthreads();
    if (tk) {
        double* Mb = RA + tk0 * ld + tk0;
#pragma unroll
        for (int r = 0; r < 8; ++r)
            if (r >= tc) Mb[r * ld + tc] = Tc[r];
    }
    __syncthreads();
    // (ii) P_ik = L_ik T_k, one (row, block column) per work item
    for (int item = tid; item < rows * kb0; item += nt) {
        const int k = item / rows, r = item - k * rows;
        const int k0 = 8 * k;
        if (r < k0 + 8) continue;
        double* row = RA + r * ld + k0;
        const double* Tb = RA + k0 * ld + k0;
        double l[8], o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) l[j] = row[j];
#pragma unroll
        for (int cc = 0; cc < 8; ++cc) {
            double sacc = 0.0;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (j >= cc) sacc = fma(l[j], Tb[j * ld + cc], sacc);
            o[cc] = sacc;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) row[j] = o[j];
    }
    __syncthreads();
}

// Row-major lower matrix RA (ld, `rows` real rows, order msp with identity rows beyond `rows`) -> staircase at Kg.
__device__ __forceinline__ void pf_write_staircase(double* Kg, const double* RA, int ld, int rows, int msp, int tid, int nt) {
    for (int r = tid >> 5; r < msp; r += nt >> 5) {
        const int i = r >> 3, len = 8 * i + 12, off = pf_rowoff(r);
        for (int c = tid & 31; c < len; c += 32) {
            double v = 0.0;
            if (c <= r) v = (r < rows) ? RA[r * ld + c] : ((r == c) ? 1.0 : 0.0);
            Kg[off + c] = v;
        }
    }
}

}  // namespace pf
}  // namespace qpb
