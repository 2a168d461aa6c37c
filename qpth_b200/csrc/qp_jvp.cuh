// qp_jvp.cuh - the right-hand side of the forward-mode (JVP) solve, shared by k_jvp_rhs (qp_kernels.cu) and
// k_box_jvp_rhs (qp_box.cu). The JVP of (z, lam, nu) at the returned point is the backward's own KKT solve,
//   [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [z. s. lam. nu.] = -[rx; 0; rz; ry],
//   rx = sym(dQ) z + dp + dG' lam + dA' nu,   rz = dG z - dh,   ry = dA z - db,
// so these kernels only form rx, rz, ry from the input tangents; the solve is the backward-with-duals entry point.
// Every tangent matrix M needs a row pass (M x) and a column pass (M' y): `contract` does both in one pass over M, so
// each element is read from HBM once. The kernels are bandwidth-bound by construction.
#pragma once
#include "qp_device.cuh"

namespace qpb {
namespace jvp {

constexpr int kJ = 4;              // columns per lane in one chunk: a warp reads 32 kJ contiguous doubles of a row
constexpr int kCW = 32 * kJ;       // chunk width

// doubles of the per-warp column partials `contract` needs in shared memory
__host__ __device__ constexpr int part_doubles(int nt) { return (nt / 32) * kCW; }

// One pass over the R x C row-major matrix M (global memory, read once):
//   row_out(r, (M xc)[r])   once per row and chunk of kCW columns, by lane 0 of the warp that owns row r;
//   col_out(c, (M' xr)[c])  once per column, after a barrier.
// xc (length C) and xr (length R) are in shared memory; part holds part_doubles(NT). Rows are owned by warps (r mod
// NT / 32) and columns by threads, so both outputs are written without atomics and every sum has a fixed order.
// Between the row and the column phase there is a barrier, so row_out and col_out may update the same array (sym(dQ) z).
template <int NT, class RowOut, class ColOut>
__device__ __forceinline__ void contract(const double* __restrict__ M, int R, int C, const double* xc, const double* xr,
                                         double* part, RowOut row_out, ColOut col_out) {
    constexpr int NW = NT / 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int c0 = 0; c0 < C; c0 += kCW) {
        double xv[kJ], cp[kJ];
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
            const int c = c0 + lane + 32 * j;
            xv[j] = c < C ? xc[c] : 0.0;
            cp[j] = 0.0;
        }
#pragma unroll 2
        for (int r = warp; r < R; r += NW) {
            const double* Mr = M + (int64_t)r * C;
            double v[kJ];
#pragma unroll
            for (int j = 0; j < kJ; ++j) {
                const int c = c0 + lane + 32 * j;
                v[j] = c < C ? __ldcs(Mr + c) : 0.0;           // streamed: every element is read once
            }
            const double y = xr[r];
            double rp = 0.0;
#pragma unroll
            for (int j = 0; j < kJ; ++j) {
                rp = fma(v[j], xv[j], rp);
                cp[j] = fma(v[j], y, cp[j]);
            }
            rp = warp_sum(rp);
            if (lane == 0) row_out(r, rp);
        }
#pragma unroll
        for (int j = 0; j < kJ; ++j) part[warp * kCW + lane + 32 * j] = cp[j];
        __syncthreads();
        for (int i = tid; i < kCW && c0 + i < C; i += NT) {
            double s = 0.0;
#pragma unroll
            for (int w = 0; w < NW; ++w) s += part[w * kCW + i];
            col_out(c0 + i, s);
        }
        __syncthreads();
    }
}

// The double backward's cotangents of the backward's clamped D = clamp(lam, 1e-8) / clamp(s, 1e-8) at one inequality
// row (k_box_ggrad_rhs, k_boxq_ggrad_rhs): with c_D = (ulam / D)(vlam / D), c_lam = c_D / clamp(s) where lam >= 1e-8
// and c_s = -c_D D / clamp(s) where s >= 1e-8, each 0 elsewhere (torch's clamp passes the gradient at the bound).
__device__ __forceinline__ void clamp_cotangents(double l, double s, double ul, double vl, double& c_lam, double& c_s) {
    const double sc = fmax(s, 1e-8), d = fmax(l, 1e-8) / sc;
    const double cd = (ul / d) * (vl / d);
    c_lam = l >= 1e-8 ? cd / sc : 0.0;
    c_s = s >= 1e-8 ? -cd * d / sc : 0.0;
}

}  // namespace jvp
}  // namespace qpb
