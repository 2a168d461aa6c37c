// Shared by qp_kernels.cu (256-thread build of every kernel) and qp_alt.cu (192- / 512-thread builds of the product-form
// solve kernels): problem dimensions, shared-memory constants, get_step, gradient output descriptor.
#pragma once
#include "qp_device.cuh"

namespace {

struct KDims {
    int n, m, e, ep, ms, msp;   // msp = ms rounded up to a multiple of 8 (identity padded)
    int ldw, lds, rows_s, vl;
    int lp;          // doubles in the packed lower factor L (rounded up to even)
    double reg;      // regularisation eps of the iterative-refinement KKT variant (batch.py:244-310); 0 on the QPFunction path
};
constexpr int kTabDoubles = 24;   // 96 uint16 tile-table entries for f_chol (build_tile_table)

__host__ __device__ inline int ld_for(int c) {
    int v = c < 4 ? 4 : c;
    while ((v & 7) != 4) ++v;
    return v;
}

// ---- shared-memory vector slots of the solve / backward kernels (each vl doubles)
enum Vec {
    V_PT = 0, V_XT, V_RXT, V_S, V_V, V_RV, V_HW, V_C2, V_W, V_WC, V_DSA, V_DS, V_DXT, V_D,
    V_BXT, V_BS, V_BV, V_HB, V_DINV, V_DINVL, V_AUG, V_T0, V_T1, V_PART /* 4 slots */, V_COUNT = V_PART + 4
};
constexpr int kRedDoubles = 4 * 32;

// vector slots + reduction scratch + 2 mbarriers (16 B) + 24 unused doubles: the `fits` and `tiny` tests of
// qpb200_plan_init are calibrated on this size, and shrinking it would move their boundaries
__host__ __device__ inline size_t solve_vec_doubles(int vl) { return (size_t)V_COUNT * vl + kRedDoubles + 2 + 24; }

// Global-scratch fallback of the K -> S copy (shared-memory mode uses one TMA bulk copy instead).
__device__ __forceinline__ void copy_K(double* LS, const double* Kg, int total, int tid, int nt) {
    int i = tid;
    for (; i + 3 * nt < total; i += 4 * nt) {
        const double a = Kg[i], b = Kg[i + nt], c = Kg[i + 2 * nt], d = Kg[i + 3 * nt];
        LS[i] = a; LS[i + nt] = b; LS[i + 2 * nt] = c; LS[i + 3 * nt] = d;
    }
    for (; i < total; i += nt) LS[i] = Kg[i];
}

// get_step (batch.py:210-213) for one QP: min over entries with dv <= 0 of -v/dv;
// 1.0 when every dv > 0 (the reference's fill value max(1.0, a.max()) at nBatch=1).
__device__ __forceinline__ double step_candidate(double v, double dv) {
    return (dv > 0.0) ? INFINITY : (-v / dv);
}

struct BwdOut {
    double* dQ; double* dp; double* dG; double* dh; double* dA; double* db;
    int mQ, mp, mG, mh, mA, mb;      // 1 = mean-reduced elsewhere (skip per-QP write)
};

}  // namespace
