// qp_alt.cu - the product-form solve kernels (qp_solve.cuh) compiled a second and a third time with another CTA size:
//   -DQPB_NT=192 -DQPB_ALT_CTAS=3   three QPs per SM (112 registers, <= 76.8 KB of shared memory per QP; W, chol(Q) from L2)
//   -DQPB_NT=512 -DQPB_ALT_CTAS=1   large problems (order 136 .. 256, e.g. nz = nineq = 200): 15 update warps instead of 7
// Same source, same arithmetic as the 256-thread build in qp_kernels.cu; only the thread count (compile-time constant
// kNT of qp_fast.cuh) and the launch bounds differ. Exports qpb200_alt<NT>_{forward,backward,solve_kkt} (and, at 192
// threads, qpb200_alt192_setup: k_setup_pf of qp_setup_pf.cuh): internal entry points that qpb200_forward /
// qpb200_backward / qpb200_solve_kkt / qpb200_pre_factor_kkt (qp_kernels.cu) dispatch to; not part of the public header.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <mutex>

#include "../../include/qpth_b200.h"
#ifndef QPB_NT
#error "compile with -DQPB_NT=192|512 -DQPB_ALT_CTAS=3|1"
#endif
// the device functions of the headers have external linkage (host stubs): give this build its own namespace
#define QPB_NS_CAT2(a, b) a##b
#define QPB_NS_CAT(a, b) QPB_NS_CAT2(a, b)
#define qpb QPB_NS_CAT(qpb_nt, QPB_NT)
#include "qp_solve.cuh"
#include "qp_setup_pf.cuh"

extern "C" void qpb200_internal_cuda_error(int err, const char* what);   // (qp_kernels.cu) records the message, per thread

namespace {

constexpr int kAltCtas = QPB_ALT_CTAS;
constexpr int kMin = (kAltCtas > 1) ? kAltCtas : 0;

KDims alt_dims(const qpb200_plan* p) {
    KDims D;
    D.n = p->nz; D.m = p->nineq; D.e = p->neq; D.ep = p->neq_pad; D.ms = p->ms; D.msp = p->ms_pad;
    D.ldw = p->ldw; D.lds = p->lds; D.rows_s = p->rows_s; D.vl = p->vl;
    D.lp = (int)p->L_elems;
    D.reg = 0.0;
    return D;
}

std::mutex g_mu;
template <typename K>
int alt_set_smem(K kernel, size_t bytes, size_t* cur) {      // cur: per-kernel high-water mark (device 0..15)
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) { qpb200_internal_cuda_error((int)e, "cudaGetDevice"); return QPB200_ERR_CUDA; }
    std::lock_guard<std::mutex> lock(g_mu);
    if (dev < 16 && cur[dev] >= bytes) return QPB200_OK;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) { qpb200_internal_cuda_error((int)e, "cudaFuncSetAttribute"); return QPB200_ERR_CUDA; }
    if (dev < 16) cur[dev] = bytes;
    return QPB200_OK;
}
int alt_check_launch() {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { qpb200_internal_cuda_error((int)e, "kernel launch (qp_alt.cu)"); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}
size_t g_fwd[16], g_kkt[16], g_bwd[16];

}  // namespace

#define QPB_CAT2(a, b, c) a##b##c
#define QPB_CAT(a, b, c) QPB_CAT2(a, b, c)
#define QPB_ALT_NAME(fn) QPB_CAT(qpb200_alt, QPB_NT, fn)

extern "C" {

int QPB_ALT_NAME(_forward)(const qpb200_plan* plan, size_t smem, int nbatch, const double* p, int64_t sp, const double* h,
                           int64_t sh, const double* b, int64_t sb, const double* Lfac, const double* Wfac,
                           const double* Kfac, int sF, double eps, double stall_tol, double best_tie, int notImprovedLim,
                           int maxIter, double* zhat, double* lam, double* slacks, double* nus, int* iters,
                           double* best_resid, double* trace, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const KDims D = alt_dims(plan);
    int rc = alt_set_smem(k_forward_fast<true, true, kMin>, smem, g_fwd);
    if (rc) return rc;
    k_forward_fast<true, true, kMin><<<nbatch, qpb::fast::kNT, smem, st>>>(
        D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam,
        slacks, nus, iters, best_resid, trace);
    return alt_check_launch();
}

// the same with W and chol(Q) staged in shared memory (one QP per SM, latency mode) - only built at 512 threads
int QPB_ALT_NAME(_forward_res)(const qpb200_plan* plan, size_t smem, int nbatch, const double* p, int64_t sp, const double* h,
                               int64_t sh, const double* b, int64_t sb, const double* Lfac, const double* Wfac,
                               const double* Kfac, int sF, double eps, double stall_tol, double best_tie, int notImprovedLim,
                               int maxIter, double* zhat, double* lam, double* slacks, double* nus, int* iters,
                               double* best_resid, double* trace, void* stream) {
#if QPB_NT == 512
    cudaStream_t st = (cudaStream_t)stream;
    const KDims D = alt_dims(plan);
    static size_t cur[16];
    int rc = alt_set_smem(k_forward_fast<false, true, 0>, smem, cur);
    if (rc) return rc;
    k_forward_fast<false, true, 0><<<nbatch, qpb::fast::kNT, smem, st>>>(
        D, p, sp, h, sh, b, sb, Lfac, Wfac, Kfac, sF, eps, stall_tol, best_tie, notImprovedLim, maxIter, zhat, lam,
        slacks, nus, iters, best_resid, trace);
    return alt_check_launch();
#else
    (void)plan; (void)smem; (void)nbatch; (void)p; (void)sp; (void)h; (void)sh; (void)b; (void)sb; (void)Lfac; (void)Wfac;
    (void)Kfac; (void)sF; (void)eps; (void)stall_tol; (void)best_tie; (void)notImprovedLim; (void)maxIter; (void)zhat;
    (void)lam; (void)slacks; (void)nus; (void)iters; (void)best_resid; (void)trace; (void)stream;
    return QPB200_ERR_BAD_ARG;
#endif
}

int QPB_ALT_NAME(_solve_kkt)(const qpb200_plan* plan, size_t smem, int nbatch, const double* d, const double* rx,
                             const double* rs, const double* rz, const double* ry, const double* Lfac, const double* Wfac,
                             const double* Kfac, int sF, double* dx, double* ds, double* dz, double* dy, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const KDims D = alt_dims(plan);
    BwdOut O;
    memset(&O, 0, sizeof(O));
    int rc = alt_set_smem(k_kkt_fast<false, true, true, kMin>, smem, g_kkt);
    if (rc) return rc;
    k_kkt_fast<false, true, true, kMin><<<nbatch, qpb::fast::kNT, smem, st>>>(
        D, d, rx, rs, rz, ry, nullptr, nullptr, nullptr, nullptr, Lfac, Wfac, Kfac, sF, dx, ds, dz, dy, O);
    return alt_check_launch();
}

#if QPB_NT == 192
// pre_factor_kkt with the footprint of the three-per-SM forward / backward CTAs (throughput mode): any of an SM's three
// slots can then hold a setup, forward or backward CTA of the pipeline
int QPB_ALT_NAME(_setup)(const qpb200_plan* plan, size_t smem, int nsys, const double* Q, int64_t sQ, const double* G,
                         int64_t sG, const double* A, int64_t sA, double reg, double* Lfac, double* Wfac, double* Kfac,
                         int* spd_flag, void* stream) {
    static size_t g_setup[16];
    cudaStream_t st = (cudaStream_t)stream;
    KDims D = alt_dims(plan);
    D.reg = reg;
    int rc = alt_set_smem(k_setup_pf<kMin>, smem, g_setup);
    if (rc) return rc;
    k_setup_pf<kMin><<<nsys, qpb::fast::kNT, smem, st>>>(D, Q, sQ, G, sG, A, sA, Lfac, Wfac, Kfac, spd_flag);
    return alt_check_launch();
}
#endif

// (the batch-mean reductions of qpb200_backward stay in qp_kernels.cu: this is only the per-QP kernel). dl_dlam, dl_dnu:
// the adjoints of the duals (NULL: zero), as in qpb200_backward_duals
int QPB_ALT_NAME(_backward)(const qpb200_plan* plan, size_t smem, int nbatch, const double* dl_dzhat,
                            const double* dl_dlam, const double* dl_dnu, const double* zhat,
                            const double* lam, const double* slacks, const double* nus, const double* Lfac,
                            const double* Wfac, const double* Kfac, int sF, double* dQ, int mean_Q, double* dp, int mean_p,
                            double* dG, int mean_G, double* dh, int mean_h, double* dA, int mean_A, double* db, int mean_b,
                            double* dxv, double* dlamv, double* dnuv, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const KDims D = alt_dims(plan);
    BwdOut O;
    O.dQ = dQ; O.dp = dp; O.dG = dG; O.dh = dh; O.dA = dA; O.db = db;
    O.mQ = mean_Q; O.mp = mean_p; O.mG = mean_G; O.mh = mean_h; O.mA = mean_A; O.mb = mean_b;
    int rc = alt_set_smem(k_kkt_fast<true, true, true, kMin>, smem, g_bwd);
    if (rc) return rc;
    k_kkt_fast<true, true, true, kMin><<<nbatch, qpb::fast::kNT, smem, st>>>(
        D, nullptr, dl_dzhat, nullptr, dl_dlam, dl_dnu, zhat, lam, slacks, nus, Lfac, Wfac, Kfac, sF, dxv, nullptr,
        dlamv, dnuv, O);
    return alt_check_launch();
}

}  // extern "C"
