// Host-side launch of the solve kernels, shared by qp_kernels.cu (the 256-thread build of every kernel) and qp_alt.cu
// (the 192- and 512-thread builds of the product-form ones): the arguments of each kind of launch in one bundle, and
// one launcher per kind that takes the kernel to run, so that each unit instantiates only its own builds.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/qpth_b200.h"
#include "qp_common.cuh"

// (qp_kernels.cu) record a CUDA error's message, per thread; raise a kernel's dynamic shared-memory limit to `bytes`
// on the current device unless it is already that high (one thread-safe cache for the whole library)
extern "C" void qpb200_internal_cuda_error(int err, const char* what);
extern "C" int qpb200_internal_set_smem(const void* kernel, size_t bytes);

// pre_factor_kkt: nsys systems (Q, G, A) -> Lfac, Wfac, Kfac, spd_flag
struct QpbSetupArgs {
    const qpb200_plan* plan; double reg; int nsys; cudaStream_t st;
    const double* Q; int64_t sQ; const double* G; int64_t sG; const double* A; int64_t sA;
    double* Lfac; double* Wfac; double* Kfac; int* spd_flag;
};

// forward: the Newton loop of nbatch QPs (ir_steps: the regularised kernels' refinement steps, else 0)
struct QpbFwdArgs {
    const qpb200_plan* plan; double reg; int nbatch; cudaStream_t st;
    const double* p; int64_t sp; const double* h; int64_t sh; const double* b; int64_t sb;
    const double* Lfac; const double* Wfac; const double* Kfac; int sF;
    double eps, stall_tol, best_tie; int notImprovedLim, maxIter;
    double* zhat; double* lam; double* slacks; double* nus; int* iters; double* best_resid; double* trace;
    int ir_steps;
};

// solve_kkt: (d, rx, rs, rz, ry) -> (dx, ds, dz, dy). The backward: rx, rz, ry = the adjoints of z*, lam, nu; zhat,
// lam, slacks, nus = the solution; dx, dz, dy = the per-QP dx, dlam, dnu; dQ .. db = the per-QP gradients, where
// mQ .. mb = 0 (1: the batch mean is reduced after the kernel)
struct QpbKktArgs {
    const qpb200_plan* plan; double reg; int nbatch; cudaStream_t st;
    const double* d; const double* rx; const double* rs; const double* rz; const double* ry;
    const double* zhat; const double* lam; const double* slacks; const double* nus;
    const double* Lfac; const double* Wfac; const double* Kfac; int sF;
    double* dx; double* ds; double* dz; double* dy;
    double* dQ; double* dp; double* dG; double* dh; double* dA; double* db;
    int mQ, mp, mG, mh, mA, mb;
    int ir_steps;
};

namespace {

KDims dims_of(const qpb200_plan* p, double reg) {
    KDims D;
    D.n = p->nz; D.m = p->nineq; D.e = p->neq; D.ep = p->neq_pad; D.ms = p->ms; D.msp = p->ms_pad;
    D.ldw = p->ldw; D.lds = p->lds; D.rows_s = p->rows_s; D.vl = p->vl;
    D.lp = (int)p->L_elems;
    D.reg = reg;
    return D;
}

template <typename... KArgs, typename... Args>
int launch(void (*kernel)(KArgs...), int grid, int threads, size_t smem, cudaStream_t st, Args... args) {
    const int rc = qpb200_internal_set_smem((const void*)kernel, smem);
    if (rc) return rc;
    kernel<<<grid, threads, smem, st>>>(args...);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { qpb200_internal_cuda_error((int)e, "kernel launch"); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}

// `tail`: the kernel's arguments after the bundle's (k_setup: scratch, scratch per system, pf; k_setup_fast: pf)
template <typename... KArgs, typename... Tail>
int launch_setup(void (*kernel)(KArgs...), int threads, size_t smem, const QpbSetupArgs& a, Tail... tail) {
    return launch(kernel, a.nsys, threads, smem, a.st, dims_of(a.plan, a.reg), a.Q, a.sQ, a.G, a.sG, a.A, a.sA, a.Lfac,
                  a.Wfac, a.Kfac, a.spd_flag, tail...);
}

// `tail`: the arguments between `trace` and `ir_steps` (k_forward: scratch, scratch per QP)
template <typename... KArgs, typename... Tail>
int launch_forward(void (*kernel)(KArgs...), int threads, size_t smem, const QpbFwdArgs& a, Tail... tail) {
    return launch(kernel, a.nbatch, threads, smem, a.st, dims_of(a.plan, a.reg), a.p, a.sp, a.h, a.sh, a.b, a.sb,
                  a.Lfac, a.Wfac, a.Kfac, a.sF, a.eps, a.stall_tol, a.best_tie, a.notImprovedLim, a.maxIter, a.zhat,
                  a.lam, a.slacks, a.nus, a.iters, a.best_resid, a.trace, tail..., a.ir_steps);
}

// `tail`: the arguments between the gradient descriptor and `ir_steps` (k_solve_kkt: scratch, scratch per QP)
template <typename... KArgs, typename... Tail>
int launch_kkt(void (*kernel)(KArgs...), int threads, size_t smem, const QpbKktArgs& a, Tail... tail) {
    const BwdOut O{a.dQ, a.dp, a.dG, a.dh, a.dA, a.db, a.mQ, a.mp, a.mG, a.mh, a.mA, a.mb};
    return launch(kernel, a.nbatch, threads, smem, a.st, dims_of(a.plan, a.reg), a.d, a.rx, a.rs, a.rz, a.ry, a.zhat,
                  a.lam, a.slacks, a.nus, a.Lfac, a.Wfac, a.Kfac, a.sF, a.dx, a.ds, a.dz, a.dy, O, tail..., a.ir_steps);
}

}  // namespace
