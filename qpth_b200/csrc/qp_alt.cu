// qp_alt.cu - the product-form solve kernels (qp_solve.cuh) compiled a second and a third time with another CTA size:
//   -DQPB_NT=192 -DQPB_ALT_CTAS=3   three QPs per SM (112 registers, <= 76.8 KB of shared memory per QP; W, chol(Q) from L2)
//   -DQPB_NT=512 -DQPB_ALT_CTAS=1   large problems (order 136 .. 256, e.g. nz = nineq = 200): 15 update warps instead of 7
// Same source, same arithmetic as the 256-thread build in qp_kernels.cu; only the thread count (compile-time constant
// kNT of qp_fast.cuh) and the launch bounds differ. Exports qpb200_alt<NT>_{forward,kkt}, qpb200_alt512_forward_res and
// qpb200_alt192_setup (k_setup_pf of qp_setup_pf.cuh): internal entry points that take the argument bundles of
// qp_launch.cuh, which the entry points of qp_kernels.cu dispatch to; not part of the public header.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

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
#include "qp_launch.cuh"

namespace {
constexpr int kMin = (QPB_ALT_CTAS > 1) ? QPB_ALT_CTAS : 0;
}  // namespace

#define QPB_CAT2(a, b, c) a##b##c
#define QPB_CAT(a, b, c) QPB_CAT2(a, b, c)
#define QPB_ALT_NAME(fn) QPB_CAT(qpb200_alt, QPB_NT, fn)

extern "C" {

// k_forward_fast with W and chol(Q) read from L2 (three per SM at 192 threads; one per SM at 512)
int QPB_ALT_NAME(_forward)(const QpbFwdArgs* a, size_t smem) {
    return launch_forward(k_forward_fast<true, true, kMin>, qpb::fast::kNT, smem, *a);
}

// k_kkt_fast, the same build: the backward (its batch-mean reductions stay in qp_kernels.cu) or solve_kkt
int QPB_ALT_NAME(_kkt)(const QpbKktArgs* a, size_t smem, int backward) {
    if (backward) return launch_kkt(k_kkt_fast<true, true, true, kMin>, qpb::fast::kNT, smem, *a);
    return launch_kkt(k_kkt_fast<false, true, true, kMin>, qpb::fast::kNT, smem, *a);
}

#if QPB_NT == 512
// the forward with W and chol(Q) staged in shared memory (one QP per SM, latency mode)
int qpb200_alt512_forward_res(const QpbFwdArgs* a, size_t smem) {
    return launch_forward(k_forward_fast<false, true, 0>, qpb::fast::kNT, smem, *a);
}
#endif

#if QPB_NT == 192
// pre_factor_kkt with the footprint of the three-per-SM forward / backward CTAs (throughput mode): any of an SM's three
// slots can then hold a setup, forward or backward CTA of the pipeline
int qpb200_alt192_setup(const QpbSetupArgs* a, size_t smem) {
    return launch_setup(k_setup_pf<kMin>, qpb::fast::kNT, smem, *a);
}
#endif

#ifdef QPB_TIMING
// the cycle accounting of this build's k_forward_fast (its own g_tim / g_cta: the namespace differs from qp_kernels.cu's)
int QPB_ALT_NAME(_debug_timing)(long long* host64, int reset) {
    cudaError_t e;
    if (reset) {
        long long z[128] = {0};
        const int target = reset >= 2 ? reset - 2 : 0;
        e = cudaMemcpyToSymbol(qpb::fast::g_tim, z, sizeof(z));
        if (e == cudaSuccess) e = cudaMemcpyToSymbol(qpb::fast::g_tim_target, &target, sizeof(int));
    } else {
        e = cudaMemcpyFromSymbol(host64, qpb::fast::g_tim, 128 * sizeof(long long));
    }
    if (e != cudaSuccess) { qpb200_internal_cuda_error((int)e, "debug_timing (qp_alt.cu)"); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}
int QPB_ALT_NAME(_debug_cta)(long long* host64, int nqp) {
    const cudaError_t e = cudaMemcpyFromSymbol(host64, qpb::fast::g_cta, (size_t)4 * nqp * sizeof(long long));
    if (e != cudaSuccess) { qpb200_internal_cuda_error((int)e, "debug_cta (qp_alt.cu)"); return QPB200_ERR_CUDA; }
    return QPB200_OK;
}
#endif

}  // extern "C"
