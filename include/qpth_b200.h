/*
 * qpth_b200 — C ABI of the H100-native batched differentiable QP solver.
 *
 * Drop-in boundary for the hot path of locuslab/qpth (reference @ 528e9f6):
 *   QPFunction()(Q,p,G,h,A,b) forward + backward
 *   = qpth/qp.py:23-182 driving qpth/solvers/pdipm/batch.py
 *     (pre_factor_kkt :375-429, forward :47-207, factor_kkt :435-470,
 *      solve_kkt :349-372, get_step :210-213).
 *
 * The reference has no native code and therefore no FFI; these entry points are
 * what a binding for that path would call.  Each one names the reference
 * function it replaces.  All pointers are DEVICE pointers to fp64 data unless a
 * name ends in `_host`; matrices are row-major and dense; `s*` arguments are
 * batch strides in ELEMENTS (0 = the tensor is shared by every QP of the batch,
 * the stride-0 `expand` of qpth/util.py:44-50).  The caller owns every buffer;
 * the library never allocates user-visible memory, never synchronises the
 * device (except the *_host convenience call) and reports errors by code.
 * `stream` is a cudaStream_t passed as void*.
 *
 * Semantics (see DESIGN.md): every QP is solved exactly as the reference
 * solves an nBatch=1 call — the batch-global exit tests (batch.py:127,140) and
 * the batch-global get_step fill value (batch.py:212) are applied per QP.
 */
#ifndef QPTH_B200_H
#define QPTH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QPB200_OK 0
#define QPB200_ERR_BAD_ARG 1      /* null pointer / non-positive size */
#define QPB200_ERR_NO_CONSTRAINTS 2 /* neq == 0 and nineq == 0  (qp.py:89 assert) */
#define QPB200_ERR_CUDA 3         /* a CUDA runtime call failed: see qpb200_last_cuda_error */
#define QPB200_ERR_TOO_LARGE 4    /* problem exceeds what the kernels support */

/* Sizes of everything the caller must allocate for one (nz, nineq, neq) shape.
 * Filled by qpb200_plan_init.  "system" = one distinct (Q,G,A) triple: the
 * factors are shared by the whole batch when Q, G and A are all un-batched. */
typedef struct qpb200_plan {
    int nz, nineq, neq;
    int neq_pad;            /* neq rounded up to a multiple of 8 (identity-padded rows) */
    int ms;                 /* neq_pad + nineq: order of the reduced KKT system S */
    int ms_pad;             /* ms rounded up to a multiple of 8 (identity rows): rows of the stored K */
    int ldw, lds, rows_s, vl;   /* shared-memory leading dimensions / row counts */
    int smem_resident;      /* 1: W and the S workspace live in shared memory; 0: global scratch */
    int threads;            /* CTA size the kernels are launched with */
    int fast;               /* 1: compact shared-memory kernels (register-resident Cholesky, nineq <= 104) */
    int setup_fast;         /* 1: pre_factor_kkt with the same building blocks (nz <= 104) */
    int64_t L_elems;        /* per system: chol(Q), packed lower triangle, row by row    [replaces Q_LU]  */
    int64_t W_elems;        /* per system: [A;G] L^-T, ms rows with stride ldw           [whitened G, A]  */
    int64_t K_elems;        /* per system: block-Cholesky template of S, ms_pad x lds    [replaces S_LU,R] */
    int64_t setup_scratch_elems;   /* per system, only when smem_resident == 0 (else 0) */
    int64_t solve_scratch_elems;   /* per QP,     only when smem_resident == 0 (else 0) */
    int64_t setup_smem_bytes, solve_smem_bytes;
    int64_t coop_smem_bytes;       /* dynamic shared memory of the co-resident solve kernels */
    int coop_ok;            /* 1: the co-resident kernels exist for this shape (two QPs per SM: W and chol(Q) are read
                             *    from L2 instead of being staged in shared memory)                                  */
    int coop;               /* 1: use them. plan_init sets 0 (they lost to the one-QP-per-SM kernels in A/B runs); the caller
                             *    may set it where coop_ok. Only the round-1 kernels (pf == 0) have this variant.        */
    int tiny;               /* 1: nz, ms_pad <= 32: one WARP per QP (32-thread CTAs, up to 16 QPs per SM) with the generic
                             *    shared-memory kernels; `threads` is then 32                                        */
    int pf;                 /* 1: product-form kernels: factor_kkt produces T_k = L_kk^-1 and P_ik = L_ik T_k directly (fp64
                             *    tensor pipe), substitutions are chain-free, K and the factor use the staircase layout
                             *    (K_elems = 32 t^2 + 64 t doubles, t = ms_pad / 8). Decided by plan_init; do not toggle.   */
    int pf_global;          /* with pf: 1 = W and chol(Q) are read from global memory (large problems, e.g. nz = nineq =
                             *    200: factor + vectors fill the shared memory), 0 = staged in shared memory             */
    int64_t pf_smem_bytes;  /* dynamic shared memory of the product-form solve kernels */
    int pf2_ok;             /* with pf: 1 = the two-QPs-per-SM variant of the solve kernels exists for this shape (factor and
                             *    vectors of a QP take <= 113 KB; W and chol(Q) are read from L2; 128 registers per thread)  */
    int pf_two;             /* with pf2_ok: 1 = use it. THE CALLER MAY SET THIS per call: two QPs per SM give the higher
                             *    throughput once more QPs are in flight than the GPU has SMs (a large batch, or several
                             *    batches on several streams); one QP per SM has the lower latency for a small batch.      */
    int64_t pf2_smem_bytes; /* dynamic shared memory of the two-QPs-per-SM variant */
    int pf3_ok;             /* with pf: 1 = a THREE-QPs-per-SM variant exists (192-thread CTAs, <= 76.8 KB per QP)               */
    int pf_three;           /* with pf3_ok: 1 = use it (takes precedence over pf_two). May be set per call like pf_two.          */
    int64_t pf3_smem_bytes;
    int pf_threads;         /* CTA size of the one-QP-per-SM product-form kernels: 256, or 512 for large orders (ms_pad > 128)  */
    int setup_pf;           /* with pf: 1 = pre_factor_kkt runs the product-form setup kernel (two systems per SM at C2; the
                             *    only shared-memory setup for nz = nineq = 200), 0 = the round-1 setup kernels               */
    int64_t setup_pf_smem_bytes;
} qpb200_plan;

int qpb200_version(void);
const char* qpb200_error_string(int code);
const char* qpb200_last_cuda_error(void);

/* Fill `plan` for a problem shape. No device work. */
int qpb200_plan_init(int nz, int nineq, int neq, qpb200_plan* plan);

/* Entry points of qpb200_plan_kernels */
enum {
    QPB200_ENTRY_SETUP = 0,     /* qpb200_pre_factor_kkt, qpb200_pre_factor_kkt_reg */
    QPB200_ENTRY_FORWARD,       /* qpb200_forward */
    QPB200_ENTRY_KKT,           /* qpb200_backward, qpb200_backward_duals, qpb200_solve_kkt, qpb200_jvp */
    QPB200_ENTRY_REG,           /* qpb200_forward_reg, qpb200_backward_reg, qpb200_backward_reg_duals, qpb200_jvp_reg */
    QPB200_ENTRY_KKT_REG,       /* qpb200_solve_kkt_reg */
    QPB200_ENTRY_COUNT
};
/* Kernels of qpb200_plan_kernels */
enum {
    QPB200_K_NONE = 0,          /* none: the entry point returns QPB200_ERR_TOO_LARGE for this plan */
    QPB200_K_SETUP_TINY,        /* pre_factor_kkt, one warp per system */
    QPB200_K_SETUP_PF192,       /* product-form setup, 192 threads (three per SM, next to the pf_three solve kernels) */
    QPB200_K_SETUP_PF,          /* product-form setup, 256 threads */
    QPB200_K_SETUP_FAST,        /* the compact shared-memory setup (setup_fast) */
    QPB200_K_SETUP_SMEM,        /* the generic setup, shared memory */
    QPB200_K_SETUP_GLOBAL,      /* the generic setup, global scratch (needs `scratch`) */
    QPB200_K_TINY,              /* solve kernels, one warp per QP */
    QPB200_K_PF192,             /* product form, three QPs per SM (pf_three), 192 threads */
    QPB200_K_PF_TWO,            /* product form, two QPs per SM (pf_two) */
    QPB200_K_PF_GLOBAL512,      /* product form, W and chol(Q) from global memory (pf_global), 512 threads */
    QPB200_K_PF_GLOBAL256,      /* the same at 256 threads */
    QPB200_K_PF_RES512,         /* product form, W and chol(Q) in shared memory, 512 threads (a forward only) */
    QPB200_K_PF_RES,            /* the same at 256 threads */
    QPB200_K_COOP,              /* the round-1 co-resident kernels (coop) */
    QPB200_K_FAST,              /* the round-1 compact shared-memory kernels (fast) */
    QPB200_K_GENERIC_SMEM,      /* the generic kernels, shared memory */
    QPB200_K_GENERIC_GLOBAL     /* the generic kernels, global scratch (needs `scratch`) */
};
/* The kernel each entry point launches for `plan` as it stands (with the caller's pf_two, pf_three and coop):
 * out[entry] = {QPB200_K_* kernel, CTA size, dynamic shared-memory bytes}. No device work. */
int qpb200_plan_kernels(const qpb200_plan* plan, int64_t out[QPB200_ENTRY_COUNT][3]);

/* pre_factor_kkt (batch.py:375-429) + the SPD check of qp.py:81-85.
 * nsys systems (1 if Q, G, A are all shared, else nBatch); sQ/sG/sA strides as above.
 * Only the lower triangle of Q is read: its strictly upper triangle may hold anything, NaN included, and the factors
 * are those of the symmetric matrix tril(Q) + tril(Q, -1)^T. The same holds for qpb200_pre_factor_kkt_reg.
 * Writes Lfac (nsys*L_elems), Wfac (nsys*W_elems), Kfac (nsys*K_elems) and
 * spd_flag[nsys] (0 = SPD, 1 = a pivot of chol(Q) was not positive). */
int qpb200_pre_factor_kkt(const qpb200_plan* plan, int nsys,
                          const double* Q, int64_t sQ, const double* G, int64_t sG,
                          const double* A, int64_t sA,
                          double* Lfac, double* Wfac, double* Kfac, int* spd_flag,
                          double* scratch, void* stream);

/* forward (batch.py:47-207): the Mehrotra predictor-corrector loop, one CTA per QP.
 * sF = 0 if the factors are shared (nsys == 1) else 1.
 * Outputs: zhat (B,nz), lam (B,nineq), slacks (B,nineq), nus (B,neq) [may be NULL if neq==0],
 * iters[B] (loop iterations run), best_resid[B] (resids of the returned iterate, batch.py:107).
 * Exit tests of batch.py:140 are applied per QP: best < eps, mu > 1e32, a NaN iterate, maxIter, and
 * notImprovedLim consecutive non-improving iterations once best < stall_tol (pass INFINITY for the
 * reference's literal nBatch=1 behaviour; QPFunction passes 1e-6, see DESIGN.md).
 * best_tie: the returned iterate is the LATEST one whose resids is below best_tie * min resids (1.0 = the
 * reference's argmin, batch.py:126-139; QPFunction passes 1.5, see DESIGN.md).
 * trace (may be NULL): (B, maxIter, 4) doubles receiving pri_resid, dual_resid, mu, resids of every
 * iteration run — the quantities the reference prints at verbose == 1 (batch.py:115-117). */
int qpb200_forward(const qpb200_plan* plan, int nbatch,
                   const double* p, int64_t sp, const double* h, int64_t sh,
                   const double* b, int64_t sb,
                   const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                   double eps, double stall_tol, double best_tie, int notImprovedLim, int maxIter,
                   double* zhat, double* lam, double* slacks, double* nus,
                   int* iters, double* best_resid, double* trace, double* scratch, void* stream);

/* QPFunctionFn.backward (qp.py:128-182): one factor_kkt + one solve_kkt per QP and
 * the gradient outer products.  Any of dQ..db may be NULL (skipped).  For an
 * input that was passed un-batched, pass mean_X = 1: the gradient is the batch
 * MEAN (qp.py:159-177) written as one (un-batched) tensor; dxv/dlamv/dnuv are
 * caller-provided (B,nz)/(B,nineq)/(B,neq) work buffers that receive
 * dx, dlam, dnu (always written; needed by the mean reduction). */
int qpb200_backward(const qpb200_plan* plan, int nbatch,
                    const double* dl_dzhat,
                    const double* zhat, const double* lam, const double* slacks, const double* nus,
                    const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                    double* dQ, int mean_Q, double* dp, int mean_p,
                    double* dG, int mean_G, double* dh, int mean_h,
                    double* dA, int mean_A, double* db, int mean_b,
                    double* dxv, double* dlamv, double* dnuv,
                    double* scratch, void* stream);

/* qpb200_backward for a loss that also depends on the returned duals (an extension: the reference returns only zhat).
 * dl_dlam (B,nineq) and dl_dnu (B,neq) are the gradients of the loss with respect to lam and nus; either may be NULL
 * (zero), and dl_dnu must be NULL when neq == 0. They enter the right-hand side of the backward solve,
 *   [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dlam dnu] = -[dl_dzhat; 0; dl_dlam; dl_dnu],   D = lam / s (clamped),
 * the row-scaled implicit derivative of Qz + p + G'lam + A'nu = 0, diag(lam)(Gz - h) = 0, Az = b at the returned
 * point. The gradients are the outer products of qpb200_backward applied to this dx, dlam, dnu. qpb200_backward is
 * this call with both NULL. */
int qpb200_backward_duals(const qpb200_plan* plan, int nbatch,
                          const double* dl_dzhat, const double* dl_dlam, const double* dl_dnu,
                          const double* zhat, const double* lam, const double* slacks, const double* nus,
                          const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                          double* dQ, int mean_Q, double* dp, int mean_p,
                          double* dG, int mean_G, double* dh, int mean_h,
                          double* dA, int mean_A, double* db, int mean_b,
                          double* dxv, double* dlamv, double* dnuv,
                          double* scratch, void* stream);

/* factor_kkt + solve_kkt (batch.py:435-470, 349-372) for caller-supplied d and
 * right-hand sides: one call = LU/Cholesky of R + D^-1 and one reduced KKT solve.
 * Used by the parity tests of rows a8/a9; not needed by QPFunction itself.
 * ry/dy may be NULL when neq == 0. All vectors are (B, len). */
int qpb200_solve_kkt(const qpb200_plan* plan, int nbatch,
                     const double* d, const double* rx, const double* rs,
                     const double* rz, const double* ry,
                     const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                     double* dx, double* ds, double* dz, double* dy,
                     double* scratch, void* stream);

/* Robust KKT variants of the reference (SURVEY 8f.2): factor_solve_kkt_reg / solve_kkt_ir (batch.py:244-310) regularise
 * the KKT matrix - Q~ = Q + eps I, D~ = D + eps I, -eps I in the two constraint blocks - so that a PSD-singular Q or a
 * rank-deficient A still factors, and recover the accuracy by iterative refinement against the un-regularised residual.
 * Here the regularised solve is the SAME pair of kernels with reg_eps threaded through: chol(Q + eps I); reduced matrix
 * W W^T + diag(eps on equality rows, 1/(d + eps) + eps on inequality rows), which is SPD whatever the rank of A. One
 * pre_factor_kkt_reg serves every refinement step (the reference refactors each time). reg_eps = 0 is the plain call.
 * The refinement loop itself (residual + correction) is host-side glue: qpth_b200/kkt.py.
 * Only the lower triangle of Q is read, as by qpb200_pre_factor_kkt: the factors are those of tril(Q) + tril(Q, -1)^T
 * (+ eps I), so a refinement residual must be formed with that symmetric matrix. */
int qpb200_pre_factor_kkt_reg(const qpb200_plan* plan, int nsys,
                              const double* Q, int64_t sQ, const double* G, int64_t sG,
                              const double* A, int64_t sA, double reg_eps,
                              double* Lfac, double* Wfac, double* Kfac, int* spd_flag,
                              double* scratch, void* stream);
int qpb200_solve_kkt_reg(const qpb200_plan* plan, int nbatch,
                         const double* d, const double* rx, const double* rs,
                         const double* rz, const double* ry, double reg_eps,
                         const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                         double* dx, double* ds, double* dz, double* dy,
                         double* scratch, void* stream);

/* Regularised QP solve (QPFunction kkt_solver=IR_UNOPT): QPs whose Q is only positive SEMIdefinite (LPs, low-rank
 * quadratic terms) or whose equality rows are linearly dependent. The Newton loop and its exits, outputs and trace are
 * those of qpb200_forward / qpb200_backward, but every KKT solve (initial point, each iteration's direction, the backward
 * solve) uses the regularised system of the pair above, [Q+eI 0 G' A'; 0 D+eI I 0; G I -eI 0; A 0 0 -eI], followed by
 * ir_steps refinement steps against the un-regularised one (0 <= ir_steps <= 8), and the residuals, best_resid and the
 * trace are those of the TRUE problem (||Qx + p + G'z + A'y||, not Q + eps I). The loop is thus an inexact Newton method
 * whose fixed point is the exact KKT point. In the forward pass the refinement is applied to each iteration's combined
 * direction (the same correction as refining the affine and corrector directions one by one: it is linear); sigma uses
 * the unrefined affine direction.
 * forward_reg and backward_reg take two kinds of plan:
 *  - one from qpb200_plan_init_reg: the product-form kernels with 256 threads and one QP per SM (W and chol(Q) in
 *    shared memory, or read from L2 when pf_global), on every shape they take, tiny ones included. plan_init_reg
 *    returns QPB200_ERR_TOO_LARGE for ms_pad > 256 (in practice about 200: shared memory) or nineq == 0. scratch is
 *    unused (may be NULL);
 *  - one from qpb200_plan_init with tiny == 0, pf == 0 and smem_resident == 0: the generic global-scratch kernels, on
 *    the larger shapes plan_init_reg refuses. scratch (nbatch * solve_scratch_elems doubles) is then required; NULL
 *    returns QPB200_ERR_BAD_ARG.
 * Every other plan returns QPB200_ERR_TOO_LARGE. The factors come from qpb200_pre_factor_kkt_reg with the same plan and
 * reg_eps; spd_flag is then 1 where a pivot of chol(Q + eps I) failed, i.e. Q has an eigenvalue below -eps. With
 * rank-deficient A the duals nus and the gradients dA, db are not unique. */
int qpb200_plan_init_reg(int nz, int nineq, int neq, qpb200_plan* plan);
int qpb200_forward_reg(const qpb200_plan* plan, int nbatch,
                       const double* p, int64_t sp, const double* h, int64_t sh,
                       const double* b, int64_t sb,
                       const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                       double eps, double stall_tol, double best_tie, int notImprovedLim, int maxIter,
                       double reg_eps, int ir_steps,
                       double* zhat, double* lam, double* slacks, double* nus,
                       int* iters, double* best_resid, double* trace, double* scratch, void* stream);
int qpb200_backward_reg(const qpb200_plan* plan, int nbatch,
                        const double* dl_dzhat,
                        const double* zhat, const double* lam, const double* slacks, const double* nus,
                        const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                        double reg_eps, int ir_steps,
                        double* dQ, int mean_Q, double* dp, int mean_p,
                        double* dG, int mean_G, double* dh, int mean_h,
                        double* dA, int mean_A, double* db, int mean_b,
                        double* dxv, double* dlamv, double* dnuv,
                        double* scratch, void* stream);
/* qpb200_backward_reg with the adjoints of the duals, as qpb200_backward_duals (the refinement steps are unchanged: each
 * works from the residual of the last correction, whatever the right-hand side). With linearly dependent equality rows
 * nus is not unique, and the gradient through it belongs to the nus returned. */
int qpb200_backward_reg_duals(const qpb200_plan* plan, int nbatch,
                              const double* dl_dzhat, const double* dl_dlam, const double* dl_dnu,
                              const double* zhat, const double* lam, const double* slacks, const double* nus,
                              const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                              double reg_eps, int ir_steps,
                              double* dQ, int mean_Q, double* dp, int mean_p,
                              double* dG, int mean_G, double* dh, int mean_h,
                              double* dA, int mean_A, double* db, int mean_b,
                              double* dxv, double* dlamv, double* dnuv,
                              double* scratch, void* stream);

/* Forward mode (JVP) at the returned point, for input tangents dQ, dp, dG, dh, dA, db. Each tangent is a pointer with
 * its own batch stride in elements (0: one tangent for every QP, as for an un-batched input) and may be NULL (zero: it is
 * never read); dG, dh must be NULL when nineq == 0, and dA, db, dnu when neq == 0. The call forms
 *   rx = sym(dQ) z + dp + dG' lam + dA' nu,   rz = dG z - dh,   ry = dA z - db,     sym(dQ) = (dQ + dQ') / 2
 * in `rhs` (B (nz + nineq + neq) doubles: rx (B,nz), then rz (B,nineq), then ry (B,neq)) and solves the backward's
 * system with it, qpb200_backward_duals(dl_dzhat = rx, dl_dlam = rz, dl_dnu = ry) with every gradient NULL:
 *   [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dz ds dlam dnu] = -[rx; 0; rz; ry],   D = lam / s (clamped at 1e-8).
 * dz (B,nz), dlam (B,nineq), dnu (B,neq) receive the tangents of zhat, lam and nus. This is the exact transpose of
 * qpb200_backward_duals: sum_b <(g_z, g_lam, g_nu), (dz, dlam, dnu)> = sum_X <grad_X, dX> for batched inputs. For an
 * un-batched input the JVP is the true derivative, while the backward returns the batch mean, so there the identity
 * carries a factor nbatch. Arguments are checked as qpb200_backward_duals checks them, before anything is launched. */
int qpb200_jvp(const qpb200_plan* plan, int nbatch,
               const double* dQ, int64_t sdQ, const double* dp, int64_t sdp,
               const double* dG, int64_t sdG, const double* dh, int64_t sdh,
               const double* dA, int64_t sdA, const double* db, int64_t sdb,
               const double* zhat, const double* lam, const double* slacks, const double* nus,
               const double* Lfac, const double* Wfac, const double* Kfac, int sF,
               double* rhs, double* dz, double* dlam, double* dnu,
               double* scratch, void* stream);
/* qpb200_jvp for the regularised mode: the solve is qpb200_backward_reg_duals with its ir_steps refinement steps (plan,
 * reg_eps and ir_steps as there). With linearly dependent equality rows dnu is not unique; dz and dlam are. */
int qpb200_jvp_reg(const qpb200_plan* plan, int nbatch,
                   const double* dQ, int64_t sdQ, const double* dp, int64_t sdp,
                   const double* dG, int64_t sdG, const double* dh, int64_t sdh,
                   const double* dA, int64_t sdA, const double* db, int64_t sdb,
                   const double* zhat, const double* lam, const double* slacks, const double* nus,
                   const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                   double reg_eps, int ir_steps,
                   double* rhs, double* dz, double* dlam, double* dnu,
                   double* scratch, void* stream);

/* Double backward (an extension): the derivative of phi = sum_X <w_X, grad_X> for cotangents w_X on the six outputs
 * grad_X of qpb200_backward_duals, with respect to its adjoints (g_z, g_lam, g_nu) and to Q, p, G, h, A, b, treating
 * that backward as computed (the 1e-8 clamps of D included). v = (dxv, dlamv, dnuv) is the first backward's solve at
 * the same point. The call runs
 *   1. qpb200_jvp with tangents w_X: u = (gg_z, gg_lam, gg_nu), the gradients of g_z, g_lam and g_nu;
 *   2. a kernel forming the cotangents of the solution, cz = sym(wQ) vx + wG' vlam + wA' vnu - G' c_s,
 *      clam = wG vx + c_lam, cnu = wA vx, from the cotangent c_D = (ulam / D)(vlam / D) of D = clamp(lam) / clamp(s):
 *      c_lam = c_D / clamp(s) where lam >= 1e-8, c_s = -c_D D / clamp(s) where s >= 1e-8 (0 elsewhere; s = h - G z);
 *   3. qpb200_backward_duals with (cz, clam, cnu): w = (wx, wlam, wnu);
 *   4. a kernel writing dQ = sym(wx z' + ux vx'), dp = wx, dG = (wlam - c_s) z' + lam wx' + vlam ux' + ulam vx',
 *      dh = c_s - wlam, dA = wnu z' + nu wx' + vnu ux' + unu vx', db = -wnu.
 * w_X: pointer and batch stride in elements (0: one cotangent for every QP); each may be NULL (zero), wG and wh must be
 * NULL when nineq == 0 and wA, wb when neq == 0. G (stride sG) is the constraint matrix of the forward. The cotangent of
 * a batch-mean gradient (an un-batched input) is the caller's w_X / nbatch. dQ .. db may be NULL (skipped); sum_X = 1
 * writes the batch sum (one un-batched tensor, the exact derivative for an un-batched input), 0 the per-QP gradients.
 * gg_z (B,nz), gg_lam (B,nineq), gg_nu (B,neq) are always written. work: QPB200_DOUBLE_BACKWARD_WORK doubles. Arguments
 * are checked as qpb200_jvp checks them, before anything is launched. */
#define QPB200_DOUBLE_BACKWARD_WORK(nbatch, nz, nineq, neq) \
    ((int64_t)(nbatch) * (2 * (int64_t)(nz) + 3 * (int64_t)(nineq) + 2 * (int64_t)(neq)))
int qpb200_double_backward(const qpb200_plan* plan, int nbatch,
                           const double* wQ, int64_t swQ, const double* wp, int64_t swp,
                           const double* wG, int64_t swG, const double* wh, int64_t swh,
                           const double* wA, int64_t swA, const double* wb, int64_t swb,
                           const double* G, int64_t sG,
                           const double* dxv, const double* dlamv, const double* dnuv,
                           const double* zhat, const double* lam, const double* slacks, const double* nus,
                           const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                           double* gg_z, double* gg_lam, double* gg_nu,
                           double* dQ, int sum_Q, double* dp, int sum_p,
                           double* dG, int sum_G, double* dh, int sum_h,
                           double* dA, int sum_A, double* db, int sum_b,
                           double* work, double* scratch, void* stream);
/* qpb200_double_backward for the regularised mode: qpb200_jvp_reg and qpb200_backward_reg_duals with their ir_steps
 * refinement steps (plan, reg_eps and ir_steps as there). */
int qpb200_double_backward_reg(const qpb200_plan* plan, int nbatch,
                               const double* wQ, int64_t swQ, const double* wp, int64_t swp,
                               const double* wG, int64_t swG, const double* wh, int64_t swh,
                               const double* wA, int64_t swA, const double* wb, int64_t swb,
                               const double* G, int64_t sG,
                               const double* dxv, const double* dlamv, const double* dnuv,
                               const double* zhat, const double* lam, const double* slacks, const double* nus,
                               const double* Lfac, const double* Wfac, const double* Kfac, int sF,
                               double reg_eps, int ir_steps,
                               double* gg_z, double* gg_lam, double* gg_nu,
                               double* dQ, int sum_Q, double* dp, int sum_p,
                               double* dG, int sum_G, double* dh, int sum_h,
                               double* dA, int sum_A, double* db, int sum_b,
                               double* work, double* scratch, void* stream);

/* Jacobians at the returned point (an extension): d(z*, lam, nu)/d(p, h, b) for every QP of the batch, the negated
 * inverse of the backward's system [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] with D = clamp(lam, 1e-8) / clamp(s, 1e-8):
 *   J_z,p = -R_xx, J_z,h = R_x,lam, J_z,b = R_x,nu (likewise for the lam and nu rows), R = that matrix's inverse.
 * One CTA per QP forms S = W W' + diag(0, 1/d) from Wfac, factors it once and solves for all the columns in blocks of 8.
 * It reads Lfac and Wfac of qpb200_pre_factor_kkt (any qpb200_plan_init plan; not the regularised factors), never K. */
/* Dynamic shared memory of qpb200_jacobian for a qpb200_plan_init plan; *smem_bytes = 0 where the kernel does not
 * cover the shape (the caller then uses qpb200_jvp column by column). No device work. */
int qpb200_jacobian_smem(const qpb200_plan* plan, int64_t* smem_bytes);
/* d(z*, lam, nu)/d(p, h, b) at the point (lam, slacks), with the backward's clamped D. rows / cols: bit 0 z / p,
 * bit 1 lam / h, bit 2 nu / b. J: nbatch row-major blocks of R x C doubles, the blocks in the order z, lam, nu and
 * p, h, b. sF as in qpb200_backward. QPB200_ERR_BAD_ARG for a NULL pointer, an empty mask, a nu or b bit with
 * neq == 0, or nbatch < 1; QPB200_ERR_TOO_LARGE where qpb200_jacobian_smem reports 0. */
int qpb200_jacobian(const qpb200_plan* plan, int nbatch, int rows, int cols, const double* lam, const double* slacks,
                    const double* Lfac, const double* Wfac, int sF, double* J, void* stream);

/* ---- Box QPs (qpth_b200/box.py BoxQPFunction): min 1/2 z' diag(q) z + p'z  s.t.  A z = b,  lb <= z <= ub -------------
 * The dense equivalent is Q = diag(q), G = [-I; I] (only the sides given: lb rows first), h = [-lb; ub]; lam and slacks
 * are laid out as [lb rows; ub rows] (nineq = (has_lb + has_ub) * nz). The inequality block of the KKT system is
 * eliminated in closed form (H = q + G'DG diagonal, M = A H^-1 A' of order neq), so there is no pre_factor_kkt: every
 * call takes q and A themselves. Strides as above (0 = shared); lb / ub may be NULL for an absent side. */
typedef struct qpb200_box_plan {
    int nz, neq, neq_pad, nineq;
    int has_lb, has_ub;
    int threads;            /* CTA size (one CTA per QP) */
    int64_t smem_bytes;     /* dynamic shared memory per CTA: A, the factor of M and every vector */
    int ok;                 /* 1: the box kernels cover this shape (neq_pad <= threads, smem_bytes <= 227 KB); 0: the entry
                             *    points below return QPB200_ERR_TOO_LARGE and the dense path is the one to use          */
    /* Thread block cluster kernels (ok == 0 but neq_pad <= threads): one cluster of cl_ctas CTAs solves one QP, CTA r
     * owning the variables [r cl_slice, (r + 1) cl_slice). cl_ctas is the smallest of 2, 4, 8 whose slice fits 227 KB
     * (0: no cluster covers the shape). The entry points below use them whenever cl_ctas != 0, and return
     * QPB200_ERR_TOO_LARGE if the device cannot make such a cluster resident. QPB200_BOX_CLUSTER=C (development knob)
     * forces C on shapes with ok == 1 too.
     * neq_pad > threads selects the distributed-M cluster kernels instead: M = A H^-1 A' is spread over the cluster by
     * 8-row block rows (rank i mod C), cl_smem_bytes is the largest rank's share. They are chosen where the dense path
     * rejects the shape or its order ms_pad exceeds 384 (the knob forces them on any neq_pad > threads shape C fits). */
    int cl_ctas;
    int cl_slice;           /* variables per CTA (the last CTA may hold fewer) */
    int64_t cl_smem_bytes;  /* dynamic shared memory per CTA */
} qpb200_box_plan;

int qpb200_box_plan_init(int nz, int neq, int has_lb, int has_ub, qpb200_box_plan* plan);

/* forward (batch.py:47-207) with the structured solve; outputs and exit rules as qpb200_forward. spd_flag[B] (may be
 * NULL): 1 where some q_i <= 0 ('Q is not SPD.'). */
int qpb200_box_forward(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* p, int64_t sp,
                       const double* A, int64_t sA, const double* b, int64_t sb, const double* lb, int64_t slb,
                       const double* ub, int64_t sub, double eps, double stall_tol, double best_tie, int notImprovedLim,
                       int maxIter, double* zhat, double* lam, double* slacks, double* nus, int* iters,
                       double* best_resid, double* trace, int* spd_flag, void* stream);

/* backward: dq = dx o z (the diagonal of QPFunction's dQ), dp = dx, dlb = dlam_lb, dub = -dlam_ub, dA = dnu z' + nu dx',
 * db = -dnu; mean_X = 1 writes the batch mean as one un-batched tensor. Any gradient may be NULL. dxv (B,nz), dlamv
 * (B,nineq), dnuv (B,neq) are caller-provided work buffers that receive dx, dlam, dnu. */
int qpb200_box_backward(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                        int64_t sA, const double* dl_dzhat, const double* zhat, const double* lam, const double* slacks,
                        const double* nus, double* dq, int mean_q, double* dp, int mean_p, double* dlb, int mean_lb,
                        double* dub, int mean_ub, double* dA, int mean_A, double* db, int mean_b, double* dxv,
                        double* dlamv, double* dnuv, void* stream);
/* qpb200_box_backward with the adjoints of the duals, as qpb200_backward_duals: dl_dlam (B,nineq) in the [lb rows; ub
 * rows] layout of lam, dl_dnu (B,neq); either may be NULL (zero), dl_dnu must be NULL when neq == 0. */
int qpb200_box_backward_duals(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                              int64_t sA, const double* dl_dzhat, const double* dl_dlam, const double* dl_dnu,
                              const double* zhat, const double* lam, const double* slacks, const double* nus, double* dq,
                              int mean_q, double* dp, int mean_p, double* dlb, int mean_lb, double* dub, int mean_ub,
                              double* dA, int mean_A, double* db, int mean_b, double* dxv, double* dlamv, double* dnuv,
                              void* stream);
/* Forward mode (JVP), as qpb200_jvp: tangents dq, dp, dA, db, dlb, dub, each with a batch stride (0: shared) and NULL
 * allowed (dA, db, dnu must be NULL when neq == 0; dlb / dub when that side is absent). rhs (B (nz + nineq + neq)
 * doubles) receives rx = dq o z + dp + dA' nu (B,nz), rz = [dlb; -dub] (B,nineq, lam's [lb rows; ub rows] layout) and
 * ry = dA z - db (B,neq); the solve is qpb200_box_backward_duals with them and every gradient NULL, on the layout the plan
 * selects. dz, dlam, dnu receive the tangents of zhat, lam and nus. */
int qpb200_box_jvp(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A, int64_t sA,
                   const double* dq, int64_t sdq, const double* dp, int64_t sdp, const double* dA, int64_t sdA,
                   const double* db, int64_t sdb, const double* dlb, int64_t sdlb, const double* dub, int64_t sdub,
                   const double* zhat, const double* lam, const double* slacks, const double* nus, double* rhs,
                   double* dz, double* dlam, double* dnu, void* stream);
/* Double backward (an extension), qpb200_double_backward with Q = diag(q) and the constant G = [-I; I]: the derivative
 * of phi = sum_X <w_X, grad_X> for cotangents w_X on the outputs of qpb200_box_backward_duals, with respect to its
 * adjoints (g_z, g_lam, g_nu) and to q, p, A, b, lb, ub, treating that backward as computed (the 1e-8 clamps of D
 * included). v = (dxv, dlamv, dnuv) is the first backward's solve at the same point. The call runs
 *   1. qpb200_box_jvp with tangents w_X: u = (gg_z, gg_lam, gg_nu), the gradients of g_z, g_lam and g_nu;
 *   2. a kernel forming cz = wq o vx + wA' vnu + c_s_lb - c_s_ub, clam = c_lam, cnu = wA vx from the cotangent
 *      c_D = (ulam / D)(vlam / D) of D: c_lam = c_D / clamp(s) where lam >= 1e-8, c_s = -c_D D / clamp(s) where
 *      s >= 1e-8 (0 elsewhere);
 *   3. qpb200_box_backward_duals with (cz, clam, cnu): w = (wx, wlam, wnu);
 *   4. a kernel writing dq = wx o z + ux o vx, dp = wx, dlb = wlam_lb - c_s_lb, dub = c_s_ub - wlam_ub,
 *      dA = wnu z' + nu wx' + vnu ux' + unu vx', db = -wnu.
 * w_X in qpb200_box_jvp's tangent order, each with a batch stride (0: one cotangent for every QP) and NULL allowed
 * (zero); wA, wb must be NULL when neq == 0, wlb / wub when that side is absent. The cotangent of a batch-mean gradient
 * (an un-batched input) is the caller's w_X / nbatch. dq .. db may be NULL (skipped); sum_X = 1 writes the batch sum
 * (one un-batched tensor, the exact derivative for an un-batched input), 0 the per-QP gradients. gg_z (B,nz), gg_lam
 * (B,nineq), gg_nu (B,neq) are always written. work: QPB200_DOUBLE_BACKWARD_WORK(nbatch, nz, nineq, neq) doubles. Every
 * argument is checked before anything is launched. */
int qpb200_box_double_backward(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                               int64_t sA, const double* wq, int64_t swq, const double* wp, int64_t swp,
                               const double* wA, int64_t swA, const double* wb, int64_t swb, const double* wlb,
                               int64_t swlb, const double* wub, int64_t swub, const double* dxv, const double* dlamv,
                               const double* dnuv, const double* zhat, const double* lam, const double* slacks,
                               const double* nus, double* gg_z, double* gg_lam, double* gg_nu, double* dq, int sum_q,
                               double* dp, int sum_p, double* dlb, int sum_lb, double* dub, int sum_ub, double* dA,
                               int sum_A, double* db, int sum_b, double* work, void* stream);

/* Jacobians of a box QP at the returned point (an extension, csrc/qp_jac.cu): d(z*, lam, nu)/d(p, lb, ub, b) per QP,
 * with the backward's clamped D = clamp(lam, 1e-8) / clamp(s, 1e-8) = [d_lb; d_ub]. With H = q + d_lb + d_ub and
 * X = [H A'; A 0]^-1: the p columns are -X e_j (z and nu rows), the b columns X e_(nz + c), the lb / ub columns the p
 * columns scaled by -d_lb_j / -d_ub_j, and the lam rows d_lb o (rz_lb - z) and d_ub o (rz_ub + z) (rz_lb = e_j in lb
 * column j, rz_ub = -e_j in ub column j, zero otherwise). One CTA per QP factors M = A H^-1 A' once and solves for
 * every column in blocks of 8; any qpb200_box_plan_init plan whose buffers fit is covered, whatever its layout. */
/* Dynamic shared memory of qpb200_box_jacobian; *smem_bytes = 0 where the kernel does not cover the shape (the caller
 * then uses qpb200_box_jvp column by column). No device work. */
int qpb200_box_jacobian_smem(const qpb200_box_plan* plan, int64_t* smem_bytes);
/* rows: bit 0/1/2 = z / lam / nu; cols: bit 0/1/2/3 = p / lb / ub / b. J: nbatch row-major blocks of R x C doubles,
 * the blocks in that order. q, A with batch strides sq, sA (0 = shared). QPB200_ERR_BAD_ARG for a NULL pointer, an
 * empty mask, an unknown bit, an lb / ub bit for an absent side, a nu / b bit with neq == 0, or nbatch < 1;
 * QPB200_ERR_TOO_LARGE where qpb200_box_jacobian_smem reports 0. */
int qpb200_box_jacobian(const qpb200_box_plan* plan, int nbatch, int rows, int cols, const double* q, int64_t sq,
                        const double* A, int64_t sA, const double* lam, const double* slacks, double* J, void* stream);

/* The structured factor and solve for caller-supplied d (B,nineq) and right-hand sides (the counterpart of
 * qpb200_solve_kkt):  [diag(q) 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dz dy] = -[rx rs rz ry].
 * ry / dy may be NULL when neq == 0. */
int qpb200_box_solve_kkt(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                         int64_t sA, const double* d, const double* rx, const double* rs, const double* rz,
                         const double* ry, double* dx, double* ds, double* dz, double* dy, void* stream);

/* ---- Box QPs with a dense Q (BoxQPFunction(dense_Q=True)): min 1/2 z'Qz + p'z  s.t.  A z = b,  lb <= z <= ub --------
 * Only the lower triangle of Q (nz x nz, batch stride sQ, 0 = shared) is read. The dense equivalent, the [lb rows; ub
 * rows] layout of lam / slacks and every stride convention are those of the qpb200_box_* entry points above. The
 * inequality block is eliminated as there, and each Newton iteration factors the bordered matrix [Q + G'DG  A'; A  0] of
 * order nz_pad + neq_pad once, as L diag(I, -I) L' (csrc/qp_boxq.cu), one CTA of `threads` threads per QP. */
typedef struct qpb200_boxq_plan {
    int nz, neq, neq_pad, nineq;
    int has_lb, has_ub;
    int order;              /* nz_pad + neq_pad: the order of the factored matrix (at most threads) */
    int threads;            /* CTA size (one CTA per QP) */
    int64_t smem_bytes;     /* dynamic shared memory per CTA: the factor, A and every vector */
    int ok;                 /* 1: the kernels cover this shape (order <= threads, smem_bytes <= 227 KB); 0: the entry points
                             *    below return QPB200_ERR_TOO_LARGE and the dense path on the dense equivalent is the
                             *    one to use */
} qpb200_boxq_plan;

int qpb200_boxq_plan_init(int nz, int neq, int has_lb, int has_ub, qpb200_boxq_plan* plan);
/* As qpb200_box_forward; spd_flag[B] (may be NULL): 1 where chol(Q) breaks down ('Q is not SPD.'). */
int qpb200_boxq_forward(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* p,
                        int64_t sp, const double* A, int64_t sA, const double* b, int64_t sb, const double* lb,
                        int64_t slb, const double* ub, int64_t sub, double eps, double stall_tol, double best_tie,
                        int notImprovedLim, int maxIter, double* zhat, double* lam, double* slacks, double* nus,
                        int* iters, double* best_resid, double* trace, int* spd_flag, void* stream);
/* As qpb200_box_backward_duals (NULL dl_dlam and dl_dnu: the loss of zhat alone), with dQ = 1/2 (dx z' + z dx')
 * (B,nz,nz), or its batch mean (nz,nz) with mean_Q = 1, in place of dq. */
int qpb200_boxq_backward_duals(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A,
                               int64_t sA, const double* dl_dzhat, const double* dl_dlam, const double* dl_dnu,
                               const double* zhat, const double* lam, const double* slacks, const double* nus,
                               double* dQ, int mean_Q, double* dp, int mean_p, double* dlb, int mean_lb, double* dub,
                               int mean_ub, double* dA, int mean_A, double* db, int mean_b, double* dxv,
                               double* dlamv, double* dnuv, void* stream);
/* As qpb200_box_jvp, with the tangent dQ (nz x nz, stride sdQ) in place of dq: rx = sym(dQ) z + dp + dA' nu. */
int qpb200_boxq_jvp(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A, int64_t sA,
                    const double* dQ, int64_t sdQ, const double* dp, int64_t sdp, const double* dA, int64_t sdA,
                    const double* db, int64_t sdb, const double* dlb, int64_t sdlb, const double* dub, int64_t sdub,
                    const double* zhat, const double* lam, const double* slacks, const double* nus, double* rhs,
                    double* dz, double* dlam, double* dnu, void* stream);
/* As qpb200_box_double_backward, with the cotangent wQ (nz x nz, stride swQ, read in full) in place of wq: cz gains
 * sym(wQ) vx, and dQ = sym(wx z' + ux vx') (B,nz,nz), or its batch sum (nz,nz) with sum_Q = 1, replaces dq. */
int qpb200_boxq_double_backward(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ,
                                const double* A, int64_t sA, const double* wQ, int64_t swQ, const double* wp,
                                int64_t swp, const double* wA, int64_t swA, const double* wb, int64_t swb,
                                const double* wlb, int64_t swlb, const double* wub, int64_t swub, const double* dxv,
                                const double* dlamv, const double* dnuv, const double* zhat, const double* lam,
                                const double* slacks, const double* nus, double* gg_z, double* gg_lam, double* gg_nu,
                                double* dQ, int sum_Q, double* dp, int sum_p, double* dlb, int sum_lb, double* dub,
                                int sum_ub, double* dA, int sum_A, double* db, int sum_b, double* work, void* stream);
/* As qpb200_box_jacobian with a dense Q (nz x nz, batch stride sQ; only its lower triangle is read): K = [H A'; A 0],
 * H = Q + diag(d_lb + d_ub), is factored once per QP as the forward factors it (L diag(I, -I) L' on the bordered
 * staircase) and every column is solved in blocks of 8. *smem_bytes = 0 where the kernel does not cover the plan (every
 * qpb200_boxq_plan_init plan with ok = 1 is covered); the caller then uses qpb200_boxq_jvp column by column. */
int qpb200_boxq_jacobian_smem(const qpb200_boxq_plan* plan, int64_t* smem_bytes);
int qpb200_boxq_jacobian(const qpb200_boxq_plan* plan, int nbatch, int rows, int cols, const double* Q, int64_t sQ,
                         const double* A, int64_t sA, const double* lam, const double* slacks, double* J, void* stream);
/* As qpb200_box_solve_kkt: [Q 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dz dy] = -[rx rs rz ry]. */
int qpb200_boxq_solve_kkt(const qpb200_boxq_plan* plan, int nbatch, const double* Q, int64_t sQ, const double* A,
                          int64_t sA, const double* d, const double* rx, const double* rs, const double* rz,
                          const double* ry, double* dx, double* ds, double* dz, double* dy, void* stream);

/* Measurement aid: launches blocks x threads threads each issuing 8*iters dependent-chain-free fp64 FMAs
 * (2*8*iters*blocks*threads flops); out needs blocks*threads doubles. bench.py times it with CUDA
 * events to obtain the fp64 roofline denominator on the box it runs on. */
int qpb200_dfma_probe(int blocks, int threads, int iters, double* out, void* stream);

/* Whole path on HOST buffers (pageable or pinned): H2D, pre_factor_kkt, forward,
 * backward, D2H, on `device`; synchronises before returning.  All six inputs
 * batched (nbatch leading dimension); gradients may be NULL to skip backward.
 * Only the lower triangle of each Q is read: the result is that of tril(Q) + tril(Q, -1)^T, whatever the
 * strictly upper triangle holds, NaN included. */
int qpb200_qp_host(int device, int nbatch, int nz, int nineq, int neq,
                   const double* Q_host, const double* p_host, const double* G_host,
                   const double* h_host, const double* A_host, const double* b_host,
                   const double* dl_host, double eps, int notImprovedLim, int maxIter,
                   double* zhat_host, double* dQ_host, double* dp_host, double* dG_host,
                   double* dh_host, double* dA_host, double* db_host, int* spd_flag_host);

/* The OptNet parameterisation either side of the path (example-cls-layer.ipynb:125-129): SHARED parameters L (nz x nz, its
 * lower triangle is used), G (nineq x nz), z0, s0 define Q = tril(L) tril(L)^T + eps I and h = G z0 + s0; `construct`
 * builds both in one launch, `chain` maps the (batch-mean) QP gradients dQ, dG_qp, dh back onto the parameters:
 * dL = tril((dQ + dQ^T) tril(L)), dG = dG_qp + dh z0^T, dz0 = G^T dh, ds0 = dh. qpth_b200/layers.py wraps them with
 * QPFunction's kernels in one autograd.Function. */
int qpb200_optnet_construct(int nz, int nineq, const double* L, const double* G, const double* z0, const double* s0,
                            double eps, double* Q, double* h, void* stream);
int qpb200_optnet_chain(int nz, int nineq, const double* L, const double* G, const double* z0, const double* dQ,
                        const double* dG_qp, const double* dh, double* dL, double* dG, double* dz0, double* ds0,
                        void* stream);

/* Transfer helper for SYMMETRIC (nbatch, n, n) matrices - Q on its way in, dQ on its way out (qp.py:157-158 builds dQ
 * as 1/2 (dx z^T + z dx^T)): only the lower triangle crosses PCIe, as `band`-row strips (strip b = rows [b band, (b+1)
 * band) x columns [0, (b+1) band)), one strided 3-D copy per strip on `stream`. The part of the destination above the
 * strips is left untouched. direction 0: host -> device, 1: device -> host. The host buffer should be pinned. Every
 * entry point that takes a dense Q reads only its lower triangle, so such a device buffer can be passed as Q whatever
 * its upper part holds. */
int qpb200_copy_lower(const double* src, double* dst, int nbatch, int n, int band, int direction, void* stream);

#ifdef __cplusplus
}
#endif
#endif
