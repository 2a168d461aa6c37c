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
    int coop;               /* 1: use them (plan_init's default when coop_ok; the caller may clear it to get the
                             *    one-QP-per-SM kernels, which have the lower latency for a batch smaller than the GPU) */
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

/* pre_factor_kkt (batch.py:375-429) + the SPD check of qp.py:81-85.
 * nsys systems (1 if Q, G, A are all shared, else nBatch); sQ/sG/sA strides as above.
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
 * The refinement loop itself (residual + correction) is host-side glue: qpth_b200/kkt.py. */
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

/* The structured factor and solve for caller-supplied d (B,nineq) and right-hand sides (the counterpart of
 * qpb200_solve_kkt):  [diag(q) 0 G' A'; 0 D I 0; G I 0 0; A 0 0 0] [dx ds dz dy] = -[rx rs rz ry].
 * ry / dy may be NULL when neq == 0. */
int qpb200_box_solve_kkt(const qpb200_box_plan* plan, int nbatch, const double* q, int64_t sq, const double* A,
                         int64_t sA, const double* d, const double* rx, const double* rs, const double* rz,
                         const double* ry, double* dx, double* ds, double* dz, double* dy, void* stream);

/* Measurement aid: launches blocks x threads threads each issuing 8*iters dependent-chain-free fp64 FMAs
 * (2*8*iters*blocks*threads flops); out needs blocks*threads doubles. bench.py times it with CUDA
 * events to obtain the fp64 roofline denominator on the box it runs on. */
int qpb200_dfma_probe(int blocks, int threads, int iters, double* out, void* stream);

/* Whole path on HOST buffers (pageable or pinned): H2D, pre_factor_kkt, forward,
 * backward, D2H, on `device`; synchronises before returning.  All six inputs
 * batched (nbatch leading dimension); gradients may be NULL to skip backward. */
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
 * strips is left untouched. direction 0: host -> device, 1: device -> host. The host buffer should be pinned. */
int qpb200_copy_lower(const double* src, double* dst, int nbatch, int n, int band, int direction, void* stream);

#ifdef __cplusplus
}
#endif
#endif
