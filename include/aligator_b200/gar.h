/* aligator_b200/gar.h -- C ABI of the CUDA-native batched Riccati sweep (H100, sm_90a).
 *
 * Drop-in boundary for ONE path of Simple-Robotics/aligator: the linear-quadratic
 * subproblem solve behind gar::RiccatiSolverBase<double>
 * (include/aligator/gar/riccati-base.hpp:13-37), i.e. what
 * gar::ProximalRiccatiSolver (gar/proximal-riccati.hpp:12-47) does for
 * SolverProxDDPTpl::innerLoop (solvers/proxddp/solver-proxddp.hxx:605-632) and
 * for bench/gar-riccati.cpp:42-50 -- for a BATCH of independent problem
 * instances of identical dimensions, on one H100.
 *
 * Plain C: opaque handle, pointers and sizes, int status codes, no exceptions.
 * All matrices are fp64.  "column-major" / "row-major" are the reference's own
 * storage orders (Eigen default column-major; fb / Z are RowMatrixXs,
 * math.hpp:23-27, riccati-kernel.hpp:96-98).
 *
 * Data layout (identical on host and device; `batch` and knot indices lead):
 *
 *   stage knots  [batch][N][stage_record]   one record = the 11 buffers of
 *       LqrKnotTpl (gar/lqr-problem.hpp:60-65) concatenated, each in the
 *       reference's own column-major storage, nx2 = nx, nth = 0:
 *           [ A (nx*nx) | B (nx*nu) | f (nx) | Q (nx*nx) | S (nx*nu) | R (nu*nu)
 *             | q (nx) | r (nu) | C (nc*nx) | D (nc*nu) | d (nc) | pad to even ]
 *   terminal knot [batch][term_record] = [ Q | q | C (nct*nx) | d (nct) ]   (nu = 0)
 *   G0 [batch][nc0*nx] column-major, g0 [batch][nc0]   (lqr-problem.hpp:126-127)
 *
 *   outputs (StageFactor members, riccati-kernel.hpp:86-101):
 *   FF   [batch][N][nu+nc+nx]          ff  = [k; z; a]
 *   FB   [batch][N][(nu+nc+nx)*nx]     fb  = [K; Z; Ahat], ROW-major
 *   VXX  [batch][N+1][nx*nx]           vm.Vxx column-major; symmetric for t>=1,
 *                                      as computed for t=0 (SURVEY A1)
 *   VX   [batch][N+1][nx]              vm.vx
 *   FFT  [batch][nct], FBT [batch][nct*nx]   terminal knot's z, Z (row-major)
 *   KKT0 [batch][nx+nc0]               kkt0.ff = [x0; lbda0]
 *   XS [batch][N+1][nx]  US [batch][N][nu]  VS [batch][N][nc]  VST [batch][nct]
 *   LBD0 [batch][nc0]    LBDAS [batch][N][nx]  (lbdas[1..N])
 *   STATUS [batch] int   0 = ok, bit0 = a stage LDL^T failed (the reference throws
 *                        "Failed stage LDL factorization", riccati-kernel.hxx:239-241),
 *                        bit1 = the initial-stage factorisation failed,
 *                        bit2 = (parallel solver) a block of the condensed system failed to factor,
 *                        bit3 = a per-instance mu given to a *_v backward / sweep in DEVICE memory was not > 0
 *                               (NaN included) while constraints are present (nc > 0 or nct > 0); that
 *                               instance's outputs are unspecified, every other instance is unaffected.
 *
 * Per-instance scalars (the *_v twins below).  Each scalar a solver keeps per problem -- the penalty mu
 * (mu_penal_, solver-proxddp.hxx:509-520), mu_dyn, the regularisation preg (:690-698) and the step length
 * alpha (:648-671) -- has a twin entry point that takes a [batch] array of doubles instead (the handle's own
 * batch: the local batch on a sharded rank).  Instance b reads element b; nothing else about the computation
 * changes, so instance b's outputs equal those of the scalar call with the value of element b.  The arrays are
 * read in stream order: a device-side update may write them on the same stream just before the call, and the
 * caller keeps them alive until that work has finished.  The twins launch as many kernels as the scalar calls,
 * and they leave no trace in the handle: a later scalar or forward-only call behaves as if the twin had never
 * run.  The streaming twins (multipliers, AL value, assembly, linear step) do not check the values, as they
 * do not check their other device inputs.
 */
#ifndef ALIGATOR_B200_GAR_H
#define ALIGATOR_B200_GAR_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ab2_gar_solver ab2_gar_solver;

enum {
  AB2_OK = 0,
  AB2_ERR_INVALID = 1,     /* bad argument */
  AB2_ERR_UNSUPPORTED = 2, /* dims not instantiated in this build */
  AB2_ERR_CUDA = 3,        /* CUDA runtime error; see ab2_gar_last_error() */
  AB2_ERR_STATE = 4        /* call order (e.g. forward before backward) */
};

enum { AB2_HOST = 0, AB2_DEVICE = 1 };

/* output selectors for ab2_gar_get / ab2_gar_output_doubles / ab2_gar_device_ptr */
enum {
  AB2_OUT_FF = 0,
  AB2_OUT_FB = 1,
  AB2_OUT_VXX = 2,
  AB2_OUT_VX = 3,
  AB2_OUT_FFT = 4,
  AB2_OUT_FBT = 5,
  AB2_OUT_KKT0 = 6,
  AB2_OUT_XS = 7,
  AB2_OUT_US = 8,
  AB2_OUT_VS = 9,
  AB2_OUT_VST = 10,
  AB2_OUT_LBD0 = 11,
  AB2_OUT_LBDAS = 12,
  /* parametric problems (nth > 0), riccati-kernel.hpp:86-101, proximal-riccati.hpp:40-43 */
  AB2_OUT_FTH = 13,     /* [batch][N][(nu+nc+nx)*nth]  row-major [Kth; Zth; Yth]      (StageFactor::fth) */
  AB2_OUT_VXT = 14,     /* [batch][N+1][nx*nth]        column-major                   (vm.Vxt) */
  AB2_OUT_VTT = 15,     /* [batch][N+1][nth*nth]                                      (vm.Vtt) */
  AB2_OUT_VT = 16,      /* [batch][N+1][nth]                                          (vm.vt)  */
  AB2_OUT_KKT0FTH = 17, /* [batch][(nx+nc0)*nth]       row-major                      (kkt0.fth) */
  AB2_OUT_THGRAD = 18,  /* [batch][nth]                                               (thGrad) */
  AB2_OUT_THHESS = 19,  /* [batch][nth*nth]            column-major                   (thHess) */
  AB2_OUT_COUNT = 20
};

typedef struct ab2_gar_dims {
  int nx;      /* state (tangent) dimension of every knot; nx2 = nx */
  int nu;      /* control dimension of the N stage knots (>= 1)     */
  int nc;      /* constraint rows of the stage knots                */
  int nct;     /* constraint rows of the terminal knot (nu = 0)     */
  int nc0;     /* rows of the initial condition G0 x0 + g0 = 0      */
  int horizon; /* N: the problem has N stage knots + 1 terminal     */
  int batch;   /* number of independent problem instances           */
  int device;  /* CUDA device ordinal                               */
} ab2_gar_dims;

/* launch tuning.  variant: -1 = automatic (the FP64 tensor-core formulation where the
 * shape allows it, else the lane-per-column one; the CTA-per-instance kernel for shapes
 * without a compile-time instantiation); 0..8 and 10 select a specific warp-per-instance build,
 * see csrc/riccati_launch.cuh; 9 forces the CTA-per-instance kernel (csrc/riccati_block.cuh). */
typedef struct ab2_gar_tuning {
  int variant;
  int stagger_ns;  /* > 0: start-up delay per resident warp slot (de-phases the warps of an SM) */
  int ctas_per_sm; /* > 0: cap on resident CTAs per SM (e.g. 7 -> 4096 instances = two full rounds) */
} ab2_gar_tuning;

/* Doubles in one stage / terminal record (stage includes the pad to even).
 * Replaces: the 11 ArenaMatrix members of LqrKnotTpl, gar/lqr-problem.hpp:60-65. */
size_t ab2_gar_stage_record_doubles(int nx, int nu, int nc);
size_t ab2_gar_term_record_doubles(int nx, int nct);
/* 1 if (nx,nu,nc,nc0) is served by a compile-time kernel instantiation of this build (one
 * warp or part of one per instance), 2 if by the run-time-dimension kernel (one CTA per
 * instance: any shape whose buffers fit 227 KB of shared memory and whose row counts
 * nx+1, nu+nc, nx+nc0, nu+nc+nx are <= 256), 0 if not served. */
int ab2_gar_supported(int nx, int nu, int nc, int nc0);

/* Replaces: ProximalRiccatiSolver(const LqrProblemTpl&), gar/proximal-riccati.hxx:13-31
 * (allocates all factor storage once; the hot calls below never allocate). */
int ab2_gar_create(const ab2_gar_dims *dims, ab2_gar_solver **out);
/* Parametric problems (LqrKnotTpl::Gth, Gx, Gu, Gv, gamma with nth > 0, gar/lqr-problem.hpp:66-71;
 * what ParallelRiccatiSolver's legs solve).  Same as ab2_gar_create with `nth` parameters: stage
 * records grow by [Gx nx*nth | Gu nu*nth | Gv nc*nth | Gth nth*nth | gamma nth], the terminal record
 * by [Gx | Gv nct*nth | Gth | gamma] (ab2_gar_*_record_doubles_th); backward also produces
 * AB2_OUT_FTH..THHESS; runs the CTA-per-instance kernel. */
int ab2_gar_create_parametric(const ab2_gar_dims *dims, int nth, ab2_gar_solver **out);
size_t ab2_gar_stage_record_doubles_th(int nx, int nu, int nc, int nth);
size_t ab2_gar_term_record_doubles_th(int nx, int nct, int nth);
/* forward(xs, us, vs, lbdas, theta) (riccati-base.hpp:21-24 with the optional theta): theta is
 * [batch][nth] in host or device memory, NULL = no parameter (like std::nullopt). */
int ab2_gar_forward_theta(ab2_gar_solver *s, const double *theta, int memspace, void *stream);
int ab2_gar_destroy(ab2_gar_solver *s);
int ab2_gar_set_tuning(ab2_gar_solver *s, const ab2_gar_tuning *t);

/* Replaces: RiccatiSolverDense(const LqrProblemTpl&), gar/dense-riccati.hxx:13-45 -- the reference's second solver
 * (LQSolverChoice::STAGEDENSE): per knot ONE Bunch-Kaufman factorisation of the (nu + nc + 2 nx)^2 matrix
 * [[R, D^T, B^T, 0],[D, -mu I, 0, 0],[B, 0, 0, -I],[0, 0, -I, P']] (gar/dense-kernel.hpp:98-113), one CTA per
 * instance.  Same problem layout and call sequence as ab2_gar_create; FF / FB have nu + nc + 2 nx rows
 * [k; z; l; y] / [K; Z; L; Y] (dense-kernel.hpp:28-31: u = k + K x, v = z + Z x, lbda' = l + L x, x' = y + Y x),
 * VXX / VX hold Pxx / px (not symmetrised).  Not the fast path: an independent algorithm on the device. */
int ab2_gar_create_dense(const ab2_gar_dims *dims, ab2_gar_solver **out);
/* Replaces: ParallelRiccatiSolver(LqrProblemTpl&, num_threads), gar/parallel-solver.hxx:32-82 -- the
 * parallel-in-time variant.  The horizon of EVERY instance is cut into `num_legs` legs
 * [i(N+1)/T, (i+1)(N+1)/T) (get_work, :23-28); backward() runs the legs of all instances as the work
 * items of one launch (each leg = the recursion of riccati-kernel.hxx:105-129 on its span, parametric
 * in the co-state at the next leg's head, nth = nx), then solves the condensed symmetric
 * block-tridiagonal system of every instance (:85-129, 166-203; block-tridiagonal.hpp:82-182) with at
 * most 5 refinement steps to 1e-10; forward() rolls the legs out in one launch (:209-243).
 * Unlike the reference this does NOT mutate the caller's problem (:52-60, :136-147): the records stay
 * the plain [A|B|f|Q|S|R|q|r|C|D|d] ones, the leg parameterisation (Gx = A^T, Gu = B^T, gamma = f on a
 * leg's last knot) is implicit.  Outputs: as ab2_gar_create plus FTH/VXT/VTT/VT with nth = nx (zero on
 * the last leg, which has no parameters).  Status bit2 = a block of the condensed system failed to
 * factor (the reference ignores that, :176-179).  num_legs < 2 is AB2_ERR_INVALID (the reference
 * throws, :42-46); horizon + 1 >= num_legs is required. */
int ab2_gar_create_parallel(const ab2_gar_dims *dims, int num_legs, ab2_gar_solver **out);
/* Replaces: RiccatiSolverBase::collapseFeedback(), riccati-base.hpp:32 (no-op for the serial solver)
 * / ParallelRiccatiSolver::collapseFeedback(), parallel-solver.hpp:41-51: K_0 -= Kth_0 * subdiagonal[1]
 * (restated as written: after the swap at parallel-solver.hxx:180-181 that block is Vxt_0^T). */
int ab2_gar_collapse_feedback(ab2_gar_solver *s, void *stream);

/* Give the solver the problem data.  Replaces the non-owning `problem_` pointer the
 * reference re-reads at every backward() (proximal-riccati.hpp:46; the knots are
 * rewritten in place by updateLQSubproblem, solver-proxddp.hxx:734-805).
 * memspace AB2_HOST: buffers are copied host->device on `stream` (pinned memory makes
 * the copy asynchronous).  AB2_DEVICE: the pointers are kept, non-owning, zero-copy.
 * Any of the four may be NULL to keep the previous one. */
int ab2_gar_set_problem(ab2_gar_solver *s, const double *stage, const double *term,
                        const double *G0, const double *g0, int memspace, void *stream);

/* Replaces: RiccatiSolverBase::backward(mueq), riccati-base.hpp:19
 * (terminal + stage recursion + initial saddle system, proximal-riccati.hxx:34-62). */
int ab2_gar_backward(ab2_gar_solver *s, double mueq, void *stream);
/* Replaces: RiccatiSolverBase::forward(xs,us,vs,lbdas), riccati-base.hpp:21-24
 * (riccati-kernel.hxx:196-207, 315-377; theta unsupported: nth = 0). */
int ab2_gar_forward(ab2_gar_solver *s, void *stream);
/* backward + forward in ONE persistent launch: the loop body of
 * bench/gar-riccati.cpp:46-49 and solver-proxddp.hxx:608-611. */
int ab2_gar_sweep(ab2_gar_solver *s, double mueq, void *stream);
/* ab2_gar_backward / ab2_gar_sweep with a per-instance mu: mueq [batch] in host or device memory.  Host arrays are
 * checked like the scalar (mu > 0 when nc > 0 or nct > 0, else AB2_ERR_INVALID and nothing is launched) and staged
 * into a buffer the handle owns, as ab2_gar_forward_theta does with theta; device arrays are read by the kernels,
 * which set status bit3 on an instance whose mu is unusable.  Every handle type the scalar calls serve. */
int ab2_gar_backward_v(ab2_gar_solver *s, const double *mueq, int memspace, void *stream);
int ab2_gar_sweep_v(ab2_gar_solver *s, const double *mueq, int memspace, void *stream);
/* Inputs of the batched LQ assembly: the derivative buffers SolverProxDDP::updateLQSubproblem
 * (solvers/proxddp/solver-proxddp.hxx:734-805) and computeProjectedJacobians (:25-69) read.
 * DEVICE pointers; stage arrays are [batch][N][block], terminal / initial arrays [batch][block],
 * blocks column-major like the reference's Eigen matrices.  Constraint sets are given per row
 * by bounds: a row is ACTIVE (kept by applyNormalConeProjectionJacobian, core/constraint-set.hxx:
 * 25-37) iff shifted > hi or shifted < lo -- equality rows: lo = +inf; negative orthant: lo = -inf,
 * hi = 0; box: its limits (computeActiveSet of equality-constraint.hpp:52, negative-orthant.hpp:30,
 * box-constraint.hpp:39). */
typedef struct ab2_lq_inputs {
  const double *Jx, *Ju, *slack;   /* dd.Jx() -> A, dd.Ju() -> B, dyn_slacks[t+1] -> f        (:755-757) */
  const double *Lxx, *Lxu, *Luu;   /* cd.Lxx_, Lxu_, Luu_ -> Q, S, R (+ preg on the diagonals) (:759-768) */
  const double *Lx, *Lu;           /* workspace Lxs[t], Lus[t] -> q, r                          (:764-765) */
  const double *Hxx, *Hxu, *Huu;   /* dd.Hxx_, Hxu_, Huu_ (HessianApprox::EXACT) or NULL        (:770-774) */
  const double *cJx, *cJu;         /* constraint Jacobians before projection [nc x nx], [nc x nu] (:40-41) */
  const double *Lv, *shifted;      /* workspace Lvs[t] -> d; shifted_constraints[t]              (:46,49,780) */
  const double *lo, *hi;           /* [nc] bounds of the stage constraint rows (shared by all knots) */
  const double *Lxx_N, *Lx_N;      /* terminal cost                                               (:787-790) */
  const double *cJx_N, *Lv_N, *shifted_N, *loN, *hiN; /* terminal constraints [nct ...]          (:55-68,791-794) */
  const double *G0, *g0;           /* init_data Jx(), value_                                      (:798-800) */
  const double *Hxx0;              /* init_data Hxx_ (added to stage 0's Q) or NULL               (:803-804) */
  double preg, mu_inv;
} ab2_lq_inputs;
/* updateLQSubproblem + computeProjectedJacobians for every instance and knot in one pass over
 * HBM: writes the solver-owned packed problem (the same bytes ab2_gar_set_problem uploads) and
 * makes it the current problem.  A device-resident caller never moves the knots over PCIe. */
int ab2_gar_assemble(ab2_gar_solver *s, const ab2_lq_inputs *in, void *stream);
/* The same with per-instance preg [batch] and mu_inv [batch] (DEVICE); in->preg and in->mu_inv are ignored. */
int ab2_gar_assemble_v(ab2_gar_solver *s, const ab2_lq_inputs *in, const double *preg, const double *mu_inv,
                       void *stream);
/* Device address of the current packed problem: what = 0 stage, 1 term, 2 G0, 3 g0
 * (the bytes workspace_.lqr_problem holds after updateLQSubproblem). */
int ab2_gar_problem_ptr(ab2_gar_solver *s, int what, const double **out);
/* Copy of it (whole array) to `dst` in host or device memory. */
int ab2_gar_get_problem(ab2_gar_solver *s, int what, double *dst, int memspace, void *stream);

/* One whole iteration of the caller's loop with HOST buffers, pipelined over the batch:
 * upload the problem (what updateLQSubproblem rewrote, solver-proxddp.hxx:734-805), sweep,
 * and download `nwhat` result arrays (`whats[i]` -> `dsts[i]`, full-size host arrays laid out
 * like ab2_gar_get's; what solver-proxddp.hxx:610-632 reads back).  The batch is cut into
 * `nchunks` slices (0 = automatic) that travel on internal streams, so the upload of slice
 * i+1, the sweep of slice i and the download of slice i-1 overlap; PCIe is full duplex, so the
 * step costs max(upload, download) instead of their sum.  Host buffers should be pinned
 * (page-locked); pageable memory works but serialises.  Ordered after prior work on `stream`;
 * work enqueued on `stream` afterwards waits for it.  Results also stay on the device. */
int ab2_gar_sweep_host(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                       const double *g0, double mueq, int nchunks, const int *whats,
                       double *const *dsts, int nwhat, void *stream);
/* The same with the symmetric blocks of every stage knot sent as LOWER TRIANGLES (what Eigen's
 * triangularView<Lower> of LqrKnotTpl::Q / ::R walks, lqr-problem.hpp:53-57; the Riccati recursion only ever
 * needs those): record [A | B | f | Qlow nx(nx+1)/2 | S | Rlow nu(nu+1)/2 | q | r | C | D | d], column j of a
 * triangle holding rows j..n-1, no padding.  The host path is PCIe-bound, so the 16 % fewer bytes at
 * config 2 take 12 % less time (H100); the full records are rebuilt in HBM by one streaming kernel per slice.
 * Plain serial handles only (nth = 0).  pack_stage_sym is the host-side helper that derives the packed
 * records from full ones (an adapter packs its Eigen matrices straight into this layout instead). */
size_t ab2_gar_stage_record_doubles_sym(int nx, int nu, int nc);
int ab2_gar_pack_stage_sym(int nx, int nu, int nc, const double *stage, double *stage_sym, long nrec);
int ab2_gar_sweep_host_sym(ab2_gar_solver *s, const double *stage_sym, const double *term, const double *G0,
                           const double *g0, double mueq, int nchunks, const int *whats,
                           double *const *dsts, int nwhat, void *stream);
/* ab2_gar_sweep_host / ab2_gar_sweep_host_sym with a per-instance mu: mueq [batch] in HOST memory, checked like the
 * scalar (AB2_ERR_INVALID, nothing launched), staged once on `stream` and sliced together with the batch. */
int ab2_gar_sweep_host_v(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                         const double *g0, const double *mueq, int nchunks, const int *whats,
                         double *const *dsts, int nwhat, void *stream);
int ab2_gar_sweep_host_sym_v(ab2_gar_solver *s, const double *stage_sym, const double *term, const double *G0,
                             const double *g0, const double *mueq, int nchunks, const int *whats,
                             double *const *dsts, int nwhat, void *stream);

/* Replaces: getFeedforward(i)/getFeedback(i) (riccati-base.hpp:33-34), the public
 * `datas[i].vm` / `kkt0` members (proximal-riccati.hpp:40-43) and the caller-owned
 * xs/us/vs/lbdas vectors.  Copies the whole [batch][...] array `what` to dst. */
size_t ab2_gar_output_doubles(const ab2_gar_solver *s, int what);
int ab2_gar_get(ab2_gar_solver *s, int what, double *dst, int memspace, void *stream);
/* Sub-range copy: knots [t0, t0+nt) of instances [b0, b0+nb) (dense [nb][nt][...]). */
int ab2_gar_get_range(ab2_gar_solver *s, int what, int b0, int nb, int t0, int nt,
                      double *dst, int memspace, void *stream);
/* Device-resident consumers: raw device pointer of an output array. */
/* First-step policy of every instance, packed [batch][nu][nx+1] = [K_0 | k_0] (row-major) into
 * the DEVICE buffer `dst` by one small kernel: what a receding-horizon consumer applies
 * (results_.gains_[0], solver-proxddp.hxx:619-626) and the payload of the one all-gather when
 * the batch is sharded across GPUs (SURVEY section 8e). */
int ab2_gar_first_step_policy(ab2_gar_solver *s, double *dst, void *stream);
/* Gains in the layout of the caller's results: for every instance and stage knot a COLUMN-major
 * (nu+nc+nx) x (nx+1) block whose column 0 is the feedforward [k; z; a] and columns 1..nx the
 * feedback [K; Z; Ahat] -- what SolverProxDDP copies into results_.gains_[i] from
 * getFeedforward(i) / getFeedback(i) (solver-proxddp.hxx:619-626, results.hxx:23-38).
 * dst: [batch][N][(nu+nc+nx)*(nx+1)], host or device. */
int ab2_gar_get_gains(ab2_gar_solver *s, double *dst, int memspace, void *stream);
/* lqrComputeKktError (gar/utils.hxx:88-182) of the current problem and the solution of the last
 * forward pass, for every instance: dst[batch][3] = infinity norms of the dynamics (incl. the
 * initial condition), constraint (C x + D u + d - mu v) and stationarity residuals.  Computed on
 * the device by ab2_gar_refine's residual kernel (one launch), with one maximum per row family; dst in
 * host or device memory. */
int ab2_gar_kkt_error(ab2_gar_solver *s, double mueq, double *dst, int memspace, void *stream);
/* The same with a per-instance mu: mueq [batch] in DEVICE memory (dst in host or device memory). */
int ab2_gar_kkt_error_v(ab2_gar_solver *s, const double *mueq, double *dst, int memspace, void *stream);
/* The device array behind an output, in its physical layout.  Every output except AB2_OUT_VXX has the layout
 * ab2_gar_get returns (up to the ring heads of ab2_gar_cycle_append).  AB2_OUT_VXX, after a backward pass of the
 * warp-per-instance kernel (every tuning variant except 9 on a plain serial handle whose shape has one; the
 * CTA-per-instance, dense and parallel solvers keep [batch][N+1][nx*nx]):
 *   [batch][N+1][P] lower triangles, P = nx(nx+1)/2 rounded up to even: knot t's Vxx, which is symmetric, packed
 *                   column by column (LAPACK 'L': column j holds rows j..nx-1; the padding double is 0);
 *   then [batch][nx*nx] the full column-major block of factor slot 0 (Vxx_0, which is not symmetric in general,
 *                   or the terminal block when N = 0); packed slot 0 is unused.
 * ab2_gar_get / ab2_gar_get_range expand this to full blocks. */
int ab2_gar_device_ptr(ab2_gar_solver *s, int what, double **out);

/* Multi-GPU (one process per GPU, the batch sharded by instance, SURVEY section 8e): the ONE exchange
 * of a sweep -- the all-gather of the first-step policy [K_0 | k_0] -- fused into the sweep over
 * NVLink peer memory instead of a separate NCCL collective.  Every rank owns a receive buffer
 * [world][batch][nu][nx+1] (three slots, alternating by step) that all peers map through CUDA IPC.
 * Once connected, every warp-per-instance backward / sweep launch stores each instance's block straight
 * into slot r of every rank's buffer as soon as that instance's backward pass is done (other kernels:
 * a pack kernel does the same stores); a step flag (release / acquire at system scope) publishes it.
 *   init:      allocate the local buffer; *ipc_handle_out = 64 bytes to hand to every peer
 *   connect:   all_handles = world x 64 bytes, rank order (exchange them with any host transport)
 *   allgather: after backward / sweep, on the same `stream` (all ranks, same batch): publish the step
 *              (pack + store first where the sweep has not done it); holds `stream` until every peer
 *              has consumed what the next step's slot held
 *   wait:      `stream` acknowledges the previous step as consumed, then waits until the blocks of every
 *              rank have arrived for the last allgather
 *   buffer:    device address of the slot holding the last allgather, [world][batch][nu][nx+1] */
int ab2_gar_peer_gather_init(ab2_gar_solver *s, int world, int rank, void *ipc_handle_out);
int ab2_gar_peer_gather_connect(ab2_gar_solver *s, const void *all_handles);
int ab2_gar_policy_allgather(ab2_gar_solver *s, void *stream);
int ab2_gar_policy_allgather_wait(ab2_gar_solver *s, void *stream);
int ab2_gar_peer_gather_buffer(ab2_gar_solver *s, double **out, long *step);
/* Per-instance status words (layout above). */
int ab2_gar_status(ab2_gar_solver *s, int *dst, int memspace, void *stream);
/* Pivot statistics of the last backward pass, one int per instance: bits 0-14 = number of
 * 2x2 pivots, bit 15 = the initial saddle system needed no interchange / 2x2 pivot and ran on the
 * register fast path, high 16 bits = number of symmetric interchanges the Bunch-Kaufman factorisations
 * of the stage KKT matrices and of the initial saddle system took (core/bunchkaufman.hpp:61-83,
 * what Eigen::BunchKaufman reports through pivots() / m_pivot_count, :158-163).  Diagnostics:
 * lets a caller (and the tests) see that the pivoted code paths actually ran. */
int ab2_gar_pivot_stats(ab2_gar_solver *s, int *dst, int memspace, void *stream);

/* The consumers of the step inside the caller's line search (SURVEY section 8f rank 2), batched over the
 * instances so that SolverProxDDP's inner loop (solver-proxddp.hxx:605-660) can stay on the device between
 * the sweep and the next model evaluation; the step (dxs, dus, dvs, dlams) is the solver's own last forward
 * pass.  All array arguments are DEVICE pointers laid out like the solver's outputs: xs [batch][N+1][nx],
 * us [batch][N][nu], vs [batch][N][nc], vsT [batch][nct], lam0 [batch][nc0], lams [batch][N][nx]. */
typedef struct ab2_ls_iterate {
  const double *xs, *us, *vs, *vsT, *lam0, *lams;
} ab2_ls_iterate;
typedef struct ab2_ls_trial {
  double *xs, *us, *vs, *vsT, *lam0, *lams;
} ab2_ls_trial;
/* Replaces: the vector part of SolverProxDDP::tryLinearStep, solver-proxddp.hxx:111-155: trial = results +
 * alpha * step for lams, vs (math::vectorMultiplyAdd, :121-124) and for xs, us with the vector-space
 * integrate (:139-150); a manifold's integrate and problem.evaluate() stay with the modelling library. */
int ab2_gar_linear_step(ab2_gar_solver *s, double alpha, const ab2_ls_iterate *current, const ab2_ls_trial *trial,
                        void *stream);
/* The same with a per-instance step length alpha [batch] (DEVICE): every element uses the alpha of the instance
 * that owns it; alpha = 0 leaves that instance's trial equal to its current iterate. */
int ab2_gar_linear_step_v(ab2_gar_solver *s, const double *alpha, const ab2_ls_iterate *current,
                          const ab2_ls_trial *trial, void *stream);
/* Replaces: ALFunction::directionalDerivative, merit-function.hxx:68-104 (Lxs [batch][N+1][nx], Lus [batch][N][nu]
 * = the Lagrangian gradients) and costDirectionalDerivative, :13-31 (pass the cost gradients): dst[batch] =
 * sum_t Lxs_t . dxs_t + sum_t Lus_t . dus_t.  dst in host or device memory. */
int ab2_gar_directional_derivative(ab2_gar_solver *s, const double *Lxs, const double *Lus, double *dst, int memspace,
                                   void *stream);
/* Replaces: ALFunction::evaluate, merit-function.hxx:33-66: dst[batch] = cost[batch] (NULL = 0) + 1/2 (mucstr
 * |lam0|^2 + mudyn sum |lams_t|^2 + mucstr sum |vs_t|^2 + mucstr |vsT|^2) of the multiplier estimates `plus`
 * (only lam0, lams, vs, vsT are read). */
int ab2_gar_al_value(ab2_gar_solver *s, const ab2_ls_iterate *plus, const double *cost, double mudyn, double mucstr,
                     double *dst, int memspace, void *stream);
/* The same with per-instance mudyn [batch] and mucstr [batch] (DEVICE). */
int ab2_gar_al_value_v(ab2_gar_solver *s, const ab2_ls_iterate *plus, const double *cost, const double *mudyn,
                       const double *mucstr, double *dst, int memspace, void *stream);

/* Gradients of the LQ solution with respect to the problem data (no reference counterpart: what learning a cost or a
 * model through an MPC layer needs).  The solve is the solution z of one symmetric KKT system K z = -h; for a loss
 * with cotangent zbar = dL/dz, w = K^-1 zbar is the solution of the SAME LQ problem with the vectors replaced by
 * q_t = -xbar_t, r_t = -ubar_t, d_t = -vbar_t, f_t = -lambdabar_{t+1}, q_N = -xbar_N, d_N = -vbar_N, g0 = -lambdabar_0,
 * and the gradients are dh = -w, dK = -w z^T read out of K's blocks.  With w = (xt, ut, vt, lt) and z = (x, u, v, l):
 *   dq = -xt_t, dr = -ut_t, dd = -vt_t, df = -lt_{t+1}, dg0 = -lt_0,
 *   dA = -(lt_{t+1} x_t^T + l_{t+1} xt_t^T), dB = -(lt_{t+1} u_t^T + l_{t+1} ut_t^T), dS = -(xt u^T + x ut^T),
 *   dC = -(vt x^T + v xt^T), dD = -(vt u^T + v ut^T), dG0 = -(lt_0 x_0^T + l_0 xt_0^T),
 *   dQ = -1/2 (xt x^T + x xt^T), dR = -1/2 (ut u^T + u ut^T), and the terminal record's dQ_N, dq_N, dC_N, dd_N alike.
 * Q and R are symmetric and the kernels may read either triangle, so their gradient is the one with respect to a
 * symmetric argument (Q_ij and Q_ji perturbed together): the right chain rule for any symmetric parametrisation,
 * such as (P + P^T) / 2 or L L^T.  mu is not differentiated.
 *
 * All arrays are DEVICE arrays.  `primal` is a solution of the handle's CURRENT problem at the same mu (in practice
 * what the last sweep returned, copied out by the caller); every field of nonzero size is required and none may
 * overlap an output array of the handle (AB2_ERR_INVALID).  A NULL `cotangent` field is a zero cotangent.  `grad`
 * arrays have the problem's layouts -- stage [batch][N][stage_record] (pad double = 0), term [batch][term_record],
 * G0 [batch][nc0*nx], g0 [batch][nc0] -- and are overwritten; a NULL field is not written.
 * In order on `stream`, without host synchronisation, three launches: a streaming kernel writes the adjoint problem
 * into a buffer the handle owns (allocated on the first call), the sweep kernel solves it (backward + forward), a
 * streaming kernel writes the gradients.  Afterwards the handle's problem is unchanged, but its OUTPUTS (FF .. LBDAS,
 * status, pivot statistics) are those of the adjoint solve: the matrix recursion is the primal one, so FB, VXX and
 * the pivot statistics equal the primal sweep's, while the vectors and the trajectory are w.  A later backward or
 * sweep restores the primal outputs.  Plain serial handles (warp, CTA and dense kernels); parametric (nth > 0) and
 * parallel handles return AB2_ERR_UNSUPPORTED; a call before set_problem returns AB2_ERR_STATE.  Nothing is launched
 * on an error. */
typedef struct ab2_lq_grad {
  double *stage, *term, *G0, *g0;
} ab2_lq_grad;
int ab2_gar_adjoint  (ab2_gar_solver *s, double mueq,
                      const ab2_ls_iterate *primal, const ab2_ls_iterate *cotangent,
                      const ab2_lq_grad *grad, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_adjoint_v(ab2_gar_solver *s, const double *mueq, int memspace,
                      const ab2_ls_iterate *primal, const ab2_ls_iterate *cotangent,
                      const ab2_lq_grad *grad, void *stream);

/* Forward mode: the derivative zdot of the LQ solution along a tangent pdot of the problem data (a perturbed model
 * A, B, a shifted reference in q, the initial state through g0, ...), for the whole batch in one call.  K is affine
 * in the data, so zdot = -K^-1 (Kdot z + hdot): the SAME LQ problem with the vectors replaced by rho = Kdot z + hdot.
 * With z = (x, u, v, l), l_{t+1} = lams[t], sym(M) = (M + M^T) / 2 and dotted blocks the tangent records, per stage knot
 *   q_t <- qdot + sym(Qdot) x_t + Sdot u_t + Cdot^T v_t + Adot^T l_{t+1}   (+ G0dot^T l_0 at t = 0)
 *   r_t <- rdot + Sdot^T x_t + sym(Rdot) u_t + Ddot^T v_t + Bdot^T l_{t+1}
 *   d_t <- ddot + Cdot x_t + Ddot u_t,       f_t <- fdot + Adot x_t + Bdot u_t
 * and q_N <- qdot_N + sym(Qdot_N) x_N + C_Ndot^T v_N, d_N <- ddot_N + C_Ndot x_N, g0 <- g0dot + G0dot x_0.
 * sym(Qdot) and sym(Rdot) make this the exact transpose of ab2_gar_adjoint's symmetric-argument gradient:
 * <zbar, zdot> = <grad, pdot> for any pdot, including an asymmetric Qdot or Rdot.  mu is not differentiated.
 *
 * `dot` holds DEVICE arrays in the problem's layouts (stage [batch][N][stage_record], pad double ignored;
 * term [batch][term_record]; G0 [batch][nc0*nx]; g0 [batch][nc0]); a NULL field is a zero tangent.  `primal` is a
 * solution of the handle's CURRENT problem at the same mu; every field of nonzero size is required.  It is read
 * completely before the sweep writes anything, so it MAY be the handle's own outputs (ab2_gar_device_ptr).
 * In order on `stream`, without host synchronisation, three launches: a streaming kernel writes -rho into a buffer
 * the handle owns (allocated on the first call), ab2_gar_adjoint's records kernel builds the tangent problem from it,
 * the sweep kernel solves it.  Afterwards the handle's problem is unchanged and its trajectory outputs (XS .. LBDAS)
 * are zdot; as after ab2_gar_adjoint, FB, VXX and the pivot statistics equal the primal sweep's, and a later backward
 * or sweep restores the primal outputs.  Plain serial handles (warp, CTA and dense kernels); parametric (nth > 0) and
 * parallel handles return AB2_ERR_UNSUPPORTED; a call before set_problem returns AB2_ERR_STATE; a NULL primal field
 * of nonzero size, or mueq <= 0 with constraints, returns AB2_ERR_INVALID.  Nothing is launched on an error. */
typedef struct ab2_lq_tangent {
  const double *stage, *term, *G0, *g0;
} ab2_lq_tangent;
int ab2_gar_tangent  (ab2_gar_solver *s, double mueq, const ab2_ls_iterate *primal,
                      const ab2_lq_tangent *dot, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_tangent_v(ab2_gar_solver *s, const double *mueq, int memspace, const ab2_ls_iterate *primal,
                      const ab2_lq_tangent *dot, void *stream);

/* Re-solve the last backward's LQ matrices for new vectors, many right-hand sides at once (Jacobians, batched VJPs
 * and JVPs, linear MPC where only g0 and the references change).  With h = (q_t, r_t, d_t, f_t, q_N, d_N, g0) in the
 * layouts of the solution (ab2_ls_iterate: q [batch][N+1][nx] with q_N last, r like us, d like vs, dN like vsT, g0 like
 * lam0, f like lams with f_t in the row of lambda_{t+1}), the call returns z = -K^-1 h: the solution of the handle's
 * current LQ problem with all its vectors replaced by h, K the symmetric KKT matrix of the whole problem.  The
 * problem's own vectors give the primal solution, h = -zbar the adjoint's w (ab2_gar_adjoint), h = rho the tangent
 * (ab2_gar_tangent).  K is symmetric and h and z pair block for block, so the call is its own transpose: the VJP of z
 * with respect to h is resolve(zbar) and the JVP is resolve(hdot).
 * Only the vector half of the recursion runs; FB = [K; Z; Ahat] and VXX are read (in the layout the last backward
 * wrote, ab2_gar_device_ptr), together with the stage records' matrices (through the ring head) and C_N, G0:
 *   terminal  z_N = d_N / mu,  vx_N = q_N + C_N^T z_N
 *   stage t   V' = Vxx_{t+1},  v+ = vx_{t+1} + V' f_t,  rhat = r_t + B^T v+,
 *             [k; z] = -[[R + B^T V' B, D^T], [D, -mu I]]^-1 [rhat; d_t]   (Bunch-Kaufman, once per knot, instance and
 *             chunk of right-hand sides),  a = f_t + B k,
 *             vx_t = (qhat + Shat k) + C^T z  with qhat = q_t + A^T v+, Shat k = S k + A^T V' B k (the reference's order)
 *   initial   [x_0; lam_0] = -[[Vxx_0, G0^T], [G0, 0]]^-1 [vx_0; g0]
 *   forward   u_t = k + K x_t,  v_t = z + Z x_t,  x_{t+1} = a + Ahat x_t,  lam_{t+1} = vx_{t+1} + Vxx_{t+1} x_{t+1},
 *             v_N = z_N + Z_N x_N.
 * Every saddle-point matrix is read from its lower triangle, as the sweep's factorisations read theirs.
 * Layout: every rhs and out field is [nrhs][batch][...] in DEVICE memory; right-hand side j of instance b is block
 * j * batch + b.  A NULL rhs field is zero; an out field of nonzero size is required.  The out arrays hold the
 * backward pass's per-knot vectors before every rhs entry has been read, so no rhs array may overlap an out array
 * (an in-place re-solve such as q -> xs is refused).  `mueq` must be the mu of the last
 * backward.  The call writes the out arrays and nothing else: every output of the handle (FF .. LBDAS, status, pivot
 * statistics) is unchanged.  One launch on `stream`; right-hand side j's result is bit for bit independent of nrhs and
 * of its position among the right-hand sides (no atomics).
 * Errors (nothing is launched): AB2_ERR_UNSUPPORTED for dense, parametric (nth > 0) and parallel handles;
 * AB2_ERR_STATE when no backward (backward, sweep, their *_v twins, sweep_host*, adjoint, tangent, fddp_backward_pass)
 * has run since the last set_problem, assemble or cycle_append; AB2_ERR_INVALID for nrhs < 0, a NULL required out
 * field, an rhs array overlapping an out array, or mueq <= 0 with constraints.  Every shape a plain serial handle accepts
 * fits (one right-hand side needs max(nx^2 + (nu+nc+nx) nx + 2 nx nu + (nu+nc)(nu+nc+1), (nx+nc0)(nx+nc0+1)) +
 * 4 nx + max(nu+nc, nx+nc0) doubles of shared memory); a shape that did not would return AB2_ERR_UNSUPPORTED.  nrhs == 0 launches nothing. */
typedef struct ab2_lq_rhs {
  const double *q, *r, *d, *dN, *g0, *f;
} ab2_lq_rhs;
int ab2_gar_resolve  (ab2_gar_solver *s, double mueq, int nrhs, const ab2_lq_rhs *rhs,
                      const ab2_ls_trial *out, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_resolve_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs,
                      const ab2_lq_rhs *rhs, const ab2_ls_trial *out, void *stream);
/* A counter that every call rewriting FB / VXX or the records bumps (set_problem, assemble, cycle_append and every
 * backward listed above): a caller that keeps derivatives for later re-solves checks that the factorisation they
 * belong to is still the handle's.  A host-side increment; it changes nothing those calls compute. */
int ab2_gar_factor_epoch(const ab2_gar_solver *s, long long *epoch);

/* Derivatives of a parametric solution with respect to theta (handles of ab2_gar_create_parametric, nth > 0).  The
 * matrices do not depend on theta, so forward_theta's solution is affine in it, z(theta) = z_0 + J theta, and J is
 * made of the factors the last backward stored: FB = [K; Z; Ahat], FTH = [Kth; Zth; Yth], VXX, VXT, FBT (Z_N) and
 * F0 = KKT0FTH (rows x_0, then lam_0).  theta_tangent returns J d for directions d, theta_adjoint J^T zbar for
 * cotangents zbar (the gradient of a loss with respect to theta); neither refactors or sweeps.
 *   theta_tangent (the theta terms of forward_theta, without its feed-forward terms):
 *     x_0 = F0_x d,  lam_0 = F0_lam d
 *     t = 0..N-1:  u_t = K_t x_t + Kth_t d,  v_t = Z_t x_t + Zth_t d,  x_{t+1} = Ahat_t x_t + Yth_t d,
 *                  lam_{t+1} = Vxx_{t+1} x_{t+1} + Vxt_{t+1} d
 *     v_N = Z_N x_N   (the terminal knot has no theta term, as in forward_theta)
 *   theta_adjoint (its exact transpose), cotangents (xbar, ubar, vbar, vbar_N, lambar_0, lambar) and c_t the
 *   cotangent of x_t:
 *     c_N = xbar_N + Z_N^T vbar_N + Vxx_N lambar_N,  thbar = Vxt_N^T lambar_N        (the Vxx and Vxt terms for N >= 1)
 *     t = N-1..0:  thbar += Kth_t^T ubar_t + Zth_t^T vbar_t + Yth_t^T c_{t+1}  (+ Vxt_t^T lambar_t for t >= 1)
 *                  c_t = xbar_t + K_t^T ubar_t + Z_t^T vbar_t + Ahat_t^T c_{t+1}  (+ Vxx_t lambar_t for t >= 1)
 *     thbar += F0_x^T c_0 + F0_lam^T lambar_0
 * Layouts: dtheta and theta_bar are [nrhs][batch][nth]; out and cot are [nrhs][batch][...] in the solution's layouts
 * (ab2_ls_trial / ab2_ls_iterate, lams[t] = lambda_{t+1}); block j * batch + b is direction j of instance b.  Every
 * array is DEVICE memory.  A NULL cot field is zero; dtheta, theta_bar and every out field of nonzero size are
 * required.  No mu argument: only the stored factorisation is read.  The calls write the caller's arrays and nothing
 * else: every handle output (FF .. THHESS), the status words, the pivot statistics and ab2_gar_factor_epoch are
 * unchanged.  One launch each on `stream`; direction j's result is bit for bit independent of nrhs and of j's
 * position (one warp per instance and chunk of directions, no atomics).
 * Errors (nothing is launched), checked in this order: AB2_ERR_UNSUPPORTED for handles without parameters (nth = 0,
 * dense) and parallel handles (their theta is implicit); AB2_ERR_STATE when no backward has run since the last
 * set_problem or assemble; AB2_ERR_INVALID for nrhs < 0, a NULL required field, dtheta or cot overlapping out or
 * theta_bar, or out or theta_bar overlapping an output of the handle.  A shape whose one direction needs more than
 * 227 KB of shared memory returns AB2_ERR_UNSUPPORTED.  nrhs == 0 launches nothing. */
int ab2_gar_theta_tangent(ab2_gar_solver *s, int nrhs, const double *dtheta, const ab2_ls_trial *out, void *stream);
int ab2_gar_theta_adjoint(ab2_gar_solver *s, int nrhs, const ab2_ls_iterate *cot, double *theta_bar, void *stream);

/* Jacobians of the LQ solution with respect to the problem data: many cotangents (reverse mode) or many tangents
 * (forward mode) on the last backward's factorisation, through ab2_gar_resolve's program (resolve(h) = -K^-1 h), without
 * re-running the matrix recursion per right-hand side.
 *   adjoint_many, for each cotangent j:  y_j = resolve(zbar_j), with the cotangent fields as resolve's rhs fields
 *     (xs -> q, us -> r, vs -> d, vsT -> dN, lam0 -> g0, lams -> f).  y_j = -w_j with w_j as in ab2_gar_adjoint, so the
 *     vector gradients are y_j itself (dq = y_x, dr = y_u, dd = y_v, df = y_l, dg0 = y_l0, and the terminal dq_N, dd_N)
 *     and the matrix gradients are ab2_gar_adjoint's with -w replaced by y: dA = y_l,t+1 x_t^T + l_t+1 y_x,t^T,
 *     dQ = 1/2 (y_x x^T + x y_x^T), dG0 = y_l0 x_0^T + l_0 y_x0^T, ...
 *   tangent_many, for each tangent j:  rho_j = ab2_gar_tangent's right-hand side Kdot_j z + hdot_j, and
 *     zdot_j = -K^-1 rho_j = resolve(rho_j).
 * Layouts: `primal` is [batch][...] in the solver's output layouts, the solution of the current problem at this mu.
 * Every per-right-hand-side array (cotangent, dot, work, grad, out) is [nrhs][batch][...] in DEVICE memory: block
 * j * batch + b is right-hand side j of instance b.  grad and dot use the problem's record layouts (stage records'
 * pad double written as 0, never read).  A NULL cotangent or dot field is zero for every right-hand side; a NULL grad
 * field is not written.  `work` is caller-owned scratch in resolve's out layout (so the calls allocate nothing):
 * adjoint_many leaves y there, which is the vector gradient in the solution's layouts (a result); tangent_many leaves
 * rho there, in resolve's rhs layouts.
 * Launches, in order on `stream` without host synchronisation: adjoint_many runs resolve (cotangent -> work), then a
 * gradient kernel (work, primal -> grad); tangent_many runs a rho kernel (dot, primal -> work), then resolve
 * (work -> out).  Only the caller's arrays are written: every handle output (FF .. LBDAS, status, pivot statistics) is
 * unchanged and ab2_gar_factor_epoch does not move.  Records are read through the ring head (correct after
 * cycle_append and a backward).  Right-hand side j's results are bit for bit independent of nrhs and of j's position.
 * `mueq` must be the mu of the last backward.
 * Errors (nothing is launched), as ab2_gar_resolve: AB2_ERR_UNSUPPORTED for dense, parametric (nth > 0) and parallel
 * handles; AB2_ERR_STATE when no backward has run since the last set_problem, assemble or cycle_append;
 * AB2_ERR_INVALID for nrhs < 0, a NULL work (or, for tangent_many, out) field of nonzero size, a NULL primal field of
 * nonzero size, mueq <= 0 with constraints, or an overlap that would let one step read what an earlier step wrote:
 * cotangent or dot with work, work with primal or out, grad or out with primal or with each other, grad with work.
 * nrhs == 0 launches and writes nothing. */
int ab2_gar_adjoint_many  (ab2_gar_solver *s, double mueq, int nrhs, const ab2_ls_iterate *primal,
                           const ab2_ls_iterate *cotangent, const ab2_ls_trial *work,
                           const ab2_lq_grad *grad, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_adjoint_many_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs,
                           const ab2_ls_iterate *primal, const ab2_ls_iterate *cotangent,
                           const ab2_ls_trial *work, const ab2_lq_grad *grad, void *stream);
int ab2_gar_tangent_many  (ab2_gar_solver *s, double mueq, int nrhs, const ab2_ls_iterate *primal,
                           const ab2_lq_tangent *dot, const ab2_ls_trial *work,
                           const ab2_ls_trial *out, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_tangent_many_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs,
                           const ab2_ls_iterate *primal, const ab2_lq_tangent *dot,
                           const ab2_ls_trial *work, const ab2_ls_trial *out, void *stream);

/* The two streaming kernels of adjoint_many / tangent_many as stateless calls, generalised for higher derivatives of
 * the solve (every derivative of z = solve(P), of resolve and of these two maps is made of resolve and these two maps;
 * DESIGN section 2p).  K is affine in the data P, so for a data direction Pdot and a vector a in the solution's layout:
 *   rho(Pdot; a)   = Kdot(Pdot) a + hdot(Pdot): ab2_gar_tangent's right-hand side with z replaced by a (sym(Qdot),
 *                    sym(Rdot) included); rho_K(Pdot; a) = Kdot(Pdot) a, the same without the tangent's vector blocks
 *                    (qdot, rdot, ddot, fdot, qdot_N, ddot_N, g0dot);
 *   Gr(y; z)       = adjoint_many's gradient records for y and the primal z: dh = y, dK = y z^T read out of K's blocks
 *                    (symmetric part for Q and R, pad = +0.0); Gr_K(y; z) the same with every vector block written 0.
 * They pair as <Gr(y; z), Pdot> = <y, rho(Pdot; z)> and <Gr_K(y; z), Pdot> = <y, rho_K(Pdot; z)> = <z, rho_K(Pdot; y)>,
 * so Gr_K(y; z) = Gr_K(z; y) and the derivatives of each map are the other map again.
 *   rho_many,  for each right-hand side j:  out_j = rho^(v)(dot1_j; a1_j) + rho_K(dot2_j; a2_j) + e_j,
 *     rho^(v) = rho when with_vectors != 0, else rho_K.  out is in resolve's rhs layouts (q like xs with q_N last, r like
 *     us, d like vs, dN like vsT, g0 like lam0, f like lams).  dot2 == NULL: no second term (a2 is ignored);
 *     e == NULL: no e.
 *   grad_many, for each right-hand side j:  grad_j = Gr^(v)(y1_j; z1_j) + Gr_K(y2_j; z2_j),
 *     Gr^(v) = Gr when with_vectors != 0, else Gr_K.  y2 == NULL: no second pair (z2 is ignored).
 * Layouts: dot1, dot2, e, y1, y2, out and grad are [nrhs][batch][...] in DEVICE memory (block j * batch + b is
 * right-hand side j of instance b); dot and grad use the problem's record layouts (stage records' pad double written as
 * 0, never read).  A vector operand a1, a2, z1, z2 is [nrhs][batch][...] when its flag (*_each) is nonzero and
 * [batch][...] shared by every right-hand side when it is 0; a shared operand is staged once per knot, a per-direction one
 * read once per (direction, knot).  A NULL dot field is zero; every field of nonzero size of a1, y1, z1, e and out (and
 * of a2 with dot2, of z2 with y2) is required; a NULL grad field is not written.
 * At with_vectors != 0, shared a1 / z1 and no second term or e, the calls run adjoint_many's and tangent_many's kernels,
 * with their bits; every other mode runs the generalised instantiation, whose one-term results equal those bits.
 * Right-hand side j's results are bit for bit independent of nrhs and of j's position (each element is summed in a fixed
 * order: term 1, term 2, then e).
 * The calls read no factorisation and no mu: no state precondition, one launch on `stream`, and every handle output,
 * the status and ab2_gar_factor_epoch are unchanged.  Dense handles are served (their records have the same layout).
 * Errors (nothing is launched): AB2_ERR_UNSUPPORTED for parametric (nth > 0) and parallel handles, whose records have
 * another layout; AB2_ERR_INVALID for nrhs < 0, a NULL required argument or field, or an output field overlapping any
 * input field or another output field.  nrhs == 0 launches and writes nothing. */
int ab2_gar_rho_many (ab2_gar_solver *s, int nrhs, int with_vectors,
                      const ab2_lq_tangent *dot1, const ab2_ls_iterate *a1, int a1_each,
                      const ab2_lq_tangent *dot2, const ab2_ls_iterate *a2, int a2_each,
                      const ab2_ls_iterate *e, const ab2_ls_trial *out, void *stream);
int ab2_gar_grad_many(ab2_gar_solver *s, int nrhs, int with_vectors,
                      const ab2_ls_iterate *y1, const ab2_ls_iterate *z1, int z1_each,
                      const ab2_ls_iterate *y2, const ab2_ls_iterate *z2, int z2_each,
                      const ab2_lq_grad *grad, void *stream);

/* Iterative refinement of the LQ solution on the last backward's factorisation (what ParallelRiccatiSolver does to its
 * condensed system, parallel-solver.hxx:185-202, here for the whole serial solve).  At small penalties (mu = 1e-8 and
 * below) the fp64 recursion loses digits to the conditioning of the stage KKT systems; a step or two of refinement
 * with resolve as the correction solver recovers them.  For a solution estimate z = (x, u, v, lam) of K z = -h:
 *   residual    r = K z + h,   correction  delta = resolve(r) = -K^-1 r,   update  z <- z + delta.
 * With lam_{t+1} = lams[t] and lam_t = lams[t-1], the rows of r in resolve's rhs layouts are
 *   q-row  Q x_t + S u_t + C^T v_t + A^T lam_{t+1} - lam_t + q_t     (t = 0: + G0^T lam_0 instead of - lam_0)
 *   r-row  S^T x_t + R u_t + D^T v_t + B^T lam_{t+1} + r_t
 *   d-row  C x_t + D u_t - mu v_t + d_t
 *   f-row  A x_t + B u_t - x_{t+1} + f_t                             (in the row of lam_{t+1})
 *   q_N    Q_N x_N + C_N^T v_N - lam_N + q_N  (N = 0: + G0^T lam_0 instead of - lam_N),   d_N  C_N x_N - mu v_N + d_N
 *   g0     G0 x_0 + g0
 * with Q and R used as stored.  These are the rows ab2_gar_kkt_error takes norms of, summed by the same kernel, so
 * ||r||_inf equals the largest of its three norms exactly.  h is the problem's own vectors (ab2_gar_refine: the primal
 * solution) or a caller's resolve right-hand sides (ab2_gar_refine_many: the adjoint's w with h = -zbar, the tangent
 * with h = rho, Jacobian columns, any resolve output).
 *
 * ab2_gar_refine / _v refine the handle's own trajectory outputs (XS, US, VS, VST, LBD0, LBDAS) in place against the
 * current problem's vectors.  Every other output (FF, FB, VXX, VX, FFT, FBT, KKT0, status, pivot statistics) is
 * bit-identical afterwards and ab2_gar_factor_epoch does not move.  The residual and correction live in a buffer the
 * handle owns, allocated on the first call.
 * ab2_gar_refine_many / _v refine z ([nrhs][batch][...] in the solution's layouts) in place against the right-hand
 * sides rhs ([nrhs][batch][...] in resolve's rhs layouts; a NULL field is zero).  `work` is caller-owned: q .. f in
 * resolve's rhs layouts for the residual, xs .. lams in the solution's layouts for the correction, all [nrhs][batch]
 * [...] on the device.  After a call with steps >= 1 it holds the last residual (of the iterate before the last
 * update) and the last correction.  Right-hand side j's result is bit for bit independent of nrhs and of j's position.
 * norms (optional, NULL = not written): [nrhs][batch][steps + 1] doubles (nrhs = 1 for ab2_gar_refine) in device or
 * host memory: ||r||_inf of the input iterate and of each refined iterate.  A host array is written by a stream-ordered
 * copy from a buffer the handle owns (allocated when a larger one is first needed): read it after synchronising
 * `stream`.  steps = 0 computes only the first column and changes nothing else; steps = 0 without norms does nothing.
 * Launches, in order on `stream` without host synchronisation: per step a residual kernel, resolve's program and an
 * update kernel; with norms, one more residual launch at the end for the last column.
 * `mueq` must be the mu of the last backward; the _v twins take a per-instance mu as ab2_gar_resolve_v does.
 * Errors (nothing is launched): AB2_ERR_UNSUPPORTED for dense, parametric (nth > 0) and parallel handles;
 * AB2_ERR_STATE when no backward has run since the last set_problem, assemble or cycle_append, and for ab2_gar_refine
 * also when the trajectory outputs do not hold the primal solution of that factorisation (no forward since the last
 * backward, a backward alone, or an ab2_gar_adjoint / ab2_gar_tangent call since the last forward); AB2_ERR_INVALID for
 * steps < 0, nrhs < 0, a NULL z or work field of nonzero size, mueq <= 0 with constraints, or an overlap that would let
 * a launch read what an earlier launch of the same step wrote: rhs with z or work, z with itself or work, the two
 * halves of work with each other or themselves.  nrhs == 0 launches and writes nothing. */
typedef struct ab2_lq_refine_work {
  double *q, *r, *d, *dN, *g0, *f;          /* residual, resolve's rhs layouts   */
  double *xs, *us, *vs, *vsT, *lam0, *lams; /* correction, the solution's layouts */
} ab2_lq_refine_work;
int ab2_gar_refine  (ab2_gar_solver *s, double mueq, int steps, double *norms, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_refine_v(ab2_gar_solver *s, const double *mueq, int memspace, int steps, double *norms, void *stream);
int ab2_gar_refine_many  (ab2_gar_solver *s, double mueq, int nrhs, int steps, const ab2_lq_rhs *rhs,
                          const ab2_ls_trial *z, const ab2_lq_refine_work *work, double *norms, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_refine_many_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs, int steps,
                          const ab2_lq_rhs *rhs, const ab2_ls_trial *z, const ab2_lq_refine_work *work,
                          double *norms, void *stream);

/* Gradients of the factorisation with respect to the problem data: the reverse mode of the backward recursion, for
 * losses on the gains and the cost-to-go (a feedback law u = k_0 + K_0 x fitted to demonstrations, inverse LQR on
 * gains, a terminal cost trained against Vxx_0, vx_0).  The backward pass maps the records and mu to, per stage knot,
 * FF_t = [k; z; a], FB_t = [K; Z; Ahat], Vxx_t, vx_t and, at the terminal knot, FFT = z_N, FBT = Z_N, Vxx_N, vx_N.  For
 * cotangents of those outputs the call returns the gradient with respect to every record entry, with Q and R as
 * symmetric arguments (as ab2_gar_adjoint).  Cotangents of Vxx_t are symmetrised, which is exact: Vxx_t is symmetric.
 * Vxx_t is read only by knot t-1, so the pass runs forward in time, carrying Vbar, vbar (seeded with the Vxx_0, vx_0
 * cotangents).  Per stage knot, with V' = Vxx_{t+1}, v' = vx_{t+1}, X = [[K, k], [Z, z]], Shat = S + A^T V' B,
 * v+ = v' + V' f, M = [[R + B^T V' B, D^T], [D, -mu I]] (factored again from its lower triangle, as resolve does),
 * sym(M) = (M + M^T) / 2 and the caller's cotangents marked 0:
 *   closed loop  Kb = Kb0 + B^T Ahatb,  kb = kb0 + B^T ab,  Bb = Ahatb K^T + ab k^T,  Ab = Ahatb,  fb = ab
 *   value        Qb = Vbar,  qb = vbar,  Shatb = Vbar K^T + vbar k^T,  Kb += Shat^T Vbar,  kb += Shat^T vbar,
 *                Cb = Z Vbar + z vbar^T,  Zb = Zb0 + C Vbar,  zb = zb0 + C vbar
 *   solve        P = -M^-1 [[Kb, kb], [Zb, zb]];  Shatb += P_u[:, :nx]^T,  rb = P_u[:, nx],  Cb += P_c[:, :nx],
 *                db = P_c[:, nx],  Rb = sym(P_u X_u^T),  Db = P_c X_u^T + X_c P_u^T  (X_u = [K, k], X_c = [Z, z]),
 *                Sb = Shatb
 *   products     Ab += 2 V' A Qb + V' B Shatb^T + v+ qb^T,  Bb += 2 V' B Rb + V' A Shatb + v+ rb^T,
 *                vb+ = A qb + B rb,  fb += V' vb+
 *   carry        Vbar_{t+1} = sym(Vxxb0_{t+1}) + sym(A Qb A^T + B Rb B^T + A Shatb B^T + vb+ f^T),  vbar_{t+1} = vxb0_{t+1} + vb+
 * and at the terminal knot (Z_N = C_N / mu, z_N = d_N / mu):  Zb = Zb0_N + C_N Vbar,  zb = zb0_N + C_N vbar,
 *   C_Nb = Z_N Vbar + z_N vbar^T + Zb / mu,  d_Nb = zb / mu,  Q_Nb = Vbar,  q_Nb = vbar.
 * G0 and g0 do not enter the factorisation: a non-NULL G0 / g0 grad field is zero-filled.  mu is not differentiated.
 *
 * Layouts (DEVICE arrays): cotangents as ab2_gar_get returns the outputs -- ff [batch][N][nu+nc+nx], fb
 * [batch][N][(nu+nc+nx)*nx] row-major, vxx [batch][N+1][nx*nx] full column-major blocks (not the packed physical
 * layout), vx [batch][N+1][nx], fft [batch][nct], fbt [batch][nct*nx]; a NULL field is a zero cotangent.  `grad` has
 * the problem's layouts (stage records' pad double written as 0) and is overwritten; a NULL field is not written.
 * One launch on `stream`: one warp per instance, or one CTA per instance when the shape's shared memory leaves room for
 * no other.  Only the caller's grad arrays are written: every output of the handle, its status, pivot statistics and
 * ab2_gar_factor_epoch are unchanged, and no memory is allocated (a host mueq array of the _v twin is staged like
 * ab2_gar_sweep_v's).  Records are read through the ring head, Vxx in the layout the last backward wrote.  The
 * results are deterministic: every entry is summed by one lane in a fixed order.  `mueq` must be the mu of the last
 * backward.
 * Errors (nothing is launched): AB2_ERR_UNSUPPORTED for dense, parametric (nth > 0) and parallel handles, and for a
 * shape whose item needs more than 227 KB of shared memory (5 nx^2 + 3 nx nu + nc nx + nu^2 + 5 nx +
 * (nu+nc)(2 nx + nu + nc + 3) doubles; C1-C5 fit);
 * AB2_ERR_STATE unless a backward on the problem's own vectors has run since the last set_problem, assemble or
 * cycle_append (after ab2_gar_adjoint or ab2_gar_tangent FF and VX hold that solve's vectors, until the next
 * backward); AB2_ERR_INVALID for mueq <= 0 with constraints, or a grad array that overlaps a cotangent array or an
 * output of the handle. */
typedef struct ab2_factor_cotangent {
  const double *ff, *fb, *vxx, *vx, *fft, *fbt;
} ab2_factor_cotangent;
int ab2_gar_factor_adjoint  (ab2_gar_solver *s, double mueq, const ab2_factor_cotangent *cot,
                             const ab2_lq_grad *grad, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_factor_adjoint_v(ab2_gar_solver *s, const double *mueq, int memspace,
                             const ab2_factor_cotangent *cot, const ab2_lq_grad *grad, void *stream);

/* Forward mode of the factorisation: the tangents of FF, FB, VXX, VX, FFT, FBT along a tangent pdot of the problem
 * records -- the sensitivity of the whole gain schedule K_t, or of every Vxx_t, to a few parameters that enter A, B,
 * Q, ... in one call per parameter.  It is the exact transpose of ab2_gar_factor_adjoint: <cbar, ydot> =
 * <factor_adjoint(cbar), pdot> for any cbar and pdot.  Q and R enter as sym(Qdot), sym(Rdot) (as ab2_gar_tangent), so an
 * asymmetric Qdot acts as its symmetric part.  G0 and g0 do not enter the factorisation (their fields are ignored);
 * mu is not differentiated.  The tangent recursion runs backward in time, as the sweep does, carrying Vd', vd' (the
 * tangents of Vxx_{t+1}, vx_{t+1}).  At the terminal knot (Z_N = C_N / mu, z_N = d_N / mu as stored):
 *   Zd_N = Cd_N / mu,  zd_N = dd_N / mu,  Vxxd_N = sym(Qd_N + Cd_N^T Z_N + C_N^T Zd_N),  vxd_N = qd_N + Cd_N^T z_N + C_N^T zd_N
 * and per stage knot, with V' = Vxx_{t+1}, X = [[K, k], [Z, z]], Shat = S + A^T V' B, v+ = vx_{t+1} + V' f and
 * M = [[R + B^T V' B, D^T], [D, -mu I]] recomputed from the record and the stored factor (M factored again from its
 * lower triangle, as resolve does):
 *   products     vd+ = vd' + Vd' f + V' fd,   Shatd = Sd + Ad^T V' B + A^T Vd' B + A^T V' Bd,
 *                Rhatd = sym(Rd) + Bd^T V' B + B^T V' Bd + B^T Vd' B,   Qhatd = sym(Qd) + Ad^T V' A + A^T V' Ad + A^T Vd' A,
 *                rhatd = rd + Bd^T v+ + B^T vd+,   qhatd = qd + Ad^T v+ + A^T vd+
 *   solve        [[Kd, kd], [Zd, zd]] = -M^-1 [[Rhatd K + Dd^T Z + Shatd^T, Rhatd k + Dd^T z + rhatd], [Dd K + Cd, Dd k + dd]]
 *   closed loop  Ahatd = Ad + Bd K + B Kd,   ad = fd + Bd k + B kd
 *   value        Vxxd_t = sym(Qhatd + Shatd K + Shat Kd + Cd^T Z + C^T Zd),   vxd_t = qhatd + Shatd k + Shat kd + Cd^T z + C^T zd
 * (Qhatd is formed as Qd + A^T (Vd' A + 2 V' Ad), which has the same symmetric part; only that part enters Vxxd_t.)
 *
 * Layouts (DEVICE arrays): `dot` is ab2_lq_tangent in the problem's layouts, logical knot order (stage
 * [batch][N][stage_record], term [batch][term_record]; the pad double is never read); a NULL field is a zero tangent.
 * `out` has ab2_gar_get's layouts, those of ab2_gar_factor_adjoint's cotangents: ff [batch][N][nu+nc+nx], fb
 * [batch][N][(nu+nc+nx)*nx] row-major, vxx [batch][N+1][nx*nx] full column-major blocks (exactly symmetric), vx
 * [batch][N+1][nx], fft [batch][nct], fbt [batch][nct*nx] row-major.  A NULL out field is not written (the recursion
 * still carries Vxxd and vxd).
 * One launch on `stream`: one warp per instance, or one CTA per instance when the shape's shared memory leaves room for
 * no other.  Only the caller's out arrays are written: every output of the handle, its status, pivot statistics and
 * ab2_gar_factor_epoch are unchanged, and no memory is allocated (a host mueq array of the _v twin is staged like
 * ab2_gar_sweep_v's).  Records are read through the ring head, Vxx in the layout the last backward wrote.  The results
 * are deterministic: every entry is summed by one lane in a fixed order.  `mueq` must be the mu of the last backward.
 * Errors (nothing is launched): AB2_ERR_UNSUPPORTED for dense, parametric (nth > 0) and parallel handles, and for a
 * shape whose item needs more than 227 KB of shared memory (4 nx^2 + 5 nx nu + nu^2 + nc nx + 4 nx +
 * (nu+nc)(2 nx + nu + nc + 3) doubles, rounded up to even; C1-C5 fit); AB2_ERR_STATE unless a backward on the
 * problem's own vectors has run since the last set_problem, assemble or cycle_append (not after ab2_gar_adjoint or
 * ab2_gar_tangent, until the next backward); AB2_ERR_INVALID for mueq <= 0 with constraints, or an out array that
 * overlaps a dot array or an output of the handle. */
typedef struct ab2_factor_tangent {
  double *ff, *fb, *vxx, *vx, *fft, *fbt;
} ab2_factor_tangent;
int ab2_gar_factor_tangent  (ab2_gar_solver *s, double mueq, const ab2_lq_tangent *dot,
                             const ab2_factor_tangent *out, void *stream);
/* The same with a per-instance mu: mueq [batch] in host or device memory, checked and staged like ab2_gar_sweep_v. */
int ab2_gar_factor_tangent_v(ab2_gar_solver *s, const double *mueq, int memspace,
                             const ab2_lq_tangent *dot, const ab2_factor_tangent *out, void *stream);

/* The rest of SolverProxDDP's inner iteration (solver-proxddp.hxx:555-699) around the sweep, batched over the
 * instances: multiplier estimates, Lagrangian gradients and stopping criteria.  With these, the LQ right-hand side
 * ab2_gar_assemble reads and the gradients ab2_gar_directional_derivative reads are produced on the device.
 * All array arguments are DEVICE pointers in the layouts of ab2_lq_inputs / ab2_ls_iterate: stage arrays
 * [batch][N][.], terminal and initial arrays [batch][.], matrices column-major, xs [batch][N+1][nx],
 * lam0 [batch][nc0], lams [batch][N][nx] (lams[1..N]), vs [batch][N][nc], vsT [batch][nct].
 *
 * Normal-cone projection per row, from the bounds encoding of ab2_lq_inputs (the same rows the active-set rule
 * above keeps): an equality row (lo = +inf) has NC(z) = z (equality-constraint.hpp:37-40); every other row has
 * NC(z) = z - max(min(z, hi), lo) (box-constraint.hpp:27-37), i.e. max(z, 0) for the negative orthant
 * (lo = -inf, hi = 0, negative-orthant.hpp:36-38). */
typedef struct ab2_mult_inputs {
  const double *xs, *lam0, *lams, *vs, *vsT; /* the iterate the estimates are computed at                       */
  const double *prev_vs, *prev_vsT;          /* workspace_.prev_vs, laid out like vs / vsT                      */
  const double *init_value;                  /* [batch][nc0] init_data value_ (assemble's g0)                   */
  const double *xnext, *fs;                  /* EXACTLY ONE: xnext [batch][N][nx] (dd.xnext_; vector-space
                                                difference fs[t+1] = xnext_t - x_{t+1}) or fs [batch][N][nx]
                                                given by a caller on a manifold                                 */
  const double *cval, *cval_N;               /* constraint values [batch][N][nc], [batch][nct]                  */
  const double *lo, *hi, *loN, *hiN;         /* [nc] / [nct] row bounds, shared by all knots and instances      */
  double mu, mu_dyn;
} ab2_mult_inputs;
typedef struct ab2_mult_outputs {
  double *slack;                                  /* [batch][N][nx] dyn_slacks[1..N] (assemble's slack)      */
  double *lam0_plus, *lams_plus, *vs_plus, *vsT_plus; /* lams_plus / vs_plus: an ab2_ls_iterate for al_value */
  double *shifted, *shifted_N;                    /* shifted_constraints                                     */
  double *Lv, *Lv_N;                              /* Lvs                                                     */
} ab2_mult_outputs;
/* Replaces: SolverProxDDP::computeMultipliers, solver-proxddp.hxx:220-318, for every instance (one warp each):
 *   fs0 = init_value,  lam0_plus = lam0 + fs0 / mu   (mu, not mu_dyn: :246-247),
 *   fs[t+1] = xnext_t - x_{t+1},  lams_plus[t+1] = lams[t+1] + fs[t+1] / mu_dyn   (:263-264),
 *   shifted = cval + mu prev_vs,  Lv = NC(shifted) - mu vs,  vs_plus = (1/mu) NC(shifted),
 *   stage_infeas = mu (vs_plus - prev_vs)   (:277-286; the terminal block likewise when nct > 0, :292-314).
 * dst [batch][2] (host or device) = [prim_infeas, finite]: prim_infeas = max(|stage_infeas|_inf over all knots,
 * |fs|_inf over fs0..fs_N) (:315-316); finite = 1.0 if every lams_plus and Lv entry is finite, else 0.0 -- the
 * reference returns false at the first non-finite one (RET_FALSE_IF_NAN, :248, 265, 289, 313); prim_infeas of
 * such an instance is unspecified.  Every output array is required (arrays of zero size may be NULL). */
int ab2_gar_multipliers(ab2_gar_solver *s, const ab2_mult_inputs *in, const ab2_mult_outputs *out, double *dst,
                        int memspace, void *stream);
/* The same with per-instance mu [batch] and mu_dyn [batch] (DEVICE; in->mu and in->mu_dyn are ignored); each
 * instance's mu_inv = 1 / mu is computed from its own mu. */
int ab2_gar_multipliers_v(ab2_gar_solver *s, const ab2_mult_inputs *in, const double *mu, const double *mu_dyn,
                          const ab2_mult_outputs *out, double *dst, int memspace, void *stream);

typedef struct ab2_lag_inputs {
  const double *lx, *lu, *lx_N;        /* cost gradients cost_data->Lx_, Lu_: [batch][N][nx], [batch][N][nu], [batch][nx] */
  const double *Jx, *Ju;               /* dynamics Jacobians [batch][N][nx*nx], [batch][N][nx*nu]                          */
  const double *cJx, *cJu, *cJx_N;     /* constraint Jacobians [batch][N][nc*nx], [batch][N][nc*nu], [batch][nct*nx]       */
  const double *G0;                    /* init_data Jx_ [batch][nc0*nx]                                                    */
  const double *lam0, *lams, *vs, *vsT; /* any multiplier set: the iterate (LQ right-hand side) or the *_plus estimates
                                           (ALFunction::directionalDerivative, merit-function.hxx:82-84)                  */
  int force_initial_condition;         /* nonzero: Lx_0 = 0, as innerLoop does after the call (solver-proxddp.hxx:592-594) */
} ab2_lag_inputs;
typedef struct ab2_lag_outputs {
  double *Lx, *Lx_N, *Lu; /* assemble layout: [batch][N][nx], [batch][nx], [batch][N][nu]      */
  double *Lxs, *Lus;      /* directional-derivative layout: [batch][N+1][nx], [batch][N][nu]   */
} ab2_lag_outputs;
/* Replaces: LagrangianDerivatives::compute, core/lagrangian.hpp:29-92, for every instance and knot:
 *   Lx_t = lx_t + Jx_t^T lam_{t+1} + cJx_t^T v_t - lam_t  (t >= 1; t = 0: + G0^T lam0 instead of - lam_0),
 *   Lu_t = lu_t + Ju_t^T lam_{t+1} + cJu_t^T v_t,
 *   Lx_N = lx_N + cJx_N^T v_N - lam_N  (N = 0: Lx_0 = lx_N + cJx_N^T v_N + G0^T lam0).
 * Writes whichever of the five outputs are non-NULL (at least one). */
int ab2_gar_lagrangian_gradient(ab2_gar_solver *s, const ab2_lag_inputs *in, const ab2_lag_outputs *out, void *stream);

/* Replaces: SolverProxDDP::computeCriterion, solver-proxddp.hxx:703-732: dst [batch][2] (host or device) =
 * [inner_criterion, dual_infeas].  Lxs [batch][N+1][nx], Lus [batch][N][nu] (lagrangian_gradient's outputs),
 * init_value [batch][nc0] = fs0, slack [batch][N][nx] = fs[1..N], Lv [batch][N][nc], Lv_N [batch][nct].
 * As in the reference, knot i's dynamics residual is dyn_slacks[i]: inner_criterion covers fs0..fs_{N-1} (fs0 only
 * when N >= 1) and never fs_N; dual_infeas = max(|Lxs|_inf over knots 0..N, |Lus|_inf). */
int ab2_gar_criterion(ab2_gar_solver *s, const double *Lxs, const double *Lus, const double *init_value,
                      const double *slack, const double *Lv, const double *Lv_N, double *dst, int memspace,
                      void *stream);

/* SolverFDDPTpl::backwardPass, solvers/fddp/solver-fddp.hxx:204-277 (SURVEY section 8f rank 4), for a batch: the
 * unconstrained recursion is the sweep's own stage step with A = Jx, B = Ju, f_i = fs[i+1], Q = Lxx + preg I,
 * S = Lxu, R = Luu + preg I, q = Lx, r = Lu (nc = 0; the LLT of Quu (:259-260) is the Bunch-Kaufman factorisation
 * on its all-1x1-pivots path), so this assembles the knots from FDDP's buffers on the device, runs backward()
 * and adds FDDP's own bookkeeping: Vx_i += Vxx_i fs[i] (:219-220, 274-276) and Quuks_i = Quu_i k_i (:264).
 * DEVICE pointers: Jx [batch][N][nx*nx], Ju [batch][N][nx*nu] (column-major), fs [batch][N+1][nx], Lxx, Lxu, Luu,
 * Lx, Lu per stage, Lxx_N [batch][nx*nx], Lx_N [batch][nx].  The solver must have nc = nct = 0, nc0 = nx.
 * After the call: K_i, k_i = the first nu rows of FB / FF (kkt_fb, kkt_ff), Vxx_i = VXX (symmetric from the lower
 * triangle, + preg on the diagonal carried by Q); Vx_out [batch][N+1][nx] and Quuks_out [batch][N][nu] (device,
 * may be NULL) receive FDDP's Vx_ (with the defect term) and Quuks_. */
typedef struct ab2_fddp_inputs {
  const double *Jx, *Ju, *fs, *Lxx, *Lxu, *Luu, *Lx, *Lu, *Lxx_N, *Lx_N;
  double preg;
} ab2_fddp_inputs;
int ab2_fddp_backward_pass(ab2_gar_solver *s, const ab2_fddp_inputs *in, double *Vx_out, double *Quuks_out, void *stream);
/* The same with a per-instance preg [batch] (DEVICE; in->preg is ignored). */
int ab2_fddp_backward_pass_v(ab2_gar_solver *s, const ab2_fddp_inputs *in, const double *preg, double *Vx_out,
                             double *Quuks_out, void *stream);

/* Replaces: cycleAppend(knot), proximal-riccati.hxx:79-86 + the problem rotation the
 * caller performs (solver-proxddp.hxx:202-209): factors and stage knots of every
 * instance shift one knot to the left; `new_last` ([batch][stage_record], memspace)
 * becomes stage knot N-1; its factor slot and kkt0 are zeroed.
 * O(1) in the horizon: the per-knot factor arrays and the solver-owned copy of the stage records are
 * rings -- the call advances a head index, zeroes ONE factor slot and writes ONE record per instance; the
 * getters (ab2_gar_get / get_range / get_gains / get_problem / first_step_policy) and the kernels apply the
 * head, and the next backward() rewrites the factors in plain knot order.  Raw device pointers
 * (ab2_gar_device_ptr, ab2_gar_problem_ptr) see the physical layout: stage knot t sits in slot
 * (t + head) mod N, heads from ab2_gar_ring_heads (0 except after a cycle).  The parallel solver drops
 * every factor instead (parallel-solver.hxx:246-258). */
int ab2_gar_cycle_append(ab2_gar_solver *s, const double *new_last, int memspace, void *stream);

int ab2_gar_ring_heads(const ab2_gar_solver *s, int *factor_head, int *stage_head);
/* Profiling aid (environment AB2_PHASE_CLOCKS=1 at create): clock64() cycles per phase of the CTA-per-instance
 * kernel, summed over the knots of instance 0 since the last call; 16 counters (csrc/riccati_block.cuh). */
int ab2_gar_phase_clocks(ab2_gar_solver *s, long long *dst16);

int ab2_gar_synchronize(ab2_gar_solver *s, void *stream);
/* Page-locked host memory for the buffers handed to set_problem / get / sweep_host: copies to and
 * from it are asynchronous (what the reference's mimalloc arena is to its hot loop,
 * solver-proxddp.hpp:177-178: allocate once, never in the loop).  free(NULL) is a no-op. */
int ab2_gar_pinned_alloc(size_t bytes, void **out);
void ab2_gar_pinned_free(void *p);
/* Kernels launched by this solver since creation (for bench accounting); the getters' copies do not count. */
long ab2_gar_launch_count(const ab2_gar_solver *s);
/* Shared memory per CTA / registers etc. of the kernel serving this solver
 * (*regs_per_thread: low 16 bits = registers, high 16 bits = resident CTAs per SM). */
int ab2_gar_kernel_info(const ab2_gar_solver *s, int *group_lanes, int *smem_bytes_per_cta,
                        int *threads_per_cta, int *grid, int *regs_per_thread);
const char *ab2_gar_last_error(void);
const char *ab2_gar_version(void);

#ifdef __cplusplus
}
#endif
#endif /* ALIGATOR_B200_GAR_H */
