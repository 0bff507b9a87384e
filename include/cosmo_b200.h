/*
 * cosmo_b200.h -- C ABI of the H100-native ADMM iteration engine that drops in
 * behind COSMO.jl's `COSMO.optimize!` hot loop.
 *
 * Boundary (reference file:line, COSMO.jl v0.8.11):
 *   - the engine owns everything between `allocate_loop_variables!` / the
 *     operator warm start (src/solver.jl:125-129) and `recover_mu!` at loop
 *     exit (src/solver.jl:167); `setup!` (src/setup.jl:18-64: Ruiz scaling,
 *     row ranges) stays upstream and `reverse_scaling!` /
 *     `reverse_decomposition!` (src/solver.jl:179-190) stay downstream, in
 *     unchanged host code.
 *   - per-plugin entry points mirror the reference's own seams:
 *       AbstractKKTSolver  ctor / solve! / update_rho! / free_memory!
 *                          (src/linear_solver/kktsolver.jl:5-13, 310-313)
 *       AbstractConvexSet  project!(x, set)          (src/convexset.jl:885-891)
 *
 * Conventions
 *   - plain pointers and sizes only; array arguments are owned by the caller
 *     (Julia GC memory under GC.@preserve, or a CuArray). The engine copies
 *     inputs to HBM inside the call and never keeps a caller pointer.  Array
 *     arguments are HOST pointers, except where "host or device" is said
 *     (see "Caller arrays in device memory" below).
 *   - matrices arrive exactly as Julia stores them: SparseMatrixCSC{T,Int64},
 *     1-based colptr/rowval (`index_base = 1`); `index_base = 0` accepts
 *     SciPy-style 0-based int64 arrays.
 *   - `dtype` selects Float64 / Float32 models (Model{Float64}, Model{Float32}).
 *   - every function returns 0 on success or a negative COSMO_B200_ERR_* code;
 *     `cosmo_b200_last_error` returns the message (the Julia shim rethrows it as
 *     ErrorException). Solver outcomes are NOT errors: they are reported in
 *     `cosmo_b200_result.status` (1:1 with the reference's status Symbols,
 *     src/solver.jl:113,161,175,311-353).
 *   - one host thread per handle; `solve` is synchronous.
 */
#ifndef COSMO_B200_H
#define COSMO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COSMO_B200_ABI_VERSION 4

typedef struct cosmo_b200_handle cosmo_b200_handle;

/* cosmo_b200_problem.flags */
#define COSMO_B200_PROBLEM_EQUILIBRATE 1 /* run scale_ruiz! on the device (data handed over unscaled) */

enum {
  COSMO_B200_OK = 0,
  COSMO_B200_ERR_INVALID = -1,     /* bad argument / dimension mismatch (interface.jl:369-392) */
  COSMO_B200_ERR_UNSUPPORTED = -2, /* unknown set type, BigFloat, unsupported option: shim falls back to Julia */
  COSMO_B200_ERR_CUDA = -3,        /* CUDA runtime error or no usable sm_90 device */
  COSMO_B200_ERR_ALLOC = -4,
  COSMO_B200_ERR_NCCL = -5,
  COSMO_B200_ERR_NUMERICAL = -6    /* eigensolver failed to converge (LAPACK info != 0, convexset.jl:186) */
};

enum { COSMO_B200_F64 = 0, COSMO_B200_F32 = 1 };

/* cone types in `sort_sets` order (src/interface.jl:466-475) */
enum {
  COSMO_B200_ZERO = 0,         /* ZeroSet,          convexset.jl:16-28   */
  COSMO_B200_NONNEG = 1,       /* Nonnegatives,     convexset.jl:52-74   */
  COSMO_B200_BOX = 2,          /* Box(l,u),         convexset.jl:803-847 */
  COSMO_B200_SOC = 3,          /* SecondOrderCone,  convexset.jl:92-114  */
  COSMO_B200_PSD_SQUARE = 4,   /* PsdCone / DensePsdCone,                 convexset.jl:271-321 */
  COSMO_B200_PSD_TRIANGLE = 5, /* PsdConeTriangle / DensePsdConeTriangle, convexset.jl:362-412 */
  /* 3-d cones (sort_sets puts every remaining type in class 6 too, interface.jl:473) */
  COSMO_B200_EXP = 6,          /* ExponentialCone,      convexset.jl:497-618 */
  COSMO_B200_DUAL_EXP = 7,     /* DualExponentialCone,  convexset.jl:749-789 */
  COSMO_B200_POW = 8,          /* PowerCone(alpha),     convexset.jl:625-742 */
  COSMO_B200_DUAL_POW = 9,     /* DualPowerCone(alpha), convexset.jl:765-789 */
  COSMO_B200_PSD_TRIANGLE_COMPLEX = 10 /* PsdConeTriangle{T, Complex{T}}(dim), dim = N^2 (convexset.jl:344-360,444-490);
                                          projected through the real 2N x 2N embedding [[A, -B], [B, A]]: in shared
                                          memory up to N = 48, through the large-cone path (tensor cores) beyond */
};

/* ---- custom convex cones (the reference's `AbstractConvexCone` subtypes with a `project!` method) --------------------
   A set with type = COSMO_B200_CUSTOM is projected by CUDA C++ that the user writes.  Its cosmo_b200_set has
   u = the const cosmo_b200_custom_cone* of its type, l = its n_params parameters in the model's element type T (NULL when
   n_params = 0; never scaled, as scale! of a custom cone is a no-op), alpha = tol = max_iter = 0.  The engine compiles
   each type with NVRTC (libnvrtc.so.12, loaded with dlopen on first use: without it create returns
   COSMO_B200_ERR_UNSUPPORTED) for sm_90a when the engine is created, once per process for each (name, source,
   granularity, n_params, flags, dtype), and launches the projection inside admm_z! after the built-in cones.
   Custom cones sort with the exponential and power cones (class 6), take one scalar scaling per cone (Ruiz) and the
   inequality rho.  `source` defines, in namespace `name`,
     template <typename T> __device__ void project(T* x, long long dim, const T* p, int lane, int width);
     template <typename T> __device__ bool in_dual(const T* x, long long dim, T tol, const T* p, int lane, int width);
     template <typename T> __device__ bool in_pol_recc(const T* x, long long dim, T tol, const T* p, int lane, int width);
   the last two only when flags has COSMO_B200_CUSTOM_HAS_IN_DUAL / _HAS_IN_POL_RECC.  All `width` lanes of a cone call a
   function together (lane = 0 .. width-1); x is the cone's `dim` rows, p its parameters.  project overwrites x (which
   holds w_s) with its projection.  The primal infeasibility certificate asks in_dual(-dy) and the dual one
   in_pol_recc(A dx) (convexset.jl:928-936); a cone is certified when every lane returns true.  A type without the hook
   never certifies, so such a problem runs to Max_iter_reached where the reference would raise a MethodError (its
   documentation calls this "infeasibility detection is disabled").  No #include is needed: a prelude defines, in
   namespace cosmo_cone, sum(v, width), max(v, width) and all(b, width) over the lanes of a cone, which every lane of
   the cone must call. */
#define COSMO_B200_CUSTOM 11 /* cosmo_b200_set.type */
enum {
  COSMO_B200_CUSTOM_THREAD = 0, /* one lane per cone */
  COSMO_B200_CUSTOM_WARP = 1,   /* 32 lanes: one warp per cone */
  COSMO_B200_CUSTOM_BLOCK = 2   /* 256 lanes: one thread block per cone */
};
#define COSMO_B200_CUSTOM_HAS_IN_DUAL 1
#define COSMO_B200_CUSTOM_HAS_IN_POL_RECC 2
typedef struct {
  const char* name;    /* C identifier: the namespace of the device functions in `source` (not "cosmo_cone") */
  const char* source;  /* CUDA C++; compiler messages name its lines as `name`(line) */
  int32_t granularity; /* COSMO_B200_CUSTOM_THREAD | _WARP | _BLOCK */
  int32_t n_params;    /* values of T per cone */
  int32_t flags;       /* COSMO_B200_CUSTOM_HAS_* */
  int32_t reserved;    /* 0 */
} cosmo_b200_custom_cone;

/* status (src/solver.jl:113,161,175,311-353) */
enum {
  COSMO_B200_UNDETERMINED = 0,
  COSMO_B200_SOLVED = 1,
  COSMO_B200_MAX_ITER_REACHED = 2,
  COSMO_B200_TIME_LIMIT_REACHED = 3,
  COSMO_B200_PRIMAL_INFEASIBLE = 4,
  COSMO_B200_DUAL_INFEASIBLE = 5,
  COSMO_B200_UNSOLVED = 6
};

/* accelerators (COSMOAccelerators.jl types selectable through settings.accelerator) */
enum { COSMO_B200_ACC_EMPTY = 0, COSMO_B200_ACC_ANDERSON = 1 };

/* AndersonAccelerator{T, type, memory, regularizer} parameters and the activation reason (accelerator_interface.jl:1-48) */
enum { COSMO_B200_AA_TYPE2_QR = 0, COSMO_B200_AA_TYPE2_NORMAL = 1, COSMO_B200_AA_TYPE1 = 2 };
enum { COSMO_B200_AA_RESTARTED_MEMORY = 0, COSMO_B200_AA_ROLLING_MEMORY = 1 };
enum { COSMO_B200_AA_NO_REGULARIZER = 0, COSMO_B200_AA_TIKONOV = 1, COSMO_B200_AA_FROBENIUS = 2 };
enum { COSMO_B200_AA_IMMEDIATE = 0, COSMO_B200_AA_ITER = 1, COSMO_B200_AA_ACCURACY = 2 };

/* ws.accelerator's type parameters and ws.activation_reason (settings.jl:96-98,136-138) */
typedef struct {
  int32_t type;          /* COSMO_B200_AA_TYPE2_QR | _TYPE2_NORMAL (Type2{NormalEquations}) | _TYPE1 */
  int32_t memory;        /* COSMO_B200_AA_RESTARTED_MEMORY | _ROLLING_MEMORY (not with TYPE2_QR) */
  int32_t regularizer;   /* COSMO_B200_AA_NO_REGULARIZER | _TIKONOV | _FROBENIUS (not with TYPE2_QR) */
  int32_t activation;    /* COSMO_B200_AA_IMMEDIATE | _ITER (IterActivation) | _ACCURACY (AccuracyActivation) */
  double lambda;         /* regulariser weight (>= 0; 1e-8 is the value the Julia shim passes by default) */
  int64_t start_iter;    /* IterActivation: active once iter >= start_iter */
  double start_accuracy; /* AccuracyActivation: active after the first termination check with r_prim < tol + tol
                            max_norm_prim and r_dual < tol + tol max_norm_dual */
} cosmo_b200_accelerator;

/* KKT plugins (src/linear_solver/kktsolver_indirect.jl:173-189) */
enum {
  COSMO_B200_KKT_CG = 0,             /* CGIndirectKKTSolver      (reduced system, CG)      :3-88   */
  COSMO_B200_KKT_MINRES_REDUCED = 1, /* IndirectReducedKKTSolver(solver_type = :MINRES)    :3-88   */
  COSMO_B200_KKT_MINRES = 2,         /* MINRESIndirectKKTSolver  (full KKT, MINRES)        :90-162 */
  COSMO_B200_KKT_LDL = 3,            /* direct LDL' of the full KKT matrix on the device, the counterpart of
                                        QdldlKKTSolver (kktsolver.jl:285-320); single-GPU */
  COSMO_B200_KKT_LDL_SUPERNODAL = 4  /* supernodal LDL' of the full KKT matrix on the device (dense panels), the
                                        counterpart of the Pardiso plugins' direct solve (kktsolver_pardiso.jl);
                                        same contract as COSMO_B200_KKT_LDL; single-GPU */
};

/* SparseMatrixCSC{T,Int64} as Julia stores it */
typedef struct {
  int64_t nrows, ncols;
  const int64_t* colptr; /* ncols+1 */
  const int64_t* rowval; /* nnz */
  const void* nzval;     /* nnz, dtype */
} cosmo_b200_csc;

/* one entry of CompositeConvexSet.sets (src/projections.jl:20-31) */
typedef struct {
  int32_t type;     /* COSMO_B200_ZERO ... */
  int32_t max_iter; /* Exp/Pow cones: MAX_ITER of the projection (0 = reference default, 100 / 20) */
  int64_t dim;      /* rows of this set (for PSD: length of the vector, N^2 or N(N+1)/2; Exp/Pow: 3) */
  const void* l;    /* Box only: lower/upper bounds, already scaled by E (convexset.jl:863-867) */
  const void* u;
  double alpha;     /* PowerCone / DualPowerCone exponent in (0,1), convexset.jl:631-634 */
  double tol;       /* Exp/Pow cones: EXP_TOL / POW_TOL (0 = reference default 1e-8) */
} cosmo_b200_set;

/* ws.p (ProblemData, types.jl:158-175) + ws.sm (ScaleMatrices, types.jl:130-151) after setup! */
typedef struct {
  int32_t dtype;      /* COSMO_B200_F64 | COSMO_B200_F32 */
  int32_t index_base; /* 1 = Julia, 0 = C */
  int32_t device;     /* CUDA device ordinal */
  int32_t flags;      /* COSMO_B200_PROBLEM_* */
  int64_t m, n;
  cosmo_b200_csc P; /* n x n, both triangles stored */
  cosmo_b200_csc A; /* m x n, model form A x + s = b */
  const void* q;    /* n */
  const void* b;    /* m */
  int64_t n_sets;
  const cosmo_b200_set* sets;
  /* diagonal scalings (NULL => identity).  With flags & COSMO_B200_PROBLEM_EQUILIBRATE and settings.scaling != 0 they
     must be NULL: (P, q, A, b) and the Box bounds are UNSCALED and the engine equilibrates them on the device
     (scale_ruiz!, scaling.jl:21-116); the host then reads D, E, c back with cosmo_b200_get_scaling for
     scale_variables! / reverse_scaling!. */
  const void* D;
  const void* Dinv;
  const void* E;
  const void* Einv;
  double c; /* cost scaling ws.sm.c[] (1.0 when unscaled) */
} cosmo_b200_problem;

/* COSMO.Settings (src/settings.jl:61-155), the fields the loop reads */
typedef struct {
  double rho, sigma, alpha;
  double eps_abs, eps_rel, eps_prim_inf, eps_dual_inf;
  int64_t max_iter;
  int32_t check_termination, check_infeasibility;
  int32_t scaling; /* != 0: residuals are unscaled with Einv / cinv*Dinv (residuals.jl:43-49) */
  int32_t adaptive_rho;
  int32_t adaptive_rho_interval; /* 0 = automatic: chosen once (time in the loop) > adaptive_rho_fraction * setup_time,
                                    rounded to a multiple of check_termination (solver.jl:244-256) */
  int32_t kkt_solver;            /* COSMO_B200_KKT_* */
  double adaptive_rho_tolerance;
  int64_t adaptive_rho_max_adaptions;
  double RHO_MIN, RHO_MAX, RHO_TOL, RHO_EQ_OVER_RHO_INEQ, COSMO_INFTY, MIN_SCALING;
  double time_limit;
  double tol_constant, tol_exponent; /* kktsolver_indirect.jl:21,168-170 */
  int32_t verbose;                   /* bit 0: settings.verbose (iteration log), bit 1: settings.verbose_timing */
  int32_t psd_max_sweeps;            /* Jacobi eigensolver sweep cap (engine-specific) */
  /* accelerator (settings.jl:96-98,136-138; accelerator_interface.jl:58-114) */
  int32_t accelerator;         /* COSMO_B200_ACC_EMPTY | COSMO_B200_ACC_ANDERSON (Type2{QRDecomp}, RestartedMemory,
                                  NoRegularizer, ImmediateActivation unless cosmo_b200_set_accelerator chose another) */
  int32_t accelerator_mem;     /* history length `mem` (reference default 15) */
  int32_t accelerator_min_mem; /* columns needed before a candidate is formed (package default 3) */
  int32_t safeguard;           /* settings.safeguard */
  double safeguard_tol;        /* settings.safeguard_tol (2.0) */
  /* ABI 3 */
  double adaptive_rho_fraction; /* settings.adaptive_rho_fraction (0.4), used by the automatic interval rule */
  double setup_time;            /* seconds the host spent in setup! (ws.times.setup_time: scaling, decomposition, the creation
                                   of this engine); 0: the engine uses its own creation time.  Feeds the automatic rho
                                   interval and the time limit, which the reference measures from before setup!
                                   (solver.jl:119,349) */
  double MAX_SCALING;           /* settings.MAX_SCALING (1e4), read by the device equilibration */
  /* ABI 4 */
  double obj_true;              /* settings.obj_true (NaN = off): has_converged additionally requires
                                   |obj_true - cost| <= obj_true_tol at a termination check (residuals.jl:127-140) */
  double obj_true_tol;          /* settings.obj_true_tol (1e-3) */
} cosmo_b200_settings;

/* COSMO.Result / ResultInfo / ResultTimes (types.jl:26-41, 65-71, 93-112) */
typedef struct {
  /* caller-allocated outputs in the SCALED coordinates the loop works in
     (ws.vars.x = view(w_prev,1:n), ws.vars.s.data, ws.vars.mu at solver.jl:167);
     reverse_scaling! stays in host code. Any of them may be NULL. */
  void* x;  /* n */
  void* s;  /* m */
  void* mu; /* m  (y = -mu) */
  double obj_val;
  int64_t iter;
  int64_t safeguarding_iter;
  int32_t status;
  int32_t _pad;
  double r_prim, r_dual, max_norm_prim, max_norm_dual;
  double rho; /* final scalar rho (ws.rho) */
  double* rho_updates;      /* optional caller buffer for ws.rho_updates */
  int64_t rho_updates_cap;
  int64_t n_rho_updates;
  /* times in seconds (ResultTimes, types.jl:26-41).  proj_time = device time of admm_z! (solver.jl:15,152; here fused
     with the right-hand side of admm_x!), kkt_time = device time of the KKT solves incl. the fused ADMM tail: CUDA
     events on the engine stream, filled when settings.verbose bit 1 is set or the problem is not latency-bound
     (n + m >= 20000 or a large PSD cone), 0 otherwise; res_time = host time inside the termination checks. */
  double solver_time, setup_time, iter_time, proj_time, kkt_time, res_time;
  double iter_time_device; /* the loop timed with CUDA events on the engine stream */
  /* statistics */
  int64_t kkt_inner_iterations; /* CG / MINRES iterations summed over the solve */
  int64_t kkt_multiplications;  /* reduced / full operator applications (S.multiplications) */
  int64_t kernel_launches;      /* engine kernels launched inside the loop */
} cosmo_b200_result;

/* ---- lifecycle ---------------------------------------------------------- */
int cosmo_b200_abi_version(void);
/* COSMO.Settings{T}() defaults (settings.jl:101-139) with kkt_solver = CG and accelerator = COSMO_B200_ACC_EMPTY
   (the reference default is the Anderson accelerator, settings.jl:136-138: set accelerator = COSMO_B200_ACC_ANDERSON;
   the Julia shim of INTEGRATION.md copies it from ws.accelerator) */
int cosmo_b200_default_settings(cosmo_b200_settings* out);
/* _make_kkt_solver! + Variables{T}(m,n,C) + classify_constraints! + set_rho_vec!
   (setup.jl:1-7,75-85; types.jl:263-279; parameters.jl:3-13): uploads the problem. */
int cosmo_b200_create(cosmo_b200_handle** out, const cosmo_b200_problem* prob, const cosmo_b200_settings* settings);
/* free_memory!(ws) (solver.jl:205-208) */
void cosmo_b200_destroy(cosmo_b200_handle* h);
/* last error message of a handle (or of the failed create when h == NULL) */
const char* cosmo_b200_last_error(const cosmo_b200_handle* h);

/* ---- model updates ------------------------------------------------------ */
int cosmo_b200_update_settings(cosmo_b200_handle* h, const cosmo_b200_settings* settings);
/* warm_start_primal!/slack!/dual! (interface.jl:117-179), already scaled; NULL = leave unchanged */
int cosmo_b200_warm_start(cosmo_b200_handle* h, const void* x, const void* s, const void* mu);
/* update!(model, q=, b=) (interface.jl:187-211), already scaled; NULL = leave unchanged */
int cosmo_b200_update_qb(cosmo_b200_handle* h, const void* q, const void* b);
/* New values of P and A on the sparsity pattern given at create, an engine extension: the closest reference entry point
   is update!(model, q=, b=) (interface.jl:187-211), which takes only q and b.  Px and Ax are the nzval arrays in the
   CSC order of create (element type T, nnzP / nnzA entries, which must equal create's: otherwise
   COSMO_B200_ERR_INVALID and nothing changes); q and b as for cosmo_b200_update_qb; NULL = leave unchanged.  Afterwards
   the handle is bit for bit in the state cosmo_b200_create with the new data and the handle's current settings leaves:
   the same scaling, rho vector (rho_updates = [settings.rho]), zero iterates and CG warm start, KKT call counter 1,
   cleared accelerator history and PSD warm starts, and under COSMO_B200_KKT_LDL a fresh factor (a non-convex P:
   COSMO_B200_ERR_INVALID "Objective function is not convex.").  Warm-start it as a new engine.  Not reset, because
   they describe the engine's history rather than its state: the setup time a later solve reports is the duration of
   this call (and so is the figure the automatic adaptive_rho_interval rule reads when settings.setup_time is 0), and
   the statistics counters (factorisations, kernel launches) keep counting.  The first call also derives the value
   maps from the resident pattern and keeps them on the device (a one-off cost about that of the slab placement).
   An engine created with COSMO_B200_PROBLEM_EQUILIBRATE (and scaling != 0) re-runs Ruiz from identity on the unscaled
   data, so it needs all four of Px, Ax, q and b, unscaled (COSMO_B200_ERR_INVALID otherwise); its Box bounds are the
   unscaled ones given at create.  With caller-supplied D, E the values are taken as given, like create does.  A
   decomposition map (cosmo_b200_set_decomposition) stays; reverse_decomposition needs a solve first.  After
   cosmo_b200_comm_init with nranks > 1: COSMO_B200_ERR_UNSUPPORTED. */
int cosmo_b200_update_matrices(cosmo_b200_handle* h, const void* Px, int64_t nnzP, const void* Ax, int64_t nnzA,
                               const void* q, const void* b);
/* update_rho!(kkt_solver, rho_vec) (kktsolver_indirect.jl:164-166): overrides the row penalties */
int cosmo_b200_update_rho(cosmo_b200_handle* h, const void* rho_vec, double rho);
/* empty_model!-like reset of iterates, rho, CG warm start and call counter */
int cosmo_b200_reset(cosmo_b200_handle* h);
/* _make_accelerator! (setup.jl:10-14) for settings.accelerator = AndersonAccelerator{T, type, memory, regularizer} with
   activation_reason (accelerator_interface.jl:1-48); read when settings.accelerator == COSMO_B200_ACC_ANDERSON and kept
   across update_settings.  NULL restores the default (Type2{QRDecomp}, RestartedMemory, NoRegularizer,
   ImmediateActivation).  TYPE2_QR with rolling memory or a regulariser: COSMO_B200_ERR_UNSUPPORTED; lambda < 0 or an
   unknown enum: COSMO_B200_ERR_INVALID. */
int cosmo_b200_set_accelerator(cosmo_b200_handle* h, const cosmo_b200_accelerator* acc);
/* what the reference logs in accelerator.acceleration_status (accelerator_interface.jl:95-111, solver.jl:272-275)
   for the last solve: out = {accepted candidates (num_accelerated_steps), safeguard declines, rejected solves
   (singular, non-finite or |eta| > 1e4), restarts after a rho adaptation, memory restarts, iteration at which the
   accelerator became active (0: never)} */
int cosmo_b200_accelerator_stats(cosmo_b200_handle* h, int64_t out[6]);

/* ---- the hot loop (solver.jl:125-167) ------------------------------------ */
int cosmo_b200_solve(cosmo_b200_handle* h, cosmo_b200_result* out);

/* ---- plugin-granularity entry points (also the parity-test hooks) -------- */
/* project!(s, C): s_out = Pi_K(w_s) (convexset.jl:885-891) */
int cosmo_b200_project(cosmo_b200_handle* h, const void* w_s, void* s_out);
/* solve!(kkt_solver, sol, rhs): rhs, sol in R^{n+m} (kktsolver_indirect.jl:36-88,123-162) */
int cosmo_b200_kkt_solve(cosmo_b200_handle* h, const void* rhs, void* sol, int64_t* inner_iterations);
/* calculate_residuals! + max_res_component_norm + calculate_cost! (residuals.jl:30-96,143-147)
   for given (x, s, mu); out = {r_prim, r_dual, max_norm_prim, max_norm_dual, cost} */
int cosmo_b200_residuals(cosmo_b200_handle* h, const void* x, const void* s, const void* mu,
                         int32_t ignore_scaling, double out[5]);
/* y = M x for M in {0: A, 1: A', 2: P} (the mul! calls at kktsolver_indirect.jl:53-63); 3: y = A' x2 + P x1 + sigma x1
   for x = [x1; x2] in R^{n+m}, y in R^n (the second half of the reduced KKT operator, kktsolver_indirect.jl:61-63) */
int cosmo_b200_spmv(cosmo_b200_handle* h, int32_t which, const void* x, void* y);
/* time `reps` back-to-back launches of one SpMV kernel with CUDA events; returns ms per launch */
int cosmo_b200_spmv_bench(cosmo_b200_handle* h, int32_t which, int32_t reps, double* ms_per_launch,
                          double* algorithmic_bytes);
/* read back the current per-row penalty vector (ws.rho_vec) */
int cosmo_b200_get_rho_vec(cosmo_b200_handle* h, void* rho_vec);
/* ws.sm.D.diag (n), ws.sm.E.diag (m), ws.sm.c[] as used by the engine: what the host passed at create, or what the
   device equilibration computed (scaling.jl:21-116); all ones when settings.scaling == 0.  NULL pointers are skipped. */
int cosmo_b200_get_scaling(cosmo_b200_handle* h, void* D, void* E, double* c);
/* read back the operator variable w = [w_x; w_s] (n+m) */
int cosmo_b200_get_w(cosmo_b200_handle* h, void* w);
/* is_primal_infeasible! (which = 0, delta = delta_y: this rank's m rows) or is_dual_infeasible! (which = 1,
   delta = delta_x: n) (infeasibility.jl:1-68) on the given delta, with the engine's D, E, c, b, q and eps_*_inf.
   out = {verdict (1: infeasible), last gate reached (1: norm, 2: A'dy resp. q'dx, 3: P dx (dual only), 4: cone tests),
          |E dy|_inf resp. |D dx|_inf, |Dinv A'dy|_inf resp. q'dx, dy'b of the normalized -dy resp. |Dinv P dx|_inf,
          Box support sum (primal), failed certificate families (bit 0: Zero/Nonnegatives/Box rows, 1: SOC, 2: PSD,
          3: Exp/Pow and their duals, 4: custom cones), PSD cones whose eigensolver missed psd_max_sweeps (counted as not certified)};
   a value that the test did not reach is NaN.  Uses the engine's dx / dy scratch vectors, as cosmo_b200_residuals
   does: call it between solves, not inside one.  With several ranks every rank calls it. */
int cosmo_b200_infeasibility_test(cosmo_b200_handle* h, int32_t which, const void* delta, double out[8]);
/* lam[k] = largest eigenvalue of mat(v[rows of the k-th PSD cone]) for every PSD cone of this rank, in set order, as
   the infeasibility certificate computes it: a PsdCone read from its upper triangle (is_pos_def!, convexset.jl:324-336),
   the same prescaling and eigensolver path (shared-memory Jacobi up to N = 96, block Jacobi beyond); +inf where the
   eigensolver did not converge within psd_max_sweeps.  v has the m rows of this rank. */
int cosmo_b200_psd_lambda_max(cosmo_b200_handle* h, const void* v, double* lam);

/* ---- direct LDL' KKT plugin (kkt_solver = COSMO_B200_KKT_LDL) ------------- */
/* K = [P + sigma I, A'; A, -diag(1/rho)] (N = n + m) is ordered by minimum degree and analysed on the host at create;
   the factorisation (at create, then lazily before the first KKT solve after rho_vec or sigma changed: adapt_rho,
   update_rho, reset, update_settings) and both triangular solves run on the device.  A factor that does not fit in
   device memory fails the create with COSMO_B200_ERR_ALLOC; a factorisation with fewer or more than n positive pivots
   fails with COSMO_B200_ERR_INVALID ("Objective function is not convex."), a zero or non-finite pivot with
   COSMO_B200_ERR_NUMERICAL.  cosmo_b200_kkt_solve reports 0 inner iterations.
   out = {N, nnz of the upper triangle of K, nnz of L (strictly lower), levels of the elimination tree, kernel launches
   per solve, factorisations so far, device seconds of the last factorisation, host seconds of the symbolic analysis};
   all 0 on a handle that never used the plugin. */
int cosmo_b200_ldl_stats(cosmo_b200_handle* h, double out[8]);
/* The symbolic analysis alone, on the host (no GPU needed).  Every array has N = n + m entries, in pivot order k:
   perm[k] = original index of pivot k (x: 0..n-1, y: n..N-1), parent[k] = parent of k in the elimination tree of the
   permuted K (-1: root), colcount[k] = entries of column k of L below the diagonal, level[k] = 0 for a leaf, else
   1 + the largest level of its children.  Errors through cosmo_b200_last_error(NULL). */
int cosmo_b200_ldl_symbolic(const cosmo_b200_problem* prob, int64_t* perm, int64_t* parent, int64_t* colcount, int64_t* level);

/* ---- supernodal LDL' KKT plugin (kkt_solver = COSMO_B200_KKT_LDL_SUPERNODAL) ---- */
/* The contract of COSMO_B200_KKT_LDL (factor at create, lazy refactorisation, the same errors, single-GPU), on the
   ordering of COSMO_B200_KKT_LDL renumbered by a postorder of the elimination tree: the factor is that plugin's up to
   a symmetric permutation.  Columns are grouped into supernodes (dense panels, relaxed amalgamation); small ones
   factor in one CTA each, large ones tiled across CTAs.  cosmo_b200_ldl_stats answers for this plugin too (nnz_L:
   stored entries, explicit zeros included; levels: supernodal levels).  out[8] = {supernodes, maximum width, explicit
   zeros, supernodal levels, supernodes on the small path, supernodes on the tiled path, kernel nodes per solve,
   flops of the descendant updates of one factorisation}; 0 where the handle never used the plugin. */
int cosmo_b200_ldl_sn_stats(cosmo_b200_handle* h, int64_t out[8]);
/* The supernodal symbolic analysis alone, on the host (no GPU needed).  perm (N = n + m entries): perm[k] = original
   index of pivot k in the postordered numbering; snode_ptr (N + 1 entries, the first supernodes + 1 used): columns of
   supernode s are [snode_ptr[s], snode_ptr[s+1]); snode_parent (N entries, the first supernodes used): the parent
   supernode, -1 for a root.  stats = {supernodes, maximum width, stored entries, explicit zeros, supernodal levels,
   simplicial levels, nnz(L), flops of the descendant updates}.  Errors through cosmo_b200_last_error(NULL). */
int cosmo_b200_ldl_sn_symbolic(const cosmo_b200_problem* prob, int64_t* perm, int64_t* snode_ptr, int64_t* snode_parent,
                               int64_t stats[8]);

/* ---- reverse of a chordal decomposition (reverse_decomposition! + psd_completion!,
        chordal_decomposition.jl:129-311) ------------------------------------ */
/* psd_complete! of one decomposed PsdConeTriangle: the clique tree in traversal order (parents first, children in
   order).  Vertices are renumbered in the order the traversal first meets them (new_of), so the vertices visited before
   step t are the leading block 0..lo-1.  Step t = steps[6t .. 6t+5] = {lo, hi, a0, a1, k0, k1}: its residual nu is the
   new indices lo..hi-1 (lo = hi of the step before, 0 for the first), its separator alpha = idx[a0..a1-1] and the other
   clique members below lo are idx[k0..k1-1] (a1 == k0).  The step sets, for every r < lo outside the clique,
       W[r, nu] = W[nu, r]' = W[r, alpha] Z,   W[alpha, alpha] Z = W[alpha, nu],
   and leaves every entry inside the clique as it is. */
typedef struct {
  int64_t N;               /* side of the matrix */
  int64_t row_offset;      /* first row of the cone in the original problem (cosmo_b200_psd_complete ignores it) */
  int64_t dim;             /* rows of the cone: N(N+1)/2 (PsdConeTriangle); a square PsdCone (N*N) only in the map of
                              cosmo_b200_set_decomposition_noncompact */
  const int64_t* new_of;   /* N: traversal position of every vertex, a permutation of 0..N-1 */
  int64_t n_steps;
  const int64_t* steps;    /* 6 * n_steps */
  int64_t n_idx;
  const int64_t* idx;      /* new indices, each below the lo of its step */
} cosmo_b200_completion;

/* The map from the decomposed problem (the handle's n, m) back to the original one (n_orig, m_orig), 0-based:
   x = the first n_orig entries; plain rows are copied; original row row[i] of a decomposed cone gets
   s = 0.0 + s'[s_src[s_ptr[i]]] + ... + s'[s_src[s_ptr[i+1]-1]] in that order and mu = mu'[mu_src[i]], which must be the
   last entry of that list (the clique the host loop writes last); rows in no clique are 0. */
typedef struct {
  int64_t n_orig, m_orig;
  int64_t n, m;            /* must equal the handle's n, m */
  int64_t n_plain;
  const int64_t* plain;    /* 3 * n_plain: old_start, new_start, dim */
  int64_t n_rows;
  const int64_t* row;      /* n_rows original rows, strictly increasing, none inside a plain block */
  const int64_t* s_ptr;    /* n_rows + 1, s_ptr[0] = 0, every list non-empty */
  const int64_t* s_src;    /* s_ptr[n_rows] rows of the decomposed problem */
  const int64_t* mu_src;   /* n_rows */
  int64_t n_cones;         /* decomposed cones (PsdConeTriangle; PsdCone too in the traditional map) */
  const cosmo_b200_completion* cones;
} cosmo_b200_decomposition;

/* Copies the map to the device (NULL clears it).  Every index is checked: out-of-range or inconsistent maps return
   COSMO_B200_ERR_INVALID; a cone with the square PsdCone layout (dim = N*N) and a sharded handle (nranks > 1) return
   COSMO_B200_ERR_UNSUPPORTED. */
int cosmo_b200_set_decomposition(cosmo_b200_handle* h, const cosmo_b200_decomposition* d);
/* The map of the traditional transformation (compact_transformation = false: A' = [A H; 0 -I], b' = [b; 0], s = H s'
   and mu = H mu' divided by each row's overlap count, chordal_decomposition.jl:136-168), in the same struct with two
   differences: mu_src must be NULL, and original row row[i] gets mu = (0.0 + mu'[s_src[s_ptr[i]]] + ... +
   mu'[s_src[s_ptr[i+1]-1]]) / (s_ptr[i+1] - s_ptr[i]); a cone may have the square PsdCone layout (dim = N*N, column-major,
   completed from its upper triangle and written back to all N*N entries).  Plain blocks point into the rows below m_orig
   (m_orig + the column of H), and their rows are 0.0 + the row, as H s' gives them.  The same checks and errors as
   cosmo_b200_set_decomposition; setting either map replaces the other, and cosmo_b200_reverse_decomposition runs the one
   that is set. */
int cosmo_b200_set_decomposition_noncompact(cosmo_b200_handle* h, const cosmo_b200_decomposition* d);
/* reverse_scaling! + reverse_decomposition! (+ psd_completion! when complete_dual != 0) of the x, s, mu that the last
   cosmo_b200_solve left on the device: x = D x', s = s' / E, mu = (E mu') / c widened to fp64, then the map.  Writes x
   (n_orig), s and mu (m_orig) in fp64 into caller buffers; NULL skips a buffer (a NULL mu skips the completion).
   stats (may be NULL) = {cones completed, separator solves that fell back to the pseudo-inverse, bytes of the dense
   workspace, device microseconds of the kernels (CUDA events; the copies to the caller's buffers excluded)}.  The dense N x N fp64 workspace of the largest cone is allocated on
   first use and kept; if it does not fit: COSMO_B200_ERR_ALLOC.  No map, or no solve since create / reset / warm_start:
   COSMO_B200_ERR_INVALID. */
int cosmo_b200_reverse_decomposition(cosmo_b200_handle* h, int32_t complete_dual, void* x, void* s, void* mu,
                                     int64_t stats[4]);
/* The completion alone on a dense column-major N x N fp64 matrix Y (host memory, read from its upper triangle,
   overwritten with the symmetric completion); the parity hook of the kernels.  No handle: uses the current device.
   stats as above.  Errors through cosmo_b200_last_error(NULL). */
int cosmo_b200_psd_complete(int64_t N, const cosmo_b200_completion* schedule, double* Y, int64_t stats[4]);

/* ---- values of the original problem onto a chordally decomposed one ------ */
/* The way forward through the decomposition for values, an engine extension: the reference refuses to update a model
   that has been chordally decomposed at all (update!, interface.jl:192,204), so every new q, b, P or A pays the
   decomposition, the augmentation and the setup again.  None of them depends on the values: the decomposition is a
   function of the sparsity pattern, and the decomposed problem (the handle's n, m, nnzA) takes its values from the
   original one (n_orig, m_orig, nnzA_orig), 0-based, as
     A' in CSC order with sorted rows: entry k = Ax[a_src[k]], or the constant +1.0 for a_src[k] = -1, -1.0 for -2
        (the overlap columns); every entry of A is used exactly once;
     b'[i] = b[b_src[i]] for a plain row, 0.0 for b_src[i] = -1, and for a row of a clique block b_src[i] = -2 - r:
        b[r], where a zero of either sign arrives as +0.0 (the decomposition writes only the nonzero values there);
     q' = [q; 0];   P' = blockdiag(P, 0): P's values in P's order.
   b_uncovered[i] != 0 marks an original row of a decomposed cone that lies in no clique: b must be zero there, a
   nonzero value changes the aggregate sparsity pattern and with it the decomposition.  Every other original row is
   the source of exactly one row of b'. */
typedef struct {
  int64_t n_orig, m_orig;
  int64_t n, m;              /* must equal the handle's n, m */
  int64_t nnzA_orig;
  int64_t nnzA;              /* must equal the nnz of the handle's A */
  const int64_t* a_src;      /* nnzA */
  const int64_t* b_src;      /* m */
  const uint8_t* b_uncovered; /* m_orig */
} cosmo_b200_forward_map;
/* Checks every index and copies the map to the device (as int32 where every index fits), where it stays; NULL clears
   it.  A size that is not the handle's, an index out of range, an entry of A used twice or not at all, a row of b used
   twice, or a row that is neither used nor marked uncovered (or both): COSMO_B200_ERR_INVALID.  A sharded handle
   (nranks > 1): COSMO_B200_ERR_UNSUPPORTED. */
int cosmo_b200_set_forward_map(cosmo_b200_handle* h, const cosmo_b200_forward_map* f);
/* cosmo_b200_update_matrices with Px (nnzP entries), Ax (nnzA_orig entries), q (n_orig) and b (m_orig) in the
   coordinates and the CSC order of the ORIGINAL problem: they are staged on the device, gathered through the forward
   map and enter the value path of cosmo_b200_update_matrices.  The same rules hold: NULL = leave unchanged, an
   equilibrating engine needs all four, unscaled, and the handle ends up bit for bit in the state cosmo_b200_create
   with the decomposed new data leaves; a decomposition map stays, reverse_decomposition needs a solve first.  No
   forward map, nnzP or nnzA_orig that differ from the pattern, or a b that is nonzero on an uncovered row (counted on
   the device before the first write): COSMO_B200_ERR_INVALID, and nothing has changed. */
int cosmo_b200_update_matrices_original(cosmo_b200_handle* h, const void* Px, int64_t nnzP, const void* Ax,
                                        int64_t nnzA_orig, const void* q, const void* b);

/* ---- caller arrays in device memory --------------------------------------- */
/* Host or device: every array of cosmo_b200_warm_start, _update_qb, _update_matrices and _update_matrices_original, the
   x, s, mu buffers of cosmo_b200_result, the outputs of cosmo_b200_reverse_decomposition and the arrays of the entry
   points below may point to host memory, to device memory on the handle's device or to managed memory (copies use
   cudaMemcpyDefault, so a host pointer takes the path it always took).  A pointer in device memory of another device:
   COSMO_B200_ERR_INVALID, and nothing is written.  "Caller device memory" means device or managed memory: when a call
   reads it, the engine stream first waits on an event recorded on the caller stream; when a call writes it, the caller
   stream waits on the engine stream before the call returns (the call is synchronous as before; no cudaDeviceSynchronize).  The entry points below refuse a sharded handle
   (nranks > 1) with COSMO_B200_ERR_UNSUPPORTED. */
/* The stream that caller device memory is ordered on (NULL: the legacy default stream, which is also the initial one;
   cudaStreamPerThread is accepted).  Kept until the next call. */
int cosmo_b200_set_caller_stream(cosmo_b200_handle* h, void* stream);
/* update!(model, q=, b=) in the model's own coordinates, unscaled, in fp64 (NULL = unchanged): with a forward map
   (cosmo_b200_set_forward_map) q has n_orig and b m_orig entries and become q' = [q; 0], b' = b[b_src] as there; without
   one they have n and m.  The device then forms (D q') c and E b' in fp64, rounded once to the element type, and changes
   the state as cosmo_b200_update_qb does (rho classes recomputed from a new b; iterates and rho kept).  A b that is
   nonzero on an uncovered row of the forward map: COSMO_B200_ERR_INVALID, and nothing has changed.  The handle keeps the
   fp64 q and b it was given on the device (8 (n_orig + m_orig) bytes, allocated on first use) for
   cosmo_b200_original_qb. */
int cosmo_b200_update_qb_original(cosmo_b200_handle* h, const double* q, const double* b);
/* Reads back the q and b last given to cosmo_b200_update_qb_original (NULL skips one); one that was never given, or was
   given before the forward map changed its sizes: COSMO_B200_ERR_INVALID. */
int cosmo_b200_original_qb(cosmo_b200_handle* h, double* q, double* b);
/* The last solve's solution in the original, unscaled coordinates, in fp64: x (n_orig), y = -mu and s (m_orig); any
   pointer may be NULL.  With a decomposition map this is cosmo_b200_reverse_decomposition's arithmetic (the completion
   when complete_dual != 0); without one it is reverse_scaling!: x = D x', s = s' / E, mu = (E mu') / c after widening,
   with n_orig = n and m_orig = m.  No solve since create / reset / warm_start / rescale_iterates: COSMO_B200_ERR_INVALID. */
int cosmo_b200_solution(cosmo_b200_handle* h, int32_t complete_dual, double* x, double* y, double* s);
/* reverse_scaling! followed by scale_variables! on the resident iterates, in fp64 and then rounded to the element type:
   x' <- (D x') / D, s' <- E (s' / E), mu' <- (((E mu') / c) / E) c: the round trip the host applies between two solves
   when it hands the unscaled solution back as the next warm start.  Like cosmo_b200_warm_start, it ends the solution
   that cosmo_b200_solution and cosmo_b200_reverse_decomposition read. */
int cosmo_b200_rescale_iterates(cosmo_b200_handle* h);

/* ---- multi-GPU (one process per GPU; rows sharded, n-vectors replicated) -- */
/* 128-byte ncclUniqueId created on rank 0 and broadcast by the host plumbing */
int cosmo_b200_comm_unique_id(void* id128);
int cosmo_b200_comm_init(cosmo_b200_handle* h, int32_t nranks, int32_t rank, const void* id128);
/* Peer-memory exchange over NVLink/NVSwitch for the reduced-KKT operator partials (optional; replaces
   the per-application NCCL allreduce by a one-shot sum fused into the consumer kernels).
   export: 128 bytes (two CUDA IPC handles) per rank; the host all-gathers them in rank order;
   attach: maps the peers' buffers.  All ranks must be on one NVLink-connected node. */
int cosmo_b200_comm_p2p_export(cosmo_b200_handle* h, void* blob128);
int cosmo_b200_comm_p2p_attach(cosmo_b200_handle* h, const void* blobs, int32_t nranks);

/* ---- custom cones --------------------------------------------------------- */
/* Checks the descriptor and compiles the type for dtype (COSMO_B200_F64 | _F32) into the process-wide cache, or finds it
   there; no device is needed.  A bad descriptor (name not an identifier, unknown granularity or flag, reserved != 0,
   n_params < 0, no source) or a compile error: COSMO_B200_ERR_INVALID, with the NVRTC log (the user's lines as
   `name`(line)) in cosmo_b200_last_error(NULL) and, truncated to log_cap bytes with a terminating 0, in `log` when it is
   not NULL.  No libnvrtc.so.12: COSMO_B200_ERR_UNSUPPORTED.  Returns 1 instead of 0 when the call compiled. */
int cosmo_b200_custom_cone_compile(const cosmo_b200_custom_cone* type, int32_t dtype, char* log, int64_t log_cap);
/* out = {custom cone types, custom cones of this handle, compilations its create caused, types its create found in the
   cache} */
int cosmo_b200_custom_cone_stats(cosmo_b200_handle* h, int64_t out[4]);

/* ---- diagnostics ---------------------------------------------------------- */
/* Which path projected the large PSD cones (N > 96) so far: out = {tensor-core projections, tensor-core fallbacks to
   block Jacobi, Newton-Schulz steps of the last one, weighted-residual checks of the last one, 0, 0 (unused, always
   zero), block-Jacobi sweeps of the last eigensolve, int8 slices per operand}. */
int cosmo_b200_psd_stats(cosmo_b200_handle* h, int64_t out[8]);
/* The product kernel of the large-cone PSD projection on its own: C = A B for symmetric, commuting N x N fp64
   matrices (column-major) through `k` int8 slices on wgmma (csrc/tc_gemm.cuh; the reference's counterpart is the
   BLAS-3 part of project!(::PsdCone), convexset.jl:244-260).  `groups` = number of slice-pair groups kept
   (0: the default of `k`); supported (k, groups): (8,10) (8,8) (7,7) (6,8) (4,6); `reserved` must be 0.
   frob2 = {|C|_F^2, |I - C|_F^2} from the fused reductions.
   No handle: uses the current device.  Errors through cosmo_b200_last_error(NULL). */
int cosmo_b200_tc_gemm_test(int32_t N, int32_t k, int32_t groups, int32_t reserved, const double* A, const double* B, double* C,
                            int32_t reps, double* ms_per_product, double* frob2);

#ifdef __cplusplus
}
#endif
#endif /* COSMO_B200_H */
