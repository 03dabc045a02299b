/*
 * cuipm.h -- C ABI of the H100-native batched OCP-QP interior-point solver.
 *
 * This is the drop-in boundary for acados' `qp_solver` plugin slot: everything the reference's
 * `ocp_qp_hpipm()` (acados/ocp_qp/ocp_qp_hpipm.c:314-405) obtains from HPIPM's
 * `d_ocp_qp_ipm_solve()` (external/hpipm/ocp_qp/x_ocp_qp_ipm.c:2684-3120) is obtained through the
 * entry points below instead.  Plain pointers and sizes only: no torch / CUDA types in signatures, so
 * the plugin source that lives inside libacados (acados_b200/plugin/ocp_qp_cuipm.c) stays plain C.
 *
 * Batch model: all QPs of one batch share a SHAPE (horizon, per-stage dimensions, box/soft index maps)
 * and differ in their numerical DATA.  One QP's data is one contiguous "QP record" of doubles; one
 * QP's primal-dual solution is one contiguous "solution record".  Record layouts are described by
 * cuipm_layout (offsets in doubles), computed by cuipm_layout_create().
 *
 * Conventions are HPIPM's (external/hpipm/include/hpipm_d_ocp_qp.h:54-71, ocp_qp/x_ocp_qp.c:1035-1267):
 *   stage k = 0..N, v_k = [u_k; x_k] (nu_k + nx_k), dynamics x_{k+1} = BAt_k' v_k + b_k,
 *   cost 1/2 v'RSQ v + rq'v (+ slacks: 1/2 s'Z s + z's), constraints
 *     lb <= v[idxb] (+ sl) , v[idxb] (- su) <= ub ; lg <= DCt' v (+ sl), DCt' v (- su) <= ug ; sl >= lls, su >= lus
 *   d = [lb, lg, -ub, -ug, lls, lus]  (UPPER BOUNDS STORED NEGATED, x_ocp_qp.c:1228-1267)
 *   lam, t ordered (lb, lg, ub, ug, ls, us); d_mask in {0.0, 1.0} disables single constraints.
 *   idxs_rev[k][i] = slack index softening constraint i (i over nb+ng), or -1.
 */
#ifndef CUIPM_H_
#define CUIPM_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CUIPM_STAT_M 20  /* columns of the per-iteration statistics table (x_ocp_qp_ipm.c:801) */

/* return / status codes: HPIPM's (external/hpipm/include/hpipm_common.h:57-64) */
enum cuipm_status {
    CUIPM_SUCCESS = 0,
    CUIPM_MAX_ITER = 1,
    CUIPM_MIN_STEP = 2,
    CUIPM_NAN_SOL = 3,
    CUIPM_INCONS_EQ = 4
};

/* error codes of the API calls themselves (not solver status) */
enum cuipm_error {
    CUIPM_OK = 0,
    CUIPM_ERR_INVALID = -1,     /* bad argument / unsupported option value */
    CUIPM_ERR_CUDA = -2,        /* CUDA runtime error (message via cuipm_last_error) */
    CUIPM_ERR_NO_DEVICE = -3,   /* no CUDA device: there is NO CPU fallback */
    CUIPM_ERR_TOO_LARGE = -4    /* stage dimensions exceed what the kernel supports: the solver's vectors alone need more shared
                                 * memory than a block may have, or a record needs offsets beyond 32 bits.  (Stage blocks that do not
                                 * fit in shared memory are not refused: they go to a per-QP device scratch buffer.) */
};

/* modes: external/hpipm/include/hpipm_common.h (enum hpipm_mode) */
enum cuipm_mode { CUIPM_SPEED_ABS = 0, CUIPM_SPEED = 1, CUIPM_BALANCE = 2, CUIPM_ROBUST = 3 };

/* Shape shared by all QPs of a batch (mirrors struct d_ocp_qp_dim + idxb/idxs_rev of struct d_ocp_qp). */
typedef struct cuipm_shape {
    int N;                        /* horizon length; stages 0..N */
    const int *nx;                /* [N+1] */
    const int *nu;                /* [N+1] */
    const int *nb;                /* [N+1] box constraints on v=[u;x] */
    const int *ng;                /* [N+1] general constraints */
    const int *ns;                /* [N+1] soft-constraint slack pairs */
    const int *const *idxb;       /* [N+1][nb_k]      index into v_k */
    const int *const *idxs_rev;   /* [N+1][nb_k+ng_k] slack index or -1 (may be NULL if all ns==0) */
} cuipm_shape;

/* Solver options: the subset of struct d_ocp_qp_ipm_arg (hpipm_d_ocp_qp_ipm.h) that the reference's
 * plugin can reach through ocp_qp_hpipm_opts_set (acados/ocp_qp/ocp_qp_hpipm.c:142-183). */
typedef struct cuipm_opts {
    int mode;             /* enum cuipm_mode the defaults were taken from */
    int iter_max;
    int stat_max;         /* rows of the statistics table kept (>= iter_max) */
    double mu0;
    double alpha_min;
    double res_g_max;     /* tol_stat */
    double res_b_max;     /* tol_eq   */
    double res_d_max;     /* tol_ineq */
    double res_m_max;     /* tol_comp */
    double dual_gap_max;
    double reg_prim;
    double lam_min;
    double t_min;
    double tau_min;
    double lam0_min;
    double t0_min;
    int pred_corr;
    int cond_pred_corr;
    int itref_pred_max;
    int itref_corr_max;
    int lq_fact;          /* 0: Cholesky only; 1: Cholesky, LQ when inaccurate; 2: always LQ */
    int warm_start;       /* 0/1 cold (the plugin zeroes ux, ocp_qp_hpipm.c:333-336); 2/3 keep pi,lam,t of `sol` (lam,t clipped) */
    int abs_form;         /* must be 0 (delta formulation) */
    int comp_dual_sol_eq; /* must be 1 */
    int comp_res_exit;    /* must be 1 */
    int split_step;       /* must be 0 */
    int var_init_scheme;  /* 0 or 1 */
    int t_lam_min;        /* 0,1,2 */
    int t0_init;          /* 0,1,2 */
    double m_relax;       /* acados "tau_min": if >0, complementarity target m_i = m_relax (ocp_qp_hpipm.c:338-342) */
} cuipm_opts;

/* Offsets (in doubles) inside one QP record / one solution record.  All sub-arrays start on an even
 * offset (16-byte aligned) and the records are a multiple of 2 doubles long.  Arrays of length N+1
 * are indexed by stage; entries for BAt/b/pi at stage N are unused (no dynamics after the last stage). */
typedef struct cuipm_layout {
    int N;
    /* QP record */
    size_t qp_stride;      /* doubles per QP record */
    size_t *qp_stage;      /* [N+2] start of stage k's sub-record; qp_stage[N+1] == qp_stride */
    size_t *off_BAt;       /* (nu+nx) x nx_next, column-major, ld = nu+nx : [B'; A'] */
    size_t *off_RSQ;       /* (nu+nx) x (nu+nx), column-major, ld = nu+nx, LOWER triangle referenced: [R S'; S Q] */
    size_t *off_DCt;       /* (nu+nx) x ng, column-major : [D'; C'] */
    size_t *off_b;         /* nx_next */
    size_t *off_rq;        /* nu+nx */
    size_t *off_d;         /* 2nb+2ng+2ns : lb, lg, -ub, -ug, lls, lus */
    size_t *off_dmask;     /* 2nb+2ng+2ns */
    size_t *off_Z;         /* 2ns : Zl, Zu (diagonals) */
    size_t *off_z;         /* 2ns : zl, zu */
    /* solution record */
    size_t sol_stride;     /* doubles per solution record */
    size_t *sol_stage;     /* [N+2] */
    size_t *off_ux;        /* nu+nx+2ns : u, x, sl, su */
    size_t *off_pi;        /* nx_next */
    size_t *off_lam;       /* 2nb+2ng+2ns */
    size_t *off_t;         /* 2nb+2ng+2ns */
} cuipm_layout;

/* Per-QP result summary written next to each solution record. */
typedef struct cuipm_info {
    int status;            /* enum cuipm_status */
    int iter;              /* IPM iterations taken */
    double res_max[4];     /* inf-norms: stationarity, equality, inequality, complementarity */
    double mu;             /* duality measure at exit */
    double obj;            /* objective value at exit */
    double dual_gap;
    int lq_count;          /* iterations factorised with the LQ refactorisation (stat column 13; x_ocp_qp_ipm.c:2299-2346) */
    int reserved;
} cuipm_info;

typedef struct cuipm_solver cuipm_solver;  /* opaque: device buffers, stream, compiled-shape tables */

/* ---- options ------------------------------------------------------------------------------------ */
/* HPIPM mode defaults (x_ocp_qp_ipm.c:69-260). */
void cuipm_opts_set_default(cuipm_opts *opts, int mode);
/* HPIPM mode defaults + the overrides acados applies after every mode switch (ocp_qp_hpipm.c:101-129):
 * this is what PARTIAL_CONDENSING_HPIPM runs with out of the box. */
void cuipm_opts_set_default_acados(cuipm_opts *opts, int mode);
/* String-keyed setter with the reference's field names (ocp_qp_hpipm.c:142-183; x_ocp_qp_ipm.c:264-384):
 * iter_max, tol_stat, tol_eq, tol_ineq, tol_comp, tol_dual_gap, mu0, alpha_min, reg_prim, warm_start,
 * pred_corr, cond_pred_corr, split_step, t_lam_min, t0_init, var_init_scheme, lam_min, t_min, tau_min,
 * lam0_min, t0_min, ric_alg, comp_res_exit, comp_dual_sol_eq, hpipm_mode (value = const char*).
 * Returns CUIPM_ERR_INVALID for an unknown field (the plugin turns that into printf+exit(1) like the reference). */
int cuipm_opts_set(cuipm_opts *opts, const char *field, const void *value);
int cuipm_opts_get(const cuipm_opts *opts, const char *field, void *value);

/* ---- layout ------------------------------------------------------------------------------------- */
cuipm_layout *cuipm_layout_create(const cuipm_shape *shape);
void cuipm_layout_destroy(cuipm_layout *layout);

/* ---- solver lifetime ---------------------------------------------------------------------------- */
/* Creates a solver bound to CUDA device `device` able to hold up to `max_batch` QPs of `shape`.
 * Returns NULL on failure (cuipm_last_error() tells why).  There is no CPU fallback. */
cuipm_solver *cuipm_create(const cuipm_shape *shape, int max_batch, int device);
void cuipm_destroy(cuipm_solver *s);
const cuipm_layout *cuipm_get_layout(const cuipm_solver *s);
const char *cuipm_last_error(void);

/* ---- solve -------------------------------------------------------------------------------------- */
/* Host-buffer entry (what the acados plugin / batch function calls):
 *   qp    : nbatch QP records, host memory (pinned memory makes the copies asynchronous)
 *   sol   : nbatch solution records, host memory.  With opts->warm_start >= 1 it is also an INPUT.
 *   info  : nbatch summaries
 *   stat  : optional nbatch x (stat_max+1) x CUIPM_STAT_M table (row-per-iteration, HPIPM's column meaning); may be NULL
 * Copies H2D, solves on the device, copies D2H, synchronises.  Returns enum cuipm_error. */
int cuipm_solve_host(cuipm_solver *s, int nbatch, const double *qp, double *sol, cuipm_info *info,
                     double *stat, const cuipm_opts *opts);
/* The same, split: cuipm_solve_host_async enqueues the copies and the kernels on the solver's own streams and returns,
 * cuipm_wait blocks until that work has completed (the host buffers must stay valid until then; pinned memory is needed
 * for the copies to overlap anything).  Two solver objects used alternately overlap the transfers of one batch with
 * the solve of the previous one; the reference has no counterpart (its batch solve is a blocking OpenMP loop,
 * c_templates_tera/acados_solver.in.c:3223-3243). */
int cuipm_solve_host_async(cuipm_solver *s, int nbatch, const double *qp, double *sol, cuipm_info *info, double *stat,
                           const cuipm_opts *opts);
int cuipm_wait(cuipm_solver *s);
/* Chunk-granular form: records lo .. lo+n-1 of the batch whose (page-locked) host buffers START at qp / sol / info are copied in,
 * solved and copied out on internal stream `slot` (0..7; a slot must have been waited for before it is used again); returns
 * once the work is enqueued.  cuipm_wait_chunk blocks until the chunk of that slot is back in the host buffers.  For callers
 * that produce their records chunk by chunk: the plugin's batched entry unpacks the ocp_qp_in structs of chunk c+1 (the loop of
 * d_ocp_qp getters of acados/ocp_qp/ocp_qp_hpipm.c:281-330 has no counterpart: HPIPM reads the structs in place) while the
 * device copies and solves chunk c. */
int cuipm_solve_host_chunk(cuipm_solver *s, int slot, int lo, int n, const double *qp, double *sol, cuipm_info *info,
                           const cuipm_opts *opts);
int cuipm_wait_chunk(cuipm_solver *s, int slot);

/* Device-buffer entry: all pointers are device pointers on the solver's device; asynchronous on the
 * solver's stream unless `sync` != 0. */
int cuipm_solve_device(cuipm_solver *s, int nbatch, const double *d_qp, double *d_sol, cuipm_info *d_info,
                       double *d_stat, const cuipm_opts *opts, int sync);

/* Page-locked host memory for the record buffers handed to cuipm_solve_host[_async]: with pageable memory the "asynchronous"
 * copies are staged synchronously by the driver.  The acados plugin keeps its batch staging buffers here (no CUDA header
 * in the plugin: it stays plain C).  cuipm_host_alloc returns NULL on failure. */
void *cuipm_host_alloc(size_t bytes);
void cuipm_host_free(void *p);

/* Device memory owned by the solver, for callers that stage data themselves (bench, multi-GPU scatter). */
double *cuipm_device_qp_buffer(cuipm_solver *s);       /* max_batch * qp_stride doubles  */
double *cuipm_device_sol_buffer(cuipm_solver *s);      /* max_batch * sol_stride doubles */
cuipm_info *cuipm_device_info_buffer(cuipm_solver *s); /* max_batch */
void *cuipm_stream(cuipm_solver *s);                   /* cudaStream_t */

/* Solution sensitivities with the factorisation of the last IPM iteration of the preceding solve on this solver
 * (reference: d_ocp_qp_ipm_sens_frw / d_ocp_qp_ipm_sens_adj, external/hpipm/ocp_qp/x_ocp_qp_ipm.c:3285-3444, reached through
 * ocp_qp_hpipm_eval_forw_sens / ocp_qp_hpipm_eval_adj_sens, acados/ocp_qp/ocp_qp_hpipm.c:481-506).
 * seed, sens: nbatch records in the SOLUTION layout -- (seed_g, seed_b, seed_d, seed_m) in the (ux, pi, lam, t) slots of
 * the seed, the sensitivities of (ux, pi, lam, t) in sens.  One substitution per QP, no refactorisation.  The host
 * variant uses the QP records the preceding cuipm_solve_host left in the solver's device buffer; the device variant is
 * handed the same d_qp as the preceding cuipm_solve_device. */
int cuipm_sens_host(cuipm_solver *s, int nbatch, const double *seed, double *sens, int adjoint, const cuipm_opts *opts);
int cuipm_sens_device(cuipm_solver *s, int nbatch, const double *d_qp, const double *d_seed, double *d_sens, int adjoint,
                      const cuipm_opts *opts, int sync);

/* ---- stage-0 equality elimination on the device ---------------------------------------------------------------------
 * Reference: d_ocp_qp_reduce_eq_dof / d_ocp_qp_restore_eq_dof (external/hpipm/ocp_qp/x_ocp_qp_red.c:278-560, 848-994), which
 * acados' ocp_qp_partial_condensing (acados/ocp_qp/ocp_qp_partial_condensing.c:523-689) runs around every QP solve; with
 * the default N2 = N they are all that module does.  `full` is the shape as the user poses it (stage 0 carries x_0 with
 * state bounds; idxe0[0..nbxe0) are the positions, in stage 0's bound list, of the bounds that are equalities lb = ub =
 * x0).  cuipm_reduce_device maps QP records of the full shape to QP records of the reduced shape (the one to create the
 * cuipm_solver with), cuipm_restore_device maps solution records back, multipliers of the dropped bounds included.
 * All pointers are device pointers; stream is a cudaStream_t (may be NULL). */
typedef struct cuipm_reducer cuipm_reducer;
cuipm_reducer *cuipm_reducer_create(const cuipm_shape *full, int nbxe0, const int *idxe0, int device);
void cuipm_reducer_destroy(cuipm_reducer *r);
const cuipm_shape *cuipm_reducer_reduced_shape(const cuipm_reducer *r);     /* owned by r */
const cuipm_layout *cuipm_reducer_full_layout(const cuipm_reducer *r);
const cuipm_layout *cuipm_reducer_reduced_layout(const cuipm_reducer *r);
int cuipm_reduce_device(cuipm_reducer *r, int nbatch, const double *d_qp_full, double *d_qp_red, void *stream);
int cuipm_restore_device(cuipm_reducer *r, int nbatch, const double *d_qp_full, const double *d_sol_red, double *d_sol_full,
                         double lam_min, double t_min, void *stream);

/* ---- partial (block) condensing on the device -----------------------------------------------------------------------
 * Reference: ocp_qp_partial_condensing (acados/ocp_qp/ocp_qp_partial_condensing.c:523-689) -> d_part_cond_qp_cond /
 * d_part_cond_qp_expand_sol (external/hpipm/cond/x_part_cond.c:410-866), for cond_N < N.  `shape` is the shape the solver
 * would otherwise be created with (after the stage-0 equality elimination); the N stages are grouped into cond_N blocks
 * (sizes as d_part_cond_qp_compute_block_size, the terminal stage stays), cuipm_condense_device maps QP records of `shape`
 * to QP records of the condensed shape (create the cuipm_solver with that one), cuipm_expand_device maps solution records
 * of the condensed QPs back (inner states from the dynamics, inner multipliers from stationarity).  Device pointers;
 * stream is a cudaStream_t (may be NULL). */
typedef struct cuipm_condenser cuipm_condenser;
cuipm_condenser *cuipm_condenser_create(const cuipm_shape *shape, int cond_N, int device);
void cuipm_condenser_destroy(cuipm_condenser *c);
const cuipm_shape *cuipm_condenser_condensed_shape(const cuipm_condenser *c);     /* owned by c */
int cuipm_condense_device(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, void *stream);
int cuipm_expand_device(cuipm_condenser *c, int nbatch, const double *d_qp, const double *d_sol_cond, double *d_sol, void *stream);
/* The lhs / rhs split of the reference's condensing module (ocp_qp_partial_condensing.c:575-630 condense_lhs / condense_rhs ->
 * d_part_cond_qp_cond_lhs / _rhs, x_part_cond.c:410,564; used by ocp_qp_xcond_solver.c:591-669 and the SQP-RTI preparation /
 * feedback phases, ocp_nlp_sqp_rti.c:461-520): cuipm_condense_lhs_device condenses the QPs and keeps the prediction matrices of
 * every stage per QP on the device; cuipm_condense_rhs_device then refreshes only the vectors of the SAME condensed records
 * (gradients, dynamics offsets, shifted bounds) from records whose matrices are unchanged and whose vectors (b, rq, d, z --
 * e.g. a new x0 folded in by the stage-0 elimination) are new.  Same arguments as cuipm_condense_device. */
int cuipm_condense_lhs_device(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, void *stream);
int cuipm_condense_rhs_device(cuipm_condenser *c, int nbatch, const double *d_qp, double *d_qp_cond, void *stream);

/* ---- the whole xcond chain behind one object -------------------------------------------------------------------------
 * Reference: ocp_qp_xcond_solver (acados/ocp_qp/ocp_qp_xcond_solver.c:523-669): condensing module + QP solver + expansion,
 * evaluate() in one piece or split into condense_lhs (:591-627, preparation phase of SQP-RTI) and condense_rhs_and_solve
 * (:629-669, feedback phase).  `full` is the shape as the user poses it, idxe0 as for cuipm_reducer_create; cond_N in 1..N
 * (<= 0 or N: no block condensing).  The reduced / condensed records, the prediction matrices of the lhs pass and all
 * intermediate solutions live on the device.  With warm_start >= 2 the solve starts from this object's previous solution in the
 * reduced / condensed layout (zeros before the first solve), as the reference runs its QP solver on the condensed solution of
 * the previous call unless initialize_next_xcond_qp_from_qp_out is set (ocp_qp_xcond_solver.c:554-569).
 *
 * Two kinds of entry run the same device chain:
 *   _host:   records of the full shape come from (page-locked) host memory; solutions of the full shape, the per-QP summaries
 *            and, if `stat` is not NULL, the statistics tables (as for cuipm_solve_host) go back; synchronises.  The object
 *            allocates its device copies of the records and solutions at the first host call.
 *   _device: as cuipm_solve_device -- device pointers on the object's device, the work enqueued on the stream of
 *            cuipm_xcond_solver(x) (cuipm_stream), a synchronise only if `sync` != 0.  The reducer and the restore read
 *            d_qp_full in place: it must stay unchanged until the call's work has completed.  d_stat may be NULL, else it holds
 *            nbatch x (stat_max+1) x CUIPM_STAT_M doubles. */
typedef struct cuipm_xcond cuipm_xcond;
cuipm_xcond *cuipm_xcond_create(const cuipm_shape *full, int nbxe0, const int *idxe0, int cond_N, int max_batch, int device);
void cuipm_xcond_destroy(cuipm_xcond *x);
const cuipm_layout *cuipm_xcond_full_layout(const cuipm_xcond *x);
int cuipm_xcond_cond_N(const cuipm_xcond *x);
/* The solver of the reduced / condensed shape (statistics, getters, sensitivities); owned by x.  Its device buffers hold the
 * reduced or condensed records and solutions of the last call. */
cuipm_solver *cuipm_xcond_solver(cuipm_xcond *x);
int cuipm_xcond_solve_host(cuipm_xcond *x, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info, double *stat,
                           const cuipm_opts *opts);
int cuipm_xcond_condense_lhs_host(cuipm_xcond *x, int nbatch, const double *qp_full);
int cuipm_xcond_condense_rhs_and_solve_host(cuipm_xcond *x, int nbatch, const double *qp_full, double *sol_full, cuipm_info *info,
                                            double *stat, const cuipm_opts *opts);
int cuipm_xcond_solve_device(cuipm_xcond *x, int nbatch, const double *d_qp_full, double *d_sol_full, cuipm_info *d_info,
                             double *d_stat, const cuipm_opts *opts, int sync);
int cuipm_xcond_condense_lhs_device(cuipm_xcond *x, int nbatch, const double *d_qp_full, int sync);
int cuipm_xcond_condense_rhs_and_solve_device(cuipm_xcond *x, int nbatch, const double *d_qp_full, double *d_sol_full,
                                              cuipm_info *d_info, double *d_stat, const cuipm_opts *opts, int sync);

/* ---- records of the full shape assembled on the device from per-field sources ------------------------------------------
 * Fields carry the names and orientation of the reference's AcadosOcpQp.set (interfaces/acados_template/acados_template/
 * acados_ocp_qp.py): A is nx_next x nx, B nx_next x nu, S nu x nx, C ng x nx, D ng x nu, Q nx x nx, R nu x nu; the others are
 * vectors.  lbu / ubu are the first nbu bounds of idxb (the entries < nu), lbx / ubx the others. */
enum cuipm_field {
    CUIPM_F_A, CUIPM_F_B, CUIPM_F_b, CUIPM_F_Q, CUIPM_F_R, CUIPM_F_S, CUIPM_F_q, CUIPM_F_r,
    CUIPM_F_lbu, CUIPM_F_ubu, CUIPM_F_lbx, CUIPM_F_ubx, CUIPM_F_C, CUIPM_F_D, CUIPM_F_lg, CUIPM_F_ug,
    CUIPM_F_Zl, CUIPM_F_Zu, CUIPM_F_zl, CUIPM_F_zu, CUIPM_F_lls, CUIPM_F_lus,
    CUIPM_F_lbu_mask, CUIPM_F_ubu_mask, CUIPM_F_lbx_mask, CUIPM_F_ubx_mask, CUIPM_F_lg_mask, CUIPM_F_ug_mask,
    CUIPM_F_lls_mask, CUIPM_F_lus_mask,
    CUIPM_F_COUNT
};
/* One field of one stage for every QP of the batch: element (r, c) of QP q is ptr[q*s_batch + r*s_row + c*s_col] (vectors:
 * element r, s_col unused).  Strides are in doubles and >= 0; s_batch = 0 gives every QP the same value. */
typedef struct cuipm_src {
    int field, stage;
    const double *ptr;
    long long s_batch, s_row, s_col;
} cuipm_src;
/* Writes nbatch records of the full shape of x into d_qp_full (device memory, nbatch x qp_stride doubles of
 * cuipm_xcond_full_layout) -- the bits the host packer writes for the same data: HPIPM's record conventions (BAt = [B'; A'],
 * both triangles of RSQ, DCt = [D'; C'], d = [lbu, lbx, lg, -ubu, -ubx, -ug, lls, lus], masks in the same order), zeros for
 * the padding and for every field without a source, ones for masks without one.  One kernel on the stream of
 * cuipm_xcond_solver(x), after the source table (built on the host each call) has been copied there; a synchronise only if
 * `sync` != 0.  A (field, stage) given twice, a field that does not exist at its stage (size 0 there: dynamics at N, slacks
 * where ns = 0, ...), a negative stride or a null pointer returns CUIPM_ERR_INVALID before anything is enqueued.  The sources
 * are read when the kernel runs. */
int cuipm_xcond_assemble_device(cuipm_xcond *x, int nbatch, const cuipm_src *src, int nsrc, double *d_qp_full, int sync);

/* Riccati quantities of the last factorisation (reference: ocp_qp_hpipm_solver_get, ocp_qp_hpipm.c:417-478).
 * field in {"P","p","K","k","Lr"}; copies column-major data of QP `iqp`, stage `stage` into `value`. */
int cuipm_get_ric(cuipm_solver *s, int iqp, const char *field, int stage, double *value, int size1, int size2);

/* number of kernels the last solve call launched (bench.py's gpu_launches claim) */
int cuipm_last_launch_count(const cuipm_solver *s);
/* device time in milliseconds of the last cuipm_solve_* call with sync, all its kernels (CUDA events on the solver's stream) */
float cuipm_last_kernel_ms(const cuipm_solver *s);
/* device time in milliseconds of the dominant kernel alone (the throughput kernel where the shape has one; CUDA events around
 * that launch) of the last synchronous cuipm_solve_device call */
float cuipm_last_main_kernel_ms(cuipm_solver *s);
/* QPs of the last solve that the throughput kernel handed back to the generic kernel (cold paths: LQ refactorisation,
 * iterative refinement, no active constraint); 0 where the generic kernel solved everything.  Synchronises. */
int cuipm_last_handed_back(cuipm_solver *s);
/* launch tuning without a reference counterpart: key "warps" = warps cooperating on one QP in the generic kernel (1, 2 or 4;
 * the default is chosen from the stage dimensions); key "pipe" = chunks (1..8, default 8) the host entry splits a batch into
 * so that the copies of one chunk overlap the solve of the others; key "fast" = 0 keeps eligible shapes off the throughput
 * kernel (several QPs per warp, acados_b200/csrc/cuipm_fast.cu); key "spill" = 1 runs the generic kernel's global-scratch
 * variant (stage-block buffers in a per-QP device scratch buffer, allocated on first use) on a shape that fits in shared
 * memory, 0 restores the default -- a test hook like "fast": the variant is chosen by itself exactly for the shapes that do
 * not fit, and gives the same results bit for bit.  Results do not depend on any of them beyond floating-point summation
 * order. */
int cuipm_set_tuning(cuipm_solver *s, const char *key, int value);

#ifdef __cplusplus
}
#endif
#endif /* CUIPM_H_ */
