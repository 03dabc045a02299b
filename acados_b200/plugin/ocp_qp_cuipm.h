/*
 * ocp_qp_cuipm.h -- acados `qp_solver` plugin backed by the cuipm CUDA library (include/cuipm.h).
 *
 * Drop-in for acados/ocp_qp/ocp_qp_hpipm.{c,h}: same vtable (acados/ocp_qp/ocp_qp_common.h:60-79), same option
 * field names, same memory_get fields, same status mapping.  Inside libacados this file would live at
 * acados/ocp_qp/ocp_qp_cuipm.h and be registered as PARTIAL_CONDENSING_CUIPM (see INTEGRATION.md).
 */
#ifndef ACADOS_OCP_QP_OCP_QP_CUIPM_H_
#define ACADOS_OCP_QP_OCP_QP_CUIPM_H_

#ifdef __cplusplus
extern "C" {
#endif

#include "acados/ocp_qp/ocp_qp_common.h"
#include "acados/utils/types.h"

#include "cuipm.h"

typedef struct ocp_qp_cuipm_opts_
{
    cuipm_opts c;       /* solver options (HPIPM field names, see cuipm_opts_set) */
    int print_level;
    int device;         /* CUDA device ordinal (default 0) */
} ocp_qp_cuipm_opts;

typedef struct ocp_qp_cuipm_memory_
{
    cuipm_solver *solver;       /* device resources; created lazily on the first evaluate, freed in terminate */
    int max_batch;              /* capacity of `solver` */
    int N;
    int *dims_i;                /* nx,nu,nb,ng,ns copies: 5*(N+1) ints */
    int *idx_pool;              /* idxb / idxs_rev copies the solver was created with */
    int **idxb_p, **idxs_rev_p; /* per-stage pointers into idx_pool */
    int idx_pool_len;
    double *qp_rec, *sol_rec;   /* host staging records for the single-QP path (pinned lazily is not possible in raw memory) */
    double *seed_rec, *sens_rec; /* staging records of eval_forw_sens / eval_adj_sens (solution layout) */
    double *stat;               /* (stat_max+1) x CUIPM_STAT_M table of the last solve (HPIPM's layout: row per iteration) */
    int stat_max_alloc;         /* stat_max the table was sized with at memory creation (the reference freezes ws->stat_max there too) */
    /* batch entry: page-locked staging buffers owned by the memory object (cuipm_host_alloc), grown on demand, freed in
     * terminate / memory_reset -- no allocation per call */
    double *b_qp, *b_sol;
    cuipm_info *b_info;
    int b_cap;                  /* QPs the staging buffers hold */
    cuipm_info info;
    double time_qp_solver_call;
    int iter;
    int status;                 /* HPIPM status code of the last solve */
} ocp_qp_cuipm_memory;

acados_size_t ocp_qp_cuipm_opts_calculate_size(void *config, void *dims);
void *ocp_qp_cuipm_opts_assign(void *config, void *dims, void *raw_memory);
void ocp_qp_cuipm_opts_initialize_default(void *config, void *dims, void *opts_);
void ocp_qp_cuipm_opts_update(void *config, void *dims, void *opts_);
void ocp_qp_cuipm_opts_set(void *config_, void *opts_, const char *field, void *value);
void ocp_qp_cuipm_opts_get(void *config_, void *opts_, const char *field, void *value);
acados_size_t ocp_qp_cuipm_memory_calculate_size(void *config, void *dims, void *opts_);
void *ocp_qp_cuipm_memory_assign(void *config, void *dims, void *opts_, void *raw_memory);
void ocp_qp_cuipm_memory_get(void *config_, void *mem_, const char *field, void *value);
acados_size_t ocp_qp_cuipm_workspace_calculate_size(void *config, void *dims, void *opts_);
int ocp_qp_cuipm(void *config, void *qp_in, void *qp_out, void *opts_, void *mem_, void *work_);
void ocp_qp_cuipm_memory_reset(void *config_, void *qp_in_, void *qp_out_, void *opts_, void *mem_, void *work_);
void ocp_qp_cuipm_solver_get(void *config_, void *qp_in_, void *qp_out_, void *opts_, void *mem_, const char *field, int stage,
                             void *value, int size1, int size2);
void ocp_qp_cuipm_eval_forw_sens(void *config_, void *qp_in, void *seed, void *qp_out, void *opts_, void *mem_, void *work_);
void ocp_qp_cuipm_eval_adj_sens(void *config_, void *qp_in, void *seed, void *qp_out, void *opts_, void *mem_, void *work_);
void ocp_qp_cuipm_terminate(void *config_, void *mem_, void *work_);
void ocp_qp_cuipm_config_initialize_default(void *config);

/* Batched entry the reference lacks (SURVEY.md section 8(b)): n structurally identical QPs in, n solutions out, one
 * kernel launch.  `mem` must come from memory_assign of this plugin; status_out[i] receives acados return codes.
 * Replaces the OpenMP loop over capsules of the generated batch solver (c_templates_tera/acados_solver.in.c:3223-3243)
 * at the QP level.  Returns the worst acados status. */
int ocp_qp_cuipm_batch_solve(void *config, int n, ocp_qp_in **qp_in, ocp_qp_out **qp_out, void *opts_, void *mem_, int *status_out);

/* The xcond chain as a batched entry: n structurally identical UNCONDENSED QPs as ocp_qp_xcond_solver holds them (x0 as stage-0
 * equality bounds, dims->nbxe[0] / qp_in->idxe[0]) in, solutions of the same shape out; the stage-0 elimination, the block
 * condensing to cond_N stages (1..N; <= 0: N), the interior-point solve, the expansion and the restore all run on the device
 * (cuipm_xcond_*, include/cuipm.h) -- the batched counterpart of ocp_qp_xcond_solver's evaluate (ocp_qp_xcond_solver.c:523-589)
 * with acados' CPU condensing module taken out of the path.  phase: 0 = one pass; 1 = condense_lhs only (:591-627, nothing is
 * written to qp_out); 2 = condense_rhs_and_solve (:629-669) on QPs whose matrices are those of the last phase-1 call.
 * With warm_start >= 2 a solve starts from the context's previous condensed solution (zeros before the first), as
 * ocp_qp_xcond_solver does with its xcond_qp_out (:554-569); the qp_out structs are not read.
 * The context owns the device objects and the page-locked staging. */
typedef struct ocp_qp_cuipm_xcond_batch ocp_qp_cuipm_xcond_batch;
ocp_qp_cuipm_xcond_batch *ocp_qp_cuipm_xcond_batch_create(ocp_qp_in *qp_in0, int n_max, int cond_N, int device);
int ocp_qp_cuipm_xcond_batch_solve(ocp_qp_cuipm_xcond_batch *ctx, int n, ocp_qp_in **qp_in, ocp_qp_out **qp_out, void *opts_, int phase,
                                   int *status_out);
void ocp_qp_cuipm_xcond_batch_destroy(ocp_qp_cuipm_xcond_batch *ctx);

#ifdef __cplusplus
}
#endif
#endif
