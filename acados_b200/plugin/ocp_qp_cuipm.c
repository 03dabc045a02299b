/*
 * ocp_qp_cuipm.c -- acados `qp_solver` plugin: plain C inside libacados, all arithmetic in the cuipm CUDA library
 * reached through the C ABI of include/cuipm.h (static- or dynamic-linked).  Supersedes acados/ocp_qp/ocp_qp_hpipm.c
 * on this path; structure follows the plugin contract of acados/ocp_qp/ocp_qp_common.h:60-79:
 * the caller owns all host memory (sizes reported by *_calculate_size, carved by *_assign, 8-byte aligned),
 * `mem` persists across calls, device resources are created lazily on the first evaluate and released in terminate.
 *
 * There is no CPU fallback: if the CUDA library cannot create a solver, evaluate prints the error and exits
 * (the reference's convention for unrecoverable plugin errors, e.g. ocp_qp_hpipm.c:287-291).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "blasfeo/include/blasfeo_d_aux.h"
#include "hpipm/include/hpipm_d_ocp_qp.h"
#include "hpipm/include/hpipm_d_ocp_qp_seed.h"
#include "hpipm/include/hpipm_d_ocp_qp_sol.h"

#include "acados/utils/mem.h"
#include "acados/utils/timing.h"

#include "ocp_qp_cuipm.h"

/************************************************
 * opts
 ************************************************/

acados_size_t ocp_qp_cuipm_opts_calculate_size(void *config_, void *dims_)
{
    acados_size_t size = sizeof(ocp_qp_cuipm_opts) + 8;
    make_int_multiple_of(8, &size);
    return size;
}

void *ocp_qp_cuipm_opts_assign(void *config_, void *dims_, void *raw_memory)
{
    char *c_ptr = (char *) raw_memory;
    align_char_to(8, &c_ptr);
    return (void *) c_ptr;
}

void ocp_qp_cuipm_opts_initialize_default(void *config_, void *dims_, void *opts_)
{
    ocp_qp_cuipm_opts *opts = opts_;
    /* BALANCE mode + the overrides acados applies (ocp_qp_hpipm.c:101-129) */
    cuipm_opts_set_default_acados(&opts->c, CUIPM_BALANCE);
    opts->print_level = 0;
    opts->device = 0;
}

void ocp_qp_cuipm_opts_update(void *config_, void *dims_, void *opts_) {}

void ocp_qp_cuipm_opts_set(void *config_, void *opts_, const char *field, void *value)
{
    ocp_qp_cuipm_opts *opts = opts_;
    if (!strcmp(field, "print_level")) opts->print_level = *(int *) value;
    else if (!strcmp(field, "device")) opts->device = *(int *) value;
    else if (!strcmp(field, "tau_min")) opts->c.m_relax = *(double *) value;   /* as ocp_qp_hpipm.c:170-174 */
    else if (cuipm_opts_set(&opts->c, field, value) != CUIPM_OK)
    {
        printf("\nerror: ocp_qp_cuipm_opts_set: field %s not available\n", field);
        exit(1);
    }
}

void ocp_qp_cuipm_opts_get(void *config_, void *opts_, const char *field, void *value)
{
    ocp_qp_cuipm_opts *opts = opts_;
    if (cuipm_opts_get(&opts->c, field, value) != CUIPM_OK)
    {
        printf("\nerror: ocp_qp_cuipm_opts_get: field %s not available\n", field);
        exit(1);
    }
}

/************************************************
 * memory
 ************************************************/

static void shape_from_dims(const ocp_qp_dims *dims, cuipm_shape *sh)
{
    sh->N = dims->N; sh->nx = dims->nx; sh->nu = dims->nu; sh->nb = dims->nb; sh->ng = dims->ng; sh->ns = dims->ns;
    sh->idxb = NULL; sh->idxs_rev = NULL;
}

static acados_size_t idx_pool_len(const ocp_qp_dims *dims)
{
    acados_size_t n = 0;
    for (int k = 0; k <= dims->N; k++) n += 2 * dims->nb[k] + dims->ng[k];
    return n;
}

/* shape of `in`, its idxb / idxs_rev (-1 on stages without slacks) copied into pool with per-stage pointers idxb_p / rev_p */
static cuipm_shape shape_from_in(const ocp_qp_in *in, int *pool, int **idxb_p, int **rev_p)
{
    const ocp_qp_dims *d = in->dim;
    int o = 0;
    for (int k = 0; k <= d->N; k++)
    {
        idxb_p[k] = pool + o;
        for (int i = 0; i < d->nb[k]; i++) pool[o++] = in->idxb[k][i];
        rev_p[k] = pool + o;
        for (int i = 0; i < d->nb[k] + d->ng[k]; i++) pool[o++] = d->ns[k] > 0 ? in->idxs_rev[k][i] : -1;
    }
    cuipm_shape sh;
    shape_from_dims(d, &sh);
    sh.idxb = (const int *const *) idxb_p;
    sh.idxs_rev = (const int *const *) rev_p;
    return sh;
}

acados_size_t ocp_qp_cuipm_memory_calculate_size(void *config_, void *dims_, void *opts_)
{
    ocp_qp_dims *dims = dims_;
    ocp_qp_cuipm_opts *opts = opts_;
    cuipm_shape sh;
    shape_from_dims(dims, &sh);
    /* record sizes depend on the dims only: borrow empty index maps */
    cuipm_layout *l = cuipm_layout_create(&sh);
    acados_size_t size = sizeof(ocp_qp_cuipm_memory);
    size += 5 * (dims->N + 1) * sizeof(int) + idx_pool_len(dims) * sizeof(int) + 8;
    size += 2 * (dims->N + 1) * sizeof(int *);
    size += (l->qp_stride + 3 * l->sol_stride) * sizeof(double);
    size += (acados_size_t) (opts->c.stat_max + 1) * CUIPM_STAT_M * sizeof(double);
    size += 3 * 8;
    cuipm_layout_destroy(l);
    make_int_multiple_of(8, &size);
    return size;
}

void *ocp_qp_cuipm_memory_assign(void *config_, void *dims_, void *opts_, void *raw_memory)
{
    ocp_qp_dims *dims = dims_;
    ocp_qp_cuipm_opts *opts = opts_;
    char *c_ptr = (char *) raw_memory;
    align_char_to(8, &c_ptr);
    ocp_qp_cuipm_memory *mem = (ocp_qp_cuipm_memory *) c_ptr;
    c_ptr += sizeof(ocp_qp_cuipm_memory);
    memset(mem, 0, sizeof(*mem));
    mem->N = dims->N;
    align_char_to(8, &c_ptr);
    mem->idxb_p = (int **) c_ptr; c_ptr += (dims->N + 1) * sizeof(int *);
    mem->idxs_rev_p = (int **) c_ptr; c_ptr += (dims->N + 1) * sizeof(int *);
    mem->dims_i = (int *) c_ptr; c_ptr += 5 * (dims->N + 1) * sizeof(int);
    mem->idx_pool = (int *) c_ptr; mem->idx_pool_len = (int) idx_pool_len(dims); c_ptr += mem->idx_pool_len * sizeof(int);
    align_char_to(8, &c_ptr);
    cuipm_shape sh;
    shape_from_dims(dims, &sh);
    cuipm_layout *l = cuipm_layout_create(&sh);
    mem->qp_rec = (double *) c_ptr; c_ptr += l->qp_stride * sizeof(double);
    mem->sol_rec = (double *) c_ptr; c_ptr += l->sol_stride * sizeof(double);
    mem->seed_rec = (double *) c_ptr; c_ptr += l->sol_stride * sizeof(double);
    mem->sens_rec = (double *) c_ptr; c_ptr += l->sol_stride * sizeof(double);
    mem->stat = (double *) c_ptr; c_ptr += (acados_size_t) (opts->c.stat_max + 1) * CUIPM_STAT_M * sizeof(double);
    mem->stat_max_alloc = opts->c.stat_max;
    cuipm_layout_destroy(l);
    mem->solver = NULL;
    mem->status = 0;
    return mem;
}

void ocp_qp_cuipm_memory_get(void *config_, void *mem_, const char *field, void *value)
{
    ocp_qp_cuipm_memory *mem = mem_;
    if (!strcmp(field, "time_qp_solver_call")) *(double *) value = mem->time_qp_solver_call;
    else if (!strcmp(field, "iter")) *(int *) value = mem->iter;
    else if (!strcmp(field, "status")) *(int *) value = mem->status;
    else if (!strcmp(field, "stat")) *(double **) value = mem->stat;
    else if (!strcmp(field, "stat_m")) *(int *) value = CUIPM_STAT_M;
    else if (!strcmp(field, "tau_iter"))
    {   /* barrier parameter of the last corrector step = sigma * mu of the last iteration (stat columns 3 and 6) */
        double tau = 0.0;
        if (mem->iter > 0 && mem->iter < mem->stat_max_alloc) tau = mem->stat[CUIPM_STAT_M * mem->iter + 3] * mem->stat[CUIPM_STAT_M * (mem->iter - 1) + 6];
        *(double *) value = tau;
    }
    else
    {
        printf("\nerror: ocp_qp_cuipm_memory_get: field %s not available\n", field);
        exit(1);
    }
}

acados_size_t ocp_qp_cuipm_workspace_calculate_size(void *config_, void *dims_, void *opts_) { return 0; }

/************************************************
 * marshalling between struct d_ocp_qp (panel-major BLASFEO) and cuipm records
 ************************************************/

static int same_structure(ocp_qp_cuipm_memory *mem, const ocp_qp_in *in)
{
    const ocp_qp_dims *d = in->dim;
    int N = d->N, *pool = mem->idx_pool, o = 0;
    if (N != mem->N) return 0;
    for (int k = 0; k <= N; k++)
    {
        int *di = mem->dims_i + 5 * k;
        if (di[0] != d->nx[k] || di[1] != d->nu[k] || di[2] != d->nb[k] || di[3] != d->ng[k] || di[4] != d->ns[k]) return 0;
        for (int i = 0; i < d->nb[k]; i++) if (pool[o++] != in->idxb[k][i]) return 0;
        for (int i = 0; i < d->nb[k] + d->ng[k]; i++) if (pool[o++] != (d->ns[k] > 0 ? in->idxs_rev[k][i] : -1)) return 0;
    }
    return 1;
}

static void ensure_solver(ocp_qp_cuipm_memory *mem, ocp_qp_cuipm_opts *opts, const ocp_qp_in *in, int nbatch)
{
    if (mem->solver && mem->max_batch >= nbatch && same_structure(mem, in)) return;
    if (mem->solver) cuipm_destroy(mem->solver);
    const ocp_qp_dims *d = in->dim;
    for (int k = 0; k <= d->N; k++)
    {
        int *di = mem->dims_i + 5 * k;
        di[0] = d->nx[k]; di[1] = d->nu[k]; di[2] = d->nb[k]; di[3] = d->ng[k]; di[4] = d->ns[k];
    }
    cuipm_shape sh = shape_from_in(in, mem->idx_pool, mem->idxb_p, mem->idxs_rev_p);
    mem->solver = cuipm_create(&sh, nbatch, opts->device);
    mem->max_batch = nbatch;
    if (!mem->solver)
    {
        printf("\nerror: ocp_qp_cuipm: %s\n", cuipm_last_error());
        exit(1);
    }
}

static void pack_qp(const ocp_qp_in *in, const cuipm_layout *l, double *rec)
{
    const ocp_qp_dims *d = in->dim;
    for (int k = 0; k <= d->N; k++)
    {
        int n = d->nu[k] + d->nx[k], nc = 2 * (d->nb[k] + d->ng[k] + d->ns[k]);
        if (k < d->N)
        {
            blasfeo_unpack_dmat(n, d->nx[k + 1], in->BAbt + k, 0, 0, rec + l->off_BAt[k], n);
            blasfeo_unpack_dvec(d->nx[k + 1], in->b + k, 0, rec + l->off_b[k], 1);
        }
        blasfeo_unpack_dmat(n, n, in->RSQrq + k, 0, 0, rec + l->off_RSQ[k], n);
        blasfeo_unpack_dvec(n, in->rqz + k, 0, rec + l->off_rq[k], 1);
        if (d->ng[k] > 0) blasfeo_unpack_dmat(n, d->ng[k], in->DCt + k, 0, 0, rec + l->off_DCt[k], n);
        blasfeo_unpack_dvec(nc, in->d + k, 0, rec + l->off_d[k], 1);
        blasfeo_unpack_dvec(nc, in->d_mask + k, 0, rec + l->off_dmask[k], 1);
        if (d->ns[k] > 0)
        {
            blasfeo_unpack_dvec(2 * d->ns[k], in->Z + k, 0, rec + l->off_Z[k], 1);
            blasfeo_unpack_dvec(2 * d->ns[k], in->rqz + k, n, rec + l->off_z[k], 1);
        }
    }
}

static void pack_sol(const ocp_qp_out *out, const ocp_qp_dims *d, const cuipm_layout *l, double *rec)
{
    for (int k = 0; k <= d->N; k++)
    {
        int n = d->nu[k] + d->nx[k], nc = 2 * (d->nb[k] + d->ng[k] + d->ns[k]);
        blasfeo_unpack_dvec(n + 2 * d->ns[k], out->ux + k, 0, rec + l->off_ux[k], 1);
        if (k < d->N) blasfeo_unpack_dvec(d->nx[k + 1], out->pi + k, 0, rec + l->off_pi[k], 1);
        blasfeo_unpack_dvec(nc, out->lam + k, 0, rec + l->off_lam[k], 1);
        blasfeo_unpack_dvec(nc, out->t + k, 0, rec + l->off_t[k], 1);
    }
}

static void unpack_sol(const double *rec, const ocp_qp_dims *d, const cuipm_layout *l, ocp_qp_out *out)
{
    for (int k = 0; k <= d->N; k++)
    {
        int n = d->nu[k] + d->nx[k], nc = 2 * (d->nb[k] + d->ng[k] + d->ns[k]);
        blasfeo_pack_dvec(n + 2 * d->ns[k], (double *) rec + l->off_ux[k], 1, out->ux + k, 0);
        if (k < d->N) blasfeo_pack_dvec(d->nx[k + 1], (double *) rec + l->off_pi[k], 1, out->pi + k, 0);
        blasfeo_pack_dvec(nc, (double *) rec + l->off_lam[k], 1, out->lam + k, 0);
        blasfeo_pack_dvec(nc, (double *) rec + l->off_t[k], 1, out->t + k, 0);
    }
}

static int acados_status(int hpipm_status)
{   /* ocp_qp_hpipm.c:398-404 */
    switch (hpipm_status)
    {
        case CUIPM_SUCCESS: return ACADOS_SUCCESS;
        case CUIPM_MAX_ITER: return ACADOS_MAXITER;
        case CUIPM_MIN_STEP: return ACADOS_MINSTEP;
        case CUIPM_NAN_SOL: return ACADOS_NAN_DETECTED;
        case CUIPM_INCONS_EQ: return ACADOS_INFEASIBLE;
        default: return ACADOS_UNKNOWN;
    }
}

/* QP i of a batch back into its struct: solution, iteration count, acados status (status_out, if given) */
static void hand_back(int i, const double *sol, const cuipm_info *infos, const cuipm_layout *l, ocp_qp_in **qp_in, ocp_qp_out **qp_out, int *status_out)
{
    unpack_sol(sol + l->sol_stride * (size_t) i, qp_in[i]->dim, l, qp_out[i]);
    qp_info *info = qp_out[i]->misc;
    info->interface_time = 0; info->num_iter = infos[i].iter; info->t_computed = 1;
    if (status_out) status_out[i] = acados_status(infos[i].status);
}

/* the batch's wall-clock time t split evenly over its QPs' qp_info; returns the batch's worst acados status (its first failure) */
static int batch_result(int n, ocp_qp_out **qp_out, const cuipm_info *infos, double t)
{
    int worst = ACADOS_SUCCESS;
    for (int i = 0; i < n; i++)
    {
        qp_info *info = qp_out[i]->misc;
        info->solve_QP_time = t / n; info->total_time = t / n;
        if (worst == ACADOS_SUCCESS) worst = acados_status(infos[i].status);
    }
    return worst;
}

/************************************************
 * functions
 ************************************************/

int ocp_qp_cuipm(void *config_, void *qp_in_, void *qp_out_, void *opts_, void *mem_, void *work_)
{
    ocp_qp_in *qp_in = qp_in_;
    ocp_qp_out *qp_out = qp_out_;
    ocp_qp_cuipm_opts *opts = opts_;
    ocp_qp_cuipm_memory *mem = mem_;
    qp_info *info = qp_out->misc;
    acados_timer tot_timer, qp_timer;
    acados_tic(&tot_timer);

    ensure_solver(mem, opts, qp_in, 1);
    const cuipm_layout *l = cuipm_get_layout(mem->solver);
    pack_qp(qp_in, l, mem->qp_rec);
    if (opts->c.warm_start >= 2) pack_sol(qp_out, qp_in->dim, l, mem->sol_rec);   /* pi, lam, t carried over; ux is zeroed by the solver */
    double interface_time = acados_toc(&tot_timer);

    acados_tic(&qp_timer);
    /* the statistics table was sized when the memory was created: iter_max may have been raised since (the reference
     * keeps ws->stat_max of the workspace creation and guards every write with it, x_ocp_qp_ipm.c:2227) */
    cuipm_opts o = opts->c;
    if (o.stat_max > mem->stat_max_alloc) o.stat_max = mem->stat_max_alloc;
    int rc = cuipm_solve_host(mem->solver, 1, mem->qp_rec, mem->sol_rec, &mem->info, mem->stat, &o);
    if (rc != CUIPM_OK)
    {
        printf("\nerror: ocp_qp_cuipm: %s\n", cuipm_last_error());
        exit(1);
    }
    info->solve_QP_time = acados_toc(&qp_timer);

    acados_tic(&qp_timer);
    unpack_sol(mem->sol_rec, qp_in->dim, l, qp_out);
    interface_time += acados_toc(&qp_timer);

    mem->status = mem->info.status;
    mem->iter = mem->info.iter;
    mem->time_qp_solver_call = info->solve_QP_time;
    info->interface_time = interface_time;
    info->total_time = acados_toc(&tot_timer);
    info->num_iter = mem->iter;
    info->t_computed = 1;

    if (opts->print_level > 0)
    {
        printf("\nalpha_prim_aff\talpha_dual_aff\tmu_aff\t\tsigma\t\talpha_prim\talpha_dual\tmu\t\tres_stat\tres_eq\t\tres_ineq\tres_comp\tdual gap\tobj\n");
        for (int i = 0; i <= mem->iter && i < mem->stat_max_alloc; i++)
        {
            for (int j = 0; j < 13; j++) printf("%e\t", mem->stat[CUIPM_STAT_M * i + j]);
            printf("\n");
        }
    }
    return acados_status(mem->status);
}

/* threads for the struct (un)packing: the OpenMP default, capped by the cgroup CPU quota (a container may show 128 CPUs and allow
 * 16 CPUs' worth of time: a team sized from the mask then burns the quota in its barriers) and by CUIPM_HOST_THREADS */
static int pack_threads(void)
{
    static int nt = 0;
    if (nt > 0) return nt;
    int n = omp_get_max_threads();
    FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f)
    {
        char q[32];
        long per = 0;
        if (fscanf(f, "%31s %ld", q, &per) == 2 && strcmp(q, "max") && per > 0)
        {
            long c = (atol(q) + per - 1) / per;
            if (c >= 1 && c < n) n = (int) c;
        }
        fclose(f);
    }
    const char *e = getenv("CUIPM_HOST_THREADS");
    if (e && atoi(e) > 0) n = atoi(e);
    nt = n > 0 ? n : 1;
    return nt;
}

/* page-locked staging of the batched entries (the plugin's raw memory is pageable and sized for one QP): records and summaries */
static void staging_free(double **qp, double **sol, cuipm_info **info, int *cap)
{
    cuipm_host_free(*qp); cuipm_host_free(*sol); cuipm_host_free(*info);
    *qp = *sol = NULL; *info = NULL; *cap = 0;
}

/* grows the staging to n QPs of layout l; 0 if an allocation failed (cuipm_last_error() says why) */
static int staging_grow(const cuipm_layout *l, int n, double **qp, double **sol, cuipm_info **info, int *cap)
{
    if (*cap >= n) return 1;
    staging_free(qp, sol, info, cap);
    *qp = cuipm_host_alloc(sizeof(double) * l->qp_stride * (size_t) n);
    *sol = cuipm_host_alloc(sizeof(double) * l->sol_stride * (size_t) n);
    *info = cuipm_host_alloc(sizeof(cuipm_info) * (size_t) n);
    if (!*qp || !*sol || !*info) return 0;
    *cap = n;
    return 1;
}

int ocp_qp_cuipm_batch_solve(void *config_, int n, ocp_qp_in **qp_in, ocp_qp_out **qp_out, void *opts_, void *mem_, int *status_out)
{
    ocp_qp_cuipm_opts *opts = opts_;
    ocp_qp_cuipm_memory *mem = mem_;
    if (n <= 0) return ACADOS_SUCCESS;
    acados_timer timer;
    acados_tic(&timer);
    ensure_solver(mem, opts, qp_in[0], n);
    const cuipm_layout *l = cuipm_get_layout(mem->solver);
    if (!staging_grow(l, n, &mem->b_qp, &mem->b_sol, &mem->b_info, &mem->b_cap)) { printf("\nerror: ocp_qp_cuipm_batch_solve: %s\n", cuipm_last_error()); exit(1); }
    double *qp = mem->b_qp, *sol = mem->b_sol;
    cuipm_info *infos = mem->b_info;
    /* Pipeline over chunks, two parallel regions in all (a region per chunk costs a barrier of the whole thread team each, which
     * dominates when the team is larger than the cores the process may use): the threads draw QPs from a counter and unpack the
     * structs into the page-locked records; whoever completes a chunk submits it (copy in, solve, copy out on the chunk's own
     * stream, the kernels of different chunks share the SMs) and goes on unpacking the later chunks.  In the second region the
     * threads draw QPs again, wait for the chunk of their QP and pack its solution into the ocp_qp_out struct while the later
     * chunks are still being solved. */
    const int nchunk = n >= 512 ? 8 : 1, per = (n + nchunk - 1) / nchunk;
    int next = 0, done_cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0}, rc_all = CUIPM_OK;
    const int nthr = pack_threads();
#pragma omp parallel num_threads(nthr)
    {
        for (;;)
        {
            int i;
#pragma omp atomic capture seq_cst
            i = next++;
            if (i >= n) break;
            pack_qp(qp_in[i], l, qp + l->qp_stride * (size_t) i);
            if (opts->c.warm_start >= 2) pack_sol(qp_out[i], qp_in[i]->dim, l, sol + l->sol_stride * (size_t) i);
            const int c = i / per, lo = c * per, m = n - lo < per ? n - lo : per;
            int d;
#pragma omp atomic capture seq_cst
            d = ++done_cnt[c];
            if (d == m)
            {
                int rc = cuipm_solve_host_chunk(mem->solver, c, lo, m, qp, sol, infos, &opts->c);
                if (rc != CUIPM_OK)
                {
#pragma omp atomic write
                    rc_all = rc;
                }
            }
        }
    }
    if (rc_all != CUIPM_OK) { printf("\nerror: ocp_qp_cuipm_batch_solve: %s\n", cuipm_last_error()); exit(1); }
    next = 0;
#pragma omp parallel num_threads(nthr)
    {
        int waited = -1;
        for (;;)
        {
            int i;
#pragma omp atomic capture seq_cst
            i = next++;
            if (i >= n) break;
            const int c = i / per;
            if (c != waited)
            {
                if (cuipm_wait_chunk(mem->solver, c) != CUIPM_OK) { printf("\nerror: ocp_qp_cuipm_batch_solve: %s\n", cuipm_last_error()); exit(1); }
                waited = c;
            }
            hand_back(i, sol, infos, l, qp_in, qp_out, status_out);
        }
    }
    const double t_solve = acados_toc(&timer);
    const int worst = batch_result(n, qp_out, infos, t_solve);
    mem->info = infos[n - 1]; mem->status = infos[n - 1].status; mem->iter = infos[n - 1].iter; mem->time_qp_solver_call = t_solve;
    return worst;
}

/************************************************
 * the xcond chain as a batched entry (device condensing behind the C plugin)
 ************************************************/

struct ocp_qp_cuipm_xcond_batch
{
    cuipm_xcond *x;
    int *pool, **idxb_p, **rev_p;
    double *b_qp, *b_sol;
    cuipm_info *b_info;
    int b_cap;                  /* n_max of create: the most QPs a call may pass */
};

void ocp_qp_cuipm_xcond_batch_destroy(ocp_qp_cuipm_xcond_batch *c)
{
    if (!c) return;
    if (c->x) cuipm_xcond_destroy(c->x);
    staging_free(&c->b_qp, &c->b_sol, &c->b_info, &c->b_cap);
    free(c->pool); free(c->idxb_p); free(c->rev_p);
    free(c);
}

ocp_qp_cuipm_xcond_batch *ocp_qp_cuipm_xcond_batch_create(ocp_qp_in *in, int n_max, int cond_N, int device)
{
    const ocp_qp_dims *d = in->dim;
    if (d->nbue[0] > 0 || d->nge[0] > 0)
    {
        printf("\nerror: ocp_qp_cuipm_xcond_batch_create: only state-bound equalities at stage 0 are eliminated on the device\n");
        return NULL;
    }
    ocp_qp_cuipm_xcond_batch *c = calloc(1, sizeof(*c));
    c->pool = calloc(idx_pool_len(d) + 1, sizeof(int));
    c->idxb_p = calloc(d->N + 1, sizeof(int *));
    c->rev_p = calloc(d->N + 1, sizeof(int *));
    cuipm_shape sh = shape_from_in(in, c->pool, c->idxb_p, c->rev_p);
    /* equalities of stage 0: positions within [bu, bx, g] (d_ocp_qp.idxe, hpipm_d_ocp_qp.h:68) = positions in the bound list */
    c->x = cuipm_xcond_create(&sh, d->nbxe[0], in->idxe[0], cond_N, n_max, device);
    if (!c->x || !staging_grow(cuipm_xcond_full_layout(c->x), n_max, &c->b_qp, &c->b_sol, &c->b_info, &c->b_cap))
    {
        printf("\nerror: ocp_qp_cuipm_xcond_batch_create: %s\n", cuipm_last_error());
        ocp_qp_cuipm_xcond_batch_destroy(c);
        return NULL;
    }
    return c;
}

int ocp_qp_cuipm_xcond_batch_solve(ocp_qp_cuipm_xcond_batch *c, int n, ocp_qp_in **qp_in, ocp_qp_out **qp_out, void *opts_, int phase,
                                   int *status_out)
{
    ocp_qp_cuipm_opts *opts = opts_;
    if (!c || n < 0 || n > c->b_cap) { printf("\nerror: ocp_qp_cuipm_xcond_batch_solve: bad arguments\n"); exit(1); }
    if (n == 0) return ACADOS_SUCCESS;
    acados_timer timer;
    acados_tic(&timer);
    const cuipm_layout *l = cuipm_xcond_full_layout(c->x);
    const int nthr = pack_threads();
#pragma omp parallel for schedule(static) num_threads(nthr)
    for (int i = 0; i < n; i++) pack_qp(qp_in[i], l, c->b_qp + l->qp_stride * (size_t) i);
    int rc;
    if (phase == 1) rc = cuipm_xcond_condense_lhs_host(c->x, n, c->b_qp);
    else if (phase == 2) rc = cuipm_xcond_condense_rhs_and_solve_host(c->x, n, c->b_qp, c->b_sol, c->b_info, NULL, &opts->c);
    else rc = cuipm_xcond_solve_host(c->x, n, c->b_qp, c->b_sol, c->b_info, NULL, &opts->c);
    if (rc != CUIPM_OK) { printf("\nerror: ocp_qp_cuipm_xcond_batch_solve: %s\n", cuipm_last_error()); exit(1); }
    if (phase == 1) return ACADOS_SUCCESS;
    const double t_solve = acados_toc(&timer);
#pragma omp parallel for schedule(static) num_threads(nthr)
    for (int i = 0; i < n; i++) hand_back(i, c->b_sol, c->b_info, l, qp_in, qp_out, status_out);
    return batch_result(n, qp_out, c->b_info, t_solve);
}

/* drops the device solver and the batch staging, rebuilt on the next evaluate (ocp_qp_hpipm_memory_reset re-assigns its workspace) */
static void release(ocp_qp_cuipm_memory *mem)
{
    if (mem->solver) cuipm_destroy(mem->solver);
    mem->solver = NULL;
    mem->max_batch = 0;
    staging_free(&mem->b_qp, &mem->b_sol, &mem->b_info, &mem->b_cap);
}

void ocp_qp_cuipm_memory_reset(void *config_, void *qp_in_, void *qp_out_, void *opts_, void *mem_, void *work_)
{
    ocp_qp_cuipm_memory *mem = mem_;
    release(mem);
    mem->status = 0;
    mem->iter = 0;
}

void ocp_qp_cuipm_solver_get(void *config_, void *qp_in_, void *qp_out_, void *opts_, void *mem_, const char *field, int stage,
                             void *value, int size1, int size2)
{
    ocp_qp_in *qp_in = qp_in_;
    ocp_qp_cuipm_memory *mem = mem_;
    int nx = qp_in->dim->nx[stage], nu = qp_in->dim->nu[stage], e1 = 0, e2 = 0;
    if (!strcmp(field, "P")) { e1 = nx; e2 = nx; }
    else if (!strcmp(field, "p")) { e1 = nx; e2 = 1; }
    else if (!strcmp(field, "K")) { e1 = nu; e2 = nx; }
    else if (!strcmp(field, "k")) { e1 = nu; e2 = 1; }
    else if (!strcmp(field, "Lr")) { e1 = nu; e2 = nu; }
    else
    {
        printf("\nocp_qp_cuipm_solver_get: field %s not supported", field);
        return;
    }
    if (size1 != e1 || size2 != e2)
        printf("\nocp_qp_cuipm_solver_get: size of field %s not as expected, got size %d %d.\n", field, size1, size2);
    if (!mem->solver || cuipm_get_ric(mem->solver, 0, field, stage, (double *) value, e1, e2) != CUIPM_OK)
        printf("\nocp_qp_cuipm_solver_get: %s\n", mem->solver ? cuipm_last_error() : "no factorisation available (call evaluate first)");
}

/* Solution sensitivities with the factorisation of the last evaluate() on this memory (reference:
 * ocp_qp_hpipm_eval_forw_sens / _adj_sens, ocp_qp_hpipm.c:481-506 -> d_ocp_qp_ipm_sens_frw / _adj).  The QP of that
 * evaluate() is still resident on the device; only the seed travels. */
static void eval_sens(void *qp_in_, void *seed_, void *qp_out_, void *opts_, void *mem_, int adjoint)
{
    ocp_qp_in *qp_in = qp_in_;
    ocp_qp_seed *seed = seed_;
    ocp_qp_out *sens = qp_out_;
    ocp_qp_cuipm_opts *opts = opts_;
    ocp_qp_cuipm_memory *mem = mem_;
    if (mem->solver == NULL)
    {
        printf("\nerror: ocp_qp_cuipm_eval_%s_sens: no factorisation available, call evaluate first\n", adjoint ? "adj" : "forw");
        exit(1);
    }
    const ocp_qp_dims *d = qp_in->dim;
    const cuipm_layout *l = cuipm_get_layout(mem->solver);
    for (int k = 0; k <= d->N; k++)
    {
        int nc = 2 * (d->nb[k] + d->ng[k] + d->ns[k]);
        blasfeo_unpack_dvec(d->nu[k] + d->nx[k] + 2 * d->ns[k], seed->seed_g + k, 0, mem->seed_rec + l->off_ux[k], 1);
        if (k < d->N) blasfeo_unpack_dvec(d->nx[k + 1], seed->seed_b + k, 0, mem->seed_rec + l->off_pi[k], 1);
        blasfeo_unpack_dvec(nc, seed->seed_d + k, 0, mem->seed_rec + l->off_lam[k], 1);
        blasfeo_unpack_dvec(nc, seed->seed_m + k, 0, mem->seed_rec + l->off_t[k], 1);
    }
    int rc = cuipm_sens_host(mem->solver, 1, mem->seed_rec, mem->sens_rec, adjoint, &opts->c);
    if (rc != CUIPM_OK)
    {
        printf("\nerror: ocp_qp_cuipm_eval_%s_sens: %s\n", adjoint ? "adj" : "forw", cuipm_last_error());
        exit(1);
    }
    unpack_sol(mem->sens_rec, d, l, sens);
}

void ocp_qp_cuipm_eval_forw_sens(void *config_, void *qp_in, void *seed, void *qp_out, void *opts_, void *mem_, void *work_)
{
    eval_sens(qp_in, seed, qp_out, opts_, mem_, 0);
}

void ocp_qp_cuipm_eval_adj_sens(void *config_, void *qp_in, void *seed, void *qp_out, void *opts_, void *mem_, void *work_)
{
    eval_sens(qp_in, seed, qp_out, opts_, mem_, 1);
}

void ocp_qp_cuipm_terminate(void *config_, void *mem_, void *work_)
{
    if (mem_) release(mem_);
}

void ocp_qp_cuipm_config_initialize_default(void *config_)
{
    qp_solver_config *config = config_;
    config->dims_set = &ocp_qp_dims_set;
    config->opts_calculate_size = &ocp_qp_cuipm_opts_calculate_size;
    config->opts_assign = &ocp_qp_cuipm_opts_assign;
    config->opts_initialize_default = &ocp_qp_cuipm_opts_initialize_default;
    config->opts_update = &ocp_qp_cuipm_opts_update;
    config->opts_set = &ocp_qp_cuipm_opts_set;
    config->opts_get = &ocp_qp_cuipm_opts_get;
    config->memory_calculate_size = &ocp_qp_cuipm_memory_calculate_size;
    config->memory_assign = &ocp_qp_cuipm_memory_assign;
    config->memory_get = &ocp_qp_cuipm_memory_get;
    config->workspace_calculate_size = &ocp_qp_cuipm_workspace_calculate_size;
    config->evaluate = &ocp_qp_cuipm;
    config->solver_get = &ocp_qp_cuipm_solver_get;
    config->memory_reset = &ocp_qp_cuipm_memory_reset;
    config->eval_forw_sens = &ocp_qp_cuipm_eval_forw_sens;
    config->eval_adj_sens = &ocp_qp_cuipm_eval_adj_sens;
    config->terminate = &ocp_qp_cuipm_terminate;
}
