// cuipm_internal.h -- declarations shared by the host and device translation units of libcuipm.
#ifndef CUIPM_INTERNAL_H_
#define CUIPM_INTERNAL_H_

#include <cstddef>
#include <string>

#include "cuipm.h"

namespace cuipm {
void set_error(const std::string &msg);
// CUIPM_OK if the option values are within what the device path implements, else CUIPM_ERR_INVALID (+ message)
int opts_check(const cuipm_opts *o);
// Dynamic shared memory (bytes) `kernel` may request per block on the current device: the device's opt-in limit less the
// kernel's static shared memory.  Returns CUIPM_OK or CUIPM_ERR_CUDA (+ message).
int smem_limit(const void *kernel, size_t *bytes);
// Sets the dynamic shared memory `kernel` may be launched with.  The attribute belongs to the kernel, not to a solver: objects of
// other shapes in the process may launch the same kernel with more or less, so it is set before every launch.
int set_dynamic_smem(const void *kernel, size_t bytes);
// Sets the message "<what>: <CUDA error string of err (a cudaError_t)>" and returns CUIPM_ERR_CUDA.
int cuda_error(const std::string &what, int err);
// The solver's statistics buffer, grown to at least n doubles (the old one is freed after the solver's stream has drained);
// null (+ message) if that fails.
double *stat_buffer(cuipm_solver *s, size_t n);
}  // namespace cuipm

namespace cuipm_asm { struct Stage; }
// the assembly's part of an xcond object (cuipm_assemble.cu): its stage table from the full shape; freed with its device tables
int asm_init(cuipm_xcond *x, const cuipm_shape *full);
void asm_free(cuipm_xcond *x);

// the xcond object (cuipm_xcond.cu; cuipm_assemble.cu writes its records)
struct cuipm_xcond
{
    int device = 0, max_batch = 0, cond_N = 0;
    cuipm_reducer *red = nullptr;
    cuipm_condenser *cond = nullptr;
    cuipm_solver *solver = nullptr;                    // its device buffers hold the records, solutions and summaries it solves
    const cuipm_layout *lf = nullptr, *lr = nullptr;
    double *d_full = nullptr, *d_sol_full = nullptr;   // host entries only: allocated at the first one
    double *d_red = nullptr, *d_sol_red = nullptr;     // condensing only
    int lhs_valid = 0;
    cuipm_asm::Stage *asm_st = nullptr;                // the assembly's stage table of the full shape (N+1 entries), no sources
    void *d_asm = nullptr;                             // device copy of the assembly's tables
    size_t asm_bytes = 0;
};

// CUDA runtime call in a function that returns a cuipm status: on failure, the message names the call
#define CK(call) do { const cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuipm::cuda_error(#call, (int) e_); } while (0)

#endif
