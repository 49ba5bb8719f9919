/* cs_debug_atan2: the device side of cs_pmath.h, exposed so that a test can check it against the host evaluation bit for bit.
 * cs_debug_nfa: the line detectors' NFA (cs_nfa.cuh) on given (n, k, p), so that a test can check it against the reference's formula. */
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "cs_internal.h"
#include "cs_nfa.cuh"
#include "cs_pmath.h"

namespace {
__global__ void k_debug_atan2(const double *__restrict__ y, const double *__restrict__ x, double *__restrict__ out, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = cs_pm_atan2(y[i], x[i]);
}

/* one warp per triple: the value from cs_nfa_warp as the detectors call it, the break index from the same body instantiated to report it */
__global__ void k_debug_nfa(const double *__restrict__ lgam, const int32_t *__restrict__ n, const int32_t *__restrict__ k, const double *__restrict__ p,
                            double logNT, bool lsd_first_term, double *__restrict__ value, int32_t *__restrict__ brk, int count)
{
    const int w = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    if (w >= count) return; /* whole warps */
    const double v = cs_nfa_warp(lgam, n[w], k[w], p[w], logNT, lsd_first_term);
    int b = 0;
    cs_nfa_warp_impl<true>(lgam, n[w], k[w], p[w], logNT, lsd_first_term, &b);
    if ((threadIdx.x & 31) == 0) {
        value[w] = v;
        brk[w] = b;
    }
}
}  // namespace

extern "C" int cs_debug_atan2(cs_ctx *c, const double *y, const double *x, double *out, int n)
{
    if (!c || !y || !x || !out || n < 0) return CS_ERR_INVALID_ARG;
    if (n == 0) return CS_OK;
    cudaSetDevice(cs_ctx_device(c));
    double *d = nullptr;
    if (cudaMalloc(&d, (size_t)n * 24) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMalloc failed");
    cudaMemcpy(d, y, (size_t)n * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d + n, x, (size_t)n * 8, cudaMemcpyHostToDevice);
    k_debug_atan2<<<(n + 255) / 256, 256>>>(d, d + n, d + 2 * (size_t)n, n);
    cudaMemcpy(out, d + 2 * (size_t)n, (size_t)n * 8, cudaMemcpyDeviceToHost);
    const cudaError_t e = cudaGetLastError();
    cudaFree(d);
    return e == cudaSuccess ? CS_OK : cs_ctx_fail(c, CS_ERR_CUDA, "cs_debug_atan2 failed: %s", cudaGetErrorString(e));
}

extern "C" int cs_debug_nfa(cs_ctx *c, const int32_t *n, const int32_t *k, const double *p, double logNT, int lsd_first_term, double *out_value,
                            int32_t *out_break, int count)
{
    if (!c || !n || !k || !p || !out_value || !out_break || count < 0) return CS_ERR_INVALID_ARG;
    if (count == 0) return CS_OK;
    cudaSetDevice(cs_ctx_device(c));
    /* the log_gamma table as the detectors build it (cs_lsd.cu, cs_edlines.cu) */
    std::vector<double> t(CS_LGAMMA_TABLE, 0.0);
    for (int i = 1; i < CS_LGAMMA_TABLE; i++) t[i] = cs_lgamma_host((double)i);
    const size_t cnt = (size_t)count, tb = (size_t)CS_LGAMMA_TABLE * 8;
    char *d = nullptr;
    if (cudaMalloc(&d, tb + cnt * 32) != cudaSuccess) return cs_ctx_fail(c, CS_ERR_CUDA, "cudaMalloc failed");
    double *d_lgam = (double *)d, *d_p = (double *)(d + tb), *d_val = d_p + cnt;
    int32_t *d_n = (int32_t *)(d_val + cnt), *d_k = d_n + cnt, *d_brk = d_k + cnt;
    cudaMemcpy(d_lgam, t.data(), tb, cudaMemcpyHostToDevice);
    cudaMemcpy(d_n, n, cnt * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_k, k, cnt * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_p, p, cnt * 8, cudaMemcpyHostToDevice);
    k_debug_nfa<<<(unsigned)((cnt * 32 + 255) / 256), 256>>>(d_lgam, d_n, d_k, d_p, logNT, lsd_first_term != 0, d_val, d_brk, count);
    cudaMemcpy(out_value, d_val, cnt * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(out_break, d_brk, cnt * 4, cudaMemcpyDeviceToHost);
    const cudaError_t e = cudaGetLastError();
    cudaFree(d);
    return e == cudaSuccess ? CS_OK : cs_ctx_fail(c, CS_ERR_CUDA, "cs_debug_nfa failed: %s", cudaGetErrorString(e));
}

/* the host evaluation of the same header (what a C++ caller of the library would get) */
extern "C" double cs_atan2_host(double y, double x) { return cs_pm_atan2(y, x); }
