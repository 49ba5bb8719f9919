/*
 * cs_nfa.cuh -- the number-of-false-alarms test both line detectors end with, evaluated by a whole warp.
 *   LSD      nfa(n, k, p)  line_lbd/libs/lsd.cpp:1100-1136 (note its first term: (n + 1), not log_gamma(n + 1) -- the vendored file's own)
 *   EDLines  nfa(n, k, p)  line_lbd/include/line_lbd/line_descriptor/descriptor.hpp:763-830
 * Both are -log10(binomial tail) - logNT with the tail summed term by term until the remainder is provably below 10 % of the result.
 * Their cost on a GPU thread is the transcendental work: three log_gamma (seven log + seven pow each) and a pow + log10 per tail term.
 *   - log_gamma is only ever taken of small integers (n + 1, k + 1, n - k + 1): a table, built once on the host with the formulas and
 *     the libm the reference uses (cs_lgamma_host below), replaces it; larger arguments fall back to the device formula;
 *   - the tail's running products stay a sequential chain (two flops per term, in the reference's order), but the break test of 32
 *     consecutive terms (a pow and a log10 each) is evaluated by the 32 lanes at once.
 * Every lane returns the same value.
 */
#ifndef CS_NFA_CUH
#define CS_NFA_CUH

#include <float.h>
#include <math.h>

#define CS_LGAMMA_TABLE 16384

/* host: log_gamma exactly as the reference evaluates it (Windschitl above 15, Lanczos below) */
static inline double cs_lgamma_host(double x)
{
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
    const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * log(x + 5.5) - (x + 5.5);
    double b = 0.0;
    for (int n = 0; n < 7; n++) {
        a -= log(x + (double)n);
        b += q[n] * pow(x, (double)n);
    }
    return a + log(b);
}

#ifdef __CUDACC__
static __device__ __noinline__ double cs_lgamma_dev(double x)
{
    if (x > 15.0) return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
    const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * log(x + 5.5) - (x + 5.5);
    double b = 0.0;
    for (int n = 0; n < 7; n++) {
        a -= log(x + (double)n);
        b += q[n] * pow(x, (double)n);
    }
    return a + log(b);
}
/* log_gamma of the integer xi >= 1 */
__device__ __forceinline__ double cs_lgamma_int(const double *__restrict__ table, int xi)
{
    return (table && xi < CS_LGAMMA_TABLE) ? __ldg(table + xi) : cs_lgamma_dev((double)xi);
}
__device__ __forceinline__ bool cs_nfa_double_equal(double a, double b)
{
    if (a == b) return true;
    const double abs_diff = fabs(a - b);
    const double aa = fabs(a), bb = fabs(b);
    double abs_max = (aa > bb) ? aa : bb;
    if (abs_max < DBL_MIN) abs_max = DBL_MIN;
    return (abs_diff / abs_max) <= (100.0 * DBL_EPSILON);
}

/* all 32 lanes call with the same arguments; lsd_first_term selects lsd.cpp's (n + 1) in place of log_gamma(n + 1).  kBreak (cs_debug_nfa
 * only) also reports the i at which the tail loop stopped: n + 1 when it ran to the end, -1 for the early returns and the underflow branch. */
template <bool kBreak>
__device__ __forceinline__ double cs_nfa_warp_impl(const double *__restrict__ lgamma_table, int n, int k, double p, double logNT, bool lsd_first_term,
                                                   int *i_break)
{
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const double LN10 = 2.30258509299404568402, tolerance = 0.1;
    if (kBreak) *i_break = -1;
    if (n == 0 || k == 0) return -logNT;
    if (n == k) return -logNT - (double)n * log10(p);
    const double p_term = p / (1.0 - p);
    const double first = lsd_first_term ? ((double)n + 1) : cs_lgamma_int(lgamma_table, n + 1);
    const double log1term = first - cs_lgamma_int(lgamma_table, k + 1) - cs_lgamma_int(lgamma_table, n - k + 1) + (double)k * log(p) + (double)(n - k) * log(1.0 - p);
    double term = exp(log1term);
    if (cs_nfa_double_equal(term, 0.0)) {
        if ((double)k > (double)n * p) return -log1term / LN10 - logNT;
        return -logNT;
    }
    double bin_tail = term;
    if (kBreak) *i_break = n + 1;
    for (int i0 = k + 1; i0 <= n; i0 += 32) {
        const int i = i0 + lane;
        const bool valid = i <= n;
        /* this lane's factor; then the running product / sum up to and including its own term, in order */
        const double bin_term = valid ? (double)(n - i + 1) / (double)i : 0.0;
        const double mult_term = bin_term * p_term;
        double my_term = 0, my_tail = 0, t = term, s = bin_tail;
#pragma unroll 4
        for (int j = 0; j < 32; j++) {
            const double m = __shfl_sync(FULL, mult_term, j);
            t *= m;
            s += t;
            if (j == lane) {
                my_term = t;
                my_tail = s;
            }
        }
        bool brk = false;
        if (valid && bin_term < 1.0) {
            const double err = my_term * ((1.0 - pow(mult_term, (double)(n - i + 1))) / (1.0 - mult_term) - 1.0);
            brk = err < tolerance * fabs(-log10(my_tail) - logNT) * my_tail;
        }
        const unsigned hit = __ballot_sync(FULL, brk);
        const int n_valid = min(32, n - i0 + 1);
        const int src = hit ? (__ffs(hit) - 1) : (n_valid - 1);
        term = __shfl_sync(FULL, my_term, src);
        bin_tail = __shfl_sync(FULL, my_tail, src);
        if (hit) {
            if (kBreak) *i_break = i0 + src;
            break;
        }
    }
    return -log10(bin_tail) - logNT;
}

/* what the detectors call */
static __device__ __noinline__ double cs_nfa_warp(const double *__restrict__ lgamma_table, int n, int k, double p, double logNT, bool lsd_first_term)
{
    return cs_nfa_warp_impl<false>(lgamma_table, n, k, p, logNT, lsd_first_term, nullptr);
}
#endif /* __CUDACC__ */

#endif /* CS_NFA_CUH */
