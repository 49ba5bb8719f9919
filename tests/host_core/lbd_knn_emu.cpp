/* tests/host_core/lbd_knn_emu.cpp -- the SOURCE of the knn / radius matching kernels (k_lbd_knn2, k_lbd_match_sorted in
 * cube_slam_b200/csrc/cs_lbd_kernels.cuh) compiled for the host against the emulation of the CUDA execution model in cuda_emu.h (a
 * std::thread per CUDA thread, a std::barrier for __syncthreads, function-local statics for __shared__ and for the sorting kernel's
 * dynamic shared memory) and run launch by launch through the launch wrappers the library uses.  tests/test_lbd_knn_host_emu.py compares
 * what the launches write with the oracle.  Test infrastructure, never shipped.  g++ -std=c++20 -O2 -ffp-contract=off -pthread. */
#include "cuda_emu.h"

#include "../../cube_slam_b200/csrc/cs_lbd_core.h"
namespace {
#include "../../cube_slam_b200/csrc/cs_lbd_kernels.cuh"
}

/* k_lbd_knn2<<<n_queries, 128>>>; q_all / t_all 16-byte aligned like device memory */
extern "C" void emu_lbd_knn2(const void *q_all, const void *t_all, const int32_t *pair_of_query, const int32_t *t_off, int n_queries, unsigned long long *keys2)
{
    launch_lbd_knn2((unsigned)n_queries, nullptr, (const uint4 *)q_all, (const uint4 *)t_all, pair_of_query, t_off, n_queries, keys2);
}

/* k_lbd_match_sorted<<<n_queries, 256>>>; keys == NULL: the counting launch */
extern "C" void emu_lbd_match_sorted(const void *q_all, const void *t_all, const int32_t *pair_of_query, const int32_t *t_off, int n_queries, int max_dist,
                                     const long long *out_off, unsigned long long *keys, int32_t *counts)
{
    launch_lbd_match_sorted((unsigned)n_queries, nullptr, 0, (const uint4 *)q_all, (const uint4 *)t_all, pair_of_query, t_off, n_queries, max_dist, out_off, keys,
                            counts);
}

extern "C" int emu_lbd_knn_max_train() { return CS_LBD_KNN_MAX_TRAIN; }
