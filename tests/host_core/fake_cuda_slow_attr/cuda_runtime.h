/* tests/host_core/fake_cuda_slow_attr/cuda_runtime.h -- stands in for <cuda_runtime.h> when tests/host_core/once_per_device.cpp compiles
 * cube_slam_b200/csrc/cs_kernels.h for the host.  Only what that header needs, and one call with behaviour: cudaFuncSetAttribute takes about
 * 50 ms, as a first call into the driver can, and only then records the value it was given (fake_attr_value) and counts the call
 * (fake_attr_calls).  A thread that launches while another is still inside it would see the attribute unset.  cudaGetDevice returns 0.
 * Never shipped. */
#ifndef CS_TEST_FAKE_CUDA_SLOW_ATTR_H
#define CS_TEST_FAKE_CUDA_SLOW_ATTR_H
#include <atomic>
#include <chrono>
#include <cstddef>
#include <thread>

typedef int cudaError_t;
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
struct int2 {
    int x, y;
};
struct int4 {
    int x, y, z, w;
};
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
enum cudaDeviceAttr { cudaDevAttrMaxSharedMemoryPerBlockOptin = 97 };
enum { cudaSuccess = 0 };
struct cudaFuncAttributes {
    size_t sharedSizeBytes = 0;
};

inline std::atomic<int> fake_attr_value{0}, fake_attr_calls{0};

static inline cudaError_t cudaGetDevice(int *d)
{
    *d = 0;
    return 0;
}
template <typename K> static inline cudaError_t cudaFuncGetAttributes(cudaFuncAttributes *a, K)
{
    a->sharedSizeBytes = 0;
    return 0;
}
static inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr, int)
{
    *v = 232448;
    return 0;
}
template <typename K> static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int value)
{
    std::this_thread::sleep_for(std::chrono::milliseconds(50));
    fake_attr_value.store(value);
    fake_attr_calls.fetch_add(1);
    return 0;
}
#endif
