/* tests/host_core/once_per_device.cpp -- CS_ONCE_PER_DEVICE (cube_slam_b200/csrc/cs_kernels.h) entered by eight host threads at once, the
 * way the first batches of several contexts reach the same launcher.  Compiled against fake_cuda_slow_attr/cuda_runtime.h, whose
 * cudaFuncSetAttribute takes 50 ms before the value is in place.  After the macro, every thread must find the attribute set: a thread that
 * went on to launch while another was still setting it would launch with more dynamic shared memory than the device allows yet.  A second
 * round checks the other half of the contract: once the body has completed, no thread runs it again.  tests/test_once_per_device.py builds
 * and runs it, with -fsanitize=thread where the compiler has it.  Never shipped. */
#include "../../cube_slam_b200/csrc/cs_kernels.h"

#include <barrier>
#include <cstdio>
#include <thread>
#include <vector>

static void k_fake() {}

static void launcher()
{
    CS_ONCE_PER_DEVICE(cudaFuncSetAttribute(k_fake, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
}

/* n threads pass a barrier, then each calls launcher() and reports whether the attribute was in place when it returned */
static int round_of(int n)
{
    std::barrier sync(n);
    std::atomic<int> unset{0};
    std::vector<std::thread> th;
    for (int i = 0; i < n; i++)
        th.emplace_back([&] {
            sync.arrive_and_wait();
            launcher();
            if (fake_attr_value.load() != 128 * 1024) unset.fetch_add(1);
        });
    for (auto &t : th) t.join();
    return unset.load();
}

int main()
{
    const int n = 8;
    const int unset_first = round_of(n);
    const int calls_first = fake_attr_calls.load();
    const int unset_second = round_of(n);
    const int calls_second = fake_attr_calls.load() - calls_first;
    printf("first round: %d of %d threads found the attribute unset, %d calls; second round: %d unset, %d calls\n", unset_first, n, calls_first,
           unset_second, calls_second);
    return (unset_first == 0 && calls_first >= 1 && unset_second == 0 && calls_second == 0) ? 0 : 1;
}
