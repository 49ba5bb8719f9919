"""CS_ONCE_PER_DEVICE (cube_slam_b200/csrc/cs_kernels.h) under concurrent first use, without a GPU: eight host threads pass a barrier and enter
the same once-per-device site, whose body (cudaFuncSetAttribute, from tests/host_core/fake_cuda_slow_attr/cuda_runtime.h) takes 50 ms before
the value is in place.  Every thread must find the attribute set when the macro returns -- the launchers go on to launch with more than 48 KB
of dynamic shared memory, which fails before the limit has been raised -- and once the body has completed, no later call may run it again.
tests/host_core/once_per_device.cpp is the harness; with ThreadSanitizer where this g++ links it."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def test_no_thread_passes_the_once_per_device_site_before_its_body_has_run():
    src = os.path.join(HERE, "host_core", "once_per_device.cpp")
    bdir = os.path.join(HERE, "host_core", "_build")
    os.makedirs(bdir, exist_ok=True)
    probe = subprocess.run(["g++", "-fsanitize=thread", "-x", "c++", "-", "-o", os.path.join(bdir, "tsan_probe")], input="int main(){return 0;}", text=True,
                           capture_output=True)
    san = ["-fsanitize=thread"] if probe.returncode == 0 else []
    exe = os.path.join(bdir, "once_per_device")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-g", "-pthread", "-I", os.path.join(HERE, "host_core", "fake_cuda_slow_attr"), "-o", exe, src] + san)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out[-3000:]
    assert "first round: 0 of 8 threads found the attribute unset" in out and "second round: 0 unset, 0 calls" in out, out[-3000:]
    assert "ThreadSanitizer" not in out, out[-3000:]
