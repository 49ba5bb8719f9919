"""shim/lsd_detector_b200.cpp without a GPU.

It compiles: against the reference's own descriptor.hpp with oracle/ref/fakecv standing in for OpenCV (every member LSDDetector.cpp defines is
defined), and with neither on the include path (the guard leaves an empty translation unit).  And it runs: the shim and its driver
(shim/test/lsd_detector_shim_driver.cpp), linked next to the reference's other line_lbd sources and against a host stand-in of
libcubeslam_b200.so (tests/host_core/lsd_octaves_standin.cpp: cs_detect_raw_lines_octaves_batch answered by the CPU oracle's pyramid, LSD and
KeyLine fill, CS_ERR_CAPACITY on demand), equal the reference's own LSDDetector (oracle/_ref/libref_lsd_detector.so) in everything but the
device: grouping and packing, the mask rule, append semantics, the flag flips and their messages, the exceptions and the capacity retry."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_gpu_lsd_detector_shim as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")
SRC = os.path.join(ROOT, "shim", "lsd_detector_b200.cpp")
REF = "/root/reference/line_lbd"
MEMBERS = ("LSDDetector::createLSDDetector()", "LSDDetector::computeGaussianPyramid(", "LSDDetector::detectImpl(")


def _cxx():
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("no g++")
    return cxx


def test_guard_leaves_an_empty_translation_unit(tmp_path):
    out = str(tmp_path / "l.o")
    r = subprocess.run([_cxx(), "-std=c++14", "-Wall", "-c", SRC, "-o", out, "-I", os.path.join(ROOT, "include")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "LSDDetector" not in subprocess.run(["nm", "-C", out], capture_output=True, text=True).stdout


def test_body_compiles_against_the_reference_header_and_defines_every_member(tmp_path):
    if not os.path.isdir(os.path.join(REF, "include")):
        lib = G.SHIM
        if not os.path.exists(lib) or not shutil.which("nm"):
            pytest.skip("needs the reference checkout's headers, or oracle/_ref/libshim_lsd.so that build() compiles from them")
        syms = subprocess.run(["nm", "-C", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    else:
        out = str(tmp_path / "l.o")
        r = subprocess.run([_cxx(), "-std=c++14", "-Wall", "-Wextra", "-c", SRC, "-o", out, "-I", os.path.join(ROOT, "include"), "-I",
                            os.path.join(ROOT, "oracle", "ref", "fakecv"), "-I", os.path.join(REF, "include")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        shim_warnings = [l for l in r.stderr.splitlines() if "lsd_detector_b200.cpp" in l and "warning" in l]
        assert not shim_warnings, shim_warnings
        syms = subprocess.run(["nm", "-C", "--defined-only", out], capture_output=True, text=True).stdout
    syms = "\n".join(l for l in syms.splitlines() if " T " in l)
    for m in MEMBERS:
        assert m in syms, m
    assert syms.count("LSDDetector::detect(") == 3                           # the flat, the per-octave and the vector overload


@pytest.fixture(scope="module")
def host(oracle):
    """(shim on the host stand-in, the reference's own LSDDetector)"""
    if not os.path.isdir(os.path.join(REF, "include")):
        pytest.skip("needs the reference checkout (its headers and line_lbd sources); the shim runs on the GPU in tests/test_gpu_lsd_detector_shim.py")
    if not os.path.exists(G.REF):
        pytest.skip("oracle/_ref/libref_lsd_detector.so is built by build() where the reference checkout exists")
    out = os.path.join(HERE, "host_core", "_build", "libshim_lsd_standin.so")
    orc = os.path.abspath(os.path.join(ROOT, "oracle", "_build"))
    ref_srcs = [os.path.join(REF, f) for f in ("libs/lsd.cpp", "libs/binary_descriptor.cpp", "libs/binary_descriptor_matcher.cpp", "class/line_lbd_allclass.cpp")]
    srcs = [SRC, os.path.join(ROOT, "shim", "test", "lsd_detector_shim_driver.cpp"), os.path.join(HERE, "host_core", "lsd_octaves_standin.cpp")]
    deps = srcs + ref_srcs + [os.path.join(ROOT, "include", "cube_slam_b200.h"), os.path.join(orc, "liboracle.so")]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call([_cxx(), "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-w", "-ffp-contract=off", "-fno-fast-math", "-DLSDD_VIEWS",
                               "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle", "ref", "fakecv"), "-I", os.path.join(REF, "include"),
                               "-o", out] + srcs + ref_srcs + ["-L", orc, "-loracle", "-Wl,-rpath," + orc])
    shim, ref = G.Driver(out), G.Driver(G.REF)
    shim.L.lsdd_cout_on()
    ref.L.lsdd_cout_on()
    shim.L.standin_reset()
    return shim, ref


def test_frames_and_octave_counts_on_the_stand_in(host, fixture_a, fixture_b):
    G.check_frames(*host, [("fixture A", fixture_a["img"]), ("fixture B 9", fixture_b["frames"][9][0]), ("211x97 gray", G.synthetic(211, 97, True))])


def test_masks_prefilled_vectors_and_flags_on_the_stand_in(host, fixture_b, capfd):
    img, boxes = fixture_b["frames"][17]
    G.check_masks(*host, img, boxes, np.random.default_rng(21), capfd=capfd, octaves=(2,))
    G.check_mask_errors(*host, img)


def test_vector_overload_on_the_stand_in(host, fixture_b):
    frames = [fixture_b["frames"][0][0], G.synthetic(211, 97, True, 2), G.synthetic(333, 251, False, 3)]
    G.check_vector(*host, frames, np.random.default_rng(22), K=2, n=12)


def test_roi_counts_depth_and_outside_points_on_the_stand_in(host, fixture_a):
    G.check_roi(*host, fixture_a["img"])
    G.check_counts_and_depth(*host, fixture_a["img"], np.random.default_rng(23))
    G.check_outside_points_are_kept(host[0], fixture_a["img"])


def test_capacity_retry_on_the_stand_in(host, fixture_a):
    """the stand-in answers CS_ERR_CAPACITY until the buffer holds 9 000 lines per octave: the drop-in doubles its buffer (2 048, 4 096,
    8 192, 16 384) and answers what the reference answers; a checkerboard past 2 048 segments needs no knob"""
    shim, ref = host
    shim.L.standin_reset()
    shim.L.standin_fail_below(9000)
    try:
        G.run_both(shim, ref, G.FLAT, fixture_a["img"], 2, 2, what="forced capacity")
        assert shim.L.standin_calls() == 4 and shim.L.standin_last_cap() == 16384
    finally:
        shim.L.standin_reset()
    G.check_capacity(shim, ref)
    assert shim.L.standin_calls() == 4                                     # 2 048 then 4 096, at 1 and at 2 octaves


def test_reference_line_lbd_detect_over_the_drop_in_on_the_stand_in(host, fixture_a):
    G.check_line_lbd(*host, fixture_a["img"], octaves=(1, 3))
