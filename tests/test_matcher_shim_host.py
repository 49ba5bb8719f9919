"""shim/binary_descriptor_matcher_b200.cpp without a GPU.

It compiles: against the reference's own descriptor.hpp with oracle/ref/fakecv standing in for OpenCV (the whole body, every member a caller
reaches defined), and with neither on the include path (the guard leaves an empty translation unit).  And its pairwise forms run: the shim
and its driver (shim/test/matcher_shim_driver.cpp), linked next to the reference's other line_lbd sources and against the emulated build of
cs_lbd.cu (tests/host_core/lbd_host_emu.cpp, the kernels under the CUDA execution-model emulation), answer the GPU test's pairwise cases
on the CPU.  The emulated build has no collection (tests/host_core/lbd_collection_absent.cpp), so the collection forms run on the GPU only."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")
SRC = os.path.join(ROOT, "shim", "binary_descriptor_matcher_b200.cpp")
REF = "/root/reference/line_lbd"
MEMBERS = ("BinaryDescriptorMatcher::BinaryDescriptorMatcher()", "BinaryDescriptorMatcher::createBinaryDescriptorMatcher()",
           "BinaryDescriptorMatcher::add(", "BinaryDescriptorMatcher::train()", "BinaryDescriptorMatcher::clear()")


def _cxx():
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("no g++")
    return cxx


def test_guard_leaves_an_empty_translation_unit(tmp_path):
    out = str(tmp_path / "m.o")
    r = subprocess.run([_cxx(), "-std=c++14", "-Wall", "-c", SRC, "-o", out, "-I", os.path.join(ROOT, "include")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "BinaryDescriptorMatcher" not in subprocess.run(["nm", "-C", out], capture_output=True, text=True).stdout


def test_body_compiles_against_the_reference_header_and_defines_every_member(tmp_path):
    if not os.path.isdir(os.path.join(REF, "include")):
        lib = os.path.join(ROOT, "oracle", "_ref", "libshim_matcher.so")
        if not os.path.exists(lib) or not shutil.which("nm"):
            pytest.skip("needs the reference checkout's headers, or oracle/_ref/libshim_matcher.so that build() compiles from them")
        syms = subprocess.run(["nm", "-C", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    else:
        out = str(tmp_path / "m.o")
        r = subprocess.run([_cxx(), "-std=c++14", "-Wall", "-Wextra", "-c", SRC, "-o", out, "-I", os.path.join(ROOT, "include"), "-I",
                            os.path.join(ROOT, "oracle", "ref", "fakecv"), "-I", os.path.join(REF, "include")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        shim_warnings = [l for l in r.stderr.splitlines() if "binary_descriptor_matcher_b200.cpp" in l and "warning" in l]
        assert not shim_warnings, shim_warnings
        syms = subprocess.run(["nm", "-C", "--defined-only", out], capture_output=True, text=True).stdout
    syms = "\n".join(l for l in syms.splitlines() if " T " in l)             # the functions the object exports
    for m in MEMBERS:
        assert m in syms, m
    for m in ("match(", "knnMatch(", "radiusMatch("):
        assert syms.count("BinaryDescriptorMatcher::" + m) == 2, m          # the pairwise and the collection form
    assert "Mihasher::" not in syms                                         # no hash on the host


@pytest.fixture(scope="module")
def emu_shim(oracle):
    if not os.path.isdir(os.path.join(REF, "include")):
        pytest.skip("needs the reference checkout (its headers and line_lbd sources); the shim runs on the GPU in tests/test_gpu_matcher_shim.py")
    import test_gpu_matcher_shim as G
    out = os.path.join(HERE, "host_core", "_build", "libshim_matcher_emu.so")
    orc = os.path.abspath(os.path.join(ROOT, "oracle", "_build"))
    ref_srcs = [os.path.join(REF, f) for f in ("libs/lsd.cpp", "libs/LSDDetector.cpp", "libs/binary_descriptor.cpp", "class/line_lbd_allclass.cpp")]
    srcs = [SRC, os.path.join(ROOT, "shim", "test", "matcher_shim_driver.cpp"), os.path.join(HERE, "host_core", "lbd_host_emu.cpp"),
            os.path.join(HERE, "host_core", "lbd_collection_absent.cpp")]
    deps = srcs + ref_srcs + [os.path.join(ROOT, "cube_slam_b200", "csrc", f) for f in ("cs_lbd.cu", "cs_lbd_core.h", "cs_lbd_kernels.cuh")] + \
        [os.path.join(ROOT, "include", "cube_slam_b200.h"), os.path.join(HERE, "host_core", "cuda_emu.h")]
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++20", "-O2", "-fPIC", "-shared", "-pthread", "-w", "-ffp-contract=off", "-fno-fast-math", "-DCS_EMU_WITH_SHIM_GLUE",
                               "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "oracle", "ref", "fakecv"), "-I", os.path.join(REF, "include"),
                               "-o", out] + srcs + ref_srcs + ["-L", orc, "-loracle", "-Wl,-rpath," + orc])
    return G, G.Shim(out)


def test_pairwise_forms_on_the_emulated_library(emu_shim, oracle, fixture_b):
    """match / knnMatch / radiusMatch of the pairwise form with and without a mask, both compactResult, against the reference's own matcher
    and the documented answer: planted ties, and LBD codes of two golden frames (the CPU oracle's descriptors, which the GPU's equal)"""
    from test_oracle_ref_lbd_knn import _planted
    G, shim = emu_shim
    rng = np.random.default_rng(41)
    m = shim.new()
    try:
        q, t = _planted(rng, 10, 70)
        G.check_pairwise(shim, m, q, t, rng)
        descs = []
        for f in (0, 9):
            img = fixture_b["frames"][f][0]
            descs.append(oracle.lbd_compute(img, oracle.lbd_detect_keylines(img, True, 15.0)))
        G.check_pairwise(shim, m, descs[0][:12], descs[1], rng, ks=(1, 2, None), radii=(25.0,))
    finally:
        shim.L.shim_bdm_free(m)


def test_reference_constructor_bdm_and_input_errors_on_the_emulated_library(emu_shim, oracle, capfd):
    """line_lbd_detect's own constructor makes the shim's matcher its bdm; the pairwise input errors print or throw as on the GPU"""
    from test_oracle_ref_lbd_knn import _planted
    G, shim = emu_shim
    rng = np.random.default_rng(42)
    q, t = _planted(rng, 8, 50)
    det = shim.L.shim_detector_new()
    try:
        m = shim.L.shim_detector_bdm(det)
        G.check_pairwise(shim, m, q, t, rng, ks=(1, 3), radii=(25.0,))
        shim.L.shim_cout_on()
        capfd.readouterr()
        assert shim.query(m, G.KNN, q[:0], t, k=2) == [] and "descriptors matrices cannot be void" in capfd.readouterr().out
        assert shim.query(m, G.KNN, q, t, k=2, mask=np.ones((len(q), 2))) == []
        assert "input mask should have %d rows and 1 column" % len(q) in capfd.readouterr().out
        assert shim.query(m, G.KNN, q, t, k=-1) == -1
        assert shim.L.shim_bdm_wrong_shape(m, 1) == 1
    finally:
        shim.L.shim_detector_free(det)


def test_built_harness_shares_the_process_cpp_runtime_and_prints_numbers(oracle, capfd):
    """oracle/_ref/libshim_matcher.so links the shared libstdc++ (a private static copy's locale facets are unknown to the process's
    std::cout, and printing a number through them crashes), and the messages the matcher prints where the reference does -- row counts
    included -- come out with the oracle's reference libraries loaded in the same process.  These input errors return before any device
    work, so this runs without a GPU."""
    import test_gpu_matcher_shim as G
    from oracle import pyoracle_knn as K
    if not os.path.exists(G.SHIM) or not shutil.which("readelf"):
        pytest.skip("oracle/_ref/libshim_matcher.so is built by build() where the reference checkout exists")
    needed = subprocess.run(["readelf", "-d", G.SHIM], capture_output=True, text=True).stdout
    assert "libstdc++.so.6" in needed
    if K.ref_available():
        K._ref_knn()                                                        # switches std::cout off as it loads
    shim = G.Shim(G.SHIM)
    m = shim.new()
    try:
        q = np.random.default_rng(43).integers(0, 256, (16, 32), dtype=np.uint8)
        shim.L.shim_cout_on()
        capfd.readouterr()
        assert shim.query(m, G.KNN, q, q, k=2, mask=np.ones((16, 2))) == []
        assert "input mask should have 16 rows and 1 column" in capfd.readouterr().out
        assert shim.query(m, G.MATCH, q, q, mask=np.ones((3, 2))) == []
        assert "input mask should have 16 rows and 1 column" in capfd.readouterr().out
    finally:
        shim.L.shim_bdm_free(m)
