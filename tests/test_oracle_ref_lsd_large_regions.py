"""Frames whose LSD regions outgrow the part of the region list the GPU seed loop keeps in shared memory, pinned on the CPU.

k_lsd_grow_seq (cube_slam_b200/csrc/cs_lsd.cu) keeps the first LSD_SEQ_SCAP = 2 048 entries of a seed's region list in shared memory and the
rest in HBM; refine's re-grow is written behind the first pass, and reduce_region_radius swaps entries anywhere in the list.  Ordinary
frames barely reach that boundary, so these generators make frames that do: concentric rings (curved regions, which refine re-grows and
reduce-radius shrinks), sawtooth ramps (straight regions of thousands of pixels) and ramp bars in a flat frame (one region of a chosen
size).  For each frame the oracle equals the reference's own lsd.cpp (oracle/_ref/liblsd_ref.so) bit for bit, and the oracle's statistics
(oracle.lsd_stats) prove the frame still reaches the regime it exists for.  tests/test_gpu_lsd_large_regions.py runs the same frames on
the GPU."""
import numpy as np
import pytest

SPILL = 2048   # LSD_SEQ_SCAP


def rings(w, h, slope):
    """concentric rings around the frame centre: gray = floor(slope * radius) mod 256"""
    y, x = np.mgrid[0:h, 0:w]
    return (np.floor(slope * np.hypot(x - w / 2, y - h / 2)) % 256).astype(np.uint8)


def sawtooth(w, h, angle_deg, slope):
    """a ramp along the direction angle_deg, wrapping every 256 levels: gray = floor(slope * (x cos a + y sin a)) mod 256"""
    y, x = np.mgrid[0:h, 0:w]
    a = np.deg2rad(angle_deg)
    return (np.floor(slope * (x * np.cos(a) + y * np.sin(a))) % 256).astype(np.uint8)


def ramp_bar(w, h, bw, bh, slope, flat=90):
    """a bw x bh bar, centred in a flat frame, whose gray rises by `slope` per column"""
    img = np.full((h, w), flat, np.uint8)
    x0, y0 = (w - bw) // 2, (h - bh) // 2
    img[y0:y0 + bh, x0:x0 + bw] = (flat + slope * (np.arange(bw) - bw // 2))[None, :].clip(0, 255).astype(np.uint8)
    return img


def bgr(gray):
    """a BGR frame with the gray pattern in blue and green and three quarters of it in red"""
    return np.ascontiguousarray(np.stack([gray, gray, (gray.astype(np.int32) * 3 // 4).astype(np.uint8)], 2))


def frames():
    """name -> frame.  The exact-size frames were found by a search over ring slopes 5.0 .. 12.0 (step 0.1) on 320 x 240 and ramp bars of
    12 / 14 / 16 x 240 .. 319 pixels at slope 7 on 96 x 320, reading the oracle's counts of first passes and region lists of exactly
    2 047, 2 048 and 2 049 entries.  rings_sxga has a region list of exactly 2 048 entries made of a first pass and a re-grow (none of its
    first passes has 2 048 entries)."""
    return {
        "rings_vga": rings(640, 480, 6),
        "rings_sxga": rings(1280, 960, 10),
        "rings_vga_bgr": bgr(rings(640, 480, 7)),
        "saw0": sawtooth(640, 480, 0, 8),
        "saw30": sawtooth(640, 480, 30, 8),
        "saw30_bgr": bgr(sawtooth(640, 480, 30, 8)),
        "saw45": sawtooth(640, 480, 45, 8),
        "saw90": sawtooth(640, 480, 90, 8),
        "saw20_sxga": sawtooth(1280, 960, 20, 8),
        "bar_vga": ramp_bar(640, 480, 40, 400, 9),
        "first_2048": ramp_bar(96, 320, 16, 259, 7),
        "first_2049": rings(320, 240, 5.8),
        "first_2047": rings(320, 240, 7.8),
        "n_all_2047": rings(320, 240, 8.7),
    }


# the regime each frame exists for: statistic -> least value (an int) or exact value (a 1-tuple)
REGIMES = {
    "rings_vga": dict(n_all_spill=100, regrow_past=90, reduce_past=300, first_max=5000),
    "rings_sxga": dict(n_all_spill=800, regrow_past=700, reduce_past=100, n_all_2048=1, n_all_2049=1, first_2049=1, nfa_past_table=40),
    "rings_vga_bgr": dict(n_all_spill=100, regrow_past=100, reduce_past=200),
    "saw0": dict(n_all_spill=15, first_max=8000),
    "saw30": dict(n_all_spill=15, reduce_past=3, first_max=9000),
    "saw30_bgr": dict(n_all_spill=15, reduce_past=3),
    "saw45": dict(n_all_spill=15, first_max=11000, nfa_past_table=10, nfa_max_n=60000),
    "saw90": dict(n_all_spill=15, first_max=11000),
    "saw20_sxga": dict(n_all_spill=70, regrow_past=4, reduce_past=10, first_max=17000, nfa_max_n=500000, nfa_past_table=1),
    "bar_vga": dict(n_all_spill=1, first_max=6000),
    "first_2048": dict(first_2048=(1,), n_all_2048=(1,), first_max=(2048,)),
    "first_2049": dict(first_2049=1, n_all_2049=1),
    "first_2047": dict(first_2047=1),
    "n_all_2047": dict(n_all_2047=1),
}


@pytest.fixture(scope="module")
def stats(oracle):
    return {name: oracle.lsd_stats(img) for name, img in frames().items()}


def test_every_frame_reaches_its_regime(stats):
    for name, want in REGIMES.items():
        got = stats[name][1]
        for key, v in want.items():
            if isinstance(v, tuple):
                assert got[key] == v[0], (name, key, got)
            else:
                assert got[key] >= v, (name, key, got)
        # n_all counts the re-grow as well: never shorter than the longest first pass
        assert got["n_all_max"] >= got["first_max"] and got["seeds"] > 0


def test_exact_boundary_sizes_are_all_covered(stats):
    """first passes and region lists (n_all) of exactly 2 047, 2 048 and 2 049 entries: the last shared-memory entry, the first HBM one"""
    for key in ("first_2047", "first_2048", "first_2049", "n_all_2047", "n_all_2048", "n_all_2049"):
        assert sum(s[key] for _, s in stats.values()) >= 1, key


def test_raw_segments_equal_the_reference(oracle, stats):
    if not oracle.ref_lsd_available():
        pytest.skip("oracle/_ref/liblsd_ref.so not built")
    for name, img in frames().items():
        raw = stats[name][0]
        ref = oracle.ref_lsd_detect(img, cap=16384)
        assert len(raw) == len(ref) > 0, name
        np.testing.assert_array_equal(raw, ref, err_msg=name)


def test_statistics_change_no_result(oracle, stats):
    """lsd_stats is lsd_detect with counters: the same raw segments"""
    for name, img in frames().items():
        np.testing.assert_array_equal(stats[name][0], oracle.lsd_detect(img, 15.0, cap=16384)["raw_lines"], err_msg=name)


def test_the_old_giant_ramp_grows_no_region(oracle):
    """The shallow ramp an earlier GPU test used as its large region (0.35 gray levels per pixel) has a gradient modulus far below LSD's
    threshold of 2 / sin(22.5 deg) = 5.23: no pixel has a defined angle, no seed grows.  Hence the frames above."""
    ramp = np.ascontiguousarray(np.tile((np.arange(640) * 0.35).astype(np.uint8)[None, :], (480, 1)))
    raw, st = oracle.lsd_stats(ramp)
    assert len(raw) == 0 and st["seeds"] == 0


def test_nfa_entry_point_matches_the_detectors_forms(oracle):
    """orc_lsd_nfa: the early returns (break index -1), a tail that breaks, and the two first terms: every term of the tail scales by
    exp(log_gamma(n + 1) - (n + 1)), so the two values differ by that exponent over ln 10 (up to where the tail is cut off)"""
    import math
    assert oracle.lsd_nfa(0, 0, 0.125, 3.0) == (-3.0, -1)
    assert oracle.lsd_nfa(10, 0, 0.125, 3.0) == (-3.0, -1)
    v, b = oracle.lsd_nfa(10, 10, 0.125, 3.0)
    assert b == -1 and v == -3.0 - 10 * math.log10(0.125)
    v1, b1 = oracle.lsd_nfa(100, 30, 0.125, 10.0, True)
    v2, b2 = oracle.lsd_nfa(100, 30, 0.125, 10.0, False)
    assert 30 < b1 <= 101 and 30 < b2 <= 101
    assert abs((v1 - v2) - (math.lgamma(101) - 101) / math.log(10)) < 1e-3
    # underflow branch: exp(log1term) == 0 -> -log1term / ln 10 - logNT, break index -1
    v, b = oracle.lsd_nfa(100000, 90000, 0.125, 10.0)
    assert b == -1 and v > 1e4
    vs, bs = oracle.lsd_nfa_many([100, 100000, 10], [30, 90000, 10], 0.125, 10.0)
    assert list(bs) == [b1, -1, -1] and vs[0] == v1
