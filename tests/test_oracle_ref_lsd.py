"""The LSD oracle (oracle/lsd_oracle.cpp) against the REFERENCE'S OWN lsd.cpp, compiled from /root/reference into
oracle/_ref/liblsd_ref.so (oracle/Makefile target `ref`, oracle/ref/lsd_ref.cpp + minicv.hpp: the reference file is included from
where it lies, nothing of it is copied).  Raw segments -- createLineSegmentDetector(LSD_REFINE_ADV)->detect(gray), what
LSDDetector::detectImpl (line_lbd/libs/LSDDetector.cpp:120-170) gets for octave 0 -- must be equal bit for bit, count and order.

The library exists where the reference checkout was present at build time (it travels to the GPU box with the snapshot); without it these
tests skip, and tests/test_goldens_sequence.py still pins the oracle to the reference through the recorded `raw_checksum_ref`."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.ref_lsd_available():
        pytest.skip("oracle/_ref/liblsd_ref.so not built (no /root/reference on this machine)")
    return oracle


def _same(ref, img, cap=8192):
    got = ref.lsd_detect(img, 15.0, cap=cap)["raw_lines"]
    want = ref.ref_lsd_detect(img, cap=cap)
    assert got.shape == want.shape
    np.testing.assert_array_equal(got, want)
    return len(want)


def test_demo_frame(ref, fixture_a):
    assert _same(ref, fixture_a["img"]) == 450


def test_sequence_frames(ref, fixture_b):
    for i in range(0, len(fixture_b["frames"]), 7):
        assert _same(ref, fixture_b["frames"][i][0]) > 0


@pytest.mark.parametrize("seed,w,h,kind", [(7, 640, 480, "indoor"), (8, 1242, 375, "kitti")])
def test_synthetic_frames(ref, seed, w, h, kind):
    from cube_slam_b200 import synthetic as S
    imgs = S.make_batch(seed, 2, w, h, 3, kind=kind, poisson=(kind == "indoor"))[0]
    for f in range(2):
        assert _same(ref, imgs[f]) > 50


def odd_and_degenerate_frames():
    """Named frames where LSD implementations part ways: ragged sizes (the 0.8 resize rounds differently), noise (thousands of seeds, few
    accepted), a constant frame (no defined pixel), sharp rectangles (long regions, the reduce-radius / refine branches) and a blurred disc
    (curved regions that fail the density test and get cut).  tests/test_gpu_*_parity.py run the same frames."""
    rng = np.random.default_rng(5)
    out = {}
    for shape in [(97, 211), (61, 64), (200, 333)]:
        out["noise_%dx%d" % shape] = rng.integers(0, 256, shape, dtype=np.uint8)
    out["constant"] = np.full((120, 160), 77, np.uint8)
    img = np.full((240, 320), 30, np.uint8)
    img[40:200, 60:260] = 200
    img[90:150, 120:180] = 90
    img += rng.integers(0, 6, img.shape, dtype=np.uint8)
    out["rectangles"] = img
    yy, xx = np.mgrid[:300, :300]
    disc = (np.hypot(yy - 150, xx - 150) < 100).astype(np.float64) * 180 + 40
    out["disc"] = np.clip(disc + rng.normal(0, 2, disc.shape), 0, 255).astype(np.uint8)
    return out


def test_odd_sizes_and_degenerate_images(ref):
    frames = odd_and_degenerate_frames()
    for shape in [(97, 211), (61, 64), (200, 333)]:
        _same(ref, frames["noise_%dx%d" % shape])
    assert _same(ref, frames["constant"]) == 0
    assert _same(ref, frames["rectangles"]) >= 6
    _same(ref, frames["disc"])


def checkerboard(w, h, cell, lo, hi, noise=0, seed=0):
    """A w x h (uint8) checkerboard of cell x cell squares of the levels lo and hi, plus uniform noise in [0, noise): thousands of short
    line-support regions, as tiled floors, shelves and facades give."""
    yy, xx = np.mgrid[:h, :w]
    img = np.where((yy // cell + xx // cell) % 2 == 0, lo, hi).astype(np.int32)
    if noise:
        img += np.random.default_rng(seed).integers(0, noise, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


# 2 850 and 13 564 raw LSD segments: more candidate rectangles per frame than the GPU seed loop's initial hand-off buffer (2 048) holds
CHECKERBOARDS = {"vga_10px": (640, 480, 10, 0, 255), "sxga_12px_noisy": (1280, 960, 12, 40, 200, 6)}


def tiny_frame(h, w, seed):
    """An h x w step edge (a dark left half, a bright right one) with a little noise."""
    img = np.full((h, w), 60, np.uint8)
    img[:, w // 2:] = 190
    return img + np.random.default_rng(seed).integers(0, 8, (h, w), dtype=np.uint8)


# down to 3 x 3 (0.8 x 3 rounds to 2, the smallest size LSD runs at); 9 x 7, 33 x 31: scaled sizes that are not multiples of 32
TINY_SHAPES = [(3, 3), (4, 5), (7, 9), (9, 7), (16, 17), (33, 31), (65, 129)]


def test_tiny_frames(ref):
    rng = np.random.default_rng(9)
    for h, w in TINY_SHAPES:
        _same(ref, tiny_frame(h, w, h * w))
        _same(ref, rng.integers(0, 256, (h, w), dtype=np.uint8))
    assert _same(ref, tiny_frame(65, 129, 1)) >= 1


@pytest.mark.parametrize("name", sorted(CHECKERBOARDS))
def test_checkerboards(ref, name):
    img = checkerboard(*CHECKERBOARDS[name])
    assert _same(ref, img, cap=16384) > 2048
    if ref.ref_detect_filter_lines_available():  # the filtered matrix as well: every segment is shorter than 15 pixels, so it is empty
        want = ref.ref_detect_filter_lines(img, True, 15.0, cap=16384)
        np.testing.assert_array_equal(ref.lsd_detect(img, 15.0, cap=16384)["lines"], want)
        assert want.shape == (0, 4)
