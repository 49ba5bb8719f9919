"""The LSD seed loop's used map on the GPU (cube_slam_b200/csrc/cs_lsd.cu, k_lsd_grow_seq).  A growth round sets the bits of the pixels
it accepts, several of them often in one 32-pixel word; refine and reduce_region_radius clear the bits of the pixels they give back; the
raster scan re-reads the words after every seed.  A lost or stale bit changes which pixels later regions may take, so the frames here are
the ones where that would show:

- dense textures and horizontal stripes, where many pixels accepted in one round share a word;
- widths whose scaled rows do not fill their last word, and ramps at angles, so regions cross word and row-padding boundaries;
- frames with many refines and reduces, whose released pixels later seeds of the same 32-word scan step grow from again;
- the KITTI and 1280 x 960 shapes bench.py's c4 and c5 run.

Each batch goes through both instantiations of k_lsd_grow_seq (cs_set_profiling bit 0 and without); raw segments and the filtered matrix
equal the oracle's bit for bit in both."""
import numpy as np
import pytest

from test_gpu_lsd_rect_reduce import SLOT_REDUCE_ITERS, SLOT_REFINES, check_batch, det, ordinary  # noqa: F401 (det: fixture)
from test_oracle_ref_lsd_large_regions import frames

pytestmark = pytest.mark.gpu


def blocks(seed, w, h, side):
    """side x side blocks of random gray levels: short regions everywhere, most of them refined or reduced"""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 256, ((h + side - 1) // side, (w + side - 1) // side), dtype=np.uint8)
    return np.ascontiguousarray(np.kron(g, np.ones((side, side), np.uint8))[:h, :w])


def stripes(seed, w, h, period):
    """horizontal bands with a little noise: long rows of pixels accepted in the same rounds, many of them in one word"""
    rng = np.random.default_rng(seed)
    y = np.arange(h)[:, None]
    g = 128 + 70 * np.sign(np.sin(2 * np.pi * (y + 0.5) / period)) + rng.normal(0, 6, (h, w))
    return np.clip(g, 0, 255).astype(np.uint8)


def gray(img):
    return np.ascontiguousarray(img[:, :, 1])


@pytest.mark.parametrize("w,h", [(640, 480), (641, 480)])
def test_dense_textures(det, oracle, w, h):
    """block textures of 2, 3 and 5 pixels and stripes of period 5 and 7; 641 wide scales to 513, one pixel into a row's 17th word"""
    named = [("blocks%d" % s, blocks(900 + s, w, h, s)) for s in (2, 3, 5)]
    named += [("stripes%d" % p, stripes(910 + p, w, h, p)) for p in (5, 7)]
    prof = check_batch(det, oracle, named)
    assert int(prof[SLOT_REFINES]) > 0 and int(prof[SLOT_REDUCE_ITERS]) > 0, prof


def test_regions_across_words_and_row_padding(det, oracle):
    """ramps at 30 and 45 degrees and concentric rings: regions of hundreds to thousands of pixels that cross many word boundaries, with
    region lists past the part kept in shared memory"""
    f = frames()
    check_batch(det, oracle, [(n, f[n]) for n in ("saw30", "saw45", "rings_vga")])


def test_released_pixels_are_seeded_again(det, oracle):
    """c3-like frames and block textures side by side: dozens of refines and reduces a frame, each giving pixels back that the raster
    scan, still inside the same step, offers as seeds again"""
    named = [("c3_%d" % s, gray(ordinary(940 + s, 640, 480))) for s in range(3)]
    named += [("blocks4_%d" % s, blocks(950 + s, 640, 480, 4)) for s in range(3)]
    prof = check_batch(det, oracle, named)
    assert int(prof[SLOT_REFINES]) > 10 and int(prof[SLOT_REDUCE_ITERS]) > 10, prof


@pytest.mark.parametrize("w,h,kind", [(1242, 375, "kitti"), (1280, 960, "indoor")], ids=["c4", "c5"])
def test_benchmark_shapes(det, oracle, w, h, kind):
    """bench.py's c4 (scaled width 994, W % 32 != 0) and c5 frames, with a block texture of the same size"""
    from cube_slam_b200 import synthetic as S
    imgs = S.make_batch(960 + w, 2, w, h, 3, kind=kind)[0]
    named = [("%s_%d" % (kind, i), gray(imgs[i])) for i in range(len(imgs))] + [("blocks3", blocks(970, w, h, 3))]
    check_batch(det, oracle, named)
