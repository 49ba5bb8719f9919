"""The LSD seed loop's seed scan (cube_slam_b200/csrc/cs_lsd.cu, k_lsd_grow_seq), checked on the CPU with the kernel's steps restated in
numpy.

The reference visits every pixel in raster order and grows a region from it iff its angle is defined and it is not USED at that moment
(lsd.cpp:478-481).  The kernel scans the row-padded bit planes defb ("angle defined") and used 32 words per step, one word per lane, takes
the bits of defb & ~used lowest first, and after every grow reads the used words of this step and the next again and recomputes what is
left of the step.  A grow here sets and clears bits anywhere -- refine and reduce_region_radius give pixels back, also later pixels of the
step being scanned and pixels already passed -- and both walks must visit the same seeds."""
import numpy as np
import pytest


def _grow(used, y, x, rng_seed):
    """a stand-in for one seed's grow -> rectangle -> refine: marks the seed and a few pixels around and after it, and gives some pixels
    back (as refine / reduce_region_radius do), also pixels later in the same row, in the next rows and before the seed"""
    H, W = used.shape
    rng = np.random.default_rng(rng_seed)
    used[y, x] = True
    n = int(rng.integers(0, 12))
    ys = np.clip(y + rng.integers(-1, 3, n), 0, H - 1)
    xs = np.clip(x + rng.integers(-3, 40, n), 0, W - 1)
    used[ys, xs] = True
    if rng.random() < 0.4:                       # give back a few: after the seed (same step), below it, and before it
        m = int(rng.integers(1, 6))
        gy = np.clip(y + rng.integers(-1, 2, m), 0, H - 1)
        gx = np.clip(x + rng.integers(-20, 60, m), 0, W - 1)
        keep_seed = (gy == y) & (gx == x)
        used[gy[~keep_seed], gx[~keep_seed]] = False


def _scan_reference(defined, used0, salt):
    used = used0.copy()
    H, W = defined.shape
    seeds = []
    for y in range(H):
        for x in range(W):
            if defined[y, x] and not used[y, x]:
                seeds.append((y, x))
                _grow(used, y, x, salt + y * W + x)
    return seeds


def _pack(plane, WW):
    H, W = plane.shape
    padded = np.zeros((H, WW * 32), np.uint8)
    padded[:, :W] = plane
    return np.packbits(padded.reshape(H, WW, 32), axis=2, bitorder="little").view("<u4").reshape(H * WW).astype(np.uint64)


def _scan_words(defined, used0, salt):
    """the kernel's loop: lane l of a step holds word w0 + l; s = defb & ~used; after a grow, used words of this step and the next are read
    again and the bits up to and including the seed (and the words of lower lanes) are masked off"""
    H, W = defined.shape
    WW = (W + 31) // 32
    n_words = WW * H
    used = used0.copy()                       # the used map as pixels; the kernel reads it as words
    defb = _pack(defined, WW)
    lanes = np.arange(32)
    full = np.uint64(0xFFFFFFFF)

    def load_used(idx):
        words = _pack(used, WW)
        return np.where(idx < n_words, words[np.minimum(idx, n_words - 1)], 0).astype(np.uint64)

    seeds = []
    u_next = load_used(lanes)
    d_next = np.where(lanes < n_words, defb[np.minimum(lanes, n_words - 1)], 0).astype(np.uint64)
    for w0 in range(0, n_words, 32):
        wi = w0 + lanes
        d, u = d_next, u_next
        d_next = np.where(wi + 32 < n_words, defb[np.minimum(wi + 32, n_words - 1)], 0).astype(np.uint64)
        u_next = load_used(wi + 32)
        s = d & ~u & full
        while True:
            nz = np.nonzero(s)[0]
            if len(nz) == 0:
                break
            j = int(nz[0])
            sw = int(s[j])
            b = (sw & -sw).bit_length() - 1
            y, xw = divmod(w0 + j, WW)
            x = xw * 32 + b
            assert x < W
            seeds.append((y, x))
            _grow(used, y, x, salt + y * W + x)
            u = load_used(wi)
            u_next = load_used(wi + 32)
            after = np.where(lanes > j, full, np.where(lanes == j, np.uint64((0xFFFFFFFE << b) & 0xFFFFFFFF), np.uint64(0)))
            s = d & ~u & after & full
    return seeds


@pytest.mark.parametrize("W", [31, 32, 33, 513, 994, 1024])
def test_word_scan_visits_the_seeds_in_raster_order(W):
    rng = np.random.default_rng(W)
    H = max(3, 6000 // W)
    for density, pre_used in ((0.5, 0.0), (0.15, 0.3), (0.9, 0.05)):
        defined = rng.random((H, W)) < density
        defined[-1, :] = False                 # the last row and column never have an angle (lsd.cpp:562-586)
        defined[:, -1] = False
        used0 = rng.random((H, W)) < pre_used
        salt = int(rng.integers(1 << 30))
        want = _scan_reference(defined, used0, salt)
        got = _scan_words(defined, used0, salt)
        assert got == want
        assert len(want) > 10
