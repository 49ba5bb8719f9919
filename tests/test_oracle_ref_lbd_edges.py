"""The LBD descriptor / matcher oracle against the REFERENCE'S OWN code (oracle/_ref/liblinelbd_ref.so, as tests/test_oracle_ref_lbd.py) on
the inputs tests/test_gpu_lbd_edges.py runs on the device, where descriptor kernels can go wrong and the demo / sequence frames never go:

 * dense frames: the EDLines routing-regime frames (test_oracle_ref_edlines.dense_frames) and the two LSD checkerboards with no length
   filter (2 760 and 13 463 key lines: thousands of describe CTAs in one launch);
 * ragged frame sizes, gray and BGR, detected and with given key lines;
 * tiny frames: given key lines in frames from 1 x 1 up to 7 x 9 (the Sobel maps reflect every tap into a 1-pixel side), LSD detection at
   the sizes the LSD accepts (3 x 3 up: no key line, no error);
 * long and border lines: full-width, full-height and full-diagonal lines of a 1280 x 960 frame (numOfPixels 1 280 / 960 / 1 280), lines on
   every border row and column, end points outside the frame, one-pixel lines, and a 1280 x 40 frame whose 63-row support regions leave the
   frame on both sides;
 * the matcher at scale and at its special cases: 2 000 queries against 5 000 codes, ties between codes in different lanes / warps / loop
   iterations of the device's scan, empty sets in the middle of a batch, thresholds equal to a distance, nearest codes further than
   D = 128, queries the multi-index hash never meets, and every consecutive frame pair of the shipped sequence.

Everything is compared bit for bit: key-line fields, 32-byte descriptors, 72-float descriptors (NaN == NaN: a one-pixel line or a flat
frame has a zero band and its normalisation divides 0 by 0), and (query, train, distance) triples -- the reference's train index only
where the distance is at most 128 (beyond it the reference never writes the index; the oracle and the library say -1).  Where the
reference and the oracle agree down to 1 x 1 the product accepts 1 x 1 (cs_edl_sobel_maps)."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.ref_detect_filter_lines_available():
        pytest.skip("oracle/_ref/liblinelbd_ref.so not built (no /root/reference on this machine)")
    return oracle


FIELDS = ("sx", "sy", "ex", "ey", "angle", "line_length", "response", "size", "num_pixels")


# ---- inputs (tests/test_gpu_lbd_edges.py builds the same) --------------------------------------------------------------------------------

def sxga_frames(n=2, seed=93):
    from cube_slam_b200 import synthetic as S
    return S.make_batch(seed, n, 1280, 960, 3)[0]


RAGGED_SHAPES = [(97, 211), (61, 64), (200, 333), (203, 241)]
# given key lines: 1-pixel sides up to the 7 x 9 ragged frame; 8 x 8 and above has always been accepted
TINY_GIVEN_SHAPES = [(1, 1), (1, 9), (9, 1), (2, 2), (2, 7), (3, 4), (5, 5), (4, 8), (8, 4), (7, 9)]
# LSD detection: lrint(0.8 * 3) = 2 is the smallest scaled side the LSD runs at
TINY_LSD_SHAPES = [(3, 3), (4, 5), (5, 5), (7, 9), (9, 7)]


def tiny_image(h, w, channels, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w) + ((3,) if channels == 3 else ()), dtype=np.uint8)


def given_rows(h, w, n_random=40, seed=0):
    """Segments of a w x h frame: corner to corner, each border, a one-pixel line, a zero-length line, end points outside the frame, and
    random segments (float end points anywhere in and a little around the frame)."""
    rng = np.random.default_rng(seed + 7 * w + h)
    W, H = w - 1, h - 1
    rows = [[0, 0, W, H], [W, 0, 0, H], [0, 0, W, 0], [0, H, W, H], [0, 0, 0, H], [W, 0, W, H], [W / 2, H / 2, W / 2 + 0.3, H / 2 + 0.2],
            [W / 3, H / 3, W / 3, H / 3], [-5, H / 2, W + 5, H / 2 + 1], [W / 2, -4, W / 2 - 1, H + 6]]
    rnd = rng.uniform(-0.1, 1.1, (n_random, 4)) * np.array([W, H, W, H])
    return np.concatenate([np.array(rows, np.float32), rnd.astype(np.float32)])


def long_and_border_rows(w=1280, h=960):
    """Lines a demo frame never has: the full width, height and diagonal; each border row and column, whole and in part; end points
    outside the frame (numOfPixels counts the clamped ends); one-pixel lines; lines 1 px inside the border."""
    W, H = w - 1, h - 1
    rows = [[0, 480, W, 480], [640, 0, 640, H], [0, 0, W, H], [W, 0, 0, H],
            [0, 0, W, 0], [0, H, W, H], [0, 0, 0, H], [W, 0, W, H], [W, H, 0, H],
            [100, 0, 400, 0], [900, H, 300, H], [0, 100, 0, 700], [W, 800, W, 50], [1, 1, W - 1, 1], [W - 1, 2, W - 1, H - 2],
            [-200, 300, W + 300, 500], [600, -100, 700, H + 100], [-50, -50, W + 50, H + 50], [-10, 10, -1, 900],
            [500.2, 300.1, 500.4, 300.3], [0, 0, 0.4, 0.4], [W, H, W - 0.3, H], [77.5, 88.5, 77.5, 88.5],
            [31, 31, W - 31, 31], [30.6, H - 30.6, W - 30.6, H - 30.6]]
    return np.array(rows, np.float32)


def short_frame_rows(w=1280, h=40):
    """A 1280 x 40 frame: every 63-row support region leaves the frame above and below."""
    W, H = w - 1, h - 1
    rows = [[0, 20, W, 20], [0, 0, W, H], [0, H, W, 0], [10, 5, 1200, 5], [1270, 35, 3, 36], [640, 0, 640, H], [100, 0, 160, H],
            [0, 0, W, 0], [0, H, W, H], [300.5, 19.5, 900.5, 19.5], [-40, 10, W + 40, 30], [5, 20, 5.2, 20.1]]
    return np.array(rows, np.float32)


def short_frame(w=1280, h=40, seed=95):
    """Bands of levels along x with a step every 32 columns and noise: plenty of gradient for long lines to sample."""
    rng = np.random.default_rng(seed)
    img = np.repeat(((np.arange(w) // 32) * 37 % 256)[None, :], h, 0)
    img = img + (np.arange(h)[:, None] > h // 2) * 60 + rng.integers(0, 12, (h, w))
    return np.ascontiguousarray(np.stack([img, 255 - img, img // 2 + 30], 2).clip(0, 255).astype(np.uint8))


def _flip_bits(code, bits):
    code = code.copy()
    for b in bits:
        code[b // 8] ^= np.uint8(1 << (b % 8))
    return code


def _near_codes(rng, train, n, max_bits):
    """n queries, each a train code with up to max_bits random bits flipped"""
    return np.stack([_flip_bits(train[int(rng.integers(0, len(train)))], rng.integers(0, 256, int(rng.integers(0, max_bits + 1))))
                     for _ in range(n)])


def _bytes_with_popcount(rng, shape, lo, hi):
    vals = np.array([v for v in range(256) if lo <= bin(v).count("1") <= hi], np.uint8)
    return vals[rng.integers(0, len(vals), shape)]


# train indices the device's scan gives to different lanes (j + 1), warps (j + 32) and loop iterations of one thread (j + 128 k)
TIE_OFFSETS = (0, 1, 32, 128, 256, 4096 + 64)
TIE_DISTANCES = [32, 4, 32, 6, 32, 4, 32, 6]      # of the 8 tie queries' planted codes (matcher_cases)


def matcher_cases():
    """name -> (list of query sets, list of train sets, thresholds); each case is one cs_match_line_descrip_batch call on the device."""
    rng = np.random.default_rng(21)
    cases = {}
    # 2 000 queries against 5 000 codes: near codes (0 .. 60 bits), some unrelated, exact duplicates in the train set
    t = rng.integers(0, 256, (5000, 32), dtype=np.uint8)
    t[4000:4100] = t[100:200]
    q = _near_codes(rng, t, 2000, 60)
    q[::10] = rng.integers(0, 256, (200, 32), dtype=np.uint8)
    cases["q2000_t5000"] = ([q], [t], (25.0, 300.0))
    # planted ties: for each of 8 queries, codes at the same distance at train indices j + TIE_OFFSETS.  Codes with one bit flipped in every
    # byte (distance 32, smallest byte distance 1 at byte 0): the flipped bit of byte 0 decides (the hash flips lower patterns first); the
    # same code twice: the lower train index.  Codes with k bits flipped in k different bytes (distance k): the first unflipped byte decides.
    t = rng.integers(0, 256, (4500, 32), dtype=np.uint8)
    qs = rng.integers(0, 256, (8, 32), dtype=np.uint8)
    for i in range(8):
        j = 7 + 9 * i
        offs = [o for o in TIE_OFFSETS if j + o < len(t)]
        if i % 2 == 0:
            for n, o in enumerate(offs):
                first = (n * 3 + i) % 8 if n < len(offs) - 2 else 5      # the last two share byte 0's bit: train index decides between them
                bits = [first] + [8 * b + int(rng.integers(0, 8)) for b in range(1, 32)]
                t[j + o] = _flip_bits(qs[i], bits)
        else:
            k = 3 + i % 4
            for n, o in enumerate(offs):
                byte_set = sorted(rng.choice(32, k, replace=False)) if n < len(offs) - 1 else list(range(k))
                t[j + o] = _flip_bits(qs[i], [8 * b + int(rng.integers(0, 8)) for b in byte_set])
    cases["ties"] = ([qs], [t], (32.0, 32.5, 33.0, 24.5, 5.0, 4.0, 300.0))
    # 64 pairs; empty query sets at positions 0 and 63, empty train sets at 31 and 40, both at 20
    queries, trains = [], []
    for p in range(64):
        nt = int(rng.integers(1, 300))
        tt = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
        qq = _near_codes(rng, tt, int(rng.integers(1, 50)), 40)
        if p in (0, 63, 20):
            qq = qq[:0]
        if p in (31, 40, 20):
            tt = tt[:0]
        queries.append(qq)
        trains.append(tt)
    cases["pairs64_with_empty_sets"] = (queries, trains, (25.0, 24.5, 300.0))
    # nearest codes further than D = 128 (every byte of the train codes has 7 or 8 bits set, the queries' at most one, except one byte of
    # each train code that is within 2 bits: the hash meets them, at distance >= 186); and a pair whose train codes all have every byte at
    # 5 or more bits from every query byte: no query is ever met, no DMatch at any threshold
    qlow = _bytes_with_popcount(rng, (30, 32), 0, 1)
    tfar = _bytes_with_popcount(rng, (40, 32), 7, 8)
    for i in range(40):
        tfar[i, i % 32] = _bytes_with_popcount(rng, (1,), 0, 1)[0]
    tnever = _bytes_with_popcount(rng, (50, 32), 6, 8)
    qnever = np.concatenate([qlow[:10], np.zeros((3, 32), np.uint8)])
    comp_q = rng.integers(0, 256, (1, 32), dtype=np.uint8)            # one query, its complement and codes 7, 6, 5 bits away in every byte
    comp_t = np.concatenate([~comp_q ^ np.uint8(m) for m in (0, 1, 3, 7, 0x38)])
    cases["far_and_never_met"] = ([qlow, qnever, comp_q, qlow[:5]], [tfar, tnever, comp_t, tfar[:0]], (25.0, 128.5, 300.0))
    return cases


# ---- comparisons --------------------------------------------------------------------------------------------------------------------

def same_keylines(ref, img, use_lsd, thres, cap=8192):
    kr, dr = ref.ref_detect_descrip_lines(img, use_lsd, thres, cap)
    ko = ref.lbd_detect_keylines(img, use_lsd, thres, cap)
    assert len(kr) == len(ko)
    for f in FIELDS:
        np.testing.assert_array_equal(kr[f], ko[f], err_msg=f)
    np.testing.assert_array_equal(ref.lbd_compute(img, ko), dr)
    return ko


def same_given(ref, img, rows):
    h, w = img.shape[:2]
    kl = ref.lbd_keylines_from_lsd(rows, w, h)
    d, f = ref.lbd_compute(img, kl, want_float=True)
    d2, f2 = ref.ref_lbd_compute(img, kl, want_float=True)
    np.testing.assert_array_equal(d, d2)
    np.testing.assert_array_equal(f, f2)          # NaN == NaN, in the same places
    return kl, f


def same_matches(ref, q, t, thres):
    a, b = ref.lbd_match(q, t, thres), ref.ref_match_line_descrip(q, t, thres)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[2], b[2])
    near = a[2] <= 128
    np.testing.assert_array_equal(a[1][near], b[1][near])
    assert (a[1][~near] == -1).all()
    return a


# ---- tests ----------------------------------------------------------------------------------------------------------------------------

def test_dense_frames_both_flavours(ref):
    from test_oracle_ref_edlines import dense_frames
    want = {"room": (212, 234), "room_noise_band": (173, 181), "checkerboard_window": (39, 43)}
    for name, img in dense_frames().items():
        n = tuple(len(same_keylines(ref, img, use_lsd, 15.0)) for use_lsd in (False, True))
        assert n == want[name], (name, n)


@pytest.mark.parametrize("name,n", [("vga_10px", 2760), ("sxga_12px_noisy", 13463)])
def test_checkerboards_every_lsd_keyline(ref, name, n):
    from test_oracle_ref_lsd import CHECKERBOARDS, checkerboard
    img = checkerboard(*CHECKERBOARDS[name])
    assert len(same_keylines(ref, img, True, -1.0, cap=16384)) == n


def test_sxga_frames_and_ragged_sizes(ref):
    from test_gpu_lsd_parity import odd_size_batch
    for img in sxga_frames():
        for use_lsd in (True, False):
            assert len(same_keylines(ref, img, use_lsd, 15.0)) > 20
    for h, w in RAGGED_SHAPES:
        for channels in (1, 3):
            for img in odd_size_batch(h, w, channels):
                for use_lsd in (True, False):
                    same_keylines(ref, img, use_lsd, 15.0)
                same_given(ref, img, given_rows(h, w))


def test_tiny_frames(ref):
    """Given key lines from 1 x 1 up: the oracle's descriptors are the reference's, bytes and floats, NaNs included.  LSD detection from
    3 x 3 up: no key line and no error (computeImpl returns before computeSobel when there is no key line)."""
    n_nan = 0
    for h, w in TINY_GIVEN_SHAPES:
        for channels in (1, 3):
            _, f = same_given(ref, tiny_image(h, w, channels, h * 100 + w), given_rows(h, w, 8))
            n_nan += int(np.isnan(f).any(1).sum())
    assert n_nan > 0                                   # flat 1-pixel-high frames and zero-length lines: 0 / 0 in the normalisation
    from test_gpu_lsd_parity import odd_size_batch
    for h, w in TINY_LSD_SHAPES:
        for channels in (1, 3):
            for img in odd_size_batch(h, w, channels):
                assert len(same_keylines(ref, img, True, 15.0)) == 0
                assert len(same_keylines(ref, img, True, -1.0)) == 0


def test_long_and_border_lines(ref):
    img = sxga_frames(1)[0]
    kl, _ = same_given(ref, img, long_and_border_rows())
    assert {1280, 960, 1} <= set(kl["num_pixels"].tolist())
    kl, _ = same_given(ref, short_frame(), short_frame_rows())
    assert kl["num_pixels"].max() == 1280


@pytest.mark.parametrize("name", ["q2000_t5000", "ties", "pairs64_with_empty_sets", "far_and_never_met"])
def test_matcher_cases(ref, name):
    queries, trains, thresholds = matcher_cases()[name]
    for thres in thresholds:
        for q, t in zip(queries, trains):
            same_matches(ref, q, t, thres)
    if name == "far_and_never_met":
        qi, ti, d = same_matches(ref, queries[0], trains[0], 300.0)
        assert len(qi) == len(queries[0]) and (d > 128).all() and (ti == -1).all()
        for k in (1, 2):
            assert len(same_matches(ref, queries[k], trains[k], 300.0)[0]) == 0
    if name == "ties":
        qi, ti, d = same_matches(ref, queries[0], trains[0], 300.0)
        np.testing.assert_array_equal(d, TIE_DISTANCES)
        picked = ti - (7 + 9 * np.arange(8))
        assert set(picked.tolist()) <= set(TIE_OFFSETS) and len(set(picked.tolist())) > 1   # not always the lowest train index


def test_sequence_pairs(ref, fixture_b):
    """The LSD key lines of every frame of the shipped sequence, matched with the next frame's."""
    descs = [ref.lbd_compute(img, ref.lbd_detect_keylines(img, True, 15.0)) for img, _ in fixture_b["frames"]]
    total = 0
    for a, b in zip(descs[:-1], descs[1:]):
        total += len(same_matches(ref, a, b, 40.0)[0])
    assert total > 100
