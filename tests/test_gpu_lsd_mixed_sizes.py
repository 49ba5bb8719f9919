"""LSD over frames of different sizes in one GPU batch (cs_detect_lines_batch_mixed, cs_detect_raw_lines_octaves_batch_mixed) and the
Python list form that uses it (line_lbd_detect.detect_filter_lines_batch on a list).

The expected value of every frame is what the one-size calls return for that frame alone, compared with assert_array_equal; a subset is also
compared with the oracle (oracle/pyoracle.py, oracle/pyoracle_octaves.py)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

THRES = 15.0


@pytest.fixture(scope="module")
def ctx():
    import cube_slam_b200 as cs
    c = cs.Context(0, 1280, 960, 1, 1, 1)
    yield c
    c.close()


def params(ctx, use_LSD=1, K=1, thres=THRES):
    from cube_slam_b200 import _lib
    p = _lib.LineParams()
    ctx.L.cs_default_line_params(C.byref(p))
    p.use_LSD, p.numoctaves, p.octaveratio, p.line_length_thres = use_LSD, K, 2.0 if K > 1 else 1.0, thres
    return p


def scenes(seed, w, h):
    from cube_slam_b200 import synthetic
    return synthetic.make_batch(seed, 1, w, h)[0][0]


def checkerboard(w, h, cell=8, seed=3):
    """a random board of cell x cell squares: thousands of short segments, more LSD candidates in one frame than the first hand-off buffer"""
    rng = np.random.default_rng(seed)
    grid = rng.integers(0, 2, ((h + cell - 1) // cell, (w + cell - 1) // cell)).astype(np.uint8) * 200 + 20
    return np.ascontiguousarray(np.kron(grid, np.ones((cell, cell), np.uint8))[:h, :w])


def frame_mix(fixture_a, fixture_b):
    big = scenes(5, 1280, 720)
    gray = lambda x: np.ascontiguousarray(x[..., 1])
    return [scenes(1, 640, 480), gray(scenes(2, 320, 240)), big, np.ascontiguousarray(big[100:579, 200:841]), gray(big[300:323, 500:537]),
            np.full((3, 3), 9, np.uint8), np.arange(27, dtype=np.uint8).reshape(3, 3, 3), fixture_a["img"], gray(fixture_b["frames"][30][0]),
            fixture_b["frames"][7][0]]


def one_size(ctx, img, p, cap):
    """cs_detect_lines_batch on one frame -> its n x 4 segments"""
    from cube_slam_b200 import _lib
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    out = np.zeros((1, cap, 4), np.float32)
    n = np.zeros(1, np.int32)
    ctx.check(ctx.L.cs_detect_lines_batch(ctx.h, img.ctypes.data, 1, w, h, w * ch, ch, C.byref(p), _lib.ptr(out, C.c_float), cap, _lib.ptr(n, C.c_int32)))
    return out[0, :n[0]]


def mixed(ctx, imgs, p, cap, views=None, buf=None):
    """cs_detect_lines_batch_mixed -> (return code, per frame n x 4 segments)"""
    from cube_slam_b200 import _lib
    if views is None:
        buf, views = _lib.pack_frames(imgs)
    F = len(views)
    out = np.zeros((F, cap, 4), np.float32)
    n = np.zeros(F, np.int32)
    rc = ctx.L.cs_detect_lines_batch_mixed(ctx.h, buf.ctypes.data if buf is not None else None, views, F, C.byref(p), _lib.ptr(out, C.c_float), cap,
                                           _lib.ptr(n, C.c_int32))
    return rc, [out[f, :n[f]].copy() for f in range(F)]


def octaves_one(ctx, img, p, cap=4096):
    from cube_slam_b200 import _lib
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    K = p.numoctaves
    kl = np.zeros((1, K, cap), _lib.OCTAVE_KEYLINE_DTYPE)
    n = np.zeros((1, K), np.int32)
    ctx.check(ctx.L.cs_detect_raw_lines_octaves_batch(ctx.h, img.ctypes.data, 1, w, h, w * ch, ch, C.byref(p), kl.ctypes.data, cap,
                                                       _lib.ptr(n, C.c_int32)))
    return [kl[0, k, :n[0, k]].copy() for k in range(K)]


def octaves_mixed(ctx, imgs, p, cap=4096):
    from cube_slam_b200 import _lib
    buf, views = _lib.pack_frames(imgs)
    F, K = len(imgs), p.numoctaves
    kl = np.zeros((F, K, cap), _lib.OCTAVE_KEYLINE_DTYPE)
    n = np.zeros((F, K), np.int32)
    rc = ctx.L.cs_detect_raw_lines_octaves_batch_mixed(ctx.h, buf.ctypes.data, views, F, C.byref(p), kl.ctypes.data, cap, _lib.ptr(n, C.c_int32))
    return rc, [[kl[f, k, :n[f, k]].copy() for k in range(K)] for f in range(F)]


def test_frame_mix_equals_each_frame_alone(ctx, oracle, fixture_a, fixture_b):
    """VGA, 320 x 240, 1280 x 720, 641 x 479, 37 x 23, the smallest frame LSD takes (3 x 3) gray and BGR, fixture frames: every frame's
    segments are those of the frame alone; a row-padded view reads the same; a subset is the oracle's"""
    imgs = frame_mix(fixture_a, fixture_b)
    p = params(ctx)
    rc, got = mixed(ctx, imgs, p, 4096)
    assert rc == 0, ctx.L.cs_last_error(ctx.h).decode()
    for f, img in enumerate(imgs):
        np.testing.assert_array_equal(got[f], one_size(ctx, img, p, 4096), err_msg="frame %d (%s)" % (f, img.shape,))
    for f in (0, 3, 4, 7):
        np.testing.assert_array_equal(got[f], oracle.lsd_detect(imgs[f], THRES)["lines"], err_msg="frame %d against the oracle" % f)
    # the same frames with padded rows and gaps between them
    from cube_slam_b200 import _lib
    views = (_lib.FrameView * len(imgs))()
    parts, off = [], 0
    for f, img in enumerate(imgs):
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else 3
        stride = w * ch + 13
        a = np.zeros((h, stride), np.uint8)
        a[:, :w * ch] = img.reshape(h, w * ch)
        views[f].offset, views[f].width, views[f].height, views[f].stride, views[f].channels = off + 5, w, h, stride, ch
        parts += [np.zeros(5, np.uint8), a.reshape(-1)]
        off += 5 + a.size
    rc, padded = mixed(ctx, None, p, 4096, views, np.concatenate(parts))
    assert rc == 0, ctx.L.cs_last_error(ctx.h).decode()
    for f in range(len(imgs)):
        np.testing.assert_array_equal(padded[f], got[f], err_msg="padded frame %d" % f)


def test_frame_order(ctx, fixture_a, fixture_b):
    imgs = frame_mix(fixture_a, fixture_b)
    p = params(ctx)
    _, got = mixed(ctx, imgs, p, 4096)
    perm = np.random.default_rng(4).permutation(len(imgs))
    rc, back = mixed(ctx, [imgs[i] for i in perm], p, 4096)
    assert rc == 0
    for j, i in enumerate(perm):
        np.testing.assert_array_equal(back[j], got[i], err_msg="permuted position %d (frame %d)" % (j, i))


def test_edlines_groups(ctx, fixture_a, fixture_b):
    """use_LSD == 0: one EDLines batch per size group, each frame what it is alone"""
    imgs = [x for x in frame_mix(fixture_a, fixture_b) if min(x.shape[:2]) >= 16]
    imgs = imgs + imgs[:2]
    p = params(ctx, use_LSD=0)
    rc, got = mixed(ctx, imgs, p, 4096)
    assert rc == 0, ctx.L.cs_last_error(ctx.h).decode()
    for f, img in enumerate(imgs):
        np.testing.assert_array_equal(got[f], one_size(ctx, img, p, 4096), err_msg="EDLines frame %d" % f)


def test_dense_frame_beside_small_ones(ctx):
    """a checkerboard overflows the candidate hand-off buffer; after the regrow every frame is exact"""
    imgs = [scenes(7, 160, 120), checkerboard(1280, 960, 4), np.ascontiguousarray(scenes(8, 200, 150)[..., 0]), checkerboard(97, 61, 3)]
    p = params(ctx, thres=-1.0)     # every segment: each one is an accepted candidate of the seed loop
    cap = 65536
    rc, got = mixed(ctx, imgs, p, cap)
    assert rc == 0, ctx.L.cs_last_error(ctx.h).decode()
    assert len(got[1]) > 2048
    for f, img in enumerate(imgs):
        np.testing.assert_array_equal(got[f], one_size(ctx, img, p, cap), err_msg="frame %d" % f)


def test_capacity_names_the_frame(ctx, fixture_a):
    imgs = [np.ascontiguousarray(scenes(9, 64, 48)[..., 0]), fixture_a["img"], scenes(10, 320, 240)]
    p = params(ctx)
    full = [one_size(ctx, x, p, 4096) for x in imgs]
    cap = len(full[1]) - 1
    assert max(len(full[0]), len(full[2])) <= cap
    rc, _ = mixed(ctx, imgs, p, cap)
    assert rc == -3
    assert "frame 1" in ctx.L.cs_last_error(ctx.h).decode()
    rc, got = mixed(ctx, imgs, p, 4096)
    assert rc == 0
    for f in range(3):
        np.testing.assert_array_equal(got[f], full[f])
    # octaves: frame and octave named
    po = params(ctx, K=2)
    one = [octaves_one(ctx, x, po) for x in imgs]
    counts = [[len(o) for o in x] for x in one]
    rc, _ = octaves_mixed(ctx, imgs, po, cap=1)
    assert rc == -3
    msg = ctx.L.cs_last_error(ctx.h).decode()
    assert "frame" in msg and "octave" in msg, msg
    rc, got = octaves_mixed(ctx, imgs, po)
    assert rc == 0 and [[len(o) for o in x] for x in got] == counts


def test_refused_before_any_launch(ctx, fixture_a):
    from cube_slam_b200 import _lib
    imgs = [fixture_a["img"], scenes(11, 320, 240)]
    buf, views = _lib.pack_frames(imgs)
    p = params(ctx)
    out = np.zeros((2, 64, 4), np.float32)
    n = np.zeros(2, np.int32)
    L, h = ctx.L, ctx.h

    def call(b, v, F, fn="lines", prm=p):
        if fn == "lines":
            return L.cs_detect_lines_batch_mixed(h, b, v, F, C.byref(prm), _lib.ptr(out, C.c_float), 64, _lib.ptr(n, C.c_int32))
        kl = np.zeros(2 * prm.numoctaves * 64, _lib.OCTAVE_KEYLINE_DTYPE)
        nn = np.zeros(2 * prm.numoctaves, np.int32)
        return L.cs_detect_raw_lines_octaves_batch_mixed(h, b, v, F, C.byref(prm), kl.ctypes.data, 64, _lib.ptr(nn, C.c_int32))

    def bad(field, value):
        v = (_lib.FrameView * 2)()
        C.memmove(v, views, C.sizeof(v))
        setattr(v[1], field, value)
        return v

    for fn in ("lines", "octaves"):
        assert call(None, views, 2, fn) == -1
        assert call(buf.ctypes.data, None, 2, fn) == -1
        assert call(buf.ctypes.data, views, 0, fn) == -1
        for field, value in (("width", 0), ("height", -1), ("channels", 2), ("stride", 100), ("offset", -1)):
            assert call(buf.ctypes.data, bad(field, value), 2, fn) == -1, (fn, field)
            assert "frame 1" in L.cs_last_error(h).decode(), (fn, field)
    tiny = bad("width", 1)
    tiny[1].stride = 3
    assert call(buf.ctypes.data, tiny, 2) == -1 and "frame 1" in L.cs_last_error(h).decode()
    assert call(buf.ctypes.data, views, 2, "octaves", params(ctx, K=9)) == -1
    assert "frame 1" in L.cs_last_error(h).decode() and "too small" in L.cs_last_error(h).decode()     # 320 x 240 at octave 8
    rc, got = mixed(ctx, imgs, p, 4096)
    assert rc == 0
    np.testing.assert_array_equal(got[1], one_size(ctx, imgs[1], p, 4096))


def test_octaves_every_frame(ctx, fixture_a, fixture_b):
    """K = 1 .. 4: the mixed octave call is the per-image call field for field; one frame per K is the oracle's"""
    from oracle import pyoracle_octaves as octo
    big = scenes(12, 1280, 720)
    imgs = [scenes(13, 640, 480), np.ascontiguousarray(scenes(14, 320, 240)[..., 2]), np.ascontiguousarray(big[11:490, 17:658]),
            np.ascontiguousarray(big[200:223, 300:337]), fixture_b["frames"][12][0], np.ascontiguousarray(fixture_a["img"][..., 0])]
    for K in (1, 2, 3, 4):
        p = params(ctx, K=K)
        rc, got = octaves_mixed(ctx, imgs, p)
        assert rc == 0, ctx.L.cs_last_error(ctx.h).decode()
        for f, img in enumerate(imgs):
            want = octaves_one(ctx, img, p)
            for k in range(K):
                np.testing.assert_array_equal(got[f][k], want[k], err_msg="K %d frame %d octave %d" % (K, f, k))
        f = K % len(imgs)
        ora = octo.lsd_octaves_raw(imgs[f], K, 2.0)
        for k in range(K):
            assert len(got[f][k]) == len(ora[k]), (K, k)
            for a, b in zip(got[f][k].dtype.names, ora[k].dtype.names):
                if not a.startswith("pad"):
                    np.testing.assert_array_equal(got[f][k][a], ora[k][b], err_msg="K %d octave %d field %s against the oracle" % (K, k, a))


def test_many_frames(ctx):
    """512 frames of four sizes, shuffled, in one call: each frame is what its size group's one-size call gives it"""
    rng = np.random.default_rng(15)
    sizes = [(160, 120), (200, 150), (96, 64), (320, 240)]
    base = {s: [scenes(20 + i * 7 + j, s[0], s[1]) for j in range(4)] for i, s in enumerate(sizes)}
    order = rng.integers(0, 4, 512)
    imgs = [base[sizes[s]][i % 4] if i % 3 else np.ascontiguousarray(base[sizes[s]][i % 4][..., 1]) for i, s in enumerate(order)]
    p = params(ctx)
    rc, got = mixed(ctx, imgs, p, 1024)
    assert rc == 0, ctx.L.cs_last_error(ctx.h).decode()
    from cube_slam_b200 import _lib
    groups = {}
    for i, img in enumerate(imgs):
        groups.setdefault(img.shape, []).append(i)
    for shape, idx in groups.items():
        a = np.ascontiguousarray(np.stack([imgs[i] for i in idx]))
        h, w = shape[:2]
        ch = 1 if len(shape) == 2 else 3
        out = np.zeros((len(idx), 1024, 4), np.float32)
        n = np.zeros(len(idx), np.int32)
        ctx.check(ctx.L.cs_detect_lines_batch(ctx.h, a.ctypes.data, len(idx), w, h, w * ch, ch, C.byref(p), _lib.ptr(out, C.c_float), 1024,
                                              _lib.ptr(n, C.c_int32)))
        for j, i in enumerate(idx):
            np.testing.assert_array_equal(got[i], out[j, :n[j]], err_msg="frame %d %s" % (i, shape))


def test_python_list_form(ctx, fixture_a, fixture_b):
    """line_lbd_detect.detect_filter_lines_batch on a list of differently sized images (one mixed call) is per-image detect_filter_lines"""
    import cube_slam_b200 as cs
    imgs = [scenes(30, 640, 480), np.ascontiguousarray(scenes(31, 320, 240)[..., 0]), fixture_b["frames"][3][0], fixture_a["img"],
            np.ascontiguousarray(scenes(32, 641, 479)[..., :3])]
    d = cs.line_lbd_detect(1, 1.0, context=ctx)
    d.use_LSD = True
    got = d.detect_filter_lines_batch(imgs)
    for i, img in enumerate(imgs):
        np.testing.assert_array_equal(got[i], d.detect_filter_lines(img, 4096), err_msg="detect_filter_lines_batch image %d" % i)


def test_edlines_sizes_checked_before_any_group(ctx, fixture_a):
    """use_LSD == 0: a frame outside EDLines' sizes is refused by name before the first group runs: no count is written"""
    imgs = [fixture_a["img"], scenes(34, 320, 240), np.full((6, 40), 50, np.uint8)]
    p = params(ctx, use_LSD=0)
    from cube_slam_b200 import _lib
    buf, views = _lib.pack_frames(imgs)
    out = np.zeros((3, 64, 4), np.float32)
    n = np.full(3, -7, np.int32)
    rc = ctx.L.cs_detect_lines_batch_mixed(ctx.h, buf.ctypes.data, views, 3, C.byref(p), _lib.ptr(out, C.c_float), 64, _lib.ptr(n, C.c_int32))
    assert rc == -1
    assert "frame 2" in ctx.L.cs_last_error(ctx.h).decode()
    assert (n == -7).all()


def test_debug_readers_refuse_after_a_mixed_run(ctx, fixture_a):
    from cube_slam_b200 import _lib
    p = params(ctx)
    rc, _ = mixed(ctx, [fixture_a["img"], scenes(33, 320, 240)], p, 4096)
    assert rc == 0
    wh = np.zeros(2, np.int32)
    assert ctx.L.cs_debug_lsd(ctx.h, 0, _lib.ptr(wh, C.c_int32), None, None, None, None, None, None, None, 0) == -6
    assert "mixed" in ctx.L.cs_last_error(ctx.h).decode()
    assert ctx.L.cs_debug_lsd_defb(ctx.h, 0, None, _lib.ptr(wh, C.c_int32)) == -6
    one_size(ctx, fixture_a["img"], p, 4096)
    assert ctx.L.cs_debug_lsd(ctx.h, 0, _lib.ptr(wh, C.c_int32), None, None, None, None, None, None, None, 0) == 0
    octaves_one(ctx, fixture_a["img"], params(ctx, K=2))       # an octave call is one LSD run over planes of two sizes
    assert ctx.L.cs_debug_lsd(ctx.h, 0, _lib.ptr(wh, C.c_int32), None, None, None, None, None, None, None, 0) == -6
