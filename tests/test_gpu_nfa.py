"""The line detectors' NFA on the device (cs_nfa_warp, cube_slam_b200/csrc/cs_nfa.cuh) against the reference's formula (the oracle's
orc_lsd_nfa: lsd.cpp:1100-1136 and descriptor.hpp:763-830), triple by triple.

cs_nfa_warp looks log_gamma up in a host-built table below CS_LGAMMA_TABLE = 16 384 and evaluates it with the device's log / pow / sinh
above; the binomial tail is summed by one lane while all 32 evaluate the break test of 32 consecutive terms.  A device NFA that drifts from
the host's by more than about 1e-7 relative can flip a segment (the smallest relative gap between two NFAs rect_improve compares, over the
fixture, benchmark and large-region frames, is 4.75e-7), and the break index is an integer: any difference there is a logic error.

The grid (built on the CPU, where its coverage is asserted): every (n, k) with n <= 1 024 at p = 1/8; n <= 256 at the five halvings of p
rect_improve tries; n sampled up to 10^6; k + 1 and n - k + 1 at 16 383 / 16 384 / 16 385 (the table's edge); triples whose log of the first
term straddles the underflow cut of double_equal(term, 0) (about -740.7) and the denormal range of exp.  Each at the logNT of a VGA, a KITTI
and a 1280 x 960 frame, in both forms (lsd.cpp's (n + 1) first term and EDLines' log_gamma(n + 1))."""
import ctypes as C
import math

import numpy as np
import pytest

P_HALVINGS = [0.125 / 2 ** i for i in range(6)]   # 22.5 / 180 and rect_improve's five halvings


def log_nt(w, h):
    """LSD's logNT of a w x h frame (scaled by 0.8, lsd.cpp:471)"""
    W, H = round(0.8 * w), round(0.8 * h)
    return 5 * (math.log10(W) + math.log10(H)) / 2 + math.log10(11.0)


LOG_NTS = {"vga": log_nt(640, 480), "kitti": log_nt(1242, 375), "sxga": log_nt(1280, 960)}


def _log1term(n, k, p, lsd_first_term):
    lg = np.vectorize(math.lgamma)
    first = (n + 1.0) if lsd_first_term else lg(n + 1.0)
    return first - lg(k + 1.0) - lg(n - k + 1.0) + k * np.log(p) + (n - k) * np.log1p(-p)


def nfa_grid():
    """-> (n, k, p) int32 / int32 / float64 arrays"""
    rng = np.random.default_rng(2048)
    parts = []
    # every (n, k), n <= 1 024, at p = 1/8; n <= 256 at every p
    for n_max, ps in ((1024, P_HALVINGS[:1]), (256, P_HALVINGS[1:])):
        n = np.repeat(np.arange(n_max + 1), np.arange(n_max + 1) + 1)
        k = np.concatenate([np.arange(m + 1) for m in range(n_max + 1)])
        for p in ps:
            parts.append((n, k, np.full(len(n), p)))
    # n sampled up to 10^6: k around n p (where the tail is summed), below it and toward n
    n = np.exp(rng.uniform(np.log(1025), np.log(1e6), 3000)).astype(np.int64)
    p = rng.choice(P_HALVINGS, len(n))
    sd = np.sqrt(n * p * (1 - p))
    for k in (n * p + rng.normal(0, 1, len(n)) * 3 * sd, n * p + rng.uniform(0, 12, len(n)) * sd, rng.uniform(0, 1, len(n)) * n):
        parts.append((n, np.clip(np.rint(k), 0, n).astype(np.int64), p))
    # the table's edge: k + 1 or n - k + 1 at 16 383, 16 384, 16 385
    for edge in (16383, 16384, 16385):
        k = np.full(200, edge - 1)
        n = k + rng.integers(0, 8 * (edge - 1), 200)                     # k + 1 at the edge, n from k to 9 k
        parts.append((n, k, rng.choice(P_HALVINGS, 200)))
        p = rng.choice(P_HALVINGS, 200)
        k2 = np.rint(p * (edge - 1) / (1 - p) + rng.normal(0, 1, 200) * 20).clip(1).astype(np.int64)
        parts.append((k2 + edge - 1, k2, p))                            # n - k + 1 at the edge, k near n p
    # log1term around the underflow cut (-740.7) and through exp's denormal range (-708.4 .. -744.4)
    cand_n = rng.integers(200, 6000, 40000)
    cand_p = rng.choice(P_HALVINGS, len(cand_n))
    cand_k = (rng.uniform(0, 1, len(cand_n)) * cand_n).astype(np.int64)
    lt = _log1term(cand_n, cand_k, cand_p, True)
    sel = (lt > -750) & (lt < -700)
    parts.append((cand_n[sel], cand_k[sel], cand_p[sel]))
    n = np.concatenate([a for a, _, _ in parts]).astype(np.int32)
    k = np.concatenate([b for _, b, _ in parts]).astype(np.int32)
    p = np.concatenate([c for _, _, c in parts]).astype(np.float64)
    return n, k, p


@pytest.fixture(scope="module")
def grid():
    return nfa_grid()


def _where_it_broke(n, k, brk):
    """break categories from the oracle's break indices"""
    tail = brk > 0
    off = brk - (k + 1)
    last_block = (n - (k + 1)) // 32
    return dict(
        last_term=tail & (brk == n),
        lane0=tail & (brk <= n) & (off % 32 == 0),
        lane31=tail & (brk <= n) & (off % 32 == 31),
        first_block=tail & (brk <= n) & (off < 32),
        later_block=tail & (brk <= n) & (off >= 32),
        last_partial_block=tail & (brk <= n) & (off // 32 == last_block) & ((n - k) % 32 != 0),
        early_or_underflow=brk == -1)


def test_the_grid_covers_every_branch(oracle, grid):
    """what the grid reaches, on the CPU: the early returns, the underflow branch on both sides of the cut, breaks at lane 0 and lane 31, in
    the first, a later and the last partial block of 32 terms and at the last term, and log_gamma past the device table.  (At p <= 1/8 a
    tail that runs past its first 32 terms breaks soon after the terms start to fall: none on this grid breaks in a partial last block
    behind full ones.)  (A tail that
    reaches i = n always stops there: the remainder bound of its last term is 0.  So no triple runs off the end of the loop.)"""
    n, k, p = grid
    assert len(n) > 700000
    for first in (True, False):
        val, brk = oracle.lsd_nfa_many(n, k, p, LOG_NTS["vga"], first)
        cats = _where_it_broke(n, k, brk)
        for name, m in cats.items():
            assert m.sum() >= 10, (first, name, int(m.sum()))
        assert np.isfinite(val).all() and not (brk == n + 1).any()
    lt = _log1term(n, k, p, True)
    assert ((lt > -740.7) & (lt < -738)).sum() >= 10 and ((lt < -740.8) & (lt > -745)).sum() >= 10
    assert ((lt > -744.4) & (lt < -708.4)).sum() >= 100                        # exp lands in the denormals
    assert (k + 1 >= 16384).sum() >= 200 and (n - k + 1 >= 16384).sum() >= 200
    for edge in (16383, 16384, 16385):
        assert (k + 1 == edge).sum() >= 100 and (n - k + 1 == edge).sum() >= 100
    assert n.max() > 900000 and set(np.unique(p)) == set(P_HALVINGS)


@pytest.mark.gpu
def test_device_nfa_equals_the_reference_formula(oracle, grid):
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    n, k, p = grid
    ctx = cs.Context(0, 64, 64, 1, 1, 16)
    worst = {}
    try:
        for form in (True, False):
            for size, lnt in LOG_NTS.items():
                val = np.zeros(len(n))
                brk = np.zeros(len(n), np.int32)
                ctx.check(ctx.L.cs_debug_nfa(ctx.h, _lib.ptr(n, C.c_int32), _lib.ptr(k, C.c_int32), _lib.ptr(p, C.c_double), lnt, int(form),
                                             _lib.ptr(val, C.c_double), _lib.ptr(brk, C.c_int32), len(n)))
                ref, ref_brk = oracle.lsd_nfa_many(n, k, p, lnt, form)
                bad = np.flatnonzero(brk != ref_brk)
                assert len(bad) == 0, ("break index", form, size, len(bad),
                                       [(int(n[i]), int(k[i]), float(p[i]), int(brk[i]), int(ref_brk[i])) for i in bad[:8]])
                rel = np.abs(val - ref) / np.maximum(np.abs(ref), 1e-300)
                i = int(np.argmax(rel))
                worst[(form, size)] = (float(rel[i]), float(np.abs(val - ref).max()), int(n[i]), int(k[i]), float(p[i]))
    finally:
        ctx.close()
    print("largest device - reference NFA difference (relative, absolute, at n, k, p):", worst)
    # far below the 4.75e-7 relative gap of the closest rect_improve comparison seen on real frames.  Measured on an H100 (CUDA 12.9): 5.1e-9
    # relative, in the EDLines form at n = 501 377, where log_gamma(n + 1) comes from the device's log / pow / sinh and the NFA is near 0.16;
    # 9.0e-12 in the LSD form; 1.9e-9 absolute at most
    assert max(w[0] for w in worst.values()) < 1e-8, worst
