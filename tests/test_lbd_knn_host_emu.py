"""The knn / radius matching kernels without a GPU: k_lbd_knn2 and k_lbd_match_sorted (cube_slam_b200/csrc/cs_lbd_kernels.cuh) compiled
from their own source against the emulation of the CUDA execution model the descriptor kernels' CPU tests use (tests/host_core/cuda_emu.h
through tests/host_core/lbd_knn_emu.cpp: a thread per CUDA thread, a barrier per __syncthreads, shuffles through a block-wide array) and run
launch by launch.  What each launch writes -- keys in order, per-query counts, the counting launch and the offset-driven one -- must be the
oracle's knnMatch / radiusMatch answer (oracle/lbd_knn_oracle.cpp, pinned to the reference by tests/test_oracle_ref_lbd_knn.py), on uneven
batches with empty pairs and on pairs at the 16384-code bound."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle_knn as K

HERE = os.path.dirname(os.path.abspath(__file__))
NEVER = np.uint64(0xFFFFFFFFFFFFFFFF)


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "host_core", "lbd_knn_emu.cpp")
    deps = [src, os.path.join(HERE, "host_core", "cuda_emu.h")] + [os.path.join(HERE, "..", "cube_slam_b200", "csrc", f) for f in ("cs_lbd_core.h", "cs_lbd_kernels.cuh")]
    out = os.path.join(HERE, "host_core", "_build", "liblbdknnemu.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-std=c++20", "-O2", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-o", out, src])
    return C.CDLL(out)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _batch(pairs):
    qo = np.concatenate([[0], np.cumsum([len(q) for q, _ in pairs])]).astype(np.int32)
    to = np.concatenate([[0], np.cumsum([len(t) for _, t in pairs])]).astype(np.int32)
    q = np.concatenate([q for q, _ in pairs] + [np.zeros((1, 32), np.uint8)])      # one spare row: never an empty buffer
    t = np.concatenate([t for _, t in pairs] + [np.zeros((1, 32), np.uint8)])
    pq = np.repeat(np.arange(len(pairs), dtype=np.int32), np.diff(qo))
    return np.ascontiguousarray(q), qo, np.ascontiguousarray(t), to, np.ascontiguousarray(pq)


def _entries(keys):
    keys = np.asarray(keys, np.uint64)
    d = (keys >> np.uint64(48)).astype(np.int64)
    ti = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    return np.where(d <= 128, ti, -1).astype(np.int32), d.astype(np.float32)


def run_knn2(emu, pairs):
    q, qo, t, to, pq = _batch(pairs)
    nq = int(qo[-1])
    keys = np.zeros(2 * max(nq, 1), np.uint64)
    emu.emu_lbd_knn2(C.c_void_p(q.ctypes.data), C.c_void_p(t.ctypes.data), _p(pq, C.c_int32), _p(to, C.c_int32), nq, _p(keys, C.c_uint64))
    return keys[:2 * nq].reshape(nq, 2), qo


def run_sorted(emu, pairs, max_dist, room):
    """the library's two launches: counts, then the keys at offsets that give query i room[i] slots (None: its count)"""
    q, qo, t, to, pq = _batch(pairs)
    nq = int(qo[-1])
    cnt = np.full(max(nq, 1), -7, np.int32)
    emu.emu_lbd_match_sorted(C.c_void_p(q.ctypes.data), C.c_void_p(t.ctypes.data), _p(pq, C.c_int32), _p(to, C.c_int32), nq, max_dist, None, None, _p(cnt, C.c_int32))
    first = cnt[:nq].copy()
    slots = first if room is None else np.asarray(room, np.int64)
    off = np.concatenate([[0], np.cumsum(slots)]).astype(np.int64)
    keys = np.full(max(int(off[-1]), 1), 7, np.uint64)
    cnt2 = np.full(max(nq, 1), -7, np.int32)
    emu.emu_lbd_match_sorted(C.c_void_p(q.ctypes.data), C.c_void_p(t.ctypes.data), _p(pq, C.c_int32), _p(to, C.c_int32), nq, max_dist, _p(off, C.c_int64), _p(keys, C.c_uint64),
                             _p(cnt2, C.c_int32))
    return first, [keys[off[i]:off[i] + cnt2[i]] for i in range(nq)], cnt2[:nq], qo


def _pairs(rng, shapes):
    out = []
    for nq, nt in shapes:
        t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
        q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
        for i in range(nq):
            if nt and rng.random() < 0.8:
                q[i] = t[int(rng.integers(0, nt))]
                flips = rng.integers(0, 256, int(rng.integers(0, 140)))
                np.bitwise_xor.at(q[i], flips // 8, (1 << (flips % 8)).astype(np.uint8))
        if nt > 3:
            t[nt - 1] = t[1]                                  # duplicates: bucket order decides
        out.append((q, t))
    return out


SHAPES = [(5, 17), (0, 9), (4, 0), (1, 1), (9, 300), (3, 2), (12, 61)]


def test_knn2_launch_equals_the_oracle(emu, oracle):
    pairs = _pairs(np.random.default_rng(1), SHAPES)
    keys, qo = run_knn2(emu, pairs)
    for p, (q, t) in enumerate(pairs):
        want = K.lbd_knn_match(q, t, 2) if len(t) else [(np.zeros(0),) * 3] * len(q)
        for i in range(len(q)):
            k = keys[qo[p] + i]
            k = k[k != NEVER]
            ti, d = _entries(k)
            np.testing.assert_array_equal(ti, want[i][1])
            np.testing.assert_array_equal(d, want[i][2])


@pytest.mark.parametrize("k", [1, 3, 5, 64])
def test_sorted_launch_knn_equals_the_oracle(emu, oracle, k):
    pairs = _pairs(np.random.default_rng(2 + k), SHAPES)
    nts = [len(t) for q, t in pairs for _ in range(len(q))]
    rng = np.random.default_rng(k)
    keep = rng.random(len(nts)) < 0.8
    room = [min(k, nt) if kp else 0 for nt, kp in zip(nts, keep)]      # the knn call's slots; a masked query has none
    _, got, cnt, qo = run_sorted(emu, pairs, 256, room)
    for p, (q, t) in enumerate(pairs):
        want = K.lbd_knn_match(q, t, k) if len(t) else [(np.zeros(0),) * 3] * len(q)
        for i in range(len(q)):
            g = qo[p] + i
            if not keep[g]:
                assert cnt[g] == 0
                continue
            ti, d = _entries(got[g])
            np.testing.assert_array_equal(ti, want[i][1])
            np.testing.assert_array_equal(d, want[i][2])


@pytest.mark.parametrize("r", [0, 25, 128, 256, -1])
def test_sorted_launch_radius_equals_the_oracle(emu, oracle, r):
    pairs = _pairs(np.random.default_rng(40 + r), SHAPES)
    first, got, cnt, qo = run_sorted(emu, pairs, r, None)
    np.testing.assert_array_equal(first, cnt)
    for p, (q, t) in enumerate(pairs):
        want = K.lbd_radius_match(q, t, float(r))
        for i in range(len(q)):
            ti, d = _entries(got[qo[p] + i])
            np.testing.assert_array_equal(ti, want[i][1])
            np.testing.assert_array_equal(d, want[i][2])


def test_pairs_at_the_shared_memory_bound(emu, oracle):
    """16384 train codes in one pair, every one of them met: the sort fills all of its staging; knn takes all and radius 256 all"""
    n = emu.emu_lbd_knn_max_train()
    assert n == 16384
    rng = np.random.default_rng(77)
    t = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    q = np.stack([t[5], t[9000]])
    t[:, 0] = q[0, 0]                                       # byte 0 equal to query 0's: every code is met by query 0
    t[n - 1] = t[3]
    pairs = [(q, t), (q[:1], t[:10])]
    _, got, cnt, qo = run_sorted(emu, pairs, 256, [n, n, 10])
    want = K.lbd_knn_match(q, t, n)
    assert cnt[0] == n
    for i in range(2):
        ti, d = _entries(got[i])
        np.testing.assert_array_equal(ti, want[i][1])
        np.testing.assert_array_equal(d, want[i][2])
    ti, d = _entries(got[2])
    np.testing.assert_array_equal(ti, K.lbd_knn_match(q[:1], t[:10], 10)[0][1])
    first, got, cnt, qo = run_sorted(emu, pairs, 25, None)
    want = K.lbd_radius_match(q, t, 25.0)
    for i in range(2):
        ti, d = _entries(got[i])
        np.testing.assert_array_equal(ti, want[i][1])
        np.testing.assert_array_equal(d, want[i][2])
