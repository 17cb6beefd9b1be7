"""The key-order reference (tests/topk_reference.py) on the CPU: its key order, its decoder, its exactness guard and its
agreement with the C oracle's FLAT search, whose L2 ids are bit-exact including their order."""
import numpy as np
import pytest

import topk_reference as R
from oracle import oracle as orc
from vearch_b200 import synth

L2, IP = R.METRIC_L2, R.METRIC_IP
assert (L2, IP) == (orc.METRIC_L2, orc.METRIC_IP)


def test_f2ord_is_order_preserving_over_the_whole_line():
    tiny = np.float32(np.finfo(np.float32).tiny)
    sub = np.float32(1e-45)  # the smallest subnormal
    vals = np.array([-R.FLT_MAX, -1e30, -1.0, -tiny, -sub, -0.0, 0.0, sub, tiny, 1.0, 1e30, R.FLT_MAX], np.float32)
    o = R.f2ord(vals).astype(np.int64)
    assert (np.diff(o) > 0).all()  # strictly: -0.0 keys before +0.0
    assert R.f2ord(np.float32(0.0)) == 0x80000000 and R.f2ord(np.float32(-0.0)) == 0x7FFFFFFF
    assert np.array_equal(R.ord2f(R.f2ord(vals)).view(np.uint32), vals.view(np.uint32))
    rng = np.random.default_rng(0)
    x = rng.normal(0, 1e3, 10000).astype(np.float32)
    assert np.array_equal(np.argsort(R.f2ord(x), kind="stable"), np.argsort(x, kind="stable"))
    # IP keys: larger score first
    assert (np.diff(R.score2ord(vals, IP).astype(np.int64)) < 0).all()


def test_keys_break_ties_by_smaller_vid_and_decode_reorders_ip_ties():
    s = np.array([[5, 3, 5, 3, 7, 5]])
    vid = np.array([10, 4, 2, 9, 1, 6])
    kl = R.topk(R.keys(s, vid, metric=L2), 8)
    d, i = R.decode(kl, L2)
    assert i.tolist() == [[4, 9, 2, 6, 10, 1, -1, -1]]
    assert d[0, :6].tolist() == [3, 3, 5, 5, 5, 7] and (d[0, 6:] == np.float32(R.FLT_MAX)).all()
    ki = R.topk(R.keys(s, vid, metric=IP), 8)
    assert ((ki[0, :6] & np.uint64(0xFFFFFFFF)).astype(int).tolist()) == [1, 2, 6, 10, 4, 9]  # key order
    d, i = R.decode(ki, IP)
    assert i.tolist() == [[1, 10, 6, 2, 9, 4, -1, -1]]  # decoder: larger id first inside a tie group
    assert d[0, :6].tolist() == [7, 5, 5, 5, 3, 3] and (d[0, 6:] == np.float32(-R.FLT_MAX)).all()
    # invalid entries become the sentinel; a row with fewer entries than k is sentinel padded
    kv = R.topk(R.keys(s, vid, valid=np.array([[True, False, True, False, True, True]]), metric=L2), 5)
    assert R.decode(kv, L2)[1].tolist() == [[2, 6, 10, 1, -1]]
    assert R.topk(np.zeros((2, 0), np.uint64), 3).tolist() == [[int(R.SENTINEL)] * 3] * 2


def test_exact_zero_is_positive_zero():
    # IP of mixed-sign rows: an exact zero must key as +0.0, between the negative and the positive scores
    xq = np.array([[1, -1, 0, 0]], np.float32)
    db = np.array([[1, 1, 0, 0], [2, 0, 0, 0], [0, 3, 0, 0], [0, 0, 0, 0], [5, 5, 1, 1]], np.float32)
    kk = R.flat_keys(xq, db, 5, IP)
    d, i = R.decode(kk, IP)
    assert d.view(np.uint32)[0].tolist() == np.array([2, 0, 0, 0, -3], np.float32).view(np.uint32).tolist()
    assert i.tolist() == [[1, 4, 3, 0, 2]]  # the +0.0 group {0, 3, 4} listed larger id first


def test_guard_fires():
    with pytest.raises(R.InexactScores):
        R.keys(np.array([1 << 24]), np.array([0]))
    with pytest.raises(R.InexactScores):
        R.exact_scores(np.full((1, 4), 3000, np.float32), np.zeros((2, 4), np.float32), L2)
    with pytest.raises(R.InexactScores):  # partial sums of an IP can exceed its (cancelled) final value
        R.exact_scores(np.array([[3000, 3000]], np.float32), np.array([[3000, -3000]], np.float32), IP)
    with pytest.raises(R.InexactScores):
        R.exact_scores(np.array([[0.5]], np.float32), np.array([[1]], np.float32), IP)
    with pytest.raises(TypeError):
        R.keys(np.array([1.0]), np.array([0]))  # float64 scores: no float32 image chosen


@pytest.mark.parametrize("ties", [False, True])
def test_flat_l2_matches_oracle_exactly(ties):
    d, n, nq = 32, 3000, 12
    if ties:
        pool = np.random.default_rng(3).integers(0, 4, (16, d)).astype(np.float32)
        db = pool[np.random.default_rng(4).integers(0, 16, n)]
        xq = pool[np.random.default_rng(5).integers(0, 16, nq)]
    else:
        db, xq = synth.sift_like(n, d, seed=11), synth.sift_like(nq, d, seed=12)
    deleted = np.random.default_rng(6).random(n) < 0.3
    delb = np.packbits(deleted, bitorder="little")
    for k, kw in [(1, {}), (10, {}), (257, {}), (n + 5, {}), (100, {"del_bitmap": delb})]:
        do, io = orc.flat_search(db, xq, k, L2, **kw)
        dr, ir = R.decode(R.flat_keys(xq, db, k, L2, **kw), L2)
        assert np.array_equal(dr.view(np.uint32), do.view(np.uint32)) and np.array_equal(ir, io), (k, kw)


def test_unpack_codes_matches_bit_layout():
    rng = np.random.default_rng(7)
    for M, nbits in [(8, 1), (12, 3), (16, 4), (10, 7)]:
        codes = rng.integers(0, 1 << nbits, (50, M))
        bits = ((codes[:, :, None] >> np.arange(nbits)) & 1).reshape(50, -1).astype(np.uint8)
        packed = np.packbits(bits, axis=1, bitorder="little")
        assert packed.shape[1] == (M * nbits + 7) // 8
        assert np.array_equal(R.unpack_codes(packed, M, nbits), codes)
