"""The numpy restatement of the list purge (oracle_purge) on hand-built lists: what is live, which lists are chosen, and
what a purge leaves behind."""
import numpy as np

from oracle_purge import purge as P

T = P.TOMBSTONE


def lists3():
    """three lists: [0, 1, 2, 3], [4, 5], [] with one byte of code per entry (the code is the entry's ordinal)"""
    off = np.array([0, 4, 6, 6], np.int64)
    ids = np.array([10, 11, 12, 13, 20, 21], np.int64)
    codes = np.arange(6, dtype=np.uint8).reshape(6, 1)
    return off, codes, ids


def test_live_is_no_tombstone_and_no_bitmap_bit():
    ids = np.array([0, 9 | T, 9, 17, 40], np.int64)
    assert P.live(ids).tolist() == [True, False, True, True, True]
    bm = P.bitmap_of([9, 17], 24)
    assert bm.tolist() == [0, 2, 2]  # LSB first
    assert P.live(ids, bm).tolist() == [True, False, False, False, True]  # 40 lies beyond the bitmap: not deleted


def test_tombstones_only():
    off, codes, ids = lists3()
    ids[1] |= T
    ids[3] |= T
    o, c, i, dropped = P.purge(off, codes, ids, [0, 1, 2])
    assert o.tolist() == [0, 2, 4, 4] and i.tolist() == [10, 12, 20, 21] and c[:, 0].tolist() == [0, 2, 4, 5]
    assert dropped == 2


def test_bitmap_only():
    off, codes, ids = lists3()
    o, c, i, dropped = P.purge(off, codes, ids, [0, 1], P.bitmap_of([10, 21], 32))
    assert o.tolist() == [0, 3, 4, 4] and i.tolist() == [11, 12, 13, 20] and c[:, 0].tolist() == [1, 2, 3, 4]
    assert dropped == 2


def test_both_and_unselected_lists_keep_their_dead():
    off, codes, ids = lists3()
    ids[0] |= T
    ids[4] |= T
    bm = P.bitmap_of([12, 21], 32)
    o, c, i, dropped = P.purge(off, codes, ids, [0], bm)
    assert o.tolist() == [0, 2, 4, 4] and dropped == 2
    assert i.tolist() == [11, 13, 20 | T, 21]  # list 1 untouched: its tombstone and its deleted doc stay
    assert c[:, 0].tolist() == [1, 3, 4, 5]


def test_all_dead_and_none_dead():
    off, codes, ids = lists3()
    o, c, i, dropped = P.purge(off, codes, ids, [0, 1, 2])
    assert dropped == 0 and np.array_equal(o, off) and np.array_equal(i, ids) and np.array_equal(c, codes)
    ids[:4] |= T
    o, c, i, dropped = P.purge(off, codes, ids, [0], P.bitmap_of([20, 21], 32))
    assert o.tolist() == [0, 0, 2, 2] and i.tolist() == [20, 21] and dropped == 4
    o, c, i, dropped = P.purge(off, codes, ids, [0, 1], P.bitmap_of([20, 21], 32))
    assert o.tolist() == [0, 0, 0, 0] and len(i) == 0 and c.shape == (0, 1) and dropped == 6


def test_threshold_is_inclusive_in_float32():
    lens = np.array([10, 10, 10, 0, 1000, 7])
    dead = np.array([3, 2, 0, 0, 299, 7])
    assert P.select_lists(dead, lens, 0.3).tolist() == [0, 5]  # 3 / 10 >= 0.3f, 2 / 10 and 299 / 1000 are not
    assert P.select_lists(dead, lens, 0.0).tolist() == [0, 1, 4, 5]  # 0: every list with a dead entry
    assert P.select_lists(dead, lens, 1.0).tolist() == [5]
    assert np.float32(3) / np.float32(10) >= np.float32(0.3)


def test_positions_follow_the_purge():
    off, codes, ids = lists3()
    ids[0] |= T  # vid 10 was updated: its live entry is the second one of list 1
    ids[5] = 10
    pos = P.vid_positions(off, ids, 24)
    assert pos[10] == (1 << 32 | 1) and pos[11] == 1 and pos[21] == -1
    o, c, i, _ = P.purge(off, codes, ids, [0, 1], P.bitmap_of([20], 24))
    pos = P.vid_positions(o, i, 24)
    assert pos[10] == (1 << 32 | 0) and pos[11] == 0 and pos[13] == 2 and pos[20] == -1
