"""Sharding of GPU_IVFPQ / GPU_IVFFLAT restated in numpy (index_shards.cu): global vid v lives in shard v % S as local
vid v / S; a vid bitmap is cut into S per-shard bitmaps (split_bitmap_kernel); the shards' sorted result keys are
merged by (score, global vid) (merge_shard_keys_kernel); a dumped list is the merge of its shard segments by global
vid (ShardedIndex::dump_gamma).  No GPU needed."""
import numpy as np
import pytest

SENT = np.uint64(0xFFFFFFFFFFFFFFFF)


def to_local(v, S):
    return v % S, v // S


def to_global(s, local, S):
    return local * S + s


def split_bitmap(words, bits, S):
    """split_bitmap_kernel: dst[s] bit j = src bit j * S + s, for j * S + s < bits"""
    nw = ((bits + S - 1) // S + 31) // 32 + 1
    src = np.unpackbits(words.view(np.uint8), bitorder="little")[:bits]
    out = np.zeros((S, nw * 32), np.uint8)
    for s in range(S):
        sel = src[s::S]
        out[s, :len(sel)] = sel
    return np.packbits(out, axis=1, bitorder="little").view(np.uint32)


def shard_key(key, S, s):
    if key == SENT:
        return key
    return np.uint64((int(key) & 0xFFFFFFFF00000000) | ((int(key) & 0xFFFFFFFF) * S + s))


def merge_keys(rows, k):
    """merge_shard_keys_kernel for one query: rows[s] = k sorted keys with local vids, sentinel padded; each key's
    place = its place in its row + the keys below it in every other row"""
    S = len(rows)
    out = np.full(k, SENT, np.uint64)
    g = [np.array([shard_key(x, S, s) for x in rows[s]], np.uint64) for s in range(S)]
    for s in range(S):
        for p, key in enumerate(g[s]):
            if key == SENT:
                break
            rank = p + sum(int(np.searchsorted(g[r], key, side="left")) for r in range(S) if r != s)
            if rank < k:
                out[rank] = key
    return out


def merge_dump_list(segments, S):
    """ShardedIndex::dump_gamma: the smallest head by global vid first (ties to the lower shard), each segment kept in
    its own order; ids global, tombstone bit kept"""
    mask = 1 << 63
    segs = [[((i & ~mask) * S + s) | (i & mask) for i in seg] for s, seg in enumerate(segments)]
    head, out = [0] * S, []
    while any(head[s] < len(segs[s]) for s in range(S)):
        best = min((s for s in range(S) if head[s] < len(segs[s])), key=lambda s: (segs[s][head[s]] & ~mask, s))
        out.append(segs[best][head[best]])
        head[best] += 1
    return out


def key_of(score_ord, vid):
    return np.uint64((int(score_ord) << 32) | int(vid))


@pytest.mark.parametrize("S", [1, 2, 3, 4, 7])
def test_vid_mapping_is_a_bijection_and_monotone(S):
    v = np.arange(10007)
    s, local = to_local(v, S)
    assert np.array_equal(to_global(s, local, S), v)
    for sh in range(S):  # local order is global order inside a shard
        assert np.all(np.diff(v[s == sh]) > 0) and np.array_equal(local[s == sh], np.arange((s == sh).sum()))


@pytest.mark.parametrize("S", [2, 3, 4, 8])
@pytest.mark.parametrize("bits", [1, 31, 32, 33, 1000, 4099])
def test_bitmap_split(S, bits):
    rng = np.random.default_rng(bits * 10 + S)
    words = rng.integers(0, 2**32, (bits + 31) // 32 + 1, dtype=np.uint64).astype(np.uint32)
    out = split_bitmap(words, bits, S)
    src = np.unpackbits(words.view(np.uint8), bitorder="little")
    for v in range(bits + 3 * S):
        s, j = to_local(v, S)
        got = (out[s, j >> 5] >> np.uint32(j & 31)) & 1
        assert got == (src[v] if v < bits else 0), (v, s, j)


def unsharded_topk(scores, k):
    """(score ord, vid) ascending: what one index returns, sentinel padded"""
    keys = sorted(key_of(o, v) for v, o in scores.items())
    return np.array((keys + [SENT] * k)[:k], np.uint64)


@pytest.mark.parametrize("S", [2, 3, 4])
@pytest.mark.parametrize("k", [1, 5, 64])
@pytest.mark.parametrize("n", [3, 40, 500])
def test_merge_equals_unsharded_topk_with_ties_and_short_shards(S, k, n):
    rng = np.random.default_rng(S * 1000 + k * 10 + n)
    # few distinct scores: equal scores across shards everywhere; n < S * k leaves shards with fewer than k results
    scores = {v: int(rng.integers(0, 6)) for v in rng.choice(10 * n, n, replace=False)}
    rows = []
    for s in range(S):
        local = {v // S: o for v, o in scores.items() if v % S == s}
        rows.append(unsharded_topk(local, k))
    assert np.array_equal(merge_keys(rows, k), unsharded_topk(scores, k))


def test_merge_all_empty():
    rows = [np.full(4, SENT, np.uint64) for _ in range(3)]
    assert np.all(merge_keys(rows, 4) == SENT)


@pytest.mark.parametrize("S", [2, 3, 4])
def test_dump_merge_after_adds_is_vid_order(S):
    rng = np.random.default_rng(S)
    lists = rng.integers(0, 5, 300)  # each vid's list, added in vid order
    for l in range(5):
        full = [v for v in range(300) if lists[v] == l]  # the unsharded list: insertion = vid order
        segs = [[v // S for v in full if v % S == s] for s in range(S)]
        assert merge_dump_list(segs, S) == full


def test_dump_merge_after_update_is_by_vid():
    S, mask = 2, 1 << 63
    # list holds vids 0..5 (local: shard 0 -> 0, 1, 2; shard 1 -> 0, 1, 2); vid 2 (shard 0, local 1) updated: its old
    # entry tombstoned, the new one appended to the end of shard 0's segment
    segs = [[0, 1 | mask, 2, 1], [0, 1, 2]]
    got = merge_dump_list(segs, S)
    # the unsharded list would end with vid 2 (insertion order); the sharded merge places it by vid where its
    # segment's head allows: shard 0's segment is [0, 2t, 4, 2], shard 1's [1, 3, 5]
    assert got == [0, 1, 2 | mask, 3, 4, 2, 5]
    assert sorted(i & ~mask for i in got) == [0, 1, 2, 2, 3, 4, 5]
