"""SOAR spilling without a GPU (DESIGN.md §8, SOAR spilling): the fp64 twin of the spilled-list choice (oracle_soar), the 2 k' - 1
containment the duplicate-free selection rests on, and the spilled index file layout (tests/soar_index_file.py)."""
import struct

import numpy as np
import pytest

from oracle_soar import soar
import quantised_index_file as qf
import soar_index_file as sf


def rows_and_centroids(seed, n=200, nlist=16, d=8):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((nlist, d)).astype(np.float32)
    x = rng.standard_normal((n, d)).astype(np.float32)
    primary = np.argmin(((x[:, None, :].astype(np.float64) - c[None]) ** 2).sum(-1), axis=1)
    return x, c, primary


@pytest.mark.parametrize("lam", [0.0, 1.5, 10.0])
def test_spilled_list_is_never_the_primary(lam):
    x, c, primary = rows_and_centroids(1)
    s = soar.spill_lists(x, c, primary, lam)
    assert np.all(s != primary)
    assert np.all((s >= 0) & (s < len(c)))


def test_lambda_zero_picks_the_second_nearest_list():
    x, c, primary = rows_and_centroids(2)
    s = soar.spill_lists(x, c, primary, 0.0)
    dist = ((x[:, None, :].astype(np.float64) - c[None]) ** 2).sum(-1)
    second = np.argsort(dist, axis=1, kind="stable")[:, 1]
    assert np.array_equal(s, second)


def test_large_lambda_prefers_orthogonal_residuals():
    # x = (1, 0); primary c0 = (0, 0), r = (1, 0).  c1 = (2, 0) is as near as c2 = (1, 1), but r' = x - c1 is parallel to
    # r and r' = x - c2 orthogonal: lambda > 0 picks c2
    x = np.array([[1, 0]], np.float32)
    c = np.array([[0, 0], [2, 0], [1, 1]], np.float32)
    assert soar.spill_lists(x, c, [0], 0.0)[0] == 1  # a tie at lambda 0: the lower id
    assert soar.spill_lists(x, c, [0], 1.5)[0] == 2


def test_ties_go_to_the_lowest_id():
    # x = (0.25, 0), primary c0 = (0, 0): c1 and c2 mirror each other across r, so their losses are equal; c3 is far
    x = np.array([[0.25, 0.0]], np.float32)
    c = np.array([[0.0, 0.0], [0.25, 1.0], [0.25, -1.0], [5, 5]], np.float32)
    loss = soar.spill_loss(x, c, [0], 1.5)[0]
    assert loss[1] == loss[2] < loss[3]
    assert soar.spill_lists(x, c, [0], 1.5)[0] == 1
    c_swapped = c[[0, 2, 1, 3]]
    assert soar.spill_lists(x, c_swapped, [0], 1.5)[0] == 1


def test_zero_residual_takes_the_fallback():
    x = np.zeros((1, 2), np.float32)
    c = np.array([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], np.float32)
    assert soar.spill_lists(x, c, [0], 1.5, vid0=7)[0] == 7 % 5  # |r| = 0: list gvid % nlist
    c_moved = c[[2, 1, 0, 3, 4]]
    assert soar.spill_lists(x, c_moved, [2], 1.5, vid0=7)[0] == 3  # gvid % nlist = 2 is the primary: the next list


def test_non_finite_rows_take_the_fallback():
    x, c, primary = rows_and_centroids(3, n=4)
    x[1, 0] = np.nan
    x[2, 3] = np.inf
    s = soar.spill_lists(x, c, primary, 1.5, vid0=100)
    for i in (1, 2):
        assert s[i] == soar.fallback_list(100 + i, primary[i], len(c))


def test_margin_accepts_the_twin_and_rejects_a_far_list():
    x, c, primary = rows_and_centroids(4)
    s = soar.spill_lists(x, c, primary, 1.5)
    assert soar.check_spill(x, c, primary, 1.5, s) == []
    loss = soar.spill_loss(x, c, primary, 1.5)
    worst = np.argmax(np.where(np.isfinite(loss), loss, -np.inf), axis=1)
    assert len(soar.check_spill(x, c, primary, 1.5, worst)) > len(x) // 2
    assert soar.check_spill(x, c, primary, 1.5, primary) == list(range(len(x)))


def entries_with_duplicates(rng, nvid, score_levels):
    """every vid one or two entries, scores from few levels (heavy ties), the copies' scores independent"""
    vids, scores = [], []
    for v in rng.permutation(nvid):
        for _ in range(1 + int(rng.integers(0, 2))):
            vids.append(int(v))
            scores.append(int(rng.integers(0, score_levels)))
    return np.array(vids), np.array(scores)


@pytest.mark.parametrize("seed,nvid,levels,k", [(0, 50, 3, 10), (1, 300, 1, 100), (2, 3000, 7, 1), (3, 5000, 40, 2048),
                                                (4, 40, 2, 64)])
def test_first_two_k_minus_one_keys_hold_the_best_copy_top_k(seed, nvid, levels, k):
    rng = np.random.default_rng(seed)
    vids, scores = entries_with_duplicates(rng, nvid, levels)
    keys = soar.make_keys(scores, vids)
    want = soar.topk_best_copy(vids, keys, k)
    keys = np.sort(keys)
    for depth in (2 * k - 1, 2 * k):
        assert np.array_equal(soar.dedupe_first(keys[:depth], k), want)


def test_two_k_minus_two_keys_are_not_enough():
    # k - 1 vids with both copies ahead of the k-th vid: it is key 2k - 1
    k = 5
    vids = np.array([v for v in range(k - 1) for _ in range(2)] + [k - 1])
    scores = np.arange(len(vids))
    keys = soar.make_keys(scores, vids)
    want = soar.topk_best_copy(vids, keys, k)
    assert want[-1] == keys[2 * k - 2]
    assert not np.array_equal(soar.dedupe_first(keys[:2 * k - 2], k), want)
    assert np.array_equal(soar.dedupe_first(keys[:2 * k - 1], k), want)


def test_dedupe_keeps_sentinel_padding():
    keys = np.array(list(soar.make_keys([1, 1, 2], [7, 7, 3])) + [soar.SENTINEL] * 3, np.uint64)
    got = soar.dedupe_first(keys, 3)
    assert list(got) == [keys[0], keys[2], soar.SENTINEL]


# ---- the spilled index file ---------------------------------------------------------------------------------------
def spilled_case(kind, metric, lam=1.5):
    buf, table, want = __import__("test_persist_quantised_cpu").case(kind, metric)
    codec = {k: want[k] for k in ("pq_centroids", "nb_bits", "qb", "nsub", "blocks", "ns_threshold", "reordering",
                                  "codebook") if k in want}
    sbuf = sf.write_spilled(kind, table["d"], metric, 3, want["centroids"], want["list_off"], want["codes"], want["ids"], 31,
                            want["code_size"], lam, **codec)
    return buf, sbuf, dict(table, soar_lambda=lam), want


KINDS = [(k, m) for k in ("IVFPQFastScan", "IVFRABITQ", "VEARCH") for m in (qf.METRIC_L2, qf.METRIC_IP)]


@pytest.mark.parametrize("kind,metric", KINDS)
def test_spilled_file_layout(kind, metric):
    buf, sbuf, table, want = spilled_case(kind, metric)
    # the unspilled file with the variant fourcc and the lambda after the codec block
    assert sbuf[:4] == sf.MAGIC[kind].encode() and buf[:4] == qf.MAGIC[kind].encode()
    at = sf._codec_end(buf, kind, table)
    assert buf[at:at + 4] == b"ilar"
    assert sbuf[4:at] == buf[4:at] and sbuf[at:at + 8] == struct.pack("<d", 1.5) and sbuf[at + 8:] == buf[at:]
    got = sf.read_spilled(sbuf, kind, table)
    for key in ("centroids", "list_off", "codes", "ids"):
        assert np.array_equal(got[key], want[key]), key
    assert got["soar_lambda"] == 1.5 and got["indexed_count"] == 31


@pytest.mark.parametrize("kind,metric", KINDS)
def test_each_kind_refuses_the_others_file(kind, metric):
    buf, sbuf, table, _ = spilled_case(kind, metric)
    with pytest.raises(ValueError, match="magic"):
        qf.read_quantised(sbuf, kind, table)
    with pytest.raises(ValueError, match="magic"):
        sf.read_spilled(buf, kind, table)
    with pytest.raises(ValueError, match="soar_lambda"):
        sf.read_spilled(sbuf, kind, dict(table, soar_lambda=2.0))
    with pytest.raises(ValueError):
        sf.read_spilled(sbuf[:sf._codec_end(buf, kind, table) + 4], kind, table)
