"""IVF-PQ list-major search with phase B's pair grouping and operand staging on a side stream beside phase A, and the
filter thresholds bound to phase A's keys afterwards (pq_bind_bounds_kernel).  Every case compares the list-major
batch key for key with the query-major LUT kernel (the same index searched three queries at a time): deletion and
filter bitmaps, queries whose phase A finds fewer than k' entries, the adversarial scales of the int8 filter, two host
threads searching one index at once, and batches that decline the list-major path (the inner-product table is then
built by the query-major path)."""
import threading

import numpy as np
import pytest

import float_contract as FC
from test_gpu_float_accuracy import IvfPq, pq_data
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = FC.METRIC_L2, FC.METRIC_IP
METRICS = [L2, IP]


def list_major(s, k, q=slice(None), **kw):
    got = s.search(k, q, **kw)
    assert s.idx.last_scan_kernel == "pqtc_scan_kernel", s.idx.last_scan_kernel
    return got


def query_major(s, k, nq, **kw):
    parts = []
    for q0 in range(0, nq, 3):  # 3 x nprobe pairs: far below 32 per list
        parts.append(s.search(k, slice(q0, min(q0 + 3, nq)), **kw))
        assert s.idx.last_scan_kernel == "ivfpq_scan_kernel", s.idx.last_scan_kernel
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def assert_same(got, want, what):
    dg, ig = got
    dw, iw = want
    bad = np.nonzero(np.any(dg.view(np.uint32) != dw.view(np.uint32), 1) | np.any(ig != iw, 1))[0]
    assert len(bad) == 0, (f"{what}: {len(bad)}/{len(dg)} queries differ from the LUT kernel; query {bad[0]}: "
                           f"{ig[bad[0]][:5]} vs {iw[bad[0]][:5]}")


def sift_index(metric, nq=128, seed=11):
    d, n = 128, 20000
    db = synth.sift_like(n, d, seed=seed)
    xq = synth.sift_like(nq, d, seed=seed + 1)
    return IvfPq(db, xq, 16, 16, 6, metric, seed=7), n


@pytest.mark.parametrize("metric", METRICS)
def test_bitmaps(metric):
    s, n = sift_index(metric)
    rng = np.random.default_rng(3)
    try:
        cases = [("del", {"del_bitmap": np.packbits(rng.random(n) < 0.3, bitorder="little")}),
                 ("filter", {"filter_bitmap": np.packbits(rng.random(n) < 0.5, bitorder="little")}),
                 ("both", {"del_bitmap": np.packbits(rng.random(n) < 0.2, bitorder="little"),
                           "filter_bitmap": np.packbits(rng.random(n) < 0.6, bitorder="little")})]
        for name, kw in cases:
            for k in (10, 100):
                assert_same(list_major(s, k, **kw), query_major(s, k, len(s.xq), **kw), f"{name} k={k}")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_queries_without_bound(metric):
    """all but 5 rows of every other list deleted: phase A plans from list lengths, which count deleted rows, so a query
    whose first probe is such a list scans that list alone there, finds fewer than k' = 10 valid entries and has no
    bound; the other queries keep theirs"""
    s, n = sift_index(metric)
    try:
        off, _, ids = s.idx.export_lists()
        dead = np.zeros(n, bool)
        for l in range(0, len(off) - 1, 2):
            dead[ids[off[l] + 5:off[l + 1]]] = True
        assert (s.probes[:, 0] % 2 == 0).any() and (s.probes[:, 0] % 2 == 1).any()
        kw = {"del_bitmap": np.packbits(dead, bitorder="little")}
        assert_same(list_major(s, 10, **kw), query_major(s, 10, len(s.xq), **kw), "no bound")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", ["offset1000", "scaled_hi30", "scaled_lo30", "codebook_span", "subnormal"])
def test_adversarial_scales(name, metric):
    db, xq, span = pq_data(name, 128, 20000, 128, seed=1608)
    s = IvfPq(db, xq, 16, 16, 6, metric, seed=7, span=span)
    try:
        for k in (10, 100):
            assert_same(list_major(s, k), query_major(s, k, len(xq)), f"{name} k={k}")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_two_threads(metric):
    """two host threads (each with its own search stream, side stream and scratch) search one index at once"""
    s, _ = sift_index(metric, nq=256)
    try:
        halves = [slice(0, 128), slice(128, 256)]
        want = [list_major(s, 100, q) for q in halves]
        assert_same(want[0], query_major(s, 100, 128), "first half, one thread")
        got, errors = [[None] * 4, [None] * 4], []

        def run(t):
            try:
                for rep in range(4):
                    got[t][rep] = s.search(100, halves[t])
            except Exception as e:  # noqa: BLE001 -- reported below
                errors.append(e)

        threads = [threading.Thread(target=run, args=(t,)) for t in range(2)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errors, errors
        for t in range(2):
            for rep in range(4):
                assert_same(got[t][rep], want[t], f"thread {t} search {rep}")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_declined_batch_builds_ip(metric):
    """k' = 2049 declines the list-major path on a list-major-sized batch; a small batch declines it too.  Both scan with
    the query-major kernel, which reads the inner-product table"""
    s, _ = sift_index(metric)
    try:
        full = s.search(2049)
        assert s.idx.last_scan_kernel == "ivfpq_scan_kernel", s.idx.last_scan_kernel
        assert_same(full, query_major(s, 2049, len(s.xq)), "k'=2049")
        lm = list_major(s, 100)
        small = s.search(100, slice(0, 3))
        assert s.idx.last_scan_kernel == "ivfpq_scan_kernel", s.idx.last_scan_kernel
        assert_same(small, (lm[0][:3], lm[1][:3]), "small batch after a list-major one")
    finally:
        s.idx.close()
