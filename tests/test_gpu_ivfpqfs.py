"""IVFPQFastScan on the H100 against the C restatement in oracle_pqfs (held byte-equal to its numpy twin by the CPU
tests): with shared index state (coarse centroids,
[M][16][dsub] codebook, probe lists) the uint8 tables, (a, b), list codes and distances are byte-equal; ids equal up to
exact ties at the k-th boundary.  Also: filters, L2 coarse search under IP, training on the device, the engine path,
dump / load and searches concurrent with adds."""
import threading

import numpy as np
import pytest

from oracle import oracle as orc
from oracle_pqfs import ivfpqfs as fso
from oracle_pqfs.twin import assert_same_results
from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
L2, IP = orc.METRIC_L2, orc.METRIC_IP


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


def shared_state_index(db, d, M, nlist, metric, seed=0):
    cent, _, _ = orc.kmeans(db[:4000], nlist, niter=5, seed=1234 + seed)
    pq, _ = fso.pq_train(db[:4096], M, niter=5)
    idx = gi().GammaIndex("IVFPQFastScan", d, {"ncentroids": nlist, "nprobe": 8, "nsubvector": M, "metric_type": mt(metric)})
    idx.set_centroids(cent)
    idx.set_pq_centroids(pq)
    idx.add_vectors(db)
    idx.add_pending()
    return idx, cent, pq


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M", [(128, 64), (128, 32), (64, 16), (32, 8), (30, 15), (24, 12)])
@pytest.mark.parametrize("data", ["int", "float"])
def test_shared_state_bit_exact(metric, d, M, data):
    n, nq, nlist = 20000, 40, 64
    db = synth.sift_like(n, d, seed=31, rounded=data == "int")
    xq = synth.sift_like(nq, d, seed=32, rounded=data == "int")
    idx, cent, pq = shared_state_index(db, d, M, nlist, metric)
    assert idx.pq_ksub == 16 and idx.code_size == (M + 1) // 2
    assert np.array_equal(idx.get_pq_centroids(), pq)
    # lists: L2 assignment (IndexFlatL2 quantiser under either metric), packed 4-bit codes of the raw rows
    off, codes, ids = idx.export_lists()
    a = orc.assign(cent, db, L2)
    ooff, order = orc.build_lists(a, nlist)
    assert np.array_equal(off, ooff) and np.array_equal(ids, order)
    want = fso.encode_packed(pq, db)
    assert np.array_equal(codes, want[order])
    assert np.array_equal(idx.pq_encode(db[:500]), want[:500])
    # tables
    lut8, ab = idx.pqfs_lut(xq)
    olut, oab = fso.lut(pq, xq, metric)
    assert np.array_equal(lut8, olut) and np.array_equal(ab.view(np.uint32), oab.view(np.uint32))
    for nprobe in (1, 8, 32):
        _, keys = orc.coarse_search(cent, xq, nprobe, L2)
        cd = np.zeros(keys.shape, np.float32)
        for k in (1, 10, 100):
            dg, ig = idx.search_preassigned(xq, k, keys, cd)
            assert idx.last_scan_kernel == "ivfpqfs_scan_kernel"
            do, io = fso.search_preassigned(off, codes, ids, olut, oab, xq, k, keys, metric, M)
            assert_same_results(dg, ig, do, io)
        if data == "int":  # exact re-rank: integer rows make every fp32 sum exact in any order
            dg, ig = idx.search_preassigned(xq, 10, keys, cd, params={"recall_num": 200})
            do, io = fso.search_preassigned(off, codes, ids, olut, oab, xq, 10, keys, metric, M, recall_num=200, raw=db)
            assert_same_results(dg, ig, do, io)
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M", [(128, 64), (30, 15)])
def test_ctas_scanning_several_lists(metric, d, M):
    """400 queries x 32 probes: every CTA scans several lists (the batch shape of the benchmark), so its TMA ring crosses
    list boundaries: producer and consumer cursors, the per-list id pointer and the tile bookkeeping."""
    n, nq, nlist, nprobe = 20000, 400, 64, 32
    db = synth.sift_like(n, d, seed=35)
    xq = synth.sift_like(nq, d, seed=36)
    idx, cent, pq = shared_state_index(db, d, M, nlist, metric)
    off, codes, ids = idx.export_lists()
    olut, oab = fso.lut(pq, xq, metric)
    _, keys = orc.coarse_search(cent, xq, nprobe, L2)
    keys[7, 5] = -1
    cd = np.zeros(keys.shape, np.float32)
    deleted = np.random.default_rng(6).random(n) < 0.1
    delb = np.packbits(deleted, bitorder="little")
    for k in (10, 100):
        dg, ig = idx.search_preassigned(xq, k, keys, cd, del_bitmap=delb)
        assert idx.last_scan_kernel == "ivfpqfs_scan_kernel" and idx.last_scan_info["probes_per_cta"] > 1
        do, io = fso.search_preassigned(off, codes, ids, olut, oab, xq, k, keys, metric, M, del_bitmap=delb)
        assert_same_results(dg, ig, do, io)
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
def test_filters_tombstones_and_score_window(metric):
    d, M, n, nq, nlist, nprobe, k = 64, 16, 20000, 30, 32, 8, 20
    db = synth.sift_like(n, d, seed=41)
    xq = synth.sift_like(nq, d, seed=42)
    idx, cent, pq = shared_state_index(db, d, M, nlist, metric)
    for vid in range(0, 3000, 7):  # tombstone the old entry, re-append the new row to its list
        idx.update_vector(vid, db[vid + 10000])
    raw = db.copy()
    raw[0:3000:7] = db[10000:13000:7]
    off, codes, ids = idx.export_lists()
    assert (ids < 0).sum() == len(range(0, 3000, 7))
    rng = np.random.default_rng(3)
    deleted, allowed = rng.random(n) < 0.3, rng.random(n) < 0.6
    delb, filb = np.packbits(deleted, bitorder="little"), np.packbits(allowed, bitorder="little")
    _, keys = orc.coarse_search(cent, xq, nprobe, L2)
    keys[3, 2] = -1
    cd = np.zeros(keys.shape, np.float32)
    olut, oab = fso.lut(pq, xq, metric)
    for recall_num in (0, 100):
        kw = dict(del_bitmap=delb, filter_bitmap=filb)
        dg, ig = idx.search_preassigned(xq, k, keys, cd, params={"recall_num": recall_num} if recall_num else None, **kw)
        do, io = fso.search_preassigned(off, codes, ids, olut, oab, xq, k, keys, metric, M, recall_num=recall_num, raw=raw,
                                        **kw)
        assert_same_results(dg, ig, do, io)
        got = ig[ig >= 0]
        assert not deleted[got].any() and allowed[got].all()
        lo, hi = sorted((float(do[0, 2]), float(do[0, 12])))
        dg, ig = idx.search_preassigned(xq, k, keys, cd, params={"recall_num": recall_num} if recall_num else None,
                                        min_score=lo, max_score=hi, **kw)
        do, io = fso.search_preassigned(off, codes, ids, olut, oab, xq, k, keys, metric, M, recall_num=recall_num, raw=raw,
                                        min_score=lo, max_score=hi, **kw)
        assert_same_results(dg, ig, do, io)
        v = dg[ig >= 0]
        assert ((v >= np.float32(lo)) & (v <= np.float32(hi))).all()
    idx.close()


def test_degenerate_table_on_device():
    d, M = 16, 8
    db = synth.sift_like(3000, d, seed=5)
    idx = gi().GammaIndex("IVFPQFastScan", d, {"ncentroids": 8, "nprobe": 8, "nsubvector": M, "metric_type": "L2"})
    idx.set_centroids(orc.kmeans(db, 8, niter=3)[0])
    idx.set_pq_centroids(np.full((M, 16, 2), 7, np.float32))  # every centroid equal: every span 0
    lut8, ab = idx.pqfs_lut(db[:5])
    olut, oab = fso.lut(np.full((M, 16, 2), 7, np.float32), db[:5], L2)
    assert (lut8 == 0).all() and (ab[:, 0] == 1).all()
    assert np.array_equal(lut8, olut) and np.array_equal(ab, oab)
    idx.add_vectors(db)
    idx.add_pending()
    dg, ig = idx.search(db[:5], 10)
    assert (dg == ab[:, 1:2]).all() and (ig >= 0).all()  # accu = 0 for every entry: score = b
    idx.close()


def test_ip_coarse_search_and_training_rank_lists_by_l2():
    d, M, n, nlist = 64, 16, 20000, 64
    db = synth.sift_like(n, d, seed=51)
    xq = synth.sift_like(50, d, seed=52)
    idx = gi().GammaIndex("IVFPQFastScan", d, {"ncentroids": nlist, "nprobe": 8, "nsubvector": M, "metric_type": "InnerProduct",
                                               "training_threshold": 8000})
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    cent = idx.get_centroids()
    norms = np.linalg.norm(cent.astype(np.float64), axis=1)
    assert np.allclose(norms, 1, atol=1e-4)  # spherical k-means under IP
    # unit-norm centroids rank alike under L2 and IP, so only the distances tell the two coarse searches apart here
    # (the next test separates them by their ids, on centroids of unequal norms)
    cd, _ = idx.coarse_search(xq, 8)
    od, _ = orc.coarse_search(cent, xq, 8, L2)
    assert np.allclose(cd, od, rtol=1e-5)
    idx.close()


def test_ip_index_probes_and_assigns_by_l2():
    """Integer centroids of unequal norms set through the hook, on which L2 and IP rankings differ: the probe ids and the
    list membership of an IP index are the L2 ones.  Integer operands keep every coarse distance exact."""
    d, M, n, nlist, nq, nprobe = 64, 16, 20000, 64, 50, 8
    db = synth.sift_like(n, d, seed=53)
    xq = synth.sift_like(nq, d, seed=54)
    cent, _, _ = orc.kmeans(db[:4000], nlist, niter=5)
    cent = np.rint(cent * np.linspace(0.5, 1.5, nlist, dtype=np.float32)[:, None]).astype(np.float32)
    idx = gi().GammaIndex("IVFPQFastScan", d, {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M,
                                               "metric_type": "InnerProduct"})
    idx.set_centroids(cent)
    idx.set_pq_centroids(fso.pq_train(db[:4096], M, niter=3)[0])
    idx.add_vectors(db)
    idx.add_pending()
    cd, keys = idx.coarse_search(xq, nprobe)
    od, ok = orc.coarse_search(cent, xq, nprobe, L2)
    assert_same_results(cd, keys, od, ok)
    _, oi = orc.coarse_search(cent, xq, nprobe, IP)
    assert (np.sort(oi, axis=1) != np.sort(ok, axis=1)).any(axis=1).mean() > 0.5  # the IP probes would differ
    off, _, ids = idx.export_lists()
    lists = np.repeat(np.arange(nlist), np.diff(off))[np.argsort(ids)]
    assert np.array_equal(lists, orc.assign(cent, db, L2))
    assert (lists != orc.assign(cent, db, IP)).mean() > 0.1
    idx.close()


def test_train_on_device_recall():
    d, M, n, nq, nlist = 128, 64, 200_000, 500, 256
    db = synth.sift_like(n, d, seed=61)
    xq = synth.sift_like(nq, d, seed=62)
    flat = gi().GammaIndex("FLAT", d, {"metric_type": "L2"})
    flat.add_vectors(db)
    _, gt = flat.search(xq, 1)
    flat.close()
    idx = gi().GammaIndex("IVFPQFastScan", d, {"ncentroids": nlist, "nprobe": 32, "nsubvector": M, "metric_type": "L2"})
    assert idx.training_threshold == nlist * 39
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()

    def recall(ids, i):
        return float(np.mean([gt[q, 0] in ids[q, :i] for q in range(nq)]))

    _, ig = idx.search(xq, 10, params={"nprobe": 32, "recall_num": 100})
    r1, r10 = recall(ig, 1), recall(ig, 10)
    _, ig0 = idx.search(xq, 10, params={"nprobe": 32})
    print(f"IVFPQFastScan recall_num 100: r@1 {r1:.3f} r@10 {r10:.3f}; recall_num 0: r@1 {recall(ig0, 1):.3f} "
          f"r@10 {recall(ig0, 10):.3f}")
    assert r1 >= 0.6 and r10 >= 0.9
    idx.close()


def test_concurrent_searches_with_realtime_adds():
    d, M, nlist, n0 = 64, 16, 8, 12000
    db = np.unique(synth.sift_like(n0 + 4000, d, seed=71), axis=0)
    n0 = min(n0, len(db) - 4000)
    idx, _, _ = shared_state_index(db[:n0], d, M, nlist, L2)
    errs, stop = [], threading.Event()

    def searcher(seed):
        rng = np.random.default_rng(seed)
        try:
            while not stop.is_set():
                pick = rng.integers(0, n0, 400)
                dg, ig = idx.search(db[pick], 1, params={"nprobe": nlist, "recall_num": 100})
                assert (dg[:, 0] == 0).all() and (ig[:, 0] == pick).all()
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=searcher, args=(s,)) for s in (1, 2)]
    for t in ts:
        t.start()
    try:
        for b in range(n0, n0 + 4000, 250):
            idx.add_vectors(db[b:b + 250])
            idx.add_pending()
    finally:
        stop.set()
        for t in ts:
            t.join()
    assert not errs, errs[:1]
    pick = np.arange(n0 + 3000, n0 + 3400)
    dg, ig = idx.search(db[pick], 1, params={"nprobe": nlist, "recall_num": 100})
    assert (dg[:, 0] == 0).all() and (ig[:, 0] == pick).all()
    idx.close()


# ---- engine (include/gamma_api.h) ------------------------------------------------------------------------------
D = 32
FS_PARAMS = {"ncentroids": 16, "nprobe": 8, "nsubvector": 16, "metric_type": "L2", "training_threshold": 1000}


def make_engine(tmp_path, params, name="fs"):
    from vearch_b200 import engine
    e = engine.GammaEngine(str(tmp_path), space_name=name)
    e.create_table(name, D, "IVFPQFastScan", params, fields=(("_id", wire.DT_STRING, False),))
    return e


def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def test_engine_flow_params_and_dump_load(tmp_path):
    from vearch_b200 import engine
    db, xq = synth.sift_like(3000, D, seed=81), synth.sift_like(16, D, seed=82)
    for bad, msg in (({"opq": {"nsubvector": 8}}, "opq"), ({"bbs": 48}, "bbs")):
        e = engine.GammaEngine(str(tmp_path / "bad"))
        with pytest.raises(engine.GammaStatusError) as ei:
            e.create_table("t", D, "IVFPQFastScan", dict(FS_PARAMS, **bad))
        assert ei.value.code == 4 and msg in ei.value.msg
        e.close()
    e = make_engine(tmp_path, dict(FS_PARAMS, bbs=64, nbits_per_idx=8, hnsw={"nlinks": 32}))
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    e.wait_indexed(len(db))
    e.delete_doc("doc7")
    before = e.search(xq, 10, index_params={"nprobe": 8, "recall_num": 50})
    got = keys_of(before)
    assert all(len(r) == 10 for r in got) and not any("doc7" in r for r in got)
    for q in range(len(xq)):  # re-ranked scores are the exact distances of the returned docs
        for key, s in zip(got[q], scores_of(before)[q]):
            assert s == float(((xq[q] - db[int(key[3:])]) ** 2).sum())
    rc, doc = e.get_doc_by_id("doc5")
    assert rc == 0
    plain = e.search(xq, 10, index_params={"nprobe": 8})
    assert e.dump() == 0
    e.close()
    e2 = make_engine(tmp_path, FS_PARAMS)
    assert e2.load() == 0
    e2.build_index()
    e2.wait_indexed(len(db))
    after = e2.search(xq, 10, index_params={"nprobe": 8, "recall_num": 50})
    assert keys_of(after) == keys_of(before) and scores_of(after) == scores_of(before)
    again = e2.search(xq, 10, index_params={"nprobe": 8})
    assert keys_of(again) == keys_of(plain) and scores_of(again) == scores_of(plain)
    assert e2.get_doc_by_id("doc7")[0] == -1
    e2.close()


def test_nsubvector_above_256_is_refused():
    with pytest.raises(gi().GammaError, match="above 256"):
        gi().GammaIndex("IVFPQFastScan", 1024, {"ncentroids": 16, "nprobe": 4, "nsubvector": 512, "metric_type": "L2"})
    idx = gi().GammaIndex("IVFPQFastScan", 512, {"ncentroids": 16, "nprobe": 4, "nsubvector": 256, "metric_type": "L2"})
    db = synth.sift_like(3000, 512, seed=9)
    idx.add_vectors(db)
    idx.set_centroids(orc.kmeans(db, 16, niter=2)[0])
    idx.add_pending()
    dg, ig = idx.search(db[:4], 100, params={"recall_num": 4096})  # the largest table with the largest queue
    assert (ig[:, 0] == np.arange(4)).all() and (dg[:, 0] == 0).all()
    idx.close()
