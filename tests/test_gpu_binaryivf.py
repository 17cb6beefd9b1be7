"""BINARYIVF on the H100 through the C-ABI: with given packed centroids the coarse search, list contents and searched
keys are exact against tests/topk_reference.py (Hamming distances are integers, so keys compare exactly, ties
included) and tie-aware equal to the heap of oracle_binary; training on the device packs the device k-means centroids
by sign and reaches the oracle-derived recall; updates, deleted rows, brute force, the realtime tail and host placement
follow the engine's IVF rules."""
import numpy as np
import pytest

import topk_reference as tr
from oracle_binary import binary_ivf as ob
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2 = tr.METRIC_L2


def gi():
    from vearch_b200 import index as gidx
    return gidx


def lists_of(idx):
    codes, lid, raw = [], [], []
    lists = {}
    for l in range(idx.nlist):
        n = idx.list_len(l)
        c, i = idx.get_list(l)
        c = np.asarray(c, np.uint8).reshape(n, idx.code_bytes)
        lists[l] = (c, np.asarray(i, np.int64))
        codes.append(c)
        lid.append(np.full(n, l, np.int64))
        raw.append(np.asarray(i, np.int64))
    return lists, np.concatenate(codes), np.concatenate(lid), np.concatenate(raw)


def built(db, cs, nlist, store_type=None, centroids=None):
    idx = gi().BinaryIVFIndex(cs * 8, {"ncentroids": nlist}, store_type=store_type)
    cent = centroids if centroids is not None else db[np.random.default_rng(cs).choice(len(db), nlist, replace=False)]
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending()
    return idx, cent


def expect(idx, xq, probes, k, **kw):
    _, codes, lid, raw = lists_of(idx)
    return tr.search_entries(ob.hamming(xq, codes), lid, raw, probes, k, L2, **kw)


def got_keys(dis, ids):
    return tr.keys(dis, np.where(ids >= 0, ids, 0), ids >= 0, L2)


def assert_ids_equal_up_to_ties(dis, ids, oids):
    """same ids, except that among the entries at a row's k-th (last) distance any equally distant ones may stand"""
    for q in range(len(dis)):
        last = dis[q][ids[q] >= 0].max(initial=-1)
        inner = dis[q] < last
        assert set(ids[q][inner].tolist()) == set(oids[q][inner].tolist())
        assert np.sum(ids[q] >= 0) == np.sum(oids[q] >= 0)


CODE_SIZES = [1, 3, 4, 8, 12, 16, 20, 24, 32, 64, 128]


@pytest.mark.parametrize("cs", CODE_SIZES)
def test_coarse_and_scan_key_exact(cs):
    db = synth.binary_clustered(6000, cs * 8, seed=cs, n_clusters=32, flip=0.2)
    xq = synth.binary_clustered(40, cs * 8, seed=100 + cs, n_clusters=32, flip=0.2)
    idx, cent = built(db, cs, 48)
    cd, cl = idx.coarse_search(xq, 36)
    wd, wl = ob.coarse_search(xq, cent, 36)
    assert np.array_equal(cl, wl) and np.array_equal(cd, wd.astype(np.float32))
    for l in range(idx.nlist):  # list entries are the raw bytes, in vid order
        c, i = lists_of(idx)[0][l]
        assert np.array_equal(c, db[i]) and np.all(np.diff(i) > 0)
    assert np.all(ob.assign(db, cent)[lists_of(idx)[3]] == lists_of(idx)[2])
    k = 17
    dis, ids = idx.search(xq, k, params={"nprobe": 36})
    assert np.array_equal(got_keys(dis, ids), expect(idx, xq, cl, k))
    # the oracle's heap: same distances, ids equal up to ties
    lists, _, _, _ = lists_of(idx)
    od, oi = ob.search_knn_hamming_heap(xq, lists, cl, k)
    assert np.array_equal(dis, od)
    assert_ids_equal_up_to_ties(dis, ids, oi)


@pytest.mark.parametrize("k", [1, 16, 17, 400, 1024, 4096])
def test_large_k_across_cta_groups(k):
    cs = 32
    db = synth.binary_clustered(30000, cs * 8, seed=k, n_clusters=16, flip=0.3)
    xq = synth.binary_clustered(12, cs * 8, seed=k + 1, n_clusters=16, flip=0.3)
    idx, cent = built(db, cs, 64)
    _, probes = ob.coarse_search(xq, cent, 48)
    dis, ids = idx.search_preassigned(xq, k, probes)
    assert np.array_equal(got_keys(dis, ids), expect(idx, xq, probes, k))


@pytest.mark.parametrize("cs", [3, 16, 128])
def test_bitmaps_tombstones_and_windows_inside_tie_groups(cs):
    db = synth.binary_clustered(5000, cs * 8, seed=7, n_clusters=8, flip=0.25)
    xq = synth.binary_clustered(16, cs * 8, seed=8, n_clusters=8, flip=0.25)
    idx, cent = built(db, cs, 40)
    rng = np.random.default_rng(cs)
    for l in range(0, 40, 3):
        if idx.list_len(l) > 2:
            idx.tombstone(l, 1)
    dele = np.packbits(rng.random(len(db)) < 0.2, bitorder="little")
    filt = np.packbits(rng.random(len(db)) < 0.7, bitorder="little")
    _, probes = ob.coarse_search(xq, cent, 40)
    d_all = ob.hamming(xq, db)
    lo, hi = float(np.percentile(d_all, 2)), float(np.percentile(d_all, 30))  # integers: edges fall inside tie groups
    for k in (10, 300):
        dis, ids = idx.search_preassigned(xq, k, probes, del_bitmap=dele, filter_bitmap=filt, min_score=lo, max_score=hi)
        want = expect(idx, xq, probes, k, del_bitmap=dele, filter_bitmap=filt, min_score=lo, max_score=hi)
        assert np.array_equal(got_keys(dis, ids), want)


def test_training_packs_device_centroids_and_reaches_recall():
    cs, nlist = 32, 64
    db = synth.binary_clustered(40000, cs * 8, seed=1, n_clusters=64, flip=0.12)
    xq = synth.binary_clustered(200, cs * 8, seed=2, n_clusters=64, flip=0.12)
    idx = gi().BinaryIVFIndex(cs * 8, {"ncentroids": nlist})
    assert idx.training_threshold == nlist * 39
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    real = idx.get_real_centroids()
    packed = idx.get_centroids()
    assert np.array_equal(packed, ob.real_to_binary(real))
    k = 10
    dis, ids = idx.search(xq, k)  # default nprobe 20
    ex = tr.topk(tr.keys(ob.hamming(xq, db), np.arange(len(db))[None, :]), k)
    kth = (ex[:, -1] >> np.uint64(32)).astype(np.uint32)
    got = tr.score2ord(dis, L2)
    recall = np.mean(got <= kth[:, None])  # tie-aware: any result within the exact k-th distance counts
    # the oracle's heap over the same centroids and lists gives the same distances
    _, probes = ob.coarse_search(xq, packed, 20)
    od, _ = ob.search_knn_hamming_heap(xq, lists_of(idx)[0], probes, k)
    assert np.array_equal(dis, od)
    # Pinned from the oracle alone on this data (numpy, no device): with the first 64 rows as untrained centroids and
    # nprobe 20 its tie-aware recall@10 is 0.991; trained centroids must come within 0.02 of it.
    assert recall >= 0.97


def test_update_deleted_rows_brute_force_tail_and_host_store():
    cs, nlist = 16, 32
    db = synth.binary_clustered(8000, cs * 8, seed=5, n_clusters=16, flip=0.2)
    xq = synth.binary_clustered(20, cs * 8, seed=6, n_clusters=16, flip=0.2)
    cent = db[:nlist].copy()
    # a row deleted before indexing is skipped, the rows after it in the batch are indexed under their own vids
    dele = np.zeros((len(db) + 7) // 8, np.uint8)
    dele[100 >> 3] |= 1 << (100 & 7)
    idx = gi().BinaryIVFIndex(cs * 8, {"ncentroids": nlist})
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending(dele)
    _, _, _, raw = lists_of(idx)
    assert sorted(raw.tolist()) == [v for v in range(len(db)) if v != 100]
    # update re-assigns: the old entry is tombstoned, the new bits are appended to their nearest list
    new = cent[3:4].copy()
    idx.update_vector(7, new)
    assert np.array_equal(idx.get_vector(7), new[0])
    _, codes, lid, raw = lists_of(idx)
    live = raw >= 0
    assert np.sum(raw[live] == 7) == 1 and lid[live][raw[live] == 7][0] == ob.assign(new, cent)[0]
    assert np.array_equal(idx.get_vectors(0, 50)[8:], db[8:50])
    # brute force = exact Hamming over the stored rows
    stored = idx.get_vectors(0, len(db))
    for k in (5, 100):
        dis, ids = idx.search(xq, k, brute_force=True)
        assert np.array_equal(got_keys(dis, ids), tr.topk(tr.keys(ob.hamming(xq, stored), np.arange(len(db))[None, :]), k))
    # realtime tail: rows stored but not indexed are searched exactly and merged
    tail = synth.binary_clustered(300, cs * 8, seed=9, n_clusters=16, flip=0.2)
    idx.add_vectors(tail)
    dis_t, ids_t = idx.search(xq, 30, params={"nprobe": nlist}, search_unindexed_tail=True)
    _, probes = ob.coarse_search(xq, cent, nlist)
    ivf = expect(idx, xq, probes, 30)
    tk = tr.topk(tr.keys(ob.hamming(xq, tail), np.arange(len(db), len(db) + 300)[None, :]), 30)
    assert np.array_equal(got_keys(dis_t, ids_t), tr.topk(np.concatenate([ivf, tk], 1), 30))
    # host placement (store_type RocksDB) gives the same results
    hidx = gi().BinaryIVFIndex(cs * 8, {"ncentroids": nlist}, store_type="RocksDB")
    hidx.set_centroids(cent)
    hidx.add_vectors(db)
    hidx.add_pending(dele)
    hidx.update_vector(7, new)
    hidx.add_vectors(tail)
    assert hidx.mem_bytes(2) > 0 and hidx.mem_bytes(1) == 0
    for kw in ({"brute_force": True}, {"params": {"nprobe": nlist}, "search_unindexed_tail": True}, {}):
        a = idx.search(xq, 30, **kw)
        b = hidx.search(xq, 30, **kw)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_parameters_and_refusals():
    g = gi()
    with pytest.raises(g.GammaError, match="multiple of 8"):
        g.BinaryIVFIndex(100)
    with pytest.raises(g.GammaError, match="invalid ncentroids"):
        g.BinaryIVFIndex(64, {"ncentroids": -5})
    idx = g.BinaryIVFIndex(64, {"ncentroids": -1, "metric_type": "InnerProduct", "nsubvector": 4})
    assert idx.nlist == 256 and idx.training_threshold == 256 * 39
    idx.add_vectors(np.zeros((3, 8), np.uint8))
    # float queries are refused, packed ones are served (untrained: brute force)
    with pytest.raises(g.GammaError, match="packed binary"):
        g.GammaIndex.search(idx, np.zeros((1, 64), np.float32), 1)
    d, i = idx.search(np.zeros((1, 8), np.uint8), 2)
    assert d.tolist() == [[0.0, 0.0]] and i.tolist() == [[0, 1]]
    # retrieval nprobe above nlist falls back to the default
    idx2, cent = built(synth.binary_clustered(2000, 64, seed=1, n_clusters=8), 8, 16)
    a = idx2.search(np.zeros((2, 8), np.uint8), 5, params={"nprobe": 99})
    b = idx2.search(np.zeros((2, 8), np.uint8), 5, params={"nprobe": 16})
    assert np.array_equal(a[0], b[0])


def searched_index(n=20000, cs=16, nlist=64, seed=41):
    db = synth.binary_clustered(n, cs * 8, seed=seed, n_clusters=32, flip=0.2)
    idx, _ = built(db, cs, nlist)
    return idx


def test_retrieval_metric_type_is_ignored():
    # Hamming distances rank smaller first whatever metric_type the retrieval parameters carry
    idx = searched_index()
    xq = synth.binary_clustered(40, 128, seed=42, n_clusters=32, flip=0.2)
    for kw in ({"params": {"nprobe": 8}}, {"brute_force": True}):
        want = idx.search(xq, 20, **kw)
        params = dict(kw.get("params", {}), metric_type="InnerProduct")
        got = idx.search(xq, 20, **dict(kw, params=params))
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.all(np.diff(got[0], axis=1) >= 0)


def test_concurrent_small_searches_equal_one_batch():
    # small searches without bitmaps from several threads are merged into shared device batches (request coalescing);
    # each caller gets exactly its slice of the one-batch result
    import threading
    idx = searched_index()
    xq = synth.binary_clustered(32, 128, seed=43, n_clusters=32, flip=0.2)
    for kw in ({"params": {"nprobe": 8}}, {"brute_force": True}):
        want = idx.search(xq, 10, **kw)
        got = [None] * 8
        start = threading.Barrier(8)

        def run(t):
            start.wait()
            for _ in range(5):
                got[t] = idx.search(xq[4 * t:4 * t + 4], 10, **kw)

        threads = [threading.Thread(target=run, args=(t,)) for t in range(8)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert np.array_equal(np.concatenate([g[0] for g in got]), want[0])
        assert np.array_equal(np.concatenate([g[1] for g in got]), want[1])


def test_large_batch_equals_its_slices():
    # an IVF search runs its queries in batches of 16384; every query's result is its own
    idx = searched_index()
    xq = synth.binary_clustered(20000, 128, seed=44, n_clusters=32, flip=0.2)
    dis, ids = idx.search(xq, 10, params={"nprobe": 8})
    for q0, q1 in ((0, 16384), (16384, 20000)):
        d, i = idx.search(xq[q0:q1], 10, params={"nprobe": 8})
        assert np.array_equal(dis[q0:q1], d) and np.array_equal(ids[q0:q1], i)


def test_scan_kernel_names():
    idx = searched_index()
    xq = synth.binary_clustered(20, 128, seed=45, n_clusters=32, flip=0.2)
    idx.search(xq, 10, brute_force=True)
    assert idx.last_scan_kernel == "hamming_tile_kernel+select_rows_kernel"
    idx.search(xq, 10, params={"nprobe": 8})
    assert idx.last_scan_kernel == "binary_ivf_scan_kernel"


# ---- the engine (gamma C-ABI): a BINARYIVF table end to end -----------------------------------------------------------
def eng_mod():
    from vearch_b200 import engine
    return engine


def ids_of(res):
    return [[int(it["fields"]["_id"].decode()[3:]) for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def binary_engine(path, d_bits, params, store_type="MemoryOnly", **kw):
    from vearch_b200 import wire
    e = eng_mod().GammaEngine(str(path), space_name="bin")
    e.create_table("bin", d_bits, "BINARYIVF", params, fields=(("_id", wire.DT_STRING, False),), store_type=store_type, **kw)
    return e


def test_engine_create_table_refusals(tmp_path):
    E = eng_mod()
    from vearch_b200 import wire
    with pytest.raises(E.GammaStatusError, match="multiple of 8"):
        binary_engine(tmp_path / "a", 100, {"ncentroids": 8})
    e = E.GammaEngine(str(tmp_path / "b"), space_name="mv")
    with pytest.raises(E.GammaStatusError, match="emb2: BINARYIVF is not supported in a multi-vector table"):
        e.create_table("mv", 64, "FLAT", {}, fields=(("_id", wire.DT_STRING, False),),
                       extra_vectors=[("emb2", 64, "BINARYIVF", {"ncentroids": 8})])
    e3 = E.GammaEngine(str(tmp_path / "c"), space_name="mv")
    with pytest.raises(E.GammaStatusError, match="emb: BINARYIVF is not supported in a multi-vector table"):
        e3.create_table("mv", 64, "BINARYIVF", {"ncentroids": 8}, fields=(("_id", wire.DT_STRING, False),),
                        extra_vectors=[("emb2", 64, "FLAT", {})])


def test_engine_flow_dump_load_and_placements(tmp_path):
    cs, nlist, n = 32, 32, 4000
    db = synth.binary_clustered(n, cs * 8, seed=21, n_clusters=16, flip=0.2)
    xq = synth.binary_clustered(6, cs * 8, seed=22, n_clusters=16, flip=0.2)
    params = {"ncentroids": nlist, "training_threshold": 2000}
    results = {}
    for store in ("MemoryOnly", "RocksDB"):
        e = binary_engine(tmp_path / store, cs * 8, params, store_type=store)
        assert e.add_doc("doc-bad", np.zeros(cs - 1, np.uint8)) == -3  # CheckDoc: d / 8 bytes exactly
        assert e.add_doc("doc-bad", np.zeros(cs, np.float32)) == -3
        for i, v in enumerate(db):
            assert e.add_doc(f"doc{i}", v) == 0
        e.wait_indexed(n)
        res = e.search(xq, 10, index_params={"nprobe": nlist})  # several queries in one request
        exact = tr.topk(tr.keys(ob.hamming(xq, db), np.arange(n)[None, :]), 10)
        want_d, want_i = tr.decode(exact, L2)
        assert np.array_equal(np.array(scores_of(res), np.float32), want_d)  # nprobe = nlist: exact
        assert_ids_equal_up_to_ties(want_d, np.array(ids_of(res)), want_i)
        # delete, then update (re-assigned; a row outside the training sample, so Load retrains on the same rows), then
        # the exact bytes back
        assert e.delete_doc("doc3") == 0
        new = db[5].copy()
        assert e.add_doc("doc3500", new) == 0
        rc, doc = e.get_doc_by_id("doc3500")
        assert rc == 0 and doc["emb"][0] == new.tobytes()
        assert e.get_doc_by_id("doc3")[0] == -1
        res = e.search(new[None, :], 3, index_params={"nprobe": nlist})
        assert sorted(ids_of(res)[0][:2]) == [5, 3500] and scores_of(res)[0][:2] == [0.0, 0.0]
        brute = e.search(xq, 10, is_brute_search=1)
        before = e.search(xq, 10)
        results[store] = (scores_of(before), ids_of(before), scores_of(brute), ids_of(brute))
        assert e.dump() == 0
        e.close()
        e2 = binary_engine(tmp_path / store, cs * 8, params, store_type=store)
        assert e2.load() == 0
        e2.wait_indexed(n)  # nothing is dumped for the index: Load trains and fills it again
        after = e2.search(xq, 10)
        assert scores_of(after) == scores_of(before) and ids_of(after) == ids_of(before)
        assert e2.get_doc_by_id("doc3500")[1]["emb"][0] == new.tobytes() and e2.get_doc_by_id("doc3")[0] == -1
        e2.close()
    assert results["MemoryOnly"] == results["RocksDB"]


def test_engine_realtime_tail(tmp_path):
    cs, nlist = 16, 16
    db = synth.binary_clustered(3000, cs * 8, seed=31, n_clusters=8, flip=0.2)
    xq = synth.binary_clustered(4, cs * 8, seed=32, n_clusters=8, flip=0.2)
    e = binary_engine(tmp_path, cs * 8, {"ncentroids": nlist, "training_threshold": 1000}, refresh_interval=600000,
                      enable_realtime=True)
    for i, v in enumerate(db[:2000]):
        assert e.add_doc(f"doc{i}", v) == 0
    e.wait_indexed(1000)
    for i, v in enumerate(db[2000:], start=2000):  # not picked up before the next indexing pass
        assert e.add_doc(f"doc{i}", v) == 0
    res = e.search(xq, 20, index_params={"nprobe": nlist})
    exact = tr.topk(tr.keys(ob.hamming(xq, db), np.arange(3000)[None, :]), 20)
    assert np.array_equal(np.array(scores_of(res), np.float32), tr.decode(exact, L2)[0])
    e.close()
