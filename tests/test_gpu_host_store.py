"""Raw vectors in pinned host memory (store_type "RocksDB") against the HBM store on the H100.  Every index is built
twice from the same seeded rows, once per placement: the trained state, the lists and every search result (ids and
score bits, under deletion and filter bitmaps and a score window) must be identical.  N is large enough that the host
store spans several segments (RawStore::kHostSegShift: 65 536 rows) and re-rank candidates come from all of them."""
import numpy as np
import pytest

from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
N, D, NQ = 200_000, 64, 96
HOST_SEG_ROWS = 1 << 16


def gi():
    from vearch_b200 import index as gidx
    return gidx


def eng_mod():
    from vearch_b200 import engine
    return engine


@pytest.fixture(scope="module")
def data():
    return synth.sift_like(N, D, seed=91), synth.sift_like(2048, D, seed=92)


def build_pair(typ, params, db, train=True):
    out = []
    for st in (None, "RocksDB"):
        idx = gi().GammaIndex(typ, D, params, store_type=st)
        idx.add_vectors(db)
        if train:
            idx.train()
            idx.add_pending()
        out.append(idx)
    return out


def assert_same_state(hbm, host, same_layout=True):
    assert hbm.mem_bytes(2) == 0 and hbm.mem_bytes(1) >= N * D * 4
    assert host.mem_bytes(1) == 0 and host.mem_bytes(2) >= N * D * 4
    assert host.ntotal == hbm.ntotal == N
    if hbm.index_type == "FLAT":
        return
    if same_layout:  # built alike; IVF-Flat on a host store adds its row-pointer table, 8 B per vector
        extra = N * 8 if hbm.index_type == "IVFFLAT" else 0
        assert host.mem_bytes(0) == hbm.mem_bytes(0) + extra
    assert np.array_equal(hbm.get_centroids(), host.get_centroids())
    if hbm.index_type != "IVFFLAT":
        assert np.array_equal(hbm.get_pq_centroids(), host.get_pq_centroids())
    if hbm.index_type == "IVFPQ" and hbm.has_opq:
        assert np.array_equal(hbm.get_opq(), host.get_opq())
    for a, b in zip(hbm.export_lists(), host.export_lists()):
        assert np.array_equal(a, b)


def search_variants(xq, k, kth_score, metric_l2):
    rng = np.random.default_rng(5)
    delb = np.packbits(rng.random(N) < 0.2, bitorder="little")
    filb = np.packbits(rng.random(N) < 0.7, bitorder="little")
    window = {"max_score": kth_score} if metric_l2 else {"min_score": kth_score}
    return [{}, {"del_bitmap": delb}, {"filter_bitmap": filb}, {"del_bitmap": delb, "filter_bitmap": filb, **window}]


def assert_same_search(hbm, host, xq, k, params=None, brute_force=False, kernel=None, l2=True):
    d0, _ = hbm.search(xq, k, params=params, brute_force=brute_force)
    kth = float(np.median(d0[:, k // 2]))
    for kw in search_variants(xq, k, kth, l2):
        dh, ih = hbm.search(xq, k, params=params, brute_force=brute_force, **kw)
        if kernel:
            assert hbm.last_scan_kernel == kernel, (hbm.last_scan_kernel, kernel)
        dr, ir = host.search(xq, k, params=params, brute_force=brute_force, **kw)
        assert host.last_scan_kernel == hbm.last_scan_kernel
        assert np.array_equal(ih, ir), kw.keys()
        assert np.array_equal(dh.view(np.uint32), dr.view(np.uint32)), kw.keys()


def close(*idx):
    for i in idx:
        i.close()


def test_flat_and_brute_force(data):
    db, xq = data
    hbm, host = build_pair("FLAT", {"metric_type": "L2"}, db, train=False)
    assert_same_state(hbm, host)
    assert host.get_vectors(0, N).tobytes() == db.tobytes()
    assert_same_search(hbm, host, xq[:NQ], 10)
    assert_same_search(hbm, host, xq, 50)  # several query blocks per staged chunk
    close(hbm, host)
    hbm, host = build_pair("IVFPQ", {"ncentroids": 256, "nprobe": 16, "nsubvector": 16, "metric_type": "L2"}, db)
    assert_same_search(hbm, host, xq[:NQ], 10, brute_force=True)
    close(hbm, host)


@pytest.mark.parametrize("metric", ["L2", "InnerProduct"])
def test_ivfflat_query_and_list_major(data, metric):
    db, xq = data
    hbm, host = build_pair("IVFFLAT", {"ncentroids": 256, "nprobe": 16, "metric_type": metric}, db)
    assert_same_state(hbm, host)
    l2 = metric == "L2"
    assert_same_search(hbm, host, xq[:NQ], 10, kernel="ivfflat_scan_warp_kernel", l2=l2)
    # 2048 x 16 pairs over 256 lists: 128 per list, so the list-major scan and its winner re-score run
    assert_same_search(hbm, host, xq, 10, l2=l2)
    assert "listmajor" in host.last_scan_kernel
    # an update moves the row to another list; the row-pointer table follows it
    for idx in (hbm, host):
        idx.update_vector(7, xq[0] + 0.5)
        idx.update_vector(HOST_SEG_ROWS + 3, xq[1])
    assert np.array_equal(host.get_vector(7), hbm.get_vector(7))
    assert_same_search(hbm, host, xq, 10, l2=l2)
    hbm.compact(), host.compact()
    assert_same_search(hbm, host, xq, 10, l2=l2)
    close(hbm, host)


def test_ivfflat_dump_load_list_major(data, tmp_path):
    """gamma's index file loaded into a host store: the winner re-score's row pointers come from the loaded lists"""
    db, xq = data
    params = {"ncentroids": 256, "nprobe": 16, "metric_type": "L2"}
    hbm, host = build_pair("IVFFLAT", params, db)
    host.dump(str(tmp_path), "emb")
    host.close()
    host = gi().GammaIndex("IVFFLAT", D, params, store_type="RocksDB")
    host.add_vectors(db)
    host.load(str(tmp_path), "emb")
    assert host.indexed_count == N
    assert_same_state(hbm, host, same_layout=False)  # a loaded list is reserved at its length
    assert_same_search(hbm, host, xq, 10)
    assert "listmajor" in host.last_scan_kernel
    close(hbm, host)


@pytest.mark.parametrize("cfg", [
    {"nsubvector": 16},
    {"nsubvector": 16, "nbits_per_idx": 4},
    {"nsubvector": 16, "opq": {"nsubvector": 16}},
], ids=["nbits8", "nbits4", "opq"])
def test_ivfpq(data, cfg):
    db, xq = data
    params = {"ncentroids": 256, "nprobe": 16, "metric_type": "L2", **cfg}
    hbm, host = build_pair("IVFPQ", params, db)
    assert_same_state(hbm, host)
    for rn in (0, 400):
        p = {"nprobe": 16, "recall_num": rn} if rn else {"nprobe": 16}
        assert_same_search(hbm, host, xq[:NQ], 10, params=p)
        if cfg.get("nbits_per_idx", 8) == 8 and "opq" not in cfg:
            assert_same_search(hbm, host, xq, 10, params=p, kernel="pqtc_scan_kernel")
    close(hbm, host)


def test_ivfpq_fastscan(data):
    db, xq = data
    hbm, host = build_pair("IVFPQFastScan", {"ncentroids": 256, "nprobe": 16, "nsubvector": 16, "metric_type": "L2"}, db)
    assert_same_state(hbm, host)
    for rn in (0, 400):
        p = {"nprobe": 16, "recall_num": rn} if rn else {"nprobe": 16}
        assert_same_search(hbm, host, xq[:NQ], 10, params=p)
    close(hbm, host)


def test_placement_parsing():
    for st, on_host in (("RocksDB", True), ("rocksdb", True), ("MemoryOnly", False), ("", False), (None, False)):
        idx = gi().GammaIndex("FLAT", 8, {"metric_type": "L2"}, store_type=st)
        idx.add_vectors(np.ones((3, 8), np.float32))
        assert (idx.mem_bytes(2) > 0) == on_host and (idx.mem_bytes(1) > 0) == (not on_host)
        idx.close()


# ---- engine ------------------------------------------------------------------------------------------------------
def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def engine_flow(path, store_type, index_type, index_params, db, xq, img):
    """CreateTable, add, delete, Update, GetDocByID, Search, the realtime tail, Dump -> Load -> Search; returns every
    observation"""
    n = 3000  # reaching training_threshold starts the one indexing pass this test sees
    params = {"ncentroids": 32, "nprobe": 8, "metric_type": "L2", "training_threshold": n}
    extra = [("img", 16, "FLAT", {"metric_type": "L2"}, "MemoryOnly" if store_type == "RocksDB" else "RocksDB")]
    e = eng_mod().GammaEngine(str(path), space_name="hs")
    e.create_table("hs", D, index_type, {**params, **index_params}, extra_vectors=extra, store_type=store_type,
                   refresh_interval=600000, enable_realtime=True)
    obs = []
    for i in range(n):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("img", img[i].tobytes(), wire.DT_VECTOR)]) == 0
    e.wait_indexed(n)
    for i in range(n, n + 300):  # stays un-indexed: the indexing loop sleeps between passes
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("img", img[i].tobytes(), wire.DT_VECTOR)]) == 0
    assert e.delete_doc("doc11") == 0
    assert e.add_doc("doc7", xq[3] + 1.0, extra_fields=[("img", img[0].tobytes(), wire.DT_VECTOR)]) == 0
    rc, doc = e.get_doc_by_id("doc7")
    obs.append((rc, doc["emb"][0], doc["img"][0]))
    rc, doc = e.get_doc_by_id("doc3100")
    obs.append((rc, doc["emb"][0], doc["img"][0]))
    assert obs[-1][1] == db[3100].tobytes()
    for kw in ({"index_params": {"nprobe": 8}}, {"index_params": {"nprobe": 8, "recall_num": 100}},
               {"is_brute_search": 1}, {"index_params": {"nprobe": 8}, "extra_vec_queries": [("img", img[:64])]}):
        res = e.search(xq[:64], 10, **kw)
        obs.append((keys_of(res), scores_of(res)))
    # 2048 queries x 8 probes over 32 lists: the list-major scans (IVF-Flat: and its winner re-score)
    big = e.search(xq, 10, index_params={"nprobe": 8})
    obs.append((keys_of(big), scores_of(big)))
    mem = e.memory_info()
    obs.append(mem["vector_mem"] > 0)
    assert e.dump() == 0
    e.close()
    e2 = eng_mod().GammaEngine(str(path), space_name="hs")
    e2.create_table("hs", D, index_type, {**params, **index_params}, extra_vectors=extra, store_type=store_type,
                    refresh_interval=600000, enable_realtime=True)
    assert e2.load() == 0
    e2.wait_indexed(n)
    res = e2.search(xq[:64], 10, index_params={"nprobe": 8, "recall_num": 100})
    obs.append((keys_of(res), scores_of(res)))
    res = e2.search(xq, 10, index_params={"nprobe": 8})
    obs.append((keys_of(res), scores_of(res)))
    rc, doc = e2.get_doc_by_id("doc7")
    obs.append((rc, doc["emb"][0]))
    e2.close()
    return obs


@pytest.mark.parametrize("index_type,index_params", [("IVFPQ", {"nsubvector": 16}), ("IVFFLAT", {})])
def test_engine_flow_matches_memory_only(tmp_path, data, index_type, index_params):
    db, xq = data
    img = synth.sift_like(3300, 16, seed=93)
    mem = engine_flow(tmp_path / "mem", "MemoryOnly", index_type, index_params, db, xq, img)
    host = engine_flow(tmp_path / "host", "RocksDB", index_type, index_params, db, xq, img)
    assert len(mem) == len(host)
    for i, (a, b) in enumerate(zip(mem, host)):
        assert a == b, i
