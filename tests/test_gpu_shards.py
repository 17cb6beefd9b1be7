"""GPU_IVFPQ and GPU_IVFFLAT sharded over several devices (gamma's IndexShards): vid v in shard v % S.  Every case is
compared with the unsharded index of the same type built from the same rows.  GPU_IVFPQ's ADC scores are bit-identical
on every scan path, and GPU_IVFFLAT's query-major kernel sums a row's score the same way whatever the list lengths, so
those (score, id) arrays must be equal element for element.  GPU_IVFFLAT's list-major scan selects each shard's
candidates on 3xTF32 scores before the exact re-score, so the shards' union of candidates is not the unsharded index's:
both placements are held to the fp64 reference under tests/float_contract.py's list-major margins instead
(DESIGN.md section 8).  Repeated ordinals put S shards on device 0, which runs every sharding path on a one-GPU
machine; distinct devices are tested when more than one is visible."""
import filecmp
import os

import numpy as np
import pytest

import float_contract as FC
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = 1, 0
D = 32


def gi():
    from vearch_b200 import index as gidx
    return gidx


def eng_mod():
    from vearch_b200 import engine
    return engine


def ndev():
    import torch
    return torch.cuda.device_count()


def params(typ, nlist, metric):
    p = {"ncentroids": nlist, "nprobe": min(nlist, 16), "metric_type": "L2" if metric == L2 else "InnerProduct",
         "training_threshold": nlist * 39}
    if typ == "GPU_IVFPQ":
        p["nsubvector"] = 8
    return p


def build(typ, nlist, metric, db, devices=None, store_type=None):
    idx = gi().GammaIndex(typ, D, params(typ, nlist, metric), devices=devices, store_type=store_type)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    return idx


def assert_same(got, want, what):
    """(score, id) arrays equal element for element, score bits included"""
    (gd, gi_), (wd, wi) = got, want
    assert np.array_equal(gi_, wi), f"{what}: ids differ"
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), f"{what}: scores differ"


def query_major(idx):
    return idx.last_scan_kernel.startswith("ivfflat_scan")


def list_major_contract(ref, xq, metric, nprobe):
    """per_query(q) -> (cand, f, m, md) of the IVF-Flat list-major scan over query q's probed lists (the coarse
    quantiser of the unsharded index, which every shard shares), as test_gpu_float_accuracy.IvfFlat builds them"""
    off, _, ids = ref.export_lists()
    db = ref.get_vectors(0, ref.ntotal)
    _, probes = ref.coarse_search(xq, nprobe)
    shifts = ref.get_list_shifts() if metric == L2 else None
    cache = {}

    def per_query(q):
        if q in cache:
            return cache[q]
        parts = []
        for l in probes[q]:
            raw = ids[off[l]:off[l + 1]]
            parts.append((l, raw[raw >= 0]))
        cand = np.concatenate([v for _, v in parts])
        f, ad = FC.scores64(xq[q:q + 1], db[cand], metric)
        f, ad = f[0], ad[0]
        md = FC.direct_margin(f, ad, D, metric)
        if metric == IP:
            cache[q] = (cand, f, FC.tc_dot_margin(ad, D) + md, md)
        else:
            m = np.empty_like(f)
            o = 0
            for l, vid in parts:
                na, nb, sad = FC.shifted_operands(xq[q:q + 1], db[vid], shifts[l])
                m[o:o + len(vid)] = FC.shifted_l2_margin(sad[0], na[0], nb[0], f[o:o + len(vid)], D)
                o += len(vid)
            cache[q] = (cand, f, m + md, md)
        return cache[q]
    return per_query


@pytest.fixture(scope="module")
def data():
    return synth.sift_like(30000, D, seed=11), synth.sift_like(512, D, seed=12)


SHARDS = [[0, 0], [0, 0, 0], [0, 0, 0, 0]]


def distinct_devices():
    n = ndev()
    if n < 2:
        pytest.skip(f"only {n} CUDA device visible: distinct-device sharding needs two or more")
    return list(range(min(n, 4)))


# ---- 1 + 2: same results, same trained state ----------------------------------------------------------------------
@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nlist", [16, 256])
@pytest.mark.parametrize("devices", SHARDS + ["distinct"], ids=["S2", "S3", "S4", "distinct"])
def test_same_results_and_trained_state(data, typ, metric, nlist, devices):
    if devices == "distinct":
        devices = distinct_devices()
    db, xq = data
    ref = build(typ, nlist, metric, db)
    sh = build(typ, nlist, metric, db, devices)
    assert sh.shard_count == len(devices) and ref.shard_count == 1
    assert sh.indexed_count == ref.indexed_count == len(db)
    for s in range(sh.shard_count):
        v = sh.shard(s)
        assert np.array_equal(v.get_centroids().view(np.uint32), ref.get_centroids().view(np.uint32))
        if typ == "GPU_IVFPQ":
            assert np.array_equal(v.get_pq_centroids().view(np.uint32), ref.get_pq_centroids().view(np.uint32))
        if typ == "GPU_IVFPQ" and metric == L2:  # the precomputed table exists under L2 only
            assert np.array_equal(v.get_precomputed_table().view(np.uint32), ref.get_precomputed_table().view(np.uint32))
        lens = [v.list_len(l) for l in range(nlist)]
        assert sum(lens) == len(range(s, len(db), len(devices)))
        v.close()
    contract = list_major_contract(ref, xq, metric, min(nlist, 16)) if typ == "GPU_IVFFLAT" else None
    for k in (1, 10, 2048):
        for nq in (7, 512):
            what = f"{typ} S={len(devices)} k={k} nq={nq}"
            got, want = sh.search(xq[:nq], k), ref.search(xq[:nq], k)
            if typ == "GPU_IVFPQ" or nq == 7:
                if typ == "GPU_IVFFLAT":
                    assert query_major(sh) and query_major(ref), (sh.last_scan_kernel, ref.last_scan_kernel)
                assert_same(got, want, what)
            else:  # list-major: both placements within the float contract of the fp64 reference
                assert sh.last_scan_kernel.startswith("ivf_listmajor"), sh.last_scan_kernel
                FC.check_all(got, contract, k, metric, f"sharded {what}")
                FC.check_all(want, contract, k, metric, f"unsharded {what}")
    # brute force stays on the primary device and is exact
    assert_same(sh.search(xq[:5], 10, brute_force=True), ref.search(xq[:5], 10, brute_force=True), "brute")
    ref.close()
    sh.close()


# ---- 3: filters and mutations ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
@pytest.mark.parametrize("devices", SHARDS, ids=["S2", "S3", "S4"])
def test_filters_and_mutations(data, typ, devices):
    db, xq = data
    db, xq = db[:12000], xq[:64]
    n = len(db)
    ref = build(typ, 64, L2, db)
    sh = build(typ, 64, L2, db, devices)
    rng = np.random.default_rng(5)
    dele = np.zeros((n + 7) // 8 + 16, np.uint8)
    flt = np.zeros_like(dele)
    for v in rng.choice(n, 3000, replace=False):
        dele[v >> 3] |= 1 << (v & 7)
    for v in rng.choice(n, 6000, replace=False):
        flt[v >> 3] |= 1 << (v & 7)
    cases = [dict(del_bitmap=dele), dict(filter_bitmap=flt), dict(del_bitmap=dele, filter_bitmap=flt)]
    base = ref.search(xq, 10)[0]
    cases.append(dict(min_score=float(np.median(base[:, 0])), max_score=float(np.median(base[:, 9]))))
    for kw in cases:
        assert_same(sh.search(xq, 50, **kw), ref.search(xq, 50, **kw), f"filters {sorted(kw)}")
        assert typ == "GPU_IVFPQ" or query_major(sh), sh.last_scan_kernel
    # Update moves rows across lists: tombstone + re-append in the owning shard
    moved = rng.choice(n, 200, replace=False)
    for v in moved:
        row = db[rng.integers(n)] + 0.5
        ref.update_vector(int(v), row)
        sh.update_vector(int(v), row)
    assert_same(sh.search(xq, 20), ref.search(xq, 20), "after update")
    gone = rng.choice(n, 2500, replace=False)
    bm = np.zeros((n + 7) // 8, np.uint8)
    for v in gone:
        bm[v >> 3] |= 1 << (v & 7)
    ref.delete_vectors(gone)
    sh.delete_vectors(gone)
    # a shard's list segment reaches the 0.3 dead share on its own count, so the lists each placement purges differ;
    # the results do not, and purging every remaining dead entry drops the same total
    d_ref, d_sh = ref.purge(0.3, bm), sh.purge(0.3, bm)
    assert d_sh > 0 and d_ref > 0
    assert_same(sh.search(xq, 20, del_bitmap=bm), ref.search(xq, 20, del_bitmap=bm), "after purge(0.3)")
    assert d_sh + sh.purge(0.0, bm) == d_ref + ref.purge(0.0, bm)
    assert_same(sh.search(xq, 20, del_bitmap=bm), ref.search(xq, 20, del_bitmap=bm), "after purge(0)")
    # appends after a purge
    extra = synth.sift_like(3000, D, seed=21)
    for ix in (ref, sh):
        ix.add_vectors(extra)
        ix.add_pending()
    assert_same(sh.search(xq, 20, del_bitmap=bm), ref.search(xq, 20, del_bitmap=bm), "append after purge")
    ref.close()
    sh.close()


# ---- 4: Dump and Load -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ,fname", [("GPU_IVFPQ", "ivfpq.index"), ("GPU_IVFFLAT", "ivfflat.index")])
@pytest.mark.parametrize("devices", SHARDS, ids=["S2", "S3", "S4"])
def test_dump_load(tmp_path, data, typ, fname, devices):
    db, xq = data
    db, xq = db[:9000], xq[:32]
    ref = build(typ, 32, L2, db)
    sh = build(typ, 32, L2, db, devices)
    ref.dump(str(tmp_path / "a"), "f")
    sh.dump(str(tmp_path / "b"), "f")
    fa, fb = str(tmp_path / "a" / "f" / fname), str(tmp_path / "b" / "f" / fname)
    assert os.path.getsize(fa) > 0 and filecmp.cmp(fa, fb, shallow=False), "sharded file differs after adds only"
    want = ref.search(xq, 10)
    # a sharded Load of the unsharded file, and an unsharded Load of the sharded file
    for src, devs in (("a", devices), ("b", None)):
        ix = gi().GammaIndex(typ, D, params(typ, 32, L2), devices=devs)
        ix.add_vectors(db)
        assert ix.load(str(tmp_path / src), "f") == len(db)
        assert ix.is_trained and ix.indexed_count == len(db)
        assert_same(ix.search(xq, 10), want, f"load {src} into {'sharded' if devs else 'unsharded'}")
        ix.close()
    # after an update the lists are the shards' segments merged by vid; the file still loads into either placement
    sh.update_vector(5, db[7] + 1.0)
    ref.update_vector(5, db[7] + 1.0)
    sh.dump(str(tmp_path / "c"), "f")
    ix = gi().GammaIndex(typ, D, params(typ, 32, L2))
    ix.add_vectors(db)
    ix.update_vector(5, db[7] + 1.0)
    ix.load(str(tmp_path / "c"), "f")
    assert_same(ix.search(xq, 10), ref.search(xq, 10), "load of a dump after update")
    for x in (ix, ref, sh):
        x.close()


# ---- 5: engine flow -------------------------------------------------------------------------------------------------
def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def run_engine(path, typ, devices, db, xq, dump=False):
    E = eng_mod()
    e = E.GammaEngine(str(path), space_name="ts", devices=devices)
    e.create_table("ts", D, typ, params(typ, 32, L2))
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    e.build_index()
    e.wait_indexed(len(db))
    res = e.search(xq, 10, index_params={"nprobe": 16})
    single = [e.search(xq[q:q + 1], 10, index_params={"nprobe": 16})[0] for q in range(4)]
    rc, doc = e.get_doc_by_id("doc17")
    assert rc == 0 and np.array_equal(np.frombuffer(doc["emb"][0], np.float32), db[17])
    mi = e.memory_info()
    assert mi["index_mem"] > 0 and mi["vector_mem"] > 0
    if dump:
        assert e.dump() == 0
    return e, res, single


@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
def test_engine_flow(tmp_path, data, typ):
    db, xq = data
    db, xq = db[:4000], xq[:16]
    e0, r0, s0 = run_engine(tmp_path / "plain", typ, None, db, xq)
    e1, r1, s1 = run_engine(tmp_path / "one", typ, [0], db, xq)
    e2, r2, s2 = run_engine(tmp_path / "two", typ, [0, 0], db, xq, dump=True)
    assert keys_of(r1) == keys_of(r0) and scores_of(r1) == scores_of(r0), "a one-entry list is today's placement"
    assert keys_of(r2) == keys_of(r0) and scores_of(r2) == scores_of(r0)  # 16-query batches: query-major
    assert [keys_of([a]) for a in s2] == [keys_of([a]) for a in r2[:4]], "coalesced single queries"
    # the GPU request contract is checked once, before the shards, with the same messages
    E = eng_mod()
    for eng in (e0, e2):
        with pytest.raises(E.GammaStatusError) as ei:
            eng.search(synth.sift_like(513, D, seed=3), 10)
        assert "req num [513] should not larger than [512]" in ei.value.msg
        with pytest.raises(E.GammaStatusError) as ei:
            eng.search(xq[:2], 2049)
        assert "topK num [2049] should not larger than [2048]" in ei.value.msg
    for x in (e0, e1, e2):
        x.close()
    # Load of the sharded dump, sharded and unsharded
    for devs in ([0, 0], None):
        e = E.GammaEngine(str(tmp_path / "two"), space_name="ts", devices=devs)
        e.create_table("ts", D, typ, params(typ, 32, L2))
        assert e.load() == 0
        e.wait_indexed(len(db))
        got = e.search(xq, 10, index_params={"nprobe": 16})
        assert keys_of(got) == keys_of(r2) and scores_of(got) == scores_of(r2)
        e.close()


def test_engine_non_gpu_type_runs_on_first_device(tmp_path, data):
    db, xq = data
    E = eng_mod()
    e = E.GammaEngine(str(tmp_path), space_name="ts", devices=[0, 0])
    e.create_table("ts", D, "IVFFLAT", {"ncentroids": 16, "nprobe": 8, "metric_type": "L2", "training_threshold": 1000})
    for i, v in enumerate(db[:2000]):
        assert e.add_doc(f"doc{i}", v) == 0
    e.build_index()
    e.wait_indexed(2000)
    assert len(keys_of(e.search(xq[:3], 5))[0]) == 5
    e.close()


def test_init_device_list_errors(tmp_path):
    E = eng_mod()
    with pytest.raises(RuntimeError):
        E.GammaEngine(str(tmp_path), devices=[ndev()])
    with pytest.raises(RuntimeError):
        E.GammaEngine(str(tmp_path), devices=[-1])
    E.GammaEngine(str(tmp_path), devices="all").close()
    with pytest.raises(gi().GammaError):
        gi().GammaIndex("GPU_IVFPQ", D, params("GPU_IVFPQ", 16, L2), devices=[0, ndev()])


# ---- host-memory raw store, the realtime tail, RebuildIndex ---------------------------------------------------------
@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
def test_host_store(data, typ):
    """store_type RocksDB: rows reach the shards in host batches, Update copies a host row, and the IVF-Flat list-major
    re-score reads each shard's list rows"""
    db, xq = data
    db = db[:12000]
    ref = build(typ, 16, L2, db, store_type="RocksDB")
    sh = build(typ, 16, L2, db, [0, 0, 0], store_type="RocksDB")
    assert sh.mem_bytes(1) == 0 and sh.mem_bytes(2) > 0
    assert_same(sh.search(xq[:7], 10), ref.search(xq[:7], 10), "host store")
    got, want = sh.search(xq, 10), ref.search(xq, 10)
    if typ == "GPU_IVFFLAT":
        assert sh.last_scan_kernel.startswith("ivf_listmajor"), sh.last_scan_kernel
        contract = list_major_contract(ref, xq, L2, 16)
        FC.check_all(got, contract, 10, L2, "sharded host store list-major")
    else:
        assert_same(got, want, "host store 512")
    rng = np.random.default_rng(9)
    for v in rng.choice(len(db), 100, replace=False):
        row = db[rng.integers(len(db))] - 0.25
        ref.update_vector(int(v), row)
        sh.update_vector(int(v), row)
    assert_same(sh.search(xq[:7], 10), ref.search(xq[:7], 10), "host store after update")
    assert np.array_equal(sh.get_vectors(0, len(db)), ref.get_vectors(0, len(db)))
    ref.close()
    sh.close()


@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
def test_engine_realtime_tail_and_rebuild(tmp_path, data, typ):
    db, xq = data
    db, xq = db[:2600], xq[:16]
    E = eng_mod()
    out = []
    for name, devs in (("plain", None), ("sharded", [0, 0])):
        e = E.GammaEngine(str(tmp_path / name), space_name="rt", devices=devs)
        p = params(typ, 16, L2)
        p["training_threshold"] = 2000
        e.create_table("rt", D, typ, p, refresh_interval=600000, enable_realtime=True)
        for i in range(2000):
            assert e.add_doc(f"doc{i}", db[i]) == 0
        e.wait_indexed(2000)
        for i in range(2000, 2300):  # stored, not indexed: searched brute force and merged
            assert e.add_doc(f"doc{i}", db[i]) == 0
        assert e.status()["min_indexed_num"] == 2000
        tail = e.search(db[2100:2104], 1, index_params={"nprobe": 16})
        assert keys_of(tail) == [[f"doc{i}"] for i in range(2100, 2104)]
        r1 = e.search(xq, 10, index_params={"nprobe": 16})
        for i in range(300):
            e.delete_doc(f"doc{i}")
        assert e.rebuild_index() == 0  # every shard reset, trained again, refilled
        e.wait_indexed(2300)
        r2 = e.search(xq, 10, index_params={"nprobe": 16})
        assert all(int(k[3:]) >= 300 for row in keys_of(r2) for k in row)
        out.append((keys_of(r1), scores_of(r1), keys_of(r2), scores_of(r2)))
        e.close()
    assert out[0] == out[1]


def test_shard_handles_are_read_only(data):
    db, _ = data
    sh = build("GPU_IVFPQ", 16, L2, db[:2000], [0, 0])
    v = sh.shard(1)
    with pytest.raises(gi().GammaError, match="read-only"):
        v.set_centroids(v.get_centroids())
    with pytest.raises(gi().GammaError, match="read-only"):
        v.add_vectors(db[:4])
    assert sh.nlist == 16 and np.array_equal(sh.get_centroids(), v.get_centroids())
    assert sum(sh.list_len(l) for l in range(16)) == 2000 and sh.dead_counts().sum() == 0
    sh.compact()
    v.close()
    sh.close()


def test_init_device_list_from_environment(tmp_path, monkeypatch):
    E = eng_mod()
    monkeypatch.setenv("GAMMA_B200_DEVICES", "")  # set but empty: as if unset
    E.GammaEngine(str(tmp_path)).close()
    monkeypatch.setenv("GAMMA_B200_DEVICES", "all")
    E.GammaEngine(str(tmp_path), devices=[-1]).close()  # the environment overrides the key
    monkeypatch.setenv("GAMMA_B200_DEVICES", "0,0")
    E.GammaEngine(str(tmp_path)).close()
    for bad in ("0,", "x", str(ndev())):
        monkeypatch.setenv("GAMMA_B200_DEVICES", bad)
        with pytest.raises(RuntimeError):
            E.GammaEngine(str(tmp_path))
