"""Backup on the H100 (DESIGN.md §8, backup and snapshots): the partition captured on the device under the table lock,
written after the lock is released.

- Every file a backup writes under backup/retrieval_model_index equals the file of the same name Dump writes, for every
  index type, both raw-vector placements, a multi-vector table, indexed scalar fields and a field whose index was changed
  at run time, each after updates, deletes and a purge.
- A follower that takes the backup as ApplySnapshot does (backup/* moved up into a fresh path) and Loads it answers
  searches, GetDocByID and Query exactly as the leader does, its persisting index loaded without training.
- While a backup is held between capture and write, writes and searches complete, backup_status reads 1 and a second
  backup is refused with code 5; the backup holds the state before the writes.
- A stage that does not fit under the memory limit goes to pinned host memory; the ledger counts it while held.
- The list-pack kernel, through the capture hook, against export_lists at code sizes from 1 byte to the largest.
- A backup that cannot be written leaves the previous one whole and no temporary directory."""
import os
import shutil
import struct
import threading
import time

import numpy as np
import pytest

from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
D, BITS, NLIST, N = 32, 256, 16, 3000
FI = ("fi", wire.DT_INT, True)


def E():
    from vearch_b200 import engine
    return engine


def gi():
    from vearch_b200 import index
    return index


BASE = {"ncentroids": NLIST, "nprobe": 8, "metric_type": "L2", "training_threshold": 1000}
CASES = {
    "FLAT": ("FLAT", {"metric_type": "L2"}, None),
    "IVFFLAT": ("IVFFLAT", BASE, None),
    "IVFPQ_opq": ("IVFPQ", dict(BASE, nsubvector=8, opq={"nsubvector": 8}), None),
    "IVFPQ_nbits4": ("IVFPQ", dict(BASE, nsubvector=8, nbits_per_idx=4), None),
    "IVFPQFastScan": ("IVFPQFastScan", dict(BASE, nsubvector=8), None),
    "IVFRABITQ": ("IVFRABITQ", dict(BASE, metric_type="InnerProduct", nb_bits=4, qb=4), None),
    "VEARCH": ("VEARCH", dict(BASE, metric_type="InnerProduct", nsubvector=8, reordering=True), None),
    "BINARYIVF": ("BINARYIVF", {"ncentroids": NLIST, "nprobe": 8, "training_threshold": 1000}, None),
    "GPU_IVFPQ_sharded": ("GPU_IVFPQ", dict(BASE, nsubvector=8), [0, 0]),
    "GPU_IVFFLAT": ("GPU_IVFFLAT", BASE, None),
}


IWPQ = ("IVFPQ", "GPU_IVFPQ")


def rows(typ, n, seed):
    if typ == "BINARYIVF":
        return synth.binary_clustered(n, BITS, seed=seed, n_clusters=16, flip=0.2)
    return synth.sift_like(n, D, seed=seed, n_clusters=32)


def make_engine(path, case, store="MemoryOnly", extra=()):
    typ, params, devices = CASES[case]
    e = E().GammaEngine(str(path), space_name="bk", devices=devices)
    e.create_table("bk", BITS if typ == "BINARYIVF" else D, typ, params, fields=(("_id", wire.DT_STRING, False), FI),
                   store_type=store, extra_vectors=extra)
    return e


def fi(i):
    return [("fi", struct.pack("<i", i % 50), wire.DT_INT)]


def churn(e, typ, db, n, extra_rows=None):
    """adds, then updates of training rows, deletes of 40 % of the documents and an update that purges the lists"""
    def ex(i, src):
        return [(name, r[src].tobytes(), wire.DT_VECTOR) for name, r in (extra_rows or {}).items()]
    for i in range(n):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=fi(i) + ex(i, i)) == 0
    e.wait_indexed(n)
    for i in range(30):
        assert e.add_doc(f"doc{i}", db[n - 1 - i], extra_fields=fi(i + 7) + ex(i, n - 1 - i)) == 0
    for i in range(200, 200 + int(0.4 * n)):
        assert e.delete_doc(f"doc{i}") == 0
    assert e.add_doc("doc5", db[n - 40], extra_fields=fi(5) + ex(5, n - 40)) == 0  # lists 30 % dead are purged


def ids_of(res):
    return [[it["fields"]["_id"] for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def answers(e, xq, extra_q=()):
    out = []
    rf = [("fi", struct.pack("<i", 10), struct.pack("<i", 30), True, True)]
    for kw in (dict(), dict(range_filters=rf), dict(term_filters=[("fi", struct.pack("<i", 7))]),
               dict(is_brute_search=1)):
        res = e.search(xq, 50, index_params={"nprobe": NLIST}, extra_vec_queries=extra_q, **kw)
        out.append((ids_of(res), scores_of(res)))
    docs = [e.get_doc_by_id(f"doc{i}") for i in (0, 5, 29, 31, 250, 1500, 2999)]
    q = e.query(range_filters=rf, limit=100, fields=["_id", "fi"])
    return out, docs, [it["fields"] for it in q["items"]]


def files(root):
    out = {}
    for dp, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(dp, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def apply_snapshot(leader, follower):
    """gammaEngine.ApplySnapshot: the files under <path>/backup/, each entry moved up into the new path"""
    src = os.path.join(leader, "backup")
    for name in os.listdir(src):
        shutil.copytree(os.path.join(src, name), os.path.join(follower, name))


def assert_backup_is_dump(path):
    dump, bk = files(os.path.join(path, "retrieval_model_index")), files(os.path.join(path, "backup", "retrieval_model_index"))
    assert sorted(bk) == sorted(dump) and "dump.done" in bk
    for name in dump:
        assert bk[name] == dump[name], name
    assert sorted(os.listdir(os.path.join(path, "backup"))) == ["retrieval_model_index"]


@pytest.mark.parametrize("store", ["MemoryOnly", "RocksDB"])
@pytest.mark.parametrize("case", list(CASES))
def test_backup_equals_dump_and_restores(tmp_path, case, store):
    typ = CASES[case][0]
    leader, follower = tmp_path / "leader", tmp_path / "follower"
    db, xq = rows(typ, N, 1), rows(typ, 5, 2)
    e = make_engine(leader, case, store)
    churn(e, typ, db, N)
    assert e.status()["backup_status"] == 0
    assert e.dump() == 0
    e.backup()
    assert e.status()["backup_status"] == 0
    assert_backup_is_dump(str(leader))
    before = answers(e, xq)
    e.close()

    apply_snapshot(str(leader), str(follower))
    f = make_engine(follower, case, store)
    assert f.load() == 0
    if typ != "FLAT":
        assert f.status()["index_status"] == 2  # trained state and lists from the backup, no training pass
    if typ in IWPQ:
        # an "IwPQ" file carries no indexed count: after a purge, Load counts fewer indexed rows than the lists cover and
        # the indexing thread adds some rows twice, whether the files came from Dump or from Backup (DESIGN §8); both
        # are compared once that thread has caught up
        f.wait_indexed(N)
        shutil.copytree(leader / "retrieval_model_index", tmp_path / "from_dump" / "retrieval_model_index")
        g = make_engine(tmp_path / "from_dump", case, store)
        assert g.load() == 0
        g.wait_indexed(N)
        before = answers(g, xq)
        g.close()
    got = answers(f, xq)
    f.close()
    assert got == before


def test_multi_vector_scalar_and_changed_index(tmp_path):
    leader, follower = tmp_path / "leader", tmp_path / "follower"
    db, xq = rows("IVFFLAT", N, 3), rows("IVFFLAT", 4, 4)
    f1, q1 = synth.sift_like(N, 16, seed=5, n_clusters=32), synth.sift_like(4, 16, seed=6, n_clusters=32)
    extra = [("f1", 16, "IVFFLAT", BASE, "RocksDB")]

    def make(path):
        e = make_engine(path, "IVFFLAT", extra=extra)
        return e

    e = make(leader)
    churn(e, "IVFFLAT", db, N, extra_rows={"f1": f1})
    e.add_field_index("f1", "IVFRABITQ", dict(BASE, nb_bits=2, qb=4))  # Dump and Backup wait for its build
    assert e.dump() == 0
    e.backup()
    assert_backup_is_dump(str(leader))
    assert os.path.exists(leader / "backup" / "retrieval_model_index" / "f1.000" / "gb_ivfrabitq.index")
    before = answers(e, xq, extra_q=[("f1", q1)])
    e.close()
    apply_snapshot(str(leader), str(follower))
    f = make(follower)
    assert f.load() == 0
    assert answers(f, xq, extra_q=[("f1", q1)]) == before
    f.close()


def wait_for(cond, what, timeout=60.0):
    t0 = time.time()
    while not cond():
        assert time.time() - t0 < timeout, what
        time.sleep(0.005)


def test_backup_is_a_point_in_time_without_blocking(tmp_path):
    leader, follower = tmp_path / "leader", tmp_path / "follower"
    db, xq = rows("IVFFLAT", N + 200, 7), rows("IVFFLAT", 5, 8)
    e = make_engine(leader, "IVFFLAT")
    churn(e, "IVFFLAT", db, N)
    before = answers(e, xq)
    errs = []

    def run():
        try:
            e.backup()
        except Exception as ex:  # noqa: BLE001 -- reported by the main thread
            errs.append(ex)

    assert E().backup_hold(1) == 1
    t = threading.Thread(target=run)
    try:
        t.start()
        wait_for(lambda: E().backup_hold(-1) == 2, "the backup did not reach its hold")
        # the lock is released: every one of these returns while the backup waits
        for i in range(N, N + 200):
            assert e.add_doc(f"doc{i}", db[i], extra_fields=fi(i)) == 0
        assert e.add_doc("doc0", db[N + 5], extra_fields=fi(3)) == 0
        assert e.add_doc("doc31", db[N + 6], extra_fields=fi(4)) == 0
        assert e.delete_doc("doc1") == 0 and e.delete_doc("doc2999") == 0
        assert len(e.search(xq, 10, index_params={"nprobe": NLIST})[0]["items"]) == 10
        assert e.status()["backup_status"] == 1
        with pytest.raises(E().GammaStatusError) as ex:
            e.backup()
        assert ex.value.code == 5 and "backup is in progress" in ex.value.msg
        assert t.is_alive() and E().backup_hold(-1) == 2
    finally:
        E().backup_hold(0)
        t.join(120)
    assert not t.is_alive() and not errs, errs
    assert e.status()["backup_status"] == 0
    e.close()

    apply_snapshot(str(leader), str(follower))
    f = make_engine(follower, "IVFFLAT")
    assert f.load() == 0
    assert answers(f, xq) == before
    assert all(f.get_doc_by_id(f"doc{i}")[0] == -1 for i in (N, N + 1, N + 199))
    assert f.get_doc_by_id("doc1")[0] == 0 and f.get_doc_by_id("doc2999")[0] == 0
    assert f.get_doc_by_id("doc0")[1]["emb"][0] == db[N - 1].tobytes()  # the update made before capture
    f.close()


def tracked(device):
    u, pool, _ = E().memory_ledger(device)
    return u - pool


@pytest.mark.parametrize("store", ["MemoryOnly", "RocksDB"])
def test_stage_placement_and_ledger(tmp_path, store):
    path = tmp_path / "p"
    db = rows("IVFPQ", N, 9)
    e = make_engine(path, "IVFPQ_opq", store)
    churn(e, "IVFPQ", db, N)
    results = []
    try:
        for limited in (False, True):
            dev0, host0 = tracked(0), tracked(-1)
            if limited:  # the device is at its limit: every stage goes to pinned host memory
                E().set_memory_limit(50)
                E().set_memory_total(0, 2 * tracked(0))
            assert E().backup_hold(1) == 1
            t = threading.Thread(target=e.backup)
            t.start()
            try:
                wait_for(lambda: E().backup_hold(-1) == 2, "the backup did not reach its hold")
                stage = E().backup_stage()
                held = (tracked(0) - dev0, tracked(-1) - host0)
            finally:
                E().backup_hold(0)
                t.join(120)
            assert tracked(0) == dev0 and tracked(-1) == host0  # the stage is freed once written
            results.append((stage, held, files(path / "backup" / "retrieval_model_index")))
    finally:
        E().set_memory_limit(0)
        E().set_memory_total(0, 0)
    (s_dev, held_dev, f_dev), (s_host, held_host, f_host) = results
    rows_bytes = N * D * 4
    assert s_dev[0] > 0 and held_dev[0] >= s_dev[0] and held_dev[1] >= s_dev[1]
    if store == "RocksDB":  # raw rows of host placement are staged on the host in either case
        assert s_dev[1] == rows_bytes
    else:
        assert s_dev[1] == 0 and s_dev[0] > rows_bytes
    assert s_host == (0, s_dev[0] + s_dev[1]) and held_host[0] == 0 and held_host[1] >= s_host[1]
    assert f_host == f_dev
    assert e.dump() == 0
    assert_backup_is_dump(str(path))
    e.close()


def test_failed_backup_leaves_the_previous_one(tmp_path):
    if os.geteuid() == 0:
        pytest.skip("permissions do not bind root")
    path = tmp_path / "p"
    db = rows("IVFPQ", N, 10)
    e = make_engine(path, "IVFFLAT")
    churn(e, "IVFFLAT", db, 2000)
    e.backup()
    good = files(path / "backup" / "retrieval_model_index")
    assert e.add_doc("docnew", db[2500], extra_fields=fi(1)) == 0
    os.chmod(path / "backup", 0o555)
    try:
        with pytest.raises(E().GammaStatusError) as ex:
            e.backup()
        assert ex.value.code == 5
    finally:
        os.chmod(path / "backup", 0o755)
    assert os.listdir(path / "backup") == ["retrieval_model_index"]
    assert files(path / "backup" / "retrieval_model_index") == good
    assert e.status()["backup_status"] == 0
    e.backup()  # writable again: the new state replaces it
    assert files(path / "backup" / "retrieval_model_index") != good
    assert os.listdir(path / "backup") == ["retrieval_model_index"]
    e.close()


# ---- the list-pack kernel, through the capture hook ---------------------------------------------------------------
PACK = [  # (type, d, params): code sizes from 1 byte to the largest the shape-limit tests reach
    ("IVFPQ", 4, {"nsubvector": 1}),                         # 1 byte, lists several chunks long
    ("IVFPQ", 10, {"nsubvector": 5, "nbits_per_idx": 3}),    # 2 bytes
    ("IVFPQ", 64, {"nsubvector": 64}),                       # 64 bytes, 16-byte units
    ("IVFPQ", 146, {"nsubvector": 146}),                     # 146 bytes
    ("IVFPQ", 234, {"nsubvector": 234, "nbits_per_idx": 7}),
    ("IVFPQ", 703, {"nsubvector": 703, "nbits_per_idx": 4}),
    ("IVFPQ", 3128, {"nsubvector": 3128, "nbits_per_idx": 1}),  # 391 bytes
    ("IVFFLAT", 1, {}),                                      # 16 bytes in memory, 4 on disk
    ("IVFFLAT", 6, {}),
    ("IVFFLAT", 128, {}),
    ("IVFPQFastScan", 14, {"nsubvector": 7}),                # 4 bytes
    ("IVFPQFastScan", 256, {"nsubvector": 256}),             # 128 bytes
    ("IVFRABITQ", 64, {"nb_bits": 4}),
    ("IVFRABITQ", 4096, {"nb_bits": 9}),
    ("VEARCH", 255, {"nsubvector": 255}),
    ("BINARYIVF", 8, {}),                                    # 1 byte
    ("BINARYIVF", 3512, {}),                                 # 439 bytes
]


def pack_index(typ, d, p):
    nlist = 2 if d == 4 else 8
    n = 140000 if d == 4 else 3000  # d = 4: lists past one 65 536-entry chunk of 1-byte codes
    params = dict(p, ncentroids=nlist, nprobe=nlist, training_threshold=min(n, 2000))
    if typ == "BINARYIVF":
        idx = gi().BinaryIVFIndex(d, params)
        idx.add_vectors(synth.binary_clustered(n, d, seed=11, n_clusters=8, flip=0.2))
    else:
        cls = {"IVFRABITQ": gi().RaBitQIndex, "VEARCH": gi().VearchIndex}.get(typ)
        idx = cls(d, params) if cls else gi().GammaIndex(typ, d, dict(params, metric_type="L2"))
        idx.add_vectors(synth.sift_like(n, d, seed=11, n_clusters=16))
    idx.train()
    idx.add_pending()
    return idx


def expected_pack(idx, file_cb):
    off, codes, ids = idx.export_lists()
    out = bytearray()
    for l in range(len(off) - 1):
        out += codes[off[l]:off[l + 1], :file_cb].tobytes() + ids[off[l]:off[l + 1]].tobytes()
    return bytes(out)


@pytest.mark.parametrize("typ,d,p", PACK, ids=[f"{t}-{d}-{'-'.join(map(str, p.values()))}" for t, d, p in PACK])
def test_list_pack_kernel(typ, d, p):
    idx = pack_index(typ, d, p)
    file_cb = d * 4 if typ == "IVFFLAT" else idx.code_size
    got, on_host = idx.capture_lists()
    assert not on_host and got.tobytes() == expected_pack(idx, file_cb)
    # list 0 emptied and a few entries of the others dropped by a purge, then one entry tombstoned where it is
    off, _, ids = idx.export_lists()
    gone = np.concatenate([ids[off[0]:off[1]], ids[off[1]:off[-1]][::7]])
    bm = np.zeros(int(ids.max()) + 1, bool)
    bm[gone] = True
    idx.delete_vectors(gone)
    idx.purge(threshold=0.0, del_bitmap=np.packbits(bm, bitorder="little"))
    lens = np.diff(idx.export_lists()[0])
    assert lens[0] == 0
    idx.tombstone(int(np.argmax(lens)), 1)
    got, _ = idx.capture_lists()
    want = expected_pack(idx, file_cb)
    assert got.tobytes() == want and len(want) == int(lens.sum()) * (file_cb + 8)
    idx.close()
