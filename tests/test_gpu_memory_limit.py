"""SetMemoryLimitConfig on the H100: the ledger of what the library holds per device and on the host, the documents,
searches and queries it refuses past the limit, and the trim it runs before refusing.  The limit is a percentage of a
total that gb_memory_set_total replaces, so the real SetMemoryLimitConfig path runs at a few MB."""
import struct
import time

import numpy as np
import pytest

from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
MiB = 1 << 20
SLACK = 4 * MiB  # device memory the memory info does not list: segment tables, list directories, small tables


def E():
    from vearch_b200 import engine
    return engine


@pytest.fixture(autouse=True)
def no_limit_after():
    yield
    E().set_memory_limit(0)
    E().set_memory_total(0, 0)
    E().set_memory_total(-1, 0)


def ledger(where=0):
    return E().memory_ledger(where)  # (usage, pool reserved, limit)


def tracked(where=0):
    u, p, _ = ledger(where)
    return u - p


def limit_to(nbytes, where=0):
    """a limit of nbytes at `where`: 50 % of a total of 2 nbytes"""
    E().set_memory_total(where, 2 * nbytes)
    E().set_memory_limit(50)
    assert ledger(where)[2] == nbytes


def make(path, typ, params, dim, store_type="MemoryOnly", **kw):
    e = E().GammaEngine(str(path), space_name="m", **kw)
    e.create_table("m", dim, typ, params, fields=(("_id", wire.DT_STRING, False), ("n", wire.DT_INT, True)),
                   store_type=store_type)
    return e


def add_one(e, v, i):
    return e.add_doc(f"d{i}", v, extra_fields=[("n", struct.pack("<i", i), wire.DT_INT)])


def add(e, xs, start=0):
    for i, v in enumerate(xs):
        assert add_one(e, v, start + i) == 0, start + i


def fill(e, xs):
    add(e, xs)
    e.build_index()
    return e.wait_indexed(len(xs))


def refused(call):
    with pytest.raises(E().GammaStatusError) as ei:
        call()
    assert ei.value.code == 8 and ei.value.msg == "Memory exceed limit: "


def trim(e, xq):
    """run the trim: a search refused under a 1-byte limit releases what the library holds unused, then lift it"""
    limit_to(1)
    refused(lambda: e.search(xq[:1], 1, is_brute_search=1))
    E().set_memory_limit(0)


def mem_of(e):
    mi = e.memory_info()
    return mi["vector_mem"] + mi["index_mem"] + mi["field_range_mem"], mi


def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def test_ledger_matches_memory_info_and_returns_to_start(tmp_path):
    d, n = 128, 20000
    db, xq = synth.sift_like(n, d, seed=1), synth.sift_like(256, d, seed=2)
    bdb = np.packbits(db > np.median(db), axis=1)
    ivf = {"ncentroids": 64, "nprobe": 8, "metric_type": "L2", "training_threshold": 4000}
    start = tracked()
    engines = []
    for typ, params in (("FLAT", {"metric_type": "L2"}), ("IVFPQ", dict(ivf, nsubvector=16)), ("IVFFLAT", ivf),
                        ("BINARYIVF", {"ncentroids": 64, "nprobe": 8, "training_threshold": 4000})):
        before = tracked()
        binary = typ == "BINARYIVF"
        e = make(tmp_path / typ, typ, params, d)
        fill(e, bdb if binary else db)
        q = np.packbits(xq > np.median(db), axis=1) if binary else xq
        e.search(q, 10)  # IVFFLAT: a 256-query batch takes the list-major scan and builds the mirror
        trim(e, q)
        delta = tracked() - before
        mem, mi = mem_of(e)
        assert mi["vector_mem"] > 0 and (typ == "FLAT" or mi["index_mem"] > 0), mi
        assert abs(delta - mem) <= SLACK, (typ, delta, mi)
        engines.append(e)
    for e in engines:
        e.close()
    assert tracked() == start


def test_refused_add_leaves_the_table_unchanged(tmp_path):
    d, n0 = 512, 33000  # 2 KiB rows: the store maps in steps of a quarter of what it holds, here >= 16 MiB
    db, xq = synth.sift_like(n0 + 20000, d, seed=3), synth.sift_like(8, d, seed=4)
    e = make(tmp_path, "IVFPQ", {"ncentroids": 64, "nprobe": 8, "metric_type": "L2", "nsubvector": 32,
                                 "training_threshold": 8000}, d)
    fill(e, db[:n0])
    trim(e, xq)
    limit_to(ledger()[0] + 8 * MiB)  # room for the open step's rows, not for the next step
    i, rc = n0, 0
    while i < len(db):
        rc = add_one(e, db[i], i)
        if rc:
            break
        i += 1
    assert rc == -5 and i > n0, (rc, i)  # the raw-vector stage code of Engine::AddOrUpdate
    assert e.status()["doc_num"] == i
    assert e.get_doc_by_id(f"d{i}")[0] != 0
    st = e.wait_indexed(i)
    assert st["index_status"] == 2 and st["min_indexed_num"] == st["doc_num"] == i
    limit_to(ledger()[0] + 512 * MiB)
    assert add_one(e, db[i], i) == 0
    assert e.status()["doc_num"] == i + 1
    rc, doc = e.get_doc_by_id(f"d{i}")
    assert rc == 0 and np.array_equal(np.frombuffer(doc["emb"][0], np.float32), db[i])
    e.close()


def test_refused_search_query_and_multi_vector_search(tmp_path):
    d, d2, n = 32, 16, 3000
    db, img = synth.sift_like(n, d, seed=5), synth.sift_like(n, d2, seed=6)
    xq, iq = db[:4], img[:4]
    e = E().GammaEngine(str(tmp_path), space_name="mv")
    e.create_table("mv", d, "FLAT", {"metric_type": "L2"}, fields=(("_id", wire.DT_STRING, False),),
                   extra_vectors=[("img", d2, "FLAT", {"metric_type": "L2"})])
    for i in range(n):
        assert e.add_doc(f"d{i}", db[i], extra_fields=[("img", img[i].tobytes(), wire.DT_VECTOR)]) == 0
    e.wait_indexed(n)
    multi = wire.encode_search_request("emb", xq, 5, is_brute_search=1, extra_vec_queries=[("img", iq)])
    calls = {
        "search": lambda: keys_of(e.search(xq, 5, is_brute_search=1)),
        "query": lambda: [it["fields"]["_id"] for it in e.query(document_ids=["d1", "d7"])["items"]],
        "multi": lambda: keys_of(wire.decode_search_response(e.search_raw(multi))),
    }
    base = {k: f() for k, f in calls.items()}
    assert base["search"][0][0] == "d0" and base["query"] == [b"d1", b"d7"]
    trim(e, xq)
    limit_to(ledger()[0] // 2)
    for f in calls.values():
        refused(f)
    E().set_memory_limit(0)
    assert {k: f() for k, f in calls.items()} == base
    e.close()


def test_trim_admits_what_fits_once_released(tmp_path):
    d, n = 128, 20000
    db, xq = synth.sift_like(n + 1, d, seed=7), synth.sift_like(4096, d, seed=8)
    e = make(tmp_path, "FLAT", {"metric_type": "L2"}, d)
    fill(e, db[:n])
    trim(e, xq)
    floor = ledger()[0]
    e.search(xq, 256, is_brute_search=1)  # scratch stays reserved in the pool (and the scan's cache) afterwards
    time.sleep(0.1)
    held = ledger()[0]
    assert held - floor >= 16 * MiB, (floor, held, ledger())
    lim = floor + (held - floor) // 2  # over the limit while the scratch is held, within it once released
    limit_to(lim)
    assert add_one(e, db[n], n) == 0
    assert e.status()["doc_num"] == n + 1
    u, p, _ = ledger()
    assert u <= lim and p < held - floor, (u, p, lim, held, floor)
    e.close()


def test_engines_share_one_budget(tmp_path):
    d = 128
    db, xq = synth.sift_like(20000, d, seed=9), synth.sift_like(4, d, seed=10)
    a = make(tmp_path / "a", "FLAT", {"metric_type": "L2"}, d)
    fill(a, db[:2000])
    trim(a, xq)
    ua = ledger()[0]
    b = make(tmp_path / "b", "FLAT", {"metric_type": "L2"}, d)
    fill(b, db)
    trim(b, xq)
    uab = ledger()[0]
    assert uab - ua >= b.memory_info()["vector_mem"], (ua, uab)
    limit_to((ua + uab) // 2)  # a alone fits, a and b together do not
    refused(lambda: a.search(xq, 5, is_brute_search=1))
    assert add_one(a, db[2000], 2000) == -5
    b.close()
    assert keys_of(a.search(db[:1], 1, is_brute_search=1)) == [["d0"]]
    assert add_one(a, db[2000], 2000) == 0
    a.close()


def test_sharded_index_charges_both_shards_to_their_device(tmp_path):
    d, n = 64, 8000
    db, xq = synth.sift_like(n, d, seed=11), synth.sift_like(4, d, seed=12)
    before = tracked()
    e = make(tmp_path, "GPU_IVFPQ", {"ncentroids": 32, "nprobe": 16, "metric_type": "L2", "nsubvector": 8,
                                     "training_threshold": 32 * 39}, d, devices=[0, 0])
    fill(e, db)
    trim(e, xq)
    mem, mi = mem_of(e)
    assert abs(tracked() - before - mem) <= SLACK, (tracked() - before, mi)
    e.close()
    assert tracked() == before


def test_host_store_charges_the_host_budget(tmp_path):
    d, n = 128, 20000
    db, xq = synth.sift_like(n + 1, d, seed=13), synth.sift_like(4, d, seed=14)
    h0, t0 = ledger(-1)[0], tracked()
    e = make(tmp_path, "FLAT", {"metric_type": "L2"}, d, store_type="RocksDB")
    fill(e, db[:n])
    mi = e.memory_info()
    host = ledger(-1)[0] - h0
    assert host >= n * d * 4 and host == mi["vector_mem"], (host, mi)
    assert tracked() - t0 < n * d * 4 // 4  # the rows are not on the device
    limit_to(ledger(-1)[0] - 1, where=-1)
    assert ledger()[2] > 0 and ledger()[0] < ledger()[2]  # the device is within its limit
    assert add_one(e, db[n], n) == -5
    refused(lambda: e.search(xq, 5, is_brute_search=1))
    E().set_memory_total(-1, 0)
    E().set_memory_limit(0)
    assert add_one(e, db[n], n) == 0
    e.close()
    assert ledger(-1)[0] == h0


def test_limit_parameters(tmp_path):
    d = 32
    db, xq = synth.sift_like(500, d, seed=15), synth.sift_like(2, d, seed=16)
    e = make(tmp_path, "FLAT", {"metric_type": "L2"}, d)
    fill(e, db)
    assert ledger()[2] == 0 and ledger(-1)[2] == 0  # no limit until one is set
    E().set_memory_total(0, 100 * MiB)
    E().set_memory_limit(10)
    assert ledger()[2] == 10 * MiB
    E().set_memory_limit(30)  # a later call replaces the limit
    assert ledger()[2] == 30 * MiB
    limit_to(1)
    refused(lambda: e.search(xq, 1, is_brute_search=1))
    E().set_memory_limit(0)  # removes it
    assert ledger()[2] == 0
    assert keys_of(e.search(db[:1], 1, is_brute_search=1)) == [["d0"]]
    e.close()
