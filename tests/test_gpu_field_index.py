"""Vector indexes changed at run time: AddFieldIndexWithParams / RemoveFieldIndex on a vector field.  A removed index
leaves the field searched exactly; an added index is trained and filled from the stored rows while the field's current
index keeps serving, then replaces it.  Dump waits for a build to end in its swap, so the tests use it to wait."""
import os
import threading

import numpy as np
import pytest

from oracle import oracle as orc
from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
L2 = orc.METRIC_L2
D, N, NQ, K = 32, 3000, 16, 10
BASE = {"ncentroids": 16, "training_threshold": 1000}
PARAMS = {
    "FLAT": {"metric_type": "L2"},
    "IVFFLAT": {**BASE, "nprobe": 16, "metric_type": "L2"},
    "IVFPQ": {**BASE, "nprobe": 8, "nsubvector": 8, "metric_type": "L2"},
    "IVFPQFastScan": {**BASE, "nprobe": 8, "nsubvector": 16, "metric_type": "L2"},
    "IVFRABITQ": {**BASE, "nprobe": 16, "metric_type": "L2"},
    "VEARCH": {**BASE, "nsubvector": 8, "metric_type": "L2"},
    "GPU_IVFPQ": {**BASE, "nprobe": 16, "nsubvector": 8, "metric_type": "L2", "training_threshold": 624},
    "GPU_IVFFLAT": {**BASE, "nprobe": 16, "metric_type": "L2", "training_threshold": 624},
}
HOST_OK = ("FLAT", "IVFFLAT", "IVFPQ", "IVFRABITQ")  # store placements tested per type
CASES = [(t, s) for t in PARAMS for s in (("MemoryOnly", "RocksDB") if t in HOST_OK else ("MemoryOnly",))]


def E():
    from vearch_b200 import engine
    return engine


@pytest.fixture(scope="module")
def data():
    return synth.sift_like(N + 400, D, seed=5), synth.sift_like(NQ, D, seed=6)


def engine(path, typ, params, store="MemoryOnly", devices=None, **kw):
    e = E().GammaEngine(str(path), space_name="fi", devices=devices)
    e.create_table("fi", D, typ, params, store_type=store, fields=(("_id", wire.DT_STRING, False),), **kw)
    return e


def feed(e, db, start=0):
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{start + i}", v) == 0


def keys(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def scores(res):
    return [[it["score"] for it in r["items"]] for r in res]


def wait_ready(e):
    assert e.dump() == 0  # waits for a run-time build to swap or fail
    return e.wait_indexed(0)


def index_dir(path):
    return os.path.join(str(path), "retrieval_model_index", "emb.000")


@pytest.mark.parametrize("typ,store", CASES)
def test_remove_serves_exact_results(tmp_path, data, typ, store):
    db, xq = data
    e = engine(tmp_path / "a", typ, PARAMS[typ], store)
    feed(e, db[:N])
    e.wait_indexed(N)
    for i in range(0, N, 7):
        assert e.delete_doc(f"doc{i}") == 0
    assert e.dump() == 0
    before = e.memory_info()["index_mem"]
    e.remove_field_index("emb")
    e.remove_field_index("emb")  # nothing left to remove: OK
    assert e.memory_info()["index_mem"] < before or typ == "FLAT"
    assert not os.path.exists(index_dir(tmp_path / "a"))
    assert os.path.exists(os.path.join(str(tmp_path / "a"), "retrieval_model_index", "fi.gbdump"))
    f = engine(tmp_path / "b", "FLAT", {"metric_type": "L2"})
    feed(f, db[:N])
    for i in range(0, N, 7):
        assert f.delete_doc(f"doc{i}") == 0
    f.wait_indexed(N)
    for kw in ({}, {"min_score": 0.0, "max_score": 2e5}):
        got, want = e.search(xq, K, **kw), f.search(xq, K, **kw)
        assert keys(got) == keys(want) and scores(got) == scores(want)
    assert e.status()["index_status"] == 2
    e.close()
    f.close()


@pytest.mark.parametrize("typ,store", CASES + [("BINARYIVF", "MemoryOnly")])
def test_add_equals_a_table_created_with_the_type(tmp_path, data, typ, store):
    db, xq = data
    if typ == "BINARYIVF":
        rng = np.random.default_rng(3)
        rows = rng.integers(0, 256, (N, D // 8), dtype=np.uint8)
        qs = rng.integers(0, 256, (NQ, D // 8), dtype=np.uint8)
        first, p = ("BINARYIVF", {"ncentroids": 16, "training_threshold": 1000})
        params = {"ncentroids": 8, "training_threshold": 1000}
    else:
        rows, qs = db[:N], xq
        first, p = "FLAT", {"metric_type": "L2"}
        params = PARAMS[typ]
    e = engine(tmp_path / "a", first, p, store)
    feed(e, rows)
    e.wait_indexed(N)
    e.remove_field_index("emb")
    e.add_field_index("emb", typ, params)
    wait_ready(e)
    f = engine(tmp_path / "b", typ, params, store)
    feed(f, rows)
    f.wait_indexed(N)
    got, want = e.search(qs, K), f.search(qs, K)
    assert keys(got) == keys(want) and scores(got) == scores(want)
    assert e.status()["min_indexed_num"] == N
    e.close()
    f.close()


def test_replace_while_serving(tmp_path, data):
    db, xq = data
    e = engine(tmp_path / "a", "IVFPQ", PARAMS["IVFPQ"])
    feed(e, db[:N])
    e.wait_indexed(N)
    errors, stop = [], threading.Event()

    def searcher():
        while not stop.is_set():
            try:
                r = e.search(xq, K)
                assert len(r) == NQ and all(len(x["items"]) == K for x in r)
            except Exception as ex:  # noqa: BLE001
                errors.append(repr(ex))

    t = threading.Thread(target=searcher)
    t.start()
    e.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
    feed(e, db[N:N + 200], start=N)  # added, deleted and updated during the build
    for i in range(N, N + 200, 5):
        assert e.delete_doc(f"doc{i}") == 0
    assert e.add_doc("doc1", db[N + 399]) == 0
    wait_ready(e)
    stop.set()
    t.join()
    assert errors == []
    e.wait_indexed(N + 200)  # the rows Dump flushed after the swap, indexed by the indexing thread
    live = [i for i in range(N + 200) if not (i >= N and (i - N) % 5 == 0)]
    rows = db[:N + 200].copy()
    rows[1] = db[N + 399]
    _, io = orc.flat_search(rows[live], xq, K, L2)
    assert keys(e.search(xq, K)) == [[f"doc{live[j]}" for j in row] for row in io]  # nprobe = nlist: exact
    r = e.search(db[N:N + 200], 1)
    for i, row in zip(range(N, N + 200), keys(r)):
        assert (row == [f"doc{i}"]) == ((i - N) % 5 != 0)
    assert keys(e.search(db[N + 399:N + 400], 1)) == [["doc1"]]
    e.close()


def test_validation_matches_create_table(tmp_path, data):
    db, _ = data
    e = engine(tmp_path / "a", "IVFFLAT", PARAMS["IVFFLAT"])
    feed(e, db[:N])
    e.wait_indexed(N)
    before = e.memory_info()
    for typ, params, code in (("", {}, 3), ("HNSW", {}, 3), ("IVFFLAT", {"ncentroids": 8, "nprobe": 32}, 4),
                              ("IVFPQ", {"ncentroids": 8, "nprobe": 4, "nsubvector": 5}, 4),
                              ("BINARYIVF", {"ncentroids": 8}, 4)):
        with pytest.raises(E().GammaStatusError) as ei:
            e.add_field_index("emb", typ, params)
        assert ei.value.code == code
        if typ and typ != "BINARYIVF":
            c = E().GammaEngine(str(tmp_path / "c"), space_name="c")
            with pytest.raises(E().GammaStatusError) as ci:
                c.create_table("c", D, typ, params)
            assert (ci.value.code, ci.value.msg) == (ei.value.code, ei.value.msg)
            c.close()
    assert e.memory_info() == before
    e.close()


def test_memory_limit(tmp_path, data):
    db, xq = data
    e = engine(tmp_path / "a", "FLAT", {"metric_type": "L2"})
    feed(e, db[:N])
    e.wait_indexed(N)
    want = keys(e.search(xq, K))
    usage, pool, _ = E().memory_ledger(0)
    try:  # what the library holds besides its pool, plus less than N IVF-Flat rows (D * 4 + 8 bytes each)
        E().set_memory_total(0, 2 * (usage - pool + 10_000))
        E().set_memory_limit(50)
        with pytest.raises(E().GammaStatusError) as ei:
            e.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
        assert ei.value.code == 8
    finally:
        E().set_memory_limit(0)
        E().set_memory_total(0, 0)
    assert keys(e.search(xq, K)) == want and e.memory_info()["index_mem"] == 0
    e.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
    wait_ready(e)
    assert e.memory_info()["index_mem"] > 0
    e.close()


@pytest.mark.parametrize("steps", [("add",), ("remove",), ("remove", "add")])
def test_dump_load(tmp_path, data, steps):
    db, xq = data
    e = engine(tmp_path, "IVFPQ", PARAMS["IVFPQ"])
    feed(e, db[:N])
    e.wait_indexed(N)
    for s in steps:
        if s == "add":
            e.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
        else:
            e.remove_field_index("emb")
    wait_ready(e)
    want = e.search(xq, K)
    e.close()
    g = engine(tmp_path, "IVFPQ", PARAMS["IVFPQ"])  # the schema CreateTable was given
    assert g.load() == 0
    g.wait_indexed(0 if steps[-1] == "remove" else N)
    got = g.search(xq, K)
    assert keys(got) == keys(want) and scores(got) == scores(want)
    g.close()


def test_unchanged_table_has_no_index_record(tmp_path, data):
    db, _ = data
    e = engine(tmp_path, "IVFFLAT", PARAMS["IVFFLAT"])
    feed(e, db[:N])
    e.wait_indexed(N)
    assert e.dump() == 0
    with open(os.path.join(str(tmp_path), "retrieval_model_index", "fi.gbdump"), "rb") as fh:
        assert not fh.read().endswith(b"GBFIDX01")
    e.close()


def test_multi_vector_table(tmp_path, data):
    db, xq = data
    d2 = 16
    img = synth.sift_like(N, d2, seed=7)
    imq = synth.sift_like(NQ, d2, seed=8)
    e = E().GammaEngine(str(tmp_path), space_name="mv")
    e.create_table("mv", D, "IVFFLAT", PARAMS["IVFFLAT"], extra_vectors=[("img", d2, "IVFFLAT", {**PARAMS["IVFFLAT"]})])
    for i in range(N):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("img", img[i].tobytes(), wire.DT_VECTOR)]) == 0
    e.wait_indexed(N)
    assert e.dump() == 0
    img_file = os.path.join(str(tmp_path), "retrieval_model_index", "img.000")
    snap = {f: open(os.path.join(img_file, f), "rb").read() for f in os.listdir(img_file)}

    def img_search():
        req = wire.encode_search_request("img", imq, K)
        return wire.decode_search_response(e.search_raw(req))

    before = img_search()
    e.remove_field_index("emb")
    assert img_search() == before
    assert {f: open(os.path.join(img_file, f), "rb").read() for f in os.listdir(img_file)} == snap
    req = wire.encode_search_request("emb", xq, 200, extra_vec_queries=[("img", imq)], multi_vector_rank=1)
    res = wire.decode_search_response(e.search_raw(req))
    _, i1 = orc.flat_search(db[:N], xq, 200, L2)
    for q, r in enumerate(res):
        sc = [it["score"] for it in r["items"]]
        assert sc == sorted(sc)
        assert all(int(it["fields"]["_id"].decode()[3:]) in set(i1[q].tolist()) for it in r["items"])
    e.close()


def test_sharded_add(tmp_path, data):
    db, xq = data
    out, mem = [], []
    for sub, devices in (("a", [0, 0]), ("b", None)):
        e = engine(tmp_path / sub, "FLAT", {"metric_type": "L2"}, devices=devices)
        feed(e, db[:N])
        e.wait_indexed(N)
        e.add_field_index("emb", "GPU_IVFPQ", PARAMS["GPU_IVFPQ"])
        wait_ready(e)
        out.append(e.search(xq, K))
        mem.append(e.memory_info()["index_mem"])
        e.close()
    assert keys(out[0]) == keys(out[1]) and scores(out[0]) == scores(out[1])
    assert mem[0] > mem[1]  # sharded: every shard holds its own centroids and codebook


@pytest.mark.parametrize("typ", ["IVFFLAT", "IVFPQ"])
def test_remove_inner_product_with_filters(tmp_path, data, typ):
    db, xq = data
    fields = (("_id", wire.DT_STRING, False), ("tag", wire.DT_STRING, True))
    ip = {**PARAMS[typ], "metric_type": "InnerProduct"}
    tables = []
    for sub, t, p in (("a", typ, ip), ("b", "FLAT", {"metric_type": "InnerProduct"})):
        e = E().GammaEngine(str(tmp_path / sub), space_name="fi")
        e.create_table("fi", D, t, p, fields=fields)
        for i in range(N):
            assert e.add_doc(f"doc{i}", db[i], extra_fields=[("tag", f"t{i % 7}".encode(), wire.DT_STRING)]) == 0
        for i in range(0, N, 11):
            assert e.delete_doc(f"doc{i}") == 0
        e.wait_indexed(N)
        tables.append(e)
    e, f = tables
    e.remove_field_index("emb")
    for kw in ({"term_filters": [("tag", b"t1\x01t4")]}, {"term_filters": [("tag", b"t3", 2)], "min_score": 1e4}):
        got, want = e.search(xq, K, **kw), f.search(xq, K, **kw)
        assert keys(got) == keys(want) and scores(got) == scores(want)
    e.close()
    f.close()


def test_add_below_training_threshold(tmp_path, data):
    """an index added while the field holds fewer rows than its threshold serves exact answers, then trains once the
    rows arrive, on the same first rows a table created with the type trains on"""
    db, xq = data
    e = engine(tmp_path / "a", "FLAT", {"metric_type": "L2"})
    feed(e, db[:500])
    e.wait_indexed(500)
    e.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
    assert e.dump() == 0  # the swap; the index stays untrained, so index_status is 0 as after CreateTable
    assert e.status()["index_status"] == 0
    _, io = orc.flat_search(db[:500], xq, K, L2)
    assert keys(e.search(xq, K)) == [[f"doc{j}" for j in row] for row in io]  # exact until trained, not refused
    feed(e, db[500:N], start=500)
    e.build_index()
    e.wait_indexed(N)
    f = engine(tmp_path / "b", "IVFFLAT", PARAMS["IVFFLAT"])
    feed(f, db[:N])
    f.build_index()
    f.wait_indexed(N)
    got, want = e.search(xq, K), f.search(xq, K)
    assert keys(got) == keys(want) and scores(got) == scores(want)
    e.close()
    f.close()
    g = engine(tmp_path / "c", "FLAT", {"metric_type": "L2"})  # an empty field: the index is changed before ingest
    g.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
    assert g.dump() == 0
    feed(g, db[:N])
    g.build_index()
    g.wait_indexed(N)
    got = g.search(xq, K)
    assert keys(got) == keys(want) and scores(got) == scores(want)
    g.close()


def test_every_answer_is_old_or_new(tmp_path, data):
    db, xq = data
    e = engine(tmp_path / "a", "IVFPQ", PARAMS["IVFPQ"])
    feed(e, db[:N])
    e.wait_indexed(N)
    old = keys(e.search(xq, K))
    _, io = orc.flat_search(db[:N], xq, K, L2)
    new = [[f"doc{j}" for j in row] for row in io]  # IVFFLAT with nprobe = nlist: exact
    assert old != new
    answers, stop = [], threading.Event()

    def searcher():
        while not stop.is_set():
            answers.append(keys(e.search(xq, K)))

    t = threading.Thread(target=searcher)
    t.start()
    e.add_field_index("emb", "IVFFLAT", PARAMS["IVFFLAT"])
    wait_ready(e)
    stop.set()
    t.join()
    assert answers and all(a in (old, new) for a in answers)
    for _ in range(5):
        assert keys(e.search(xq, K)) == new
    e.close()
