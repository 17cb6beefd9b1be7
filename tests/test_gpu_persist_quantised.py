"""IVFPQFastScan, IVFRABITQ, VEARCH and BINARYIVF kept across Dump / Load through their own index files, on the H100.

At the index seam, for every type under each metric it takes and both raw-vector placements: the dump equals the
struct.pack restatement (tests/quantised_index_file.py) byte for byte; a loaded index holds the same lists, dead counts and
trained state, and answers key for key as the dumped one (scores compared bit for bit) at k up to 4096, with recall_num 0
and > 0, filters, tombstones and a score window, also after the rows that trained it were updated or deleted and the
lists purged; adds, updates, deletes and purges after the load act as on the original.  A refused file (wrong magic,
truncated, wrong dimension, metric or codec parameter) leaves the index untrained, and it trains as before.

Through the engine: the first search right after Load is answered from the file; a dump without the file (as written
before the file existed) is trained again and answers as before; a multi-vector table round-trips every field."""
import math
import os

import numpy as np
import pytest

import quantised_index_file as qf
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = qf.METRIC_L2, qf.METRIC_IP
MNAME = {L2: "L2", IP: "InnerProduct"}
D, BITS, NLIST, N = 32, 256, 16, 3000
CASES = [("IVFPQFastScan", L2), ("IVFPQFastScan", IP), ("IVFRABITQ", L2), ("IVFRABITQ", IP), ("VEARCH", L2),
         ("VEARCH", IP), ("BINARYIVF", L2)]
STORES = ["MemoryOnly", "RocksDB"]


def gi():
    from vearch_b200 import index as gidx
    return gidx


def params_of(kind, metric, **over):
    p = {"ncentroids": NLIST, "nprobe": 8, "training_threshold": 1000}
    if kind != "BINARYIVF":
        p["metric_type"] = MNAME[metric]
    if kind == "IVFPQFastScan":
        p["nsubvector"] = 8
    elif kind == "IVFRABITQ":
        p.update(nb_bits=4, qb=4)
    elif kind == "VEARCH":
        p.update(nsubvector=8, reordering=True)
    p.update(over)
    return p


def make(kind, metric, store="MemoryOnly", d=None, **over):
    p = params_of(kind, metric, **over)
    if kind == "BINARYIVF":
        return gi().BinaryIVFIndex(d or BITS, p, store_type=store)
    cls = {"IVFPQFastScan": gi().GammaIndex, "IVFRABITQ": gi().RaBitQIndex, "VEARCH": gi().VearchIndex}[kind]
    if kind == "IVFPQFastScan":
        return cls(kind, d or D, p, store_type=store)
    return cls(d or D, p, store_type=store)


def rows(kind, n, seed, d=None):
    if kind == "BINARYIVF":
        return synth.binary_clustered(n, d or BITS, seed=seed, n_clusters=16, flip=0.2)
    return synth.sift_like(n, d or D, seed=seed, n_clusters=32)


def bitmap(n, vids):
    b = np.zeros(n, bool)
    b[np.asarray(vids, np.int64)] = True
    return np.packbits(b, bitorder="little")


def restate(kind, idx, metric, nprobe):
    off, codes, ids = idx.export_lists()
    codec = {}
    if kind == "BINARYIVF":
        cent = idx.get_real_centroids()
        codec["binary_centroids"] = idx.get_centroids()
    else:
        cent = idx.get_centroids()
    if kind == "IVFPQFastScan":
        codec["pq_centroids"] = idx.get_pq_centroids()
    elif kind == "IVFRABITQ":
        codec.update(nb_bits=idx.nb_bits, qb=idx.qb)
    elif kind == "VEARCH":
        codec.update(nsub=idx.nsub, blocks=idx.blocks, ns_threshold=0.2 if metric == IP else math.nan, reordering=True,
                     codebook=idx.get_codebook())
    return qf.write_quantised(kind, idx.d, metric, nprobe, cent, off, codes, ids, idx.indexed_count, idx.code_size,
                              **codec)


def table_of(kind, idx, metric):
    t = dict(d=idx.d, nlist=idx.nlist, metric=metric)
    if kind == "IVFPQFastScan":
        t["M"] = idx.pq_m
    elif kind == "IVFRABITQ":
        t.update(nb_bits=idx.nb_bits, qb=idx.qb)
    elif kind == "VEARCH":
        t.update(nsub=idx.nsub, blocks=idx.blocks, ns_threshold=0.2 if metric == IP else math.nan, reordering=True)
    return t


def conditions(kind, total, del_bm, seed):
    """search settings: k up to 4096, recall_num 0 and > 0, a filter, tombstones (always in the lists), the deletion
    bitmap, a score window (filled in from the first answer)"""
    filt = np.packbits(np.random.default_rng(seed).random(total) < 0.5, bitorder="little")
    every = {"nprobe": NLIST}
    return [dict(k=10, params=every, del_bitmap=del_bm),
            dict(k=4096, params=every, del_bitmap=del_bm),
            dict(k=20, params={"nprobe": 4, "recall_num": 0}),
            dict(k=20, params={"nprobe": 6, "recall_num": 150}, del_bitmap=del_bm),
            dict(k=64, params=every, del_bitmap=del_bm, filter_bitmap=filt),
            dict(k=64, params=every, del_bitmap=del_bm, window=True)]


def answers(idx, xq, conds):
    out = []
    for c in conds:
        c = dict(c)
        k = c.pop("k")
        if c.pop("window", False):
            dis, _ = idx.search(xq, k, params=c["params"], del_bitmap=c.get("del_bitmap"))
            lo, hi = sorted((float(np.min(dis[:, 8])), float(np.max(dis[:, 40]))))
            c.update(min_score=lo, max_score=hi)
        dis, ids = idx.search(xq, k, **c)
        out.append((dis.view(np.uint32).copy(), ids.copy()))
    return out


def assert_same_answers(a, b):
    assert len(a) == len(b)
    for (da, ia), (db_, ib) in zip(a, b):
        assert np.array_equal(ia, ib)
        assert np.array_equal(da, db_)


def assert_same_lists(a, b):
    for x, y in zip(a.export_lists(), b.export_lists()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.dead_counts(), b.dead_counts())
    assert a.indexed_count == b.indexed_count


def churn(kind, idx, seed, vids_upd, vids_del, del_bm_vids):
    """updates (the rows' old entries tombstoned), then deletes (counted dead; their vids join del_bm_vids)"""
    new = rows(kind, len(vids_upd), seed)
    for v, x in zip(vids_upd, new):
        idx.update_vector(int(v), x)
    idx.delete_vectors(np.asarray(vids_del, np.int64))
    del_bm_vids.extend(int(v) for v in vids_del)


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("kind,metric", CASES)
def test_index_round_trip(tmp_path, kind, metric, store):
    idx = make(kind, metric, store)
    db = rows(kind, N, 1)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    # the rows that trained the index are updated and deleted, then purged: retraining could not restore this state
    dead = []
    churn(kind, idx, 2, np.arange(0, 60), [100, 101, 205, 999, 1500], dead)
    assert idx.purge(0.0, del_bitmap=bitmap(N, dead)) > 0
    # tombstones and counted-dead entries left in the file, and rows appended after the purge
    churn(kind, idx, 3, np.arange(60, 90), [300, 301, 2999], dead)
    idx.add_vectors(rows(kind, 200, 4))
    idx.add_pending()
    total = N + 200
    del_bm = bitmap(total, dead)
    xq = rows(kind, 5, 9)
    conds = conditions(kind, total, del_bm, 5)
    before = answers(idx, xq, conds)

    idx.dump(tmp_path, "emb.000")
    path = tmp_path / "emb.000" / qf.FILE[kind]
    buf = path.read_bytes()
    parsed = qf.read_quantised(buf, kind, table_of(kind, idx, metric))
    assert parsed["indexed_count"] == idx.indexed_count == total
    assert buf == restate(kind, idx, metric, parsed["nprobe"])
    assert (parsed["ids"] < 0).sum() > 0  # tombstones travel

    idx2 = make(kind, metric, store)
    idx2.add_vectors(idx.get_vectors(0, total))
    assert not idx2.is_trained
    assert idx2.load(tmp_path, "emb.000") == total
    assert idx2.is_trained
    # the file's tombstones are counted dead; deletions are the owner's to count again (DESIGN section 8, T1)
    idx2.delete_vectors(np.asarray(dead, np.int64))
    assert_same_lists(idx, idx2)
    assert np.array_equal(idx.get_centroids(), idx2.get_centroids())
    assert_same_answers(answers(idx2, xq, conds), before)
    idx2.dump(tmp_path, "again.000")
    assert (tmp_path / "again.000" / qf.FILE[kind]).read_bytes() == buf

    # after the load both indexes take the same adds, updates, deletes and purge
    more = rows(kind, 150, 6)
    for ix in (idx, idx2):
        ix.add_vectors(more)
        ix.add_pending()
        d2 = list(dead)
        churn(kind, ix, 7, np.arange(0, 20), [7, 1234], d2)
        ix.purge(0.3, del_bitmap=bitmap(total + 150, d2))
    dead += [7, 1234]
    assert_same_lists(idx, idx2)
    conds = conditions(kind, total + 150, bitmap(total + 150, dead), 8)
    assert_same_answers(answers(idx2, xq, conds), answers(idx, xq, conds))
    idx.close()
    idx2.close()


def refused(kind, metric, tmp_path, buf, name, rows_, **make_kw):
    """the file `buf` under `name`, loaded into a fresh index: refused, nothing of it kept, and the index trains"""
    d = tmp_path / name / "emb.000"
    d.mkdir(parents=True)
    (d / qf.FILE[kind]).write_bytes(buf)
    ix = make(kind, metric, **make_kw)
    ix.add_vectors(rows_)
    with pytest.raises(gi().GammaError):
        ix.load(tmp_path / name, "emb.000")
    assert not ix.is_trained and ix.indexed_count == 0
    ix.train()
    ix.add_pending()
    assert ix.is_trained and ix.indexed_count == len(rows_)
    ix.close()


@pytest.mark.parametrize("kind,metric", [("IVFPQFastScan", IP), ("IVFRABITQ", L2), ("VEARCH", IP), ("BINARYIVF", L2)])
def test_refused_files_leave_the_index_untrained(tmp_path, kind, metric):
    idx = make(kind, metric)
    db = rows(kind, 2000, 11)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    idx.dump(tmp_path, "emb.000")
    buf = (tmp_path / "emb.000" / qf.FILE[kind]).read_bytes()
    refused(kind, metric, tmp_path, b"IwPQ" + buf[4:], "magic", db)
    refused(kind, metric, tmp_path, buf[:len(buf) // 2], "half", db)
    refused(kind, metric, tmp_path, buf[:-2], "tail", db)  # the trailing indexed count cut
    if kind == "BINARYIVF":
        refused(kind, metric, tmp_path, buf, "nlist", db, ncentroids=NLIST * 2)
        refused(kind, metric, tmp_path, buf, "dim", rows(kind, 2000, 11, d=BITS * 2), d=BITS * 2)
    else:
        refused(kind, metric, tmp_path, buf, "metric", db, metric_type=MNAME[IP if metric == L2 else L2])
        refused(kind, metric, tmp_path, buf, "dim", rows(kind, 2000, 11, d=D * 2), d=D * 2)
        wrong = {"IVFPQFastScan": dict(nsubvector=4), "IVFRABITQ": dict(nb_bits=5),
                 "VEARCH": dict(nsubvector=4)}[kind]
        refused(kind, metric, tmp_path, buf, "param", db, **wrong)
    if kind == "IVFRABITQ":
        refused(kind, metric, tmp_path, buf, "qb", db, qb=2)
    if kind == "VEARCH":
        refused(kind, metric, tmp_path, buf, "reordering", db, reordering=False)
    # a file of the same layout read back into a matching index still loads
    ok = make(kind, metric)
    ok.add_vectors(db)
    assert ok.load(tmp_path, "emb.000") == 2000 and ok.is_trained
    ok.close()
    idx.close()


def test_reference_ivfrabitq_file_is_ignored(tmp_path):
    """a CPU partition's ivfrabitq.index (faiss IndexIVFRaBitQ) is not this engine's file: it is never read"""
    d = tmp_path / "emb.000"
    d.mkdir()
    (d / "ivfrabitq.index").write_bytes(b"Iwrq" + bytes(64))
    ix = make("IVFRABITQ", L2)
    ix.add_vectors(rows("IVFRABITQ", 1500, 12))
    assert ix.load(tmp_path, "emb.000") == 0 and not ix.is_trained
    ix.close()


# ---- the engine ------------------------------------------------------------------------------------------------------
def eng_mod():
    from vearch_b200 import engine
    return engine


def ids_of(res):
    return [[int(it["fields"]["_id"].decode()[3:]) for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


ENGINE_METRIC = {"IVFPQFastScan": L2, "IVFRABITQ": IP, "VEARCH": IP, "BINARYIVF": L2}


def engine(path, kind, store="MemoryOnly", **kw):
    from vearch_b200 import wire
    e = eng_mod().GammaEngine(str(path), space_name="pq")
    p = params_of(kind, ENGINE_METRIC[kind], training_threshold=2000)
    e.create_table("pq", BITS if kind == "BINARYIVF" else D, kind, p, fields=(("_id", wire.DT_STRING, False),),
                   store_type=store, **kw)
    return e


ENGINE_QUERIES = [dict(topn=10, index_params={"nprobe": NLIST}), dict(topn=1000, index_params={"nprobe": 4}),
                  dict(topn=20, index_params={"nprobe": 8, "recall_num": 200})]


def engine_answers(e, xq):
    out = []
    for q in ENGINE_QUERIES:
        res = e.search(xq, q["topn"], index_params=q["index_params"])
        out.append((ids_of(res), scores_of(res)))
    return out


@pytest.mark.parametrize("store", STORES)
@pytest.mark.parametrize("kind", ["IVFPQFastScan", "IVFRABITQ", "VEARCH", "BINARYIVF"])
def test_engine_load_answers_at_once(tmp_path, kind, store):
    n = 2500
    db, xq = rows(kind, n, 21), rows(kind, 4, 22)
    e = engine(tmp_path, kind, store)
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    assert e.wait_indexed(n)["index_status"] == 2
    new = rows(kind, 40, 23)
    for i in range(40):  # rows of the training sample updated: retraining would see other rows
        assert e.add_doc(f"doc{i}", new[i]) == 0
    for i in (50, 51, 52):
        assert e.delete_doc(f"doc{i}") == 0
    before = engine_answers(e, xq)
    assert e.dump() == 0
    e.close()
    f = tmp_path / "retrieval_model_index" / "emb.000" / qf.FILE[kind]
    assert f.exists()

    e2 = engine(tmp_path, kind, store)
    assert e2.load() == 0
    assert e2.status()["index_status"] == 2  # trained from the file, before any indexing pass
    assert engine_answers(e2, xq) == before  # no wait_indexed
    assert e2.get_doc_by_id("doc51")[0] == -1
    # the loaded engine takes updates and deletes
    assert e2.add_doc("doc3", new[5]) == 0 and e2.delete_doc("doc60") == 0
    e2.wait_indexed(n)
    assert e2.get_doc_by_id("doc3")[1]["emb"][0] == new[5].tobytes()
    res = e2.search(xq, 1000, index_params={"nprobe": NLIST})
    assert all(60 not in r and 51 not in r for r in ids_of(res))
    e2.close()

    # a dump without the file (written before the file existed): Load trains the index again from the raw rows; until
    # that is done a search of this table (more than 100 documents) is refused as IndexNotTrained (code 2)
    os.remove(f)
    e3 = engine(tmp_path, kind, store)
    assert e3.load() == 0
    try:
        e3.search(xq, 10, index_params={"nprobe": NLIST})
    except eng_mod().GammaStatusError as ex:
        assert ex.code == 2
    e3.wait_indexed(n)
    assert len(e3.search(xq, 10, index_params={"nprobe": NLIST})[0]["items"]) == 10
    e3.close()


@pytest.mark.parametrize("kind", ["IVFPQFastScan", "IVFRABITQ", "VEARCH", "BINARYIVF"])
def test_engine_dump_without_the_file_answers_as_before(tmp_path, kind):
    """no update touched the training rows: retraining restores the same state, as a dump written before this file
    existed always did"""
    n = 2500
    db, xq = rows(kind, n, 31), rows(kind, 4, 32)
    e = engine(tmp_path, kind)
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    e.wait_indexed(n)
    assert e.delete_doc("doc7") == 0
    before = engine_answers(e, xq)
    assert e.dump() == 0
    e.close()
    os.remove(tmp_path / "retrieval_model_index" / "emb.000" / qf.FILE[kind])
    e2 = engine(tmp_path, kind)
    assert e2.load() == 0
    e2.wait_indexed(n)
    assert engine_answers(e2, xq) == before
    e2.close()


def test_multi_vector_table_round_trips(tmp_path):
    from vearch_b200 import wire
    n, nq, topn = 2500, 5, 300
    db, xq = rows("IVFPQFastScan", n, 41), rows("IVFPQFastScan", nq, 42)
    f1, q1 = rows("IVFRABITQ", n, 43, d=16), rows("IVFRABITQ", nq, 44, d=16)
    f2, q2 = rows("VEARCH", n, 45, d=24), rows("VEARCH", nq, 46, d=24)

    def make_engine():
        e = eng_mod().GammaEngine(str(tmp_path), space_name="mv")
        e.create_table("mv", D, "IVFPQFastScan", params_of("IVFPQFastScan", L2, training_threshold=2000),
                       extra_vectors=[("f1", 16, "IVFRABITQ", params_of("IVFRABITQ", L2, training_threshold=2000)),
                                      ("f2", 24, "VEARCH", params_of("VEARCH", IP, nsubvector=6,
                                                                     training_threshold=2000))])
        return e

    def ask(e):
        res = e.search(xq, topn, extra_vec_queries=[("f1", q1), ("f2", q2)], multi_vector_rank=1,
                       index_params={"nprobe": NLIST, "recall_num": 500})
        return ids_of(res), scores_of(res)

    e = make_engine()
    for i in range(n):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("f1", f1[i].tobytes(), wire.DT_VECTOR),
                                                         ("f2", f2[i].tobytes(), wire.DT_VECTOR)]) == 0
    e.wait_indexed(n)
    for i in range(20):  # training rows of every field updated
        assert e.add_doc(f"doc{i}", db[n - 1 - i], extra_fields=[("f1", f1[n - 1 - i].tobytes(), wire.DT_VECTOR),
                                                                 ("f2", f2[n - 1 - i].tobytes(), wire.DT_VECTOR)]) == 0
    e.wait_indexed(n)
    before = ask(e)
    assert sum(len(r) for r in before[0]) > nq
    assert e.dump() == 0
    e.close()
    base = tmp_path / "retrieval_model_index"
    for field, kind in (("emb", "IVFPQFastScan"), ("f1", "IVFRABITQ"), ("f2", "VEARCH")):
        assert (base / f"{field}.000" / qf.FILE[kind]).exists()
    e2 = make_engine()
    assert e2.load() == 0
    assert ask(e2) == before
    e2.close()
