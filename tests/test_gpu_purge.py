"""GPU tests of the inverted-list purge (RealTimeMemData::CompactIfNeed on the device): dead entries leave the lists of
every IVF type exactly as the numpy restatement (oracle_purge) says, no search result changes, and everything keyed on
the lists (vid positions, dead counters, the list-major caches, the host-store row pointers, the index file, the engine)
follows."""
import threading
import time

import numpy as np
import pytest

from oracle_purge import purge as P
from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
T = P.TOMBSTONE


def gi():
    from vearch_b200 import index
    return index


def make(kind, n=6000, seed=1, **over):
    """(index, rows, queries, a maker of fresh rows) of one IVF type, trained and filled on the device"""
    g = gi()
    rng = np.random.default_rng(seed)
    base = {"ncentroids": 16, "nprobe": 8, "metric_type": "L2", "training_threshold": 2000}
    if kind == "BINARYIVF":
        cs = over.pop("code_bytes", 24)
        rows = lambda m, s: np.random.default_rng(s).integers(0, 256, (m, cs), dtype=np.uint8)
        db, xq = rows(n, seed), rows(40, seed + 1)
        idx = g.BinaryIVFIndex(cs * 8, {"ncentroids": 16})
        idx.set_centroids(db[rng.choice(n, 16, replace=False)])
        idx.add_vectors(db)
        idx.add_pending()
        return idx, db, xq, rows
    d, cls, typ, extra = {
        "IVFFLAT": (32, g.GammaIndex, "IVFFLAT", {}),
        "IVFPQ8": (32, g.GammaIndex, "IVFPQ", {"nsubvector": 8}),
        "IVFPQ4": (48, g.GammaIndex, "IVFPQ", {"nsubvector": 12, "nbits_per_idx": 4}),  # 6-byte packed rows
        "IVFPQFastScan": (32, g.GammaIndex, "IVFPQFastScan", {"nsubvector": 16}),
        "IVFRABITQ": (32, g.RaBitQIndex, None, {"nb_bits": 4, "qb": 4}),
        "VEARCH": (32, g.VearchIndex, None, {"nsubvector": 8}),
    }[kind]
    d = over.pop("d", d)
    rows = lambda m, s: synth.sift_like(m, d, seed=s)
    db, xq = rows(n, seed), rows(40, seed + 1)
    params = {**base, **extra, **over}
    idx = cls(typ, d, params) if typ else cls(d, params)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    return idx, db, xq, rows


def churn(idx, db, rows, seed, hot_share=0.45, cold_share=0.04):
    """Delete and update a seeded mix: every other list loses hot_share of its entries (two thirds deleted, one third
    updated to fresh rows), the others cold_share.  Returns the deletion bitmap and the deleted vids."""
    rng = np.random.default_rng(seed)
    off, _, ids = idx.export_lists()
    deleted, updated = [], []
    for l in range(len(off) - 1):
        v = ids[off[l]:off[l + 1]]
        m = int(len(v) * (hot_share if l % 2 == 0 else cold_share))
        pick = rng.choice(v, m, replace=False)
        deleted += pick[: (2 * m + 2) // 3].tolist()
        updated += pick[(2 * m + 2) // 3:].tolist()
    fresh = rows(len(updated), seed + 7)
    for vid, x in zip(updated, fresh):
        idx.update_vector(int(vid), x)
    idx.delete_vectors(deleted)
    idx.delete_vectors(deleted[:5])  # counted once
    return P.bitmap_of(deleted, len(db)), np.array(deleted, np.int64)


def expected_dead(off, ids, bm):
    lst = np.repeat(np.arange(len(off) - 1), np.diff(off))
    return np.bincount(lst[~P.live(ids, bm)], minlength=len(off) - 1)


def same(a, b):
    return np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])


def searches(idx, xq, bm, kind):
    out = [idx.search(xq, 10, del_bitmap=bm)]
    if kind in ("IVFPQ8", "IVFPQ4", "IVFPQFastScan", "IVFRABITQ"):  # the exact re-rank of the 60 best estimates
        out.append(idx.search(xq, 10, params={"recall_num": 60}, del_bitmap=bm))
    out.append(idx.search(xq[:3], 100, del_bitmap=bm))
    return out


def purge_and_check(idx, db, xq, rows, kind, seed):
    bm, deleted = churn(idx, db, rows, seed)
    off, codes, ids = idx.export_lists()
    dead = expected_dead(off, ids, bm)
    assert np.array_equal(idx.dead_counts(), dead)
    sel = P.select_lists(dead, np.diff(off), 0.3)
    assert 0 < len(sel) < len(off) - 1, "the mix must leave lists on both sides of the threshold"
    before = searches(idx, xq, bm, kind)
    off2, codes2, ids2, dropped = P.purge(off, codes, ids, sel, bm)
    assert idx.purge(0.3, bm) == dropped > 0
    o, c, i = idx.export_lists()
    assert np.array_equal(o, off2) and np.array_equal(i, ids2) and np.array_equal(c, codes2)
    assert np.array_equal(idx.dead_counts(), np.where(np.isin(np.arange(len(dead)), sel), 0, dead))
    assert idx.purge(0.3, bm) == 0  # nothing is left above the threshold
    after = searches(idx, xq, bm, kind)
    assert all(same(a, b) for a, b in zip(before, after))
    # positions were refreshed: an update of a survivor of a purged list tombstones that entry and no other
    pos = P.vid_positions(off2, ids2, len(db))
    l = int(sel[0])
    vid = int(ids2[off2[l] + 1])
    idx.update_vector(vid, rows(1, seed + 9)[0])
    o3, _, i3 = idx.export_lists()
    at = int(o3[l] + (pos[vid] & 0xFFFFFFFF))
    assert pos[vid] >> 32 == l and i3[at] == (vid | T) and (i3 < 0).sum() == (ids2 < 0).sum() + 1
    want = idx.dead_counts()
    assert want[l] == 1
    # a purged vid is in no list any more: deleting it again counts nothing
    gone = [int(v) for v in deleted if pos[v] < 0][:3]
    assert len(gone) == 3
    idx.delete_vectors(gone)
    assert np.array_equal(idx.dead_counts(), want)
    # threshold 0 takes every list that has a dead entry
    assert idx.purge(0.0, bm) > 0 and not idx.dead_counts().any()
    _, _, i4 = idx.export_lists()
    assert P.live(i4, bm).all()


@pytest.mark.parametrize("kind", ["IVFFLAT", "IVFPQ8", "IVFPQ4", "IVFPQFastScan", "BINARYIVF", "IVFRABITQ", "VEARCH"])
def test_purge_matches_the_restatement_and_changes_no_result(kind):
    idx, db, xq, rows = make(kind, seed=11)
    try:
        purge_and_check(idx, db, xq, rows, kind, seed=12)
    finally:
        idx.close()


@pytest.mark.parametrize("kind,over,code_size", [
    ("IVFPQ4", {"d": 8, "nsubvector": 2}, 1),        # byte copies
    ("IVFPQ8", {"d": 48, "nsubvector": 24}, 24),     # 8-byte units
    ("BINARYIVF", {"code_bytes": 439}, 439),         # BINARYIVF's longest row, odd
    ("IVFFLAT", {"d": 128}, 512),                    # 16-byte units, 32 per row
    ("IVFFLAT", {"d": 18}, 80),                      # a row padded to whole 16-byte units
])
def test_purge_code_sizes(kind, over, code_size):
    idx, db, xq, rows = make(kind, n=4000, seed=21, **over)
    try:
        assert idx.code_size == code_size
        bm, _ = churn(idx, db, rows, seed=22)
        off, codes, ids = idx.export_lists()
        sel = P.select_lists(expected_dead(off, ids, bm), np.diff(off), 0.3)
        before = idx.search(xq, 10, del_bitmap=bm)
        off2, codes2, ids2, dropped = P.purge(off, codes, ids, sel, bm)
        assert idx.purge(0.3, bm) == dropped > 0
        o, c, i = idx.export_lists()
        assert np.array_equal(o, off2) and np.array_equal(i, ids2) and np.array_equal(c, codes2)
        assert same(before, idx.search(xq, 10, del_bitmap=bm))
    finally:
        idx.close()


def test_purge_long_list_beside_a_single_entry_and_an_empty_list():
    d, n = 8, 50000  # list 0: 48 chunks and a ragged tail; list 1: one entry; list 2: none
    rng = np.random.default_rng(31)
    cent = np.zeros((3, d), np.float32)
    cent[1], cent[2] = 100, 10000
    db = rng.normal(0, 1, (n + 1, d)).astype(np.float32)
    db[n] += 100
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": 3, "nprobe": 3, "metric_type": "L2"})
    try:
        idx.set_centroids(cent)
        idx.add(db)
        assert [idx.list_len(l) for l in range(3)] == [n, 1, 0]
        deleted = np.concatenate([rng.choice(n, int(n * 0.4), replace=False), [n]])
        idx.delete_vectors(deleted)
        bm = P.bitmap_of(deleted, n + 1)
        xq = db[rng.choice(n, 20)] + np.float32(0.01)
        before = idx.search(xq, 10, del_bitmap=bm)
        off, codes, ids = idx.export_lists()
        off2, codes2, ids2, dropped = P.purge(off, codes, ids, [0, 1], bm)
        assert idx.purge(0.3, bm) == dropped == len(deleted)
        o, c, i = idx.export_lists()
        assert o.tolist() == [0, n - int(n * 0.4), n - int(n * 0.4), n - int(n * 0.4)]
        assert np.array_equal(o, off2) and np.array_equal(i, ids2) and np.array_equal(c, codes2)
        # the scan picks its kernel variant by list length, and the variants sum the 8 dimensions in different orders:
        # the same documents, scores to the last bit or two
        after = idx.search(xq, 10, del_bitmap=bm)
        assert np.array_equal(before[1], after[1]) and np.allclose(before[0], after[0], rtol=1e-6, atol=0)
        idx.add(db[n:n + 1])  # the emptied list takes entries again
        assert idx.list_len(1) == 1 and idx.get_list(1)[1].tolist() == [n + 1]
    finally:
        idx.close()


# ---- list-major searches: the caches beside the lists ---------------------------------------------------------------
def listmajor_index(kind, store_type=None):
    """d = 128, 16 lists, 128 queries x 4 probes: 32 (query, probe) pairs per list, the list-major paths"""
    d, n, nlist = 128, 20000, 16
    db, xq = synth.sift_like(n, d, seed=41), synth.sift_like(128, d, seed=42)
    params = {"ncentroids": nlist, "nprobe": 4, "metric_type": "L2", "training_threshold": 4000}
    if kind == "IVFPQ":
        params["nsubvector"] = 16
    idx = gi().GammaIndex(kind, d, params, store_type=store_type)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    return idx, db, xq


LM_KERNEL = {"IVFFLAT": "ivf_listmajor", "IVFPQ": "pqtc_scan_kernel"}


@pytest.mark.parametrize("kind,store_type", [("IVFFLAT", None), ("IVFFLAT", "RocksDB"), ("IVFPQ", None)])
def test_list_major_search_is_unchanged_by_a_purge(kind, store_type):
    idx, db, xq = listmajor_index(kind, store_type)
    try:
        bm, _ = churn(idx, db, lambda m, s: synth.sift_like(m, 128, seed=s), seed=43)
        before = idx.search(xq, 10, del_bitmap=bm)
        assert idx.last_scan_kernel.startswith(LM_KERNEL[kind]), idx.last_scan_kernel
        assert idx.purge(0.3, bm) > 0
        after = idx.search(xq, 10, del_bitmap=bm)  # host store: the winners are re-scored through the rebuilt row pointers
        assert idx.last_scan_kernel.startswith(LM_KERNEL[kind]), idx.last_scan_kernel
        assert same(before, after)
    finally:
        idx.close()


@pytest.mark.parametrize("kind", ["IVFFLAT", "IVFPQ"])
def test_purge_then_append_back_to_the_old_length_rebuilds_the_caches(kind):
    """Lengths alone do not identify the content of a list any more: a purge followed by appends restores every length
    with other entries.  The list-major caches (the IVF-Flat mirror, IVF-PQ's per-entry |r|^2) must notice."""
    idx, db, xq = listmajor_index(kind)
    try:
        idx.search(xq, 10)  # builds the caches
        assert idx.last_scan_kernel.startswith(LM_KERNEL[kind])
        off, _, ids = idx.export_lists()
        l = int(np.argmax(np.diff(off)))
        v = ids[off[l]:off[l + 1]]
        gone, stay = v[: len(v) // 2], v[len(v) // 2:]  # the first half goes: every survivor moves
        idx.delete_vectors(gone)
        bm = P.bitmap_of(gone, len(db) + len(gone))
        assert idx.purge(0.3, bm) == len(gone)
        idx.add(db[stay[: len(gone)]])  # copies of survivors: they land in list l again
        assert [idx.list_len(j) for j in range(16)] == np.diff(off).tolist()
        got = idx.search(xq, 10, del_bitmap=bm)
        assert idx.last_scan_kernel.startswith(LM_KERNEL[kind]), idx.last_scan_kernel
        # the same index three queries at a time scans query-major, which reads no cache
        parts = [idx.search(xq[q:q + 3], 10, del_bitmap=bm) for q in range(0, len(xq), 3)]
        assert not idx.last_scan_kernel.startswith(LM_KERNEL[kind])
        qd, qi = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
        if kind == "IVFPQ":  # the filter's bound is rigorous: byte-equal to the exact table scan
            assert same(got, (qd, qi))
        else:  # 3xTF32 scores against exact ones (duplicates tie: compare the scores)
            assert np.allclose(got[0], qd, rtol=1e-4, atol=1e-2)
            assert np.mean([len(set(a) & set(b)) for a, b in zip(got[1], qi)]) >= 9.5
    finally:
        idx.close()


def test_dump_after_a_purge_is_the_restated_file_and_loads_back(tmp_path):
    import gamma_index_file as gif
    idx, db, xq, rows = make("IVFFLAT", seed=51)
    try:
        bm, _ = churn(idx, db, rows, seed=52)
        assert idx.purge(0.3, bm) > 0
        off, codes, ids = idx.export_lists()
        want = idx.search(xq, 10, del_bitmap=bm)
        dead = idx.dead_counts()
        idx.dump(tmp_path, "emb.000")
        with open(tmp_path / "emb.000" / "ivfflat.index", "rb") as fh:
            buf = fh.read()
        assert buf == gif.write_ivfflat(32, gif.METRIC_L2, 8, idx.get_centroids(), off, codes.view(np.float32), ids,
                                        idx.indexed_count)
        again = gi().GammaIndex("IVFFLAT", 32, {"ncentroids": 16, "nprobe": 8, "metric_type": "L2"})
        again.add_vectors(db)
        assert again.load(tmp_path, "emb.000") > 0
        o, c, i = again.export_lists()
        assert np.array_equal(o, off) and np.array_equal(c, codes) and np.array_equal(i, ids)
        lst = np.repeat(np.arange(16), np.diff(off))
        assert np.array_equal(again.dead_counts(), np.bincount(lst[ids < 0], minlength=16))  # the file's tombstones
        assert (again.dead_counts() <= dead).all()
        assert same(want, again.search(xq, 10, del_bitmap=bm))
        again.close()
    finally:
        idx.close()


# ---- the engine -----------------------------------------------------------------------------------------------------
def test_engine_purges_behind_deletes_and_updates_while_searches_run(tmp_path):
    import gamma_index_file as gif
    from oracle import oracle as orc
    from vearch_b200 import engine
    d, n, nlist = 32, 4000, 16
    db, xq = synth.sift_like(n, d, seed=61), synth.sift_like(16, d, seed=62)
    params = {"ncentroids": nlist, "nprobe": nlist, "metric_type": "L2", "training_threshold": 1000}
    e = engine.GammaEngine(str(tmp_path), space_name="pg")
    e.create_table("pg", d, "IVFFLAT", params, fields=(("_id", wire.DT_STRING, False),))
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    e.wait_indexed(n)
    mem0 = e.memory_info()["index_mem"]
    rng = np.random.default_rng(63)
    perm = rng.permutation(n)
    deleted, updated = perm[:1600], perm[1600:2000]
    cur = db.copy()
    cur[updated] = synth.sift_like(len(updated), d, seed=64)
    dead = np.zeros(n, bool)
    seen, errors, stop = [], [], threading.Event()

    def reader():  # every answer is made of documents that were not deleted before the search began
        while not stop.is_set():
            gone = dead.copy()
            try:
                res = e.search(xq[:4], 10, index_params={"nprobe": nlist})
                seen.append((gone, [[int(it["fields"]["_id"].decode()[3:]) for it in r["items"]] for r in res]))
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)
            time.sleep(0.002)

    t = threading.Thread(target=reader)
    t.start()
    try:
        for v in deleted:
            assert e.delete_doc(f"doc{v}") == 0
            dead[v] = True
        for v in updated:  # every update is followed by a purge of the lists that are 30 % dead
            assert e.add_doc(f"doc{v}", cur[v]) == 0
        time.sleep(0.5)  # a pass of the indexing thread
    finally:
        stop.set()
        t.join()
    assert not errors and len(seen) > 0
    for gone, rows in seen:
        assert all(len(r) == 10 and not gone[r].any() for r in rows)
    bm = np.packbits(dead, bitorder="little")
    do, io = orc.flat_search(cur, xq, 10, orc.METRIC_L2, del_bitmap=bm)  # nprobe = nlist: exact
    res = e.search(xq, 10, index_params={"nprobe": nlist})
    assert [[int(it["fields"]["_id"].decode()[3:]) for it in r["items"]] for r in res] == io.tolist()
    assert np.array_equal(np.array([[it["score"] for it in r["items"]] for r in res], np.float32), do)
    assert e.memory_info()["index_mem"] <= mem0
    assert e.dump() == 0
    e.close()
    with open(tmp_path / "retrieval_model_index" / "emb.000" / "ivfflat.index", "rb") as fh:
        buf = fh.read()
    f = gif.read_index_file(buf)
    lens = np.diff(f["list_off"])
    # 2000 of 4000 entries died; whatever is still dead sits in lists below the threshold
    assert len(f["ids"]) < n + len(updated) - 1200
    share = np.bincount(np.repeat(np.arange(nlist), lens)[~P.live(f["ids"], bm)], minlength=nlist) / np.maximum(lens, 1)
    assert (share < 0.3).all()
    assert buf == gif.write_ivfflat(d, f["metric"], f["nprobe"], f["centroids"], f["list_off"], f["codes"].view(np.float32),
                                    f["ids"], f["indexed_count"])
    e2 = engine.GammaEngine(str(tmp_path), space_name="pg")
    e2.create_table("pg", d, "IVFFLAT", params, fields=(("_id", wire.DT_STRING, False),))
    assert e2.load() == 0
    e2.wait_indexed(n)
    res2 = e2.search(xq, 10, index_params={"nprobe": nlist})
    assert [[it["fields"]["_id"] for it in r["items"]] for r in res2] == [[it["fields"]["_id"] for it in r["items"]] for r in res]
    e2.close()
