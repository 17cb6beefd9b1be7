"""Each vid's list entries as an IVF index keeps them (vid_slots) and the dead counts keyed on them, on the H100.

1. Unspilled IVFFLAT, IVFPQ, IVFPQFastScan, BINARYIVF and a two-shard GPU_IVFFLAT (read through its shard handles in
   local vids), through add, update (also of a deleted vid), delete (repeated, negative and past the table), a purge
   without and with the deletion bitmap, Dump / Load, and a refused Load followed by a rebuild: every live vid has one
   slot, at an entry holding it; a purged vid has none; each list's dead count is its tombstones plus the entries of the
   vids delete_vectors counted (once each; an update takes the count back, a purge that keeps the entry counts it again
   in its new list, a loaded index has counted none).
2. Spilled IVFPQFastScan, IVFRABITQ and VEARCH: after updates, deletes and a purge, Dump / Load gives every vid the same
   two slots.
3. A spilled file with a vid in three lists, or twice in one list, is refused with its message; the refused index has
   no slots, and a rebuild gives every vid two."""
import numpy as np
import pytest

import soar_index_file as sf
from oracle_purge import purge as P
from test_gpu_persist_quantised import table_of
from test_gpu_soar import LAM, built as built_spilled, spilled as make_spilled
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
N, NLIST, CB = 6000, 16, 24  # rows, lists, BINARYIVF bytes per row
UNSPILLED = ["IVFFLAT", "IVFPQ", "IVFPQFastScan", "BINARYIVF", "GPU_IVFFLAT"]


def gi():
    from vearch_b200 import index
    return index


def rows(kind, m, seed):
    if kind == "BINARYIVF":
        return np.random.default_rng(seed).integers(0, 256, (m, CB), dtype=np.uint8)
    return synth.sift_like(m, 32, seed=seed)


def fresh(kind):
    """an empty index of `kind`; GPU_IVFFLAT sharded in two on device 0"""
    if kind == "BINARYIVF":
        return gi().BinaryIVFIndex(CB * 8, {"ncentroids": NLIST})
    p = {"ncentroids": NLIST, "nprobe": 8, "metric_type": "L2", "training_threshold": 2000}
    p.update({"IVFPQ": {"nsubvector": 8}, "IVFPQFastScan": {"nsubvector": 16}}.get(kind, {}))
    return gi().GammaIndex(kind, 32, p, devices=[0, 0] if kind == "GPU_IVFFLAT" else None)


def build(kind, db):
    idx = fresh(kind)
    idx.add_vectors(db)
    if kind == "BINARYIVF":
        idx.set_centroids(db[np.random.default_rng(2).choice(len(db), NLIST, replace=False)])
    else:
        idx.train()
    idx.add_pending()
    return idx


def handles(idx):
    """(handle, shard, shard count): the index itself, or each shard of a sharded one (its lists hold local vids)"""
    S = idx.shard_count
    return [(idx.shard(s) if S > 1 else idx, s, S) for s in range(S)]


def check(idx, counted, gone):
    """every vid not in `gone` has one slot, at a live entry holding it, and is in its lists once; every vid in `gone`
    has no slot and no entry; each list's dead count is its tombstones plus the entries of the vids in `counted`"""
    n = idx.ntotal
    for h, s, S in handles(idx):
        off, _, ids = h.export_lists()
        lst = np.repeat(np.arange(len(off) - 1), np.diff(off))
        live = ids >= 0
        local = np.arange(s, n, S) // S
        want_n = np.ones(len(local), np.int64)
        want_n[[v // S for v in gone if v % S == s]] = 0
        assert np.array_equal(np.bincount(ids[live], minlength=len(local)), want_n)
        for v in local:
            slots = h.vid_slots(int(v))
            assert len(slots) == want_n[v], (s, v, slots)
            for l, p in slots:
                assert ids[off[l] + p] == v, (s, v, l, p)
        cnt = live & np.isin(ids, [v // S for v in counted if v % S == s])
        want = np.bincount(lst[~live], minlength=NLIST) + np.bincount(lst[cnt], minlength=NLIST)
        assert np.array_equal(h.dead_counts(), want), s
        if h is not idx:
            h.close()


@pytest.mark.parametrize("kind", UNSPILLED)
def test_unspilled_one_slot_per_vid(tmp_path, kind):
    db = rows(kind, N, 1)
    idx = build(kind, db)
    counted, gone = set(), set()
    check(idx, counted, gone)
    pick = np.random.default_rng(3).permutation(N)
    dele, upd, upd_del = pick[:600], pick[600:900], pick[900:1000]
    idx.delete_vectors(upd_del)
    counted |= set(upd_del.tolist())
    check(idx, counted, gone)
    for v, x in zip(np.concatenate([upd, upd_del]), rows(kind, 400, 9)):  # tombstoned: the tombstone takes the count
        idx.update_vector(int(v), x)
    counted -= set(upd_del.tolist())
    check(idx, counted, gone)
    idx.delete_vectors(dele)
    idx.delete_vectors(dele[:50])  # counted once
    idx.delete_vectors(np.array([-1, N, N + 1000], np.int64))  # no such vid
    counted |= set(dele.tolist())
    check(idx, counted, gone)
    # the tombstones go; the deleted rows stay, counted again in the lists they moved within
    assert idx.purge(0.0) == 400
    check(idx, counted, gone)
    assert idx.purge(0.0, P.bitmap_of(dele, N)) == len(dele)
    gone |= set(dele.tolist())
    counted -= set(dele.tolist())
    check(idx, counted, gone)
    idx.delete_vectors(dele[:10])  # in no list: nothing counted
    check(idx, counted, gone)
    idx.update_vector(int(upd[0]), rows(kind, 1, 10)[0])  # one tombstone
    check(idx, counted, gone)

    idx.dump(tmp_path, "emb.000")
    again = fresh(kind)
    again.add_vectors(idx.get_vectors(0, N))
    assert again.load(tmp_path, "emb.000") > 0
    check(again, set(), gone)  # the file's tombstones counted dead, no deletion counted
    if kind != "GPU_IVFFLAT":
        for v in range(N):
            assert again.vid_slots(v) == idx.vid_slots(v), v
    more = pick[1000:1100]
    again.delete_vectors(more)
    check(again, set(more.tolist()), gone)
    assert again.purge(0.0, P.bitmap_of(np.concatenate([dele, more]), N)) == len(more) + 1
    check(again, set(), gone | set(more.tolist()))
    again.close()

    if kind in ("IVFPQFastScan", "BINARYIVF"):  # a refused file leaves the index untrained and without slots
        name = sf.qf.FILE[kind]
        (tmp_path / "half" / "emb.000").mkdir(parents=True)
        (tmp_path / "half" / "emb.000" / name).write_bytes((tmp_path / "emb.000" / name).read_bytes()[:-2])
        cut = fresh(kind)
        cut.add_vectors(db)
        with pytest.raises(gi().GammaError):
            cut.load(tmp_path / "half", "emb.000")
        assert not cut.is_trained and all(cut.vid_slots(v) == [] for v in range(0, N, 97))
        cut.close()
    idx.close()


@pytest.mark.parametrize("kind", ["IVFPQFastScan", "IVFRABITQ", "VEARCH"])
def test_spilled_slots_survive_dump_and_load(tmp_path, kind):
    idx, db = built_spilled(kind, sf.qf.METRIC_L2)
    n = len(db)
    for v, x in zip(range(30), rows(kind, 30, 5)):
        idx.update_vector(v, x)
    dead = np.arange(100, 160)
    idx.delete_vectors(dead)
    assert idx.purge(0.0, P.bitmap_of(dead, n)) == 2 * 30 + 2 * len(dead)
    idx.update_vector(200, rows(kind, 1, 6)[0])  # two tombstones in the file
    idx.dump(tmp_path, "s.000")
    again = make_spilled(kind, sf.qf.METRIC_L2)
    again.add_vectors(idx.get_vectors(0, n))
    assert again.load(tmp_path, "s.000") == n
    for v in range(n):
        a, b = idx.vid_slots(v), again.vid_slots(v)
        assert set(a) == set(b) and len(b) == (0 if 100 <= v < 160 else 2), (v, a, b)
    idx.close()
    again.close()


def test_spilled_load_refuses_a_third_entry_and_two_in_one_list(tmp_path):
    kind, metric = "IVFPQFastScan", sf.qf.METRIC_L2
    idx, db = built_spilled(kind, metric)
    idx.dump(tmp_path, "s.000")
    buf = (tmp_path / "s.000" / sf.FILE[kind]).read_bytes()
    f = sf.read_spilled(buf, kind, dict(table_of(kind, idx, metric), soar_lambda=LAM, reordering=False))
    off = f["list_off"]

    def write(ids):
        return sf.write_spilled(kind, f["d"], metric, f["nprobe"], f["centroids"], off, f["codes"], ids,
                                f["indexed_count"], f["code_size"], LAM, pq_centroids=f["pq_centroids"])

    assert write(f["ids"]) == buf
    v = 7
    a, b = sorted(idx.vid_slots(v))

    def another(l):  # the position in list l of a live entry of a vid other than v
        return next(p for p in range(off[l + 1] - off[l]) if f["ids"][off[l] + p] >= 0 and f["ids"][off[l] + p] != v)

    third = f["ids"].copy()
    c = next(l for l in range(idx.nlist) if l not in (a[0], b[0]) and off[l + 1] > off[l])
    third[off[c] + another(c)] = v
    twice = f["ids"].copy()  # in the first of its lists: met twice there before its other list
    twice[off[a[0]] + another(a[0])] = v
    for name, ids, msg in (("third", third, "more than two live entries"), ("twice", twice, "two live entries in list")):
        d = tmp_path / name / "s.000"
        d.mkdir(parents=True)
        (d / sf.FILE[kind]).write_bytes(write(ids))
        ix = make_spilled(kind, metric)
        ix.add_vectors(db)
        with pytest.raises(gi().GammaError, match=msg):
            ix.load(tmp_path / name, "s.000")
        assert not ix.is_trained and all(ix.vid_slots(u) == [] for u in range(0, len(db), 97))
        ix.train()
        ix.add_pending()
        assert all(len(ix.vid_slots(u)) == 2 for u in range(0, len(db), 97))
        ix.close()
    idx.close()
