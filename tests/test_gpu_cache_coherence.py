"""The caches the IVF indexes keep beside their lists, held to the lists after every mutation.  One scripted sequence per
index type -- train and add, appends that fit the tensor-core mirror's reserve and one that outgrows it, updates (twice
the same row, and a deleted row), deletes, purges with and without the deletion bitmap, appends back to the old lengths,
compaction, new centroids, a new PQ codebook, Dump and Load, and for a sharded index a refused Load followed by a Load of
other rows at the same lengths -- and after every step:
  * wherever the index calls a cache current, the live cache equals one rebuilt from scratch, byte for byte: the IVF-Flat
    mirror tiles and norms (gb_debug_mirror / gb_debug_mirror_rebuilt), the IVF-PQ |r_e|^2 segments (gb_debug_pq_norms);
  * the IVF-PQ caches equal their fp32 restatement (cache_reference.py), the host-store row pointers point at the list row
    of their vid, equal to its raw-store row, and the int8 shadow rows follow the raw rows;
  * the mirror is rebuilt exactly when it must be (mirror_builds);
  * a list-major and a query-major batch, with deletion and filter bitmaps and a score window, give the oracle's keys.
A cache that is not current must not be served: every step that searches checks afterwards that the list-major scan
ran and left every cache current."""
import os

import numpy as np
import pytest

import cache_reference as CR
import gamma_index_file as gif
import rerank_reference as RR
from oracle import oracle as orc
from oracle_purge import purge as P
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = 1, 0
NLIST, NPROBE, K, KK = 16, 8, 10, 50
NQ_LM, NQ_QM = 128, 6  # 128 queries x 8 probes: 64 (query, probe) pairs per list, the list-major paths; 6: query-major
N0 = 20000             # ~1250 rows per list: every list's mirror reserve (1/8 more rows) holds the 129-row append


def gi():
    from vearch_b200 import index
    return index


def metric_name(metric):
    return "L2" if metric == L2 else "InnerProduct"


# ---- comparisons ------------------------------------------------------------------------------------------------------
def assert_keys(got, want, what):
    """(score, id) rows equal: scores bit for bit, ids as sets among equal scores (the last score's group may be cut
    differently by k)"""
    (gd, gid), (wd, wid) = got, want
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), f"{what}: scores differ"
    for q in range(len(gd)):
        inner = gd[q] != gd[q][-1]
        a = sorted(zip(gd[q][inner].tolist(), gid[q][inner].tolist()))
        b = sorted(zip(wd[q][inner].tolist(), wid[q][inner].tolist()))
        assert a == b, f"{what}: query {q} ids differ"


def bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


class Case:
    """One index under the sequence: its rows (by global vid), deleted vids, queries and the checks of its type"""

    def __init__(self, kind, metric=L2, store_type=None, seed=1):
        self.kind, self.metric, self.store_type = kind, metric, store_type
        self.sharded = kind == "GPU_IVFFLAT"
        self.flat = kind in ("IVFFLAT", "GPU_IVFFLAT")
        self.pq = kind in ("IVFPQ", "IVFPQ_OPQ")
        self.d = 128 if self.pq else 32
        self.rng = np.random.default_rng(seed)
        self.db = synth.sift_like(N0, self.d, seed=seed)
        self.xq = synth.sift_like(NQ_LM, self.d, seed=seed + 1)
        self.deleted = set()
        self.idx = self.make()
        self.idx.add_vectors(self.db)
        self.idx.train()
        self.idx.add_pending()
        self.builds = self.mirror_builds()

    def params(self):
        p = {"ncentroids": NLIST, "nprobe": NPROBE, "metric_type": metric_name(self.metric), "training_threshold": 4000}
        if self.pq:
            p["nsubvector"] = 16
        if self.kind == "IVFPQ_OPQ":
            p["opq"] = {"nsubvector": 16}
        if self.kind == "IVFPQFastScan":
            p.update(nsubvector=16, soar_lambda=1.0)
        if self.kind == "IVFRABITQ":
            p.update(nb_bits=4, qb=4, soar_lambda=1.0)
        return p

    def make(self):
        g = gi()
        if self.kind == "IVFRABITQ":
            return g.RaBitQIndex(self.d, self.params(), store_type=self.store_type)
        typ = "IVFPQ" if self.pq else self.kind
        return g.GammaIndex(typ, self.d, self.params(), store_type=self.store_type,
                            devices=[0, 0] if self.sharded else None)

    def parts(self, idx=None):
        idx = idx or self.idx
        return [idx.shard(s) for s in range(idx.shard_count)] if self.sharded else [idx]

    def mirror_builds(self, idx=None):
        return [p.mirror_builds for p in self.parts(idx)] if self.flat else []

    def lens(self, idx=None):
        return [[p.list_len(l) for l in range(NLIST)] for p in self.parts(idx)]

    # ---- mutations ----------------------------------------------------------------------------------------------------
    def append(self, x):
        self.db = np.concatenate([self.db, x])
        self.idx.add(x)

    def rows_of_list(self, l, n):
        """n copies of rows that list l already holds (a copy goes to the list its original is in)"""
        vids = [v for v in self.list_vids(l) if v not in self.deleted]
        return self.db[np.resize(np.array(vids), n)]

    def list_vids(self, l):
        out = []
        for s, p in enumerate(self.parts()):
            _, ids = p.get_list(l)
            ids = ids[ids >= 0]
            out += (ids * len(self.parts()) + s).tolist() if self.sharded else ids.tolist()
        return sorted(out)

    def bitmap(self):
        return P.bitmap_of(sorted(self.deleted), len(self.db)) if self.deleted else None

    # ---- checks -------------------------------------------------------------------------------------------------------
    def check(self, what, search=True, rebuild=None, idx=None):
        """rebuild: per part, whether the step must have made the next list-major search rebuild the mirror"""
        idx = idx or self.idx
        self.check_caches(what + " (before searching)", idx)
        if search:
            self.check_search(what, idx)
            self.check_caches(what, idx, after_search=True)
            if self.flat:
                now = self.mirror_builds(idx)
                if rebuild is not None:
                    want = [b + int(r) for b, r in zip(self.builds, rebuild)]
                    assert now == want, f"{what}: mirror builds {now}, expected {want}"
                self.builds = now

    def check_caches(self, what, idx, after_search=False):
        for s, part in enumerate(self.parts(idx)):
            where = f"{what}, part {s}"
            if self.flat:
                self.check_mirror(part, where, after_search)
                if self.store_type or self.sharded:
                    self.check_rowptrs(part, s, where, idx)
            if self.pq:
                self.check_pq(part, where, after_search)
            if self.kind in ("IVFPQFastScan", "IVFRABITQ"):
                self.check_slots(part, where)
        if self.kind in ("IVFPQFastScan", "IVFRABITQ"):
            err = RR.shadow_mismatch(RR.pad4(self.db), *idx.debug_shadow_rows(0, len(self.db)))
            assert err is None, f"{what}: shadow rows: {err}"

    def check_mirror(self, part, where, after_search):
        for l in range(NLIST):
            live = part.debug_mirror(l)
            if live["disabled"]:
                pytest.fail(f"{where}: the tensor-core mirror is disabled (HBM too full), nothing was checked")
            if after_search:
                assert live["current"], f"{where}: list {l}'s mirror is not current after a list-major search"
            if not live["current"]:
                continue
            reb = part.debug_mirror_rebuilt(l)
            assert len(live["tiles"]) == (part.list_len(l) + 127) // 128, f"{where}: list {l} tiles"
            assert bits_equal(live["tiles"], reb["tiles"]), f"{where}: list {l}'s live mirror tiles differ from a rebuild"
            assert bits_equal(live["norms"], reb["norms"]), f"{where}: list {l}'s live mirror norms differ from a rebuild"

    def check_rowptrs(self, part, s, where, idx):
        S = len(self.parts(idx))
        lists = [part.get_list(l) for l in range(NLIST)]
        top = max([int(i.max()) + 1 for _, i in lists if len(i)], default=0)
        got, st = part.debug_rowptr_rows(0, top)
        for codes, ids in lists:
            keep = ids >= 0
            vids, rows = ids[keep], codes[keep].view(np.float32)[:, :self.d]
            bad = np.nonzero(st[vids] != gi().GammaIndex.ROW_LIVE)[0]
            assert not len(bad), f"{where}: vid {vids[bad[0]]}'s row pointer is {st[vids[bad[0]]]}, not a list row"
            assert bits_equal(got[vids], rows), f"{where}: a row pointer is not its vid's list row"
            gv = vids * S + s if self.sharded else vids
            assert bits_equal(rows, self.db[gv]), f"{where}: a list row is not its vid's raw row"

    def check_pq(self, part, where, after_search):
        cb8, nrm = part.debug_pq_tables()
        w8, wn = CR.pq_tables(part.get_pq_centroids())
        assert np.array_equal(cb8, w8), f"{where}: int8 codebook differs from its restatement"
        assert bits_equal(nrm[:-1], wn), f"{where}: |pq|^2, R^2, sb, D differ from their restatement"
        T = orc.ivfpq_precompute_table(part.get_centroids(), part.get_pq_centroids())
        assert bits_equal(part.get_precomputed_table(), T), f"{where}: the precomputed table does not follow the centroids"
        M = part.pq_m
        for l in range(NLIST):
            live, rec, cur = part.debug_pq_norms(l)
            if after_search:
                assert cur, f"{where}: list {l}'s |r_e|^2 cache is not current after a list-major search"
            codes, _ = part.get_list(l)
            assert bits_equal(rec, CR.entry_norms(codes, wn, M)), f"{where}: list {l}'s |r_e|^2 differs from its restatement"
            if cur:
                assert bits_equal(live, rec), f"{where}: list {l}'s cached |r_e|^2 differs from a recomputation"

    def check_slots(self, part, where):
        slots = {}
        for l in range(NLIST):
            _, ids = part.get_list(l)
            for pos, v in enumerate(ids.tolist()):
                if v >= 0:
                    slots.setdefault(v, []).append((l, pos))
        for v in self.rng.choice(len(self.db), 200, replace=False).tolist():
            assert sorted(part.vid_slots(v)) == sorted(slots.get(v, [])), f"{where}: vid {v}'s slots"
            assert len(slots.get(v, [])) in (0, 2), f"{where}: vid {v} has {len(slots.get(v, []))} live entries"

    def windowed(self, want_fn):
        """deletion and filter bitmaps over every vid, and a score window that cuts both ends of the results"""
        n = len(self.db)
        fb = P.bitmap_of(np.nonzero(np.random.default_rng(n).random(n) < 0.8)[0], n)
        db_ = self.bitmap()
        if db_ is None:
            db_ = np.zeros_like(fb)
        d0, _ = want_fn(db_, fb, -np.finfo(np.float32).max, np.finfo(np.float32).max)
        lo, hi = sorted((float(np.percentile(d0[:, 0], 30)), float(np.percentile(d0[:, -1], 70))))
        return db_, fb, lo, hi

    def global_lists(self, idx):
        """every list's entries over all parts, as global vids: (off, vecs or codes, ids)"""
        S = len(self.parts(idx))
        cs, ids, lens = [], [], []
        for l in range(NLIST):
            n = 0
            for s, p in enumerate(self.parts(idx)):
                c, i = p.get_list(l)
                cs.append(c)
                ids.append(np.where(i >= 0, i * S + s, i) if self.sharded else i)
                n += len(i)
            lens.append(n)
        off = np.zeros(NLIST + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        return off, np.concatenate(cs), np.concatenate(ids)

    def check_search(self, what, idx):
        xq = self.xq
        part0 = self.parts(idx)[0]
        cd, keys = part0.coarse_search(xq, NPROBE)
        off, codes, ids = self.global_lists(idx)
        if self.flat:
            vecs = codes.view(np.float32)[:, :self.d]

            def want(db_, fb, lo, hi, rows=slice(None)):
                return orc.ivfflat_search_preassigned(off, vecs, ids, xq[rows], K, keys[rows], self.metric, db_, fb, lo, hi)
            db_, fb, lo, hi = self.windowed(want)
            for rows, lm in ((slice(None), True), (slice(0, NQ_QM), False)):
                got = idx.search(xq[rows], K, del_bitmap=db_, filter_bitmap=fb, min_score=lo, max_score=hi)
                assert idx.last_scan_kernel.startswith("ivf_listmajor") == lm, f"{what}: {idx.last_scan_kernel}"
                assert_keys(got, want(db_, fb, lo, hi, rows), f"{what}, {'list' if lm else 'query'}-major")
        elif self.pq:
            cent, pqc, T = idx.get_centroids(), idx.get_pq_centroids(), idx.get_precomputed_table()
            xr = idx.apply_opq(xq) if self.kind == "IVFPQ_OPQ" else xq

            def want(db_, fb, lo, hi, rows=slice(None)):
                return orc.ivfpq_search_preassigned(off, codes, ids, cent, pqc, T, xr[rows], KK, keys[rows], cd[rows],
                                                    self.metric, del_bitmap=db_, filter_bitmap=fb, min_score=lo,
                                                    max_score=hi)
            db_, fb, lo, hi = self.windowed(want)
            for rows, kern in ((slice(None), "pqtc_scan_kernel"), (slice(0, NQ_QM), "ivfpq_scan_kernel")):
                got = idx.search_preassigned(xq[rows], KK, keys[rows], cd[rows], del_bitmap=db_, filter_bitmap=fb,
                                             min_score=lo, max_score=hi)
                assert idx.last_scan_kernel == kern, f"{what}: {idx.last_scan_kernel}"
                assert_keys(got, want(db_, fb, lo, hi, rows), f"{what}, {kern}")
        else:  # estimating codecs: the exact re-rank of the estimated candidates
            db_ = self.bitmap()
            n = len(self.db)
            fb = P.bitmap_of(np.nonzero(np.random.default_rng(n).random(n) < 0.8)[0], n)
            dis, vid = idx.search(xq, K, params={"recall_num": 100}, del_bitmap=db_, filter_bitmap=fb)
            ok = vid >= 0
            assert ok[:, 0].all(), what
            v = vid[ok]
            assert not np.isin(v, sorted(self.deleted)).any(), f"{what}: a deleted vid was returned"
            assert ((fb[v >> 3] >> (v & 7)) & 1).all(), f"{what}: a filtered-out vid was returned"
            ex = ((xq[np.nonzero(ok)[0]].astype(np.float64) - self.db[v]) ** 2).sum(1) if self.metric == L2 else None
            assert np.allclose(dis[ok], ex, rtol=1e-5), f"{what}: re-ranked scores are not the exact distances"


# ---- the sequence -----------------------------------------------------------------------------------------------------
def run_sequence(c, tmp_path):
    S = len(c.parts())
    all_, none = [True] * S, [False] * S
    c.check("1 build", rebuild=all_ if c.flat else None)
    # 2: appends inside every list's reserve: 1, 127, 128 and 129 rows into one list each.  A build reserves
    # ceil(9 len / 8 / 128) tiles per list (len + len / 8 rows, whole tiles); a shard takes every S-th new row.
    at_build, used = c.lens(), set()
    room = lambda l: min((-(-(n + n // 8) // 128)) * 128 - n for n in (p[l] for p in at_build))  # noqa: E731
    for n in (1, 127, 128, 129):
        l = max((j for j in range(NLIST) if j not in used), key=room)
        assert room(l) >= -(-n // S), f"fixture: no list has room for {n} rows"
        used.add(l)
        c.append(c.rows_of_list(l, n))
        c.check(f"2 append {n} rows to list {l}", rebuild=none)
    # 3: a list outgrows its reserved tiles
    c.append(c.rows_of_list(0, 1000))
    c.check("3 outgrow list 0", rebuild=all_)
    # 4: update a row, the same row again, then a deleted row
    v1, v2 = 11, 12
    c.idx.update_vector(v1, c.db[100])
    c.db[v1] = c.db[100]
    c.check("4a update", rebuild=none)
    c.idx.update_vector(v1, c.db[200])
    c.db[v1] = c.db[200]
    c.check("4b update the same row", rebuild=none)
    c.idx.delete_vectors([v2])
    c.deleted.add(v2)
    c.idx.update_vector(v2, c.db[300])  # the document stays deleted: its new entry is hidden by the bitmap
    c.db[v2] = c.db[300]
    c.check("4c update a deleted row", rebuild=none)
    # 5: delete a tenth of the rows
    gone = c.rng.choice(len(c.db), len(c.db) // 10, replace=False)
    c.idx.delete_vectors(gone)
    c.deleted.update(gone.tolist())
    c.check("5 delete", rebuild=none)
    # 6: purge without the bitmap (the updates' tombstones), then with it (the deleted entries)
    before = c.lens()
    assert c.idx.purge(0.0) > 0
    c.check("6a purge without the bitmap", rebuild=[b != a for b, a in zip(before, c.lens())])
    old = [sum(p[l] for p in c.lens()) for l in range(NLIST)]
    assert c.idx.purge(0.0, c.bitmap()) > 0
    c.check("6b purge with the bitmap", search=False)
    # 7: back to the old lengths with other rows; no search in between
    for l in range(NLIST):
        short = old[l] - sum(p[l] for p in c.lens())
        if short > 0:
            c.append(c.rows_of_list(l, short))
    if c.flat and not c.sharded or c.pq:  # a spilled row's copy goes to its primary list only
        assert [c.idx.list_len(l) for l in range(NLIST)] == old
    c.check("7 append back to the old lengths", rebuild=all_)
    # 8: compaction moves every list, the mirror stays valid
    c.idx.compact()
    c.check("8 compact", rebuild=none)
    if not c.sharded:
        # 9: new centroids (the lists keep their entries; under L2 the mirror's shifts change)
        c.idx.set_centroids(c.idx.get_centroids() + np.float32(0.5))
        c.check("9 set_centroids", rebuild=[c.metric == L2] if c.flat else None)
    if c.pq:
        # 10: a new codebook: the tables and every |r_e|^2 change
        c.idx.set_pq_centroids(c.idx.get_pq_centroids() * np.float32(1.03125))
        c.check("10 set_pq_centroids")
    # 11: Dump, then Load into a fresh index
    c.idx.dump(str(tmp_path / "a"), "f")
    fresh = c.make()
    fresh.add_vectors(c.db)
    assert fresh.load(str(tmp_path / "a"), "f") > 0
    c.builds = c.mirror_builds(fresh)
    assert not any(c.builds), "a fresh index has no mirror before its first list-major search"
    c.check("11 load into a fresh index", rebuild=all_ if c.flat else None, idx=fresh)
    if c.sharded:
        step12(c, fresh, tmp_path)
    fresh.close()


def step12(c, idx, tmp_path):
    """A refused Load empties every shard's lists (clear_lists); a Load of other rows at the same list lengths must not
    find the old mirror current"""
    fname = "ivfflat.index"
    src = tmp_path / "a" / "f" / fname
    os.makedirs(tmp_path / "t" / "f")
    with open(src, "rb") as fh:
        buf = fh.read()
    with open(tmp_path / "t" / "f" / fname, "wb") as fh:
        fh.write(buf[: len(buf) // 2])
    with pytest.raises(gi().GammaError):
        idx.load(str(tmp_path / "t"), "f")
    assert all(n == 0 for p in c.lens(idx) for n in p)
    c.check("12a refused load", search=False, idx=idx)
    # the same file with every list row moved by one: same lengths, same ids, other rows
    ref = gi().GammaIndex(c.kind, c.d, c.params())
    ref.add_vectors(c.db)
    assert ref.load(str(tmp_path / "a"), "f") > 0
    off, codes, ids = ref.export_lists()
    vecs = codes.view(np.float32)[:, :c.d] + np.float32(1)
    os.makedirs(tmp_path / "b" / "f")
    with open(tmp_path / "b" / "f" / fname, "wb") as fh:
        fh.write(gif.write_ivfflat(c.d, gif.METRIC_L2 if c.metric == L2 else gif.METRIC_IP, NPROBE, ref.get_centroids(),
                                   off, vecs, ids, ref.indexed_count))
    ref.close()
    assert idx.load(str(tmp_path / "b"), "f") > 0
    assert [sum(p[l] for p in c.lens(idx)) for l in range(NLIST)] == np.diff(off).tolist()
    c.db = c.db.copy()
    c.db[ids[ids >= 0]] = vecs[ids >= 0]  # the list rows the index now scores (the raw store keeps the old rows)
    c.check("12b load other rows at the same lengths", rebuild=[True] * len(c.parts(idx)), idx=idx)


CASES = [
    ("IVFFLAT", L2, None), ("IVFFLAT", IP, None), ("IVFFLAT", L2, "RocksDB"), ("IVFFLAT", IP, "RocksDB"),
    ("GPU_IVFFLAT", L2, None), ("GPU_IVFFLAT", IP, None),
    ("IVFPQ", L2, None), ("IVFPQ_OPQ", L2, None),
    ("IVFPQFastScan", L2, None), ("IVFRABITQ", L2, None),
]


@pytest.mark.parametrize("kind,metric,store_type", CASES,
                         ids=[f"{k}-{metric_name(m)}-{s or 'HBM'}" for k, m, s in CASES])
def test_caches_follow_every_mutation(tmp_path, kind, metric, store_type):
    c = Case(kind, metric, store_type)
    try:
        run_sequence(c, tmp_path)
    finally:
        c.idx.close()
