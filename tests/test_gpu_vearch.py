"""VEARCH on the H100 through the C-ABI and the engine: list codes byte-equal to the numpy twin (oracle_scann) under IP at
several noise-shaping thresholds and under L2, remainder blocks included; tables, multipliers and scan scores bit-equal;
searched keys exact against tests/topk_reference.py over the twin's scores (ties, tombstones, bitmaps, score windows);
reordering equal to the exact re-score on both placements; parameter rules; the engine flow; recall."""
import numpy as np
import pytest

import topk_reference as tr
from oracle_scann import ah
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = tr.METRIC_L2, tr.METRIC_IP
MNAME = {L2: "L2", IP: "InnerProduct"}
F32 = np.float32


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mips_rows(n, d, seed):
    """rows of varied norm (maximum inner product search data)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)) / np.sqrt(d)
    return (x * rng.uniform(0.3, 1.5, (n, 1))).astype(F32)


def unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(F32)


def make(d, nsub, metric, nlist, cent, cb, t=0.2, **extra):
    idx = gi().VearchIndex(d, {"ncentroids": nlist, "nsubvector": nsub, "ns_threshold": t,
                               "metric_type": MNAME[metric], **extra})
    idx.set_codebook(cb)
    idx.set_centroids(cent)
    return idx


def codebook(d, seed, scale=0.3):
    return (np.random.default_rng(seed).standard_normal(16 * d) * scale).astype(F32)


def lists_of(idx):
    codes, lid, raw = [], [], []
    for l in range(idx.nlist):
        c, i = idx.get_list(l)
        codes.append(c)
        lid.append(np.full(len(i), l, np.int64))
        raw.append(i)
    return codes, np.concatenate(lid), np.concatenate(raw)


def twin_scores(idx, cent, cb, xq, d, nsub, metric):
    """[nq, N] twin score of every list entry (lists in order) for every query"""
    codes, _, _ = lists_of(idx)
    rows = []
    for q in xq:
        tab, m = ah.lut(q, cb, d, nsub, metric)
        rows.append(np.concatenate([ah.scores(codes[l], tab, m, metric, ah.leaf(q, cent[l]) if metric == IP else F32(0))
                                    if len(codes[l]) else np.zeros(0, F32) for l in range(idx.nlist)]))
    return np.stack(rows)


def got_keys(dis, ids, metric):
    return np.sort(tr.keys(dis, np.where(ids >= 0, ids, 0), ids >= 0, metric), axis=1)


SHAPES = [(32, 8), (30, 8), (128, 64), (96, 40), (20, 20)]  # (30, 8) and (96, 40) have a remainder block


@pytest.mark.parametrize("d,nsub", SHAPES)
@pytest.mark.parametrize("metric,t", [(IP, 0.2), (IP, 0.6), (IP, 0.0), (IP, -1.0), (L2, 0.2)])
def test_codes_byte_equal_to_the_twin(d, nsub, metric, t):
    n = 300
    x = mips_rows(n, d, d + nsub)
    x[7] = 0  # a zero row keeps its minimum-residual-norm code
    x[11, d // 2] = np.nan  # a NaN coordinate: NaN norms in its block, NaN costs, no move
    cent = unit(np.random.default_rng(3).standard_normal((4, d)))
    cb = codebook(d, d)
    idx = make(d, nsub, metric, 4, cent, cb, t)
    assert idx.blocks == len(ah.blocks(d, nsub)) and idx.code_size == ah.code_bytes(d, nsub)
    assign = np.arange(n) % 4
    got = idx.encode(x, assign)
    want = ah.encode(x, cb, d, nsub, metric, t, cent, assign)
    assert np.array_equal(got, want)
    if metric == IP and t > 0:  # the anisotropic codes differ from the plain ones on these rows
        assert not np.array_equal(want, ah.encode(x, cb, d, nsub, metric, -1.0, cent, assign))


@pytest.mark.parametrize("d,nsub", SHAPES)
@pytest.mark.parametrize("metric", [IP, L2])
def test_tables_multipliers_and_scan_scores_bit_equal(d, nsub, metric):
    n, nlist = 800, 4
    db = mips_rows(n, d, 7 * d)
    cent = unit(db[:nlist].copy()) if metric == IP else db[:nlist].copy()
    cb = codebook(d, d + 1)
    idx = make(d, nsub, metric, nlist, cent, cb)
    idx.add(db)
    xq = mips_rows(5, d, 99)
    xq[4] = 0  # an all-zero table: the multiplier's sqrt(FLT_EPSILON) floor
    lut, mult = idx.lut(xq)
    for j, q in enumerate(xq):
        tab, m = ah.lut(q, cb, d, nsub, metric)
        assert np.array_equal(lut[j], tab) and mult[j].view(np.uint32) == m.view(np.uint32)
    codes, lid, raw = lists_of(idx)
    for l in range(nlist):
        assert np.array_equal(codes[l], ah.encode(db[raw[lid == l]], cb, d, nsub, metric, 0.2, cent, np.full(len(codes[l]), l)))
    scores = twin_scores(idx, cent, cb, xq, d, nsub, metric)
    probes = np.tile(np.arange(nlist), (len(xq), 1))
    dis, ids = idx.search_preassigned(xq, n, probes, np.zeros(probes.shape, F32))
    for q in range(len(xq)):
        want = dict(zip(raw.tolist(), scores[q].tolist()))
        assert sorted(ids[q].tolist()) == sorted(want)
        assert np.array_equal(dis[q].view(np.uint32), np.array([want[v] for v in ids[q]], F32).view(np.uint32))


@pytest.mark.parametrize("metric", [IP, L2])
def test_rows_deleted_before_indexing_are_not_encoded(metric):
    """rows deleted before add_pending reach the encoder with list -1: they get no entry, and every other row's entry is
    the twin's code"""
    d, nsub, nlist, n = 32, 8, 4, 600
    db = mips_rows(n, d, 91)
    cent = unit(db[:nlist].copy())
    cb = codebook(d, 92)
    idx = make(d, nsub, metric, nlist, cent, cb)
    idx.add_vectors(db)
    deleted = np.random.default_rng(93).random(n) < 0.3
    idx.add_pending(np.packbits(deleted, bitorder="little"))
    codes, lid, raw = lists_of(idx)
    assert sorted(raw.tolist()) == np.flatnonzero(~deleted).tolist()
    for l in range(nlist):
        rows = raw[lid == l]
        assert np.array_equal(codes[l], ah.encode(db[rows], cb, d, nsub, metric, 0.2, cent, np.full(len(rows), l)))


def tied_rows(n, d, seed):
    base = mips_rows(n // 4, d, seed)
    return np.concatenate([base, base, base[: n // 4], base[: n - 3 * (n // 4)]])


@pytest.mark.parametrize("metric", [IP, L2])
@pytest.mark.parametrize("k", [1, 17, 400, 4096])
def test_topk_key_exact_under_ties_tombstones_bitmaps_and_windows(metric, k):
    d, nsub, nlist = 64, 32, 12
    db = tied_rows(12000, d, k)
    cent = unit(db[np.random.default_rng(k).choice(len(db), nlist, replace=False)])
    cb = codebook(d, 5)
    idx = make(d, nsub, metric, nlist, cent, cb)
    idx.add(db)
    for l in range(0, nlist, 3):
        if idx.list_len(l) > 2:
            idx.tombstone(l, 1)
    rng = np.random.default_rng(9)
    dele = np.packbits(rng.random(len(db)) < 0.2, bitorder="little")
    filt = np.packbits(rng.random(len(db)) < 0.7, bitorder="little")
    xq = mips_rows(6, d, k + 5)
    _, probes = idx.coarse_search(xq, 8)
    cd = np.zeros(probes.shape, F32)
    scores = twin_scores(idx, cent, cb, xq, d, nsub, metric)
    _, lid, raw = lists_of(idx)
    dis, ids = idx.search_preassigned(xq, k, probes, cd)
    assert np.array_equal(got_keys(dis, ids, metric), tr.search_entries(scores, lid, raw, probes, k, metric))
    lo, hi = float(np.percentile(scores, 10)), float(np.percentile(scores, 60))
    dis, ids = idx.search_preassigned(xq, k, probes, cd, del_bitmap=dele, filter_bitmap=filt, min_score=lo, max_score=hi)
    want = tr.search_entries(scores, lid, raw, probes, k, metric, del_bitmap=dele, filter_bitmap=filt, min_score=lo,
                             max_score=hi)
    assert np.array_equal(got_keys(dis, ids, metric), want)
    assert idx.last_scan_kernel == "vearch_scan_kernel"


@pytest.mark.parametrize("metric", [IP, L2])
def test_reordering_equals_the_exact_rescore_on_both_placements(metric):
    d, nlist, n = 64, 8, 4000
    db = np.random.default_rng(17).integers(-6, 7, (n, d)).astype(F32)
    xq = np.random.default_rng(18).integers(-6, 7, (5, d)).astype(F32)
    flat = gi().GammaIndex("FLAT", d, {"metric_type": MNAME[metric]})
    flat.add(db)
    fd, fi = flat.search(xq, n)
    got = {}
    for store in ("MemoryOnly", "RocksDB"):
        idx = gi().VearchIndex(d, {"ncentroids": nlist, "nsubvector": 16, "metric_type": MNAME[metric], "reordering": True,
                                   "training_threshold": 3000}, store_type=store)
        idx.add_vectors(db)
        idx.train()
        idx.add_pending()
        k = 10
        dis, ids = idx.search(xq, k, params={"nprobe": nlist, "recall_num": 300})
        for q in range(len(xq)):
            pos = {int(v): j for j, v in enumerate(fi[q])}
            assert np.array_equal(dis[q], np.array([fd[q][pos[int(v)]] for v in ids[q]], F32))
        # k' = max(k, recall_num): the exact re-rank of the 300 best codes, key-exact
        cb, cent = idx.get_codebook(), idx.get_centroids()
        scores = twin_scores(idx, cent, cb, xq, d, 16, metric)
        _, lid, raw = lists_of(idx)
        probes = np.tile(np.arange(nlist), (len(xq), 1))
        cand = tr.search_entries(scores, lid, raw, probes, 300, metric)
        want = tr.rerank_keys(cand, xq, db, k, metric)
        assert np.array_equal(got_keys(dis, ids, metric), want)
        got[store] = (dis, ids)
        idx.close()
    assert np.array_equal(got["MemoryOnly"][0], got["RocksDB"][0]) and np.array_equal(got["MemoryOnly"][1], got["RocksDB"][1])


def test_parameters_defaults_and_refusals():
    V, E = gi().VearchIndex, gi().GammaError
    with pytest.raises(E, match="cannot get ncentroids for vearch, set it when create space"):
        V(32, {"nsubvector": 8})
    with pytest.raises(E, match="cannot get nsubvector for vearch, set it when create space"):
        V(32, {"ncentroids": 8})
    with pytest.raises(E, match="invalid ncentroids =-2"):
        V(32, {"ncentroids": -2, "nsubvector": 8})
    with pytest.raises(E, match="invalid nsubvector =-5"):
        V(32, {"ncentroids": 8, "nsubvector": -5})
    with pytest.raises(E, match="invalid metric_type = cosine"):
        V(32, {"ncentroids": 8, "nsubvector": 8, "metric_type": "cosine"})
    with pytest.raises(E, match=r"nsubvector \[40\] above the dimension \[32\] is not supported by this engine"):
        V(32, {"ncentroids": 8, "nsubvector": 40})
    with pytest.raises(E, match="301 blocks .* above 256 is not supported by this engine"):
        V(601, {"ncentroids": 8, "nsubvector": 300})
    idx = V(128, {"ncentroids": 0, "nsubvector": -1, "thread_num": 4})
    assert idx.nlist == 2048 and idx.nsub == 64 and idx.blocks == 64 and idx.code_size == 32
    assert idx.training_threshold == 2048 * 256
    idx = V(100, {"ncentroids": 8, "nsubvector": 256 // 4, "metric_type": "l2"})
    assert idx.blocks == 65 and idx.code_size == 33  # 64 blocks of 1 dim, one of 36
    assert idx.mem_bytes(0) >= 16 * 100 * 4 + 8 * 100 * 4


def test_retrieval_defaults_nprobe_and_recall_num():
    """an empty parameter string takes VearchRetrievalParameters(type): nprobe 50, recall_num 100; a non-empty one
    VearchRetrievalParameters(): nprobe 80, recall_num 100; a request nprobe >= ncentroids gives the index's 512 leaves,
    clamped to nlist"""
    d, nlist, n = 32, 600, 12000
    db = mips_rows(n, d, 61)
    cent = unit(np.random.default_rng(62).standard_normal((nlist, d)))
    cb = codebook(d, 63)
    xq = mips_rows(8, d, 64)
    idx = make(d, 8, IP, nlist, cent, cb, reordering=True)
    idx.add(db)
    k = 200

    def same(a, b):
        return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])

    empty = idx.search(xq, k)
    assert same(empty, idx.search(xq, k, params={"nprobe": 50, "recall_num": 100}))
    assert not same(empty, idx.search(xq, k, params={"nprobe": 80}))
    assert same(idx.search(xq, k, params={"recall_num": -3}), idx.search(xq, k, params={"nprobe": 80, "recall_num": 100}))
    assert same(idx.search(xq, k, params={"nprobe": 600}), idx.search(xq, k, params={"nprobe": 512}))
    assert same(idx.search(xq, k, params={"nprobe": 10 ** 6}), idx.search(xq, k, params={"nprobe": 512}))
    small = make(d, 8, IP, 40, cent[:40], cb)
    small.add(db[:2000])
    assert same(small.search(xq, 10, params={"nprobe": 40}), small.search_preassigned(
        xq, 10, np.tile(np.arange(40), (len(xq), 1)), np.zeros((len(xq), 40), F32)))
    # the request's metric_type does not change the ranking (the codes are built for the index metric)
    assert same(idx.search(xq, k, params={"metric_type": "L2", "nprobe": 50}), empty)


def recall_at(ids, exact, k=10):
    return float(np.mean([len(set(ids[q][:k]) & set(exact[q][:k])) / k for q in range(len(ids))]))


# Floors set from the first H100 run of this test, less a margin of about 0.05.  Keys: (ns_threshold, reordering, nprobe,
# recall_num).  Measured on an H100 80GB HBM3 at 700 W on these rows (nlist 64, 32 blocks of 2 dims):
#   ns_threshold 0.2: codes alone 0.467 (every list) / 0.392 (16 lists); recall_num 100: 0.911 / 0.605; 1000: 0.998
#   ns_threshold -1:  codes alone 0.473 / 0.398;                          recall_num 100: 0.926 / 0.606; 1000: 0.999
# On these isotropic Gaussian rows the anisotropic codes do not rank better than the plain ones; no test assumes either.
RECALL_FLOORS = {}
for _t in (0.2, -1.0):
    RECALL_FLOORS.update({(_t, False, 64, 0): 0.42, (_t, False, 16, 0): 0.34, (_t, True, 64, 100): 0.86,
                          (_t, True, 16, 100): 0.55})


def test_recall_of_the_codes_the_probing_and_the_reordering():
    """recall@10 of the codes alone (every list probed, no re-rank), of the codes and the probing (16 of 64 lists), of
    the default re-rank depth (recall_num 100) and of a deep exact re-rank (recall_num 1000, every list)"""
    d, n, nlist = 64, 30000, 64
    db = mips_rows(n, d, 71)
    xq = mips_rows(200, d, 72)
    exact = np.argsort(-(xq.astype(np.float64) @ db.astype(np.float64).T), axis=1, kind="stable")[:, :10]
    got = {}
    for t in (0.2, -1.0):
        for ro in (False, True):
            idx = gi().VearchIndex(d, {"ncentroids": nlist, "nsubvector": 32, "ns_threshold": t, "reordering": ro,
                                       "training_threshold": 16384})
            idx.add_vectors(db)
            idx.train()
            idx.add_pending()
            for nprobe, rn in ((nlist, 1000), (nlist, 100), (16, 100)) if ro else ((nlist, 0), (16, 0)):
                _, ids = idx.search(xq, 10, params={"nprobe": nprobe, "recall_num": rn} if rn else {"nprobe": nprobe})
                got[(t, ro, nprobe, rn)] = recall_at(ids, exact)
            idx.close()
    print("VEARCH recall@10 (ns_threshold, reordering, nprobe, recall_num):", got)
    # the exact re-rank of 1000 candidates (3 % of the rows) from every list finds the true top 10
    assert got[(0.2, True, nlist, 1000)] >= 0.99 and got[(-1.0, True, nlist, 1000)] >= 0.99
    for key, floor in RECALL_FLOORS.items():
        assert got[key] >= floor, (key, got[key])
    for t in (0.2, -1.0):  # probing fewer lists and re-ranking fewer candidates can only lose neighbours here
        assert got[(t, False, 16, 0)] <= got[(t, False, nlist, 0)] + 0.02
        assert got[(t, True, 16, 100)] <= got[(t, True, nlist, 100)] + 0.02 <= got[(t, True, nlist, 1000)] + 0.04


def test_trained_codebooks_are_ordered_by_cluster_size():
    """train() stores each block's 16 centres by the size of their cluster in the training sample, largest first, and
    reversed in odd blocks (asymmetric_hashing_impl.cc:220-243)"""
    d, nsub, nlist, tt = 16, 4, 8, 2000
    db = synth.sift_like(3000, d, seed=81).astype(F32)
    idx = gi().VearchIndex(d, {"ncentroids": nlist, "nsubvector": nsub, "metric_type": "L2", "training_threshold": tt})
    idx.add_vectors(db)
    idx.train()
    sample = db[:tt].astype(np.float64)
    for b, ((s0, w), cents) in enumerate(zip(ah.blocks(d, nsub), ah.block_centres(idx.get_codebook(), d, nsub))):
        dist = ((sample[:, None, s0:s0 + w] - cents.astype(np.float64)[None]) ** 2).sum(-1)
        sizes = np.bincount(np.argmin(dist, axis=1), minlength=16)
        assert sizes.max() > sizes.min()
        steps = np.diff(sizes) if b & 1 else -np.diff(sizes)
        # the engine assigns in fp32: a point within rounding of two centres may land on the other one (one count)
        assert steps.min() >= -1, (b, sizes)


# ---- the engine (gamma C-ABI): a VEARCH table end to end ---------------------------------------------------------------
def eng_mod():
    from vearch_b200 import engine
    return engine


def ids_of(res):
    return [[int(it["fields"]["_id"].decode()[3:]) for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def vr_engine(path, d, params, **kw):
    from vearch_b200 import wire
    e = eng_mod().GammaEngine(str(path), space_name="vr")
    e.create_table("vr", d, "VEARCH", params, fields=(("_id", wire.DT_STRING, False),), **kw)
    return e


def test_engine_refuses_bad_parameters(tmp_path):
    E = eng_mod()
    with pytest.raises(E.GammaStatusError) as ei:
        vr_engine(tmp_path / "a", 32, {"ncentroids": 8})
    assert ei.value.code == 4 and "cannot get nsubvector for vearch" in ei.value.msg


def test_engine_flow_delete_update_dump_load(tmp_path):
    d, nlist, n = 32, 16, 3000
    db = np.random.default_rng(21).integers(-6, 7, (n, d)).astype(F32)
    xq = np.random.default_rng(22).integers(-6, 7, (4, d)).astype(F32)
    params = {"ncentroids": nlist, "nsubvector": 8, "training_threshold": 2000, "reordering": True}
    e = vr_engine(tmp_path, d, params)
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    st = e.wait_indexed(n)
    assert st["index_status"] == 2
    assert e.memory_info()["index_mem"] > 0
    exact = tr.exact_scores(xq, db.astype(np.int64), IP)
    want_d, _ = tr.decode(tr.topk(tr.keys(exact.astype(F32), np.arange(n)[None, :], metric=IP), 5), IP)
    res = e.search(xq, 5, index_params={"recall_num": n, "nprobe": nlist})  # every entry re-ranked: exact scores
    assert np.array_equal(np.array(scores_of(res), F32), want_d)
    # scores are signed inner products: the last of all documents is negative, as the exact score
    every = e.search(xq[:1], n, index_params={"recall_num": n, "nprobe": nlist})
    assert scores_of(every)[0][-1] < 0 and scores_of(every)[0][-1] == F32(exact[0].min())
    assert e.delete_doc("doc3") == 0
    assert e.get_doc_by_id("doc3")[0] == -1
    new = db[5].copy()
    assert e.add_doc("doc2999", new) == 0  # update: re-encoded into its new list
    res = e.search(new[None, :], 3, index_params={"recall_num": n, "nprobe": nlist})
    assert 2999 in ids_of(res)[0] and 3 not in ids_of(res)[0]
    queries = [dict(), dict(index_params={"nprobe": 4}), dict(index_params={"nprobe": nlist, "recall_num": 50})]
    before = [e.search(xq, 10, **q) for q in queries]
    assert e.dump() == 0
    e.close()
    e2 = vr_engine(tmp_path, d, params)
    assert e2.load() == 0
    e2.wait_indexed(n)  # nothing is dumped for the index: Load trains and fills it again
    after = [e2.search(xq, 10, **q) for q in queries]
    for a, b in zip(after, before):
        assert ids_of(a) == ids_of(b) and scores_of(a) == scores_of(b)
    assert e2.get_doc_by_id("doc3")[0] == -1
    e2.close()


def test_multi_vector_table_with_a_vearch_field(tmp_path):
    from vearch_b200 import wire
    n, d, d2, topn, nq = 2500, 32, 16, 400, 6
    db, xq = synth.sift_like(n, d, seed=51), synth.sift_like(nq, d, seed=52)
    img, imq = synth.sift_like(n, d2, seed=53), synth.sift_like(nq, d2, seed=54)
    e = eng_mod().GammaEngine(str(tmp_path), space_name="mv")
    e.create_table("mv", d, "IVFFLAT", {"ncentroids": 16, "nprobe": 16, "metric_type": "L2", "training_threshold": 2000},
                   extra_vectors=[("img", d2, "VEARCH", {"ncentroids": 16, "nsubvector": 8, "metric_type": "L2",
                                                         "reordering": True, "training_threshold": 2000})])
    for i in range(n):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("img", img[i].tobytes(), wire.DT_VECTOR)]) == 0
    assert e.wait_indexed(n)["index_status"] == 2
    res = e.search(xq, topn, extra_vec_queries=[("img", imq)], multi_vector_rank=1,
                   index_params={"nprobe": 16, "recall_num": n})
    e1 = ((xq.astype(np.float64)[:, None] - db.astype(np.float64)[None]) ** 2).sum(-1)
    e2 = ((imq.astype(np.float64)[:, None] - img.astype(np.float64)[None]) ** 2).sum(-1)
    g1 = np.argsort(e1, axis=1, kind="stable")[:, :topn]
    g2 = np.argsort(e2, axis=1, kind="stable")[:, :topn]
    joined = [set(a) & set(b) for a, b in zip(g1.tolist(), g2.tolist())]
    got = [set(row) for row in ids_of(res)]
    assert sum(len(g) for g in got) > nq
    # both fields are searched exactly here (every list probed, every code re-ranked): the join is the exact one
    assert np.mean([len(g & j) / max(1, len(j)) for g, j in zip(got, joined)]) >= 0.95
    e.close()
