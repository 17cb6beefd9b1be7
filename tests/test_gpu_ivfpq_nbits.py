"""IVFPQ at nbits_per_idx 1..7 on the H100 against the ksub-generic oracle (oracle_pqnb, held equal to the 8-bit oracle
and to a numpy restatement by tests/test_ivfpq_nbits_cpu.py).  With shared index state (coarse centroids, [M][2^nbits]
[dsub] codebook, probe lists) the bit-packed list codes, the precomputed table and the ADC scores are byte-equal; ids
equal up to exact ties at the k-th boundary.  Also: filters, tombstones, score window, re-rank, batches large enough
for the 8-bit list-major path, device training, updates and compaction, OPQ, gamma's index file, the engine path and
the parameter checks."""
import struct

import numpy as np
import pytest

import gamma_index_file as gif
from oracle import oracle as orc
from oracle_pqfs.twin import assert_same_results
from oracle_pqnb import ivfpq_nbits as pqnb
from test_ivfpq_nbits_cpu import write_ivfpq_nbits
from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
L2, IP = orc.METRIC_L2, orc.METRIC_IP
PACKED_KERNEL = "ivfpq_packed_scan_kernel"


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


def recall_1nn(ids, gt1, i):
    return float(np.mean([(gt1[q] in ids[q, :i]) for q in range(ids.shape[0])]))


def shared_state_index(db, d, M, nbits, nlist, metric, nprobe=8, extra=None):
    cent, _, _ = orc.kmeans(db[:4000], nlist, niter=5)
    a = orc.assign(cent, db, metric)
    pq = pqnb.pq_train(db[:4000] - cent[a[:4000]], M, 1 << nbits, niter=4)
    params = {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M, "nbits_per_idx": nbits, "metric_type": mt(metric)}
    params.update(extra or {})
    idx = gi().GammaIndex("IVFPQ", d, params)
    idx.set_centroids(cent)
    idx.set_pq_centroids(pq)
    idx.add_vectors(db)
    idx.add_pending()
    return idx, cent, a, pq, params


# M = 15: M nbits % 8 != 0 at every nbits < 8 (rows of 2..14 bytes, most not word-aligned), outside {8, 16, 32, 64}
@pytest.mark.parametrize("nbits", range(1, 8))
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M,data", [(64, 16, "int"), (60, 15, "int"), (60, 15, "float")])
def test_shared_state_bit_exact(nbits, metric, d, M, data):
    n, nq, nlist = 12000, 40, 32
    db = synth.sift_like(n, d, seed=41, rounded=data == "int")
    xq = synth.sift_like(nq, d, seed=42, rounded=data == "int")
    idx, cent, a, pq, _ = shared_state_index(db, d, M, nbits, nlist, metric)
    assert idx.pq_ksub == 1 << nbits and idx.code_size == pqnb.code_size(M, nbits)
    assert np.array_equal(idx.get_pq_centroids(), pq)
    # lists: layout and bit-packed residual codes byte-equal to the oracle's packing
    off_o, order = orc.build_lists(a, nlist)
    want = pqnb.ivfpq_encode(cent, pq, db, a)
    off, codes, ids = idx.export_lists()
    assert np.array_equal(off, off_o) and np.array_equal(ids, order) and np.array_equal(codes, want[order])
    assert np.array_equal(idx.pq_encode(db[:500], a[:500]), want[:500])
    T = None
    if metric == L2:
        T = pqnb.ivfpq_precompute_table(cent, pq)
        assert np.array_equal(idx.get_precomputed_table(), T)
    for k, nprobe in [(10, 8), (100, 16), (1, 1)]:
        cd, keys = orc.coarse_search(cent, xq, nprobe, metric)
        dg, ig = idx.search_preassigned(xq, k, keys, cd)
        assert idx.last_scan_kernel == PACKED_KERNEL
        do, io = pqnb.ivfpq_search_preassigned(off, codes, ids, cent, pq, T, xq, k, keys, cd, metric)
        assert_same_results(dg, ig, do, io)
    # tombstone, deletion and filter bitmaps, a missing probe, the score window
    cd, keys = orc.coarse_search(cent, xq, 8, metric)
    keys[3, 2] = -1
    l0 = int(np.flatnonzero(np.diff(off))[0])
    idx.tombstone(l0, 0)
    ids2 = ids.copy()
    ids2[off[l0]] |= orc.DEL_MASK
    rng = np.random.default_rng(nbits)
    delb = np.packbits(rng.random(n) < 0.2, bitorder="little")
    filb = np.packbits(rng.random(n) < 0.7, bitorder="little")
    for kw in ({"del_bitmap": delb}, {"filter_bitmap": filb}, {"del_bitmap": delb, "filter_bitmap": filb}):
        dg, ig = idx.search_preassigned(xq, 20, keys, cd, **kw)
        do, io = pqnb.ivfpq_search_preassigned(off, codes, ids2, cent, pq, T, xq, 20, keys, cd, metric, **kw)
        assert_same_results(dg, ig, do, io)
    do, io = pqnb.ivfpq_search_preassigned(off, codes, ids2, cent, pq, T, xq, 50, keys, cd, metric)
    lo, hi = float(min(do[0, 3], do[0, 40])), float(max(do[0, 3], do[0, 40]))
    dg, ig = idx.search_preassigned(xq, 50, keys, cd, min_score=lo, max_score=hi)
    do, io = pqnb.ivfpq_search_preassigned(off, codes, ids2, cent, pq, T, xq, 50, keys, cd, metric, min_score=lo,
                                           max_score=hi)
    assert_same_results(dg, ig, do, io)
    # exact re-rank (ivfpq.cc:675-726): the best k of the recall_num ADC candidates by exact score, checked against the
    # device's own candidates (tied ADC candidates at the recall_num boundary are scan-order dependent in the reference)
    dc, ic = idx.search_preassigned(xq, 60, keys, cd)
    dr, ir = idx.search_preassigned(xq, 10, keys, cd, params={"recall_num": 60})
    for q in range(nq):
        cand = ic[q][ic[q] >= 0]
        v = db[cand].astype(np.float64)
        exact = (((xq[q] - v) ** 2).sum(1) if metric == L2 else v @ xq[q]).astype(np.float32)
        order = np.lexsort((cand, exact if metric == L2 else -exact))[:10]
        if data == "int":  # exact sums
            assert np.array_equal(dr[q][:len(order)], exact[order])
            inner = exact[order] != exact[order][-1]
            assert set(ir[q][:len(order)][inner]) == set(cand[order][inner])
        else:
            assert np.allclose(dr[q][:len(order)], exact[order], rtol=1e-5)
    # nq * nprobe >= 32 nlist: an 8-bit index would go list-major; packed codes stay on the query-major kernel
    xb = synth.sift_like(160, d, seed=43, rounded=data == "int")
    cd, keys = orc.coarse_search(cent, xb, 8, metric)
    dg, ig = idx.search_preassigned(xb, 10, keys, cd)
    assert idx.last_scan_kernel == PACKED_KERNEL
    do, io = pqnb.ivfpq_search_preassigned(off, codes, ids2, cent, pq, T, xb, 10, keys, cd, metric)
    assert_same_results(dg, ig, do, io)
    idx.close()


def _train_on_device(db, d, M, nbits, nlist):
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nlist, "nsubvector": M, "nbits_per_idx": nbits,
                                       "metric_type": "L2", "training_threshold": 12800})
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    assert idx.indexed_count == len(db) and idx.pq_ksub == 1 << nbits
    return idx


def test_train_on_device_recall():
    """Device-trained ksub-means codebooks are as good as the oracle's (same algorithm, same seeds, statistical
    parity, tolerance 0.08 of recall@10 as for 8 bits); 4-bit codes rank worse than 8-bit ones on the same data."""
    d, n, nlist, M = 64, 40000, 64, 16
    db = synth.sift_like(n, d, seed=71)
    xq = synth.sift_like(200, d, seed=72)
    _, gt = orc.flat_search(db, xq, 1, L2)
    cent_o, _, _ = orc.kmeans(db[:12800], nlist, niter=10)
    a_o = orc.assign(cent_o, db, L2)
    off_o, order_o = orc.build_lists(a_o, nlist)
    cd_o, keys_o = orc.coarse_search(cent_o, xq, nlist, L2)
    recall = {}
    for nbits in (4, 6, 8):
        idx = _train_on_device(db, d, M, nbits, nlist)
        _, ig = idx.search(xq, 10)
        recall[nbits] = recall_1nn(ig, gt[:, 0], 10)
        if nbits < 8:
            pq_o = pqnb.pq_train(db[:12800] - cent_o[a_o[:12800]], M, 1 << nbits)
            codes_o = pqnb.ivfpq_encode(cent_o, pq_o, db, a_o)
            _, io_ref = pqnb.ivfpq_search_preassigned(off_o, codes_o[order_o], order_o, cent_o, pq_o,
                                                      pqnb.ivfpq_precompute_table(cent_o, pq_o), xq, 10, keys_o, cd_o, L2)
            assert recall[nbits] >= recall_1nn(io_ref, gt[:, 0], 10) - 0.08, (nbits, recall)
            # parity with the oracle on the device-built state
            off, codes, ids = idx.export_lists()
            cent, pqc, T = idx.get_centroids(), idx.get_pq_centroids(), idx.get_precomputed_table()
            assert np.array_equal(T, pqnb.ivfpq_precompute_table(cent, pqc))
            cd, keys = idx.coarse_search(xq, nlist)
            dg, ig = idx.search_preassigned(xq, 10, keys, cd)
            do, io = pqnb.ivfpq_search_preassigned(off, codes, ids, cent, pqc, T, xq, 10, keys, cd, L2)
            assert_same_results(dg, ig, do, io)
        idx.close()
    assert recall[4] < recall[8], recall


def test_update_and_compact_at_4_bits():
    d, M, n, nlist, nbits = 48, 12, 8000, 16, 4  # 6-byte rows
    db = synth.sift_like(n, d, seed=61)
    xq = synth.sift_like(30, d, seed=62)
    idx, cent, a, pq, _ = shared_state_index(db, d, M, nbits, nlist, L2)
    cur = db.copy()
    for vid, src in ((3, 5000), (100, 7000), (2500, 11), (3, 6000)):  # vid 3 twice: its first new entry dies too
        cur[vid] = db[src] + 1.0
        idx.update_vector(vid, cur[vid])
    off, codes, ids = idx.export_lists()
    live = ids >= 0
    assert (~live).sum() == 4 and live.sum() == n
    # every live entry holds the packed code of the vector's current value in its current list
    lst = np.repeat(np.arange(nlist), np.diff(off))
    vids = ids[live]
    assert np.array_equal(codes[live], pqnb.ivfpq_encode(cent, pq, cur[vids], lst[live]))
    assert np.array_equal(lst[live][np.argsort(vids)], orc.assign(cent, cur, L2))
    T = pqnb.ivfpq_precompute_table(cent, pq)
    cd, keys = orc.coarse_search(cent, xq, 8, L2)
    dg, ig = idx.search_preassigned(xq, 20, keys, cd)
    do, io = pqnb.ivfpq_search_preassigned(off, codes, ids, cent, pq, T, xq, 20, keys, cd, L2)
    assert_same_results(dg, ig, do, io)
    idx.compact()
    off2, codes2, ids2 = idx.export_lists()
    assert np.array_equal(off2, off) and np.array_equal(codes2, codes) and np.array_equal(ids2, ids)
    d2, i2 = idx.search_preassigned(xq, 20, keys, cd)
    assert np.array_equal(d2, dg) and np.array_equal(i2, ig)
    idx.close()


def test_opq_at_4_bits_trains_searches_dumps_and_loads(tmp_path):
    d, n, nlist, M = 32, 20000, 32, 8
    db = synth.sift_like(n, d, seed=83)
    xq = synth.sift_like(100, d, seed=84)
    params = {"ncentroids": nlist, "nprobe": 8, "nsubvector": M, "nbits_per_idx": 4, "metric_type": "L2",
              "training_threshold": 8000, "opq": {"nsubvector": M}}
    idx = gi().GammaIndex("IVFPQ", d, params)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    assert idx.has_opq and idx.pq_ksub == 16 and idx.code_size == 4
    A = idx.get_opq()
    assert np.allclose(A @ A.T, np.eye(d), atol=2e-5)
    _, gt = orc.flat_search(db, xq, 1, L2)
    dr, ir = idx.search(xq, 10, params={"recall_num": 100})
    assert idx.last_scan_kernel == PACKED_KERNEL
    assert np.array_equal(((xq[:, None, :] - db[ir]) ** 2).sum(-1), dr)  # re-rank: raw queries x raw vectors
    assert recall_1nn(ir, gt[:, 0], 10) >= 0.7
    xr = idx.apply_opq(xq)
    off, codes, ids = idx.export_lists()
    cent, pqc, T = idx.get_centroids(), idx.get_pq_centroids(), idx.get_precomputed_table()
    cd, keys = idx.coarse_search(xq, 8)
    dg, ig = idx.search_preassigned(xq, 50, keys, cd)
    do, io = pqnb.ivfpq_search_preassigned(off, codes, ids, cent, pqc, T, xr, 50, keys, cd, L2)
    assert_same_results(dg, ig, do, io)
    idx.dump(tmp_path, "emb.000")
    with open(tmp_path / "emb.000" / "ivfpq.index", "rb") as fh:
        assert fh.read() == write_ivfpq_nbits(d, gif.METRIC_L2, 8, cent, pqc, off, codes, ids, n, opq=A)
    again = gi().GammaIndex("IVFPQ", d, params)
    again.add_vectors(db)
    assert again.load(tmp_path, "emb.000") == n and np.array_equal(again.get_opq(), A)
    d2, i2 = again.search_preassigned(xq, 50, keys, cd)
    assert np.array_equal(d2, dg) and np.array_equal(i2, ig)
    idx.close()
    again.close()


@pytest.mark.parametrize("nbits", [1, 3, 4, 7])
@pytest.mark.parametrize("metric", [L2, IP])
def test_index_file_dump_load_and_refusals(tmp_path, nbits, metric):
    d, M, n, nlist = 60, 15, 6000, 16
    db = synth.sift_like(n, d, seed=91)
    xq = synth.sift_like(20, d, seed=92)
    idx, cent, a, pq, params = shared_state_index(db, d, M, nbits, nlist, metric)
    off, codes, ids = idx.export_lists()
    idx.dump(tmp_path, "emb.000")
    with open(tmp_path / "emb.000" / "ivfpq.index", "rb") as fh:
        buf = fh.read()
    assert buf == write_ivfpq_nbits(d, metric, 8, cent, pq, off, codes, ids, n)
    cd, keys = idx.coarse_search(xq, 8)
    dg, ig = idx.search_preassigned(xq, 30, keys, cd)
    again = gi().GammaIndex("IVFPQ", d, params)
    again.add_vectors(db)
    assert again.load(tmp_path, "emb.000") == n
    d2, i2 = again.search_preassigned(xq, 30, keys, cd)
    assert np.array_equal(d2, dg) and np.array_equal(i2, ig)
    again.close()
    # a file of another width, and one whose code_size field disagrees with its nbits, are refused
    other = 8 if nbits == 7 else nbits + 1
    pq_o = np.random.default_rng(0).normal(size=(M, 1 << other, d // M)).astype(np.float32)
    codes_o = np.zeros((len(ids), pqnb.code_size(M, other)), np.uint8)
    head = len(gif.fourcc("IwPQ") + gif._ivf_header(d, n, metric, nlist, 8, cent))
    bad_cs = bytearray(buf)
    struct.pack_into("<Q", bad_cs, head + 1, pqnb.code_size(M, nbits) + 1)
    for name, blob, what in (("wide.000", write_ivfpq_nbits(d, metric, 8, cent, pq_o, off, codes_o, ids, n), "nbits"),
                             ("cs.000", bytes(bad_cs), "code_size")):
        (tmp_path / name).mkdir()
        (tmp_path / name / "ivfpq.index").write_bytes(blob)
        fresh = gi().GammaIndex("IVFPQ", d, params)
        fresh.add_vectors(db)
        with pytest.raises(gi().GammaError, match=what):
            fresh.load(tmp_path, name)
        fresh.close()
    idx.close()


def test_nbits_parameter_range():
    d = 32
    base = {"ncentroids": 16, "nprobe": 4, "nsubvector": 8, "metric_type": "L2"}
    for nbits in (9, 16):
        with pytest.raises(gi().GammaError, match="nbits_per_idx \\[%d\\] above 8 is not supported" % nbits):
            gi().GammaIndex("IVFPQ", d, dict(base, nbits_per_idx=nbits))
    with pytest.raises(gi().GammaError, match="invalid nbits_per_idx"):
        gi().GammaIndex("IVFPQ", d, dict(base, nbits_per_idx=-2))
    for nbits, ksub, cs in ((0, 256, 8), (-1, 256, 8), (8, 256, 8), (1, 2, 1), (5, 32, 5)):
        idx = gi().GammaIndex("IVFPQ", d, dict(base, nbits_per_idx=nbits))
        assert (idx.pq_ksub, idx.code_size) == (ksub, cs)
        idx.close()


def test_index_factory_pq32x4():
    d, n = 128, 12000
    db = synth.sift_like(n, d, seed=95)
    xq = synth.sift_like(20, d, seed=96)
    idx = gi().index_factory(d, "IVF256,PQ32x4", nprobe=32, training_threshold=10000)
    assert idx.pq_ksub == 16 and idx.code_size == 16
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    dr, ir = idx.search(xq, 10, params={"recall_num": 100})
    assert idx.last_scan_kernel == PACKED_KERNEL
    _, gt = orc.flat_search(db, xq, 1, L2)
    assert recall_1nn(ir, gt[:, 0], 10) >= 0.8
    idx.close()


# ---- engine (include/gamma_api.h) ------------------------------------------------------------------------------
D = 32
PQ4 = {"ncentroids": 16, "nprobe": 8, "nsubvector": 8, "nbits_per_idx": 4, "metric_type": "L2", "training_threshold": 1000}


def make_engine(tmp_path, params, name="pq4"):
    from vearch_b200 import engine
    e = engine.GammaEngine(str(tmp_path), space_name=name)
    e.create_table(name, D, "IVFPQ", params, fields=(("_id", wire.DT_STRING, False),))
    return e


def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def test_engine_flow_and_dump_load(tmp_path):
    from vearch_b200 import engine
    for nbits in (9, 16):
        e = engine.GammaEngine(str(tmp_path / "bad"))
        with pytest.raises(engine.GammaStatusError) as ei:
            e.create_table("t", D, "IVFPQ", dict(PQ4, nbits_per_idx=nbits))
        assert "above 8 is not supported" in ei.value.msg
        e.close()
    for nbits in (0, -1):  # the default, 8
        e = engine.GammaEngine(str(tmp_path / f"def{nbits}"))
        e.create_table("t", D, "IVFPQ", dict(PQ4, nbits_per_idx=nbits))
        e.close()
    db, xq = synth.sift_like(3000, D, seed=81), synth.sift_like(16, D, seed=82)
    e = make_engine(tmp_path / "sp", PQ4)
    for i, v in enumerate(db):
        assert e.add_doc(f"doc{i}", v) == 0
    e.build_index()
    e.wait_indexed(len(db))
    e.delete_doc("doc7")
    before = e.search(xq, 10, index_params={"nprobe": 8, "recall_num": 50})
    got = keys_of(before)
    assert all(len(r) == 10 for r in got) and not any("doc7" in r for r in got)
    for q in range(len(xq)):  # re-ranked scores are the exact distances of the returned docs
        for key, s in zip(got[q], scores_of(before)[q]):
            assert s == float(((xq[q] - db[int(key[3:])]) ** 2).sum())
    plain = e.search(xq, 10, index_params={"nprobe": 8})
    assert e.dump() == 0
    e.close()
    # the lists travel in gamma's index file at 4 bits: code_size 4, nbits 4, [8][16][4] centroids
    with open(tmp_path / "sp" / "retrieval_model_index" / "emb.000" / "ivfpq.index", "rb") as fh:
        buf = fh.read()
    head = len(gif.fourcc("IwPQ") + gif._ivf_header(D, 0, L2, 16, 8, np.zeros((16, D), np.float32)))
    assert struct.unpack_from("<?QQQQQ", buf, head) == (True, 4, D, 8, 4, 8 * 16 * 4)
    e2 = make_engine(tmp_path / "sp", PQ4)
    assert e2.load() == 0
    e2.wait_indexed(len(db))
    after = e2.search(xq, 10, index_params={"nprobe": 8, "recall_num": 50})
    assert keys_of(after) == keys_of(before) and scores_of(after) == scores_of(before)
    again = e2.search(xq, 10, index_params={"nprobe": 8})
    assert keys_of(again) == keys_of(plain) and scores_of(again) == scores_of(plain)
    assert e2.get_doc_by_id("doc7")[0] == -1
    e2.close()
