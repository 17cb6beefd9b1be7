"""GPU parity tests: the sm_90a path (through the C-ABI in vearch_b200/libgamma.so) against the
CPU oracle on the same seeded inputs.

Bars (north_star): integer/byte/index work bit-exact; floating point within 1e-4 relative.
 * SIFT-shaped integer-valued data makes every fp32 partial sum exact, so scores must be
   BIT-EQUAL and ids equal, except inside a group of exactly tied scores at the k-th boundary,
   where the reference itself is scan-order dependent (DESIGN.md "tie rule").
 * With shared index state (centroids, codebooks, list contents, probe lists, coarse distances)
   the IVF-PQ ADC distances are bit-equal on float data too (same table arithmetic, same order).
"""
import numpy as np
import pytest

from oracle import oracle as orc
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = orc.METRIC_L2, orc.METRIC_IP
FLT_MAX = np.finfo(np.float32).max


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


def assert_same_results(dg, ig, do, io, bit_exact=True, rtol=1e-4):
    """scores equal (bitwise or rtol); ids equal except inside the tie group at the k-th boundary."""
    assert dg.shape == do.shape and ig.shape == io.shape
    if bit_exact:
        assert np.array_equal(dg, do), f"score mismatch: max abs diff {np.abs(dg - do).max()}"
    else:
        ok = np.isclose(dg, do, rtol=rtol, atol=1e-6) | ((ig < 0) & (io < 0))
        assert ok.all(), f"score mismatch beyond rtol={rtol}"
    for q in range(dg.shape[0]):
        if np.array_equal(ig[q], io[q]):
            continue
        valid = io[q] >= 0
        assert np.array_equal(valid, ig[q] >= 0), "different number of results"
        if not valid.any():
            continue
        boundary = do[q][valid][-1]
        for v in np.unique(do[q][valid]):
            grp = valid & (do[q] == v)
            if v == boundary:
                continue  # boundary tie group: membership is scan-order dependent in the reference
            if bit_exact:
                assert set(ig[q][grp]) == set(io[q][grp]), f"query {q}: ids differ at score {v}"
        if not bit_exact:
            # float data: allow swaps between near-equal neighbours only
            common = len(set(ig[q][valid]) & set(io[q][valid]))
            assert common >= valid.sum() - 1, f"query {q}: {valid.sum() - common} ids differ"


def recall_1nn(ids, gt1, i):
    return float(np.mean([(gt1[q] in ids[q, :i]) for q in range(ids.shape[0])]))


# ----------------------------------------------------------------------------------------------
# K1 FLAT
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("n,d,nq,k", [(5000, 128, 37, 10), (3000, 32, 5, 100), (777, 30, 3, 7), (40, 8, 2, 64)])
def test_flat_matches_oracle(metric, n, d, nq, k):
    db = synth.sift_like(n, d, seed=11)
    xq = synth.sift_like(nq, d, seed=12)
    idx = gi().GammaIndex("FLAT", d, {"metric_type": mt(metric)})
    idx.add_vectors(db[: n // 2])
    idx.add_vectors(db[n // 2:])
    assert idx.ntotal == n
    dg, ig = idx.search(xq, k)
    do, io = orc.flat_search(db, xq, k, metric)
    assert_same_results(dg, ig, do, io)
    if metric == L2:
        assert np.array_equal(ig, io)  # FLAT L2: ids bit-exact including order
    idx.close()


def test_flat_multi_chunk_and_filters():
    n, d, nq, k = 300_000, 16, 16, 20  # > 131072 rows => several distance blocks + key merge
    db = synth.sift_like(n, d, seed=21)
    xq = synth.sift_like(nq, d, seed=22)
    idx = gi().GammaIndex("FLAT", d, {"metric_type": "L2"})
    idx.add_vectors(db)
    dg, ig = idx.search(xq, k)
    do, io = orc.flat_search(db, xq, k, L2)
    assert np.array_equal(dg, do) and np.array_equal(ig, io)
    rng = np.random.default_rng(0)
    deleted = rng.random(n) < 0.4
    allowed = rng.random(n) < 0.5
    delb, filb = np.packbits(deleted, bitorder="little"), np.packbits(allowed, bitorder="little")
    dg, ig = idx.search(xq, k, del_bitmap=delb, filter_bitmap=filb)
    do, io = orc.flat_search(db, xq, k, L2, del_bitmap=delb, filter_bitmap=filb)
    assert np.array_equal(dg, do) and np.array_equal(ig, io)
    assert not deleted[ig[ig >= 0]].any() and allowed[ig[ig >= 0]].all()
    lo, hi = float(do[0, 3]), float(do[0, 12])
    dg, ig = idx.search(xq, k, min_score=lo, max_score=hi)
    do, io = orc.flat_search(db, xq, k, L2, min_score=lo, max_score=hi)
    assert np.array_equal(dg, do) and np.array_equal(ig, io)
    idx.close()


def test_flat_empty_and_tiny():
    idx = gi().GammaIndex("FLAT", 8, {"metric_type": "L2"})
    xq = synth.sift_like(3, 8, seed=1)
    dg, ig = idx.search(xq, 5)
    assert (ig == -1).all() and (dg == FLT_MAX).all()
    db = synth.sift_like(2, 8, seed=2)
    idx.add_vectors(db)
    dg, ig = idx.search(xq, 5)
    do, io = orc.flat_search(db, xq, 5, L2)
    assert np.array_equal(dg, do) and np.array_equal(ig, io)
    idx.close()


def test_flat_float_data_and_reference_pins():
    db = synth.embed_like(4000, 64, seed=3)
    idx = gi().GammaIndex("FLAT", 64, {"metric_type": "InnerProduct"})
    idx.add_vectors(db)
    dg, ig = idx.search(db[:64], 10)
    do, io = orc.flat_search(db, db[:64], 10, IP)
    assert_same_results(dg, ig, do, io, bit_exact=False)
    # self-query top-1 ~ 1.0 for normalised IP (internal/engine/tests/test.h:554-565)
    assert np.array_equal(ig[:, 0], np.arange(64)) and np.abs(dg[:, 0] - 1).max() < 1e-5
    # L2 score == sum (x-y)^2 within 0.01 (test/test_module_vector.py:337-364)
    dl, il = idx.search(db[:8], 5, params={"metric_type": "L2"})
    manual = ((db[:8, None, :] - db[il]) ** 2).sum(-1)
    assert np.abs(manual - dl).max() < 0.01
    idx.close()


# ----------------------------------------------------------------------------------------------
# K2 coarse quantiser, K6 k-means
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ivf_state():
    d, n, nlist = 64, 20000, 64
    db = synth.sift_like(n, d, seed=31)
    xq = synth.sift_like(48, d, seed=32)
    cent, _, _ = orc.kmeans(db[:8000], nlist, niter=6)
    cent = np.rint(cent).astype(np.float32)  # integer-valued shared state => exact arithmetic
    a = orc.assign(cent, db, L2)
    off, order = orc.build_lists(a, nlist)
    return dict(d=d, n=n, nlist=nlist, db=db, xq=xq, cent=cent, assign=a, off=off, order=order)


@pytest.mark.parametrize("metric", [L2, IP])
def test_coarse_search_exact(ivf_state, metric):
    s = ivf_state
    idx = gi().GammaIndex("IVFFLAT", s["d"], {"ncentroids": s["nlist"], "nprobe": 8, "metric_type": mt(metric)})
    idx.set_centroids(s["cent"])
    dg, ig = idx.coarse_search(s["xq"], 8)
    do, io = orc.coarse_search(s["cent"], s["xq"], 8, metric)
    assert_same_results(dg, ig, do, io)
    idx.close()


def test_kmeans_update_bit_exact(ivf_state):
    s = ivf_state
    x = synth.embed_like(5000, 48, seed=5)  # float data: order of summation matters
    a = np.random.default_rng(1).integers(0, 37, size=5000)
    a[a == 5] = 6  # leave one cluster empty
    co, h = orc.kmeans_update(x, 37, a)
    cg = gi().kmeans_update(x, 37, a)
    assert np.array_equal(co, cg)


def test_kmeans_device_quality():
    x = synth.sift_like(8000, 32, seed=41)
    cg, og = gi().kmeans(x, 32, niter=10)
    co, _, oo = orc.kmeans(x, 32, niter=10)
    # same seeded initialisation and integer data => identical first objective
    assert og[0] == oo[0]
    assert og[-1] <= og[0] and abs(og[-1] - oo[-1]) <= 0.02 * oo[-1]
    ag = orc.assign(cg, x, L2)
    ao = orc.assign(co, x, L2)
    ig_, io_ = ((x - cg[ag]) ** 2).sum(), ((x - co[ao]) ** 2).sum()
    assert abs(ig_ - io_) <= 0.02 * io_


# ----------------------------------------------------------------------------------------------
# K3 IVF-Flat
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ivfflat_index(ivf_state):
    s = ivf_state
    idx = gi().GammaIndex("IVFFLAT", s["d"], {"ncentroids": s["nlist"], "nprobe": 8, "metric_type": "L2"})
    idx.set_centroids(s["cent"])
    idx.add_vectors(s["db"][:12000])
    idx.add_pending()
    idx.add_vectors(s["db"][12000:])  # second batch exercises list growth (copy-on-grow)
    idx.add_pending()
    assert idx.indexed_count == s["n"]
    yield idx
    idx.close()


def test_ivf_lists_match_oracle_layout(ivf_state, ivfflat_index):
    s = ivf_state
    off, codes, ids = ivfflat_index.export_lists()
    assert np.array_equal(off, s["off"])  # same assignment
    assert np.array_equal(ids, s["order"])  # insertion (vid) order inside each list
    vecs = codes.view(np.float32).reshape(len(ids), -1)[:, : s["d"]]
    assert np.array_equal(vecs, s["db"][s["order"]])


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("k,nprobe", [(10, 8), (100, 16), (1, 1)])
def test_ivfflat_search_preassigned_exact(ivf_state, ivfflat_index, metric, k, nprobe):
    s = ivf_state
    cd, keys = orc.coarse_search(s["cent"], s["xq"], nprobe, metric)
    dg, ig = ivfflat_index.search_preassigned(s["xq"], k, keys, cd, params={"metric_type": mt(metric)})
    do, io = orc.ivfflat_search_preassigned(s["off"], s["db"][s["order"]], s["order"], s["xq"], k, keys, metric)
    assert_same_results(dg, ig, do, io)


def test_ivfflat_search_end_to_end_and_filters(ivf_state, ivfflat_index):
    s = ivf_state
    nprobe, k = 8, 10
    dg, ig = ivfflat_index.search(s["xq"], k, params={"nprobe": nprobe})
    cd, keys = orc.coarse_search(s["cent"], s["xq"], nprobe, L2)
    do, io = orc.ivfflat_search_preassigned(s["off"], s["db"][s["order"]], s["order"], s["xq"], k, keys, L2)
    assert_same_results(dg, ig, do, io)
    rng = np.random.default_rng(3)
    deleted = rng.random(s["n"]) < 0.3
    delb = np.packbits(deleted, bitorder="little")
    dg, ig = ivfflat_index.search(s["xq"], k, params={"nprobe": nprobe}, del_bitmap=delb)
    do, io = orc.ivfflat_search_preassigned(s["off"], s["db"][s["order"]], s["order"], s["xq"], k, keys, L2,
                                            del_bitmap=delb)
    assert_same_results(dg, ig, do, io)
    lo, hi = float(do[0, 2]), float(do[0, 7])
    dg, ig = ivfflat_index.search(s["xq"], k, params={"nprobe": nprobe}, min_score=lo, max_score=hi)
    do, io = orc.ivfflat_search_preassigned(s["off"], s["db"][s["order"]], s["order"], s["xq"], k, keys, L2,
                                            min_score=lo, max_score=hi)
    assert_same_results(dg, ig, do, io)
    # brute-force request on an IVF index == FLAT (gamma_index_ivfflat.cc:541-550)
    dg, ig = ivfflat_index.search(s["xq"], k, brute_force=True)
    do, io = orc.flat_search(s["db"], s["xq"], k, L2)
    assert np.array_equal(dg, do) and np.array_equal(ig, io)
    # reference CI pins (test/test_vector_index_ivfflat.py:89-94)
    dg, ig = ivfflat_index.search(s["xq"], 100, params={"nprobe": 16})
    assert recall_1nn(ig, io[:, 0], 1) >= 0.8 and recall_1nn(ig, io[:, 0], 10) >= 0.9


def test_ivfflat_tombstone_and_bad_keys(ivf_state):
    s = ivf_state
    idx = gi().GammaIndex("IVFFLAT", s["d"], {"ncentroids": s["nlist"], "nprobe": 4, "metric_type": "L2"})
    idx.set_centroids(s["cent"])
    idx.add_vectors(s["db"][:5000])
    deleted = np.zeros(5000, bool)
    deleted[::7] = True  # deleted before indexing => never enter the lists (ivfflat.cc:436)
    idx.add_pending(del_bitmap=np.packbits(deleted, bitorder="little"))
    off, codes, ids = idx.export_lists()
    assert len(ids) == 5000 - deleted.sum() and not deleted[ids].any()
    cd, keys = orc.coarse_search(s["cent"], s["xq"], 4, L2)
    vecs = codes.view(np.float32).reshape(len(ids), -1)
    d0, i0 = idx.search_preassigned(s["xq"], 5, keys, cd)
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids, s["xq"], 5, keys, L2)
    assert_same_results(d0, i0, do, io)
    # tombstone the best hit of query 0 (Update path, realtime_mem_data.cc:298-320)
    victim = int(i0[0, 0])
    pos_global = int(np.flatnonzero(ids == victim)[0])
    l = int(np.searchsorted(off, pos_global, side="right") - 1)
    idx.tombstone(l, pos_global - int(off[l]))
    ids2 = ids.copy()
    ids2[pos_global] |= orc.DEL_MASK
    d1, i1 = idx.search_preassigned(s["xq"], 5, keys, cd)
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids2, s["xq"], 5, keys, L2)
    assert_same_results(d1, i1, do, io)
    assert victim not in i1[0]
    keys2 = keys.copy()
    keys2[:, 1] = -1  # "not enough centroids for multiprobe"
    d2, i2 = idx.search_preassigned(s["xq"], 5, keys2, cd)
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids2, s["xq"], 5, keys2, L2)
    assert_same_results(d2, i2, do, io)
    idx.close()


def test_ivfflat_train_on_device_recall():
    d, n, nlist = 32, 30000, 64
    db = synth.sift_like(n, d, seed=51)
    xq = synth.sift_like(100, d, seed=52)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 16, "metric_type": "L2",
                                         "training_threshold": 10000})
    idx.add_vectors(db)
    assert not idx.is_trained
    dg, ig = idx.search(xq, 10)  # untrained => FLAT fallback over all stored vectors
    do, io = orc.flat_search(db, xq, 10, L2)
    assert np.array_equal(dg, do) and np.array_equal(ig, io)
    idx.train()
    idx.add_pending()
    assert idx.is_trained and idx.indexed_count == n
    dg, ig = idx.search(xq, 10)
    assert recall_1nn(ig, io[:, 0], 1) >= 0.8 and recall_1nn(ig, io[:, 0], 10) >= 0.9
    # exact parity against the oracle on the index state the device produced
    off, codes, ids = idx.export_lists()
    cent = idx.get_centroids()
    cd, keys = idx.coarse_search(xq, 16)
    dref, iref = orc.ivfflat_search_preassigned(off, codes.view(np.float32).reshape(len(ids), -1), ids, xq, 10, keys, L2)
    assert_same_results(dg, ig, dref, iref)
    idx.close()


def test_ivfflat_d768_inner_product():
    d, n, nlist = 768, 6000, 16
    db = synth.embed_like(n, d, seed=61)
    xq = synth.embed_like(20, d, seed=62)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 4, "metric_type": "InnerProduct",
                                         "training_threshold": 2000})
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    dg, ig = idx.search(xq, 10)
    off, codes, ids = idx.export_lists()
    cd, keys = idx.coarse_search(xq, 4)
    dref, iref = orc.ivfflat_search_preassigned(off, codes.view(np.float32).reshape(len(ids), -1), ids, xq, 10, keys, IP)
    assert_same_results(dg, ig, dref, iref, bit_exact=False)
    idx.close()


# ----------------------------------------------------------------------------------------------
# K4 / K5 / K8 IVF-PQ
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pq_state(ivf_state):
    s = ivf_state
    M = 8
    resid = s["db"][:8000] - s["cent"][s["assign"][:8000]]
    pqc = orc.pq_train(resid, M, niter=6)  # float codebooks
    return dict(M=M, pqc=pqc)


@pytest.mark.parametrize("metric", [L2, IP])
def test_ivfpq_shared_state_bit_exact(ivf_state, pq_state, metric):
    s, M, pqc = ivf_state, pq_state["M"], pq_state["pqc"]
    idx = gi().GammaIndex("IVFPQ", s["d"], {"ncentroids": s["nlist"], "nprobe": 8, "nsubvector": M,
                                            "metric_type": mt(metric)})
    idx.set_centroids(s["cent"])
    idx.set_pq_centroids(pqc)
    idx.add_vectors(s["db"])
    idx.add_pending()
    a = orc.assign(s["cent"], s["db"], metric)
    off_o, order = orc.build_lists(a, s["nlist"])
    codes_o = orc.ivfpq_encode(s["cent"], pqc, s["db"], a)
    # K8: codes byte-exact, list layout identical
    assert np.array_equal(idx.pq_encode(s["db"][:3000], a[:3000]), codes_o[:3000])
    off, codes, ids = idx.export_lists()
    assert np.array_equal(off, off_o) and np.array_equal(ids, order) and np.array_equal(codes, codes_o[order])
    T = None
    if metric == L2:
        T = orc.ivfpq_precompute_table(s["cent"], pqc)
        assert np.array_equal(idx.get_precomputed_table(), T)  # K4 table bit-equal
    for k, nprobe, recall_num in [(10, 8, 0), (50, 16, 0), (100, 8, 0), (10, 8, 100), (10, 8, 5)]:
        cd, keys = orc.coarse_search(s["cent"], s["xq"], nprobe, metric)
        kk = max(k, recall_num)
        # ADC stage (K4+K5): bit-equal scores, ids equal up to exact ties at the kk-th boundary
        dc, ic = idx.search_preassigned(s["xq"], kk, keys, cd)
        do, io = orc.ivfpq_search_preassigned(off, codes, ids, s["cent"], pqc, T, s["xq"], kk, keys, cd, metric)
        assert_same_results(dc, ic, do, io)
        if not recall_num:
            continue
        # K5r exact re-rank (ivfpq.cc:675-726): the best k of the ADC candidates by exact score.
        # Checked against the device's own candidate set because candidates tied at the ADC
        # boundary are scan-order dependent in the reference.
        dg, ig = idx.search_preassigned(s["xq"], k, keys, cd, params={"recall_num": recall_num})
        for q in range(s["xq"].shape[0]):
            cand = ic[q][ic[q] >= 0]
            v = s["db"][cand]
            exact = ((s["xq"][q] - v) ** 2).sum(1) if metric == L2 else v @ s["xq"][q]
            order = np.lexsort((cand, exact if metric == L2 else -exact))[:k]
            assert np.array_equal(dg[q][: len(order)], exact[order].astype(np.float32))
            for val in np.unique(exact[order][:-1]):
                if val != exact[order][-1]:
                    assert set(ig[q][dg[q] == val]) == set(cand[order][exact[order] == val])
    # filters
    deleted = np.random.default_rng(5).random(s["n"]) < 0.25
    delb = np.packbits(deleted, bitorder="little")
    cd, keys = orc.coarse_search(s["cent"], s["xq"], 8, metric)
    dg, ig = idx.search_preassigned(s["xq"], 10, keys, cd, del_bitmap=delb)
    do, io = orc.ivfpq_search_preassigned(off, codes, ids, s["cent"], pqc, T, s["xq"], 10, keys, cd, metric,
                                          del_bitmap=delb)
    assert_same_results(dg, ig, do, io)
    idx.close()


def test_ivfpq_train_on_device_recall():
    d, n, nlist, M = 64, 40000, 64, 16
    db = synth.sift_like(n, d, seed=71)
    xq = synth.sift_like(100, d, seed=72)
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": 16, "nsubvector": M, "metric_type": "L2",
                                       "training_threshold": 12800})
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    assert idx.indexed_count == n
    _, gt = orc.flat_search(db, xq, 1, L2)
    dg, ig = idx.search(xq, 100)
    # device-trained codebooks must be as good as the oracle's (same algorithm, same seeds)
    cent_o, _, _ = orc.kmeans(db[:12800], nlist, niter=10)
    a_o = orc.assign(cent_o, db, L2)
    off_o, order_o = orc.build_lists(a_o, nlist)
    pq_o = orc.pq_train(db[:12800] - cent_o[a_o[:12800]], M, niter=25)
    codes_o = orc.ivfpq_encode(cent_o, pq_o, db, a_o)
    cd_o, keys_o = orc.coarse_search(cent_o, xq, 16, L2)
    _, io_ref = orc.ivfpq_search_preassigned(off_o, codes_o[order_o], order_o, cent_o, pq_o,
                                             orc.ivfpq_precompute_table(cent_o, pq_o), xq, 100, keys_o, cd_o, L2)
    assert recall_1nn(ig, gt[:, 0], 10) >= recall_1nn(io_ref, gt[:, 0], 10) - 0.08
    # reference CI pins for IVFPQ (test/test_vector_index_ivfpq.py:105-111): r@100 >= 0.95, and with
    # gamma's exact re-rank r@1 >= 0.6, r@10 >= 0.9
    assert recall_1nn(ig, gt[:, 0], 100) >= 0.95
    dr, ir = idx.search(xq, 10, params={"recall_num": 100})
    assert recall_1nn(ir, gt[:, 0], 1) >= 0.8 and recall_1nn(ir, gt[:, 0], 10) >= 0.9
    exact = ((xq[:, None, :] - db[ir]) ** 2).sum(-1)
    assert np.array_equal(exact, dr)  # re-ranked scores are exact L2 (integer data)
    # parity with the oracle on the device-built state (same probes & coarse distances)
    off, codes, ids = idx.export_lists()
    cent, pqc, T = idx.get_centroids(), idx.get_pq_centroids(), idx.get_precomputed_table()
    assert np.array_equal(T, orc.ivfpq_precompute_table(cent, pqc))
    cd, keys = idx.coarse_search(xq, 16)
    do, io = orc.ivfpq_search_preassigned(off, codes, ids, cent, pqc, T, xq, 100, keys, cd, L2)
    assert_same_results(dg, ig, do, io)
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M,data", [(128, 16, "float"), (128, 16, "int"), (64, 8, "float"), (64, 16, "float"),
                                      (128, 8, "float"), (32, 4, "float"), (96, 12, "float"), (128, 32, "float"),
                                      (128, 64, "float")])
def test_ivfpq_listmajor_tensor_core_filter_matches_oracle(metric, d, M, data):
    """Many queries per list => the IVF-PQ scan runs list-major (kernels_pqtc.cu): exact LUT scan of the
    first probes -> per-query bound -> fp16 wgmma FILTER over the other probes -> candidates re-scored
    with the reference arithmetic.  The filter must never lose an entry: ADC scores bit-equal to the
    oracle and ids equal (tie-aware) on float data (every mantissa bit in use) as on integer data, at
    k = 10 and at re-rank depth 400, with tombstones, deletion bitmap, missing probes, score window."""
    n, nq, nlist, nprobe = 40000, 900, 16, 6
    if data == "int":
        db, xq = synth.sift_like(n, d, seed=195), synth.sift_like(nq, d, seed=196)
    else:
        rng = np.random.default_rng(197)
        centers = rng.normal(0, 1, (64, d)).astype(np.float32)
        db = (centers[rng.integers(0, 64, n)] + 0.35 * rng.normal(0, 1, (n, d))).astype(np.float32)
        xq = (centers[rng.integers(0, 64, nq)] + 0.35 * rng.normal(0, 1, (nq, d))).astype(np.float32)
    cent, _, _ = orc.kmeans(db[:4000], nlist, niter=5)
    a = orc.assign(cent, db, metric)
    pqc = orc.pq_train(db[:6000] - cent[a[:6000]], M, niter=4)
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M,
                                       "metric_type": mt(metric)})
    idx.set_centroids(cent)
    idx.set_pq_centroids(pqc)
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids = idx.export_lists()
    T = orc.ivfpq_precompute_table(cent, pqc) if metric == L2 else None
    cd, keys = orc.coarse_search(cent, xq, nprobe, metric)
    keys[5, 2] = -1   # "not enough centroids" (gamma_index_ivfpq.cc:640)
    keys[7, 0] = -1   # ... in the probe the bound comes from
    deleted = np.random.default_rng(2).random(n) < 0.2
    delb = np.packbits(deleted, bitorder="little")
    idx.tombstone(int(np.searchsorted(off, 0, side="right") - 1), 0)
    ids2 = ids.copy()
    ids2[0] |= orc.DEL_MASK
    for kk, kw in [(10, {}), (400, {}), (10, {"del_bitmap": delb}), (100, {"del_bitmap": delb})]:
        dg, ig = idx.search_preassigned(xq, kk, keys, cd, **kw)
        # shapes outside the filter's list (M = 12, 32, 64) take the LUT kernel for every probe; same answers either way
        assert idx.last_scan_kernel == ("pqtc_scan_kernel" if M in (4, 8, 16) else "ivfpq_scan_kernel")
        do, io = orc.ivfpq_search_preassigned(off, codes, ids2, cent, pqc, T, xq, kk, keys, cd, metric, **kw)
        assert_same_results(dg, ig, do, io)
    do, io = orc.ivfpq_search_preassigned(off, codes, ids2, cent, pqc, T, xq, 50, keys, cd, metric)
    lo, hi = float(min(do[0, 3], do[0, 40])), float(max(do[0, 3], do[0, 40]))
    dg, ig = idx.search_preassigned(xq, 50, keys, cd, min_score=lo, max_score=hi)
    do, io = orc.ivfpq_search_preassigned(off, codes, ids2, cent, pqc, T, xq, 50, keys, cd, metric, min_score=lo,
                                          max_score=hi)
    assert_same_results(dg, ig, do, io)
    # exact re-rank on top of the filtered ADC stage: same final answer as the LUT-only pipeline
    dr, ir = idx.search_preassigned(xq, 10, keys, cd, params={"recall_num": 400})
    dc, ic = idx.search_preassigned(xq, 400, keys, cd)
    for q in range(0, nq, 37):
        cand = ic[q][ic[q] >= 0]
        v = db[cand]
        exact = (((xq[q] - v) ** 2).sum(1) if metric == L2 else v @ xq[q]).astype(np.float32)
        order = np.lexsort((cand, exact if metric == L2 else -exact))[:10]
        assert np.allclose(dr[q][: len(order)], exact[order], rtol=1e-5)
    # a small batch of the same index goes through the LUT kernel and must agree with the big one
    d1, i1 = idx.search_preassigned(xq[:3], 10, keys[:3], cd[:3])
    assert idx.last_scan_kernel == "ivfpq_scan_kernel"
    d2, i2 = idx.search_preassigned(xq, 10, keys, cd)
    assert np.array_equal(d1, d2[:3]) and np.array_equal(i1, i2[:3])
    idx.close()


# ----------------------------------------------------------------------------------------------
# K7 merge / multi-partition
# ----------------------------------------------------------------------------------------------
def test_merge_partitions_matches_router_order():
    import torch
    rng = np.random.default_rng(9)
    nparts, nq, k = 4, 33, 10
    for metric in (L2, IP):
        dis = np.sort(rng.integers(0, 40, size=(nparts, nq, k)).astype(np.float32), axis=2)
        if metric == IP:
            dis = dis[:, :, ::-1].copy()
        ids = rng.integers(0, 1000, size=(nparts, nq, k)).astype(np.int64)
        ids[1, :, 7:] = -1
        od, oi = orc.merge_partitions(dis, ids, metric)
        gd, gi_ = gi().merge_partitions_device(torch.from_numpy(dis).cuda(), torch.from_numpy(ids).cuda(), metric)
        assert np.array_equal(gd.cpu().numpy(), od) and np.array_equal(gi_.cpu().numpy(), oi)


def test_search_device_resident_matches_host(ivf_state, ivfflat_index):
    import torch
    s = ivf_state
    dg, ig = ivfflat_index.search(s["xq"], 10, params={"nprobe": 8})
    xq_dev = torch.from_numpy(s["xq"]).cuda()
    dd, di = ivfflat_index.search_device(xq_dev, 10, params={"nprobe": 8})
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy(), dg) and np.array_equal(di.cpu().numpy(), ig)


# ----------------------------------------------------------------------------------------------
# K2 tensor-core variant (wgmma 3xTF32) against the exact CUDA-core kernel
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("n,m,d", [(128, 128, 32), (300, 200, 100), (129, 257, 128), (1000, 4096, 64), (70, 33, 8)])
def test_tensor_core_distance_kernel(metric, n, m, d):
    # integer-valued operands: TF32 holds them exactly => bit-equal to the exact kernel and to fp64 maths
    x = synth.sift_like(n, d, seed=91)
    c = synth.sift_like(m, d, seed=92)
    exact = gi().debug_dist_matrix(x, c, metric, 0)
    tc = gi().debug_dist_matrix(x, c, metric, 1)
    ref = ((x[:, None, :].astype(np.float64) - c[None].astype(np.float64)) ** 2).sum(-1) if metric == L2 \
        else x.astype(np.float64) @ c.astype(np.float64).T
    assert np.array_equal(exact.astype(np.float64), ref)
    assert np.array_equal(tc, exact)
    # float operands: error-compensated 3xTF32 stays within ~1e-6 of fp32 (north_star bar: 1e-4 relative)
    xf = synth.embed_like(n, d, seed=93) * 3.0
    cf = synth.embed_like(m, d, seed=94) * 3.0
    exact = gi().debug_dist_matrix(xf, cf, metric, 0)
    tc = gi().debug_dist_matrix(xf, cf, metric, 1)
    scale = np.abs(exact).max()
    assert np.abs(tc - exact).max() <= 2e-5 * scale


def test_request_coalescing_matches_direct_search(ivf_state, ivfflat_index):
    """Many concurrent nq=1..3 Search calls are merged into device batches by the index's worker
    thread (reference: gamma_index_ivfflat_gpu.cc:302-396); every caller must get exactly the rows
    a direct search returns."""
    import threading
    s = ivf_state
    xq = s["xq"]
    ref_d, ref_i = ivfflat_index.search(xq, 10, params={"nprobe": 8})  # nq = 48 > 16: not coalesced
    slices = [(i, min(i + 1 + (i % 3), len(xq))) for i in range(0, len(xq), 2)]
    out = {}
    errs = []

    def work(a, b):
        try:
            for _ in range(5):
                out[(a, b)] = ivfflat_index.search(xq[a:b], 10, params={"nprobe": 8})
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=ab) for ab in slices]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs
    for (a, b), (d, i) in out.items():
        assert np.array_equal(d, ref_d[a:b]) and np.array_equal(i, ref_i[a:b])
    # a different k / params must not be merged into the same batch
    d5, i5 = ivfflat_index.search(xq[:2], 5, params={"nprobe": 8})
    assert np.array_equal(d5, ref_d[:2, :5]) and np.array_equal(i5, ref_i[:2, :5])


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nlist,k,d,kernel", [
    (16, 10, 64, "ivf_listmajor_tma_kernel"),   # TMA-fed pipeline over the pre-tiled mirror
    (6, 10, 64, "ivf_listmajor_tma_kernel"),    # lists > 2048 rows: row segments
    (16, 10, 72, "ivf_listmajor_tma_kernel"),   # d not a multiple of the K chunk: zero-padded tail
    (16, 64, 64, "ivf_listmajor_pipe_kernel"),  # 32 < k <= 64: register-staged pipeline
    (16, 10, 16, "ivf_listmajor_pipe_kernel"),  # d <= 16: one K chunk of data, padded to two
    (16, 100, 64, "ivf_listmajor_tc_kernel+seg_select_kernel")])
def test_ivfflat_listmajor_tensor_core_scan_matches_oracle(metric, nlist, k, d, kernel):
    """Many queries per list => the list-major grouped-GEMM scan (kernels_tc.cu) is selected: fused
    top-k epilogue for k <= 64 (fed by TMA from the mirror for k <= 32 and d > 16, else the
    register-staged pipeline), dense score segments + segment select above.  Integer data: scores
    bit-equal to the oracle; filters and tombstones honoured."""
    n, nq, nprobe = 30000, 700, 6
    db = synth.sift_like(n, d, seed=95)
    xq = synth.sift_like(nq, d, seed=96)
    cent, _, _ = orc.kmeans(db[:4000], nlist, niter=5)
    cent = np.rint(cent).astype(np.float32)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": mt(metric)})
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids = idx.export_lists()
    vecs = codes.view(np.float32).reshape(len(ids), -1)[:, :d]
    cd, keys = orc.coarse_search(cent, xq, nprobe, metric)
    keys[5, 2] = -1  # "not enough centroids"
    deleted = np.random.default_rng(2).random(n) < 0.2
    delb = np.packbits(deleted, bitorder="little")
    idx.tombstone(int(np.searchsorted(off, 0, side="right") - 1), 0)
    ids2 = ids.copy()
    ids2[0] |= orc.DEL_MASK
    dg, ig = idx.search_preassigned(xq, k, keys, cd, del_bitmap=delb)
    assert idx.last_scan_kernel == kernel
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids2, xq, k, keys, metric, del_bitmap=delb)
    assert_same_results(dg, ig, do, io)
    lo, hi = float(min(do[0, 1], do[0, 6])), float(max(do[0, 1], do[0, 6]))
    dg, ig = idx.search_preassigned(xq, k, keys, cd, min_score=lo, max_score=hi)
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids2, xq, k, keys, metric, min_score=lo, max_score=hi)
    assert_same_results(dg, ig, do, io)
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d", [96, 200])
def test_ivfflat_listmajor_float_data_within_tolerance(metric, d):
    """General fp32 data (unit-norm embeddings, every mantissa bit in use): the error-compensated
    3xTF32 contraction must stay within 1e-5 relative of the fp32 oracle on inner products -- a
    tensor-core path that dropped or mis-rounded the low 13 mantissa bits would be off by ~5e-4.
    L2 goes through |x|^2 + |y|^2 - 2 x.y (as faiss's own blocked path does), so near neighbours of
    unit vectors lose digits to cancellation: the north-star tolerance 1e-4 applies there."""
    n, nlist, nq, nprobe, k = 20000, 8, 600, 4, 10
    db = synth.embed_like(n, d, seed=97, n_clusters=32)
    xq = synth.embed_like(nq, d, seed=98, n_clusters=32)
    cent, _, _ = orc.kmeans(db[:3000], nlist, niter=5)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": mt(metric)})
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids = idx.export_lists()
    vecs = codes.view(np.float32).reshape(len(ids), -1)[:, :d]
    cd, keys = orc.coarse_search(cent, xq, nprobe, metric)
    dg, ig = idx.search_preassigned(xq, k, keys, cd)
    assert idx.last_scan_kernel == "ivf_listmajor_tma_kernel"
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids, xq, k, keys, metric)
    assert_same_results(dg, ig, do, io, bit_exact=False, rtol=1e-5 if metric == IP else 1e-4)
    # the mirror follows the lists: vectors added after it was built are found by the next search
    more = synth.embed_like(300, d, seed=99, n_clusters=32)
    idx.add_vectors(more)
    idx.add_pending()
    dg2, ig2 = idx.search_preassigned(more[:40], 1, *reversed(orc.coarse_search(cent, more[:40], nlist, metric)))
    assert idx.last_scan_kernel == "ivf_listmajor_tma_kernel"
    assert np.array_equal(ig2[:, 0], n + np.arange(40))
    idx.close()


def test_ivf_lists_compaction_keeps_results(ivf_state):
    """Lists grown in many small steps leave dead regions behind; compact() re-packs them: same
    lists, same answers, less memory, and the index keeps accepting vectors afterwards."""
    s = ivf_state
    idx = gi().GammaIndex("IVFFLAT", s["d"], {"ncentroids": s["nlist"], "nprobe": 8, "metric_type": "L2"})
    idx.set_centroids(s["cent"])
    for a in range(0, 12000, 500):
        idx.add_vectors(s["db"][a:a + 500])
        idx.add_pending()
    before = idx.export_lists()
    ref = idx.search(s["xq"], 10, params={"nprobe": 8})
    mem0 = idx.mem_bytes(0)
    idx.compact()
    after = idx.export_lists()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert idx.mem_bytes(0) < mem0
    got = idx.search(s["xq"], 10, params={"nprobe": 8})
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    idx.add_vectors(s["db"][12000:13000])
    idx.add_pending()
    do, io = orc.flat_search(s["db"][:13000], s["db"][12500:12501], 1, L2)
    dg, ig = idx.search(s["db"][12500:12501], 1, params={"nprobe": s["nlist"]})
    assert ig[0, 0] == io[0, 0] == 12500 and dg[0, 0] == do[0, 0]
    idx.close()


def test_listmajor_mirror_survives_concurrent_adds_and_searches():
    """Big-batch searches (list-major, TMA kernel over the mirror) from two threads while a third
    keeps adding vectors: every search must see a consistent index (each probe vector finds itself),
    and the mirror is rebuilt behind the readers' backs without tearing."""
    import threading
    d, nlist, n0 = 64, 8, 8000
    db = synth.sift_like(n0 + 4000, d, seed=51)
    cent, _, _ = orc.kmeans(db[:3000], nlist, niter=4)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nlist, "metric_type": "L2"})
    idx.set_centroids(cent)
    idx.add_vectors(db[:n0])
    idx.add_pending()
    errs, stop = [], threading.Event()

    def searcher(seed):
        rng = np.random.default_rng(seed)
        try:
            while not stop.is_set():
                pick = rng.integers(0, n0, 300)
                dg, ig = idx.search(db[pick], 1, params={"nprobe": nlist})
                assert idx.last_scan_kernel.startswith("ivf_listmajor")
                ok = (dg[:, 0] == 0) & (np.all(db[ig[:, 0]] == db[pick], axis=1))
                assert ok.all()
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=searcher, args=(s,)) for s in (1, 2)]
    for t in ts:
        t.start()
    try:
        for a in range(n0, n0 + 4000, 250):
            idx.add_vectors(db[a:a + 250])
            idx.add_pending()
    finally:
        stop.set()
        for t in ts:
            t.join()
    assert not errs, errs[:1]
    dg, ig = idx.search(db[n0 + 3000:n0 + 3300], 1, params={"nprobe": nlist})
    assert np.all(dg[:, 0] == 0) and np.all(np.all(db[ig[:, 0]] == db[n0 + 3000:n0 + 3300], axis=1))
    idx.close()


def test_listmajor_mirror_is_updated_in_place_by_small_appends():
    """The pre-tiled mirror reserves 1/8 more rows per list: appends that fit go in place (no rebuild),
    and what they added is found by the next list-major search; outgrowing the reserve rebuilds once."""
    d, nlist, n0 = 64, 8, 16000
    db = synth.sift_like(n0 + 12000, d, seed=61)
    cent, _, _ = orc.kmeans(db[:3000], nlist, niter=4)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nlist, "metric_type": "L2"})
    idx.set_centroids(cent)
    idx.add_vectors(db[:n0])
    idx.add_pending()

    def finds_itself(a, b):
        dg, ig = idx.search(db[a:b], 1, params={"nprobe": nlist})
        assert idx.last_scan_kernel == "ivf_listmajor_tma_kernel"
        return bool(np.all(dg[:, 0] == 0) and np.all(np.all(db[ig[:, 0]] == db[a:b], axis=1)))

    assert finds_itself(0, 300) and idx.mirror_builds == 1
    for a in range(n0, n0 + 600, 200):  # 600 rows over 8 lists: well inside the reserve
        idx.add_vectors(db[a:a + 200])
        idx.add_pending()
        assert finds_itself(a, a + 200) and finds_itself(100, 400)
    assert idx.mirror_builds == 1
    idx.update_vector(5, db[n0 + 700])  # tombstone + re-append goes through the same path
    dg, ig = idx.search(np.repeat(db[n0 + 700:n0 + 701], 300, axis=0), 1, params={"nprobe": nlist})
    assert np.all(dg[:, 0] == 0) and idx.mirror_builds == 1
    idx.add_vectors(db[n0 + 600:n0 + 11000])  # far beyond the reserve
    idx.add_pending()
    assert finds_itself(n0 + 10000, n0 + 10300) and idx.mirror_builds == 2
    idx.close()


def test_ivfpq_opq_rotation_train_apply_search_and_file(tmp_path):
    """"opq": {"nsubvector": M} (gamma_index_ivfpq.cc:168-178, 362-364, 470, 585-590): an orthonormal rotation is
    learnt in front of the PQ, vectors and queries pass through it, the exact re-rank keeps using the raw
    vectors, and the rotation travels in the index file as the reference's "LTra" block."""
    import gamma_index_file as gif
    d, n, nlist, M = 32, 20000, 32, 8
    db = synth.sift_like(n, d, seed=83)
    xq = synth.sift_like(100, d, seed=84)
    base = {"ncentroids": nlist, "nprobe": 8, "nsubvector": M, "metric_type": "L2", "training_threshold": 8000}
    plain = gi().GammaIndex("IVFPQ", d, base)
    opq = gi().GammaIndex("IVFPQ", d, dict(base, opq={"nsubvector": M}))
    with pytest.raises(gi().GammaError):
        gi().GammaIndex("IVFPQ", d, dict(base, opq={"nsubvector": 5}))  # d % nsubvector != 0
    assert opq.has_opq and not plain.has_opq
    for idx in (plain, opq):
        idx.add_vectors(db)
        idx.train()
        idx.add_pending()
        assert idx.indexed_count == n
    A = opq.get_opq()
    assert np.allclose(A @ A.T, np.eye(d), atol=2e-5)  # orthonormal: distances are preserved
    xr = opq.apply_opq(xq)
    assert np.allclose(xr, xq @ A.T, rtol=1e-5, atol=1e-3)
    _, gt = orc.flat_search(db, xq, 1, L2)
    r_plain = recall_1nn(plain.search(xq, 10)[1], gt[:, 0], 10)
    r_opq = recall_1nn(opq.search(xq, 10)[1], gt[:, 0], 10)
    assert r_opq >= r_plain - 0.05 and r_opq >= 0.5  # the rotation must not hurt the ADC ranking
    dr, ir = opq.search(xq, 10, params={"recall_num": 100})
    assert np.array_equal(((xq[:, None, :] - db[ir]) ** 2).sum(-1), dr)  # re-rank: raw queries x raw vectors
    assert recall_1nn(ir, gt[:, 0], 10) >= 0.9
    # parity with the oracle on the device-built state: same rotated queries, same probes => same ADC results
    off, codes, ids = opq.export_lists()
    cent, pqc, T = opq.get_centroids(), opq.get_pq_centroids(), opq.get_precomputed_table()
    cd, keys = opq.coarse_search(xq, 8)  # coarse search happens on the rotated queries
    cdo, keyso = orc.coarse_search(cent, xr, 8, L2)
    assert np.array_equal(keys, keyso)
    dg, ig = opq.search_preassigned(xq, 50, keys, cd)
    do, io = orc.ivfpq_search_preassigned(off, codes, ids, cent, pqc, T, xr, 50, keys, cd, L2)
    assert_same_results(dg, ig, do, io)
    # index file: byte-identical to the independent writer, and it loads back with the rotation
    opq.dump(tmp_path, "emb.000")
    with open(tmp_path / "emb.000" / "ivfpq.index", "rb") as fh:
        assert fh.read() == gif.write_ivfpq(d, gif.METRIC_L2, 8, cent, pqc, off, codes, ids, n, opq=A)
    again = gi().GammaIndex("IVFPQ", d, dict(base, opq={"nsubvector": M}))
    again.add_vectors(db)
    assert again.load(tmp_path, "emb.000") == n and np.array_equal(again.get_opq(), A)
    d2, i2 = again.search_preassigned(xq, 50, keys, cd)
    assert np.array_equal(d2, dg) and np.array_equal(i2, ig)
    for idx in (plain, opq, again):
        idx.close()


# ----------------------------------------------------------------------------------------------
# BASELINE.json shapes (C2: IVF-Flat d=128 nlist=1024 nprobe=32; C3: IVF-PQ d=128 M=16 nlist=4096, re-rank 400)
# at database sizes the oracle finishes in seconds: same kernel instantiations as bench.py runs
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["query_major", "list_major"])
@pytest.mark.parametrize("data", ["int", "float"])
def test_baseline_shape_ivfflat_d128_nlist1024_nprobe32(path, data):
    d, n, nlist, nprobe, k = 128, 200_000, 1024, 32, 10
    nq = 1100 if path == "list_major" else 200  # >= 32 (query, probe) pairs per list selects the list-major scan
    if data == "int":
        db, xq = synth.sift_like(n, d, seed=301), synth.sift_like(nq, d, seed=302)
    else:
        db, xq = synth.sift_like(n, d, seed=303, rounded=False), synth.sift_like(nq, d, seed=304, rounded=False)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": "L2",
                                         "training_threshold": nlist * 39})
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    assert idx.indexed_count == n
    off, codes, ids = idx.export_lists()
    vecs = codes.view(np.float32).reshape(len(ids), -1)[:, :d]
    cd, keys = idx.coarse_search(xq, nprobe)
    dg, ig = idx.search_preassigned(xq, k, keys, cd)
    want = "ivf_listmajor_tma_kernel" if path == "list_major" else "ivfflat_scan_warp_kernel"
    assert idx.last_scan_kernel == want
    do, io = orc.ivfflat_search_preassigned(off, vecs, ids, xq, k, keys, L2)
    if data == "int":
        assert_same_results(dg, ig, do, io)  # bit-equal scores
    else:  # float data: summation order differs from the scalar loop (north-star tolerance 1e-4 relative)
        assert_same_results(dg, ig, do, io, bit_exact=False, rtol=1e-4)
    assert (ig == io).mean() >= 0.999
    # the end-to-end call (own coarse quantiser) returns the same thing
    d2, i2 = idx.search(xq, k)
    assert np.array_equal(i2, ig)
    idx.close()


@pytest.mark.parametrize("data", ["int", "float"])
def test_baseline_shape_ivfpq_d128_m16_nlist4096_rerank400(data):
    d, n, nlist, M, nprobe, k, recall_num = 128, 200_000, 4096, 16, 32, 10, 400
    nq = 4200  # nq * nprobe >= 32 * nlist: the tensor-core filter path of bench.py's default workload
    if data == "int":
        db, xq = synth.sift_like(n, d, seed=311), synth.sift_like(nq, d, seed=312)
    else:
        db, xq = synth.sift_like(n, d, seed=313, rounded=False), synth.sift_like(nq, d, seed=314, rounded=False)
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M, "metric_type": "L2",
                                       "training_threshold": nlist * 39})
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    off, codes, ids = idx.export_lists()
    cent, pqc, T = idx.get_centroids(), idx.get_pq_centroids(), idx.get_precomputed_table()
    assert np.array_equal(T, orc.ivfpq_precompute_table(cent, pqc))
    cd, keys = idx.coarse_search(xq, nprobe)
    # ADC stage at the re-rank depth: bit-equal scores, ids equal outside boundary ties
    dg, ig = idx.search_preassigned(xq, recall_num, keys, cd)
    assert idx.last_scan_kernel == "pqtc_scan_kernel"
    do, io = orc.ivfpq_search_preassigned(off, codes, ids, cent, pqc, T, xq, recall_num, keys, cd, L2)
    assert_same_results(dg, ig, do, io)
    # the same through the exact LUT kernel (small batch): identical answers
    d1, i1 = idx.search_preassigned(xq[:64], recall_num, keys[:64], cd[:64])
    assert idx.last_scan_kernel == "ivfpq_scan_kernel"
    assert np.array_equal(d1, dg[:64]) and np.array_equal(i1, ig[:64])
    # final answer with the exact re-rank (what bench.py times): exact L2 of the ADC candidates, best k
    dr, ir = idx.search_preassigned(xq, k, keys, cd, params={"recall_num": recall_num})
    agree = []
    for q in range(0, nq, 7):
        cand = io[q][io[q] >= 0]
        exact = ((xq[q].astype(np.float64) - db[cand]) ** 2).sum(1)
        order = np.lexsort((cand, exact))[:k]
        assert np.allclose(dr[q][: len(order)], exact[order], rtol=1e-5)
        agree.append(np.mean(ir[q][: len(order)] == cand[order]))
    assert np.mean(agree) >= 0.999
    idx.close()


def test_ivfpq_filter_follows_appends_and_codebook_changes():
    """The tensor-core filter streams a cached |r_e|^2 per list entry next to the codes.  The cache must follow the
    lists (vectors appended between two searches) and the codebook (set_pq_centroids): answers stay those of the oracle."""
    d, M, n, nq, nlist, nprobe, kk = 64, 8, 30000, 700, 16, 6, 50
    rng = np.random.default_rng(401)
    centers = rng.normal(0, 1, (32, d)).astype(np.float32)
    gen = lambda m: (centers[rng.integers(0, 32, m)] + 0.4 * rng.normal(0, 1, (m, d))).astype(np.float32)  # noqa: E731
    db, xq = gen(n), gen(nq)
    cent, _, _ = orc.kmeans(db[:4000], nlist, niter=5)
    a = orc.assign(cent, db, L2)
    pqc = orc.pq_train(db[:6000] - cent[a[:6000]], M, niter=4)
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M, "metric_type": "L2"})
    idx.set_centroids(cent)
    idx.set_pq_centroids(pqc)
    idx.add_vectors(db[:20000])
    idx.add_pending()
    T = orc.ivfpq_precompute_table(cent, pqc)
    cd, keys = orc.coarse_search(cent, xq, nprobe, L2)

    def check(pq_now, T_now):
        off, codes, ids = idx.export_lists()
        dg, ig = idx.search_preassigned(xq, kk, keys, cd)
        assert idx.last_scan_kernel == "pqtc_scan_kernel"
        do, io = orc.ivfpq_search_preassigned(off, codes, ids, cent, pq_now, T_now, xq, kk, keys, cd, L2)
        assert_same_results(dg, ig, do, io)

    check(pqc, T)
    idx.add_vectors(db[20000:])   # lists grow: the cache is rebuilt by the next search
    idx.add_pending()
    check(pqc, T)
    check(pqc, T)                 # and reused when nothing changed
    idx.close()


def test_ivfpq_filter_survives_concurrent_adds_and_searches():
    """Big-batch IVF-PQ searches (tensor-core filter, per-entry norm cache) from two threads while a third keeps adding
    vectors: every search sees a consistent index -- with exact re-rank each probe vector finds itself at distance 0 --
    and the norm cache is rebuilt between searches without tearing (appends drain in-flight searches first)."""
    import threading
    d, M, nlist, n0 = 64, 8, 8, 12000
    db = synth.sift_like(n0 + 4000, d, seed=61)
    # distinct rows only: a duplicate would make "finds itself" ambiguous
    db = np.unique(db, axis=0)
    n0 = min(n0, len(db) - 4000)
    cent, _, _ = orc.kmeans(db[:3000], nlist, niter=4)
    a = orc.assign(cent, db[:6000], L2)
    pqc = orc.pq_train(db[:6000] - cent[a], M, niter=4)
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nlist, "nsubvector": M, "metric_type": "L2"})
    idx.set_centroids(cent)
    idx.set_pq_centroids(pqc)
    idx.add_vectors(db[:n0])
    idx.add_pending()
    errs, stop = [], threading.Event()

    def searcher(seed):
        rng = np.random.default_rng(seed)
        try:
            while not stop.is_set():
                pick = rng.integers(0, n0, 400)
                dg, ig = idx.search(db[pick], 1, params={"nprobe": nlist, "recall_num": 100})
                assert idx.last_scan_kernel == "pqtc_scan_kernel"
                assert (dg[:, 0] == 0).all() and (ig[:, 0] == pick).all()
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=searcher, args=(s,)) for s in (1, 2)]
    for t in ts:
        t.start()
    try:
        for b in range(n0, n0 + 4000, 250):
            idx.add_vectors(db[b:b + 250])
            idx.add_pending()
    finally:
        stop.set()
        for t in ts:
            t.join()
    assert not errs, errs[:1]
    pick = np.arange(n0 + 3000, n0 + 3400)
    dg, ig = idx.search(db[pick], 1, params={"nprobe": nlist, "recall_num": 100})
    assert (dg[:, 0] == 0).all() and (ig[:, 0] == pick).all()
    idx.close()

