"""OPQ at embedding dimensions (d 512 to 1024), held to the OPQ bar of DESIGN.md §5 (tests/opq_reference.py).

Each round's rotation is solved on the device (kernels_opq.cu): a one-sided Jacobi SVD of X^T Y in fp64 and R = V U^T.
These tests run traced rounds at d = 512, 768 and 1024 over SIFT-like rows and the rank-deficient regimes (constant
dimensions, a zero tail), a whole 50-round run at d = 768, an IVFPQ index trained with that rotation (codes, searches,
Dump / Load), and an engine table at d = 768 that becomes searchable once trained.  The per-subspace k-means, unchanged
by the device solver, is checked at small d by tests/test_gpu_opq.py; here the trace checks skip it to keep the run
short."""
import numpy as np
import pytest

import float_contract as fc
import kmeans_reference as kr
import opq_reference as orf
from oracle import oracle as orc
from oracle_pqfs.twin import assert_same_results
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2 = fc.METRIC_L2
F32 = np.float32


def gi():
    from vearch_b200 import index as gidx
    return gidx


def rows(case, n, d):
    """SIFT-like rows, or the rank-deficient regimes of tests/test_gpu_opq.py: 1 or 8 constant dimensions (a zero row
    of X^T Y each) and an embedding whose last 16 dimensions are 0"""
    if case == "sift_float":
        return fc.regime(case, n, d, 1, 5)[0]
    if case.startswith("const"):
        x = synth.sift_like(n, d, seed=13, rounded=False)
        ncon = int(case[5:])
        cols = np.random.default_rng(13).choice(d, ncon, replace=False)
        x[:, cols] = np.linspace(-3, 40, ncon, dtype=F32)[None, :]
        return x
    if case == "zero_tail":
        x = synth.embed_like(n, d, seed=14)
        x[:, -16:] = 0
        return x
    raise ValueError(case)


def converged(tr):
    """every round's SVD stopped on the off-diagonal test, not on the 60-sweep cap.  Only for full-rank X^T Y: columns
    of a vanishing singular value are rounding noise that every rotation re-mixes, so there the cap ends the run, as it
    does in jacobi_svd.h"""
    assert np.all(tr["sweeps"] >= 1) and np.all(tr["sweeps"] < 60), tr["sweeps"]


SHAPES = [(512, 64), (768, 96), (1024, 128)]


@pytest.mark.parametrize("case", ["sift_float", "const1", "const8", "zero_tail"])
@pytest.mark.parametrize("d,M", SHAPES, ids=[f"d{d}-M{M}" for d, M in SHAPES])
def test_rounds_large_d(d, M, case):
    x = rows(case, 2000, d)
    tr = gi().debug_opq_trace(x, M, niter=2)
    orf.check_trace(x, M, tr, check_kmeans=False)
    if case == "sift_float":
        converged(tr)


@pytest.mark.parametrize("case", ["sift_float", "const1"])
def test_rounds_odd_d(case):
    """an odd d leaves one column out of every step of the round-robin pairing"""
    x = rows(case, 700, 33)
    tr = gi().debug_opq_trace(x, 11, niter=2)
    orf.check_trace(x, 11, tr)
    if case == "sift_float":
        converged(tr)


# ---- d = 768: a whole training, and the index that holds its rotation -------------------------------------------------
D, M, N, NLIST = 768, 96, 20000, 80  # 256 NLIST >= N: the index trains on every row, as the trace does


@pytest.fixture(scope="module")
def whole():
    x = synth.sift_like(N, D, seed=41, rounded=False)
    tr = gi().debug_opq_trace(x, M, niter=50, detail=False)
    return x, tr


@pytest.fixture(scope="module")
def table(whole):
    x, _ = whole
    p = {"ncentroids": NLIST, "nprobe": 16, "nsubvector": M, "metric_type": "L2", "training_threshold": N,
         "opq": {"nsubvector": M}}
    idx = gi().GammaIndex("IVFPQ", D, p)
    idx.add_vectors(x)
    idx.train()
    idx.add_pending()
    yield idx, p
    idx.close()


def test_whole_run_d768(whole):
    _, tr = whole
    orf.check_rotations(tr)
    converged(tr)


def test_index_rotation_is_the_trained_one(whole, table):
    _, tr = whole
    idx, _ = table
    assert np.array_equal(kr.bits(idx.get_opq()), kr.bits(tr["r"][-1].astype(F32)))


def check_lists(idx, x):
    """every live entry in the oracle's list of its rotated row, coded as the oracle codes it; returns the lists"""
    A = idx.get_opq()
    xr = idx.apply_opq(x)
    r = orf.check_ip_product(xr, x, A, "rotated coordinate")
    assert r is None, r
    cent, pq = idx.get_centroids(), idx.get_pq_centroids()
    off, codes, ids = idx.export_lists()
    live = (ids & orc.DEL_MASK) == 0
    lst = np.repeat(np.arange(idx.nlist), np.diff(off))
    vid = ids & 0xFFFFFFFF
    assert np.array_equal(lst[live], orc.assign(cent, xr, L2)[vid[live]]), "list of a rotated row"
    assert np.array_equal(codes[live], orc.ivfpq_encode(cent, pq, xr[vid[live]], lst[live])), "list code"
    return off, codes, ids


def test_list_codes(whole, table):
    x, _ = whole
    idx, _ = table
    check_lists(idx, x)


def test_search_key_exact(table):
    idx, _ = table
    xq = synth.sift_like(64, D, seed=42, rounded=False)
    xr = idx.apply_opq(xq)
    cent, pq = idx.get_centroids(), idx.get_pq_centroids()
    off, codes, ids = idx.export_lists()
    T = idx.get_precomputed_table()
    for k, nprobe in ((10, 8), (100, 16)):
        cd, keys = orc.coarse_search(cent, xr, nprobe, L2)
        dg, ig = idx.search_preassigned(xq, k, keys, cd)
        assert_same_results(dg, ig, *orc.ivfpq_search_preassigned(off, codes, ids, cent, pq, T, xr, k, keys, cd, L2))
    cd, keys = idx.coarse_search(xq, 16)
    assert np.array_equal(keys, orc.coarse_search(cent, xr, 16, L2)[1])
    dg, ig = idx.search(xq, 10)
    assert_same_results(dg, ig, *orc.ivfpq_search_preassigned(off, codes, ids, cent, pq, T, xr, 10, keys, cd, L2))


def test_search_recall_num(whole, table):
    """recall_num: the ADC candidates are the oracle's, key for key, and the best k of them by the raw query against
    the raw rows meet the float contract"""
    x, _ = whole
    idx, _ = table
    rn, k = 60, 10
    xq = synth.sift_like(32, D, seed=43, rounded=False)
    xr = idx.apply_opq(xq)
    cent, pq = idx.get_centroids(), idx.get_pq_centroids()
    off, codes, ids = idx.export_lists()
    cd, keys = orc.coarse_search(cent, xr, 16, L2)
    dc, ic = idx.search_preassigned(xq, rn, keys, cd)
    assert_same_results(dc, ic, *orc.ivfpq_search_preassigned(off, codes, ids, cent, pq, idx.get_precomputed_table(),
                                                              xr, rn, keys, cd, L2))
    got = idx.search_preassigned(xq, k, keys, cd, params={"recall_num": rn})

    def per_query(q):
        cand = ic[q][ic[q] >= 0]
        f, absdot = fc.scores64(xq[q:q + 1], x[cand], L2)
        m = fc.direct_margin(f[0], absdot[0], D, L2)
        return cand, f[0], m, m

    fc.check_all(got, per_query, k, L2, "opq re-rank at d 768")


def test_dump_load(whole, table, tmp_path):
    x, _ = whole
    idx, p = table
    idx.dump(tmp_path, "emb.000")
    again = gi().GammaIndex("IVFPQ", D, p)
    try:
        again.add_vectors(x)
        assert again.load(tmp_path, "emb.000") == N
        assert np.array_equal(kr.bits(again.get_opq()), kr.bits(idx.get_opq()))
        want = idx.export_lists()
        got = check_lists(again, x)
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
    finally:
        again.close()


def test_engine_table_d768_becomes_searchable(tmp_path, whole):
    """CreateTable with "opq" at d 768, adds past training_threshold: the table trains in the background and then
    answers searches through the index (before training, past 100 documents, it refuses them as not trained)"""
    from vearch_b200 import engine
    x, _ = whole
    n = 8000
    db = x[:n]
    e = engine.GammaEngine(str(tmp_path), space_name="opq")
    try:
        e.create_table("opq", D, "IVFPQ", {"ncentroids": 16, "nprobe": 16, "nsubvector": M, "metric_type": "L2",
                                           "training_threshold": n, "opq": {"nsubvector": M}})
        for i in range(200):
            assert e.add_doc(f"doc{i}", db[i]) == 0
        with pytest.raises(engine.GammaStatusError) as ei:
            e.search(db[:4], 10)
        assert ei.value.code == 2
        for i in range(200, n):
            assert e.add_doc(f"doc{i}", db[i]) == 0
        e.wait_indexed(n, timeout=600)
        xq = db[:32]
        res = e.search(xq, 10, index_params={"nprobe": 16})
        got = [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]
        assert all(len(g) == 10 for g in got)
        _, gt = orc.flat_search(db, xq, 1, L2)
        assert np.mean([f"doc{gt[q, 0]}" in got[q] for q in range(len(xq))]) >= 0.9
    finally:
        e.close()
