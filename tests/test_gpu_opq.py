"""OPQ on the H100, held to the restatement of tests/opq_reference.py (DESIGN.md §5, OPQ bar).

Every round of a traced OPQ training run (index.debug_opq_trace) is checked from the state the device reached: the
subsample, the column means, the centred rows, the random start, the projection, each subspace's k-means (the training
bar of tests/kmeans_reference.py), the codes, the reconstruction, X^T Y and the next rotation, which must be
orthonormal and Procrustes-optimal.  Then the rotation in use: every coordinate the device rotates, every list code,
searches key for key against the oracle on the device's rotated queries, the exact re-rank, and the trained state."""
import numpy as np
import pytest

import float_contract as fc
import kmeans_reference as kr
import opq_reference as orf
from oracle import oracle as orc
from oracle_pqnb import ivfpq_nbits as pqnb
from oracle_pqfs.twin import assert_same_results
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = fc.METRIC_L2, fc.METRIC_IP
F32 = np.float32


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


_open = []


@pytest.fixture(autouse=True)
def _close_indexes():
    """every index a test made is closed after it, whether it passed or not"""
    yield
    while _open:
        _open.pop().close()


def opened(idx):
    _open.append(idx)
    return idx


def traced(x, M, niter=2, check_kmeans=True):
    tr = gi().debug_opq_trace(x, M, niter=niter)
    orf.check_trace(x, M, tr, check_kmeans)
    return tr


# ---- every step of a round, across the data regimes -------------------------------------------------------------------
def regime_rows(name, n, d, seed=5):
    return fc.regime(name, n, d, 1, seed)[0]


def constant_dims(n, d, ncon, seed):
    x = synth.sift_like(n, d, seed=seed, rounded=False)
    cols = np.random.default_rng(seed).choice(d, ncon, replace=False)
    x[:, cols] = np.linspace(-3, 40, ncon, dtype=F32)[None, :]  # the centred column is exactly 0
    return x


def data(case, n, d):
    if case in ("sift_float", "offset1000", "scaled_hi", "scaled_lo", "near_dup"):
        return regime_rows(case, n, d)
    if case.startswith("const"):
        return constant_dims(n, d, int(case[5:]), 13)
    if case == "zero_tail":  # an embedding whose last 16 dimensions are 0
        x = synth.embed_like(n, d, seed=14)
        x[:, -16:] = 0
        return x
    if case == "few_distinct":  # fewer distinct rows than 256: every subspace k-means splits
        rng = np.random.default_rng(15)
        return rng.standard_normal((100, d)).astype(F32)[rng.integers(0, 100, n)]
    raise ValueError(case)


CASES = ["sift_float", "offset1000", "scaled_hi", "scaled_lo", "near_dup", "const1", "const8", "zero_tail",
         "few_distinct"]


@pytest.mark.parametrize("case", CASES)
def test_rounds(case):
    d, M = 64, 8
    x = data(case, 1200, d)
    tr = traced(x, M, niter=2)
    if case == "few_distinct":
        assert any(len(np.unique(lab)) < 256 for lab in tr["km"][0][0]["labels"])


@pytest.mark.parametrize("M", [3, 5, 15, 30])
def test_rounds_d30(M):
    """d = 30: subspace widths 10, 6, 2, 1, none a multiple of 4 (the slices are padded to it)"""
    traced(synth.sift_like(700, 30, seed=16, rounded=False), M, niter=2)


@pytest.mark.parametrize("n", [65535, 65536, 65537, 200000])
def test_subsample_edges(n):
    """around max_train_points: the subsample, mean, centring, projection, codes, reconstruction, X^T Y and rotation of
    a round; the per-iteration k-means check runs on the smaller cases above"""
    x = synth.sift_like(n, 8, seed=17, rounded=False)
    tr = traced(x, 2, niter=1, check_kmeans=False)
    assert len(tr["sample"]) == min(n, orf.MAX_TRAIN)


def test_below_256_rows_refused():
    """fewer rows than the 256 centroids of a subspace: the k-means refuses them, so training fails by name"""
    x = synth.sift_like(255, 16, seed=18, rounded=False)
    with pytest.raises(gi().GammaError, match="fewer training points than centroids"):
        gi().debug_opq_trace(x, 4, niter=1)
    idx = opened(gi().GammaIndex("IVFPQ", 16, {"ncentroids": 1, "nprobe": 1, "nsubvector": 4, "metric_type": "L2",
                                                "training_threshold": 255, "opq": {"nsubvector": 4}}))
    idx.add_vectors(x)
    with pytest.raises(gi().GammaError, match="fewer training points than centroids"):
        idx.train()
    assert not idx.is_trained


# ---- whole runs: 50 rounds, the rotation an index learns -------------------------------------------------------------
WHOLE = [("sift_float", 64, 8, 20000), ("const1", 64, 8, 20000), ("const8", 64, 16, 20000),
         ("zero_tail", 64, 8, 20000), ("sift_float", 128, 16, 70000), ("scaled_hi", 32, 4, 8000)]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("i", range(len(WHOLE)), ids=[f"{c}-d{d}-M{M}-n{n}" for c, d, M, n in WHOLE])
def test_whole_run_rotation(i, metric):
    """50 rounds: every round's rotation orthonormal and Procrustes-optimal, and the rotation an index trained on the
    same rows (with a different PQ nsubvector) holds is float32 of the last"""
    case, d, M, n = WHOLE[i]
    x = data(case, n, d)
    tr = gi().debug_opq_trace(x, M, niter=50, detail=False)
    orf.check_rotations(tr)
    nlist = max(16, -(-n // 256))
    idx = opened(gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": 4, "nsubvector": d // 4,
                                              "metric_type": mt(metric), "training_threshold": n,
                                              "opq": {"nsubvector": M}}))
    idx.add_vectors(x)
    idx.train()
    assert np.array_equal(kr.bits(idx.get_opq()), kr.bits(tr["r"][-1].astype(F32)))


# ---- the rotation in use ----------------------------------------------------------------------------------------------
def check_rotated(idx, x):
    """apply_opq(x) within ip_direct_margin of the fp64 A x, coordinate by coordinate; returns it"""
    A = idx.get_opq()
    xr = idx.apply_opq(x)
    r = orf.check_ip_product(xr, x, A, "rotated coordinate")
    assert r is None, r
    return xr


def check_lists(idx, x, nbits, metric):
    """each row is in the list the oracle assigns its rotated row to, and its code is the oracle's encoding of the
    rotated row's residual, byte for byte.  Returns (off, codes, ids) of the lists."""
    xr = check_rotated(idx, x)
    cent, pq = idx.get_centroids(), idx.get_pq_centroids()
    off, codes, ids = idx.export_lists()
    live = (ids & orc.DEL_MASK) == 0
    lst = np.repeat(np.arange(idx.nlist), np.diff(off))
    vid = ids & 0xFFFFFFFF
    assert np.array_equal(lst[live], orc.assign(cent, xr, metric)[vid[live]]), "list of a rotated row"
    enc = orc.ivfpq_encode if nbits == 8 else pqnb.ivfpq_encode
    want = enc(cent, pq, xr[vid[live]], lst[live])
    assert np.array_equal(codes[live], want), "list code of a rotated row"
    return off, codes, ids


def opq_index(d, M, nbits, metric, n, nlist=16, store_type=None, seed=31):
    x = synth.sift_like(n, d, seed=seed, rounded=False)
    p = {"ncentroids": nlist, "nprobe": 8, "nsubvector": d // 4, "nbits_per_idx": nbits, "metric_type": mt(metric),
         "training_threshold": 8000, "opq": {"nsubvector": M}}
    idx = opened(gi().GammaIndex("IVFPQ", d, p, store_type=store_type))
    idx.add_vectors(x)
    idx.train()
    idx.add_pending()
    return idx, x, p


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nbits", [8, 4, 7])
def test_codes_after_add_update_and_load(nbits, metric, tmp_path):
    d, M = 32, 8
    idx, x, p = opq_index(d, M, nbits, metric, 12000)
    check_lists(idx, x, nbits, metric)
    extra = synth.sift_like(3000, d, seed=32, rounded=False)
    for a in range(0, 3000, 700):  # adds after training, batch by batch
        idx.add_vectors(extra[a:a + 700])
        idx.add_pending()
    x = np.concatenate([x, extra])
    check_lists(idx, x, nbits, metric)
    for vid, src in ((5, 100), (12001, 7), (len(x) - 1, 0)):
        idx.update_vector(vid, x[src])
        x[vid] = x[src]
    check_lists(idx, x, nbits, metric)
    idx.dump(tmp_path, "emb.000")
    again = opened(gi().GammaIndex("IVFPQ", d, p))
    again.add_vectors(x)
    assert again.load(tmp_path, "emb.000") == len(x)
    assert np.array_equal(again.get_opq(), idx.get_opq())
    check_lists(again, x, nbits, metric)


def preassigned_ref(idx, xr, k, keys, cd, metric, nbits, **kw):
    off, codes, ids = idx.export_lists()
    cent, pq = idx.get_centroids(), idx.get_pq_centroids()
    T = idx.get_precomputed_table() if metric == L2 else None
    fn = orc.ivfpq_search_preassigned if nbits == 8 else pqnb.ivfpq_search_preassigned
    return fn(off, codes, ids, cent, pq, T, xr, k, keys, cd, metric, **kw)


SEARCH = [(8, 40, None), (4, 40, None), (7, 40, None), (8, 1100, None), (8, 40, "RocksDB"), (4, 40, "RocksDB")]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("i", range(len(SEARCH)), ids=[f"nbits{b}-nq{q}-{s or 'hbm'}" for b, q, s in SEARCH])
def test_search_key_exact(i, metric):
    """the device's rotated queries through the oracle's ADC scan on the device's lists give the device's results,
    score for score: query-major at nbits 8, packed nbits 4 and 7, the list-major tensor-core filter (a batch past its
    switch), and raw vectors in host memory"""
    nbits, nq, store = SEARCH[i]
    d, M = 32, 8
    idx, x, _ = opq_index(d, M, nbits, metric, 12000, store_type=store)
    xq = synth.sift_like(nq, d, seed=33, rounded=False)
    xr = check_rotated(idx, xq)
    cent = idx.get_centroids()
    for k, nprobe in ((10, 8), (100, 16)):
        cd, keys = orc.coarse_search(cent, xr, nprobe, metric)
        dg, ig = idx.search_preassigned(xq, k, keys, cd)
        if nq >= 1000:
            assert idx.last_scan_kernel == "pqtc_scan_kernel", idx.last_scan_kernel
        assert_same_results(dg, ig, *preassigned_ref(idx, xr, k, keys, cd, metric, nbits))
    # the whole search: the device's own coarse step, then the same scan.  Under IP the ADC score adds the query's
    # coarse dot, which search() takes from the tensor-core coarse quantiser (float contract, §5), so only L2 is exact
    cd, keys = idx.coarse_search(xq, 8)
    ck, ckeys = orc.coarse_search(cent, xr, 8, metric)
    assert np.array_equal(keys, ckeys)
    if metric == L2:
        dg, ig = idx.search(xq, 10)
        assert_same_results(dg, ig, *preassigned_ref(idx, xr, 10, keys, cd, metric, nbits))


@pytest.mark.parametrize("metric", [L2, IP])
def test_probe_groups(metric):
    """nprobe = nlist and a batch that splits each query's probes over groups (pg > 1): key-exact on rotated queries"""
    from test_gpu_probe_groups import nq_for, sm_count
    d, M, nlist = 32, 8, 64
    idx, x, _ = opq_index(d, M, 8, metric, 20000, nlist=nlist)
    nq = nq_for(2, nlist, sm_count())
    xq = synth.sift_like(nq, d, seed=34, rounded=False)
    xr = check_rotated(idx, xq)
    cd, keys = orc.coarse_search(idx.get_centroids(), xr, nlist, metric)
    dg, ig = idx.search_preassigned(xq, 10, keys, cd)
    assert_same_results(dg, ig, *preassigned_ref(idx, xr, 10, keys, cd, metric, 8))


@pytest.mark.parametrize("metric", [L2, IP])
def test_exact_rerank(metric):
    """recall_num: the best k of the device's ADC candidates by the raw query against the raw rows, within the float
    contract (the rotation never touches the re-rank)"""
    d, M, k, rn = 32, 8, 10, 60
    idx, x, _ = opq_index(d, M, 8, metric, 12000)
    xq = synth.sift_like(40, d, seed=35, rounded=False)
    cd, keys = idx.coarse_search(xq, 8)
    _, ic = idx.search_preassigned(xq, rn, keys, cd)
    got = idx.search_preassigned(xq, k, keys, cd, params={"recall_num": rn})

    def per_query(q):
        cand = ic[q][ic[q] >= 0]
        f, absdot = fc.scores64(xq[q:q + 1], x[cand], metric)
        m = fc.direct_margin(f[0], absdot[0], d, metric)
        return cand, f[0], m, m

    fc.check_all(got, per_query, k, metric, "opq re-rank")


# ---- trained state: the coarse quantiser and the codebook see the rotated rows -----------------------------------------
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nbits", [8, 4])
def test_trained_state(nbits, metric):
    import test_gpu_training as tg
    d, M, nlist = 32, 8, 16
    ksub = 1 << nbits
    x = synth.sift_like(256 * nlist + 100, d, seed=21, rounded=False)
    idx = opened(gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": 4, "nsubvector": d // 4,
                                              "nbits_per_idx": nbits, "metric_type": mt(metric),
                                              "opq": {"nsubvector": M}}))
    idx.add_vectors(x)
    t = idx.training_threshold
    idx.train()
    xt = idx.apply_opq(x[:t])  # the rotated training slab
    kp = dict(niter=10, spherical=metric == IP, l2_assign=False)
    cent = idx.get_centroids()
    assert np.array_equal(kr.bits(cent), kr.bits(tg.coarse_trace(xt, kp)))
    idx.add_pending()
    npq = min(t, 256 * ksub)
    rows = tg.codebook_rows(t, npq)
    lst = tg.vid_lists(idx)[rows]
    tg.check_codebook(idx, (xt[rows] - cent[lst]).astype(F32), ksub)
