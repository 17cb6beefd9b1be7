"""GPU_IVFPQ and GPU_IVFFLAT, gamma's two GPU index types (index/impl/gpu/): IVFPQ and IVFFLAT created under the
reference's GPU parameter contract (IVFPQGPUModelParams, IVFFlatGPUModelParams) and searched under its GPU request
contract (CommonSearch, gamma_gpu_search_base.h): at most 512 queries and k' = max(k, recall_num) <= 2048 per call, no
exact re-rank, a request nprobe outside (0, min(nlist, 2048)] falls back to the model's.  The index behind each is the
engine's IVFPQ / IVFFLAT, so its results are checked key-exact against the same references (test_gpu_topk_keys.py) and
against the CPU type built from the same trained state.  The deliberate deviations of DESIGN.md section 8 (filters
before selection, Delete / Update act on the index, Dump writes gamma's index file) are tested in the engine flow."""
import struct

import numpy as np
import pytest

import test_gpu_topk_keys as T
import topk_reference as R
from oracle import oracle as orc
from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
L2, IP = R.METRIC_L2, R.METRIC_IP
D, N, NQ = 32, 3000, 24


def gi():
    from vearch_b200 import index as gidx
    return gidx


def eng_mod():
    from vearch_b200 import engine
    return engine


def create_error(path, index_type, params, d=D):
    """CreateTable of a one-field table: the engine's status code and the message after the code's name"""
    E = eng_mod()
    e = E.GammaEngine(str(path))
    try:
        with pytest.raises(E.GammaStatusError) as ei:
            e.create_table("t", d, index_type, params)
    finally:
        e.close()
    return ei.value.code, ei.value.msg.split(": ", 1)[1]


# ---- parameters ---------------------------------------------------------------------------------------------------
GPU_IVFPQ_REFUSED = [  # IVFPQGPUModelParams::Parse / Validate, GammaIVFPQGPUIndex::Init, in that order
    ({"ncentroids": 0}, "invalid ncentroids =0"),
    ({"ncentroids": -3, "nsubvector": 0}, "invalid ncentroids =-3"),
    ({"nsubvector": 0}, "invalid nsubvector =0"),
    ({"nsubvector": -1, "nbits_per_idx": 0}, "invalid nsubvector =-1"),
    ({"nsubvector": 8, "nbits_per_idx": 0}, "invalid nbits_per_idx =0"),
    ({"nsubvector": 8, "nprobe": 0}, "invalid nprobe =0"),
    ({"nsubvector": 8, "nprobe": -1}, "invalid nprobe =-1"),
    ({"nsubvector": 8, "ncentroids": 8, "nprobe": 32}, "nprobe should less than ncentroids"),
    ({"nsubvector": 2, "nbits_per_idx": 4, "metric_type": "cosine"}, "invalid metric_type = cosine"),
    ({"nsubvector": 2, "nbits_per_idx": 4}, "only support multiple of 4 now, nsubvector=2"),
    ({"nsubvector": 8, "nbits_per_idx": 4}, "only support 8 now, nbits_per_idx=4"),
    ({"nsubvector": 8, "nbits_per_idx": 16}, "only support 8 now, nbits_per_idx=16"),
    ({"nsubvector": 12}, "Dimension [32] cannot divide by nsubvector [12]."),
    ({}, "Dimension [32] cannot divide by nsubvector [64]."),  # the default nsubvector is 64, not d / 2
]
GPU_IVFFLAT_REFUSED = [  # IVFFlatGPUModelParams::Validate
    {"ncentroids": 0}, {"ncentroids": -1}, {"nprobe": 0}, {"nprobe": -2}, {"bucket_init_size": 0},
    {"bucket_max_size": -5}, {"bucket_init_size": 2000, "bucket_max_size": 1000},
]


@pytest.mark.parametrize("params,msg", GPU_IVFPQ_REFUSED)
def test_gpu_ivfpq_parameter_refusals(tmp_path, params, msg):
    code, got = create_error(tmp_path, "GPU_IVFPQ", params)
    assert code == 4 and got == msg
    with pytest.raises(gi().GammaError) as ei:
        gi().GammaIndex("GPU_IVFPQ", D, params)
    assert ei.value.args[0].endswith(msg)


def test_gpu_ivfflat_parameter_refusals(tmp_path):
    for params in GPU_IVFFLAT_REFUSED:
        assert create_error(tmp_path, "GPU_IVFFLAT", params) == (4, "Invalid parameters"), params
    from vearch_b200 import _lib
    assert not _lib.lib().gb_index_create(b"GPU_IVFFLAT", D, b"{not json", 0)
    assert _lib.last_error() == "Parse model parameters error"
    assert not _lib.lib().gb_index_create(b"GPU_IVFPQ", D, b"{not json", 0)
    assert _lib.last_error() == "failed to parse IVFPQ retrieval parameters"


def test_defaults_and_accepted_parameters(tmp_path):
    # GPU_IVFPQ: nsubvector 64, nbits 8, ncentroids 2048, training threshold ncentroids * 256
    idx = gi().GammaIndex("GPU_IVFPQ", 128, {})
    assert idx.type == "GPU_IVFPQ" and idx.pq_m == 64 and idx.pq_ksub == 256 and idx.nlist == 2048
    assert idx.training_threshold == 2048 * 256
    idx.close()
    code, msg = create_error(tmp_path, "GPU_IVFPQ", {}, d=96)
    assert code == 4 and msg == "Dimension [96] cannot divide by nsubvector [64]."
    idx = gi().GammaIndex("GPU_IVFPQ", 32, {"ncentroids": 16, "nsubvector": 8})
    assert idx.pq_m == 8 and idx.training_threshold == 16 * 256
    idx.close()
    # the query-major scan must select k' = 2048 beside the [M][256] table: nsubvector 128 is, 200 is refused
    gi().GammaIndex("GPU_IVFPQ", 256, {"ncentroids": 16, "nprobe": 4, "nsubvector": 128}).close()
    code, msg = create_error(tmp_path, "GPU_IVFPQ", {"ncentroids": 16, "nprobe": 4, "nsubvector": 200}, d=400)
    assert code == 4 and "nsubvector [200]" in msg
    # GPU_IVFFLAT: nprobe > ncentroids is accepted, an unknown metric_type is ignored (InnerProduct stays)
    idx = gi().GammaIndex("GPU_IVFFLAT", D, {"ncentroids": 8, "nprobe": 32, "metric_type": "cosine"})
    assert idx.type == "GPU_IVFFLAT" and idx.nlist == 8 and idx.training_threshold == 8 * 256
    db, xq = synth.sift_like(4000, D, seed=3), synth.sift_like(8, D, seed=4)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    d_ip, i_ip = orc.flat_search(db, xq, 10, orc.METRIC_IP)
    dg, ig = idx.search(xq, 10)  # nprobe 32 > nlist 8: every list, so exact
    assert np.array_equal(ig, i_ip) and np.allclose(dg, d_ip, rtol=1e-5)
    idx.close()
    gi().GammaIndex("GPU_IVFFLAT", D, {}).close()


# ---- results against the references -------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", T.METRICS)
def test_gpu_ivfpq_query_major_is_key_exact(metric):
    """the default M = 64 has no tensor-core filter shape: every batch scans query-major"""
    d, M, n, nq, nlist, nprobe = 128, 64, 20000, 6, 64, 40
    db, xq = T.make_data("sift", n, d, nq, metric, seed=M)
    st = T.PqState("GPU_IVFPQ", d, M, 8, nlist, metric, db, xq, seed=3)
    assert st.idx.type == "GPU_IVFPQ"
    probes = st.probes(nprobe)
    for k in (1, 16, 400, 1024, 2048):
        T.assert_results(st.search(probes, k), st.ref(probes, k), metric, f"GPU_IVFPQ k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_scan_kernel"
    # no re-rank: recall_num 400 returns the ADC results of recall_num 0
    base = st.search(probes, 10)
    T.assert_results(base, st.ref(probes, 10), metric, "GPU_IVFPQ k=10")
    got = st.search(probes, 10, params={"recall_num": 400})
    assert np.array_equal(got[1], base[1]) and np.array_equal(got[0].view(np.uint32), base[0].view(np.uint32))
    # deletions, bitmaps and the score window apply before selection
    sc = R.decode(st.ref(probes, 100), metric)[0][0]
    for name, kw in T.filter_cases(n, 100, sc, metric, seed=M):
        T.assert_results(st.search(probes, 100, **kw), st.ref(probes, 100, **kw), metric, f"GPU_IVFPQ {name}")
    st.idx.close()


@pytest.mark.parametrize("metric", T.METRICS)
def test_gpu_ivfpq_list_major_is_key_exact(metric):
    d, M, n, nq, nlist, nprobe = 128, 16, 20000, 128, 16, 6
    db, xq = T.make_data("sift", n, d, nq, metric, seed=7)
    st = T.PqState("GPU_IVFPQ", d, M, 8, nlist, metric, db, xq, seed=6)
    probes = st.probes(nprobe)
    for k in (10, 257, 2048):
        T.assert_results(st.search(probes, k), st.ref(probes, k), metric, f"GPU_IVFPQ list-major k'={k}")
        assert st.idx.last_scan_kernel == "pqtc_scan_kernel"
    got = st.search(probes, 10, params={"recall_num": 400})
    T.assert_results(got, st.ref(probes, 10), metric, "GPU_IVFPQ list-major recall_num 400")
    st.idx.close()


@pytest.mark.parametrize("metric", T.METRICS)
def test_gpu_ivfflat_equals_ivfflat(metric):
    d, n, nlist, nprobe = 64, 20000, 32, 8
    db = synth.sift_like(n, d, seed=11)
    cent = T.pick_centroids(db, nlist, seed=2)
    idx = {}
    for typ in ("IVFFLAT", "GPU_IVFFLAT"):
        idx[typ] = gi().GammaIndex(typ, d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": T.mt(metric)})
        idx[typ].set_centroids(cent)
        idx[typ].add_vectors(db)
        idx[typ].add_pending()
    for nq, ks in ((6, (1, 100, 2048)), (256, (10, 64, 1024))):  # query-major, then the list-major kernels
        xq = synth.sift_like(nq, d, seed=nq)
        for k in ks:
            a, b = idx["IVFFLAT"].search(xq, k), idx["GPU_IVFFLAT"].search(xq, k)
            assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)), (nq, k)
            assert idx["IVFFLAT"].last_scan_kernel == idx["GPU_IVFFLAT"].last_scan_kernel
    for i in idx.values():
        i.close()


# ---- request limits -----------------------------------------------------------------------------------------------
def test_request_limits():
    d, n = 32, 6000
    db = synth.sift_like(n, d, seed=21)
    xq = synth.sift_like(513, d, seed=22)
    for typ, extra in (("GPU_IVFPQ", {"nsubvector": 8}), ("GPU_IVFFLAT", {})):
        idx = gi().GammaIndex(typ, d, dict(extra, ncentroids=16, nprobe=16, metric_type="L2"))
        idx.set_centroids(T.pick_centroids(db, 16, seed=1))
        if typ == "GPU_IVFPQ":
            idx.set_pq_centroids(np.random.default_rng(0).normal(0, 8, (8, 256, 4)).astype(np.float32))
        idx.add_vectors(db)
        idx.add_pending()
        dg, ig = idx.search(xq[:512], 2048)  # the largest call the type serves
        assert ig.shape == (512, 2048) and (ig >= 0).all()
        with pytest.raises(gi().GammaError, match=r"req num \[513\] should not larger than \[512\]"):
            idx.search(xq, 10)
        with pytest.raises(gi().GammaError, match=r"topK num \[2049\] should not larger than \[2048\]"):
            idx.search(xq[:2], 2049)
        if typ == "GPU_IVFPQ":  # k' = max(k, recall_num)
            with pytest.raises(gi().GammaError, match=r"topK num \[2049\] should not larger than \[2048\]"):
                idx.search(xq[:2], 10, params={"recall_num": 2049})
            assert np.array_equal(idx.search(xq[:4], 10, params={"recall_num": 2048})[1], idx.search(xq[:4], 10)[1])
        else:  # GPU_IVFFLAT's recall number is always k
            assert np.array_equal(idx.search(xq[:4], 10, params={"recall_num": 4096})[1], idx.search(xq[:4], 10)[1])
        idx.close()


@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
def test_request_nprobe_fallback(typ):
    """a request nprobe of 0, above nlist or above 2048 searches with the model's nprobe"""
    d, n, nlist = 32, 20000, 4096
    db = synth.sift_like(n, d, seed=31)
    xq = synth.sift_like(16, d, seed=32)
    params = {"ncentroids": nlist, "nprobe": 1, "metric_type": "L2"}  # ~5 entries per list: fewer than k at nprobe 1
    if typ == "GPU_IVFPQ":
        params["nsubvector"] = 8
    idx = gi().GammaIndex(typ, d, params)
    idx.set_centroids(T.pick_centroids(db, nlist, seed=3))
    if typ == "GPU_IVFPQ":
        idx.set_pq_centroids(np.random.default_rng(1).normal(0, 8, (8, 256, 4)).astype(np.float32))
    idx.add_vectors(db)
    idx.add_pending()
    base = idx.search(xq, 10)
    for nprobe in (0, -1, nlist + 1, 3000, 2049):
        got = idx.search(xq, 10, params={"nprobe": nprobe})
        assert np.array_equal(got[1], base[1]) and np.array_equal(got[0], base[0]), nprobe
    assert (base[1] < 0).any() and (idx.search(xq, 10, params={"nprobe": 2048})[1] >= 0).all()  # in range: honoured
    idx.close()


# ---- engine -------------------------------------------------------------------------------------------------------
ENGINE_PARAMS = {
    "GPU_IVFPQ": {"ncentroids": 16, "nprobe": 16, "nsubvector": 8, "metric_type": "L2", "training_threshold": 1000},
    "GPU_IVFFLAT": {"ncentroids": 16, "nprobe": 16, "metric_type": "L2", "training_threshold": 1000},
}


def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def scores_of(res):
    return [[it["score"] for it in r["items"]] for r in res]


def make_engine(path, typ):
    e = eng_mod().GammaEngine(str(path), space_name="ts")
    e.create_table("ts", D, typ, ENGINE_PARAMS[typ],
                   fields=(("_id", wire.DT_STRING, False), ("price", wire.DT_INT, True), ("tag", wire.DT_STRING, True)))
    return e


@pytest.mark.parametrize("typ", ["GPU_IVFPQ", "GPU_IVFFLAT"])
def test_engine_flow(tmp_path, typ):
    db, xq = synth.sift_like(N, D, seed=41), synth.sift_like(NQ, D, seed=42)
    price = (np.arange(N) * 37) % 1000
    e = make_engine(tmp_path, typ)
    i32 = lambda v: struct.pack("<i", v)
    for i in range(N):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("price", i32(int(price[i])), wire.DT_INT),
                                                         ("tag", f"t{i % 7}".encode(), wire.DT_STRING)]) == 0
    st = e.wait_indexed(N)
    assert st["index_status"] == 2 and st["doc_num"] == N
    assert e.memory_info()["index_mem"] > 0
    exact = typ == "GPU_IVFFLAT"  # nprobe == nlist: IVF-Flat is exact; IVF-PQ returns ADC distances
    res = e.search(xq, 10)
    _, gt = orc.flat_search(db, xq, 10, L2)
    if exact:
        assert keys_of(res) == [[f"doc{i}" for i in row] for row in gt]
    else:
        assert np.mean([f"doc{gt[q, 0]}" in keys_of(res)[q] for q in range(NQ)]) >= 0.9
    # range / term filters apply before selection: k results whenever k documents pass (the reference keeps only the
    # survivors among recall_num unfiltered candidates)
    sel = (price < 40) & (np.arange(N) % 7 == 3)  # 0.6 % of the documents
    kw = dict(range_filters=[("price", b"", i32(40), False, False)], term_filters=[("tag", b"t3")])
    res = e.search(xq, 10, **kw)
    assert all(len(r) == 10 and all(sel[int(k[3:])] for k in r) for r in keys_of(res))
    if exact:
        _, io = orc.flat_search(db, xq, 10, L2, filter_bitmap=np.packbits(sel, bitorder="little"))
        assert keys_of(res) == [[f"doc{i}" for i in row] for row in io]
    # Delete drops the entry; Update moves it (the reference's GPU index keeps serving the stale vector)
    victim = keys_of(e.search(xq[:1], 1))[0][0]
    assert e.delete_doc(victim) == 0
    assert victim not in keys_of(e.search(xq[:1], 10))[0]
    top = 1 if exact else 10  # a query equal to a stored vector finds it first (IVF-Flat) or among the ADC top 10
    assert "doc7" in keys_of(e.search(db[7:8], top))[0]
    assert e.add_doc("doc7", xq[3], extra_fields=[("price", i32(7), wire.DT_INT), ("tag", b"t0", wire.DT_STRING)]) == 0
    assert "doc7" in keys_of(e.search(xq[3:4], top))[0]
    assert "doc7" not in keys_of(e.search(db[7:8], 10))[0]
    # requests above the GPU limits are invalid arguments
    with pytest.raises(eng_mod().GammaStatusError) as ei:
        e.search(xq[:1], 2049)
    assert ei.value.code == 4 and "topK num [2049] should not larger than [2048]" in ei.value.msg
    # Dump writes gamma's index file of the CPU type; Load repeats every search exactly
    queries = [dict(), dict(index_params={"nprobe": 4}), kw]
    before = [e.search(xq, 10, **q) for q in queries]
    assert e.dump() == 0
    e.close()
    fname = "ivfpq.index" if typ == "GPU_IVFPQ" else "ivfflat.index"
    assert (tmp_path / "retrieval_model_index" / "emb.000" / fname).exists()
    e2 = make_engine(tmp_path, typ)
    assert e2.load() == 0
    e2.wait_indexed(N)
    after = [e2.search(xq, 10, **q) for q in queries]
    for a, b in zip(after, before):
        assert keys_of(a) == keys_of(b) and scores_of(a) == scores_of(b)
    assert e2.get_doc_by_id(victim)[0] == -1
    e2.close()


def test_multi_vector_table_with_a_gpu_ivfpq_field(tmp_path):
    n, d2, topn = 2500, 16, 60
    db, xq = synth.sift_like(n, D, seed=51), synth.sift_like(NQ, D, seed=52)
    img, imq = synth.sift_like(n, d2, seed=53), synth.sift_like(NQ, d2, seed=54)
    e = eng_mod().GammaEngine(str(tmp_path), space_name="ts")
    e.create_table("ts", D, "GPU_IVFFLAT", ENGINE_PARAMS["GPU_IVFFLAT"],
                   extra_vectors=[("img", d2, "GPU_IVFPQ", {"ncentroids": 16, "nprobe": 16, "nsubvector": 4,
                                                            "metric_type": "L2"})])
    for i in range(n):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("img", img[i].tobytes(), wire.DT_VECTOR)]) == 0
    assert e.wait_indexed(n)["index_status"] == 2
    res = e.search(xq, topn, extra_vec_queries=[("img", imq)], multi_vector_rank=1)
    _, g1 = orc.flat_search(db, xq, topn, L2)
    _, g2 = orc.flat_search(img, imq, topn, L2)
    joined = [set(a) & set(b) for a, b in zip(g1.tolist(), g2.tolist())]
    got = [set(int(k[3:]) for k in row) for row in keys_of(res)]
    assert sum(len(g) for g in got) > NQ  # the join is not empty
    assert np.mean([len(g & j) / max(1, len(j)) for g, j in zip(got, joined)]) >= 0.8
    e.close()
