"""Search cancellation on the H100 (DESIGN.md section 8, cancellation): a search given a set cancel token stops early,
raises the kill error (-2), and leaves its index exactly as a normal search does; a token that is never set changes no
result.  The per-kernel skip counters (gb_debug_cancel_stats) prove that the kernel each path names in
last_scan_kernel skipped its work, without timing anything."""
import threading
import time

import numpy as np
import pytest

from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu

D, N, NLIST, K = 64, 20000, 32, 10


def gi():
    from vearch_b200 import index
    return index


# last_scan_kernel labels -> the polling kernel behind each part (the query-major codecs share list_scan_kernel)
LIST_SCAN_LABELS = ("ivfpq_scan_kernel", "ivfpq_packed_scan_kernel", "ivfpqfs_scan_kernel", "rabitq_scan_kernel",
                    "vearch_scan_kernel", "binary_ivf_scan_kernel")


def polled_sites(label):
    out = []
    for part in label.split("+"):
        if part in LIST_SCAN_LABELS:
            out.append("list_scan_kernel")
        elif part != "ivf_listmajor_tc_kernel":  # its seg_select_kernel polls
            out.append(part)
    return out


@pytest.fixture(scope="module")
def data():
    return synth.sift_like(N, D, seed=501), synth.sift_like(256, D, seed=502)


def binary_rows(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, D // 8), dtype=np.uint8)


def build(kind, db):
    """(index, queries-of-the-right-kind selector, extra search kwargs) of one path"""
    g = gi()
    ivf = {"ncentroids": NLIST, "nprobe": 8, "metric_type": "L2", "training_threshold": 8000}
    if kind == "binaryivf":
        idx = g.BinaryIVFIndex(D, {"ncentroids": NLIST, "nprobe": 8, "training_threshold": 8000})
        idx.add_vectors(binary_rows(N, 7))
    elif kind in ("flat", "flat_host"):
        idx = g.GammaIndex("FLAT", D, {"metric_type": "L2"}, store_type="RocksDB" if kind == "flat_host" else None)
        idx.add_vectors(db)
        return idx
    elif kind.startswith("ivfflat"):
        idx = g.GammaIndex("IVFFLAT", D, ivf)
        idx.add_vectors(db)
    elif kind in ("ivfpq", "ivfpq_pqtc", "rerank2", "rerank1"):
        idx = g.GammaIndex("IVFPQ", D, dict(ivf, nsubvector=16),
                           store_type="RocksDB" if kind == "rerank1" else None)
        idx.add_vectors(db)
    elif kind == "ivfpq_nb4":
        idx = g.GammaIndex("IVFPQ", D, dict(ivf, nsubvector=16, nbits_per_idx=4))
        idx.add_vectors(db)
    elif kind in ("pqfs", "soar"):
        p = dict(ivf, nsubvector=16)
        if kind == "soar":
            p["soar_lambda"] = 1.0
        idx = g.GammaIndex("IVFPQFastScan", D, p)
        idx.add_vectors(db)
    elif kind == "rabitq":
        idx = g.RaBitQIndex(D, dict(ivf, nb_bits=2))
        idx.add_vectors(db)
    elif kind == "vearch":
        idx = g.VearchIndex(D, dict(ivf, nsubvector=16))
        idx.add_vectors(db)
    elif kind == "sharded":
        idx = g.GammaIndex("GPU_IVFPQ", D, dict(ivf, nsubvector=16), devices=[0, 0])
        idx.add_vectors(db)
    else:
        raise AssertionError(kind)
    idx.train()
    idx.add_pending()
    return idx


# path -> (build kind, queries used, retrieval params, the label's expected prefix)
PATHS = {
    "flat_hbm": ("flat", 16, None, "dist_tile_kernel"),
    "flat_host": ("flat_host", 16, None, "dist_tile_kernel"),
    "ivfflat_query_major": ("ivfflat", 16, None, "ivfflat_scan"),
    "ivfflat_list_major": ("ivfflat", 256, None, "ivf_listmajor"),
    "ivfpq_query_major": ("ivfpq", 16, None, "ivfpq_scan_kernel"),
    "ivfpq_pqtc": ("ivfpq_pqtc", 256, None, "pqtc_scan_kernel"),
    "ivfpq_nbits4": ("ivfpq_nb4", 16, None, "ivfpq_packed_scan_kernel"),
    "rerank_two_pass": ("rerank2", 16, {"recall_num": 50}, "ivfpq_scan_kernel"),
    "rerank_one_pass": ("rerank1", 16, {"recall_num": 50}, "ivfpq_scan_kernel"),
    "ivfpqfastscan": ("pqfs", 16, None, "ivfpqfs_scan_kernel"),
    "ivfrabitq": ("rabitq", 16, None, "rabitq_scan_kernel"),
    "vearch": ("vearch", 16, None, "vearch_scan_kernel"),
    "binaryivf": ("binaryivf", 16, None, "binary_ivf_scan_kernel"),
    "soar_spilled": ("soar", 16, None, "ivfpqfs_scan_kernel"),
    "gpu_ivfpq_sharded": ("sharded", 16, None, ""),
}
RERANK_SITE = {"rerank_two_pass": "rerank_prefilter_kernel", "rerank_one_pass": "rerank_kernel"}


def queries(kind, xq, nq):
    return binary_rows(nq, 11) if kind == "binaryivf" else xq[:nq]


@pytest.mark.parametrize("path", sorted(PATHS))
def test_every_path_is_cancelled_and_an_unset_token_changes_nothing(path, data):
    g = gi()
    db, xq = data
    kind, nq, params, label = PATHS[path]
    idx = build(kind, db)
    x = queries(kind, xq, nq)
    try:
        ref = idx.search(x, K, params=params)
        assert idx.last_scan_kernel.startswith(label), idx.last_scan_kernel
        scan_label = idx.last_scan_kernel
        used0 = g.pool_usage()[0]
        # a token that is never set: byte-equal results
        t = g.CancelToken()
        got = idx.search(x, K, params=params, cancel=t)
        assert np.array_equal(got[0].view(np.uint32), ref[0].view(np.uint32)) and np.array_equal(got[1], ref[1])
        # a token set before the call: the kill error, and the path's kernels skipped their CTAs
        g.debug_cancel_stats()  # clears the counters
        t2 = g.CancelToken()
        t2.set()
        with pytest.raises(g.SearchKilled):
            idx.search(x, K, params=params, cancel=t2)
        stats = g.debug_cancel_stats()
        for site in polled_sites(scan_label) + ([RERANK_SITE[path]] if path in RERANK_SITE else []):
            assert stats[site] > 0, (site, stats)
        # the index answers as before, and the scratch came back
        again = idx.search(x, K, params=params)
        assert np.array_equal(again[0].view(np.uint32), ref[0].view(np.uint32)) and np.array_equal(again[1], ref[1])
        assert g.pool_usage()[0] == used0
    finally:
        idx.close()


def test_realtime_tail_and_search_device(data):
    import torch
    g = gi()
    db, xq = data
    idx = build("ivfflat", db[:15000])
    idx.add_vectors(db[15000:])  # stored, not indexed: the enable_realtime tail
    try:
        ref = idx.search(xq[:16], K, search_unindexed_tail=True)
        t = g.CancelToken()
        got = idx.search(xq[:16], K, search_unindexed_tail=True, cancel=t)
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[0], ref[0])
        t2 = g.CancelToken()
        t2.set()
        g.debug_cancel_stats()
        with pytest.raises(g.SearchKilled):
            idx.search(xq[:16], K, search_unindexed_tail=True, cancel=t2)
        assert np.array_equal(idx.search(xq[:16], K, search_unindexed_tail=True)[1], ref[1])
        # search_device: the same results for an unset token, the kill error for a set one
        xd = torch.from_numpy(xq[:64]).cuda()
        dref, iref = idx.search_device(xd, K)
        unset = g.CancelToken()  # kept alive until the asynchronous search is done with it
        dg, ig = idx.search_device(xd, K, cancel=unset)
        torch.cuda.synchronize()
        assert torch.equal(ig, iref) and torch.equal(dg, dref)
        t3 = g.CancelToken()
        t3.set()
        g.debug_cancel_stats()
        with pytest.raises(g.SearchKilled):
            idx.search_device(xd, K, cancel=t3)
        torch.cuda.synchronize()
        st = g.debug_cancel_stats()
        assert sum(st[s] for s in polled_sites(idx.last_scan_kernel)) > 0, st
        d2, i2 = idx.search_device(xd, K)
        torch.cuda.synchronize()
        assert torch.equal(i2, iref)
    finally:
        idx.close()


def _cancel_after(token, delay_s):
    th = threading.Timer(delay_s, token.set)
    th.start()
    return th


def _mid_flight(idx, x, k, params=None, delay_s=0.002):
    g = gi()
    t0 = time.perf_counter()
    ref = idx.search(x, k, params=params)
    full = time.perf_counter() - t0
    assert full >= 0.05, f"the uncancelled search takes {full * 1e3:.1f} ms; the case needs >= 50 ms"
    tok = g.CancelToken()
    th = _cancel_after(tok, delay_s)
    t0 = time.perf_counter()
    with pytest.raises(g.SearchKilled):
        idx.search(x, k, params=params, cancel=tok)
    killed = time.perf_counter() - t0
    th.join()
    again = idx.search(x, k, params=params)
    assert np.array_equal(again[1], ref[1]) and np.array_equal(again[0], ref[0])
    print(f"uncancelled {full * 1e3:.1f} ms, cancelled after {delay_s * 1e3:.0f} ms: {killed * 1e3:.1f} ms")
    return full, killed


def test_mid_flight_cancel_flat_host_store():
    g = gi()
    import torch
    # 1 GB of rows over PCIe, scored against 8192 queries: about 2e12 fp32 distance terms keep the uncancelled search
    # on the CUDA cores for well over 50 ms, however fast the host link is
    d, n, nq = 256, 1_000_000, 8192
    idx = g.GammaIndex("FLAT", d, {"metric_type": "L2"}, store_type="RocksDB")
    idx.add_vectors(synth.sift_like_torch(n, d, seed=503, device=torch.device("cuda:0")))
    torch.cuda.synchronize()
    try:
        full, killed = _mid_flight(idx, synth.sift_like(nq, d, seed=504), 10)
        assert killed < full
    finally:
        idx.close()


def test_mid_flight_cancel_large_ivfpq_batch():
    g = gi()
    import torch
    d, n = 128, 2_000_000
    idx = g.GammaIndex("IVFPQ", d, {"ncentroids": 1024, "nprobe": 128, "nsubvector": 32, "metric_type": "L2",
                                    "training_threshold": 65536})
    idx.add_vectors(synth.sift_like_torch(n, d, seed=505, device=torch.device("cuda:0")))
    idx.train()
    idx.add_pending()
    try:
        full, killed = _mid_flight(idx, synth.sift_like(40000, d, seed=506), 100)
        assert killed < full
    finally:
        idx.close()


def test_coalesced_requests_keep_their_own_tokens(data):
    g = gi()
    db, xq = data
    idx = build("ivfflat", db)
    try:
        alone = [idx.search(xq[i:i + 1], K) for i in range(24)]
        killed = g.CancelToken()
        killed.set()
        res, errs = [None] * 24, [None] * 24
        barrier = threading.Barrier(24)

        def one(i):
            barrier.wait()
            try:
                res[i] = idx.search(xq[i:i + 1], K, cancel=killed if i == 5 else g.CancelToken())
            except g.SearchKilled as e:
                errs[i] = e

        ths = [threading.Thread(target=one, args=(i,)) for i in range(24)]
        for th in ths:
            th.start()
        for th in ths:
            th.join()
        assert errs[5] is not None and res[5] is None
        for i in range(24):
            if i != 5:
                assert errs[i] is None
                assert np.array_equal(res[i][1], alone[i][1]) and np.array_equal(res[i][0], alone[i][0])
    finally:
        idx.close()


def _engine_kill_mid_flight(api, search, rid):
    """SetKillStatus from another thread while `search(rid)` runs: set half a millisecond into the call and again every
    half millisecond until it returns, so the kill lands while it runs whatever its length"""
    from vearch_b200 import engine as E
    done = threading.Event()

    def killer():
        while not done.wait(0.0005):
            api.SetKillStatus(rid.encode(), 3, 1)

    th = threading.Thread(target=killer)
    th.start()
    try:
        with pytest.raises(E.GammaStatusError) as ei:
            search(rid)
    finally:
        done.set()
        th.join()
    assert ei.value.code == 8
    api.DeleteKillStatus(rid.encode(), 3)
    assert len(wire.decode_search_response(search(rid))[0]["items"]) > 0  # the same request id is served again


def test_engine_kill_mid_flight(tmp_path):
    from vearch_b200 import engine as E
    d, n, nq = 256, 20000, 16000
    db = synth.sift_like(n, d, seed=507)
    e = E.GammaEngine(str(tmp_path), space_name="kc")
    e.create_table("kc", d, "FLAT", {"metric_type": "L2"}, extra_vectors=[("img", d, "FLAT", {"metric_type": "L2"})])
    for i in range(n):
        assert e.add_doc(f"doc{i}", db[i], extra_fields=[("img", db[i].tobytes(), wire.DT_VECTOR)]) == 0
    api = E._api()
    xq = synth.sift_like(nq, d, seed=508)
    single = wire.encode_search_request("emb", xq, 10, request_id="kill-single", partition_id=3)
    multi = wire.encode_search_request("emb", xq, 10, request_id="kill-multi", partition_id=3,
                                       extra_vec_queries=[("img", xq)])
    try:
        e.search_raw(single)  # warm
        _engine_kill_mid_flight(api, lambda rid: e.search_raw(single), "kill-single")
        _engine_kill_mid_flight(api, lambda rid: e.search_raw(multi), "kill-multi")  # SearchMulti
    finally:
        e.close()
