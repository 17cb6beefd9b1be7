"""Key-exact top-k on every search path (DESIGN section 5): results compared with tests/topk_reference.py id for id and
score bit for bit, tie groups included, at k on each side of the queue-geometry boundaries up to 4096.

The data keep every score an integer below 2^24 (IVF-PQ with integer centroids and codebooks, so its reconstructions
are integers too), so the reference is exact and independent of the kernels' evaluation order.  Three regimes: natural
rows (synth.sift_like scaled down), a pool of 64 small-integer vectors (mixed sign under IP, with zero rows and a zero
query), where every k cuts a tie group and ties cross lists, and identical rows.  IVF searches go through
search_preassigned with probes and coarse distances computed here, exactly.  Every case asserts the kernel that served
it."""
import numpy as np
import pytest

import topk_reference as R
from oracle_pqfs import twin
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = R.METRIC_L2, R.METRIC_IP
METRICS = [L2, IP]


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


# ---- data -----------------------------------------------------------------------------------------------------------
def make_data(regime, n, d, nq, metric, seed):
    rng = np.random.default_rng(seed)
    if regime == "sift":
        db = np.rint(synth.sift_like(n, d, seed=seed) / 8)
        xq = np.rint(synth.sift_like(nq, d, seed=seed + 1) / 8)
    elif regime == "pool":
        lo, hi = (-2, 3) if metric == IP else (0, 4)
        pool = rng.integers(lo, hi, (64, d))
        pool[0] = 0  # zero rows
        db = pool[rng.integers(0, 64, n)]
        xq = pool[rng.integers(0, 64, nq)]
        xq[-1] = 0  # a zero query: every IP score is +0.0
    else:  # degenerate: every row (and so every code) identical
        db = np.tile(rng.integers(0, 4, d), (n, 1))
        xq = rng.integers(0, 4, (nq, d))
    return db.astype(np.float32), xq.astype(np.float32)


def assert_results(got, ref_keys, metric, what=""):
    dg, ig = got
    dr, ir = R.decode(ref_keys, metric)
    bad = np.nonzero(~(np.all(ig == ir, 1) & np.all(dg.view(np.uint32) == dr.view(np.uint32), 1)))[0]
    if len(bad):
        q = bad[0]
        j = np.nonzero((ig[q] != ir[q]) | (dg[q].view(np.uint32) != dr[q].view(np.uint32)))[0][0]
        raise AssertionError(f"{what}: {len(bad)} queries differ; query {q} slot {j}: got ({dg[q, j]!r}, {ig[q, j]}), "
                             f"want ({dr[q, j]!r}, {ir[q, j]})")


def filter_cases(n, k, ref_scores, metric, seed):
    """deletion / filter bitmaps leaving fewer than k valid rows, exactly k and none; a score window [s, s] on a tied
    score and a window edge inside a tie group (ref_scores: one query's unfiltered reference scores)"""
    rng = np.random.default_rng(seed)
    few = np.zeros(n, bool)
    few[rng.choice(n, k // 2, replace=False)] = True
    exact_k = np.zeros(n, bool)
    exact_k[rng.choice(n, min(k, n), replace=False)] = True
    cases = [("fewer_than_k", {"del_bitmap": np.packbits(~few, bitorder="little")}),
             ("exactly_k", {"filter_bitmap": np.packbits(exact_k, bitorder="little")}),
             ("none", {"filter_bitmap": np.zeros((n + 7) // 8, np.uint8)})]
    live = ref_scores[np.abs(ref_scores) < R.FLT_MAX]
    if len(live):
        s = float(live[min(len(live), 5) - 1])
        cases.append(("window_point", {"min_score": s, "max_score": s}))
        e = float(live[len(live) // 2])
        cases.append(("window_edge", {"max_score": e} if metric == L2 else {"min_score": e}))
    return cases


# ---- FLAT -----------------------------------------------------------------------------------------------------------
FLAT_K = [1, 16, 17, 257, 400, 1024, 4095, 4096]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("regime", ["sift", "pool", "degenerate"])
def test_flat(metric, regime):
    import torch
    d, n, nq = 32, 140000, 6  # two distance chunks of 131072 rows
    db, xq = make_data(regime, n, d, nq, metric, seed=10)
    idx = gi().GammaIndex("FLAT", d, {"metric_type": mt(metric)})
    idx.add(db)
    small = gi().GammaIndex("FLAT", d, {"metric_type": mt(metric)})  # n < k
    small.add(db[:3000])
    xt = torch.from_numpy(xq).cuda()
    for k in FLAT_K:
        ref = R.flat_keys(xq, db, k, metric)
        assert_results(idx.search(xq, k), ref, metric, f"FLAT k={k}")
        assert idx.last_scan_kernel == "dist_tile_kernel+select_rows_kernel"
        got = idx.search_device_keys(xt, k).cpu().numpy().view(np.uint64)
        assert np.array_equal(got, ref), f"FLAT raw keys k={k}"
        assert_results(small.search(xq, k), R.flat_keys(xq, db[:3000], k, metric), metric, f"FLAT n<k k={k}")
    for k in (17, 1024):
        ref = R.flat_keys(xq, db, k, metric)
        sc = R.decode(ref, metric)[0][0]
        for name, kw in filter_cases(n, k, sc, metric, seed=k):
            assert_results(idx.search(xq, k, **kw), R.flat_keys(xq, db, k, metric, **kw), metric, f"FLAT {name} k={k}")
    idx.close()
    small.close()


# ---- IVF helpers ------------------------------------------------------------------------------------------------------
def coarse_exact(xq, cent, metric, nprobe):
    """exact coarse scores, and the nprobe best lists (ties to the smaller list)"""
    s = R.exact_scores(xq, cent, metric)
    kk = R.keys(s, np.arange(len(cent))[None, :], None, metric)
    order = np.argsort(kk, axis=1, kind="stable")[:, :nprobe]
    return s, order.astype(np.int64)


def pick_centroids(db, nlist, seed):
    return db[np.random.default_rng(seed).choice(len(db), nlist, replace=False)]


def entries(idx, nlist):
    off, codes, ids = idx.export_lists()
    return off, codes, ids, np.repeat(np.arange(nlist), np.diff(off))


def tombstone_some(idx, off, ids, lists):
    """tombstone the first entry of each given list; returns the raw ids with the tombstone bit, as the kernels see them"""
    ids = ids.copy()
    for l in lists:
        if off[l + 1] > off[l]:
            idx.tombstone(int(l), 0)
            ids[off[l]] |= np.iinfo(np.int64).min
    return ids


def make_ivfflat(d, nlist, nprobe, metric, db, seed, tombstones=True):
    cent = pick_centroids(db, nlist, seed)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": mt(metric)})
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending()
    off, _, ids, el = entries(idx, nlist)
    if tombstones:
        ids = tombstone_some(idx, off, ids, range(0, nlist, 5))
    return idx, cent, ids, el


def ivfflat_ref(xq, db, ids, el, probes, k, metric, **kw):
    vid = np.where(ids >= 0, ids, ids & 0xFFFFFFFF)
    return R.search_entries(R.exact_scores(xq, db[vid], metric), el, ids, probes, k, metric, **kw)


# ---- IVF-Flat query-major ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d,ladder", [
    (64, [(1, "warp"), (100, "warp"), (2048, "warp"), (2049, "generic"), (4096, "generic")]),
    (128, [(16, "warp"), (2048, "warp"), (2049, "generic"), (4096, "generic")]),
    (1536, [(1024, "warp"), (1025, "generic"), (4096, "generic")]),
    (20, [(1, "generic"), (17, "generic"), (1024, "generic"), (4096, "generic")]),
    (100, [(33, "generic"), (4096, "generic")]),
])
@pytest.mark.parametrize("regime", ["sift", "pool"])
def test_ivfflat_query_major(metric, d, ladder, regime):
    n, nq, nlist, nprobe = (12000, 4, 16, 12) if d == 1536 else (20000, 6, 32, 20)
    db, xq = make_data(regime, n, d, nq, metric, seed=d)
    if d == 1536:  # keep |x|^2 below 2^24
        db, xq = np.minimum(db, 15), np.minimum(xq, 15)
    idx, cent, ids, el = make_ivfflat(d, nlist, nprobe, metric, db, seed=1)
    _, probes = coarse_exact(xq, cent, metric, nprobe)
    cd = np.zeros(probes.shape, np.float32)
    names = {"warp": "ivfflat_scan_warp_kernel", "generic": "ivfflat_scan_kernel"}
    for k, kern in ladder:
        ref = ivfflat_ref(xq, db, ids, el, probes, k, metric)
        assert_results(idx.search_preassigned(xq, k, probes, cd), ref, metric, f"IVFFLAT d={d} k={k}")
        assert idx.last_scan_kernel == names[kern], (k, idx.last_scan_kernel)
    k = ladder[-1][0]
    sc = R.decode(ivfflat_ref(xq, db, ids, el, probes, k, metric), metric)[0][0]
    for name, kw in filter_cases(n, k, sc, metric, seed=d):
        assert_results(idx.search_preassigned(xq, k, probes, cd, **kw), ivfflat_ref(xq, db, ids, el, probes, k, metric, **kw),
                       metric, f"IVFFLAT d={d} {name} k={k}")
    idx.close()


# ---- IVF-Flat list-major ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("regime", ["sift", "pool", "degenerate"])
def test_ivfflat_list_major(metric, regime):
    d, n, nq, nlist, nprobe = 64, 20000, 128, 16, 4  # 32 (query, probe) pairs per list
    db, xq = make_data(regime, n, d, nq, metric, seed=7)
    idx, cent, ids, el = make_ivfflat(d, nlist, nprobe, metric, db, seed=2)
    if regime == "degenerate":  # one list holds every row: probe it first
        probes = np.argsort(-np.diff(idx.export_lists()[0]))[None, :nprobe].repeat(nq, 0).astype(np.int64)
    else:
        _, probes = coarse_exact(xq, cent, metric, nprobe)
    cd = np.zeros(probes.shape, np.float32)
    ladder = [(32, "ivf_listmajor_tma_kernel"), (33, "ivf_listmajor_pipe_kernel"), (64, "ivf_listmajor_pipe_kernel"),
              (65, "ivf_listmajor_tc_kernel+seg_select_kernel"), (1024, "ivf_listmajor_tc_kernel+seg_select_kernel"),
              (4096, "ivf_listmajor_tc_kernel+seg_select_kernel")]
    for k, kern in ladder:
        ref = ivfflat_ref(xq, db, ids, el, probes, k, metric)
        assert_results(idx.search_preassigned(xq, k, probes, cd), ref, metric, f"IVFFLAT list-major k={k}")
        assert idx.last_scan_kernel == kern, (k, idx.last_scan_kernel)
    for k in (32, 65):
        sc = R.decode(ivfflat_ref(xq, db, ids, el, probes, k, metric), metric)[0][0]
        for name, kw in filter_cases(n, k, sc, metric, seed=k):
            assert_results(idx.search_preassigned(xq, k, probes, cd, **kw),
                           ivfflat_ref(xq, db, ids, el, probes, k, metric, **kw), metric, f"IVFFLAT list-major {name} k={k}")
    idx.close()


# ---- IVF-PQ -------------------------------------------------------------------------------------------------------------
class PqState:
    """an IVFPQ / IVFPQFastScan index on integer centroids and codebooks, with every list entry's exact score"""

    def __init__(self, typ, d, M, nbits, nlist, metric, db, xq, seed, tombstones=True):
        rng = np.random.default_rng(seed)
        self.metric, self.db, self.xq, self.nlist = metric, db, xq, nlist
        self.cent = pick_centroids(db, nlist, seed)
        ksub = 16 if typ == "IVFPQFastScan" else 1 << nbits
        self.pq = rng.integers(-2, 3, (M, ksub, d // M)).astype(np.float32)
        params = {"ncentroids": nlist, "nprobe": min(nlist, 8), "nsubvector": M, "metric_type": mt(metric)}
        if typ == "IVFPQ":
            params["nbits_per_idx"] = nbits
        self.idx = gi().GammaIndex(typ, d, params)
        self.idx.set_centroids(self.cent)
        self.idx.set_pq_centroids(self.pq)
        self.idx.add_vectors(db)
        self.idx.add_pending()
        self.off, codes, ids, self.el = entries(self.idx, nlist)
        self.ids = tombstone_some(self.idx, self.off, ids, range(1, nlist, 7)) if tombstones else ids
        self.coarse, _ = coarse_exact(xq, self.cent, metric, 1)
        if typ == "IVFPQFastScan":
            lut8, ab = twin.lut(self.pq, xq, metric)
            cu = twin.unpack(codes, M)
            self.scores = np.stack([twin.scores(lut8[q], ab[q], cu) for q in range(len(xq))])
        else:
            R.pq_guard(xq, self.cent, self.pq, metric)
            rec = R.pq_reconstruct(self.cent, self.pq, self.el, R.unpack_codes(codes, M, nbits))
            self.scores = R.exact_scores(xq, rec, metric)

    def probes(self, nprobe):
        return coarse_exact(self.xq, self.cent, self.metric, nprobe)[1]

    def ref(self, probes, k, q=slice(None), **kw):
        return R.search_entries(self.scores[q], self.el, self.ids, probes, k, self.metric, **kw)

    def search(self, probes, k, q=slice(None), **kw):
        cd = np.take_along_axis(self.coarse[q], probes, 1).astype(np.float32)
        return self.idx.search_preassigned(self.xq[q], k, probes, cd, **kw)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d,M", [(64, 8), (64, 16), (128, 32), (128, 64), (96, 12)])
@pytest.mark.parametrize("regime", ["sift", "pool"])
def test_ivfpq_query_major(metric, d, M, regime):
    n, nq, nlist, nprobe = 20000, 6, 64, 40  # nprobe > 32: the CTA groups' partials are merged
    db, xq = make_data(regime, n, d, nq, metric, seed=M)
    st = PqState("IVFPQ", d, M, 8, nlist, metric, db, xq, seed=3)
    probes = st.probes(nprobe)
    for k in (1, 16, 17, 400, 1024, 4096):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQ M={M} k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_scan_kernel"
    sc = R.decode(st.ref(probes, 100), metric)[0][0]
    for name, kw in filter_cases(n, 100, sc, metric, seed=M):
        assert_results(st.search(probes, 100, **kw), st.ref(probes, 100, **kw), metric, f"IVFPQ M={M} {name}")
    st.idx.close()


def test_ivfpq_large_m_limits():
    """M = 128: the [128][256] fp32 table leaves room for a queue of k' <= 2048 only; M >= 147 cannot search at all and
    is refused at create, naming nsubvector (the default nsubvector = d / 2 included)"""
    d, n, nq = 256, 6000, 4
    db, xq = make_data("pool", n, d, nq, L2, seed=5)
    st = PqState("IVFPQ", d, 128, 8, 16, L2, db, xq, seed=4)
    probes = st.probes(12)
    for k in (1, 1024, 2048):
        assert_results(st.search(probes, k), st.ref(probes, k), L2, f"IVFPQ M=128 k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_scan_kernel"
    with pytest.raises(gi().GammaError, match="recall_num / topn.*2048"):
        st.search(probes, 2049)
    with pytest.raises(gi().GammaError, match="recall_num / topn.*2048"):
        st.search(probes, 10, params={"recall_num": 4096})
    st.idx.close()
    for d, params in ((320, {"nsubvector": 160}), (384, {})):
        with pytest.raises(gi().GammaError, match="nsubvector"):
            gi().GammaIndex("IVFPQ", d, dict(params, ncentroids=16, nprobe=4, metric_type="L2"))
    gi().GammaIndex("IVFPQ", 256, {"ncentroids": 16, "nprobe": 4, "nsubvector": 128, "metric_type": "L2"}).close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d,M", [(128, 16), (64, 8)])
@pytest.mark.parametrize("regime", ["sift", "pool"])
def test_ivfpq_list_major(metric, d, M, regime):
    n, nq, nlist, nprobe = 20000, 128, 16, 6
    db, xq = make_data(regime, n, d, nq, metric, seed=M + 100)
    st = PqState("IVFPQ", d, M, 8, nlist, metric, db, xq, seed=6)
    probes = st.probes(nprobe)
    for k in (10, 256, 257, 1024, 2048, 2049):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQ list-major M={M} k'={k}")
        assert st.idx.last_scan_kernel == ("pqtc_scan_kernel" if k <= 2048 else "ivfpq_scan_kernel")
    sc = R.decode(st.ref(probes, 100), metric)[0][0]
    for name, kw in filter_cases(n, 100, sc, metric, seed=M):
        assert_results(st.search(probes, 100, **kw), st.ref(probes, 100, **kw), metric, f"IVFPQ list-major {name}")
        assert st.idx.last_scan_kernel == "pqtc_scan_kernel"
    st.idx.close()


def pqtc_flags(st, probes, k, cap=None, **kw):
    """which queries the tensor-core filter must hand to its safety net, computed from the exported lists as the engine
    plans phase A: 'no bound' (fewer than k' valid entries in the leading probes that hold >= 4 k' entries, at most
    min(nprobe - 1, 8)) or 'overflow' (more than cap valid entries of the other probes score <= that bound)"""
    nq, nprobe = probes.shape
    cap = cap or max(2048, min(8192, 1 << (8 * k - 1).bit_length()))
    lens = np.diff(st.off)
    pa_max = min(nprobe - 1, 8)
    cum = np.cumsum(np.where(probes >= 0, lens[np.maximum(probes, 0)], 0), 1)
    pa = np.minimum(np.argmax(cum >= 4 * k, 1) + 1, pa_max)
    pa[cum[:, pa_max - 1] < 4 * k] = pa_max
    no_bound, overflow = np.zeros(nq, bool), np.zeros(nq, bool)
    for q in range(nq):
        ka = st.ref(probes[q:q + 1, :pa[q]], k, q=slice(q, q + 1), **kw)[0]
        if ka[-1] == R.SENTINEL:
            no_bound[q] = True
            continue
        kb = st.ref(probes[q:q + 1, pa[q]:], 8192 + 1, q=slice(q, q + 1), **kw)[0]
        overflow[q] = (kb <= ka[-1]).sum() > cap
    return no_bound, overflow


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("shape", ["nprobe6", "nprobe40", "kprime2048_nprobe258"])
def test_ivfpq_pqtc_safety_net(metric, shape):
    """queries the filter cannot bound (deleted phase-A lists) or whose candidates overflow (a far list probed first), in
    one batch with ordinary queries: every answer equals the reference and the query-major scan's"""
    d, M = 64, 8
    nlist, nprobe, nq, k = {"nprobe6": (16, 6, 128, 10), "nprobe40": (64, 40, 64, 10),
                            "kprime2048_nprobe258": (260, 258, 40, 2048)}[shape]
    n = 20000
    db, xq = make_data("sift", n, d, nq, metric, seed=nlist)
    st = PqState("IVFPQ", d, M, 8, nlist, metric, db, xq, seed=8, tombstones=False)
    probes = st.probes(nprobe)
    lens = np.diff(st.off)
    kw = {}
    if shape != "kprime2048_nprobe258":
        # one list keeps only k' / 2 of its rows: probed first by queries 1, 4, 7, ..., it leaves them no bound
        dl = int(np.argmax(lens))
        vids = st.ids[st.off[dl]:st.off[dl + 1]]
        dead = np.zeros(n, bool)
        dead[vids[k // 2:]] = True
        kw = {"del_bitmap": np.packbits(dead, bitorder="little")}
        ranked = st.probes(nlist)
        for q in range(nq):
            if q % 3 == 0:  # the farthest other list with >= 4 k' entries first: a loose bound, candidates overflow
                first = next(l for l in ranked[q][::-1] if lens[l] >= 4 * k and l != dl and l != ranked[q, 0])
            elif q % 3 == 1:
                first = dl
            else:
                continue
            rest = [l for l in ranked[q] if l != first and l != dl]
            probes[q] = [first] + rest[:nprobe - 1]
    no_bound, overflow = pqtc_flags(st, probes, k, **kw)
    flagged = no_bound | overflow
    assert flagged.any(), "precondition: no query reaches the safety net"
    if shape != "kprime2048_nprobe258":  # there, 8 leading probes of ~77 entries leave most queries no bound
        assert overflow.any() and no_bound.any() and not flagged.all(), (overflow.sum(), no_bound.sum())
    ref = st.ref(probes, k, **kw)
    assert_results(st.search(probes, k, **kw), ref, metric, f"pqtc safety net {shape}")
    assert st.idx.last_scan_kernel == "pqtc_scan_kernel"
    qs = np.nonzero(flagged)[0][:4].tolist() + np.nonzero(~flagged)[0][:2].tolist()
    qm = st.search(probes[qs], k, q=qs, **kw)  # a small batch: query-major
    assert st.idx.last_scan_kernel == "ivfpq_scan_kernel"
    assert_results(qm, ref[qs], metric, f"query-major {shape}")
    st.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("nbits", [1, 4, 7])
@pytest.mark.parametrize("regime", ["sift", "pool"])
def test_ivfpq_packed(metric, nbits, regime):
    d, M, n, nq, nlist, nprobe = 64, 16, 20000, 6, 32, 34
    db, xq = make_data(regime, n, d, nq, metric, seed=nbits)
    st = PqState("IVFPQ", d, M, nbits, nlist, metric, db, xq, seed=9)
    probes = st.probes(nprobe)
    for k in (1, 17, 400, 1024, 4096):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQ nbits={nbits} k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_packed_scan_kernel"
    sc = R.decode(st.ref(probes, 100), metric)[0][0]
    for name, kw in filter_cases(n, 100, sc, metric, seed=nbits):
        assert_results(st.search(probes, 100, **kw), st.ref(probes, 100, **kw), metric, f"IVFPQ nbits={nbits} {name}")
    st.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("regime", ["sift", "pool"])
def test_ivfpqfs(metric, regime):
    d, M, n, nq, nlist, nprobe = 64, 16, 20000, 6, 32, 34
    db, xq = make_data(regime, n, d, nq, metric, seed=40)
    st = PqState("IVFPQFastScan", d, M, 4, nlist, metric, db, xq, seed=10)
    probes = st.probes(nprobe)
    for k in (1, 17, 400, 1024, 4096):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQFastScan k'={k}")
        assert st.idx.last_scan_kernel == "ivfpqfs_scan_kernel"
    sc = R.decode(st.ref(probes, 100), metric)[0][0]
    for name, kw in filter_cases(n, 100, sc, metric, seed=3):
        assert_results(st.search(probes, 100, **kw), st.ref(probes, 100, **kw), metric, f"IVFPQFastScan {name}")
    st.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("typ", ["IVFPQ", "IVFPQFastScan"])
def test_exact_rerank(metric, typ):
    """recall_num = k and 4096, and fewer valid candidates than recall_num: the k best, by exact score from the raw
    rows, of the ADC top recall_num"""
    d, M, n, nq, nlist, nprobe = 64, 16, 20000, 6, 32, 16
    db, xq = make_data("pool", n, d, nq, metric, seed=50)
    st = PqState(typ, d, M, 8 if typ == "IVFPQ" else 4, nlist, metric, db, xq, seed=11)
    probes = st.probes(nprobe)
    keep = np.zeros(n, bool)
    keep[np.random.default_rng(1).choice(n, 1500, replace=False)] = True
    for k, rn, kw in [(10, 10, {}), (100, 4096, {}), (10, 4096, {"filter_bitmap": np.packbits(keep, bitorder="little")})]:
        ref = R.rerank_keys(st.ref(probes, rn, **kw), xq, db, k, metric, **kw)
        assert_results(st.search(probes, k, params={"recall_num": rn}, **kw), ref, metric, f"{typ} re-rank {rn}")
    st.idx.close()


def test_ivf_brute_force_is_flat():
    d, n, nq = 32, 20000, 6
    db, xq = make_data("pool", n, d, nq, L2, seed=60)
    idx, _, _, _ = make_ivfflat(d, 16, 4, L2, db, seed=3, tombstones=False)
    for k in (17, 4096):
        assert_results(idx.search(xq, k, brute_force=True), R.flat_keys(xq, db, k, L2), L2, f"brute force k={k}")
        assert idx.last_scan_kernel == "dist_tile_kernel+select_rows_kernel"
    idx.close()
