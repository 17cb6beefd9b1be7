"""FLAT, the coarse quantiser and every IVF-Flat kernel at the largest dimensions, list lengths, batches and k they accept.

Two bars, as in tests/test_gpu_topk_keys.py and tests/test_gpu_float_accuracy.py: key-exact (ids and score bits equal
tests/topk_reference.py on small-integer rows, every score an integer below 2^24) and the float contract
(tests/float_contract.py) on ill-conditioned float rows.  Every case asserts the kernel that served it.

The query-major scan's dimension bound is restated (test_float_shape_limits_cpu.py), pinned, and found again from the
engine by bisecting create.  The scratch of the query-major IVF-Flat partials and of FLAT's chunk partials is read from
the device's memory pool and held to a restated bound."""
import re

import numpy as np
import pytest

import float_contract as FC
import topk_reference as R
from test_float_shape_limits_cpu import IVFFLAT_MAX_DIM, max_dim, pad, stages
from test_gpu_float_accuracy import IvfFlat
from test_gpu_topk_keys import assert_results, coarse_exact, entries, filter_cases, make_data, tombstone_some

pytestmark = pytest.mark.gpu
L2, IP = R.METRIC_L2, R.METRIC_IP
METRICS = [L2, IP]
F32 = np.float32
GENERIC, WARP = "ivfflat_scan_kernel", "ivfflat_scan_warp_kernel"
TMA, PIPE, TC = "ivf_listmajor_tma_kernel", "ivf_listmajor_pipe_kernel", "ivf_listmajor_tc_kernel+seg_select_kernel"
BRUTE = "dist_tile_kernel+select_rows_kernel"
PARTIAL_BUDGET = 1 << 30  # Index::kScanPartialBudget
CHUNK_ROWS = 8192  # IVF_CHUNK_ROWS: rows per query-major CTA


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


def small_ints(regime, n, d, nq, metric, seed):
    """make_data rows, clipped so that every score stays an integer below 2^24 at any d <= 4576 (|v| <= 3 at most)"""
    db, xq = make_data(regime, n, d, nq, metric, seed)
    if d > 256:
        db, xq = np.clip(db, -3, 3), np.clip(xq, -3, 3)
    return db, xq


def exact_ref(xq, db, ids, el, probes, k, metric, **kw):
    vid = np.where(ids >= 0, ids, ids & 0xFFFFFFFF)
    return R.search_entries(R.exact_scores(xq, db[vid], metric), el, ids, probes, k, metric, **kw)


def ivfflat(typ, d, nlist, metric, db, cent, **extra):
    idx = gi().GammaIndex(typ, d, {"ncentroids": nlist, "nprobe": min(nlist, 8), "metric_type": mt(metric), **extra})
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending()
    return idx


# ---- the dimension bound --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("typ", ["IVFFLAT", "GPU_IVFFLAT"])
def test_dimension_bound_from_the_engine_equals_the_restatement(typ):
    E = gi().GammaError

    def accepted(d):
        try:
            idx = gi().GammaIndex(typ, d, {"ncentroids": 4, "nprobe": 4})
        except E as e:
            assert re.search(rf"{typ}: dimension \[{d}\] above (\d+)", str(e)), str(e)
            return False
        idx.close()
        return True

    lo, hi = 1, 8000
    assert accepted(lo) and not accepted(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if accepted(mid) else (lo, mid)
    with pytest.raises(E) as ei:
        gi().GammaIndex(typ, lo + 1, {"ncentroids": 4, "nprobe": 4})
    named = int(re.search(r"above (\d+)", str(ei.value)).group(1))
    assert lo == named == IVFFLAT_MAX_DIM == max_dim(), (lo, named)


@pytest.mark.parametrize("metric", METRICS)
def test_search_at_the_dimension_bound(metric):
    """d = N: a two-stage ring at k = 4096, key-exact, with a deletion bitmap and a score window"""
    d, n, nq, nlist = IVFFLAT_MAX_DIM, 5000, 2, 2
    assert stages(pad(d), 4096) == 2
    db, xq = small_ints("pool", n, d, nq, metric, seed=3)
    idx = ivfflat("IVFFLAT", d, nlist, metric, db, db[:nlist])
    try:
        off, _, ids, el = entries(idx, nlist)
        probes = np.tile(np.arange(nlist), (nq, 1))
        cd = np.zeros(probes.shape, F32)
        for k in (1, 4096):
            assert_results(idx.search_preassigned(xq, k, probes, cd), exact_ref(xq, db, ids, el, probes, k, metric),
                           metric, f"d={d} k={k}")
            assert idx.last_scan_kernel == GENERIC
        sc = R.decode(exact_ref(xq, db, ids, el, probes, 4096, metric), metric)[0][0]
        for name, kw in filter_cases(n, 4096, sc, metric, seed=d)[::2]:
            assert_results(idx.search_preassigned(xq, 4096, probes, cd, **kw),
                           exact_ref(xq, db, ids, el, probes, 4096, metric, **kw), metric, f"d={d} {name}")
            assert idx.last_scan_kernel == GENERIC
    finally:
        idx.close()


# ---- dimension ladder, key-exact ------------------------------------------------------------------------------------
LADDER = [1, 3, 5, 17, 1536, 1540, 2048, 2560, 3072, 4096]
QM_K = [1, 17, 1024, 1025, 2048, 4096]


def qm_kernel(d, k):
    return WARP if d == 1536 and k <= 1024 else GENERIC


def lm_kernel(d, k):
    if k <= 32 and pad(d) > 16:
        return TMA
    return PIPE if k <= 64 else TC


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", LADDER)
def test_dimension_ladder_key_exact(d, metric):
    n, nlist, nprobe = 6000, 8, 8
    regime = "sift" if d <= 17 else "pool"
    db, xq = small_ints(regime, n, d, 32, metric, seed=d)
    idx = ivfflat("IVFFLAT", d, nlist, metric, db, db[:nlist])
    try:
        q4 = slice(0, 4)  # 32 pairs over 8 lists: query-major
        for k in (17, 4096):
            got = idx.search(xq[q4], k, brute_force=True)
            assert idx.last_scan_kernel == BRUTE
            assert_results(got, R.flat_keys(xq[q4], db, k, metric), metric, f"brute force d={d} k={k}")
        off, _, ids, el = entries(idx, nlist)
        ids = tombstone_some(idx, off, ids, range(0, nlist, 3))
        _, probes = coarse_exact(xq, db[:nlist], metric, nprobe)
        cd = np.zeros(probes.shape, F32)
        for k in QM_K:
            got = idx.search_preassigned(xq[q4], k, probes[q4], cd[q4])
            assert idx.last_scan_kernel == qm_kernel(d, k), (k, idx.last_scan_kernel)
            assert_results(got, exact_ref(xq[q4], db, ids, el, probes[q4], k, metric), metric, f"qm d={d} k={k}")
        for k in (32, 64, 65, 4096):  # 256 pairs = 32 per list: list-major
            got = idx.search_preassigned(xq, k, probes, cd)
            assert idx.last_scan_kernel == lm_kernel(d, k), (k, idx.last_scan_kernel)
            assert_results(got, exact_ref(xq, db, ids, el, probes, k, metric), metric, f"lm d={d} k={k}")
        # deletion / filter bitmaps and score windows at one k per kernel
        cases = [(q4, 1025, GENERIC), (slice(None), 32, lm_kernel(d, 32)), (slice(None), 64, PIPE),
                 (slice(None), 65, TC)]
        if d == 1536:
            cases.append((q4, 1024, WARP))
        for q, k, kern in cases:
            sc = R.decode(exact_ref(xq[:1], db, ids, el, probes[:1], k, metric), metric)[0][0]
            for name, kw in filter_cases(n, k, sc, metric, seed=k):
                got = idx.search_preassigned(xq[q], k, probes[q], cd[q], **kw)
                assert idx.last_scan_kernel == kern, (name, idx.last_scan_kernel)
                assert_results(got, exact_ref(xq[q], db, ids, el, probes[q], k, metric, **kw), metric,
                               f"d={d} {kern} {name} k={k}")
    finally:
        idx.close()


def test_gpu_ivfflat_at_d_4096():
    d, n, nq, nlist = 4096, 5000, 3, 4
    db, xq = small_ints("pool", n, d, nq, L2, seed=41)
    idx = ivfflat("GPU_IVFFLAT", d, nlist, L2, db, db[:nlist])
    try:
        _, _, ids, el = entries(idx, nlist)
        probes = np.tile(np.arange(nlist), (nq, 1))
        for k in (1, 2048):
            got = idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, F32))
            assert idx.last_scan_kernel == GENERIC
            assert_results(got, exact_ref(xq, db, ids, el, probes, k, L2), L2, f"GPU_IVFFLAT k={k}")
    finally:
        idx.close()


# ---- dimension ladder, float contract -------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", ["offset1000", "near_dup"])
@pytest.mark.parametrize("d", [3, 17, 1540, 2560, 4096])
def test_dimension_ladder_float_contract(d, name, metric):
    s = IvfFlat(name, d, 3000, 128, 16, 4, metric, seed=d + 7)  # 32 (query, probe) pairs per list
    try:
        for k, kern in ((10, lm_kernel(d, 10)), (48, PIPE), (100, TC)):
            got = s.search(k)
            assert s.idx.last_scan_kernel == kern, (k, s.idx.last_scan_kernel)
            s.check(got, k, True, f"list-major {name} d={d} k={k}")
        bm = np.packbits(~s.deleted, bitorder="little")
        got = s.search(100, filter_bitmap=bm)
        assert s.idx.last_scan_kernel == TC
        s.check(got, 100, True, f"list-major {name} d={d} bitmap", deleted=s.deleted)
        for k in (10, 1025):
            got = s.search(k, slice(0, 4))
            assert s.idx.last_scan_kernel == GENERIC
            s.check(got, k, False, f"query-major {name} d={d} k={k}")
        w = s.window(10)
        got = s.search(10, slice(0, 4), **w)
        assert s.idx.last_scan_kernel == GENERIC
        s.check(got, 10, False, f"query-major {name} d={d} window", **w)
        got = s.idx.search(s.xq[:4], 10, brute_force=True)
        assert s.idx.last_scan_kernel == BRUTE
        f, ad = FC.scores64(s.xq[:4], s.db, metric)
        md = FC.direct_margin(f, ad, d, metric)
        cand = np.arange(len(s.db))
        FC.check_all(got, lambda q: (cand, f[q], md[q], md[q]), 10, metric, f"brute force {name} d={d}")
    finally:
        s.idx.close()


def coarse_margins(xq, cent, metric, d):
    f, ad = FC.scores64(xq, cent, metric)
    na, nb = (xq.astype(np.float64) ** 2).sum(1)[:, None], (cent.astype(np.float64) ** 2).sum(1)[None, :]
    tcm = FC.expanded_l2_margin(ad, na, nb, f, d) if metric == L2 else FC.tc_dot_margin(ad, d)
    return f, tcm, FC.direct_margin(f, ad, d, metric)


def coarse_path(nlist, nq, nprobe, d, fused):
    """IvfIndex::coarse_dev: tensor cores from 64 lists and 32 queries, fused for nprobe <= 64 above one K chunk"""
    if nlist < 64 or nq < 32:
        return "dist_tile_kernel+select_rows_kernel"
    if fused and nprobe <= 64 and (pad(d) + 15) // 16 * 16 > 16:
        return "coarse_topk_kernel"
    return "dist_tc_kernel+select_rows_kernel"


def check_coarse(monkeypatch, idx, xq, cent, metric, d, nprobe, what):
    """nq 64 (the fused kernel), 64 under GB_COARSE_FUSED=0 (the score matrix) and 31 (the exact kernel)"""
    f, tcm, dm = coarse_margins(xq, cent, metric, d)
    cand = np.arange(len(cent))
    for nq, fused in ((64, True), (64, False), (31, True)):
        if not fused:
            monkeypatch.setenv("GB_COARSE_FUSED", "0")
        dis, ids = idx.coarse_search(xq[:nq], nprobe)
        monkeypatch.delenv("GB_COARSE_FUSED", raising=False)
        path = coarse_path(len(cent), nq, nprobe, d, fused)
        m = dm if path.startswith("dist_tile") else tcm
        assert idx.last_coarse_kernel == path, (path, idx.last_coarse_kernel)
        FC.check_all((dis, ids), lambda q: (cand, f[q], m[q], m[q]), nprobe, metric, f"coarse {path} {what}",
                     ip_ties_desc=False)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", ["offset1000", "near_dup", "wide"])
@pytest.mark.parametrize("d", LADDER)
def test_coarse_at_large_d(monkeypatch, d, name, metric):
    nlist, nprobe = 256, 16
    cent, xq = FC.regime(name, nlist, d, 64, seed=d + 3)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": mt(metric)})
    try:
        idx.set_centroids(cent)
        check_coarse(monkeypatch, idx, xq, cent, metric, d, nprobe, f"{name} d={d}")
    finally:
        idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [1, 3, 5, 1536, 4096])
@pytest.mark.parametrize("name", FC.REGIMES)
def test_dist_tiles_at_large_d(name, d, metric):
    """element-wise, as test_gpu_float_accuracy.test_dist_tiles: the dot margin holds with one K chunk, where the TF32
    split's representation error dominates, and where 96 and 256 K chunks accumulate"""
    db, xq = FC.regime(name, 200, d, 64, seed=d)
    f, ad = FC.scores64(xq, db, metric)
    exact = gi().debug_dist_matrix(xq, db, metric, 0)
    assert np.all(np.abs(exact - f) <= FC.direct_margin(f, ad, d, metric)), f"{name}: exact kernel"
    tc = gi().debug_dist_matrix(xq, db, metric, 1).astype(np.float64)
    if metric == L2:
        na, nb = (xq.astype(np.float64) ** 2).sum(1)[:, None], (db.astype(np.float64) ** 2).sum(1)[None, :]
        m = FC.expanded_l2_margin(ad, na, nb, f, d)
    else:
        m = FC.tc_dot_margin(ad, d)
    ratio = np.abs(tc - f) / np.maximum(m, np.finfo(np.float64).tiny)
    assert ratio.max() <= 1, f"{name}: dist_tc_kernel exceeds its margin by x{ratio.max():.3g}"


# ---- list lengths ---------------------------------------------------------------------------------------------------
LENS = [(1 << 17) + 3, 0, 1, 127, 128, 129, 2047, 2048, 2049, 8191, 8192, 8193]
BOUNDARY_POS = [0, 2047, 2048, 8191, 8192, 16383, 16384, 16385, 65536, 1 << 17]


def placed_rows(lens, d, seed):
    """integer rows around centroids 100 e_l: row r of list l is 100 e_l + a pool row with entries in [0, 3]"""
    rng = np.random.default_rng(seed)
    cent = np.zeros((len(lens), d), F32)
    cent[np.arange(len(lens)), np.arange(len(lens))] = 100
    pool = rng.integers(0, 4, (64, d))
    el = np.repeat(np.arange(len(lens)), lens)
    db = (cent[el] + pool[rng.integers(0, 64, len(el))]).astype(F32)
    perm = rng.permutation(len(el))
    return cent, db[perm]


@pytest.mark.parametrize("metric", METRICS)
def test_list_lengths(metric):
    d = 32
    cent, db = placed_rows(LENS, d, seed=5)
    nlist, n = len(LENS), len(db)
    idx = ivfflat("IVFFLAT", d, nlist, metric, db, cent)
    try:
        off, _, ids, el = entries(idx, nlist)
        assert list(np.diff(off)) == LENS
        rng = np.random.default_rng(6)
        xq = (cent[rng.integers(0, nlist, 64)] + rng.integers(0, 4, (64, d))).astype(F32)
        got = idx.search(xq[:4], 4096, brute_force=True)
        assert idx.last_scan_kernel == BRUTE
        assert_results(got, R.flat_keys(xq[:4], db, 4096, metric), metric, "brute force")
        for p in BOUNDARY_POS[1:]:  # tombstones at split and segment boundaries of the long list
            idx.tombstone(0, p)
            ids[p] |= np.iinfo(np.int64).min
        dead = np.zeros(n, bool)
        dead[ids[[p + 1 for p in BOUNDARY_POS]] & 0xFFFFFFFF] = True
        probes = np.tile(np.arange(nlist), (64, 1))  # 768 pairs = 64 per list: list-major
        cd = np.zeros(probes.shape, F32)
        for q, kerns in ((slice(0, 4), {1: WARP, 64: WARP, 65: WARP, 4096: GENERIC}),
                         (slice(None), {1: TMA, 64: PIPE, 65: TC, 4096: TC})):
            for k, kern in kerns.items():
                for kw in ({}, {"del_bitmap": np.packbits(dead, bitorder="little")}):
                    got = idx.search_preassigned(xq[q], k, probes[q], cd[q], **kw)
                    assert idx.last_scan_kernel == kern, (k, idx.last_scan_kernel)
                    assert_results(got, exact_ref(xq[q], db, ids, el, probes[q], k, metric, **kw), metric,
                                   f"lengths {kern} k={k} {sorted(kw)}")
    finally:
        idx.close()


def pool_rows(n, d, seed):
    """n rows drawn from 64 integer pool rows: (db, pool index of each row, pool)"""
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 4, (64, d)).astype(F32)
    which = rng.integers(0, 64, n)
    return pool[which], which, pool


def pooled_keys(xq, pool, which, vids, k, metric):
    """exact top-k keys of queries over rows vids, each row equal to pool[which[vid]]: per query the best pool groups,
    taken whole until k rows are in, are the only rows that can reach the top k"""
    out = np.full((len(xq), k), R.SENTINEL, np.uint64)
    s = R.exact_scores(xq, pool, metric)
    grp = which[vids]
    for q in range(len(xq)):
        order = np.argsort(s[q] if metric == L2 else -s[q], kind="stable")
        take, cnt = [], 0
        counts = np.bincount(grp, minlength=len(pool))
        for g in order:
            if cnt >= k and s[q, g] != s[q, take[-1]]:
                break
            take.append(g)
            cnt += counts[g]
        sel = vids[np.isin(grp, take)]
        kk = np.sort(R.keys(s[q:q + 1, which[sel]], sel[None, :], None, metric)[0])[:k]
        out[q, :len(kk)] = kk
    return out


def test_listmajor_score_cap_sends_the_batch_query_major():
    """4096 queries on one 2^20-row list at k = 65: 2^32 scores, above the tensor-core path's 12 GiB cap, so the batch
    scans query-major though it has 2048 pairs per list"""
    d, n, nq, k = 32, 1 << 20, 4096, 65
    db, which, pool = pool_rows(n, d, seed=8)
    cent = np.stack([pool.mean(0), np.full(d, 1000.0)]).astype(F32)
    idx = ivfflat("IVFFLAT", d, 2, L2, db, cent)
    try:
        off, _, ids, el = entries(idx, 2)
        assert off[1] == n
        rng = np.random.default_rng(9)
        qi = rng.integers(0, 64, nq)
        xq = pool[qi]
        probes = np.zeros((nq, 1), np.int64)
        got = idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, F32))
        assert idx.last_scan_kernel == WARP, idx.last_scan_kernel  # d = 32, k = 65: the warp kernel's queue fits
        uq, inv = np.unique(qi, return_inverse=True)
        ref = pooled_keys(pool[uq], pool, which, ids, k, L2)[inv]
        assert_results(got, ref, L2, "12 GiB cap")
    finally:
        idx.close()


# ---- batches and pairs ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_pairs_at_the_query_major_switch_and_pair_groups(metric):
    d, n, nlist = 32, 20000, 16
    db, xq = small_ints("pool", n, d, 300, metric, seed=11)
    idx = ivfflat("IVFFLAT", d, nlist, metric, db, db[:nlist])
    try:
        off, _, ids, el = entries(idx, nlist)
        ids = tombstone_some(idx, off, ids, range(0, nlist, 4))
        for nq, nprobe, kern in ((73, 7, WARP), (64, 8, TC)):  # 511 = 32 nlist - 1 pairs, then 512
            _, probes = coarse_exact(xq[:nq], db[:nlist], metric, nprobe)
            got = idx.search_preassigned(xq[:nq], 100, probes, np.zeros(probes.shape, F32))
            assert idx.last_scan_kernel == kern, (nq * nprobe, idx.last_scan_kernel)
            assert_results(got, exact_ref(xq[:nq], db, ids, el, probes, 100, metric), metric, f"{nq * nprobe} pairs")
    finally:
        idx.close()
    idx = ivfflat("IVFFLAT", d, 4, metric, db, db[:4])
    try:
        _, _, ids, el = entries(idx, 4)
        for nq in (127, 128, 129, 300):  # every query probes every list: nq pairs per list
            probes = np.tile(np.arange(4), (nq, 1))
            for k in (32, 64, 65):
                got = idx.search_preassigned(xq[:nq], k, probes, np.zeros(probes.shape, F32))
                assert idx.last_scan_kernel == lm_kernel(d, k)
                assert_results(got, exact_ref(xq[:nq], db, ids, el, probes, k, metric), metric,
                               f"{nq} pairs per list k={k}")
    finally:
        idx.close()


def test_search_across_query_blocks():
    """nq = 16385 crosses search_keys_dev's 16384-query blocks; the index's own coarse quantiser picks the lists"""
    d, n, nlist, nprobe, k = 32, 20000, 16, 4, 64
    db, which, pool = pool_rows(n, d, seed=12)
    cent = pool[:nlist]
    idx = ivfflat("IVFFLAT", d, nlist, L2, db, cent, nprobe=nprobe)
    try:
        off, _, ids, el = entries(idx, nlist)
        qi = np.random.default_rng(13).integers(0, 64, 16385)
        got = idx.search(pool[qi], k)
        assert idx.last_scan_kernel == WARP  # the second block, of one query, scans query-major (the first: list-major)
        _, probes = coarse_exact(pool, cent, L2, nprobe)
        ref = exact_ref(pool, db, ids, el, probes, k, L2)[qi]
        assert_results(got, ref, L2, "16385 queries")
    finally:
        idx.close()


def test_flat_across_query_and_row_blocks():
    """2049 queries over 140000 rows at k = 4096: flat_search_dev's 2048-query score blocks and 131072-row chunks"""
    d, n, k = 32, 140000, 4096
    db, which, pool = pool_rows(n, d, seed=14)
    idx = gi().GammaIndex("FLAT", d, {"metric_type": "L2"})
    try:
        idx.add(db)
        qi = np.random.default_rng(15).integers(0, 64, 2049)
        got = idx.search(pool[qi], k)
        assert idx.last_scan_kernel == BRUTE
        uq, inv = np.unique(qi, return_inverse=True)
        assert_results(got, pooled_keys(pool[uq], pool, which, np.arange(n), k, L2)[inv], L2, "FLAT 2049 x 140000")
    finally:
        idx.close()


# ---- nlist and nprobe -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nlist", [1, 63, 64, 129, 65536])
def test_nlist_and_nprobe(monkeypatch, nlist):
    d, metric = 32, L2
    n = max(20000, 4 * nlist)
    db, xq = FC.regime("offset1000", n, d, 64, seed=nlist)
    cent = db[np.random.default_rng(nlist).choice(n, nlist, replace=False)]
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 1, "metric_type": "L2"})
    try:
        idx.set_centroids(cent)
        idx.add(db)
        off, _, ids = idx.export_lists()
        for nprobe in sorted({p for p in (1, 64, 65, nlist) if p <= min(nlist, 4096)}):
            check_coarse(monkeypatch, idx, xq, cent, metric, d, nprobe, f"nlist={nlist} nprobe={nprobe}")
        if nlist == 65536:  # add-time assignment (dist_argmin): within the direct margin of the fp64-nearest centroid
            el = np.repeat(np.arange(nlist), np.diff(off))
            assign = np.empty(n, np.int64)
            assign[ids] = el
            for r0 in range(0, 4096, 512):
                rows = db[r0:r0 + 512]
                f, ad = FC.scores64(rows, cent, L2)
                m = FC.direct_margin(f, ad, d, L2)
                j = np.arange(len(rows))
                a, b = assign[r0:r0 + len(rows)], f.argmin(1)
                assert np.all(f[j, a] - m[j, a] <= f[j, b] + m[j, b]), f"rows {r0}..: assigned beyond the margin"
    finally:
        idx.close()


# ---- scratch bound --------------------------------------------------------------------------------------------------
def pool_peak(search):
    gidx = gi()
    used0, _ = gidx.pool_usage(reset_peak=True)
    out = search()
    _, peak = gidx.pool_usage()
    return out, peak - used0


def test_query_major_partials_are_bounded():
    """one 2^20-row list in 4096: its 128 splits per probe used to multiply every query's partials (2048 x 16 x 128 x
    4096 keys, 137 GB); the batch now scans in query blocks of at most 1 GiB of partials"""
    d, nlist, nq, nprobe, k, small = 32, 4096, 2048, 16, 4096, 8
    big, which, pool = pool_rows(1 << 20, d, seed=16)
    rng = np.random.default_rng(17)
    cent = np.zeros((nlist, d), F32)
    cent[0] = np.rint(pool.mean(0))
    # apart enough that every small row lands on its own centroid, small enough that scores stay below 2^24
    cent[1:] = 8 + rng.integers(0, 64, (nlist - 1, d)) * 4
    rest = np.repeat(cent[1:], small, 0) + rng.integers(0, 4, ((nlist - 1) * small, d))
    db = np.concatenate([big, rest]).astype(F32)
    idx = ivfflat("IVFFLAT", d, nlist, L2, db, cent)
    try:
        off, _, ids, el = entries(idx, nlist)
        assert off[1] == 1 << 20 and np.all(np.diff(off)[1:] == small)
        probes = 1 + (np.arange(nq)[:, None] * nprobe + np.arange(nprobe)[None, :]) % (nlist - 1)
        probes[::256, 0] = 0  # 8 queries also probe the long list
        xq = (cent[probes[:, 0]] + rng.integers(0, 4, (nq, d))).astype(F32)
        got, peak = pool_peak(lambda: idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, F32)))
        assert idx.last_scan_kernel == GENERIC
        nparts = nprobe * -(-(1 << 20) // CHUNK_ROWS)
        qb = max(1, min(nq, PARTIAL_BUDGET // (nparts * k * 8)))
        # partials, the list-major and final keys, the decoded scores and ids, queries and probes
        bound = qb * nparts * k * 8 + 2 * nq * k * 8 + nq * k * 12 + (32 << 20)
        assert peak <= bound, (peak, bound)
        ref = np.empty((nq, k), np.uint64)
        for q in range(nq):
            sel = np.concatenate([np.arange(off[l], off[l + 1]) for l in probes[q]])
            kk = np.sort(R.keys(R.exact_scores(xq[q:q + 1], db[ids[sel]], L2), ids[sel][None, :], None, L2)[0])[:k]
            ref[q] = R.SENTINEL
            ref[q, :len(kk)] = kk
        assert_results(got, ref, L2, "2^20-row list, k = 4096")
    finally:
        idx.close()


def test_flat_chunk_partials_are_bounded():
    """8192 queries over 5 row chunks at k = 4096: 1.34 GB of chunk partials, now merged in query blocks of <= 1 GiB"""
    d, n, nq, k = 8, 600000, 8192, 4096
    db, which, pool = pool_rows(n, d, seed=18)
    idx = gi().GammaIndex("FLAT", d, {"metric_type": "L2"})
    try:
        idx.add(db)
        qi = np.random.default_rng(19).integers(0, 64, nq)
        got, peak = pool_peak(lambda: idx.search(pool[qi], k))
        assert idx.last_scan_kernel == BRUTE
        nch = -(-n // 131072)
        ldo = 131072
        scores = min(nq, (1 << 28) // ldo) * ldo * 4
        pb = min(nq, PARTIAL_BUDGET // (nch * k * 8))
        assert nq * nch * k * 8 > PARTIAL_BUDGET >= pb * nch * k * 8
        bound = scores + pb * nch * k * 8 + nq * k * (8 + 12) + (32 << 20)  # score tile, partials, keys, decoded
        assert peak <= bound, (peak, bound)
        uq, inv = np.unique(qi, return_inverse=True)
        assert_results(got, pooled_keys(pool[uq], pool, which, np.arange(n), k, L2)[inv], L2, "FLAT partials")
    finally:
        idx.close()
