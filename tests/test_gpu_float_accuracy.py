"""Every floating-point search path against fp64 within the error its arithmetic allows (tests/float_contract.py), on
ill-conditioned float data: clustered rows with a common offset of 100 and 1000, SIFT-like floats, unit embeddings
scaled by 2^+-40, per-dimension scales over 2^+-10 and near-duplicate rows.  Each case asserts the kernel that served
it.  IVF searches go through search_preassigned with probes chosen exactly in fp64, so a case tests the list scan and
nothing else.

The list-major IVF-Flat kernels select on the expanded form |x - s|^2 + |y - s|^2 - 2 (x - s).(y - s) over operands
shifted by the list shift s_l; their selection margin is the expanded margin over those shifted operands plus the
direct margin of the re-score.  Kernels that stage the raw operands instead break the contract on the offset regimes,
even against margins computed as if s_l were the centroid.

IVF-PQ: the exact re-rank against fp64 over its ADC candidates, and the tensor-core filter (pqtc_scan_kernel) against the
LUT kernel of small batches, key for key, on adversarial scales: offsets, 2^+-30, codebooks over 2^+-10 and 2^-64, where
the squared terms are subnormal in fp32."""
import numpy as np
import pytest

import float_contract as FC

pytestmark = pytest.mark.gpu
L2, IP = FC.METRIC_L2, FC.METRIC_IP
METRICS = [L2, IP]


def gi():
    from vearch_b200 import index as gidx
    return gidx


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


def best(f, k, metric):
    return np.argsort(f if metric == L2 else -f, axis=1, kind="stable")[:, :k]


# ---- FLAT and the distance tiles --------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d,n", [(30, 140000), (128, 20000), (1536, 6000)])  # 140000: two distance chunks
@pytest.mark.parametrize("name", FC.REGIMES)
def test_flat(name, d, n, metric):
    db, xq = FC.regime(name, n, d, 3, seed=d)
    idx = gi().GammaIndex("FLAT", d, {"metric_type": mt(metric)})
    try:
        idx.add(db)
        f, ad = FC.scores64(xq, db, metric)
        md = FC.direct_margin(f, ad, d, metric)
        cand = np.arange(n)
        for k in (1, 10, 100):
            got = idx.search(xq, k)
            assert idx.last_scan_kernel == "dist_tile_kernel+select_rows_kernel"
            FC.check_all(got, lambda q: (cand, f[q], md[q], md[q]), k, metric, f"FLAT {name} d={d} k={k}")
    finally:
        idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("name", FC.REGIMES)
def test_dist_tiles(name, d, metric):
    # element-wise: the exact kernel within the direct margin, dist_tc_kernel within the expanded (L2) or 3xTF32 dot (IP)
    # margin with C_TC -- the model constant of wgmma's fp32 accumulation is checked here, on every regime
    db, xq = FC.regime(name, 700, d, 300, seed=3)
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


# ---- coarse quantiser -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", FC.REGIMES)
def test_coarse(monkeypatch, name, metric):
    d, nlist, nprobe = 128, 512, 16
    cent, xq = FC.regime(name, nlist, d, 64, seed=9)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": mt(metric)})
    try:
        idx.set_centroids(cent)
        f, ad = FC.scores64(xq, cent, metric)
        na, nb = (xq.astype(np.float64) ** 2).sum(1)[:, None], (cent.astype(np.float64) ** 2).sum(1)[None, :]
        tcm = FC.expanded_l2_margin(ad, na, nb, f, d) if metric == L2 else FC.tc_dot_margin(ad, d)
        dm = FC.direct_margin(f, ad, d, metric)
        cand = np.arange(nlist)
        # the fused kernel and the score matrix (nq >= 32: 3xTF32 expanded form, as faiss's IndexFlat BLAS path), the
        # exact kernel below 32 queries
        for path, nq, m in (("coarse_topk_kernel", 64, tcm), ("dist_tc_kernel+select_rows_kernel", 64, tcm),
                            ("dist_tile_kernel+select_rows_kernel", 31, dm)):
            if path.startswith("dist_tc"):
                monkeypatch.setenv("GB_COARSE_FUSED", "0")
            dis, ids = idx.coarse_search(xq[:nq], nprobe)
            monkeypatch.delenv("GB_COARSE_FUSED", raising=False)
            assert idx.last_coarse_kernel == path, (path, idx.last_coarse_kernel)
            FC.check_all((dis, ids), lambda q: (cand, f[q], m[q], m[q]), nprobe, metric, f"coarse {path} {name}",
                         ip_ties_desc=False)
    finally:
        idx.close()


# ---- IVF-Flat ---------------------------------------------------------------------------------------------------------
class IvfFlat:
    """an IVFFLAT index on float centroids (rows of db), exact fp64 probes, a deletion bitmap, per-query candidates"""

    def __init__(self, name, d, n, nq, nlist, nprobe, metric, seed):
        self.metric, self.d, self.nprobe = metric, d, nprobe
        self.db, self.xq = FC.regime(name, n, d, nq, seed=seed)
        rng = np.random.default_rng(seed)
        self.cent = self.db[rng.choice(n, nlist, replace=False)]
        self.idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": nprobe, "metric_type": mt(metric)})
        self.idx.set_centroids(self.cent)
        self.idx.add(self.db)
        self.refresh()
        fc, _ = FC.scores64(self.xq, self.cent, metric)
        self.probes = best(fc, nprobe, metric).astype(np.int64)
        self.deleted = rng.random(n) < 0.1

    def refresh(self):
        off, _, ids = self.idx.export_lists()
        self.off, self.ids = off, ids
        self.shifts = self.idx.get_list_shifts() if self.metric == L2 else None  # IP: scanned unshifted
        self.cache = {}

    def candidates(self, q, listmajor, deleted=None):
        """(cand, f, m, md) of query q over its probed lists"""
        key = (q, listmajor, deleted is not None)
        if key not in self.cache:
            self.cache[key] = self.candidates_of(q, listmajor, deleted)
        return self.cache[key]

    def candidates_of(self, q, listmajor, deleted):
        parts = []
        for l in self.probes[q]:
            raw = self.ids[self.off[l]:self.off[l + 1]]
            vid = raw[raw >= 0]
            if deleted is not None:
                vid = vid[~deleted[vid]]
            parts.append((l, vid))
        cand = np.concatenate([v for _, v in parts])
        f, ad = FC.scores64(self.xq[q:q + 1], self.db[cand], self.metric)
        f, ad = f[0], ad[0]
        md = FC.direct_margin(f, ad, self.d, self.metric)
        if not listmajor:
            return cand, f, md, md
        if self.metric == IP:
            return cand, f, FC.tc_dot_margin(ad, self.d) + md, md
        m = np.empty_like(f)
        o = 0
        for l, vid in parts:
            na, nb, sad = FC.shifted_operands(self.xq[q:q + 1], self.db[vid], self.shifts[l])
            m[o:o + len(vid)] = FC.shifted_l2_margin(sad[0], na[0], nb[0], f[o:o + len(vid)], self.d)
            o += len(vid)
        return cand, f, m + md, md

    def search(self, k, q=slice(None), **kw):
        xq = self.xq[q]
        return self.idx.search_preassigned(xq, k, self.probes[q], np.zeros(self.probes[q].shape, np.float32), **kw)

    def check(self, got, k, listmajor, what, q0=0, deleted=None, **window):
        FC.check_all(got, lambda q: self.candidates(q0 + q, listmajor, deleted), k, self.metric, what, **window)

    def window(self, k):
        """a score window whose edge cuts query 0's top-k"""
        cand, f, _, _ = self.candidates(0, False)
        e = float(np.sort(f)[k // 2] if self.metric == L2 else -np.sort(-f)[k // 2])
        return {"max_score": e} if self.metric == L2 else {"min_score": e}


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", FC.REGIMES)
def test_ivfflat_list_major(name, metric):
    s = IvfFlat(name, 128, 20000, 128, 16, 4, metric, seed=21)  # 32 (query, probe) pairs per list
    try:
        for k, kern in ((10, "ivf_listmajor_tma_kernel"), (48, "ivf_listmajor_pipe_kernel"),
                        (100, "ivf_listmajor_tc_kernel+seg_select_kernel")):
            got = s.search(k)
            assert s.idx.last_scan_kernel == kern, (k, s.idx.last_scan_kernel)
            s.check(got, k, True, f"list-major {name} k={k}")
            bm = np.packbits(~s.deleted, bitorder="little")
            got = s.search(k, filter_bitmap=bm)
            assert s.idx.last_scan_kernel == kern
            s.check(got, k, True, f"list-major {name} k={k} bitmap", deleted=s.deleted)
            w = s.window(k)
            got = s.search(k, **w)
            assert s.idx.last_scan_kernel == kern
            s.check(got, k, True, f"list-major {name} k={k} window", **w)
        # the answer must not depend on the batch: the same queries in 3-query batches run query-major
        for q0 in range(0, 6, 3):
            got = s.search(10, slice(q0, q0 + 3))
            assert s.idx.last_scan_kernel.startswith("ivfflat_scan"), s.idx.last_scan_kernel
            s.check(got, 10, False, f"query-major batch {name}", q0=q0)
        # brute force of the same index: the exact FLAT tiles over every row
        got = s.idx.search(s.xq[:4], 10, brute_force=True)
        assert s.idx.last_scan_kernel == "dist_tile_kernel+select_rows_kernel"
        f, ad = FC.scores64(s.xq[:4], s.db, metric)
        md = FC.direct_margin(f, ad, 128, metric)
        cand = np.arange(len(s.db))
        FC.check_all(got, lambda q: (cand, f[q], md[q], md[q]), 10, metric, f"brute force {name}")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", FC.REGIMES)
def test_ivfflat_list_major_d16(name, metric):
    s = IvfFlat(name, 16, 20000, 128, 16, 4, metric, seed=22)  # d = 16: the register-staged pipeline even at k <= 32
    try:
        got = s.search(10)
        assert s.idx.last_scan_kernel == "ivf_listmajor_pipe_kernel"
        s.check(got, 10, True, f"list-major d=16 {name}")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d,kern", [(64, "ivfflat_scan_warp_kernel"), (128, "ivfflat_scan_warp_kernel"),
                                    (20, "ivfflat_scan_kernel"), (100, "ivfflat_scan_kernel")])
@pytest.mark.parametrize("name", FC.REGIMES)
def test_ivfflat_query_major(name, d, kern, metric):
    s = IvfFlat(name, d, 20000, 6, 32, 8, metric, seed=d)
    try:
        for k in (1, 10, 100):
            got = s.search(k)
            assert s.idx.last_scan_kernel == kern, (k, s.idx.last_scan_kernel)
            s.check(got, k, False, f"query-major {name} d={d} k={k}")
        bm = np.packbits(s.deleted, bitorder="little")
        got = s.search(10, del_bitmap=bm)
        assert s.idx.last_scan_kernel == kern
        s.check(got, 10, False, f"query-major {name} d={d} deleted", deleted=s.deleted)
        w = s.window(10)
        got = s.search(10, **w)
        assert s.idx.last_scan_kernel == kern
        s.check(got, 10, False, f"query-major {name} d={d} window", **w)
    finally:
        s.idx.close()


def test_ivfflat_list_major_append_and_update():
    # rows appended in small batches after the mirror is built go through tc_mirror_append_kernel, which must stage them
    # with their list's shift; an update re-appends the row.  The new rows sit right next to the queries, so they must
    # be found: staged unshifted, their expanded-form scores would be off by far more than the gaps
    s = IvfFlat("offset1000", 128, 20000, 128, 16, 4, L2, seed=23)
    try:
        n0 = len(s.db)
        s.check(s.search(10), 10, True, "before appends")
        builds = s.idx.mirror_builds
        rng = np.random.default_rng(24)
        # one row next to each of the first 64 queries, in batches of 16: few enough per list for the mirror's reserve
        extra = (s.xq[:64] + 0.05 * rng.standard_normal((64, 128))).astype(np.float32)
        for a in range(0, 64, 16):
            s.idx.add(extra[a:a + 16])
        moved = (s.xq[5] + 0.01 * rng.standard_normal(128)).astype(np.float32)
        s.idx.update_vector(7, moved)
        s.db = np.concatenate([s.db, extra])
        s.db[7] = moved
        s.refresh()
        got = s.search(10)
        assert s.idx.last_scan_kernel == "ivf_listmajor_tma_kernel"
        assert s.idx.mirror_builds == builds, "the appends should fit the mirror's reserve"
        s.check(got, 10, True, "after appends and an update")
        found = np.array([n0 + q in got[1][q] for q in range(64)])
        assert found.mean() > 0.9, f"rows appended next to queries found for only {found.sum()} of 64"
        assert 7 in got[1][5], "the updated row sits next to query 5"
    finally:
        s.idx.close()


def test_ivfflat_list_major_mirror_follows_centroids():
    # new centroids give new shifts: a mirror staged with the old ones must be rebuilt before the next list-major search
    s = IvfFlat("offset1000", 128, 20000, 128, 16, 4, L2, seed=25)
    try:
        s.check(s.search(10), 10, True, "before")
        builds = s.idx.mirror_builds
        old = s.shifts
        s.idx.set_centroids(s.cent + np.float32(3.0))
        s.refresh()
        assert not np.array_equal(s.shifts, old)
        got = s.search(10)
        assert s.idx.last_scan_kernel == "ivf_listmajor_tma_kernel"
        assert s.idx.mirror_builds == builds + 1, "the mirror kept the old shifts"
        s.check(got, 10, True, "after set_centroids")
    finally:
        s.idx.close()


# ---- the list shifts --------------------------------------------------------------------------------------------------
def grid(cent):
    """g_l: the largest power of two <= rho_l / sqrt(d), rho_l half the distance to the nearest other centroid"""
    c = cent.astype(np.float64)
    f = ((c[:, None, :] - c[None, :, :]) ** 2).sum(-1)
    np.fill_diagonal(f, np.inf)
    t = f.min(1) / 4 / c.shape[1]
    ok = np.isfinite(t) & (t > 0)  # rho = 0, or no other centroid (nlist = 1): s = c
    e = np.frexp(np.where(ok, t, 1.0))[1] - 1
    return np.where(ok, np.ldexp(1.0, np.floor_divide(e, 2)), 0.0)


def assert_shifts(s, cent, what):
    g = grid(cent)
    for l in range(len(cent)):
        if g[l] == 0:
            assert np.array_equal(s[l], cent[l]), what
        else:
            assert np.max(np.abs(s[l].astype(np.float64) - cent[l])) <= g[l] / 2, (what, l)
    integer = np.all(cent == np.rint(cent), axis=1)
    assert np.all(s[integer] == np.rint(s[integer])), f"{what}: integer centroid, fractional shift"


def test_list_shifts(tmp_path):
    d, nlist = 64, 64
    db, _ = FC.regime("offset1000", 8000, d, 1, seed=31)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 4, "metric_type": "L2",
                                         "training_threshold": 4000})
    try:
        cent = db[:nlist].copy()
        cent[::2] = np.rint(cent[::2])  # integer centroids keep integer shifts
        cent[5] = cent[4]                # rho = 0: the shift is the centroid
        idx.set_centroids(cent)
        s0 = idx.get_list_shifts()
        assert_shifts(s0, cent, "set_centroids")
        idx.add(db)
        assert np.array_equal(idx.get_list_shifts(), s0), "adds changed the shifts"
        idx.set_centroids(cent + np.float32(0.5))
        assert_shifts(idx.get_list_shifts(), cent + np.float32(0.5), "set_centroids again")
        idx.dump(tmp_path, "f")
        tr = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 4, "metric_type": "L2",
                                            "training_threshold": 4000})
        tr.add_vectors(db)
        tr.train()
        assert_shifts(tr.get_list_shifts(), tr.get_centroids(), "train")
        tr.close()
        ld = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 4, "metric_type": "L2"})
        ld.add_vectors(db)
        assert ld.load(tmp_path, "f") > 0
        assert np.array_equal(ld.get_list_shifts(), idx.get_list_shifts()), "load"
        ld.close()
        one = gi().GammaIndex("IVFFLAT", d, {"ncentroids": 1, "nprobe": 1, "metric_type": "L2"})
        one.set_centroids(cent[:1])
        assert_shifts(one.get_list_shifts(), cent[:1], "nlist = 1")
        one.close()
        ip = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 4, "metric_type": "InnerProduct"})
        with pytest.raises(gi().GammaError):  # inner product: scanned unshifted, no shift table
            ip.get_list_shifts()
        ip.close()
    finally:
        idx.close()


def test_metric_override_declines_list_major():
    # the mirror of an L2 index is shifted: a search under inner product scans query-major, within the direct margin
    s = IvfFlat("offset100", 128, 20000, 128, 16, 4, L2, seed=41)
    try:
        got = s.search(10, params={"metric_type": "InnerProduct"})
        assert s.idx.last_scan_kernel.startswith("ivfflat_scan"), s.idx.last_scan_kernel
        s.metric = IP
        s.check(got, 10, False, "L2 index searched under IP")
    finally:
        s.idx.close()


# ---- IVF-PQ -----------------------------------------------------------------------------------------------------------
PQTC_SHAPES = [(16, 8), (8, 16), (8, 8), (16, 4), (4, 16), (4, 32), (4, 8), (8, 4)]  # every (M, dsub) pqtc_supported takes


def pq_data(name, d, n, nq, seed):
    """(db, xq, codebook scale per sub-quantiser) of one adversarial IVF-PQ regime"""
    from vearch_b200 import synth
    if name in ("scaled_hi30", "scaled_lo30", "subnormal"):  # 2^-64: squared terms below fp32's normal range
        sc = {"scaled_hi30": 2.0 ** 30, "scaled_lo30": 2.0 ** -30, "subnormal": 2.0 ** -64}[name]
        db = synth.embed_like(n, d, seed=seed).astype(np.float64) * sc
        xq = synth.embed_like(nq, d, seed=seed + 1).astype(np.float64) * sc
        return db.astype(np.float32), xq.astype(np.float32), None
    if name == "codebook_span":  # sub-quantisers whose magnitudes span 2^+-10
        db, xq = FC.regime("offset100", n, d, nq, seed)
        return db - np.float32(100), xq - np.float32(100), 2.0 ** np.random.default_rng(seed).uniform(-10, 10, d)
    db, xq = FC.regime(name, n, d, nq, seed)
    return db, xq, None


class IvfPq:
    """an IVFPQ index (8-bit codes) on centroids drawn from db and a codebook of residual slices, exact fp64 probes"""

    def __init__(self, db, xq, M, nlist, nprobe, metric, seed, span=None):
        rng = np.random.default_rng(seed)
        n, d = db.shape
        self.db, self.xq, self.metric = db, xq, metric
        cent = db[rng.choice(n, nlist, replace=False)]
        fc, _ = FC.scores64(db[:4000], cent, L2)
        resid = db[:4000] - cent[fc.argmin(1)]
        pq = resid[rng.choice(len(resid), 256, replace=False)].reshape(256, M, d // M).transpose(1, 0, 2).copy()
        if span is not None:
            pq *= span.reshape(M, 1, d // M)[:, :, :1].astype(np.float32)
        self.idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M,
                                                "metric_type": mt(metric)})
        self.idx.set_centroids(cent)
        self.idx.set_pq_centroids(pq.astype(np.float32))
        self.idx.add(db)
        fq, _ = FC.scores64(xq, cent, metric)
        self.probes = best(fq, nprobe, metric).astype(np.int64)
        self.cd = np.take_along_axis(fq, self.probes, 1).astype(np.float32)

    def search(self, k, q=slice(None), **kw):
        return self.idx.search_preassigned(self.xq[q], k, self.probes[q], self.cd[q], **kw)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("M,dsub", PQTC_SHAPES)
@pytest.mark.parametrize("name", ["offset1000", "scaled_hi30", "scaled_lo30", "codebook_span", "subnormal"])
def test_ivfpq_filter_adversarial_scales(name, M, dsub, metric):
    # the filter's bound is claimed rigorous, so its ADC keys must be byte-equal to the exact LUT kernel's
    d = M * dsub
    db, xq, span = pq_data(name, d, 20000, 128, seed=M * 100 + dsub)
    s = IvfPq(db, xq, M, 16, 6, metric, seed=7, span=span)
    try:
        for k in (10, 100):
            dg, ig = s.search(k)
            assert s.idx.last_scan_kernel == "pqtc_scan_kernel", s.idx.last_scan_kernel
            parts = []
            for q0 in range(0, len(xq), 3):
                parts.append(s.search(k, slice(q0, q0 + 3)))
                assert s.idx.last_scan_kernel == "ivfpq_scan_kernel", s.idx.last_scan_kernel
            ds, is_ = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
            bad = np.nonzero(np.any(dg.view(np.uint32) != ds.view(np.uint32), 1) | np.any(ig != is_, 1))[0]
            assert len(bad) == 0, (f"{name} M={M} dsub={dsub} k={k}: {len(bad)}/{len(xq)} queries differ from the LUT "
                                   f"kernel; query {bad[0]}: {ig[bad[0]][:5]} vs {is_[bad[0]][:5]}")
    finally:
        s.idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("name", ["offset100", "offset1000", "scaled_hi", "scaled_lo"])
def test_ivfpq_exact_rerank(name, metric):
    # recall_num 400: the final top-10 is the exact (direct-form) best of the ADC candidates -- the same index searched at
    # k = 400 without re-rank
    db, xq = FC.regime(name, 20000, 128, 128, seed=51)
    s = IvfPq(db, xq, 16, 16, 6, metric, seed=8)
    try:
        _, ic = s.search(400)
        assert s.idx.last_scan_kernel == "pqtc_scan_kernel"
        got = s.search(10, params={"recall_num": 400})
        assert s.idx.last_scan_kernel == "pqtc_scan_kernel"

        def per_query(q):
            cand = ic[q][ic[q] >= 0]
            f, ad = FC.scores64(xq[q:q + 1], db[cand], metric)
            md = FC.direct_margin(f[0], ad[0], 128, metric)
            return cand, f[0], md, md

        FC.check_all(got, per_query, 10, metric, f"IVF-PQ re-rank {name}")
    finally:
        s.idx.close()
