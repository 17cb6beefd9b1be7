"""The two-pass exact re-rank (rerank_prefilter_kernel) at its limits, candidate by candidate, through the test hooks
index.debug_shadow_rows (the int8 shadow rows the raw store keeps) and index.debug_rerank (the re-rank of caller-given
candidates by either kernel, with each candidate's pass-1 interval).  Held against the numpy restatement of the bound
(test_rerank_prefilter_cpu.py, rerank_reference.py) and the key-exact CPU re-rank (topk_reference.rerank_keys):

* shadow rows follow encode() at every row width the kernels see (nch < 8 idle lanes, nch not a multiple of 8, zero
  padding between d, dpad and cols16, long chunk loops), in every float regime and at the encoder's edges;
* every interval holds the one-pass fp32 score and equals the restated interval of the device's own shadow bytes;
* keys are the one-pass kernel's and the CPU re-rank's at every candidate depth up to the launcher's 8192, with
  sentinels anywhere, bitmaps, score windows, and survivor counts on both sides of the 32-key sort;
* the same holds through search at each shadow type's deepest recall_num, and past the first raw-store segment."""
import re

import numpy as np
import pytest

import float_contract as FC
import rerank_reference as RR
import topk_reference as R
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
F32 = np.float32
L2, IP = R.METRIC_L2, R.METRIC_IP
MNAME = {L2: "L2", IP: "InnerProduct"}
DIMS = [1, 3, 4, 12, 16, 17, 30, 100, 112, 128, 129, 768, 1536, 4096]
NC = 2048  # candidates per query of the interval tests


def gi():
    from vearch_b200 import index as gidx
    return gidx


def holder(typ, d, metric, **extra):
    """an index whose raw store keeps shadow rows; debug_rerank and debug_shadow_rows need no training"""
    p = dict(ncentroids=4, nprobe=4, metric_type=MNAME[metric], **extra)
    if typ == "IVFRABITQ":
        return gi().RaBitQIndex(d, dict({"nb_bits": 4}, **p))
    if typ == "VEARCH":
        return gi().VearchIndex(d, dict({"nsubvector": 16, "reordering": True}, **p))
    return gi().GammaIndex(typ, d, dict({"nsubvector": 16}, **p))


def edge_rows(d, rng):
    """rows at the encoder's edges: zero, one dominant component, scales 2^30, 2^-30 and 2^-64, a row whose scale is
    subnormal, one whose scale rounds to 0 (unbounded) and one nearly so"""
    base = rng.standard_normal((6, d))
    one = np.zeros(d)
    one[d // 2] = 7.0
    big = np.zeros(d)
    big[0] = 1e3
    big += 1e-3 * rng.standard_normal(d)
    rows = [np.zeros(d), one, big, base[0] * 2.0 ** 30, base[1] * 2.0 ** -30, base[2] * 2.0 ** -64,
            base[3] / np.abs(base[3]).max() * 2.0 ** -130]
    tiny = np.zeros((2, d))
    tiny[0, 0] = 50 * 2.0 ** -149  # s = 50 / 127 ulps of the smallest subnormal: rounds to 0
    tiny[1, -1] = -70 * 2.0 ** -149  # rounds to the smallest subnormal: bounded
    return np.concatenate([np.array(rows), tiny]).astype(F32)


def regime_block(name, d, n, nq, seed):
    """n rows (the regime's, then the edge rows) and nq queries (the regime's, then one in the 2^-64 range)"""
    rng = np.random.default_rng(seed)
    edge = edge_rows(d, rng)
    db, xq = FC.regime(name, n - len(edge), d, nq - 1, seed=seed)
    db = np.concatenate([db, edge])
    return db, np.concatenate([xq, edge[5:6] * F32(1.5)])


def shadow_of(idx, vids):
    vids = np.asarray(vids, np.int64)
    rows = [idx.debug_shadow_rows(int(v), 1) for v in vids]
    return (np.concatenate([r[0] for r in rows]),) + tuple(np.concatenate([r[i] for r in rows]) for i in (1, 2, 3))


def assert_shadow(idx, db, start=0, vids=None, what=""):
    if vids is None:
        got = idx.debug_shadow_rows(start, len(db))
    else:
        got = shadow_of(idx, vids)
    err = RR.shadow_mismatch(RR.pad4(db), *got)
    assert err is None, f"{what}: {err}"


def same_results(a, b):
    return np.array_equal(a["dis"].view(np.uint32), b["dis"].view(np.uint32)) and np.array_equal(a["ids"], b["ids"])


def want_results(want, metric):
    dis, ids = R.decode(want, metric)
    return {"dis": dis, "ids": ids}


# ---- 1. shadow rows ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DIMS)
def test_shadow_rows_follow_encode(d):
    blocks = [regime_block(name, d, 64, 2, seed=40 + i)[0] for i, name in enumerate(FC.REGIMES)]
    db = np.concatenate(blocks)
    idx = holder("IVFRABITQ", d, L2)
    idx.add_vectors(db)
    assert_shadow(idx, db, what=f"d={d}")
    idx.close()


@pytest.mark.parametrize("typ", ["IVFPQ", "IVFPQFastScan", "VEARCH"])
def test_shadow_rows_of_each_type(typ):
    db = np.concatenate([regime_block(name, 128, 64, 2, seed=60 + i)[0] for i, name in enumerate(FC.REGIMES)])
    idx = holder(typ, 128, L2)
    idx.add_vectors(db)
    assert_shadow(idx, db, what=typ)
    idx.close()


# ---- 2. intervals, per candidate -----------------------------------------------------------------------------------
def check_intervals(idx, db, xq, cand, metric, what, k=10):
    """cand [nq, ncand] vids (-1: none) into db; every candidate's interval against the one-pass score and the
    restatement of the device's own shadow row; the survivor count against the intervals; keys of both kernels"""
    two = idx.debug_rerank(xq, cand, k)
    one_all = idx.debug_rerank(xq, cand, cand.shape[1], two_pass=False)
    one = idx.debug_rerank(xq, cand, k, two_pass=False)
    assert same_results(two, one), f"{what}: the two kernels' keys differ"
    xp = RR.pad4(xq)
    live = cand >= 0
    assert np.all((two["state"] == RR.DEAD) == ~live), what
    for q in range(len(xq)):
        vids = cand[q][live[q]]
        # the one-pass score of every live candidate, and the direct fp32 form restated
        by_vid = dict(zip(one_all["ids"][q].tolist(), one_all["dis"][q].tolist()))
        ref = np.array([by_vid[v] for v in vids.tolist()], F32)
        direct = RR.direct_fp32(xp[q:q + 1], RR.pad4(db[vids]), metric)[0]
        assert np.array_equal(ref.view(np.uint32), direct.view(np.uint32)), f"{what} q{q}: one-pass scores"
        lo, hi, st = two["lo"][q][live[q]], two["hi"][q][live[q]], two["state"][q][live[q]]
        qy, s, e, nrm = gather_shadow(idx, vids)
        lo_min, lo_max, hi_min, hi_max, bounded = (a[0] for a in RR.brackets(xp[q:q + 1], qy, s, e, nrm, metric))
        bounded &= np.isfinite(e)
        assert np.array_equal(st == RR.UNBOUNDED, ~bounded), f"{what} q{q}: unbounded candidates"
        b = st == RR.BOUNDED
        assert np.all(st[~b] == RR.UNBOUNDED), what
        # sound: the interval holds the score the one-pass kernel computes
        bad = np.nonzero(b & ~((lo <= ref) & (ref <= hi)))[0]
        assert not len(bad), (f"{what} q{q}: {len(bad)} intervals miss the fp32 score; first: vid {vids[bad[0]]}, "
                              f"{ref[bad[0]]!r} not in [{lo[bad[0]]!r}, {hi[bad[0]]!r}]")
        # tight: the restated interval of the same shadow row, to the rounding of its fp64 steps
        for name, got, a, z in (("lo", lo, lo_min, lo_max), ("hi", hi, hi_min, hi_max)):
            bad = np.nonzero(b & ~((a <= got) & (got <= z)))[0]
            assert not len(bad), (f"{what} q{q}: {len(bad)} {name} ends differ from the restatement; first: vid "
                                  f"{vids[bad[0]]}, {got[bad[0]]!r} not in [{a[bad[0]]!r}, {z[bad[0]]!r}]")
    assert np.array_equal(two["surv"], RR.expected_survivors(two["lo"], two["hi"], two["state"], k, metric)), what
    return two


def gather_shadow(idx, vids):
    """shadow rows of arbitrary vids: one contiguous read of the range they span"""
    lo, hi = int(vids.min()), int(vids.max()) + 1
    qy, s, e, nrm = idx.debug_shadow_rows(lo, hi - lo)
    j = vids - lo
    return qy[j], s[j], e[j], nrm[j]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d", DIMS)
def test_intervals_hold_and_match_the_restatement(d, metric):
    nq = 2
    blocks = [regime_block(name, d, NC, nq, seed=70 + i) for i, name in enumerate(FC.REGIMES)]
    db = np.concatenate([b[0] for b in blocks])
    xq = np.concatenate([b[1] for b in blocks])
    rng = np.random.default_rng(d)
    cand = np.concatenate([np.tile(np.arange(NC) + i * NC, (nq, 1)) for i in range(len(blocks))])
    cand = rng.permuted(cand, axis=1)
    cand[rng.random(cand.shape) < 0.003] = -1  # dead candidates anywhere
    idx = holder("IVFRABITQ", d, metric)
    idx.add_vectors(db)
    two = check_intervals(idx, db, xq, cand, metric, f"d={d} {MNAME[metric]}")
    # the zero and scale-0 rows are unbounded, ordinary rows bounded; pruning happens
    assert np.mean(two["state"] == RR.BOUNDED) > 0.9 and np.any(two["state"] == RR.UNBOUNDED)
    assert np.median(two["surv"]) < NC / 2
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
def test_overflowing_magnitudes_are_unbounded(metric):
    """scores that stay finite in fp32 but whose bound passes 2^126: every candidate is unbounded, so all survive"""
    d, n = 16, 256
    rng = np.random.default_rng(5)
    sign = np.where(rng.random((n + 2, d)) < 0.5, -1.0, 1.0)
    if metric == L2:  # |q - y|^2 = 16 (1.2 2^61)^2 ~ 2^126.5
        db, xq = (sign[:n] * 1.2 * 2.0 ** 61).astype(F32), np.zeros((2, d), F32)
    else:  # |<q, y>| <= |q| |y| = 16 (1.5 2^61)^2 ~ 2^127.2
        db, xq = (sign[:n] * 1.5 * 2.0 ** 61).astype(F32), (sign[n:] * 1.5 * 2.0 ** 61).astype(F32)
    idx = holder("IVFRABITQ", d, metric)
    idx.add_vectors(db)
    cand = np.tile(np.arange(n), (2, 1))
    two = idx.debug_rerank(xq, cand, 10)
    one = idx.debug_rerank(xq, cand, n, two_pass=False)
    assert np.all(np.isfinite(one["dis"])), "the scores must stay finite"
    assert np.all(two["state"] == RR.UNBOUNDED) and np.all(two["surv"] == n)
    assert same_results(two, idx.debug_rerank(xq, cand, 10, two_pass=False))
    idx.close()


def test_a_lo_equal_to_the_bound_survives():
    """two candidates whose pass-1 ends meet: y's lo equals x's hi, the bound at k = 1, so y must be read (its score
    may tie x's); found among rows one fp32 step apart"""
    d, n = 16, 2048
    a = (1.0 + np.arange(n) * 2.0 ** -23).astype(F32)
    db = np.zeros((n, d), F32)
    db[:, 0] = a
    xq = np.zeros((1, d), F32)
    idx = holder("IVFRABITQ", d, L2)
    idx.add_vectors(db)
    two = idx.debug_rerank(xq, np.arange(n)[None], 1)
    lo, hi = two["lo"][0], two["hi"][0]
    assert np.all(two["state"] == RR.BOUNDED)
    pos = {float(v): i for i, v in enumerate(lo)}
    pairs = [(x, pos[float(hi[x])]) for x in range(n) if float(hi[x]) in pos]
    assert pairs, "no two intervals meet"
    for x, y in pairs[:16]:
        r = idx.debug_rerank(xq, np.array([[x, y]]), 1)
        assert r["lo"][0, 1] == r["hi"][0, 0] and r["surv"][0] == 2, (x, y, r["lo"], r["hi"], r["surv"])
    idx.close()


# ---- 3. keys at every depth ----------------------------------------------------------------------------------------
DEPTHS = [1, 2, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 8192]
KD, KN, KQ = 64, 24_000, 3


@pytest.fixture(scope="module", params=[L2, IP], ids=["L2", "IP"])
def int_index(request):
    """integer-valued sift-like rows (exact fp32 scores) with 40 copies of a row next to each query at vids 20000 +
    40 q ..., for the survivor sets"""
    metric = request.param
    db = np.rint(synth.sift_like(KN, KD, seed=3) / 8)
    xq = np.rint(synth.sift_like(KQ, KD, seed=4) / 8)
    if metric == IP:
        db, xq = db - 16, xq - 16
    for q in range(KQ):
        near = xq[q] * (4 if metric == IP else 1)
        near[q] += 1
        db[20_000 + 40 * q:20_000 + 40 * (q + 1)] = near
    db, xq = db.astype(F32), xq.astype(F32)
    idx = holder("IVFPQ", KD, metric, nsubvector=8)
    idx.add_vectors(db)
    yield metric, idx, db, xq
    idx.close()


def check_keys(idx, db, xq, cand, k, metric, what, **kw):
    """both kernels' keys against the CPU re-rank; returns the two-pass run"""
    adc = np.where(cand >= 0, cand, 0).astype(np.uint64)
    adc = np.where(cand >= 0, adc, R.SENTINEL)
    want = want_results(R.rerank_keys(adc, xq, db, k, metric, **kw), metric)
    two = idx.debug_rerank(xq, cand, k, **kw)
    one = idx.debug_rerank(xq, cand, k, two_pass=False, **kw)
    for name, got in (("two-pass", two), ("one-pass", one)):
        bad = np.nonzero(~(np.all(got["dis"].view(np.uint32) == want["dis"].view(np.uint32), 1) &
                           np.all(got["ids"] == want["ids"], 1)))[0]
        assert not len(bad), f"{what}: {name} keys differ from the CPU re-rank (first: query {bad[0]})"
    assert np.array_equal(two["surv"], RR.expected_survivors(two["lo"], two["hi"], two["state"], k, metric)), what
    return two


@pytest.mark.parametrize("ncand", DEPTHS)
def test_keys_at_every_depth(int_index, ncand):
    metric, idx, db, xq = int_index
    rng = np.random.default_rng(ncand)
    n = len(db)
    cand = np.stack([rng.choice(n, ncand, replace=False) for _ in range(KQ)])
    cand[:, :min(ncand, 40)] = 20_000 + 40 * np.arange(KQ)[:, None] + np.arange(min(ncand, 40))  # ties at the top
    cand = rng.permuted(cand, axis=1)
    if ncand > 1:
        cand[rng.random(cand.shape) < 0.06] = -1  # sentinels anywhere
    dead = np.packbits(rng.random(n) < 0.3, bitorder="little")
    keep = np.packbits(rng.random(n) < 0.5, bitorder="little")
    s = np.sort(np.concatenate([R.exact_scores(xq[q:q + 1], db[cand[q][cand[q] >= 0]], metric)[0]
                                for q in range(KQ)]))
    a, b = float(s[len(s) // 8]), float(s[len(s) // 2])
    for k in sorted({1, 10, ncand} & set(range(1, ncand + 1))):
        w = f"{MNAME[metric]} ncand={ncand} k={k}"
        check_keys(idx, db, xq, cand, k, metric, w)
        check_keys(idx, db, xq, cand, k, metric, w + " deletion bitmap", del_bitmap=dead)
        check_keys(idx, db, xq, cand, k, metric, w + " filter bitmap", filter_bitmap=keep)
        check_keys(idx, db, xq, cand, k, metric, w + " window", min_score=a, max_score=b)
        check_keys(idx, db, xq, cand, k, metric, w + " single-point window", min_score=a, max_score=a)
        # a window no score meets: no results; every live candidate is read (none bounds the k-th result)
        r = check_keys(idx, db, xq, cand, k, metric, w + " empty window", min_score=0.5, max_score=0.5)
        assert np.all(r["ids"] == -1) and np.array_equal(r["surv"], (cand >= 0).sum(1)), w
        # every candidate screened out by the filter: nothing to read
        none = np.zeros_like(keep)
        r = check_keys(idx, db, xq, cand, k, metric, w + " empty filter", filter_bitmap=none)
        assert np.all(r["surv"] == 0) and np.all(r["state"] == RR.DEAD), w


@pytest.mark.parametrize("m", [31, 32, 33, 34])
def test_survivor_counts_around_the_warp_sort(int_index, m):
    """m copies of one row next to the query and 300 rows far behind: exactly the m copies survive at k <= m, so
    the survivors are sorted by one warp (m <= 32) or by the block sort (m > 32); keys in several candidate orders"""
    metric, idx, db, xq = int_index
    rng = np.random.default_rng(m)
    for rep in range(6):
        cand = np.stack([RR.copies_and_far(xq[q], db, 20_000 + 40 * q + np.arange(40), m, 300, metric, rng)
                         for q in range(KQ)])
        for k in sorted({1, 10, m, len(cand[0])}):
            r = check_keys(idx, db, xq, cand, k, metric, f"{MNAME[metric]} m={m} k={k} order {rep}")
            if k <= m:
                assert np.all(r["surv"] == m), (m, k, r["surv"])


# ---- 4. through search ---------------------------------------------------------------------------------------------
SEARCH_TYPES = {
    "IVFPQ": lambda d: ("IVFPQ", {"nsubvector": {16: 8, 132: 12, 768: 48}[d]}),
    "IVFPQFastScan": lambda d: ("IVFPQFastScan", {"nsubvector": {16: 8, 132: 12, 768: 48}[d]}),
    "IVFRABITQ": lambda d: ("IVFRABITQ", {"nb_bits": 4}),
    "VEARCH": lambda d: ("VEARCH", {"nsubvector": {16: 8, 132: 12, 768: 48}[d], "reordering": True}),
}


def deepest_recall(idx, xq, k):
    """the largest recall_num the index accepts here, from its refusal of 2^20"""
    try:
        idx.search(xq[:1], k, params={"nprobe": 16, "recall_num": 1 << 20})
    except gi().GammaError as e:
        m = re.search(r"above (\d+)", str(e))
        assert m, str(e)
        return int(m.group(1))
    raise AssertionError("recall_num 2^20 was accepted")


@pytest.mark.parametrize("d", [16, 132, 768])
@pytest.mark.parametrize("typ", list(SEARCH_TYPES))
def test_search_at_the_deepest_recall_num(typ, d):
    n, nq, k = 20_000, 8, 10
    name, extra = SEARCH_TYPES[typ](d)
    db = np.rint(synth.sift_like(n, d, seed=d) / 8).astype(F32)
    xq = np.rint(synth.sift_like(nq, d, seed=d + 1) / 8).astype(F32)
    p = dict(extra, ncentroids=64, nprobe=16, metric_type="L2", training_threshold=n)
    idx = gi().RaBitQIndex(d, p) if name == "IVFRABITQ" else (gi().VearchIndex(d, p) if name == "VEARCH" else
                                                            gi().GammaIndex(name, d, p))
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    idx.set_rerank_stats(True)
    kk = deepest_recall(idx, xq, k)
    assert kk >= 400, kk
    _, ids = idx.search(xq, kk, params={"nprobe": 16})
    adc = np.where(ids >= 0, ids.astype(np.uint64), R.SENTINEL)
    want = R.rerank_keys(adc, xq, db, k, L2)
    idx.rerank_survivors()
    dis, ids = idx.search(xq, k, params={"nprobe": 16, "recall_num": kk})
    wd, wi = R.decode(want, L2)
    assert np.array_equal(dis.view(np.uint32), wd.view(np.uint32)) and np.array_equal(ids, wi), (typ, d, kk)
    surv = idx.rerank_survivors()
    assert len(surv) == nq, f"{typ} d={d}: the two-pass kernel did not serve every query"
    assert np.all(surv < kk), (typ, d, kk, surv)  # the screen still prunes
    idx.close()


# ---- 5. the second raw-store segment -------------------------------------------------------------------------------
SEG = 1 << 20
NSEG = SEG + 4099


@pytest.mark.parametrize("typ,cuts", [("IVFPQ", [SEG - 3, SEG + 2000]), ("IVFPQFastScan", [SEG - 3, SEG])],
                         ids=["straddle", "at-boundary"])
def test_second_segment(typ, cuts, tmp_path):
    d, metric, nq = 32, L2, 6
    rng = np.random.default_rng(17)
    db = rng.integers(0, 24, (NSEG, d)).astype(F32)
    xq = rng.integers(0, 24, (nq, d)).astype(F32)
    p = dict(nsubvector=8, ncentroids=32, nprobe=8, metric_type="L2", training_threshold=20_000)
    idx = gi().GammaIndex(typ, d, p)
    for a, b in zip([0] + cuts, cuts + [NSEG]):
        idx.add_vectors(db[a:b])
    idx.train()
    idx.add_pending()
    watch = np.r_[SEG - 2:SEG + 3, NSEG - 1]
    assert_shadow(idx, db[watch], vids=watch, what=f"{typ} shadow rows at the boundary")

    def cands():
        c = np.stack([rng.choice(NSEG, 3000, replace=False) for _ in range(nq)])
        c[:, :8] = np.r_[SEG - 4:SEG + 4]
        c[:, 8:12] = rng.integers(SEG, NSEG, 4)
        c[:, 12] = NSEG - 1
        return rng.permuted(c, axis=1)

    cand = cands()
    for k in (1, 10, 3000):
        check_keys(idx, db, xq, cand, k, metric, f"{typ} both segments k={k}")
    # rows moved next to queries 0-2, across the boundary: each must come back first
    for q, v in enumerate((SEG - 1, SEG, SEG + 1)):
        row = xq[q].copy()
        row[q] += 1
        idx.update_vector(v, row)
        db[v] = row
    assert_shadow(idx, db[watch], vids=watch, what=f"{typ} shadow rows after update_vector")
    r = check_keys(idx, db, xq, cand, 10, metric, f"{typ} after update_vector")
    assert list(r["ids"][:3, 0]) == [SEG - 1, SEG, SEG + 1]
    before = idx.debug_rerank(xq, cand, 10)
    idx.dump(str(tmp_path), "emb")
    idx.close()
    idx2 = gi().GammaIndex(typ, d, p)
    idx2.add_vectors(db)
    idx2.load(str(tmp_path), "emb")
    assert_shadow(idx2, db[watch], vids=watch, what=f"{typ} shadow rows after load")
    after = check_keys(idx2, db, xq, cand, 10, metric, f"{typ} after dump / load")
    assert same_results(before, after)
    idx2.close()
