"""Query-major list scans at batch shapes: every codec of the shared list scan (list_scan.cuh) and the BINARYIVF scan with
several probes per CTA, key-exact against the restatements.

The scans split a batch by  pg = clamp(nprobe * nq / (nsm * 32), 1, 32)  probes per CTA, so a small test batch only
ever runs pg = 1.  Here nq is derived from the device's SM count for pg in {1, 2, 3, 7, 32} (nprobe % 3 and % 7 != 0:
the last group is shorter), and every case asserts the kernel and the pg it reached.  A CTA then walks several lists:
long lists of several tiles, single-entry lists, empty lists and -1 probes, in an order shuffled per row, so the
groups' boundaries fall everywhere.  The batch repeats Q distinct queries, each row with its own probe order; the
reference (tests/topk_reference.py over the twins' scores) is computed per distinct query, and the same queries
searched alone (pg = 1) give byte-identical keys.

Rows and queries are integer vectors whose largest coordinate (4) is unique: the row's home list, centroid e_home.
Lists -e_j never win a row under either metric, so they are empty; homes H - 8 .. H - 5 have no rows, H - 4 .. H - 1
one row each, and home 1 about a third of them.

Beside the split: IVF-PQ phase A on both sides of nq >= 4 nsm (one CTA per query, or its leading probes split and
merged), and batches across the 16384-query blocks and past 65535 queries."""
import numpy as np
import pytest

import topk_reference as R
from oracle_binary import binary_ivf as ob
from oracle_pqfs import twin
from oracle_rabitq import rabitq as rq
from test_gpu_shape_limits import (binary_scan, ivfpq_scan, nibble_scan, rabitq_scan, scan_max_k,
                                   vearch_twin_scores)
from test_gpu_topk_keys import coarse_exact, entries, filter_cases, tombstone_some

pytestmark = pytest.mark.gpu
L2, IP = R.METRIC_L2, R.METRIC_IP
MNAME = {L2: "L2", IP: "InnerProduct"}
F32 = np.float32

# ---- the split, restated (index.cu scan_query_major_dev, BinaryIvfIndex::scan_dev) ---------------------------------
PG = [1, 2, 3, 7, 32]
MAX_PG = 32


def probes_per_cta(nprobe, nq, nsm):
    return min(MAX_PG, max(1, nprobe * nq // (nsm * 32)))


def nq_for(pg, nprobe, nsm):
    """the smallest batch whose split is pg probes per CTA"""
    return -(-pg * nsm * 32 // nprobe)


def ngroups(nprobe, pg):
    return -(-nprobe // pg)


# codec family -> (nprobe, largest batch the type accepts); the GPU_* types take at most 512 queries a request
NPROBE = {"list_scan": (64, None), "binary": (50, None), "gpu_ivfpq": (265, 512)}
PHASE_A_QUERIES_PER_SM = 4  # IVF-PQ phase A keeps a query's leading probes in one CTA from nq >= 4 nsm on
QUERY_BLOCK = 16384  # IvfIndex::kQueryBlock


def gi():
    from vearch_b200 import index as gidx
    return gidx


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- data: rows with a home list -----------------------------------------------------------------------------------
def home_rows(n, d, H, seed, singles=True):
    """integer rows in {-1, 0, 1} with a 4 at the home coordinate; home 1 holds ~35 %, homes H-8..H-5 none, H-4..H-1
    one row each (singles=True)"""
    rng = np.random.default_rng(seed)
    k = H - 8
    p = np.full(k, 0.65 / (k - 1))
    p[1] = 0.35
    home = rng.choice(k, n - 4, p=p)
    home = np.concatenate([home, np.arange(H - 4, H)]) if singles else rng.choice(k, n, p=p)
    x = rng.integers(-1, 2, (n, d))
    x[np.arange(n), home] = 4
    return x.astype(F32)


def home_queries(Q, d, H, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(-1, 2, (Q, d))
    x[np.arange(Q), rng.integers(0, H, Q)] = 4
    x[-1] = 0  # a zero query: every score of a row ties with its neighbours' under IP
    return x.astype(F32)


def basis_centroids(H, d, negated=1):
    """e_0 .. e_{H-1}, then -e_j (and -2 e_j): lists no row reaches under L2 or IP"""
    e = np.eye(H, d, dtype=F32)
    return np.concatenate([e] + [-(i + 1) * e for i in range(negated)]).astype(F32)


def dead_bitmap(n, seed, frac):
    return np.packbits(np.random.default_rng(seed).random(n) < frac, bitorder="little")


# ---- one index per codec, with every list entry's score for the Q distinct queries ---------------------------------
class Codec:
    def __init__(self, name, kernel, metric, idx, xq, scores, el, ids, nprobe, kmax, H, coarse=None, db=None,
                 params=None, binary=False, rr=None):
        self.name, self.kernel, self.metric, self.idx = name, kernel, metric, idx
        self.xq, self.scores, self.el, self.ids = xq, scores, el, ids
        self.nprobe, self.kmax, self.H, self.coarse, self.db = nprobe, kmax, H, coarse, db
        self.params, self.binary = params or {}, binary
        self.rr = rr  # VEARCH: the same lists with reordering on, which re-ranks every search
        self.Q, self.nlist, self.n = len(xq), idx.nlist, len(ids)
        self.lens = np.bincount(el, minlength=self.nlist)
        self.base = self.base_probes(seed=5)
        self._dec = {}

    def base_probes(self, seed):
        """each query's probes: the long list, a single-entry list, two empty ones, then the others; -1 in a third of
        the rows"""
        rng = np.random.default_rng(seed)
        H, out = self.H, []
        for q in range(self.Q):
            must = [1, H - 4 + q % 4, H - 8 + q % 4, H + q % H]
            rest = [l for l in rng.permutation(self.nlist) if l not in must]
            row = np.array(must + rest[:self.nprobe - 4], np.int64)
            rng.shuffle(row)
            if q % 3 == 0:
                row[rng.choice(self.nprobe, 5, replace=False)] = -1
            out.append(row)
        return np.stack(out)

    def batch_probes(self, rows, seed):
        """row r: query r % Q's probes in an order of its own"""
        rng = np.random.default_rng(seed)
        return np.stack([rng.permutation(self.base[q]) for q in rows])

    def coarse_dis(self, rows, probes):
        if self.coarse is None:
            return np.zeros(probes.shape, F32)
        cd = np.take_along_axis(self.coarse[rows], np.maximum(probes, 0), 1)
        return np.where(probes >= 0, cd, 0).astype(F32)

    def search(self, rows, k, probes, params=None, idx=None, **kw):
        if self.binary:
            return self.idx.search_preassigned(self.xq[rows], k, probes, **kw)
        p = dict(self.params, **(params or {}))
        return (idx or self.idx).search_preassigned(self.xq[rows], k, probes, self.coarse_dis(rows, probes), params=p or None,
                                           **kw)

    def ref(self, k, probes=None, **kw):
        return R.search_entries(self.scores, self.el, self.ids, self.base if probes is None else probes, k,
                                self.metric, **kw)

    def dec(self, key, keys):
        if key not in self._dec:
            self._dec[key] = R.decode(keys(), self.metric)
        return self._dec[key]

    def close(self):
        self.idx.close()
        if self.rr is not None:
            self.rr.close()


def check(got, want, rows, what):
    """got: the batch's (scores, ids); want: the decoded reference of the Q distinct queries"""
    dg, ig = got
    dr, ir = want[0][rows], want[1][rows]
    bad = np.nonzero(~(np.all(ig == ir, 1) & np.all(dg.view(np.uint32) == dr.view(np.uint32), 1)))[0]
    if len(bad):
        r = bad[0]
        j = np.nonzero((ig[r] != ir[r]) | (dg[r].view(np.uint32) != dr[r].view(np.uint32)))[0][0]
        raise AssertionError(f"{what}: {len(bad)}/{len(rows)} rows differ; row {r} (query {rows[r]}) slot {j}: got "
                             f"({dg[r, j]!r}, {ig[r, j]}), want ({dr[r, j]!r}, {ir[r, j]})")


def assert_split(c, pg, what, idx=None):
    idx = idx or c.idx
    info = idx.last_scan_info
    assert idx.last_scan_kernel == c.kernel, (what, idx.last_scan_kernel)
    assert info.get("probes_per_cta") == pg, (what, info)


def pq_codec(name, typ, d, M, nbits, metric, H=48, nprobe=64, Q=64, negated=1, seed=0):
    db = home_rows(20000, d, H, seed=seed + 1)
    xq = home_queries(Q, d, H, seed=seed + 2)
    cent = basis_centroids(H, d, negated)
    rng = np.random.default_rng(seed + 3)
    ksub = 16 if typ == "IVFPQFastScan" else 1 << nbits
    pq = rng.integers(-2, 3, (M, ksub, d // M)).astype(F32)
    params = {"ncentroids": len(cent), "nprobe": nprobe, "nsubvector": M, "metric_type": MNAME[metric]}
    if typ == "IVFPQ":
        params["nbits_per_idx"] = nbits
    idx = gi().GammaIndex(typ, d, params)
    idx.set_centroids(cent)
    idx.set_pq_centroids(pq)
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids, el = entries(idx, len(cent))
    ids = tombstone_some(idx, off, ids, range(0, H, 5))
    coarse = None
    if typ == "IVFPQFastScan":
        lut8, ab = twin.lut(pq, xq, metric)
        cu = twin.unpack(codes, M)
        scores = np.stack([twin.scores(lut8[q], ab[q], cu) for q in range(Q)])
        kernel, kmax = "ivfpqfs_scan_kernel", 4096
    else:
        R.pq_guard(xq, cent, pq, metric)
        rec = R.pq_reconstruct(cent, pq, el, R.unpack_codes(codes, M, nbits))
        scores = R.exact_scores(xq, rec, metric)
        coarse = R.exact_scores(xq, cent, metric).astype(F32)  # dis0 of each probe (IVF-PQ by residual)
        kernel = "ivfpq_scan_kernel" if nbits == 8 else "ivfpq_packed_scan_kernel"
        kmax = 2048 if typ == "GPU_IVFPQ" else scan_max_k(ivfpq_scan(M, nbits))
    return Codec(name, kernel, metric, idx, xq, scores, el, ids, nprobe, kmax, H, coarse=coarse,
                 db=None if typ == "GPU_IVFPQ" else db)


def rabitq_codec(name, metric, B, qb, d=64, H=48, nprobe=64, Q=64):
    db = home_rows(20000, d, H, seed=11)
    xq = home_queries(Q, d, H, seed=12)
    cent = basis_centroids(H, d)
    idx = gi().RaBitQIndex(d, {"ncentroids": len(cent), "nprobe": nprobe, "nb_bits": B, "metric_type": MNAME[metric]})
    idx.set_centroids(cent)
    idx.add(db)
    off, codes, ids, el = entries(idx, len(cent))
    ids = tombstone_some(idx, off, ids, range(0, H, 5))
    scores = np.zeros((Q, len(ids)), F32)
    for l in np.unique(el):
        sel = el == l
        for j in range(Q):
            scores[j, sel] = rq.estimate(codes[sel], xq[j], cent[l], d, B, metric, qb)
    return Codec(name, "rabitq_scan_kernel", metric, idx, xq, scores, el, ids, nprobe,
                 scan_max_k(rabitq_scan(d, B, qb)), H, db=db, params={"qb": qb})


def vearch_codec(name, metric, d=64, nsub=16, H=48, nprobe=64, Q=64):
    db = home_rows(20000, d, H, seed=21)
    xq = home_queries(Q, d, H, seed=22)
    cent = basis_centroids(H, d)  # unit rows: VEARCH's spherical partitions under IP
    cb = (np.random.default_rng(23).standard_normal(16 * d) * 1.5).astype(F32)
    p = {"ncentroids": len(cent), "nsubvector": nsub, "metric_type": MNAME[metric]}
    if metric == IP:
        p["ns_threshold"] = 0.2
    idx, rr = gi().VearchIndex(d, p), gi().VearchIndex(d, dict(p, reordering=True))
    for i in (idx, rr):
        i.set_codebook(cb)
        i.set_centroids(cent)
        i.add(db)
    off, codes, ids, el = entries(idx, len(cent))
    o2, c2, i2, _ = entries(rr, len(cent))
    assert np.array_equal(off, o2) and np.array_equal(codes, c2) and np.array_equal(ids, i2)
    ids = tombstone_some(idx, off, ids, range(0, H, 5))
    tombstone_some(rr, off, i2, range(0, H, 5))
    scores = vearch_twin_scores(codes, el, cent, cb, xq, d, nsub, metric)
    return Codec(name, "vearch_scan_kernel", metric, idx, xq, scores, el, ids, nprobe, scan_max_k(nibble_scan(nsub)),
                 H, db=db, rr=rr)


def binary_codec(name, cs=16, H=32, nprobe=50, Q=64, n=20000):
    """packed rows: pattern P_home with <= 6 bits flipped; lists H.. hold the complements, which no row reaches"""
    rng = np.random.default_rng(31)
    pat = rng.integers(0, 256, (H, cs), dtype=np.uint8)
    cent = np.concatenate([pat, ~pat])

    def near(homes):
        x = pat[homes].copy()
        for r in range(len(x)):
            b = rng.choice(cs * 8, rng.integers(0, 7), replace=False)
            np.bitwise_xor.at(x[r], b >> 3, (1 << (b & 7)).astype(np.uint8))
        return x

    k = H - 8
    p = np.full(k, 0.65 / (k - 1))
    p[1] = 0.35
    db = near(np.concatenate([rng.choice(k, n - 4, p=p), np.arange(H - 4, H)]))
    xq = near(rng.integers(0, H, Q))
    idx = gi().BinaryIVFIndex(cs * 8, {"ncentroids": len(cent)})
    idx.set_centroids(cent)
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids, el = entries(idx, len(cent))
    ids = tombstone_some(idx, off, ids, range(0, H, 5))
    return Codec(name, "binary_ivf_scan_kernel", L2, idx, xq, ob.hamming(xq, codes), el, ids, nprobe,
                 scan_max_k(binary_scan(cs)), H, binary=True)


CASES = {
    "IVFPQ8_M32_L2": lambda: pq_codec("IVFPQ8_M32_L2", "IVFPQ", 64, 32, 8, L2),  # 32-byte codes: a vector-load layout
    "IVFPQ8_M32_IP": lambda: pq_codec("IVFPQ8_M32_IP", "IVFPQ", 64, 32, 8, IP),
    "IVFPQ8_M12_L2": lambda: pq_codec("IVFPQ8_M12_L2", "IVFPQ", 60, 12, 8, L2),  # the generic (MW = 0) layout
    "IVFPQ8_M12_IP": lambda: pq_codec("IVFPQ8_M12_IP", "IVFPQ", 60, 12, 8, IP),
    **{f"IVFPQ_nbits{b}_L2": (lambda b=b: pq_codec(f"IVFPQ_nbits{b}_L2", "IVFPQ", 64, 16, b, L2)) for b in range(1, 8)},
    "IVFPQ_nbits3_IP": lambda: pq_codec("IVFPQ_nbits3_IP", "IVFPQ", 64, 16, 3, IP),
    "IVFPQFastScan_L2": lambda: pq_codec("IVFPQFastScan_L2", "IVFPQFastScan", 64, 16, 4, L2),
    "IVFPQFastScan_IP": lambda: pq_codec("IVFPQFastScan_IP", "IVFPQFastScan", 64, 16, 4, IP),
    "IVFRABITQ_qb0_L2": lambda: rabitq_codec("IVFRABITQ_qb0_L2", L2, 3, 0),
    "IVFRABITQ_qb0_IP": lambda: rabitq_codec("IVFRABITQ_qb0_IP", IP, 3, 0),
    "IVFRABITQ_qb4_L2": lambda: rabitq_codec("IVFRABITQ_qb4_L2", L2, 3, 4),
    "IVFRABITQ_qb4_IP": lambda: rabitq_codec("IVFRABITQ_qb4_IP", IP, 3, 4),
    "VEARCH_IP": lambda: vearch_codec("VEARCH_IP", IP),
    "VEARCH_L2": lambda: vearch_codec("VEARCH_L2", L2),
    "BINARYIVF": lambda: binary_codec("BINARYIVF"),
    # M = 64 declines the tensor-core filter; 3 x 128 lists so that nq <= 512 reaches pg = 32
    "GPU_IVFPQ_M64_L2": lambda: pq_codec("GPU_IVFPQ_M64_L2", "GPU_IVFPQ", 128, 64, 8, L2, H=128, nprobe=265, Q=24,
                                         negated=2),
    "GPU_IVFPQ_M64_IP": lambda: pq_codec("GPU_IVFPQ_M64_IP", "GPU_IVFPQ", 128, 64, 8, IP, H=128, nprobe=265, Q=24,
                                         negated=2),
}


def family(case):
    return "binary" if case.startswith("BINARY") else ("gpu_ivfpq" if case.startswith("GPU_IVFPQ") else "list_scan")


_live = {}


def state(case):
    """one index alive at a time: the cases run one codec's pg ladder after another"""
    if case not in _live:
        for c in _live.values():
            c.close()
        _live.clear()
        _live[case] = CASES[case]()
    return _live[case]


@pytest.fixture(scope="module", autouse=True)
def _close_indexes():
    yield
    for c in _live.values():
        c.close()
    _live.clear()


@pytest.mark.parametrize("pg", PG)
@pytest.mark.parametrize("case", list(CASES))
def test_probe_groups_key_exact(case, pg):
    c = state(case)
    nprobe, cap = NPROBE[family(case)]
    assert c.nprobe == nprobe
    nq = nq_for(pg, nprobe, sm_count())
    assert cap is None or nq <= cap, (nq, cap)
    assert probes_per_cta(nprobe, nq, sm_count()) == pg
    # preconditions: the probe rows reach a long list (>= 3 tiles of every codec), single-entry lists and empty ones
    assert c.lens[1] >= 3 * 1024 and (c.lens[c.H - 4:c.H] == 1).all() and (c.lens[c.H - 8:c.H - 4] == 0).all()
    assert (c.lens[c.H:] == 0).all() and (c.base < 0).any()
    rows = np.arange(nq) % c.Q
    probes = c.batch_probes(rows, seed=pg)
    what = f"{case} pg={pg} nq={nq}"
    for k in (1, 17, c.kmax):
        got = c.search(rows, k, probes)
        assert_split(c, pg, what)
        check(got, c.dec(("k", k), lambda: c.ref(k)), rows, f"{what} k'={k}")
        small = c.search(np.arange(c.Q), k, c.base)  # the same queries alone: one probe per CTA
        assert_split(c, 1, f"{what} small batch")
        assert np.array_equal(got[0].view(np.uint32), small[0][rows].view(np.uint32)) and np.array_equal(
            got[1], small[1][rows]), f"{what} k'={k}: batch and single-query keys differ"
    sc = c.dec(("k", 17), lambda: c.ref(17))[0][c.Q // 2]
    cases = filter_cases(c.n, 17, sc, c.metric, seed=1) + [
        ("del_and_filter", {"del_bitmap": dead_bitmap(c.n, 1, 0.3), "filter_bitmap": dead_bitmap(c.n, 2, 0.6)})]
    for name, kw in cases:
        got = c.search(rows, 17, probes, **kw)
        assert_split(c, pg, what)
        check(got, c.dec((name, 17), lambda: c.ref(17, **kw)), rows, f"{what} {name}")
    dele = {"del_bitmap": dead_bitmap(c.n, 3, 0.25)}
    check(c.search(rows, c.kmax, probes, **dele), c.dec(("del", c.kmax), lambda: c.ref(c.kmax, **dele)), rows,
          f"{what} deleted k'={c.kmax}")
    if c.db is not None:  # the exact re-rank of the kmax best codes
        got = c.search(rows, 17, probes, params={"recall_num": c.kmax}, idx=c.rr)
        assert_split(c, pg, what, idx=c.rr)
        want = c.dec(("rerank", c.kmax), lambda: R.rerank_keys(c.ref(c.kmax), c.xq, c.db, 17, c.metric))
        check(got, want, rows, f"{what} recall_num={c.kmax}")
    if pg == MAX_PG:  # through search: the index's own coarse quantiser picks the lists
        xb = c.xq[rows]
        _, pr = c.idx.coarse_search(xb, nprobe)
        assert all(np.array_equal(np.sort(pr[r]), np.sort(pr[rows[r]])) for r in range(nq))  # equal queries, equal lists
        got = c.idx.search(xb, 17, params=dict(c.params, nprobe=nprobe))
        assert_split(c, pg, f"{what} search")
        check(got, R.decode(c.ref(17, probes=pr[:c.Q]), c.metric), rows, f"{what} search")


# ---- IVF-PQ phase A: both sides of nq >= 4 nsm -------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("side", [-1, 0])
def test_ivfpq_phase_a_sides(metric, side):
    """nq = 4 nsm - 1: phase A splits each query's leading probes over CTAs and merges them; nq = 4 nsm: one CTA per
    query.  Both key for key equal to the query-major LUT kernel, under a deletion and a filter bitmap"""
    from test_gpu_pq_overlap import assert_same, list_major, query_major, sift_index
    nq = PHASE_A_QUERIES_PER_SM * sm_count() + side
    s, n = sift_index(metric, nq=nq)
    try:
        rng = np.random.default_rng(7)
        kw = {"del_bitmap": np.packbits(rng.random(n) < 0.3, bitorder="little"),
              "filter_bitmap": np.packbits(rng.random(n) < 0.7, bitorder="little")}
        for k in (10, 100):
            got = list_major(s, k, **kw)
            info = s.idx.last_scan_info
            assert info["phase_a_probes_per_cta"] == (info["phase_a_max_probes"] if side == 0 else 1), info
            assert_same(got, query_major(s, k, nq, **kw), f"nq={nq} k={k}")
    finally:
        s.idx.close()


# ---- query blocks ------------------------------------------------------------------------------------------------------
def block_data(d, H, npool, seed):
    """rows with a home list; a pool of queries with a unique nearest and second-nearest list (no coarse ties at
    nprobe 2)"""
    db = home_rows(20000, d, H, seed=seed, singles=False)
    rng = np.random.default_rng(seed + 1)
    pool = rng.integers(-1, 2, (npool, d))
    h = rng.integers(0, H, npool)
    s2 = (h + rng.integers(1, H, npool)) % H
    pool[np.arange(npool), h] = 4
    pool[np.arange(npool), s2] = 2
    return db, pool.astype(F32)


def block_index(typ, d, H, metric, db, nprobe):
    cent = basis_centroids(H, d)
    p = {"ncentroids": len(cent), "nprobe": nprobe, "metric_type": MNAME[metric]}
    if typ == "IVFPQFastScan":
        p["nsubvector"] = d // 2
    if typ == "IVFPQ_OPQ":  # a permutation as the rotation: rotated integer rows stay integers
        p.update(nsubvector=d // 2, opq={"nsubvector": d // 2})
    idx = gi().GammaIndex("IVFPQ" if typ == "IVFPQ_OPQ" else typ, d, p)
    perm = np.random.default_rng(d).permutation(d)
    rot = np.arange(d)
    if typ == "IVFPQ_OPQ":
        A = np.zeros((d, d), F32)
        A[np.arange(d), perm] = 1  # y[i] = x[perm[i]]
        idx.set_opq(A)
        rot = perm
    idx.set_centroids(cent[:, rot])
    pq = None
    if typ != "IVFFLAT":
        ksub = 16 if typ == "IVFPQFastScan" else 256
        pq = np.random.default_rng(d + 1).integers(-2, 3, (d // 2, ksub, 2)).astype(F32)
        idx.set_pq_centroids(pq)
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids, el = entries(idx, len(cent))
    ids = tombstone_some(idx, off, ids, range(0, H, 3))
    return idx, cent, rot, pq, codes, ids, el


def block_scores(typ, pool, db, rot, pq, codes, ids, el, cent, metric):
    if typ == "IVFFLAT":
        return R.exact_scores(pool, db[ids & 0xFFFFFFFF], metric)
    M = pq.shape[0]
    if typ == "IVFPQFastScan":
        lut8, ab = twin.lut(pq, pool, metric)
        cu = twin.unpack(codes, M)
        return np.stack([twin.scores(lut8[q], ab[q], cu) for q in range(len(pool))])
    rec = R.pq_reconstruct(cent[:, rot], pq, el, R.unpack_codes(codes, M, 8))
    return R.exact_scores(pool[:, rot], rec, metric)


@pytest.mark.parametrize("typ", ["IVFFLAT", "IVFPQ_OPQ", "IVFPQFastScan"])
def test_query_blocks(typ):
    """16384 + 129 queries (two blocks of search_keys_dev), then 65545 (past one launch's 65535 queries) through search and
    search_preassigned; d = 30, so a query row (120 bytes) is shorter than its 128-byte stride"""
    d, H, nprobe, k, metric = 30, 30, 2, 17, L2
    db, pool = block_data(d, H, 257, seed=41)
    idx, cent, rot, pq, codes, ids, el = block_index(typ, d, H, metric, db, nprobe)
    try:
        n = len(db)
        kw = {"del_bitmap": dead_bitmap(n, 42, 0.2), "filter_bitmap": dead_bitmap(n, 43, 0.8)}
        scores = block_scores(typ, pool, db, rot, pq, codes, ids, el, cent, metric)
        _, probes = coarse_exact(pool, cent, metric, nprobe)
        params = {"recall_num": 64} if typ == "IVFPQ_OPQ" else None
        ref = R.search_entries(scores, el, ids, probes, 64 if params else k, metric, **kw)
        if params:
            ref = R.rerank_keys(ref, pool, db, k, metric, **kw)
        want = R.decode(ref, metric)
        rng = np.random.default_rng(44)
        for nq in (QUERY_BLOCK + 129, 65545):
            qi = rng.integers(0, len(pool), nq)
            m = min(len(pool), nq - QUERY_BLOCK)
            qi[QUERY_BLOCK:QUERY_BLOCK + m] = np.arange(m)  # the second block starts with the pool in order
            check(idx.search(pool[qi], k, params=params, **kw), want, qi, f"{typ} search nq={nq}")
            cd = np.take_along_axis(R.exact_scores(pool, cent, metric), probes, 1).astype(F32)[qi]
            got = idx.search_preassigned(pool[qi], k, probes[qi], cd, params=params, **kw)
            check(got, want, qi, f"{typ} search_preassigned nq={nq}")
    finally:
        idx.close()
