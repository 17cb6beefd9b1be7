"""The two-pass exact re-rank (rerank_prefilter_kernel) on the H100: candidates screened on the int8 shadow of the raw
rows, fp32 rows read only for those that can still reach the top k.  Its keys must be the one-pass re-rank's, bit for
bit: against the CPU restatement (topk_reference.rerank_keys, integer-valued rows so that every fp32 order is exact)
and, on float rows, against the same index with its raw vectors in host memory, which re-ranks through the one-pass
kernel.  Each search must have been served by the two-pass kernel (its per-query survivor counts are recorded)."""
import numpy as np
import pytest

import topk_reference as R
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
F32 = np.float32
L2, IP = R.METRIC_L2, R.METRIC_IP
MNAME = {L2: "L2", IP: "InnerProduct"}
N, D, NQ, NLIST, NPROBE = 30_000, 128, 24, 64, 16

TYPES = {
    "IVFPQ": ("IVFPQ", {"nsubvector": 16}),
    "IVFPQ_nbits4": ("IVFPQ", {"nsubvector": 16, "nbits_per_idx": 4}),
    "IVFPQFastScan": ("IVFPQFastScan", {"nsubvector": 16}),
    "IVFRABITQ": ("IVFRABITQ", {"nb_bits": 4}),
}


def gi():
    from vearch_b200 import index as gidx
    return gidx


def int_data(metric, seed):
    """integer-valued sift-like rows (exact fp32 scores) with near-duplicates: 48 copies of a row next to each of the
    first queries, so the k-th score is tied many times over; plus zero rows and rows with one dominant component"""
    rng = np.random.default_rng(seed)
    db = np.rint(synth.sift_like(N, D, seed=seed) / 8)
    xq = np.rint(synth.sift_like(NQ, D, seed=seed + 1) / 8)
    if metric == IP:
        db -= 16
        xq -= 16
    for q in range(6):
        near = xq[q].copy()
        near[q] += 1
        db[1000 + 48 * q:1000 + 48 * (q + 1)] = near
    db[5:9] = 0
    db[9:13] = 0
    db[9:13, rng.integers(0, D, 4)] = 200
    return db.astype(F32), xq.astype(F32)


def make(typ, metric, store_type=None, extra=None):
    name, p = TYPES.get(typ, (typ, {}))
    params = dict(p, ncentroids=NLIST, nprobe=NPROBE, metric_type=MNAME[metric], training_threshold=N)
    params.update(extra or {})
    if name == "IVFRABITQ":
        return gi().RaBitQIndex(D, params, store_type=store_type)
    if name == "VEARCH":
        return gi().VearchIndex(D, params, store_type=store_type)
    return gi().GammaIndex(name, D, params, store_type=store_type)


def build(typ, metric, db, store_type=None, extra=None):
    idx = make(typ, metric, store_type, extra)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    idx.set_rerank_stats(True)
    return idx


def as_keys(dis, ids, metric):
    """the engine's result rows as keys, in key order (IP lists equal scores with the larger id first)"""
    return np.sort(R.keys(dis, np.where(ids >= 0, ids, 0), ids >= 0, metric), axis=1)


def adc_candidates(idx, xq, kk, **kw):
    """the ADC top kk of each query, what the re-rank is given: the same search without recall_num"""
    _, ids = idx.search(xq, kk, params={"nprobe": NPROBE}, **kw)
    return np.where(ids >= 0, ids.astype(np.uint64), R.SENTINEL)


def check(idx, xq, db, k, kk, metric, what, **kw):
    want = R.rerank_keys(adc_candidates(idx, xq, kk, **kw), xq, db, k, metric, **kw)
    idx.rerank_survivors()
    dis, ids = idx.search(xq, k, params={"nprobe": NPROBE, "recall_num": kk}, **kw)
    got = as_keys(dis, ids, metric)
    bad = np.nonzero(~np.all(got == want, 1))[0]
    assert not len(bad), f"{what}: {len(bad)} queries differ from the CPU re-rank (first: query {bad[0]})"
    wd, wi = R.decode(want, metric)
    assert np.array_equal(dis.view(np.uint32), wd.view(np.uint32)) and np.array_equal(ids, wi), what
    surv = idx.rerank_survivors()
    assert len(surv) == len(xq), f"{what}: the two-pass kernel did not serve the search"
    assert np.all(surv <= kk), what
    return surv


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("typ", list(TYPES))
def test_keys_equal_the_cpu_rerank(typ, metric):
    db, xq = int_data(metric, seed=3)
    idx = build(typ, metric, db)
    deep = typ in ("IVFPQ", "IVFPQFastScan")
    # (the 48 copies next to each of the first queries tie the k-th score at k = 1 and 10)
    for k, kk in [(1, 400), (10, 400), (400, 400)] + ([(10, 4096), (4096, 4096)] if deep else []):
        check(idx, xq, db, k, kk, metric, f"{typ} k={k} recall_num={kk}")
    # bitmaps and a score window
    n = len(db)
    rng = np.random.default_rng(5)
    dead = np.packbits(rng.random(n) < 0.3, bitorder="little")
    keep = np.packbits(rng.random(n) < 0.5, bitorder="little")
    check(idx, xq, db, 10, 400, metric, f"{typ} deletion bitmap", del_bitmap=dead)
    check(idx, xq, db, 10, 400, metric, f"{typ} filter bitmap", filter_bitmap=keep)
    ref = R.decode(R.rerank_keys(adc_candidates(idx, xq, 400), xq, db, 400, metric), metric)[0][0]
    lo_s, hi_s = sorted((float(ref[3]), float(ref[60])))
    check(idx, xq, db, 10, 400, metric, f"{typ} score window", min_score=lo_s, max_score=hi_s)
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
def test_update_append_and_dump_load(metric, tmp_path):
    db, xq = int_data(metric, seed=11)
    idx = build("IVFPQ", metric, db)
    check(idx, xq, db, 10, 400, metric, "before")
    # an update moves a far row next to query 0: it must come back first (a stale shadow row would screen it out)
    s = R.exact_scores(xq[:1], db, metric)[0]
    far = int(np.argmax(s) if metric == L2 else np.argmin(s))
    row = xq[0] * (4 if metric == IP else 1)  # same coarse list as the query under either metric
    idx.update_vector(far, row)
    db[far] = row
    check(idx, xq, db, 10, 400, metric, "after update_vector")
    _, ids = idx.search(xq[:1], 1, params={"nprobe": NPROBE, "recall_num": 400})
    assert ids[0, 0] == far
    # appends after a search: new rows get their shadow rows with them
    more = np.rint(synth.sift_like(5000, D, seed=12) / 8).astype(F32) - (16 if metric == IP else 0)
    more[:8] = xq[:8]
    idx.add_vectors(more)
    idx.add_pending()
    db = np.concatenate([db, more])
    check(idx, xq, db, 10, 400, metric, "after append")
    before = idx.search(xq, 10, params={"nprobe": NPROBE, "recall_num": 400})
    idx.dump(str(tmp_path), "emb")
    idx.close()
    idx2 = make("IVFPQ", metric)
    idx2.add_vectors(db)
    idx2.load(str(tmp_path), "emb")
    idx2.set_rerank_stats(True)
    after = idx2.search(xq, 10, params={"nprobe": NPROBE, "recall_num": 400})
    assert np.array_equal(before[0].view(np.uint32), after[0].view(np.uint32)) and np.array_equal(before[1], after[1])
    assert len(idx2.rerank_survivors()) == len(xq)
    idx2.close()


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("typ", ["IVFPQ", "IVFPQFastScan", "IVFRABITQ", "VEARCH"])
def test_float_rows_bit_equal_to_the_one_pass_kernel(typ, metric):
    """float rows (sums depend on the evaluation order): the HBM index (two-pass kernel) against the same index with
    its raw vectors in host memory (one-pass kernel), score bits and ids"""
    db = synth.sift_like(N, D, seed=21, rounded=False).astype(F32)
    xq = synth.sift_like(NQ, D, seed=22, rounded=False).astype(F32)
    if metric == IP:
        db, xq = db - 60, xq - 60
    db[100:164] = db[99]  # exact ties
    xq[0] = db[99] + 0.25
    db[7] = 0
    extra = {"reordering": True, "nsubvector": 16} if typ == "VEARCH" else None
    hbm = build(typ, metric, db, extra=extra)
    host = build(typ, metric, db, store_type="RocksDB", extra=extra)
    for k, kk in ((1, 200), (10, 400), (100, 100)):
        p = {"nprobe": NPROBE, "recall_num": kk}
        a, b = hbm.search(xq, k, params=p), host.search(xq, k, params=p)
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]), (typ, k, kk)
        assert len(hbm.rerank_survivors()) == len(xq) and len(host.rerank_survivors()) == 0
    assert hbm.mem_bytes(1) >= N * (4 * D + D + 16) and host.mem_bytes(1) == 0  # the shadow is counted with the store
    hbm.close()
    host.close()


def test_no_shadow_without_reordering():
    db, xq = int_data(L2, seed=31)
    a = build("VEARCH", L2, db, extra={"nsubvector": 16})
    b = build("VEARCH", L2, db, extra={"nsubvector": 16, "reordering": True})
    a.search(xq, 10, params={"nprobe": NPROBE})
    assert len(a.rerank_survivors()) == 0
    assert b.mem_bytes(1) - a.mem_bytes(1) >= N * (D + 16)  # the shadow rows of the reordering index
    a.close()
    b.close()
