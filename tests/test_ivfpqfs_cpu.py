"""IVFPQFastScan on the CPU: the C restatement (oracle_pqfs/ivfpqfs_oracle.c) and its numpy twin agree byte for byte;
both are pinned by hand-computed answers, fp64 argmin checks and an independent per-entry loop of the search; the
ksub = 16 training is checked against a plain numpy Lloyd run."""
import numpy as np
import pytest

from oracle import oracle as orc
from oracle_pqfs import ivfpqfs as cfs
from oracle_pqfs import twin as fso
from vearch_b200 import synth

L2, IP = orc.METRIC_L2, orc.METRIC_IP
F32 = np.float32


def test_quantisation_formula_and_nibble_order_known_answer():
    # d = 4, M = 2: sub-quantiser 0 has centroids (i, 0), sub-quantiser 1 has (0, 2i)
    pq = np.zeros((2, 16, 2), F32)
    pq[0, :, 0] = np.arange(16)
    pq[1, :, 1] = 2 * np.arange(16)
    lut8, ab = fso.lut(pq, np.zeros((1, 4), F32), L2)
    # tables i^2 and 4 i^2: mins 0, widest span 900, a = 255 / 900
    a = F32(255) / F32(900)
    assert ab[0, 0] == a and ab[0, 1] == 0
    assert lut8[0, 0, :4].tolist() == [0, 0, 1, 3]    # floor(i^2 a + 0.5): 0, 0.78, 1.63, 3.05
    assert lut8[0, 1, :4].tolist() == [0, 1, 5, 10]   # floor(4 i^2 a + 0.5): 0, 1.63, 5.03, 10.7
    assert lut8[0, 0, 15] == 64 and lut8[0, 1, 15] == 255
    # x = (3, 0, 0, 10): codes 3 and 5; byte = 3 | 5 << 4
    codes = fso.encode(pq, np.array([[3, 0, 0, 10]], F32))
    assert codes.tolist() == [[3, 5]]
    assert fso.pack(codes).tolist() == [[0x53]]
    # its score: accu = lut8[0][3] + lut8[1][5] = 3 + 28, de-quantised as accu * (1 / a) + b
    assert lut8[0, 1, 5] == 28
    s = fso.scores(lut8[0], ab[0], codes)
    assert s[0] == F32(31) * (F32(1) / a) + F32(0)


def test_degenerate_table_gives_a_one_and_zero_table():
    pq = np.zeros((3, 16, 2), F32)  # every centroid equal: every span 0
    xq = synth.sift_like(4, 6, seed=3)
    tab = fso.float_lut(pq, xq, L2)
    lut8, ab = fso.quantize_lut(tab)
    assert (lut8 == 0).all() and (ab[:, 0] == 1).all()
    b = np.zeros(4, F32)
    for m in range(3):
        b = b + tab[:, m, 0]
    assert np.array_equal(ab[:, 1], b)


@pytest.mark.parametrize("M", [15, 16, 3])
def test_pack_unpack_roundtrip_and_odd_tail(M):
    rng = np.random.default_rng(M)
    codes = rng.integers(0, 16, size=(50, M)).astype(np.uint8)
    packed = fso.pack(codes)
    assert packed.shape == (50, (M + 1) // 2)
    assert np.array_equal(fso.unpack(packed, M), codes)
    assert np.array_equal(packed[:, 0] & 15, codes[:, 0]) and np.array_equal(packed[:, 0] >> 4, codes[:, 1])
    if M % 2:
        assert (packed[:, -1] >> 4 == 0).all()


@pytest.mark.parametrize("d,M", [(32, 16), (30, 15)])
def test_codes_are_per_slice_argmin(d, M):
    x = synth.sift_like(3000, d, seed=5, rounded=False)
    pq, _ = cfs.pq_train(x[:2000], M, niter=5)
    codes = fso.encode(pq, x)
    dsub = d // M
    for m in range(M):
        xs = x[:, m * dsub:(m + 1) * dsub].astype(np.float64)
        dis = ((xs[:, None, :] - pq[m][None].astype(np.float64)) ** 2).sum(axis=2)
        chosen = dis[np.arange(len(x)), codes[:, m]]
        # fp32 evaluation may pick a different centroid only when the two are tied to within rounding
        assert (chosen <= dis.min(axis=1) * (1 + 1e-5) + 1e-6).all()


def _lloyd_inertia(x, k, niter, seed):
    rng = np.random.default_rng(seed)
    c = x[rng.choice(len(x), k, replace=False)].astype(np.float64)
    for _ in range(niter):
        dis = ((x[:, None, :] - c[None]) ** 2).sum(axis=2)
        a = dis.argmin(axis=1)
        for j in range(k):
            if (a == j).any():
                c[j] = x[a == j].mean(axis=0)
    return ((x[:, None, :] - c[None]) ** 2).sum(axis=2).min(axis=1).sum()


def test_ksub16_training_lowers_error_and_matches_numpy_lloyd():
    d, M = 16, 8
    x = np.random.default_rng(7).normal(0, 1, size=(4096, d)).astype(F32) * np.linspace(1, 4, d, dtype=F32)
    pq, objs = cfs.pq_train(x, M)
    dsub = d // M
    for m in range(M):
        xs = x[:, m * dsub:(m + 1) * dsub].astype(np.float64)
        assert objs[m][-1] < objs[m][0]  # assignment error at the last iteration below the initial centroids'
        inertia = ((xs[:, None, :] - pq[m][None].astype(np.float64)) ** 2).sum(axis=2).min(axis=1).sum()
        ref = _lloyd_inertia(xs, 16, 25, m)
        # two local optima of the same objective from different starts: within 5 % of each other
        assert abs(inertia - ref) <= 0.05 * ref, (m, inertia, ref)


def _loop_search(list_off, list_codes, list_ids, lut8, ab, keys, k, metric, M, deleted):
    """the search as a plain per-entry loop: an independent restatement of search_preassigned"""
    nq = keys.shape[0]
    out = []
    for q in range(nq):
        cand = []
        for l in keys[q]:
            if l < 0:
                continue
            for p in range(list_off[l], list_off[l + 1]):
                vid = int(list_ids[p])
                if vid < 0 or deleted[vid]:
                    continue
                accu = 0
                for m in range(M):
                    byte = int(list_codes[p, m // 2])
                    accu += int(lut8[q, m, (byte >> (4 * (m % 2))) & 15])
                s = F32(accu) * (F32(1) / ab[q, 0]) + ab[q, 1]
                cand.append((float(s) if metric == L2 else -float(s), vid, s))
        cand.sort()
        out.append([(c[2], c[1]) for c in cand[:k]])
    return out


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M", [(16, 8), (30, 15)])
def test_search_matches_a_per_entry_loop(metric, d, M):
    n, nq, nlist, nprobe, k = 1500, 6, 8, 3, 10
    db = synth.sift_like(n, d, seed=11)
    xq = synth.sift_like(nq, d, seed=12)
    cent, _, _ = orc.kmeans(db, nlist, niter=4)
    assign = orc.assign(cent, db, L2)
    off, order = orc.build_lists(assign, nlist)
    pq, _ = cfs.pq_train(db, M, niter=4)
    codes = fso.pack(fso.encode(pq, db))[order]
    ids = order.astype(np.int64)
    ids[5] |= np.int64(-(2 ** 63))  # a tombstone
    deleted = np.random.default_rng(1).random(n) < 0.1
    _, keys = orc.coarse_search(cent, xq, nprobe, L2)
    keys[2, 1] = -1
    lut8, ab = fso.lut(pq, xq, metric)
    dg, ig = fso.search_preassigned(off, codes, ids, lut8, ab, xq, k, keys, metric, M,
                                    del_bitmap=np.packbits(deleted, bitorder="little"))
    ref = _loop_search(off, codes, ids, lut8, ab, keys, k, metric, M, deleted)
    for q in range(nq):
        got = [(dg[q, i], ig[q, i]) for i in range(k) if ig[q, i] >= 0]
        assert [s for s, _ in got] == [s for s, _ in ref[q]]
        for s in {s for s, _ in got}:  # equal scores: the same ids (the output order inside them is the decoder's)
            assert {i for t, i in got if t == s} == {i for t, i in ref[q] if t == s} or s == got[-1][0]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M,data", [(32, 16, "int"), (30, 15, "float"), (24, 12, "float"), (16, 8, "int")])
def test_c_restatement_and_numpy_twin_agree_byte_for_byte(metric, d, M, data):
    n, nq, nlist, nprobe = 3000, 12, 16, 5
    db = synth.sift_like(n, d, seed=21, rounded=data == "int")
    xq = synth.sift_like(nq, d, seed=22, rounded=data == "int")
    pq, _ = cfs.pq_train(db, M, niter=4)
    packed = cfs.encode_packed(pq, db)
    assert np.array_equal(packed, fso.pack(fso.encode(pq, db)))
    for tab_pq in (pq, np.full_like(pq, 3)):  # the second: every span 0 (degenerate table)
        l8c, abc = cfs.lut(tab_pq, xq, metric)
        l8n, abn = fso.lut(tab_pq, xq, metric)
        assert np.array_equal(l8c, l8n) and np.array_equal(abc.view(np.uint32), abn.view(np.uint32))
    lut8, ab = cfs.lut(pq, xq, metric)
    cent, _, _ = orc.kmeans(db, nlist, niter=4)
    off, order = orc.build_lists(orc.assign(cent, db, L2), nlist)
    codes, ids = packed[order], order.astype(np.int64)
    ids[7] |= np.int64(-(2 ** 63))  # a tombstone
    _, keys = orc.coarse_search(cent, xq, nprobe, L2)
    keys[1, 3] = -1
    rng = np.random.default_rng(4)
    delb = np.packbits(rng.random(n) < 0.2, bitorder="little")
    filb = np.packbits(rng.random(n) < 0.7, bitorder="little")
    base = dict(del_bitmap=delb, filter_bitmap=filb)
    dw, _ = fso.search_preassigned(off, codes, ids, lut8, ab, xq, 20, keys, metric, M, **base)
    lo, hi = sorted((float(dw[0, 3]), float(dw[0, 15])))
    for k, recall_num, extra in ((1, 0, {}), (10, 0, base), (100, 0, {}), (10, 50, base),
                                 (20, 0, dict(base, min_score=lo, max_score=hi)),
                                 (10, 60, dict(base, min_score=lo, max_score=hi))):
        dc, ic = cfs.search_preassigned(off, codes, ids, lut8, ab, xq, k, keys, metric, M, recall_num=recall_num, raw=db,
                                        **extra)
        dn, in_ = fso.search_preassigned(off, codes, ids, lut8, ab, xq, k, keys, metric, M, recall_num=recall_num, raw=db,
                                         **extra)
        assert np.array_equal(dc.view(np.uint32), dn.view(np.uint32)) and np.array_equal(ic, in_), (k, recall_num, extra)
