"""numpy twin of the C restatement in ivfpqfs_oracle.c (TEST INFRASTRUCTURE ONLY): the IVFPQFastScan index (faiss
IndexIVFPQFastScan with by_residual = false, as gamma's index/impl/gamma_index_ivfpqfs.cc builds it) -- 4-bit
encoding and packing, the float table, its uint8 quantisation (faiss quantize_lut::round_uint8_per_column) and the
search over given probes.  PQ training is ivfpqfs.pq_train.

Every floating-point step is a float32 numpy operation, one rounding per operation and no fused multiply-add, in the
order the device kernels use: per sub-vector the sum runs sequentially over the dsub columns.  After quantisation the
arithmetic is integer until the score  accu * (1 / a) + b.
"""
import numpy as np

from oracle import oracle as orc

KSUB = 16
F32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)


def encode(pq, x):
    """codes [n, M]: per sub-vector the nearest of the 16 centroids, lowest index on ties."""
    M, ksub, dsub = pq.shape
    x = np.ascontiguousarray(x, F32)
    codes = np.empty((x.shape[0], M), np.uint8)
    for m in range(M):
        dis = np.zeros((x.shape[0], ksub), F32)
        for j in range(dsub):
            t = x[:, m * dsub + j][:, None] - pq[m, :, j][None, :]
            dis = dis + t * t
        codes[:, m] = np.argmin(dis, axis=1)
    return codes


def pack(codes):
    """two codes per byte, sub-quantiser 2j in the low nibble of byte j (BitstringWriter order); odd M: last high nibble 0"""
    n, M = codes.shape
    out = np.zeros((n, (M + 1) // 2), np.uint8)
    out[:] = codes[:, 0::2]
    out[:, :M // 2] |= codes[:, 1::2] << 4
    return out


def unpack(packed, M):
    codes = np.empty((packed.shape[0], M), np.uint8)
    codes[:, 0::2] = packed[:, :(M + 1) // 2] & 15
    codes[:, 1::2] = packed[:, :M // 2] >> 4
    return codes


def float_lut(pq, xq, metric):
    """[nq, M, 16]: sum_j (x_j - c_j)^2 (L2) or sum_j x_j c_j (IP), sequentially over j"""
    M, ksub, dsub = pq.shape
    xq = np.ascontiguousarray(xq, F32)
    tab = np.zeros((xq.shape[0], M, ksub), F32)
    for j in range(dsub):
        xj = xq[:, j::dsub][:, :M, None]  # column m * dsub + j of every sub-vector
        cj = pq[None, :, :, j]
        tab = tab + ((xj - cj) * (xj - cj) if metric == orc.METRIC_L2 else xj * cj)
    return tab


def quantize_lut(tab):
    """round_uint8_per_column: lut8 = floor((v - min_m) * a + 0.5), a = 255 / max_m span_m, b = sum_m min_m (m order).
    Every span 0: faiss divides by zero; here a = 1 and the table is all zero."""
    nq, M, _ = tab.shape
    mins = tab.min(axis=2)
    spans = tab.max(axis=2) - mins
    max_span = np.maximum(spans.max(axis=1), F32(0))
    a = np.where(max_span > 0, F32(255) / np.where(max_span > 0, max_span, F32(1)), F32(1)).astype(F32)
    b = np.zeros(nq, F32)
    for m in range(M):
        b = b + mins[:, m]
    lut8 = np.floor((tab - mins[:, :, None]) * a[:, None, None] + F32(0.5)).astype(np.uint8)
    return lut8, np.stack([a, b], axis=1).astype(F32)


def lut(pq, xq, metric):
    return quantize_lut(float_lut(pq, xq, metric))


def scores(lut8_q, ab_q, codes):
    """accu * (1 / a) + b of entries with unpacked codes [n, M] under one query's table"""
    M = lut8_q.shape[0]
    accu = lut8_q[np.arange(M)[None, :], codes.astype(np.int64)].astype(np.int64).sum(axis=1)
    one_a = F32(1) / ab_q[0]
    return accu.astype(F32) * one_a + ab_q[1]


def _bit(bitmap, ids):
    return (bitmap[ids >> 3] >> (ids & 7)) & 1


def _top(dis, ids, k, metric):
    """the k best by the engine's key (score, then smaller id), in the output order of its decoder: L2 ascending,
    IP descending with the larger id first among equal scores"""
    order = np.lexsort((ids, dis if metric == orc.METRIC_L2 else -dis))[:k]
    d, i = dis[order], ids[order]
    if metric != orc.METRIC_L2:
        o = np.lexsort((-i, -d))
        d, i = d[o], i[o]
    od = np.full(k, FLT_MAX if metric == orc.METRIC_L2 else -FLT_MAX, F32)
    oi = np.full(k, -1, np.int64)
    od[:len(d)], oi[:len(i)] = d, i
    return od, oi


def search_preassigned(list_off, list_codes, list_ids, lut8, ab, xq, k, keys, metric, M, recall_num=0, raw=None,
                       del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX, max_score=FLT_MAX):
    """fast-scan search over the probed lists keys[q] (-1 = none).  Filters and the score window apply to every
    entry before selection; recall_num > 0 keeps the max(k, recall_num) best and re-ranks them exactly from raw."""
    nq = keys.shape[0]
    kk = max(k, recall_num) if recall_num > 0 else k
    out_d = np.empty((nq, k), F32)
    out_i = np.empty((nq, k), np.int64)
    for q in range(nq):
        sel = [np.arange(list_off[l], list_off[l + 1]) for l in keys[q] if l >= 0]
        pos = np.concatenate(sel) if sel else np.zeros(0, np.int64)
        ids = list_ids[pos]
        dis = scores(lut8[q], ab[q], unpack(list_codes[pos], M))
        ok = (ids >= 0) & (dis >= F32(min_score)) & (dis <= F32(max_score))
        vid = np.where(ids >= 0, ids, 0)
        if del_bitmap is not None:
            ok &= _bit(del_bitmap, vid) == 0
        if filter_bitmap is not None:
            ok &= _bit(filter_bitmap, vid) == 1
        d, i = _top(dis[ok], ids[ok], kk, metric)
        if recall_num > 0:
            i = i[i >= 0]
            rows, x = np.ascontiguousarray(raw[i], F32), np.ascontiguousarray(xq[q], F32)
            ex = np.zeros(len(i), F32)
            for j in range(rows.shape[1]):  # sequentially over d, as the C restatement
                ex = ex + ((rows[:, j] - x[j]) * (rows[:, j] - x[j]) if metric == orc.METRIC_L2 else rows[:, j] * x[j])
            w = (ex >= F32(min_score)) & (ex <= F32(max_score))
            d, i = _top(ex[w], i[w], k, metric)
        out_d[q], out_i[q] = d[:k], i[:k]
    return out_d, out_i


def assert_same_results(dg, ig, do, io):
    """scores bit-equal; ids equal except inside the group of exactly tied scores at the k-th boundary"""
    assert dg.shape == do.shape and ig.shape == io.shape
    assert np.array_equal(dg, do), f"score mismatch: max abs diff {np.abs(dg - do).max()}"
    for q in range(dg.shape[0]):
        if np.array_equal(ig[q], io[q]):
            continue
        valid = io[q] >= 0
        assert np.array_equal(valid, ig[q] >= 0), "different number of results"
        boundary = do[q][valid][-1]
        for v in np.unique(do[q][valid]):
            grp = valid & (do[q] == v)
            if v != boundary:
                assert set(ig[q][grp]) == set(io[q][grp]), f"query {q}: ids differ at score {v}"
