"""Plain key-order reference of the engine's top-k contract (test infrastructure only).

Every search path orders its results by the 64-bit key  (order-preserving score bits << 32) | vid: the best score
first, the smaller vid first among equal scores (common.cuh f2ord / score2ord / make_key).  The decoder
(kernels_select.cu decode_keys_kernel) lists equal IP scores with the larger id first and fills empty slots with id -1
and score +-FLT_MAX.

The scores fed in here are exact: integers computed in int64 and checked against 2^24, below which every fp32
evaluation order of the same sum gives the same float, or scores that are themselves the float32 result of a restated
computation (IVFPQFastScan's quantised tables).  The comparison with the engine can then be exact, key for key.
"""
import numpy as np

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)
SENTINEL = np.uint64(0xFFFFFFFFFFFFFFFF)
EXACT_LIMIT = 1 << 24
METRIC_IP, METRIC_L2 = 0, 1  # DistanceComputeType (oracle.METRIC_*)


class InexactScores(ValueError):
    """a score, or a bound on a partial sum of one, is not exactly representable in fp32"""


def guard(bound, what="score"):
    """raise unless |bound| < 2^24 everywhere: integers below it are exact in fp32, so is every partial sum below it"""
    b = np.max(np.abs(np.asarray(bound, np.int64))) if np.size(bound) else 0
    if b >= EXACT_LIMIT:
        raise InexactScores(f"{what} bound {int(b)} reaches 2^24: fp32 sums of it depend on the evaluation order")


def f2ord(s):
    """float32 -> uint32, order-preserving over the whole line: -FLT_MAX < ... < -0.0 < +0.0 < ... < FLT_MAX"""
    b = np.ascontiguousarray(s, F32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def ord2f(o):
    o = np.asarray(o, np.uint32)
    b = np.where(o & np.uint32(0x80000000), o & np.uint32(0x7FFFFFFF), ~o).astype(np.uint32)
    return b.view(F32)


def score2ord(s, metric):
    o = f2ord(s)
    return o if metric == METRIC_L2 else ~o


def to_f32(scores):
    """the float32 image of exact scores: integers are guarded, float32 passes through; exact zero is +0.0"""
    s = np.asarray(scores)
    if s.dtype.kind in "iu":
        guard(s)
        return s.astype(F32)
    if s.dtype != F32:
        raise TypeError(f"scores must be integers or float32, not {s.dtype}")
    return s


def keys(scores, vids, valid=None, metric=METRIC_L2):
    """the engine's keys of (score, vid) pairs; invalid pairs get the sentinel"""
    s = to_f32(scores)
    k = (score2ord(s, metric).astype(np.uint64) << np.uint64(32)) | (np.asarray(vids).astype(np.uint64) & np.uint64(0xFFFFFFFF))
    if valid is not None:
        k = np.where(valid, k, SENTINEL)
    return k


def topk(key_rows, k):
    """the k smallest keys of every row, ascending, padded with the sentinel when a row has fewer than k columns"""
    key_rows = np.atleast_2d(key_rows)
    n = key_rows.shape[1]
    out = np.full((key_rows.shape[0], k), SENTINEL, np.uint64)
    if n:
        kk = min(k, n)
        part = np.partition(key_rows, kk - 1, axis=1)[:, :kk] if kk < n else key_rows
        out[:, :kk] = np.sort(part, axis=1)[:, :kk]
    return out


def decode(key_rows, metric):
    """(scores float32, ids int64) in the engine's output order"""
    key_rows = np.atleast_2d(np.asarray(key_rows, np.uint64))
    nq, k = key_rows.shape
    empty = key_rows == SENTINEL
    dis = ord2f(score2ord_inv(key_rows >> np.uint64(32), metric))
    ids = (key_rows & np.uint64(0xFFFFFFFF)).astype(np.int64)
    dis = np.where(empty, F32(FLT_MAX if metric == METRIC_L2 else -FLT_MAX), dis).astype(F32)
    ids = np.where(empty, -1, ids)
    if metric == METRIC_IP:  # heap_reorder on a CMin heap: equal scores with the larger id first
        hi = (key_rows >> np.uint64(32)).astype(np.int64)
        for q in range(nq):
            i = 0
            while i < k and not empty[q, i]:
                j = i
                while j + 1 < k and not empty[q, j + 1] and hi[q, j + 1] == hi[q, i]:
                    j += 1
                ids[q, i:j + 1] = ids[q, i:j + 1][::-1]
                i = j + 1
    return dis, ids


def score2ord_inv(hi, metric):
    hi = np.asarray(hi).astype(np.uint32)
    return hi if metric == METRIC_L2 else ~hi


def bit(bitmap, vids):
    """bit vid of an LSB-first byte bitmap (the engine reads it as 32-bit words: the same bits on little-endian)"""
    vids = np.asarray(vids, np.int64)
    return (bitmap[vids >> 3] >> (vids & 7)) & 1


def validity(raw_ids, del_bitmap=None, filter_bitmap=None):
    """tombstones (top bit of the list id) and RetrievalContext::IsValid over raw list ids; -> (valid, vid)"""
    raw_ids = np.asarray(raw_ids, np.int64)
    ok = raw_ids >= 0
    vid = np.where(ok, raw_ids, 0) & 0xFFFFFFFF
    if filter_bitmap is not None:
        ok &= bit(filter_bitmap, vid) == 1
    if del_bitmap is not None:
        ok &= bit(del_bitmap, vid) == 0
    return ok, vid


def in_window(s32, min_score, max_score):
    return (s32 >= F32(min_score)) & (s32 <= F32(max_score))


# ---- exact scores -------------------------------------------------------------------------------------------------
def exact_scores(xq, rows, metric):
    """[nq, n] int64 L2 / IP scores of integer-valued rows, guarded so that every fp32 evaluation order is exact (the
    L2 bound also covers the |x|^2 + |y|^2 - 2 x.y form of the tensor-core kernels)"""
    x = _ints(xq)
    y = _ints(rows)
    if metric == METRIC_L2:
        xn, yn = (x * x).sum(1), (y * y).sum(1)
        guard(xn.max(initial=0) + yn.max(initial=0), "L2 norm")
        return xn[:, None] + yn[None, :] - 2 * (x @ y.T)
    guard(np.abs(x) @ np.abs(y).T, "inner-product partial sum")
    return x @ y.T


def _ints(a):
    a = np.asarray(a)
    r = np.rint(a).astype(np.int64)
    if not np.array_equal(r, a):
        raise InexactScores("rows are not integer-valued")
    return r


def unpack_codes(codes, M, nbits):
    """[n, code_size] bit-packed rows (code m at bits [m nbits, (m + 1) nbits), LSB-first) -> [n, M] codes"""
    codes = np.asarray(codes, np.uint8)
    if nbits == 8:
        return codes[:, :M].astype(np.int64)
    bits = np.unpackbits(codes, axis=1, bitorder="little")[:, :M * nbits].reshape(len(codes), M, nbits)
    return (bits.astype(np.int64) << np.arange(nbits)).sum(2)


def pq_reconstruct(cent, pq, entry_list, codes):
    """[n, d] int64 reconstructions c_l + sum_m pq[m][code_m] of list entries, integer centroids and codebooks"""
    c, p = _ints(cent), _ints(pq)
    M, _, dsub = p.shape
    rec = c[entry_list].copy()
    for m in range(M):
        rec[:, m * dsub:(m + 1) * dsub] += p[m][codes[:, m]]
    return rec


def pq_guard(xq, cent, pq, metric):
    """bound on every partial sum of the engine's IVF-PQ arithmetic: dis0 + sum_m lut[m][code_m], with lut = T - 2 ip
    (L2, T = |pq|^2 + 2 <c|m, pq>) or ip (IP); each table entry is itself a guarded sum of products"""
    x, c, p = _ints(xq), _ints(cent), _ints(pq)
    M, ksub, dsub = p.shape
    ax, ac, ap = np.abs(x), np.abs(c), np.abs(p)
    ipb = np.einsum("qmj,mcj->qmc", ax.reshape(len(x), M, dsub), ap).max(2).sum(1)  # sum_m max_c |<x|m, pq>|
    if metric == METRIC_L2:
        d0 = (x * x).sum(1).max() + (c * c).sum(1).max() + 2 * (ax @ ac.T).max()
        tb = ((ap * ap).sum(2)[None] + 2 * np.einsum("lmj,mcj->lmc", ac.reshape(len(c), M, dsub), ap)).max(2).sum(1)
        guard(d0 + tb.max() + 2 * ipb.max(), "IVF-PQ partial sum")
    else:
        guard((ax @ ac.T).max() + ipb.max(), "IVF-PQ partial sum")


# ---- searches over given probes ----------------------------------------------------------------------------------
def search_entries(entry_scores, entry_list, entry_raw_ids, probes, k, metric, del_bitmap=None, filter_bitmap=None,
                   min_score=-FLT_MAX, max_score=FLT_MAX):
    """keys [nq, k] of a search over probed lists.  entry_scores [nq, N]: exact score of every list entry for every
    query (int64 or float32); entry_list / entry_raw_ids [N]: each entry's list and raw list id; probes [nq, nprobe]
    (-1 = no list)"""
    s32 = to_f32(entry_scores)
    ok, vid = validity(entry_raw_ids, del_bitmap, filter_bitmap)
    nl = max(int(entry_list.max(initial=0)), int(np.max(probes, initial=0))) + 1
    probed = np.zeros((len(probes), nl + 1), bool)
    pr = np.where(probes >= 0, probes, nl)
    probed[np.arange(len(probes))[:, None], pr] = True
    probed[:, nl] = False
    valid = probed[:, entry_list] & ok[None, :] & in_window(s32, min_score, max_score)
    return topk(keys(s32, vid[None, :], valid, metric), k)


def flat_keys(xq, db, k, metric, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX, max_score=FLT_MAX):
    s = exact_scores(xq, db, metric)
    n = db.shape[0]
    return search_entries(s, np.zeros(n, np.int64), np.arange(n), np.zeros((len(xq), 1), np.int64), k, metric, del_bitmap,
                          filter_bitmap, min_score, max_score)


def rerank_keys(adc_keys, xq, db, k, metric, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX,
                max_score=FLT_MAX):
    """exact re-rank: the k best, by exact score from the raw rows, of each query's ADC candidates"""
    out = np.full((len(xq), k), SENTINEL, np.uint64)
    for q in range(len(xq)):
        cand = adc_keys[q][adc_keys[q] != SENTINEL]
        vid = (cand & np.uint64(0xFFFFFFFF)).astype(np.int64)
        s = exact_scores(xq[q:q + 1], db[vid], metric)
        ok, _ = validity(vid, del_bitmap, filter_bitmap)
        out[q] = topk(keys(s, vid[None, :], ok[None, :] & in_window(to_f32(s), min_score, max_score), metric), k)[0]
    return out
