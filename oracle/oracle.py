"""ctypes binding of oracle/liboracle.so (gamma_oracle.c).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (vearch_b200) never imports it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle.so")

METRIC_IP = 0
METRIC_L2 = 1
DEL_MASK = np.int64(-(2**63))

_lib = None


def build(force=False):
    src = os.path.join(_HERE, "gamma_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        _lib = C.CDLL(_SO)
        _lib.orc_l2sqr.restype = C.c_float
        _lib.orc_inner_product.restype = C.c_float
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _bm(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.uint8)


def num_threads():
    return int(lib().orc_num_threads())


def flat_search(db, xq, k, metric, del_bitmap=None, filter_bitmap=None, min_score=-3.4028235e38,
                max_score=3.4028235e38):
    db, xq = _f32(db), _f32(xq)
    n, d = db.shape
    nq = xq.shape[0]
    dis = np.empty((nq, k), np.float32)
    ids = np.empty((nq, k), np.int64)
    delb, filb = _bm(del_bitmap), _bm(filter_bitmap)
    rc = lib().orc_flat_search(_p(db), C.c_int64(d), C.c_int64(n), C.c_int(d), _p(xq), C.c_int(nq), C.c_int(k),
                               C.c_int(metric), _p(delb), _p(filb), C.c_float(min_score), C.c_float(max_score),
                               _p(dis), _p(ids))
    assert rc == 0
    return dis, ids


def coarse_search(centroids, xq, nprobe, metric):
    centroids, xq = _f32(centroids), _f32(xq)
    L, d = centroids.shape
    nq = xq.shape[0]
    dis = np.empty((nq, nprobe), np.float32)
    ids = np.empty((nq, nprobe), np.int64)
    rc = lib().orc_coarse_search(_p(centroids), C.c_int(L), C.c_int(d), _p(xq), C.c_int(nq), C.c_int(nprobe),
                                 C.c_int(metric), _p(dis), _p(ids))
    assert rc == 0
    return dis, ids


def assign(centroids, x, metric):
    centroids, x = _f32(centroids), _f32(x)
    L, d = centroids.shape
    out = np.empty(x.shape[0], np.int64)
    rc = lib().orc_assign(_p(centroids), C.c_int(L), C.c_int(d), _p(x), C.c_int64(x.shape[0]), C.c_int(metric), _p(out))
    assert rc == 0
    return out


def build_lists(assign_ids, nlist):
    """CSR inverted lists in insertion (vid) order -- RTInvertIndex semantics
    (index/realtime/realtime_mem_data.cc:258-296). Returns (list_off, order)."""
    assign_ids = np.asarray(assign_ids, np.int64)
    order = np.argsort(assign_ids, kind="stable")
    counts = np.bincount(assign_ids, minlength=nlist)
    off = np.zeros(nlist + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    return off, order


def ivfflat_search_preassigned(list_off, list_vecs, list_ids, xq, k, keys, metric, del_bitmap=None,
                               filter_bitmap=None, min_score=-3.4028235e38, max_score=3.4028235e38):
    list_off, list_vecs, list_ids = _i64(list_off), _f32(list_vecs), _i64(list_ids)
    xq, keys = _f32(xq), _i64(keys)
    nq, d = xq.shape
    nprobe = keys.shape[1]
    nlist = list_off.shape[0] - 1
    dis = np.empty((nq, k), np.float32)
    ids = np.empty((nq, k), np.int64)
    delb, filb = _bm(del_bitmap), _bm(filter_bitmap)
    rc = lib().orc_ivfflat_search_preassigned(_p(list_off), _p(list_vecs), _p(list_ids), C.c_int(nlist), C.c_int(d),
                                              _p(xq), C.c_int(nq), C.c_int(k), _p(keys), C.c_int(nprobe),
                                              C.c_int(metric), _p(delb), _p(filb), C.c_float(min_score),
                                              C.c_float(max_score), _p(dis), _p(ids))
    assert rc == 0
    return dis, ids


def pq_compute_codes(pq_centroids, x):
    pq_centroids, x = _f32(pq_centroids), _f32(x)
    M, ksub, dsub = pq_centroids.shape
    assert ksub == 256
    n = x.shape[0]
    codes = np.empty((n, M), np.uint8)
    rc = lib().orc_pq_compute_codes(_p(pq_centroids), C.c_int(M), C.c_int(dsub), _p(x), C.c_int64(n), _p(codes))
    assert rc == 0
    return codes


def ivfpq_encode(coarse_centroids, pq_centroids, x, assign_ids):
    coarse_centroids, pq_centroids, x, assign_ids = _f32(coarse_centroids), _f32(pq_centroids), _f32(x), _i64(assign_ids)
    M = pq_centroids.shape[0]
    n, d = x.shape
    codes = np.empty((n, M), np.uint8)
    rc = lib().orc_ivfpq_encode(_p(coarse_centroids), C.c_int(d), _p(pq_centroids), C.c_int(M), _p(x), C.c_int64(n),
                                _p(assign_ids), _p(codes))
    assert rc == 0
    return codes


def ivfpq_precompute_table(coarse_centroids, pq_centroids):
    coarse_centroids, pq_centroids = _f32(coarse_centroids), _f32(pq_centroids)
    L, d = coarse_centroids.shape
    M = pq_centroids.shape[0]
    T = np.empty((L, M, 256), np.float32)
    rc = lib().orc_ivfpq_precompute_table(_p(coarse_centroids), C.c_int(L), C.c_int(d), _p(pq_centroids), C.c_int(M), _p(T))
    assert rc == 0
    return T


def ivfpq_search_preassigned(list_off, list_codes, list_ids, coarse_centroids, pq_centroids, precomputed_table, xq, k,
                             keys, coarse_dis, metric, recall_num=0, raw=None, del_bitmap=None, filter_bitmap=None,
                             min_score=-3.4028235e38, max_score=3.4028235e38):
    list_off, list_ids = _i64(list_off), _i64(list_ids)
    list_codes = np.ascontiguousarray(list_codes, np.uint8)
    coarse_centroids, pq_centroids, xq = _f32(coarse_centroids), _f32(pq_centroids), _f32(xq)
    keys, coarse_dis = _i64(keys), _f32(coarse_dis)
    T = None if precomputed_table is None else _f32(precomputed_table)
    rawc = None if raw is None else _f32(raw)
    nq, d = xq.shape
    M = pq_centroids.shape[0]
    nprobe = keys.shape[1]
    nlist = list_off.shape[0] - 1
    dis = np.empty((nq, k), np.float32)
    ids = np.empty((nq, k), np.int64)
    delb, filb = _bm(del_bitmap), _bm(filter_bitmap)
    rc = lib().orc_ivfpq_search_preassigned(
        _p(list_off), _p(list_codes), _p(list_ids), C.c_int(nlist), C.c_int(d), C.c_int(M), _p(coarse_centroids),
        _p(pq_centroids), _p(T), _p(xq), C.c_int(nq), C.c_int(k), _p(keys), _p(coarse_dis), C.c_int(nprobe),
        C.c_int(metric), C.c_int(recall_num), _p(rawc), C.c_int64(0 if rawc is None else rawc.shape[1]), _p(delb),
        _p(filb), C.c_float(min_score), C.c_float(max_score), _p(dis), _p(ids))
    assert rc == 0
    return dis, ids


def rand_perm(n, seed):
    perm = np.empty(n, np.int64)
    lib().orc_rand_perm(_p(perm), C.c_int64(n), C.c_int64(seed))
    return perm


def kmeans_update(x, k, assign_ids):
    x, assign_ids = _f32(x), _i64(assign_ids)
    n, d = x.shape
    cent = np.empty((k, d), np.float32)
    hassign = np.empty(k, np.float32)
    lib().orc_kmeans_update(_p(x), C.c_int64(n), C.c_int(d), C.c_int(k), _p(assign_ids), _p(cent), _p(hassign))
    return cent, hassign


def kmeans_split(hassign, centroids, n):
    """faiss's split_clusters (EPS = 1/1024, rng(1234)) on copies: every empty cluster re-seeded from a big one.  n: the
    rows trained on.  Returns (centroids, hassign, number of splits)."""
    cent = _f32(centroids).copy()
    h = _f32(hassign).copy()
    k, d = cent.shape
    ns = lib().orc_kmeans_split(C.c_int(d), C.c_int(k), C.c_int64(n), _p(h), _p(cent))
    return cent, h, int(ns)


def kmeans_normalize(centroids):
    """spherical k-means' renormalisation of the centroids, on a copy (a zero row stays zero)"""
    cent = _f32(centroids).copy()
    k, d = cent.shape
    lib().orc_kmeans_normalize(_p(cent), C.c_int(k), C.c_int(d))
    return cent


def kmeans(x, k, niter=25, seed=1234, spherical=False, max_points_per_centroid=256, l2_assign=False):
    """l2_assign: spherical, but assigned by L2 (the clustering index IVFPQFastScan and VEARCH keep under IP)"""
    x = _f32(x)
    n, d = x.shape
    cent = np.empty((k, d), np.float32)
    assign_ids = np.full(n, -1, np.int64)
    obj = np.zeros(niter, np.float32)
    rc = lib().orc_kmeans(_p(x), C.c_int64(n), C.c_int(d), C.c_int(k), C.c_int(niter), C.c_int64(seed),
                          C.c_int(1 if spherical else 0), C.c_int(1 if l2_assign else 0), C.c_int(max_points_per_centroid),
                          _p(cent), _p(assign_ids), _p(obj))
    assert rc == 0
    return cent, assign_ids, obj


def pq_train(x, M, niter=25, seed=1234):
    x = _f32(x)
    n, d = x.shape
    out = np.empty((M, 256, d // M), np.float32)
    rc = lib().orc_pq_train(_p(x), C.c_int64(n), C.c_int(d), C.c_int(M), C.c_int(niter), C.c_int64(seed), _p(out))
    assert rc == 0
    return out


def merge_partitions(dis, ids, metric):
    """dis/ids: [nparts, nq, k] per-partition sorted results -> merged [nq, k] (router order)."""
    dis, ids = _f32(dis), _i64(ids)
    nparts, nq, k = dis.shape
    od = np.empty((nq, k), np.float32)
    oi = np.empty((nq, k), np.int64)
    lib().orc_merge_partitions(_p(dis), _p(ids), C.c_int(nparts), C.c_int(nq), C.c_int(k), C.c_int(metric), _p(od), _p(oi))
    return od, oi
