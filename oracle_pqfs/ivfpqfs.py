"""ctypes binding of oracle_pqfs/libivfpqfs_oracle.so (ivfpqfs_oracle.c): the IVFPQFastScan restatement in C.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py.  Same arguments and results as the numpy twin in twin.py; the CPU
tests hold the two byte-equal."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libivfpqfs_oracle.so")
KSUB = 16
FLT_MAX = float(np.finfo(np.float32).max)
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "ivfpqfs_oracle.c")
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", _HERE, "-s"])
        _lib = C.CDLL(_SO)
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def pq_train(x, M, ksub=KSUB, niter=25, seed=1234):
    """ProductQuantizer::train: M independent ksub-means (oracle/gamma_oracle.c's k-means, at most 256 points per
    centroid) on the dsub-wide slices of the raw rows.  Returns ([M][ksub][dsub], per-sub-quantiser objectives)."""
    x = _f32(x)
    dsub = x.shape[1] // M
    out = np.empty((M, ksub, dsub), np.float32)
    objs = []
    for m in range(M):
        c, _, obj = orc.kmeans(x[:, m * dsub:(m + 1) * dsub], ksub, niter=niter, seed=seed)
        out[m] = c
        objs.append(obj)
    return out, objs


def encode_packed(pq, x):
    pq, x = _f32(pq), _f32(x)
    M, _, dsub = pq.shape
    codes = np.empty((x.shape[0], (M + 1) // 2), np.uint8)
    assert lib().orcfs_encode(_p(pq), C.c_int(M), C.c_int(dsub), _p(x), C.c_int64(x.shape[0]), _p(codes)) == 0
    return codes


def lut(pq, xq, metric):
    pq, xq = _f32(pq), _f32(xq)
    M, _, dsub = pq.shape
    nq = xq.shape[0]
    lut8 = np.empty((nq, M, KSUB), np.uint8)
    ab = np.empty((nq, 2), np.float32)
    assert lib().orcfs_lut(_p(pq), C.c_int(M), C.c_int(dsub), _p(xq), C.c_int(nq), C.c_int(metric), _p(lut8), _p(ab)) == 0
    return lut8, ab


def search_preassigned(list_off, list_codes, list_ids, lut8, ab, xq, k, keys, metric, M, recall_num=0, raw=None,
                       del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX, max_score=FLT_MAX):
    list_off = np.ascontiguousarray(list_off, np.int64)
    list_ids = np.ascontiguousarray(list_ids, np.int64)
    list_codes = np.ascontiguousarray(list_codes, np.uint8)
    lut8, ab, xq = np.ascontiguousarray(lut8, np.uint8), _f32(ab), _f32(xq)
    keys = np.ascontiguousarray(keys, np.int64)
    rawc = None if raw is None else _f32(raw)
    delb = None if del_bitmap is None else np.ascontiguousarray(del_bitmap, np.uint8)
    filb = None if filter_bitmap is None else np.ascontiguousarray(filter_bitmap, np.uint8)
    nq, d = xq.shape
    dis = np.empty((nq, k), np.float32)
    ids = np.empty((nq, k), np.int64)
    rc = lib().orcfs_search_preassigned(
        _p(list_off), _p(list_codes), _p(list_ids), C.c_int(len(list_off) - 1), C.c_int(M), _p(lut8), _p(ab), _p(xq),
        C.c_int(d), C.c_int(nq), C.c_int(k), _p(keys), C.c_int(keys.shape[1]), C.c_int(metric), C.c_int(recall_num),
        _p(rawc), C.c_int64(0 if rawc is None else rawc.shape[1]), _p(delb), _p(filb), C.c_float(min_score),
        C.c_float(max_score), _p(dis), _p(ids))
    assert rc == 0
    return dis, ids
