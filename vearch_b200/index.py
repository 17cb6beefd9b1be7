"""Host-side mirror of the reference's index interface for the hot path.

Names follow the reference: `index_factory`, `train / add / search` of the faiss-like wrappers
(internal/engine/index/index.h:  vearch::IndexIVFFlat, vearch::IndexIVFPQ, index_factory) and
the IndexModel plug-in verbs `Indexing / Add / Search` (internal/engine/index/index_model.h:229-335).
Everything below is a thin ctypes shim over include/gamma_b200_index.h; all compute happens in
vearch_b200/libgamma.so (sm_90a CUDA).  There is no CPU fallback.
"""
import ctypes as C
import json

import numpy as np

from . import _lib

METRIC_IP = 0  # DistanceComputeType::INNER_PRODUCT (gamma's default)
METRIC_L2 = 1
FLT_MAX = 3.4028234663852886e38


class GammaError(RuntimeError):
    pass


class SearchKilled(GammaError):
    """A search whose cancel token was set before it finished (the C-ABI's -2)."""


def _check(rc, what):
    if rc == -2:
        raise SearchKilled(f"{what} killed")
    if rc != 0:
        raise GammaError(f"{what} failed (rc={rc}): {_lib.last_error()}")


class CancelToken:
    """One cancel word of a search (gb_cancel_token): set() stops the searches given it early, and they raise
    SearchKilled.  It only ever goes from unset to set; one search at a time may hold it."""

    def __init__(self):
        self._h = _lib.lib().gb_cancel_token_create()
        if not self._h:
            raise GammaError(f"cancel token: {_lib.last_error()}")

    def set(self):
        _lib.lib().gb_cancel_token_set(self._h)

    def is_set(self):
        return bool(_lib.lib().gb_cancel_token_is_set(self._h))

    def close(self):
        if self._h:
            _lib.lib().gb_cancel_token_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _token(cancel):
    return None if cancel is None else C.c_void_p(cancel._h)


def debug_cancel_stats(device=0):
    """{kernel: CTAs that skipped their work on a set cancel word} on `device` since the last call, which clears them"""
    p, n = C.c_void_p(), C.c_int()
    _check(_lib.lib().gb_debug_cancel_stats(device, C.byref(p), C.byref(n)), "debug_cancel_stats")
    js = C.string_at(p.value, n.value).decode()
    C.CDLL(None).free(C.c_void_p(p.value))
    return json.loads(js)


def debug_cancel_register(request_id, partition_id, token, register=True):
    """the kill registry behind SetKillStatus, with `token` standing in for a running search's cancel word"""
    _check(_lib.lib().gb_debug_cancel_register(request_id.encode(), partition_id, C.c_void_p(token._h), int(register)),
           "debug_cancel_register")


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _bitmap(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.uint8)


class GammaIndex:
    """One vector field's raw store + index model on one GPU."""

    def __init__(self, index_type, d, params=None, device=0, store_type=None, devices=None):
        """store_type: where the raw vectors live, as a table's VectorInfo.store_type: "RocksDB" (any case) keeps them
        in pinned host memory, read over PCIe, so HBM holds only the index; anything else keeps them in HBM.
        devices: CUDA ordinals (one may repeat) a GPU_IVFPQ / GPU_IVFFLAT index is sharded over, vid v in shard
        v % len(devices); devices[0] holds the raw vectors and replaces `device`.  One entry, or another type: the index
        lives on devices[0]."""
        t = index_type.upper()
        self.index_type = "IVFPQFastScan" if t == "IVFPQFASTSCAN" else t  # gamma's spelling of the registered name
        self.d = int(d)
        self.device = device if not devices else int(devices[0])
        self._view = False
        params = dict(params or {})
        if store_type is not None:
            params["store_type"] = store_type
        pj = json.dumps(params).encode()
        if devices is None:
            self._h = _lib.lib().gb_index_create(self.index_type.encode(), self.d, pj, device)
        else:
            devs = (C.c_int * len(devices))(*[int(v) for v in devices])
            self._h = _lib.lib().gb_index_create_sharded(self.index_type.encode(), self.d, pj, devs, len(devices))
        if not self._h:
            raise GammaError(f"create {index_type}: {_lib.last_error()}")

    @property
    def shard_count(self):
        """Shards of the index: 1 unless it was created sharded over two devices or more."""
        return int(_lib.lib().gb_index_shard_count(self._h))

    def shard(self, i):
        """Shard i's index structures (lists, centroids, codebook, tables) as a GammaIndex, valid while this index
        lives; its raw store is empty (the rows stay with the sharded index).  close() frees only the handle."""
        h = _lib.lib().gb_index_shard(self._h, int(i))
        if not h:
            raise GammaError(f"shard {i}: {_lib.last_error()}")
        v = object.__new__(type(self))
        v.index_type, v.d, v.device, v._view, v._h, v._owner = self.index_type, self.d, None, True, h, self
        return v

    def close(self):
        if getattr(self, "_h", None):
            _lib.lib().gb_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- properties -------------------------------------------------------------------
    @property
    def ntotal(self):
        return int(_lib.lib().gb_index_ntotal(self._h))

    @property
    def indexed_count(self):
        return int(_lib.lib().gb_index_indexed_count(self._h))

    @property
    def is_trained(self):
        return bool(_lib.lib().gb_index_is_trained(self._h))

    @property
    def training_threshold(self):
        return int(_lib.lib().gb_index_training_threshold(self._h))

    @property
    def type(self):
        """The registered type name the index was created under ("GPU_IVFPQ" is an IVFPQ index under that name)."""
        return _lib.lib().gb_index_type(self._h).decode()

    @property
    def nlist(self):
        return int(_lib.lib().gb_index_nlist(self._h))

    @property
    def code_size(self):
        return int(_lib.lib().gb_index_code_size(self._h))

    def mem_bytes(self, which=0):
        """0: the index's HBM; 1: the raw vectors' HBM; 2: the raw vectors' pinned host memory."""
        return int(_lib.lib().gb_index_mem_bytes(self._h, which))

    # ---- build --------------------------------------------------------------------------
    def add_vectors(self, x):
        """VectorManager::AddToStore: append raw vectors (host ndarray or torch CUDA tensor)."""
        if hasattr(x, "is_cuda") and x.is_cuda:
            assert x.dtype.is_floating_point and x.dim() == 2 and x.shape[1] == self.d and x.stride(1) == 1
            _check(_lib.lib().gb_index_add_vectors_device(self._h, x.shape[0], C.c_void_p(x.data_ptr()), x.stride(0)),
                   "add_vectors_device")
            return
        x = _f32(x)
        assert x.ndim == 2 and x.shape[1] == self.d
        _check(_lib.lib().gb_index_add_vectors(self._h, x.shape[0], _ptr(x)), "add_vectors")

    def train(self):
        """IndexModel::Indexing(): train on the first training_threshold stored vectors."""
        _check(_lib.lib().gb_index_train(self._h), "train")

    def add_pending(self, del_bitmap=None):
        """VectorManager::AddRTVecsToIndex: index everything stored but not yet indexed."""
        b = _bitmap(del_bitmap)
        _check(_lib.lib().gb_index_add_pending(self._h, _ptr(b)), "add_pending")

    def add(self, x):
        """faiss-like add (index/index.h): store + index."""
        self.add_vectors(x)
        self.add_pending()

    def update_vector(self, vid, x):
        x = _f32(x).reshape(-1)
        _check(_lib.lib().gb_index_update_vector(self._h, vid, _ptr(x)), "update_vector")

    def get_vector(self, vid):
        out = np.empty(self.d, np.float32)
        _check(_lib.lib().gb_index_get_vector(self._h, vid, _ptr(out)), "get_vector")
        return out

    def get_vectors(self, start, n):
        out = np.empty((n, self.d), np.float32)
        _check(_lib.lib().gb_index_get_vectors(self._h, start, n, _ptr(out)), "get_vectors")
        return out

    # ---- search -------------------------------------------------------------------------
    def search(self, x, k, params=None, brute_force=False, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX,
               max_score=FLT_MAX, cancel=None, search_unindexed_tail=False):
        """IndexModel::Search. Returns (scores[nq,k] float32, ids[nq,k] int64).  cancel: a CancelToken; the search
        raises SearchKilled when it was set before the search finished.  search_unindexed_tail: enable_realtime's
        brute-force pass over the stored rows not yet indexed."""
        x = _f32(x)
        assert x.ndim == 2 and x.shape[1] == self.d
        nq = x.shape[0]
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        pj = json.dumps(params).encode() if params else b""
        db, fb = _bitmap(del_bitmap), _bitmap(filter_bitmap)
        bits = 0
        for b in (db, fb):
            if b is not None:
                bits = max(bits, b.size * 8)
        if cancel is None and not search_unindexed_tail:
            rc = _lib.lib().gb_index_search(self._h, nq, _ptr(x), k, pj, int(brute_force), _ptr(db), _ptr(fb), bits,
                                            C.c_float(min_score), C.c_float(max_score), _ptr(dis), _ptr(ids))
        else:
            rc = _lib.lib().gb_index_search_cancellable(self._h, nq, _ptr(x), k, pj, int(brute_force), _ptr(db), _ptr(fb),
                                                        bits, C.c_float(min_score), C.c_float(max_score),
                                                        int(search_unindexed_tail), _token(cancel), _ptr(dis), _ptr(ids))
        _check(rc, "search")
        return dis, ids

    def search_device(self, x, k, params=None, brute_force=False, out=None, del_bitmap=None, filter_bitmap=None,
                      min_score=-FLT_MAX, max_score=FLT_MAX, cancel=None):
        """Queries and results stay in HBM (torch CUDA tensors); asynchronous on torch's current stream.
        del_bitmap / filter_bitmap: CUDA uint8 tensors of one length on the index's device in search()'s layout
        (LSB-first, bit set => deleted / allowed, ids past the bitmap neither), read on that stream.  cancel: a
        CancelToken (without bitmaps or a score window); SearchKilled when it was set by the time the search was
        enqueued, and the outputs are undefined when it is set later."""
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
        nq = x.shape[0]
        if out is None:
            out = (torch.empty((nq, k), dtype=torch.float32, device=x.device),
                   torch.empty((nq, k), dtype=torch.int64, device=x.device))
        pj = json.dumps(params).encode() if params else b""
        st = torch.cuda.current_stream(x.device).cuda_stream
        if cancel is not None:
            assert del_bitmap is None and filter_bitmap is None and min_score == -FLT_MAX and max_score == FLT_MAX
            rc = _lib.lib().gb_index_search_device_cancellable(self._h, nq, C.c_void_p(x.data_ptr()), x.stride(0), k, pj,
                                                               int(brute_force), _token(cancel),
                                                               C.c_void_p(out[0].data_ptr()),
                                                               C.c_void_p(out[1].data_ptr()), C.c_void_p(st))
            _check(rc, "search_device")
            return out
        if del_bitmap is None and filter_bitmap is None and min_score == -FLT_MAX and max_score == FLT_MAX:
            rc = _lib.lib().gb_index_search_device(self._h, nq, C.c_void_p(x.data_ptr()), x.stride(0), k, pj,
                                                   int(brute_force), C.c_void_p(out[0].data_ptr()),
                                                   C.c_void_p(out[1].data_ptr()), C.c_void_p(st))
            _check(rc, "search_device")
            return out
        # one bitmap_bits covers both bitmaps, as in search()
        assert del_bitmap is None or filter_bitmap is None or del_bitmap.numel() == filter_bitmap.numel()
        bits, ptrs = 0, []
        for b in (del_bitmap, filter_bitmap):
            if b is None:
                ptrs.append(None)
                continue
            assert b.is_cuda and b.dtype == torch.uint8 and b.dim() == 1 and b.is_contiguous()
            bits = max(bits, b.numel() * 8)
            if b.numel() == 0:  # an empty bitmap is still a bitmap: it allows (or deletes) nothing
                b = torch.zeros(1, dtype=torch.uint8, device=b.device)
            ptrs.append(C.c_void_p(b.data_ptr()))
        rc = _lib.lib().gb_index_search_device_filtered(self._h, nq, C.c_void_p(x.data_ptr()), x.stride(0), k, pj,
                                                        int(brute_force), ptrs[0], ptrs[1], bits, C.c_float(min_score),
                                                        C.c_float(max_score), C.c_void_p(out[0].data_ptr()),
                                                        C.c_void_p(out[1].data_ptr()), C.c_void_p(st))
        _check(rc, "search_device")
        return out

    def search_device_keys(self, x, k, params=None, brute_force=False, out_keys=None):
        """Like search_device, returning only the nq x k int64 result keys (score bits << 32 | doc id, best first):
        what a partition contributes to merge_partition_keys_device."""
        import torch
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
        nq = x.shape[0]
        if out_keys is None:
            out_keys = torch.empty((nq, k), dtype=torch.int64, device=x.device)
        pj = json.dumps(params).encode() if params else b""
        st = torch.cuda.current_stream(x.device).cuda_stream
        rc = _lib.lib().gb_index_search_device_keys(self._h, nq, C.c_void_p(x.data_ptr()), x.stride(0), k, pj, int(brute_force),
                                                    C.c_void_p(out_keys.data_ptr()), None, None, C.c_void_p(st))
        _check(rc, "search_device_keys")
        return out_keys

    def stage_times(self):
        """{stage: ms} summed over the searches since the last call (set_scan_timing(True) first)."""
        p, n = C.c_void_p(), C.c_int()
        _check(_lib.lib().gb_index_stage_times(self._h, C.byref(p), C.byref(n)), "stage_times")
        js = C.string_at(p.value, n.value).decode()
        C.CDLL(None).free(C.c_void_p(p.value))
        return json.loads(js)

    def set_rerank_stats(self, on):
        """while on, every search that re-ranks through the two-pass kernel records, per query, the candidates whose
        fp32 rows it read (the search then waits for the count)"""
        _lib.lib().gb_index_set_rerank_stats(self._h, int(on))

    def rerank_survivors(self):
        """int32 array of the per-query survivor counts recorded since the last call (set_rerank_stats(True) first)"""
        p, n = C.c_void_p(), C.c_int64()
        _check(_lib.lib().gb_index_rerank_survivors(self._h, C.byref(p), C.byref(n)), "rerank_survivors")
        out = np.frombuffer(C.string_at(p.value, 4 * n.value), np.int32).copy()
        C.CDLL(None).free(C.c_void_p(p.value))
        return out

    RR_BOUNDED, RR_WITHHELD, RR_UNBOUNDED, RR_DEAD = 0, 1, 2, 3  # debug_rerank's per-candidate states

    def debug_rerank(self, x, cand, k, two_pass=True, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX,
                     max_score=FLT_MAX):
        """The exact re-rank of caller-given candidates (int64 vids [nq, ncand], -1: none, anywhere) over this index's
        HBM rows, by the two-pass kernel or the one-pass kernel.  The bitmaps screen the candidates as the list scans do
        before a re-rank (a deleted or filtered-out vid is no candidate).  Returns a dict: dis, ids [nq, k]; two-pass also
        surv [nq] (candidates whose fp32 rows were read) and per candidate lo, hi [nq, ncand] float32 (its pass-1
        interval as scores, NaN where there is none) and state (RR_BOUNDED; RR_WITHHELD: bounded, but the interval
        crosses the score window, so it does not set the k-th bound; RR_UNBOUNDED; RR_DEAD: no candidate)."""
        x = _f32(x)
        cand = np.ascontiguousarray(cand, np.int64)
        nq, ncand = cand.shape
        assert x.shape == (nq, self.d)
        out = {"dis": np.empty((nq, k), np.float32), "ids": np.empty((nq, k), np.int64)}
        if two_pass:
            out.update(surv=np.empty(nq, np.int32), lo=np.empty((nq, ncand), np.float32),
                       hi=np.empty((nq, ncand), np.float32), state=np.empty((nq, ncand), np.int32))
        db, fb = _bitmap(del_bitmap), _bitmap(filter_bitmap)
        bits = max([b.size * 8 for b in (db, fb) if b is not None], default=0)
        _check(_lib.lib().gb_debug_rerank(self._h, nq, _ptr(x), ncand, _ptr(cand), k, _ptr(db), _ptr(fb), bits,
                                          C.c_float(min_score), C.c_float(max_score), int(two_pass), _ptr(out["dis"]),
                                          _ptr(out["ids"]), _ptr(out.get("surv")), _ptr(out.get("lo")),
                                          _ptr(out.get("hi")), _ptr(out.get("state"))), "debug_rerank")
        return out

    def debug_shadow_rows(self, start, n):
        """The raw store's int8 shadow rows [start, start + n): (qy int8 [n, cols16], s, e, nrm float32 [n])."""
        rb = C.c_int64()
        _check(_lib.lib().gb_debug_shadow_rows(self._h, start, n, None, C.byref(rb)), "debug_shadow_rows")
        raw = np.empty((n, rb.value), np.uint8)
        _check(_lib.lib().gb_debug_shadow_rows(self._h, start, n, _ptr(raw), C.byref(rb)), "debug_shadow_rows")
        cols16 = rb.value - 16
        meta = raw[:, cols16:].copy().view(np.float32)
        return raw[:, :cols16].view(np.int8), meta[:, 0].copy(), meta[:, 1].copy(), meta[:, 2].copy()

    def set_scan_timing(self, on):
        _lib.lib().gb_index_set_scan_timing(self._h, int(on))

    @property
    def last_scan_ms(self):
        return float(_lib.lib().gb_index_last_scan_ms(self._h))

    @property
    def last_scan_kernel(self):
        return _lib.lib().gb_index_last_scan_kernel(self._h).decode()

    @property
    def last_scan_info(self):
        return json.loads(_lib.lib().gb_index_last_scan_info(self._h).decode() or "{}")

    # ---- index-state exchange (parity tests) -------------------------------------------
    def set_centroids(self, c):
        c = _f32(c)
        _check(_lib.lib().gb_index_set_centroids(self._h, _ptr(c), c.shape[0]), "set_centroids")

    def get_centroids(self):
        out = np.empty((self.nlist, self.d), np.float32)
        _check(_lib.lib().gb_index_get_centroids(self._h, _ptr(out)), "get_centroids")
        return out

    @property
    def pq_m(self):
        return int(_lib.lib().gb_index_pq_m(self._h))

    @property
    def pq_ksub(self):
        """Centroids per sub-quantiser: 2^nbits_per_idx (IVFPQ; 256 at the default 8 bits), 16 (IVFPQFastScan)."""
        return int(_lib.lib().gb_index_pq_ksub(self._h))

    def set_pq_centroids(self, pq):
        pq = _f32(pq)
        assert pq.shape == (self.pq_m, self.pq_ksub, self.d // self.pq_m)
        _check(_lib.lib().gb_index_set_pq_centroids(self._h, _ptr(pq)), "set_pq_centroids")

    def get_pq_centroids(self):
        m = self.pq_m
        out = np.empty((m, self.pq_ksub, self.d // m), np.float32)
        _check(_lib.lib().gb_index_get_pq_centroids(self._h, _ptr(out)), "get_pq_centroids")
        return out

    def get_precomputed_table(self):
        """IVFPQ under L2: T[l][m][c] = |pq_m[c]|^2 + 2 <centroid_l|m, pq_m[c]>, shape (nlist, M, pq_ksub)."""
        out = np.empty((self.nlist, self.pq_m, self.pq_ksub), np.float32)
        _check(_lib.lib().gb_index_get_precomputed_table(self._h, _ptr(out)), "get_precomputed_table")
        return out

    @property
    def has_opq(self):
        return bool(_lib.lib().gb_index_has_opq(self._h))

    def set_opq(self, A):
        A = _f32(A)
        assert A.shape == (self.d, self.d)
        _check(_lib.lib().gb_index_set_opq(self._h, _ptr(A)), "set_opq")

    def get_opq(self):
        A = np.empty((self.d, self.d), np.float32)
        _check(_lib.lib().gb_index_get_opq(self._h, _ptr(A)), "get_opq")
        return A

    def apply_opq(self, x):
        x = _f32(x)
        out = np.empty_like(x)
        _check(_lib.lib().gb_index_apply_opq(self._h, x.shape[0], _ptr(x), _ptr(out)), "apply_opq")
        return out

    def list_len(self, l):
        return int(_lib.lib().gb_index_list_len(self._h, l))

    def get_list(self, l):
        n = self.list_len(l)
        codes = np.empty((n, self.code_size), np.uint8)
        ids = np.empty(n, np.int64)
        if n:
            _check(_lib.lib().gb_index_get_list(self._h, l, _ptr(codes), _ptr(ids)), "get_list")
        return codes, ids

    def export_lists(self):
        """CSR view (list_off, codes, ids) of every inverted list, for the oracle."""
        lens = np.array([self.list_len(l) for l in range(self.nlist)], np.int64)
        off = np.zeros(self.nlist + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        codes = np.empty((int(off[-1]), self.code_size), np.uint8)
        ids = np.empty(int(off[-1]), np.int64)
        for l in range(self.nlist):
            if lens[l]:
                c, i = self.get_list(l)
                codes[off[l]:off[l + 1]] = c
                ids[off[l]:off[l + 1]] = i
        return off, codes, ids

    @property
    def mirror_builds(self):
        return int(_lib.lib().gb_index_mirror_builds(self._h))

    @property
    def last_coarse_kernel(self):
        return _lib.lib().gb_index_last_coarse_kernel(self._h).decode()

    def get_list_shifts(self):
        """IVFFLAT under L2: the per-list shifts s_l (nlist x d) the list-major scan subtracts from both operands."""
        out = np.empty((self.nlist, self.d), np.float32)
        _check(_lib.lib().gb_index_get_list_shifts(self._h, _ptr(out)), "get_list_shifts")
        return out

    MIRROR_CURRENT, MIRROR_DISABLED = 1, 2  # debug_mirror's state bits
    ROW_LIVE, ROW_NULL, ROW_STRAY = 0, 1, 2  # debug_rowptr_rows' per-vid states

    def _debug_mirror(self, fn, l):
        nt, tf, st = C.c_int64(), C.c_int64(), C.c_int32()
        _check(fn(self._h, int(l), 0, None, None, C.byref(nt), C.byref(tf), C.byref(st)), "debug_mirror")
        want = (self.list_len(l) + 127) // 128
        tiles, norms = np.zeros((want, tf.value), np.float32), np.zeros((want, 128), np.float32)
        _check(fn(self._h, int(l), want, _ptr(tiles), _ptr(norms), C.byref(nt), C.byref(tf), C.byref(st)), "debug_mirror")
        return {"tiles": tiles[:nt.value], "norms": norms[:nt.value], "current": bool(st.value & self.MIRROR_CURRENT),
                "disabled": bool(st.value & self.MIRROR_DISABLED)}

    def debug_mirror(self, l):
        """IVFFLAT (or a shard of GPU_IVFFLAT): list l's first ceil(len / 128) tiles of the live tensor-core mirror, as a
        dict: tiles [n, 2 * 128 * k16] float32 (hi then lo operand), norms [n, 128], and whether the mirror is current
        and whether it is disabled.  n is 0 when no mirror exists."""
        return self._debug_mirror(_lib.lib().gb_debug_mirror, l)

    def debug_mirror_rebuilt(self, l):
        """The same tiles as a build of the mirror from the current lists writes them (into scratch; the live mirror is
        left as it is)."""
        return self._debug_mirror(_lib.lib().gb_debug_mirror_rebuilt, l)

    def debug_rowptr_rows(self, v0, n):
        """IVFFLAT on a "RocksDB" store (or a shard of GPU_IVFFLAT, local vids): the rows the winner re-score's row
        pointers give vids [v0, v0 + n), and per vid ROW_LIVE (a list entry), ROW_NULL or ROW_STRAY (no list entry; row
        zero).  Returns (rows [n, d] float32, state [n] int32)."""
        rows, state = np.zeros((n, self.d), np.float32), np.zeros(n, np.int32)
        _check(_lib.lib().gb_debug_rowptr_rows(self._h, int(v0), int(n), _ptr(rows), _ptr(state)), "debug_rowptr_rows")
        return rows, state

    def debug_pq_norms(self, l):
        """IVFPQ at 8 bits: list l's cached |r_e|^2 segment and the same segment recomputed from the lists, as
        (live float32 [<= len], recomputed float32 [len], current: whether the cache's key matches)."""
        n, cur = C.c_int64(), C.c_int32()
        _check(_lib.lib().gb_debug_pq_norms(self._h, int(l), None, None, C.byref(n), C.byref(cur)), "debug_pq_norms")
        live, rec = np.zeros(n.value, np.float32), np.zeros(n.value, np.float32)
        _check(_lib.lib().gb_debug_pq_norms(self._h, int(l), _ptr(live), _ptr(rec), C.byref(n), C.byref(cur)),
               "debug_pq_norms")
        return live, rec, bool(cur.value)

    def debug_pq_tables(self):
        """IVFPQ at 8 bits: the tensor-core filter's tables, (int8 codebook [M, 256, dsub], cbnrm float32 [M * 256 + 4]:
        |pq[m][c]|^2, then R^2, sb, D and one unused float)."""
        m = self.pq_m
        cb8 = np.zeros((m, 256, self.d // m), np.int8)
        nrm = np.zeros(m * 256 + 4, np.float32)
        _check(_lib.lib().gb_debug_pq_tables(self._h, _ptr(cb8), _ptr(nrm)), "debug_pq_tables")
        return cb8, nrm

    def compact(self):
        _check(_lib.lib().gb_index_compact(self._h), "compact")

    def dump(self, directory, abs_name):
        """IndexModel::Dump: <directory>/<abs_name>/{ivfflat,ivfpq}.index in gamma's own format; IVFPQFastScan, IVFRABITQ,
        VEARCH and BINARYIVF write this engine's own gb_{ivfpqfs,ivfrabitq,vearch,binaryivf}.index."""
        _check(_lib.lib().gb_index_dump(self._h, str(directory).encode(), abs_name.encode()), "dump")

    def capture_lists(self):
        """The lists as Dump and Backup capture them: (bytes, on_host), the bytes in the index file's order (per list its
        codes at the file's code size, then its ids as stored) and whether they were staged in pinned host memory."""
        n, host = C.c_int64(), C.c_int32()
        _check(_lib.lib().gb_index_capture_lists(self._h, None, 0, C.byref(n), C.byref(host)), "capture_lists")
        out = np.empty(n.value, np.uint8)
        _check(_lib.lib().gb_index_capture_lists(self._h, _ptr(out), n.value, C.byref(n), C.byref(host)), "capture_lists")
        return out, bool(host.value)

    def load(self, directory, abs_name):
        """IndexModel::Load; returns load_num (0: no file).  The vectors must already be in the store.  A refused file raises;
        an index of the four quantised types is then left untrained."""
        n = np.zeros(1, np.int64)
        _check(_lib.lib().gb_index_load(self._h, str(directory).encode(), abs_name.encode(), _ptr(n)), "load")
        return int(n[0])

    def tombstone(self, l, pos):
        _check(_lib.lib().gb_index_tombstone(self._h, l, pos), "tombstone")

    def delete_vectors(self, vids):
        """The documents `vids` were deleted: their list entries are counted dead (a search still needs the deletion
        bitmap to hide them).  A vid that is in no list, or already counted, is ignored."""
        v = np.ascontiguousarray(np.atleast_1d(vids), np.int64)
        _check(_lib.lib().gb_index_delete(self._h, _ptr(v), v.size), "delete_vectors")

    def purge(self, threshold=0.3, del_bitmap=None):
        """RealTimeMemData::CompactIfNeed: rewrite every list whose counted dead share is >= threshold without its
        tombstoned entries and the entries set in del_bitmap; threshold 0 purges every list with a dead entry.
        Returns the number of entries dropped."""
        b = _bitmap(del_bitmap)
        n = np.zeros(1, np.int64)
        _check(_lib.lib().gb_index_purge(self._h, C.c_float(threshold), _ptr(b), 0 if b is None else b.size, _ptr(n)),
               "purge")
        return int(n[0])

    def vid_slots(self, vid):
        """The list entries of vid as [(list, position), ...]: two for an index with SOAR spilling ("soar_lambda" > 0),
        one otherwise, none for a vid in no list.  A fresh build lists the primary entry first."""
        out = np.zeros(2, np.uint64)
        _check(_lib.lib().gb_index_vid_slots(self._h, int(vid), _ptr(out)), "vid_slots")
        return [(int(v) >> 32, int(v) & 0xFFFFFFFF) for v in out if int(v) != 2**64 - 1]

    def memory_charge(self, n_total):
        """What admission under the memory limit charges for storing rows up to n_total: (store growth bytes, rows that
        growth makes room for, index bytes of those rows once indexed)."""
        out = np.zeros(3, np.int64)
        _check(_lib.lib().gb_index_memory_charge(self._h, int(n_total), _ptr(out[0:]), _ptr(out[1:]), _ptr(out[2:])),
               "memory_charge")
        return int(out[0]), int(out[1]), int(out[2])

    def dead_counts(self):
        """Dead entries counted per list (updates' tombstones + delete_vectors) since the list's last purge."""
        out = np.zeros(self.nlist, np.int32)
        _check(_lib.lib().gb_index_dead_counts(self._h, _ptr(out)), "dead_counts")
        return out

    def coarse_search(self, x, nprobe):
        x = _f32(x)
        nq = x.shape[0]
        dis = np.empty((nq, nprobe), np.float32)
        ids = np.empty((nq, nprobe), np.int64)
        _check(_lib.lib().gb_index_coarse_search(self._h, nq, _ptr(x), nprobe, _ptr(dis), _ptr(ids)), "coarse_search")
        return dis, ids

    def search_preassigned(self, x, k, keys, coarse_dis, params=None, del_bitmap=None, filter_bitmap=None,
                           min_score=-FLT_MAX, max_score=FLT_MAX):
        x = _f32(x)
        keys = np.ascontiguousarray(keys, np.int64)
        coarse_dis = _f32(coarse_dis)
        nq, nprobe = keys.shape
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        pj = json.dumps(params).encode() if params else b""
        db, fb = _bitmap(del_bitmap), _bitmap(filter_bitmap)
        bits = 0
        for b in (db, fb):
            if b is not None:
                bits = max(bits, b.size * 8)
        rc = _lib.lib().gb_index_search_preassigned(self._h, nq, _ptr(x), k, _ptr(keys), _ptr(coarse_dis), nprobe, pj,
                                                    _ptr(db), _ptr(fb), bits, C.c_float(min_score),
                                                    C.c_float(max_score), _ptr(dis), _ptr(ids))
        _check(rc, "search_preassigned")
        return dis, ids

    def pq_encode(self, x, assign=None):
        """IVFPQ: codes of the residuals w.r.t. the assigned lists.  IVFPQFastScan: packed 4-bit codes of the raw
        vectors (no assign), ceil(M/2) bytes each, sub-quantiser 2j in the low nibble of byte j."""
        x = _f32(x)
        assign = None if assign is None else np.ascontiguousarray(assign, np.int64)
        codes = np.empty((x.shape[0], self.code_size), np.uint8)
        _check(_lib.lib().gb_index_pq_encode(self._h, x.shape[0], _ptr(x), _ptr(assign), _ptr(codes)), "pq_encode")
        return codes

    def pqfs_lut(self, x, metric=-1):
        """IVFPQFastScan: the uint8 tables [nq, M, 16] of a query batch and (a, b) [nq, 2]; an entry scores
        accu * (1 / a) + b, accu the sum of its M table entries."""
        x = _f32(x)
        nq = x.shape[0]
        lut = np.empty((nq, self.pq_m, 16), np.uint8)
        ab = np.empty((nq, 2), np.float32)
        _check(_lib.lib().gb_index_pqfs_lut(self._h, nq, _ptr(x), metric, _ptr(lut), _ptr(ab)), "pqfs_lut")
        return lut, ab


class BinaryIVFIndex(GammaIndex):
    """BINARYIVF (gamma_index_binary_ivf.cc): d is in bits, a multiple of 8; rows, queries and centroids are uint8 arrays
    of shape [n, d / 8], bit i at bit (i & 7) of byte i >> 3 (numpy.packbits(..., bitorder="little")).  Scores are
    Hamming distances as float32, smaller first."""

    def __init__(self, d, params=None, device=0, store_type=None):
        super().__init__("BINARYIVF", d, params, device, store_type)
        self.code_bytes = self.d // 8

    def _rows(self, x):
        x = np.ascontiguousarray(x, dtype=np.uint8)
        if x.ndim == 1:
            x = x.reshape(1, -1)
        assert x.ndim == 2 and x.shape[1] == self.code_bytes, f"expected uint8 rows of {self.code_bytes} bytes"
        return x

    def add_vectors(self, x):
        x = self._rows(x)
        _check(_lib.lib().gb_index_add_binary(self._h, x.shape[0], _ptr(x)), "add_binary")

    def update_vector(self, vid, x):
        x = self._rows(x)
        _check(_lib.lib().gb_index_update_binary(self._h, vid, _ptr(x)), "update_binary")

    def get_vectors(self, start, n):
        out = np.empty((n, self.code_bytes), np.uint8)
        _check(_lib.lib().gb_index_get_binary(self._h, start, n, _ptr(out)), "get_binary")
        return out

    def get_vector(self, vid):
        return self.get_vectors(vid, 1)[0]

    def search(self, x, k, params=None, brute_force=False, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX,
               max_score=FLT_MAX, search_unindexed_tail=False, cancel=None):
        x = self._rows(x)
        nq = x.shape[0]
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        pj = json.dumps(params).encode() if params else b""
        db, fb = _bitmap(del_bitmap), _bitmap(filter_bitmap)
        bits = max([b.size * 8 for b in (db, fb) if b is not None], default=0)
        rc = _lib.lib().gb_index_search_binary_cancellable(self._h, nq, _ptr(x), k, pj, int(brute_force), _ptr(db),
                                                           _ptr(fb), bits, C.c_float(min_score), C.c_float(max_score),
                                                           int(search_unindexed_tail), _token(cancel), _ptr(dis),
                                                           _ptr(ids))
        _check(rc, "search_binary")
        return dis, ids

    def set_centroids(self, c):
        c = self._rows(c)
        _check(_lib.lib().gb_index_set_binary_centroids(self._h, _ptr(c), c.shape[0]), "set_binary_centroids")

    def get_centroids(self):
        out = np.empty((self.nlist, self.code_bytes), np.uint8)
        _check(_lib.lib().gb_index_get_binary_centroids(self._h, _ptr(out)), "get_binary_centroids")
        return out

    def get_real_centroids(self):
        """The float k-means centroids behind the packed ones (training's +-1 space)."""
        out = np.empty((self.nlist, self.d), np.float32)
        _check(_lib.lib().gb_index_get_real_centroids(self._h, _ptr(out)), "get_real_centroids")
        return out

    def coarse_search(self, x, nprobe):
        x = self._rows(x)
        dis = np.empty((x.shape[0], nprobe), np.float32)
        ids = np.empty((x.shape[0], nprobe), np.int64)
        _check(_lib.lib().gb_index_coarse_search_binary(self._h, x.shape[0], _ptr(x), nprobe, _ptr(dis), _ptr(ids)),
               "coarse_search_binary")
        return dis, ids

    def search_preassigned(self, x, k, keys, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX,
                           max_score=FLT_MAX):
        x = self._rows(x)
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        nq, nprobe = keys.shape
        dis = np.empty((nq, k), np.float32)
        ids = np.empty((nq, k), np.int64)
        db, fb = _bitmap(del_bitmap), _bitmap(filter_bitmap)
        bits = max([b.size * 8 for b in (db, fb) if b is not None], default=0)
        rc = _lib.lib().gb_index_search_preassigned_binary(self._h, nq, _ptr(x), k, _ptr(keys), nprobe, _ptr(db), _ptr(fb),
                                                           bits, C.c_float(min_score), C.c_float(max_score), _ptr(dis),
                                                           _ptr(ids))
        _check(rc, "search_preassigned_binary")
        return dis, ids


class RaBitQIndex(GammaIndex):
    """IVFRABITQ (gamma_index_ivfrabitq.cc): IVF over multi-bit RaBitQ codes of the residuals, nb_bits in [1, 9] per
    dimension, queries quantised to qb in [0, 8] bits per (query, list).  Rows and queries are float32 [n, d] as for
    the other float types; the estimator contract is DESIGN.md section 3, K13 (numpy twin: oracle_rabitq)."""

    def __init__(self, d, params=None, device=0, store_type=None):
        super().__init__("IVFRABITQ", d, params, device, store_type)

    @property
    def nb_bits(self):
        return int(_lib.lib().gb_index_rabitq_nb_bits(self._h))

    @property
    def qb(self):
        return int(_lib.lib().gb_index_rabitq_qb(self._h))

    def encode(self, x, assign):
        """List entries (uint8 [n, code_size]) of rows x whose residuals are taken to the lists `assign`."""
        x = _f32(x)
        assign = np.ascontiguousarray(assign, np.int64)
        assert x.ndim == 2 and x.shape[1] == self.d and assign.shape == (x.shape[0],)
        codes = np.empty((x.shape[0], self.code_size), np.uint8)
        _check(_lib.lib().gb_index_rabitq_encode(self._h, x.shape[0], _ptr(x), _ptr(assign), _ptr(codes)), "rabitq_encode")
        return codes

    def estimate(self, x, lists, qb=None, metric=-1):
        """The scan's scores of every entry of list lists[j] for query x[j]: a list of float32 arrays, one per query,
        in list order."""
        x = _f32(x)
        lists = np.ascontiguousarray(lists, np.int64)
        assert x.ndim == 2 and x.shape[1] == self.d and lists.shape == (x.shape[0],)
        lens = [self.list_len(int(l)) for l in lists]
        out = np.empty(max(1, sum(lens)), np.float32)
        q = self.qb if qb is None else int(qb)
        _check(_lib.lib().gb_index_rabitq_estimate(self._h, x.shape[0], _ptr(x), _ptr(lists), q, metric, _ptr(out)),
               "rabitq_estimate")
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        return [out[off[j]:off[j + 1]].copy() for j in range(len(lens))]


class VearchIndex(GammaIndex):
    """VEARCH (gamma_index_vearch.cc over ScaNN's asymmetric hashing): IVF over 4-bit codes, one per block of
    d / nsubvector dims (plus one block of the d % nsubvector remaining dims).  Under InnerProduct the codes are the
    anisotropic (noise-shaped) codes of the residuals to spherical centroids, under L2 the nearest-centre codes of the raw
    rows.  ncentroids and nsubvector are required parameters.  The contract is DESIGN.md section 3, K14 (numpy twin:
    oracle_scann)."""

    def __init__(self, d, params=None, device=0, store_type=None):
        super().__init__("VEARCH", d, params, device, store_type)

    @property
    def nsub(self):
        return int(_lib.lib().gb_index_vearch_nsub(self._h))

    @property
    def blocks(self):
        return int(_lib.lib().gb_index_vearch_blocks(self._h))

    def set_codebook(self, cb):
        """The 16 d floats of the per-block codebooks (block b's 16 centres, from float 16 b (d // nsub))."""
        cb = _f32(cb).reshape(-1)
        assert cb.size == 16 * self.d
        _check(_lib.lib().gb_index_vearch_set_codebook(self._h, _ptr(cb)), "vearch_set_codebook")

    def get_codebook(self):
        out = np.empty(16 * self.d, np.float32)
        _check(_lib.lib().gb_index_vearch_get_codebook(self._h, _ptr(out)), "vearch_get_codebook")
        return out

    def encode(self, x, assign=None):
        """List codes (uint8 [n, code_size]) of rows x: of their residuals to the lists `assign` under InnerProduct, of
        the rows themselves under L2 (assign ignored)."""
        x = _f32(x)
        assign = None if assign is None else np.ascontiguousarray(assign, np.int64)
        codes = np.empty((x.shape[0], self.code_size), np.uint8)
        _check(_lib.lib().gb_index_vearch_encode(self._h, x.shape[0], _ptr(x), _ptr(assign), _ptr(codes)), "vearch_encode")
        return codes

    def lut(self, x):
        """The biased uint8 tables [nq, blocks, 16] of a query batch and their fixed-point multipliers [nq]."""
        x = _f32(x)
        nq = x.shape[0]
        lut = np.empty((nq, self.blocks, 16), np.uint8)
        mult = np.empty(nq, np.float32)
        _check(_lib.lib().gb_index_vearch_lut(self._h, nq, _ptr(x), _ptr(lut), _ptr(mult)), "vearch_lut")
        return lut, mult


def index_factory(d, description, metric=METRIC_L2, device=0, **extra):
    """index/index.h index_factory: "IVF1024,Flat" | "IVF4096,PQ16x8" | "IVF256,PQ32x4" (PQ<M>x<nbits>) | "Flat"."""
    parts = [p.strip() for p in description.split(",")]
    params = dict(extra)
    params["metric_type"] = "L2" if metric == METRIC_L2 else "InnerProduct"
    if len(parts) == 1 and parts[0].lower() == "flat":
        return GammaIndex("FLAT", d, params, device)
    if len(parts) == 2 and parts[0].upper().startswith("IVF"):
        params["ncentroids"] = int(parts[0][3:])
        params.setdefault("nprobe", min(params.get("nprobe", 80), params["ncentroids"]))
        if parts[1].lower() == "flat":
            return GammaIndex("IVFFLAT", d, params, device)
        if parts[1].upper().startswith("PQ"):
            m, _, nbits = parts[1][2:].partition("x")
            params["nsubvector"] = int(m)
            params["nbits_per_idx"] = int(nbits or 8)
            return GammaIndex("IVFPQ", d, params, device)
    raise GammaError(f"unsupported index description {description!r}")


def kmeans(x, k, niter=25, seed=1234, spherical=False, max_points_per_centroid=256, device=0):
    x = _f32(x)
    n, d = x.shape
    cent = np.empty((k, d), np.float32)
    obj = np.zeros(niter, np.float32)
    _check(_lib.lib().gb_kmeans(device, _ptr(x), n, d, k, niter, seed, int(spherical), max_points_per_centroid,
                                _ptr(cent), _ptr(obj)), "kmeans")
    return cent, obj


def debug_kmeans_trace(x, k, niter=25, seed=1234, spherical=False, l2_assign=False, max_points_per_centroid=256,
                       init=None, device=0):
    """One k-means run (the engine's training k-means), traced step by step: a dict of numpy arrays.  sample [n_s]:
    the rows of x trained on; init [k, d]: the initial centroids (`init` given: a hot start from them); labels and
    scores [niter, n_s]: each row's cluster and the score its key carried; mean, split, norm [niter, k, d]: the
    centroids after the segmented mean, the empty-cluster split and the spherical renormalisation."""
    x = _f32(x)
    n, d = x.shape
    ns = min(n, k * max_points_per_centroid) if max_points_per_centroid > 0 else n
    out = {"sample": np.empty(ns, np.int64), "init": np.empty((k, d), np.float32),
           "labels": np.empty((niter, ns), np.int32), "scores": np.empty((niter, ns), np.float32)}
    for s in ("mean", "split", "norm"):
        out[s] = np.empty((niter, k, d), np.float32)
    init = None if init is None else _f32(init).reshape(k, d)
    _check(_lib.lib().gb_debug_kmeans_trace(device, _ptr(x), n, d, k, niter, seed, int(spherical), int(l2_assign),
                                            max_points_per_centroid, _ptr(init), _ptr(out["sample"]),
                                            _ptr(out["init"]), _ptr(out["labels"]), _ptr(out["scores"]),
                                            _ptr(out["mean"]), _ptr(out["split"]), _ptr(out["norm"])),
           "debug_kmeans_trace")
    return out


OPQ_MAX_TRAIN = 65536  # the rows OPQ trains on at most (faiss OPQMatrix max_train_points)


def opq_kmeans_iters(t):
    """k-means iterations of each subspace in OPQ round t"""
    return 40 if t == 0 else 4


def debug_opq_trace(x, M, niter=3, detail=True, device=0):
    """One OPQ training run (the rotation "opq": {"nsubvector": M} learns), niter rounds, traced: a dict of numpy
    arrays.  sample [n_s]: the rows trained on; mean [d]; r0 [d, d] float64: the random orthonormal start; rf
    [niter, d, d]: the float32 rotation of each round; xty [niter, d, d]: X^T Y as the device formed it; r [niter, d, d]
    float64: the rotation each round solves for; sweeps [niter]: the Jacobi sweeps of each round's SVD; solve_ms
    [niter]: the device time of each round's SVD and R = V U^T (CUDA events).  With detail: centred [n_s, d]; proj, recon [niter, n_s, d]; codes
    [niter, n_s, M]; km [niter][M]: each subspace's k-means trace, as debug_kmeans_trace gives it."""
    x = _f32(x)
    n, d = x.shape
    ns, ds, T = min(n, OPQ_MAX_TRAIN), d // M, niter
    out = {"sample": np.empty(ns, np.int64), "mean": np.empty(d, np.float32), "r0": np.empty((d, d), np.float64),
           "rf": np.empty((T, d, d), np.float32), "xty": np.empty((T, d, d), np.float32),
           "r": np.empty((T, d, d), np.float64), "sweeps": np.empty(T, np.int32), "solve_ms": np.empty(T, np.float32)}
    its = [opq_kmeans_iters(t) for t in range(T)]
    tot = sum(its) * M
    bulk = dict(centred=np.empty((ns, d), np.float32), proj=np.empty((T, ns, d), np.float32),
                codes=np.empty((T, ns, M), np.uint8), recon=np.empty((T, ns, d), np.float32),
                init=np.empty((T * M, 256, ds), np.float32), labels=np.empty((tot, ns), np.int32),
                scores=np.empty((tot, ns), np.float32), kmean=np.empty((tot, 256, ds), np.float32),
                split=np.empty((tot, 256, ds), np.float32), norm=np.empty((tot, 256, ds), np.float32)) if detail else {}
    b = lambda key: _ptr(bulk.get(key))  # noqa: E731
    _check(_lib.lib().gb_debug_opq_trace(device, _ptr(x), n, d, M, niter, int(detail), _ptr(out["sample"]),
                                         _ptr(out["mean"]), b("centred"), _ptr(out["r0"]), _ptr(out["rf"]), b("proj"),
                                         b("codes"), b("recon"), _ptr(out["xty"]), _ptr(out["r"]), b("init"),
                                         b("labels"), b("scores"), b("kmean"), b("split"), b("norm"),
                                         _ptr(out["sweeps"]), _ptr(out["solve_ms"])),
           "debug_opq_trace")
    if detail:
        for key in ("centred", "proj", "codes", "recon"):
            out[key] = bulk[key]
        out["km"], at = [], 0
        for t in range(T):
            row = []
            for m in range(M):
                sl = slice(at, at + its[t])
                row.append({"sample": np.arange(ns, dtype=np.int64), "init": bulk["init"][t * M + m],
                            "labels": bulk["labels"][sl], "scores": bulk["scores"][sl], "mean": bulk["kmean"][sl],
                            "split": bulk["split"][sl], "norm": bulk["norm"][sl]})
                at += its[t]
            out["km"].append(row)
    return out


def kmeans_update(x, k, assign, device=0):
    x = _f32(x)
    assign = np.ascontiguousarray(assign, np.int64)
    cent = np.empty((k, x.shape[1]), np.float32)
    _check(_lib.lib().gb_kmeans_update(device, _ptr(x), x.shape[0], x.shape[1], k, _ptr(assign), _ptr(cent)),
           "kmeans_update")
    return cent


def merge_partitions_device(dis, ids, metric):
    """dis/ids: torch CUDA tensors [nparts, nq, k] -> merged ([nq,k], [nq,k]) on the same device."""
    import torch
    nparts, nq, k = dis.shape
    od = torch.empty((nq, k), dtype=torch.float32, device=dis.device)
    oi = torch.empty((nq, k), dtype=torch.int64, device=dis.device)
    st = torch.cuda.current_stream(dis.device).cuda_stream
    _check(_lib.lib().gb_merge_partitions_device(dis.device.index or 0, C.c_void_p(dis.data_ptr()),
                                                 C.c_void_p(ids.data_ptr()), nparts, nq, k, metric,
                                                 C.c_void_p(od.data_ptr()), C.c_void_p(oi.data_ptr()), C.c_void_p(st)),
           "merge_partitions_device")
    return od, oi


def merge_partition_keys_device(keys, metric):
    """keys: torch CUDA int64 tensor [nparts, nq, k] of partition result keys -> merged ([nq,k] scores, [nq,k] ids with
    ids = partition << 32 | local id) in the router's order (internal/client/client.go:1530-1609)."""
    import torch
    nparts, nq, k = keys.shape
    od = torch.empty((nq, k), dtype=torch.float32, device=keys.device)
    oi = torch.empty((nq, k), dtype=torch.int64, device=keys.device)
    st = torch.cuda.current_stream(keys.device).cuda_stream
    _check(_lib.lib().gb_merge_partition_keys_device(keys.device.index or 0, C.c_void_p(keys.data_ptr()), nparts, nq, k, metric,
                                                     C.c_void_p(od.data_ptr()), C.c_void_p(oi.data_ptr()), C.c_void_p(st)),
           "merge_partition_keys_device")
    return od, oi


def pool_usage(reset_peak=False, device=0):
    """(bytes in use, high-water mark) of the device's default memory pool, where search scratch is allocated, after
    the device's pending work; reset_peak=True then restarts the mark at the current use."""
    used, peak = C.c_int64(), C.c_int64()
    _check(_lib.lib().gb_device_pool_usage(device, int(reset_peak), C.byref(used), C.byref(peak)), "pool_usage")
    return used.value, peak.value


def debug_dist_matrix(x, c, metric, use_tc, device=0):
    """score matrix through the exact CUDA-core kernel (use_tc=0) or the wgmma 3xTF32 kernel (use_tc=1)."""
    x, c = _f32(x), _f32(c)
    out = np.empty((x.shape[0], c.shape[0]), np.float32)
    fn = _lib.lib().gb_debug_dist_matrix
    fn.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    _check(fn(device, _ptr(x), x.shape[0], _ptr(c), c.shape[0], x.shape[1], metric, int(use_tc), _ptr(out)),
           "debug_dist_matrix")
    return out
