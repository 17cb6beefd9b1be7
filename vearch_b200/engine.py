"""ctypes binding of the gamma C-ABI (include/gamma_api.h) exported by libgamma.so -- the same
23 entry points the Go partition server reaches through cgo (internal/engine/sdk/go/gamma/gamma.go).
The method names and argument meaning follow that Go wrapper (Init / CreateTable / AddOrUpdateDoc /
DeleteDoc / Search / BuildIndex / GetEngineStatus ...), so tests read like the reference's
internal/engine/tests/test.h flow: Init -> CreateTable -> Add docs -> wait index_status == 2 ->
Search -> Dump -> Load.
"""
import ctypes as C
import json
import time

import numpy as np

from . import _lib, wire

libc = C.CDLL(None)
libc.free.argtypes = [C.c_void_p]


class CStatus(C.Structure):
    _fields_ = [("code", C.c_int), ("msg", C.c_void_p)]


class GammaStatusError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"code={code}: {msg}")
        self.code, self.msg = code, msg


_declared = False


def _api():
    global _declared
    l = _lib.lib()
    if not _declared:
        vp, i32, cp = C.c_void_p, C.c_int, C.c_char_p
        pp, pi = C.POINTER(C.c_void_p), C.POINTER(C.c_int)
        l.Init.restype = vp
        l.Init.argtypes = [cp, i32]
        l.Close.argtypes = [vp]
        l.CreateTable.restype = CStatus
        l.CreateTable.argtypes = [vp, cp, i32]
        l.AddOrUpdateDoc.argtypes = [vp, cp, i32]
        l.DeleteDoc.argtypes = [vp, cp, i32]
        l.GetEngineStatus.restype = None
        l.GetEngineStatus.argtypes = [vp, pp, pi]
        l.GetMemoryInfo.restype = None
        l.GetMemoryInfo.argtypes = [vp, pp, pi]
        l.GetDocByID.argtypes = [vp, cp, i32, pp, pi]
        l.GetDocByDocID.argtypes = [vp, i32, C.c_char, pp, pi]
        l.BuildIndex.argtypes = [vp]
        l.RebuildIndex.argtypes = [vp, i32, i32, i32]
        l.Dump.argtypes = [vp]
        l.Load.argtypes = [vp]
        l.Search.restype = CStatus
        l.Search.argtypes = [vp, cp, i32, pp, pi]
        l.Query.restype = CStatus
        l.Query.argtypes = [vp, cp, i32, pp, pi]
        l.SetConfig.argtypes = [vp, cp, i32]
        l.GetConfig.argtypes = [vp, pp, pi]
        l.Backup.restype = CStatus
        l.Backup.argtypes = [vp, i32]
        l.AddFieldIndexWithParams.restype = CStatus
        l.AddFieldIndexWithParams.argtypes = [vp, cp, i32, cp, i32, cp, i32]
        l.RemoveFieldIndex.restype = CStatus
        l.RemoveFieldIndex.argtypes = [vp, cp, i32]
        l.SetMemoryLimitConfig.restype = None
        l.SetMemoryLimitConfig.argtypes = [i32]
        l.SetKillStatus.restype = None
        l.SetKillStatus.argtypes = [cp, i32, i32]
        l.DeleteKillStatus.restype = None
        l.DeleteKillStatus.argtypes = [cp, i32]
        _declared = True
    return l


def _take(ptr, ln):
    """copy a malloc'd output buffer and free it, like C.GoBytes + C.free (gamma.go:78-81)."""
    if not ptr.value:
        return b""
    data = C.string_at(ptr.value, ln.value)
    libc.free(ptr.value)
    return data


def _status(st):
    if st.code != 0:
        msg = C.string_at(st.msg).decode("utf-8", "replace") if st.msg else ""
        if st.msg:
            libc.free(st.msg)
        raise GammaStatusError(st.code, msg)


def set_memory_limit(percent):
    """SetMemoryLimitConfig: limit this process to `percent` % of each device's HBM and of host memory (0: no limit)."""
    _api().SetMemoryLimitConfig(int(percent))


def memory_ledger(device):
    """(usage, pool_reserved, limit) in bytes on a device, or the host for device -1 (limit 0: none)."""
    u, p, lim = C.c_int64(), C.c_int64(), C.c_int64()
    _api().gb_memory_ledger(device, C.byref(u), C.byref(p), C.byref(lim))
    return u.value, p.value, lim.value


def backup_hold(op):
    """test hook: 1 makes the next backup wait between its capture and its write, 0 lets it go on, -1 only reads.
    Returns 0 (off), 1 (set) or 2 (a backup is waiting)."""
    return _api().gb_debug_backup_hold(int(op))


def backup_stage():
    """(bytes in HBM, bytes in pinned host memory) the last finished capture of a dump or backup staged."""
    d, h = C.c_int64(), C.c_int64()
    _api().gb_debug_backup_stage(C.byref(d), C.byref(h))
    return d.value, h.value


def set_memory_total(device, nbytes):
    """test hook: the total memory the limit's percentage applies to on a device (-1: host); 0 restores the real one."""
    _api().gb_memory_set_total(device, int(nbytes))


class GammaEngine:
    def __init__(self, path, space_name="default", log_dir="/tmp/gamma_b200_logs", device=0, devices=None):
        """devices: CUDA ordinals or "all" (Init's "devices"): GPU_IVFPQ / GPU_IVFFLAT fields are sharded over them and
        devices[0] replaces `device`."""
        conf = {"path": path, "space_name": space_name, "log_dir": log_dir, "device": device}
        if devices is not None:
            conf["devices"] = devices if isinstance(devices, str) else [int(v) for v in devices]
        cfg = json.dumps(conf).encode()
        self._h = _api().Init(cfg, len(cfg))
        if not self._h:
            raise RuntimeError("gamma Init failed (no CUDA device or bad config)")
        self.vec_name = None
        self.dim = 0

    def close(self):
        if getattr(self, "_h", None):
            _api().Close(self._h)
            self._h = None

    def create_table(self, name, dim, index_type, index_params, vec_name="emb", fields=(("_id", wire.DT_STRING, False),),
                     refresh_interval=100, extra_vectors=(), store_type="MemoryOnly", **kw):
        """extra_vectors: further vector fields [(name, dim, index_type, index_params[, store_type])] of a multi-vector
        table.  store_type "RocksDB" keeps a field's raw vectors in pinned host memory instead of HBM."""
        self.vec_name, self.dim = vec_name, dim
        vectors = [(vec_name, dim, store_type, "")] + \
                  [(e[0], e[1], e[4] if len(e) > 4 else "MemoryOnly", "") for e in extra_vectors]
        indexes = [("idx", index_type, vec_name, json.dumps(index_params))] + \
                  [(f"idx_{e[0]}", e[2], e[0], json.dumps(e[3])) for e in extra_vectors]
        tb = wire.build_table(name, list(fields), vectors, indexes, refresh_interval=refresh_interval, **kw)
        _status(_api().CreateTable(self._h, tb, len(tb)))

    def create_table_raw(self, table_bytes, vec_name, dim):
        """CreateTable with caller-supplied gamma_api.Table flatbuffer bytes (fixtures written by the reference's builders)"""
        self.vec_name, self.dim = vec_name, dim
        _status(_api().CreateTable(self._h, table_bytes, len(table_bytes)))

    def add_doc(self, key, vector, extra_fields=()):
        """vector: float32 values, or for a BINARYIVF table a uint8 array of dimension / 8 packed bytes"""
        vector = np.asarray(vector)
        v = (vector if vector.dtype == np.uint8 else vector.astype(np.float32)).tobytes()
        fields = [("_id", key.encode() if isinstance(key, str) else key, wire.DT_STRING)]
        fields += list(extra_fields)
        fields.append((self.vec_name, v, wire.DT_VECTOR))
        doc = wire.build_doc(fields)
        return _api().AddOrUpdateDoc(self._h, doc, len(doc))

    def add_doc_raw(self, doc_bytes):
        return _api().AddOrUpdateDoc(self._h, doc_bytes, len(doc_bytes))

    def delete_doc(self, key):
        k = key.encode() if isinstance(key, str) else key
        return _api().DeleteDoc(self._h, k, len(k))

    def get_doc_by_id(self, key):
        k = key.encode() if isinstance(key, str) else key
        p, n = C.c_void_p(), C.c_int()
        rc = _api().GetDocByID(self._h, k, len(k), C.byref(p), C.byref(n))
        return rc, wire.parse_doc(_take(p, n))

    def get_doc_by_docid(self, docid, next_=False):
        p, n = C.c_void_p(), C.c_int()
        rc = _api().GetDocByDocID(self._h, docid, C.c_char(1 if next_ else 0), C.byref(p), C.byref(n))
        return rc, wire.parse_doc(_take(p, n))

    def build_index(self):
        return _api().BuildIndex(self._h)

    def status(self):
        p, n = C.c_void_p(), C.c_int()
        _api().GetEngineStatus(self._h, C.byref(p), C.byref(n))
        return json.loads(_take(p, n))

    def memory_info(self):
        p, n = C.c_void_p(), C.c_int()
        _api().GetMemoryInfo(self._h, C.byref(p), C.byref(n))
        return json.loads(_take(p, n))

    def wait_indexed(self, min_indexed, timeout=120.0):
        """poll like tests/test.h:862-879 / test/utils/vearch_utils.py:1386"""
        t0 = time.time()
        while time.time() - t0 < timeout:
            st = self.status()
            if st["index_status"] == 2 and st["min_indexed_num"] >= min_indexed:
                return st
            time.sleep(0.02)
        raise TimeoutError(f"index not ready: {self.status()}")

    def search_raw(self, request_bytes):
        p, n = C.c_void_p(), C.c_int()
        st = _api().Search(self._h, request_bytes, len(request_bytes), C.byref(p), C.byref(n))
        _status(st)
        return _take(p, n)

    def search(self, queries, topn, index_params=None, **kw):
        req = wire.encode_search_request(self.vec_name, queries, topn,
                                         index_params=json.dumps(index_params) if index_params else "", **kw)
        return wire.decode_search_response(self.search_raw(req))

    def rebuild_index(self, drop_before_rebuild=1, limit_cpu=0, describe=0):
        return _api().RebuildIndex(self._h, drop_before_rebuild, limit_cpu, describe)

    def add_field_index(self, field, index_type="", index_params=None):
        """AddFieldIndexWithParams.  A scalar field becomes filterable (type and params are ignored); a vector field gets
        an index of `index_type` with `index_params` (a dict), built in the background while its current index keeps
        serving, which replaces it once every stored row is indexed."""
        f, t = field.encode(), index_type.encode()
        p = json.dumps(index_params).encode() if index_params is not None else b""
        _status(_api().AddFieldIndexWithParams(self._h, f, len(f), t, len(t), p, len(p)))

    def remove_field_index(self, field):
        """RemoveFieldIndex: a scalar field is no longer filterable; a vector field drops its index and is then searched
        exactly (the brute-force path)."""
        f = field.encode()
        _status(_api().RemoveFieldIndex(self._h, f, len(f)))

    def dump(self):
        return _api().Dump(self._h)

    def load(self):
        return _api().Load(self._h)

    def backup(self, command=0):
        """Backup: 0 ("create") captures the partition as Dump does and writes it to <path>/backup/retrieval_model_index,
        replacing the previous backup only once complete; 1 ("restore") does nothing.  Raises GammaStatusError."""
        _status(_api().Backup(self._h, int(command)))

    def set_config(self, cfg):
        b = json.dumps(cfg).encode()
        return _api().SetConfig(self._h, b, len(b))

    def get_config(self):
        p, n = C.c_void_p(), C.c_int()
        _api().GetConfig(self._h, C.byref(p), C.byref(n))
        return json.loads(_take(p, n))

    def query(self, **kw):
        """Query (search/engine.cc:404-523): documents by key / docid or by scalar filters; one result."""
        req = wire.encode_query_request(**kw)
        p, n = C.c_void_p(), C.c_int()
        _status(_api().Query(self._h, req, len(req), C.byref(p), C.byref(n)))
        return wire.decode_search_response(_take(p, n))[0]
