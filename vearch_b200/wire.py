"""Client-side encoders/decoders for the gamma C-ABI payloads, playing the role of the Go SDK
(internal/engine/sdk/go/gamma/{table,doc}.go build the flatbuffers; internal/ps/engine/gammacb/
reader.go marshals vearchpb.SearchRequest and the router decodes SearchResponse).

Used by tests, bench.py's e2e leg and examples; the engine itself parses these formats in C++
(vearch_b200/csrc/wire.h).  No flatbuffers/protoc dependency: both formats are implemented here
from their specifications.
"""
import struct

# ---- flatbuffers ---------------------------------------------------------------------------
DT_INT, DT_LONG, DT_FLOAT, DT_DOUBLE, DT_STRING, DT_VECTOR, DT_BOOL, DT_DATE, DT_STRINGARRAY = range(9)


class FbBuilder:
    """Back-to-front builder with the official layout rules (offsets counted from the buffer end)."""

    def __init__(self):
        self.buf = bytearray()  # stored reversed-growth: we prepend
        self.minalign = 1
        self.fields = None
        self.object_start = 0

    @property
    def used(self):
        return len(self.buf)

    def _prepend(self, b):
        self.buf[0:0] = b

    def _pad(self, n):
        if n:
            self._prepend(b"\x00" * n)

    def _align(self, a):
        self.minalign = max(self.minalign, a)
        self._pad((-self.used) % a)

    def _prealign(self, ln, a):
        self.minalign = max(self.minalign, a)
        self._pad((-(self.used + ln)) % a)

    def _push(self, fmt, v):
        self._align(struct.calcsize(fmt))
        self._prepend(struct.pack("<" + fmt, v))

    def _refer(self, off):
        self._align(4)
        return self.used - off + 4

    def create_bytes(self, data, is_string=False):
        data = bytes(data)
        self._prealign(len(data) + (1 if is_string else 0), 4)
        if is_string:
            self._prepend(b"\x00")
        self._prepend(data)
        self._push("I", len(data))
        return self.used

    def create_string(self, s):
        return self.create_bytes(s.encode() if isinstance(s, str) else s, True)

    def create_offset_vector(self, offs):
        self._prealign(len(offs) * 4, 4)
        for o in reversed(offs):
            self._push("I", self._refer(o))
        self._push("I", len(offs))
        return self.used

    def start_table(self, nfields):
        self.fields = [0] * nfields
        self.object_start = self.used

    def add_offset(self, fid, off):
        if off:
            self._push("I", self._refer(off))
            self.fields[fid] = self.used

    def add_scalar(self, fid, fmt, v, default=0):
        if v != default:
            self._push(fmt, v)
            self.fields[fid] = self.used

    def end_table(self):
        self._push("i", 0)
        table_start = self.used
        nf = len(self.fields)
        while nf and not self.fields[nf - 1]:
            nf -= 1
        for i in reversed(range(nf)):
            self._push("H", table_start - self.fields[i] if self.fields[i] else 0)
        self._push("H", table_start - self.object_start)
        self._push("H", (nf + 2) * 2)
        so = self.used - table_start
        pos = len(self.buf) - table_start
        self.buf[pos:pos + 4] = struct.pack("<i", so)
        return table_start

    def finish(self, root):
        self._prealign(4, self.minalign)
        self._push("I", self._refer(root))
        return bytes(self.buf)


class FbTable:
    def __init__(self, buf, pos):
        self.buf, self.pos = buf, pos
        so = struct.unpack_from("<i", buf, pos)[0]
        self.vt = pos - so
        self.vtsize = struct.unpack_from("<H", buf, self.vt)[0]

    @staticmethod
    def root(buf):
        return FbTable(buf, struct.unpack_from("<I", buf, 0)[0])

    def _off(self, fid):
        slot = 4 + 2 * fid
        if slot + 2 > self.vtsize:
            return 0
        return struct.unpack_from("<H", self.buf, self.vt + slot)[0]

    def scalar(self, fid, fmt, default=0):
        o = self._off(fid)
        return struct.unpack_from("<" + fmt, self.buf, self.pos + o)[0] if o else default

    def _indirect(self, fid):
        o = self._off(fid)
        if not o:
            return 0
        return self.pos + o + struct.unpack_from("<I", self.buf, self.pos + o)[0]

    def bytes(self, fid):
        t = self._indirect(fid)
        if not t:
            return b""
        n = struct.unpack_from("<I", self.buf, t)[0]
        return bytes(self.buf[t + 4:t + 4 + n])

    def str(self, fid):
        return self.bytes(fid).decode()

    def tables(self, fid):
        t = self._indirect(fid)
        if not t:
            return []
        n = struct.unpack_from("<I", self.buf, t)[0]
        out = []
        for i in range(n):
            e = t + 4 + 4 * i
            out.append(FbTable(self.buf, e + struct.unpack_from("<I", self.buf, e)[0]))
        return out


def build_table(name, fields, vectors, indexes, refresh_interval=1000, enable_id_cache=False, enable_realtime=False,
                index_type="", index_params=""):
    """gamma_api.Table (idl/fbs/table.fbs).  fields: [(name, data_type, is_index)];
    vectors: [(name, dimension, store_type, store_param)]; indexes: [(name, type, field_name, params_json)]."""
    b = FbBuilder()
    idx_offs = []
    for iname, itype, ifield, iparams in indexes:
        p, fn, t, n = b.create_string(iparams), b.create_string(ifield), b.create_string(itype), b.create_string(iname)
        fns = b.create_offset_vector([])
        b.start_table(5)
        b.add_offset(0, n)
        b.add_offset(1, t)
        b.add_offset(2, fn)
        b.add_offset(3, fns)
        b.add_offset(4, p)
        idx_offs.append(b.end_table())
    vec_offs = []
    for vname, dim, store_type, store_param in vectors:
        sp, stt, n = b.create_string(store_param), b.create_string(store_type), b.create_string(vname)
        b.start_table(6)
        b.add_offset(0, n)
        b.add_scalar(1, "b", DT_VECTOR)
        b.add_scalar(2, "B", 1)
        b.add_scalar(3, "i", dim)
        b.add_offset(4, stt)
        b.add_offset(5, sp)
        vec_offs.append(b.end_table())
    fld_offs = []
    for fname, dt, is_index in fields:
        n = b.create_string(fname)
        b.start_table(4)
        b.add_offset(0, n)
        b.add_scalar(1, "b", dt)
        b.add_scalar(2, "B", 1 if is_index else 0)
        fld_offs.append(b.end_table())
    iv, vv, fv = b.create_offset_vector(idx_offs), b.create_offset_vector(vec_offs), b.create_offset_vector(fld_offs)
    ip, it, n = b.create_string(index_params), b.create_string(index_type), b.create_string(name)
    b.start_table(9)
    b.add_offset(0, n)
    b.add_offset(1, fv)
    b.add_offset(2, vv)
    b.add_offset(3, it)
    b.add_offset(4, ip)
    b.add_scalar(5, "i", refresh_interval, default=1000)
    b.add_scalar(6, "B", 1 if enable_id_cache else 0)
    b.add_scalar(7, "B", 1 if enable_realtime else 0)
    b.add_offset(8, iv)
    return b.finish(b.end_table())


def build_doc(fields, value_as_string=True):
    """gamma_api.Doc (idl/fbs/doc.fbs).  fields: [(name, value_bytes, data_type)].
    value_as_string=True reproduces the Go SDK, which writes `value` with CreateString
    (length-prefixed + NUL) although the schema says [ubyte] (sdk/go/gamma/doc.go:28-42)."""
    b = FbBuilder()
    offs = []
    for name, value, dt in fields:
        v = b.create_bytes(value, is_string=value_as_string)
        n = b.create_string(name)
        b.start_table(3)
        b.add_offset(0, n)
        b.add_offset(1, v)
        b.add_scalar(2, "b", dt)
        offs.append(b.end_table())
    fv = b.create_offset_vector(offs)
    b.start_table(1)
    b.add_offset(0, fv)
    return b.finish(b.end_table())


def parse_doc(buf):
    """-> {name: (value_bytes, data_type)}"""
    if not buf:
        return {}
    t = FbTable.root(bytes(buf))
    return {f.str(0): (f.bytes(1), f.scalar(2, "b")) for f in t.tables(0)}


# ---- protobuf (proto3 wire format) ---------------------------------------------------------
def _varint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _key(num, wire):
    return _varint((num << 3) | wire)


def _ld(num, payload):
    return _key(num, 2) + _varint(len(payload)) + payload


def encode_search_request(vec_name, queries, topn, index_params="", is_brute_search=0, fields=("_id",), request_id="",
                          partition_id=None, min_score=None, max_score=None, offset=0, trace=False, req_num=None,
                          range_filters=(), term_filters=(), operator=0, extra_vec_queries=(), ranker="",
                          multi_vector_rank=0):
    """vearchpb.SearchRequest (internal/proto/router_grpc.proto:168-191). queries: float32 ndarray [nq, d].
    range_filters: (field, lower_bytes, upper_bytes, include_lower, include_upper[, is_union]);
    term_filters: (field, value_bytes[, is_union]); operator: 0 And / 1 Or between the filters.
    extra_vec_queries: further (vector field, queries) pairs of a multi-vector search; ranker: WeightedRanker JSON;
    multi_vector_rank=1: order the joined documents by the combined score."""
    import numpy as np
    q = np.ascontiguousarray(queries)  # uint8: packed binary queries of a BINARYIVF field, d / 8 bytes each
    if q.dtype != np.uint8:
        q = np.ascontiguousarray(q, dtype=np.float32)
    out = bytearray()
    params = {}
    if request_id:
        params["request_id"] = request_id
    if partition_id is not None:
        params["partition_id"] = str(partition_id)
    if params:
        head = b"".join(_ld(7, _ld(1, k.encode()) + _ld(2, v.encode())) for k, v in params.items())
        out += _ld(1, head)
    n = q.shape[0] if req_num is None else req_num
    if n:
        out += _key(2, 0) + _varint(n)
    if topn:
        out += _key(3, 0) + _varint(topn)
    if is_brute_search:
        out += _key(4, 0) + _varint(is_brute_search)
    vq = _ld(1, vec_name.encode()) + _ld(2, q.tobytes())
    if min_score is not None and min_score != 0:
        vq += _key(3, 1) + struct.pack("<d", min_score)
    if max_score is not None and max_score != 0:
        vq += _key(4, 1) + struct.pack("<d", max_score)
    out += _ld(5, vq)
    for ename, eq in extra_vec_queries:
        out += _ld(5, _ld(1, ename.encode()) + _ld(2, np.ascontiguousarray(eq, dtype=np.float32).tobytes()))
    for f in fields:
        out += _ld(6, f.encode())
    for rf in range_filters:
        out += _ld(7, _enc_range_filter(rf))
    for tf in term_filters:
        out += _ld(8, _enc_term_filter(tf))
    if index_params:
        out += _ld(9, index_params.encode())
    if multi_vector_rank:
        out += _key(10, 0) + _varint(multi_vector_rank)
    if ranker:
        out += _ld(15, ranker.encode())
    if trace:
        out += _key(16, 0) + _varint(1)
    if operator:
        out += _key(17, 0) + _varint(operator)
    if offset:
        out += _key(20, 0) + _varint(offset)
    return bytes(out)


def _enc_range_filter(rf):
    field, lo, hi, inc_lo, inc_hi = rf[:5]
    m = _ld(1, field.encode())
    if lo:
        m += _ld(2, lo)
    if hi:
        m += _ld(3, hi)
    if inc_lo:
        m += _key(4, 0) + _varint(1)
    if inc_hi:
        m += _key(5, 0) + _varint(1)
    if len(rf) > 5 and rf[5]:
        m += _key(6, 0) + _varint(rf[5])
    return m


def _enc_term_filter(tf):
    m = _ld(1, tf[0].encode()) + (_ld(2, tf[1]) if tf[1] else b"")
    if len(tf) > 2 and tf[2]:
        m += _key(3, 0) + _varint(tf[2])
    return m


def encode_query_request(document_ids=(), partition_id=0, range_filters=(), term_filters=(), fields=(), limit=0,
                         operator=0, offset=0):
    """vearchpb.QueryRequest (internal/proto/router_grpc.proto:147-166): documents by key (by docid when
    partition_id > 0) or by scalar filters."""
    out = bytearray()
    for d in document_ids:
        out += _ld(2, d.encode() if isinstance(d, str) else d)
    if partition_id:
        out += _key(3, 0) + _varint(partition_id)
    for rf in range_filters:
        out += _ld(5, _enc_range_filter(rf))
    for tf in term_filters:
        out += _ld(6, _enc_term_filter(tf))
    for f in fields:
        out += _ld(7, f.encode())
    if limit:
        out += _key(9, 0) + _varint(limit)
    if operator:
        out += _key(15, 0) + _varint(operator)
    if offset:
        out += _key(17, 0) + _varint(offset)
    return bytes(out)


def _parse(buf):
    """-> list of (field number, wire type, value)"""
    i, out = 0, []
    n = len(buf)
    while i < n:
        key = 0
        shift = 0
        while True:
            b = buf[i]
            i += 1
            key |= (b & 0x7F) << shift
            shift += 7
            if not b & 0x80:
                break
        num, wire = key >> 3, key & 7
        if wire == 0:
            v = 0
            shift = 0
            while True:
                b = buf[i]
                i += 1
                v |= (b & 0x7F) << shift
                shift += 7
                if not b & 0x80:
                    break
            out.append((num, wire, v))
        elif wire == 1:
            out.append((num, wire, bytes(buf[i:i + 8])))
            i += 8
        elif wire == 5:
            out.append((num, wire, bytes(buf[i:i + 4])))
            i += 4
        elif wire == 2:
            ln = 0
            shift = 0
            while True:
                b = buf[i]
                i += 1
                ln |= (b & 0x7F) << shift
                shift += 7
                if not b & 0x80:
                    break
            out.append((num, wire, bytes(buf[i:i + ln])))
            i += ln
        else:
            raise ValueError(f"unsupported wire type {wire}")
    return out


def decode_search_response(buf):
    """vearchpb.SearchResponse (router_grpc.proto:195-219) ->
    [{"total": int, "msg": str, "max_score": float, "items": [{"score": float, "fields": {name: bytes}}]}]"""
    results = []
    for num, wire, v in _parse(bytes(buf)):
        if num != 2 or wire != 2:
            continue
        res = {"total": 0, "msg": "", "max_score": 0.0, "items": []}
        for n2, w2, v2 in _parse(v):
            if n2 == 2 and w2 == 1:
                res["max_score"] = struct.unpack("<d", v2)[0]
            elif n2 == 5 and w2 == 2:
                for n3, w3, v3 in _parse(v2):
                    if n3 == 1:
                        res["total"] = v3
            elif n2 == 6 and w2 == 2:
                res["msg"] = v2.decode()
            elif n2 == 7 and w2 == 2:
                item = {"score": 0.0, "fields": {}}
                for n3, w3, v3 in _parse(v2):
                    if n3 == 1 and w3 == 1:
                        item["score"] = struct.unpack("<d", v3)[0]
                    elif n3 == 2 and w3 == 2:
                        name, val = "", b""
                        for n4, w4, v4 in _parse(v3):
                            if n4 == 1:
                                name = v4.decode()
                            elif n4 == 3:
                                val = v4
                        item["fields"][name] = val
                res["items"].append(item)
        results.append(res)
    return results
