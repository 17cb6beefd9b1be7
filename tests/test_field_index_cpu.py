"""The run-time index record at the end of a `.gbdump` snapshot (DESIGN §8, vector indexes at run time), decoded by
the same code Load runs, without a GPU: per changed vector field (name, has index, type, params) as u64-length strings
and an i32, the count first, then the part's u64 length and the magic GBFIDX01.  A snapshot without it decodes to no
record."""
import ctypes as C
import json
import struct

import numpy as np
import pytest

from vearch_b200 import _lib

MAGIC = b"GBFIDX01"


def s(v):
    b = v.encode()
    return struct.pack("<Q", len(b)) + b


def record(recs):
    body = struct.pack("<I", len(recs))
    for field, has, typ, params in recs:
        body += s(field) + struct.pack("<i", 1 if has else 0) + s(typ) + s(params)
    return body + struct.pack("<Q", len(body)) + MAGIC


def decode(tail):
    p, n = C.c_void_p(), C.c_int()
    rc = _lib.lib().gb_debug_index_records(tail, len(tail), C.byref(p), C.byref(n))
    if rc != 0:
        return rc, None
    out = C.string_at(p.value, n.value).decode()
    C.CDLL(None).free(p)
    return rc, json.loads(out)


SNAPSHOT = np.random.default_rng(1).random(4096, dtype=np.float32).tobytes()  # rows and trained state


def test_snapshot_without_record():
    assert decode(SNAPSHOT) == (0, {"bytes": 0, "records": []})
    assert decode(b"") == (0, {"bytes": 0, "records": []})
    assert decode(b"GBFIDX01") == (0, {"bytes": 0, "records": []})  # too short to hold a length


def test_records_round_trip():
    recs = [("emb", True, "IVFPQ", '{"ncentroids": 16, "nsubvector": 8}'), ("img", False, "FLAT", '{"metric_type": "L2"}'),
            ("bin", False, "BINARYIVF", "")]
    rec = record(recs)
    rc, got = decode(SNAPSHOT + rec)
    assert rc == 0 and got["bytes"] == len(rec)
    assert [tuple(r) for r in got["records"]] == recs


@pytest.mark.parametrize("cut", ["length_past_file", "truncated_string", "trailing_bytes", "short_count"])
def test_malformed_records_are_refused(cut):
    rec = record([("emb", True, "IVFFLAT", "{}")])
    body, tail = rec[:-16], rec[-16:]
    if cut == "length_past_file":
        bad = body + struct.pack("<Q", len(body) + 10 ** 6) + MAGIC
    elif cut == "truncated_string":  # the params string claims more bytes than the part holds
        b = body[:-(8 + 2)] + struct.pack("<Q", 50) + b"{}"
        bad = b + struct.pack("<Q", len(b)) + MAGIC
    elif cut == "trailing_bytes":  # bytes after the last record, inside the part
        b = body + b"xx"
        bad = b + struct.pack("<Q", len(b)) + MAGIC
    else:
        bad = b"\x01\x00" + struct.pack("<Q", 2) + MAGIC
    assert decode(bad)[0] == -1
    assert decode(body + tail)[0] == 0
