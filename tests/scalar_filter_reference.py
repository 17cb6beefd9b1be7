"""Restatement of the engine's scalar filters (table/scalar_index_manager.cc Filter / Search as the engine serves
them), in plain Python over the stored field bytes: the specification the device evaluator is held to.

A table is {field: (data_type, indexed)} plus, per field, one bytes value per docid ("" when a document never had
the field).  A filter is a dict with field, lower, upper, include_lower, include_upper, is_union."""
import struct

import numpy as np

DT_INT, DT_LONG, DT_FLOAT, DT_DOUBLE, DT_STRING, DT_VECTOR, DT_BOOL, DT_DATE, DT_STRINGARRAY = range(9)
FMT = {DT_INT: "<i", DT_LONG: "<q", DT_FLOAT: "<f", DT_DOUBLE: "<d", DT_BOOL: "<B", DT_DATE: "<q"}
STRING_TYPES = (DT_STRING, DT_STRINGARRAY)


def decode(dt, raw):
    """The value the engine compares (int for the integer types, float for FLOAT / DOUBLE), None for a wrong width."""
    if len(raw) != struct.calcsize(FMT[dt]):
        return None
    return struct.unpack(FMT[dt], raw)[0]


def one_filter(dt, values, f):
    """bool[n]: the documents filter f selects on a field of type dt with the given values."""
    n = len(values)
    cur = np.zeros(n, bool)
    neg = f.get("is_union", 0) == 2
    lower, upper = f.get("lower", b""), f.get("upper", b"")
    if dt in STRING_TYPES:
        items = set(lower.split(b"\x01"))
        for d, v in enumerate(values):
            elems = v.split(b"\x01") if dt == DT_STRINGARRAY else [v]
            cur[d] = any(e in items for e in elems)
        return ~cur if neg else cur  # NotIn: every document below n, with or without a value, deleted or not
    lo = decode(dt, lower) if lower else None
    hi = decode(dt, upper) if upper else None
    equal = lower == upper
    for d, raw in enumerate(values):
        v = decode(dt, raw)
        if v is None:  # absent or invalid: never matches, NotEqual included
            continue
        if equal:
            hit = lo is not None and (v != lo if neg else v == lo)
        else:
            hit = True
            if lower:
                hit = lo is not None and (v > lo or (v == lo and f.get("include_lower", False)))
            if hit and upper:
                hit = hi is not None and (v < hi or (v == hi and f.get("include_upper", False)))
        cur[d] = hit
    return cur


def eval_filters(schema, columns, filters, op, n):
    """bool[n] of the documents that pass, or None for "no result" (unknown or unindexed field, every filter skipped,
    nothing selected).  op 0 intersects, 1 unites, anything else keeps the first evaluated filter's set."""
    acc = None
    for f in filters:
        if f["field"] not in schema or not schema[f["field"]][1]:
            return None
        dt = schema[f["field"]][0]
        if not f.get("lower", b"") and (dt in STRING_TYPES or not f.get("upper", b"")):
            continue  # skipped
        vals = list(columns[f["field"]][:n]) + [b""] * (n - len(columns[f["field"]]))
        cur = one_filter(dt, vals, f)
        if acc is None:
            acc = cur
        elif op == 0:
            acc = acc & cur
        elif op == 1:
            acc = acc | cur
    if acc is None or not acc.any():
        return None
    return acc


def query_hits(bitmap, deleted, limit, offset):
    """Query's selection: `offset` filter hits (deleted ones included) are dropped, then the first `limit` live ones."""
    out, skipped = [], 0
    for d in np.flatnonzero(bitmap):
        if len(out) >= limit:
            break
        skipped += 1
        if skipped <= offset:
            continue
        if not deleted[d]:
            out.append(int(d))
    return out
