"""The scalar filter restatement (scalar_filter_reference.py) pinned on hand-written cases: the semantics the device
evaluator must keep."""
import math
import struct

import numpy as np

import scalar_filter_reference as R

i32 = lambda v: struct.pack("<i", v)
f32 = lambda v: struct.pack("<f", v)
f64 = lambda v: struct.pack("<d", v)


def rng(field, lower=b"", upper=b"", il=False, iu=False, is_union=0):
    return {"field": field, "lower": lower, "upper": upper, "include_lower": il, "include_upper": iu, "is_union": is_union}


def term(field, items, is_union=0):
    return {"field": field, "lower": items, "is_union": is_union}


SCHEMA = {"p": (R.DT_INT, True), "f": (R.DT_FLOAT, True), "d": (R.DT_DOUBLE, True), "b": (R.DT_BOOL, True),
          "s": (R.DT_STRING, True), "a": (R.DT_STRINGARRAY, True), "plain": (R.DT_INT, False)}
# doc 0..5; doc 4 has no p / f / s / a (""), doc 5 a wrong-width p
COLS = {
    "p": [i32(1), i32(5), i32(5), i32(-3), b"", b"\x01\x02"],
    "f": [f32(1.5), f32(math.nan), f32(-0.0), f32(0.0), b"", f32(2.0)],
    "d": [f64(1.0)] * 6,
    "b": [b"\x00", b"\x01", b"\x01", b"\x00", b"", b"\x02"],
    "s": [b"x", b"y", b"", b"x", b"", b"z"],
    "a": [b"u\x01v", b"v\x01v", b"", b"w", b"", b"\x01u"],
    "plain": [i32(i) for i in range(6)],
}
N = 6


def ev(filters, op=0, n=N):
    r = R.eval_filters(SCHEMA, COLS, filters, op, n)
    return None if r is None else np.flatnonzero(r).tolist()


def test_numeric_forms():
    assert ev([rng("p", i32(5), i32(5))]) == [1, 2]  # Equal
    assert ev([rng("p", i32(5), i32(5), is_union=2)]) == [0, 3]  # NotEqual: absent / invalid never match
    assert ev([rng("p", i32(1), i32(5), True, False)]) == [0]
    assert ev([rng("p", i32(1), i32(5), False, True)]) == [1, 2]
    assert ev([rng("p", i32(-3))]) == [0, 1, 2]  # one bound: >
    assert ev([rng("p", upper=i32(1), iu=True)]) == [0, 3]  # <=
    assert ev([rng("p", i32(1), i32(6), True, True, is_union=2)]) == [0, 1, 2]  # is_union means nothing to a range
    assert ev([rng("b", b"\x01", b"\x01")]) == [1, 2]
    assert ev([rng("b", b"\x01")]) == [5]  # BOOL compares the byte


def test_wrong_width_bound_matches_nothing():
    assert ev([rng("p", b"\x05\x00")]) is None
    assert ev([rng("p", b"\x05\x00", b"\x05\x00", is_union=2)]) is None
    assert ev([rng("p", i32(0), b"\x05")]) is None  # a bad upper bound spoils a good lower one


def test_nan_and_signed_zero():
    nan = f32(math.nan)
    assert ev([rng("f", nan, nan)]) is None  # NaN equals nothing, itself included
    assert ev([rng("f", nan, nan, is_union=2)]) == [0, 1, 2, 3, 5]  # ... and differs from every valid value
    assert ev([rng("f", f32(-1.0), nan, True, True)]) is None
    assert ev([rng("f", f32(0.0), f32(0.0))]) == [2, 3]  # -0 == +0
    assert ev([rng("f", f32(0.0), f32(3.0), False, True)]) == [0, 5]
    assert ev([rng("d", f64(math.nan))]) is None


def test_strings_items_and_empty_terms():
    assert ev([term("s", b"x\x01z")]) == [0, 3, 5]
    assert ev([term("s", b"\x01q")]) == [2, 4]  # the empty item is a real term: documents without the field match
    assert ev([term("s", b"nope")]) is None
    assert ev([term("s", b"x", is_union=2)]) == [1, 2, 4, 5]
    assert ev([term("a", b"u")]) == [0, 5]
    assert ev([term("a", b"v")]) == [0, 1]  # a duplicated element matches once
    assert ev([term("a", b"\x01zz")]) == [2, 4, 5]  # empty elements, and "" of the documents without the field
    assert ev([term("a", b"v\x01w", is_union=2)]) == [2, 4, 5]


def test_not_in_covers_every_document_below_n():
    deleted = np.array([False, True, False, False, False, False])
    hits = R.eval_filters(SCHEMA, COLS, [term("s", b"zz", is_union=2)], 0, N)
    assert hits.tolist() == [True] * N  # deleted documents included: the scan, not the filter, drops them
    assert R.query_hits(hits, deleted, limit=3, offset=1) == [2, 3, 4]  # the offset counts the deleted hit too
    assert R.query_hits(hits, deleted, limit=10, offset=2) == [2, 3, 4, 5]


def test_skipping_combining_and_no_result():
    assert ev([rng("p")]) is None  # every filter skipped: no result
    assert ev([term("s", b""), rng("p")]) is None
    assert ev([rng("p"), rng("p", i32(4))]) == [1, 2]  # skipped filters do not take part
    assert ev([rng("p", i32(4)), term("s", b"y")]) == [1]
    assert ev([rng("p", i32(4)), term("s", b"y")], op=1) == [1, 2]
    assert ev([rng("p", i32(4)), term("s", b"y")], op=7) == [1, 2]  # another operator keeps the first set
    assert ev([rng("p", i32(4)), rng("plain", i32(0))]) is None  # unindexed field: no result, whatever came before
    assert ev([rng("nofield", i32(0)), rng("p", i32(4))]) is None
    assert ev([rng("p", i32(100))]) is None  # cardinality 0


def test_documents_past_the_columns_have_no_value():
    assert ev([rng("p", i32(-10))], n=8) == [0, 1, 2, 3]
    assert ev([term("s", b"x", is_union=2)], n=8) == [1, 2, 4, 5, 6, 7]
