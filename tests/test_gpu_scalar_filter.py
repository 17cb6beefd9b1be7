"""Scalar filters evaluated on the device columns, held to the restatement (scalar_filter_reference.py): every scalar
type, absent values and NaNs, more documents than one flush batch and one column allocation, updates (string-array
pool re-pack included), deletes, AddFieldIndex / RemoveFieldIndex and Dump / Load.  Brute-force and exact IVF searches
are key-exact against the CPU oracle searched with the restated bitmap; Query returns the restatement's hits."""
import struct

import numpy as np
import pytest

import scalar_filter_reference as R
from oracle import oracle as orc
from vearch_b200 import synth, wire

pytestmark = pytest.mark.gpu
L2 = orc.METRIC_L2
D, N, NQ, K = 16, 9000, 8, 10
FIELDS = [("fi", R.DT_INT), ("fl", R.DT_LONG), ("ff", R.DT_FLOAT), ("fd", R.DT_DOUBLE), ("fb", R.DT_BOOL),
          ("ft", R.DT_DATE), ("fs", R.DT_STRING), ("fa", R.DT_STRINGARRAY)]
NUM_FMT = {R.DT_INT: "<i", R.DT_LONG: "<q", R.DT_FLOAT: "<f", R.DT_DOUBLE: "<d", R.DT_BOOL: "<B", R.DT_DATE: "<q"}


def eng_mod():
    from vearch_b200 import engine
    return engine


def num_bytes(dt, v):
    return struct.pack(NUM_FMT[dt], v)


def rand_num(rng, dt):
    if dt == R.DT_BOOL:
        return int(rng.integers(0, 3))
    v = int(rng.integers(-40, 40))
    if dt in (R.DT_FLOAT, R.DT_DOUBLE):
        return float("nan") if rng.random() < 0.05 else v / 2
    return v


def rand_value(rng, dt):
    """bytes, or None: the document does not carry the field"""
    u = rng.random()
    if u < 0.08:
        return None
    if dt == R.DT_STRING:
        return b"" if u < 0.12 else f"s{rng.integers(0, 24)}".encode()
    if dt == R.DT_STRINGARRAY:
        return b"\x01".join(f"a{x}".encode() for x in rng.integers(0, 30, size=int(rng.integers(0, 4))))
    if u < 0.1:
        return b"\x01\x02\x03"  # wrong width: no valid value
    return num_bytes(dt, rand_num(rng, dt))


def rand_filter(rng, schema):
    names = list(schema)
    f = names[int(rng.integers(len(names)))]
    dt = schema[f][0]
    neg = 2 if rng.random() < 0.3 else 0
    if dt in R.STRING_TYPES:
        pre = "s" if dt == R.DT_STRING else "a"
        items = [f"{pre}{x}".encode() for x in rng.integers(0, 32, size=int(rng.integers(1, 4)))]
        if rng.random() < 0.15:
            items.append(b"")
        if rng.random() < 0.05:
            items = [b""]  # one empty item
        lower = b"\x01".join(items)
        if rng.random() < 0.05:
            lower = b""  # skipped
        return ("term", f, lower, neg)
    form = rng.integers(0, 6)
    a, b = sorted(rand_num(rng, dt) for _ in range(2))
    lo, hi = num_bytes(dt, a), num_bytes(dt, b)
    if form == 0:
        return ("range", f, lo, lo, True, True, neg)  # Equal / NotEqual
    if form == 1:
        return ("range", f, lo, b"", bool(rng.integers(2)), False, neg)
    if form == 2:
        return ("range", f, b"", hi, False, bool(rng.integers(2)), neg)
    if form == 3:
        return ("range", f, lo, hi, bool(rng.integers(2)), bool(rng.integers(2)), neg)
    if form == 4:
        return ("range", f, lo[:-1] if len(lo) > 1 else lo + b"\x00", hi, True, True, 0)  # wrong width
    if dt in (R.DT_FLOAT, R.DT_DOUBLE):
        nan = num_bytes(dt, float("nan"))
        return ("range", f, nan, nan, True, True, neg)
    return ("term", f, lo, neg)  # a term filter on a numeric field: lower bound only


def as_request(filters):
    rf = [(f[1], f[2], f[3], f[4], f[5], f[6]) for f in filters if f[0] == "range"]
    tf = [(f[1], f[2], f[3]) for f in filters if f[0] == "term"]
    # the engine sees the range filters first, then the term filters
    spec = [{"field": f[0], "lower": f[1], "upper": f[2], "include_lower": f[3], "include_upper": f[4],
             "is_union": f[5]} for f in rf]
    spec += [{"field": f[0], "lower": f[1], "is_union": f[2]} for f in tf]
    return rf, tf, spec


class Model:
    """the table as the restatement sees it"""

    def __init__(self, schema):
        self.schema = dict(schema)
        self.cols = {f: [] for f in schema}
        self.deleted = []

    def set(self, d, f, v):
        col = self.cols[f]
        while len(col) <= d:
            col.append(b"")
        if v is not None:
            col[d] = v


def make_table(e, n_extra=()):
    fields = [("_id", wire.DT_STRING, False)] + [(f, dt, True) for f, dt in FIELDS] + [("plain", wire.DT_INT, False)]
    e.create_table("ts", D, "IVFFLAT", {"ncentroids": 16, "nprobe": 16, "metric_type": "L2", "training_threshold": 2000},
                   fields=tuple(fields), extra_vectors=n_extra)


def doc_fields(rng, m, d, plain=True):
    out = []
    for f, dt in FIELDS:
        v = rand_value(rng, dt)
        m.set(d, f, v)
        if v is not None:
            out.append((f, v, dt))
    if plain:
        v = struct.pack("<i", d % 97)
        m.set(d, "plain", v)
        out.append(("plain", v, wire.DT_INT))
    return out


def keys_of(res):
    return [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]


def check_requests(e, m, db, xq, rng, n_req, brute_only=False):
    n = len(db)
    alive = ~np.asarray(m.deleted[:n], bool)
    for _ in range(n_req):
        filters = [rand_filter(rng, m.schema) for _ in range(int(rng.integers(1, 4)))]
        op = int(rng.choice([0, 0, 1, 1, 2]))
        rf, tf, spec = as_request(filters)
        want = R.eval_filters(m.schema, m.cols, spec, op, n)
        for brute in ((1,) if brute_only else (1, 0)):
            res = e.search(xq, K, index_params={"nprobe": 16}, is_brute_search=brute, range_filters=rf, term_filters=tf,
                           operator=op)
            assert len(res) == NQ
            if want is None:
                assert all(r["items"] == [] and "no result" in r["msg"] for r in res), (spec, op)
                continue
            do, io = orc.flat_search(db, xq, K, L2, filter_bitmap=np.packbits(want & alive, bitorder="little"))
            assert keys_of(res) == [[f"doc{i}" for i in row if i >= 0] for row in io], (spec, op, brute)
            assert [[it["score"] for it in r["items"]] for r in res] == \
                [[float(s) for s, i in zip(dr, ir) if i >= 0] for dr, ir in zip(do, io)], (spec, op, brute)
        limit, offset = int(rng.integers(1, 40)), int(rng.integers(0, 30))
        r = e.query(range_filters=rf, term_filters=tf, operator=op, limit=limit, offset=offset, fields=["_id"])
        if want is None:
            assert r["items"] == [] and "no result" in r["msg"]
        else:
            got = [int(it["fields"]["_id"][3:]) for it in r["items"]]
            assert got == R.query_hits(want, np.asarray(m.deleted[:n], bool), limit, offset), (spec, op)


def test_filters_over_every_scalar_type_and_mutation(tmp_path):
    rng = np.random.default_rng(2024)
    db = synth.sift_like(N, D, seed=91)
    xq = synth.sift_like(NQ, D, seed=92)
    E = eng_mod()
    e = E.GammaEngine(str(tmp_path), space_name="ts")
    make_table(e)
    m = Model({f: (dt, True) for f, dt in FIELDS} | {"plain": (R.DT_INT, False)})
    assert e.memory_info()["field_range_mem"] == 0
    for d in range(N):  # > 8192: one staged batch flushes from ingest, the columns grow past their first allocation
        assert e.add_doc(f"doc{d}", db[d], extra_fields=doc_fields(rng, m, d)) == 0
        m.deleted.append(False)
    e.wait_indexed(N)
    check_requests(e, m, db, xq, rng, 25)
    assert e.memory_info()["field_range_mem"] > 0
    # updates: scalar values change (a field an update leaves out keeps its value); string arrays are rewritten until
    # most of the pool is dead, which re-packs it
    for rnd in range(3):
        for d in range(N) if rnd < 2 else rng.choice(N, 700, replace=False):
            d = int(d)
            if rnd < 2:
                v = rand_value(rng, R.DT_STRINGARRAY) or b"a1\x01a1"
                m.set(d, "fa", v)
                fl = [("fa", v, wire.DT_STRINGARRAY)]
            else:
                fl = doc_fields(rng, m, d, plain=False)
            assert e.add_doc_raw(wire.build_doc([("_id", f"doc{d}".encode(), wire.DT_STRING)] + fl)) == 0
    for d in rng.choice(N, 400, replace=False):
        assert e.delete_doc(f"doc{int(d)}") == 0
        m.deleted[int(d)] = True
    check_requests(e, m, db, xq, rng, 25)
    # AddFieldIndex / RemoveFieldIndex
    e.add_field_index("plain")
    m.schema["plain"] = (R.DT_INT, True)
    e.remove_field_index("fi")
    m.schema["fi"] = (R.DT_INT, False)
    check_requests(e, m, db, xq, rng, 15, brute_only=True)
    e.add_field_index("fi")
    m.schema["fi"] = (R.DT_INT, True)
    # Dump / Load: the columns are built again from the stored values
    assert e.dump() == 0
    e.close()
    e2 = E.GammaEngine(str(tmp_path), space_name="ts")
    make_table(e2)
    assert e2.load() == 0
    e2.wait_indexed(N)
    m.schema["plain"] = (R.DT_INT, False)  # AddFieldIndex is not part of the schema a Load starts from
    check_requests(e2, m, db, xq, rng, 20)
    e2.close()


def test_ivfpq_filtered_search_is_exact_when_every_candidate_is_reranked(tmp_path):
    rng = np.random.default_rng(5)
    n = 3000
    db = synth.sift_like(n, D, seed=93)
    xq = synth.sift_like(NQ, D, seed=94)
    e = eng_mod().GammaEngine(str(tmp_path), space_name="ts")
    e.create_table("ts", D, "IVFPQ", {"ncentroids": 16, "nprobe": 16, "nsubvector": 4, "metric_type": "L2",
                                      "training_threshold": 1000},
                   fields=(("_id", wire.DT_STRING, False), ("fi", wire.DT_INT, True), ("fs", wire.DT_STRING, True)))
    vi = rng.integers(0, 50, n)
    vs = rng.integers(0, 40, n)
    for d in range(n):
        assert e.add_doc(f"doc{d}", db[d], extra_fields=[("fi", struct.pack("<i", int(vi[d])), wire.DT_INT),
                                                         ("fs", f"s{vs[d]}".encode(), wire.DT_STRING)]) == 0
    e.wait_indexed(n)
    for lo, terms in ((7, b"s3"), (20, b"s1\x01s2\x01s39"), (0, b"s5")):
        mask = (vi == lo) | np.isin(vs, [int(t[1:]) for t in terms.split(b"\x01")])
        res = e.search(xq, K, index_params={"nprobe": 16, "recall_num": 400}, operator=1,
                       range_filters=[("fi", struct.pack("<i", lo), struct.pack("<i", lo), True, True)],
                       term_filters=[("fs", terms)])
        assert mask.sum() <= 400
        _, io = orc.flat_search(db, xq, K, L2, filter_bitmap=np.packbits(mask, bitorder="little"))
        assert keys_of(res) == [[f"doc{i}" for i in row if i >= 0] for row in io]
    e.close()


def test_multi_vector_filtered_search(tmp_path):
    rng = np.random.default_rng(6)
    n, d2, topn = 2500, 8, 40
    db = synth.sift_like(n, D, seed=95)
    db2 = synth.sift_like(n, d2, seed=96)
    xq = synth.sift_like(NQ, D, seed=97)
    xq2 = synth.sift_like(NQ, d2, seed=98)
    e = eng_mod().GammaEngine(str(tmp_path), space_name="ts")
    e.create_table("ts", D, "FLAT", {"metric_type": "L2"},
                   fields=(("_id", wire.DT_STRING, False), ("fi", wire.DT_INT, True)),
                   extra_vectors=[("emb2", d2, "FLAT", {"metric_type": "L2"})])
    vi = rng.integers(0, 10, n)
    for d in range(n):
        doc = wire.build_doc([("_id", f"doc{d}".encode(), wire.DT_STRING), ("fi", struct.pack("<i", int(vi[d])), wire.DT_INT),
                              ("emb", db[d].tobytes(), wire.DT_VECTOR), ("emb2", db2[d].tobytes(), wire.DT_VECTOR)])
        assert e.add_doc_raw(doc) == 0
    mask = vi < 3
    rf = [("fi", b"", struct.pack("<i", 3), False, False)]
    res = e.search(xq, topn, is_brute_search=1, range_filters=rf, extra_vec_queries=[("emb2", xq2)])
    fb = np.packbits(mask, bitorder="little")
    _, i1 = orc.flat_search(db, xq, topn, L2, filter_bitmap=fb)
    _, i2 = orc.flat_search(db2, xq2, topn, L2, filter_bitmap=fb)
    for q in range(NQ):
        common = sorted(set(i1[q][i1[q] >= 0]) & set(i2[q][i2[q] >= 0]))[:topn]  # docid order
        assert keys_of(res)[q] == [f"doc{i}" for i in common]
    res = e.search(xq, topn, is_brute_search=1, range_filters=[("fi", struct.pack("<i", 99), b"", True, False)],
                   extra_vec_queries=[("emb2", xq2)])
    assert all(r["items"] == [] and "no result" in r["msg"] for r in res)
    e.close()
