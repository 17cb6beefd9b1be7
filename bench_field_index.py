"""AddFieldIndexWithParams at scale: how long a FLAT field takes to be served by an IVFPQ index built at run time, against
the alternative of a new table re-ingested through the C API, and what the build costs the searches that keep running
on the old index meanwhile.

    python bench_field_index.py [--n 10000000] [--d 128] [--nlist 4096] [--m 16]

Defaults are the C3 shape.  Prints one JSON line with the card's name, power limit and maximum SM clock."""
import argparse
import json
import subprocess
import tempfile
import time

import numpy as np

from vearch_b200 import engine as E, synth, wire


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True).splitlines()[0]
        return [v.strip() for v in out.split(",")]
    except (OSError, subprocess.CalledProcessError):
        return ["unknown", "unknown", "unknown"]


def table(path, typ, params, d):
    e = E.GammaEngine(path, space_name="b")
    e.create_table("b", d, typ, params, fields=(("_id", wire.DT_STRING, False),))
    return e


def ingest(e, db):
    for i in range(len(db)):
        assert e.add_doc(f"d{i}", db[i]) == 0


def pct(v):
    v = np.asarray(v) * 1e3
    return {"median_ms": round(float(np.median(v)), 3), "p99_ms": round(float(np.percentile(v, 99)), 3), "n": len(v)}


def timed(e, q, k):
    t = time.perf_counter()
    r = e.search(q, k)
    return time.perf_counter() - t, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--idle-rounds", type=int, default=50)
    a = ap.parse_args()
    db = synth.sift_like(a.n, a.d, seed=11)
    xq = synth.sift_like(512, a.d, seed=12)
    params = {"ncentroids": a.nlist, "nprobe": 64, "nsubvector": a.m, "metric_type": "L2"}
    res = {"n": a.n, "d": a.d, "nlist": a.nlist, "M": a.m}
    with tempfile.TemporaryDirectory() as tmp:
        e = table(tmp + "/a", "FLAT", {"metric_type": "L2"}, a.d)
        ingest(e, db)
        e.wait_indexed(a.n, timeout=3600)
        probe = e.search(xq[:1], 10)[0]
        idle1, idle512 = [], []
        for _ in range(a.idle_rounds):  # the old index with no build running
            idle1.append(timed(e, xq[:1], 10)[0])
            idle512.append(timed(e, xq, 10)[0])
        busy1, busy512 = [], []
        t0 = time.perf_counter()
        e.add_field_index("emb", "IVFPQ", params)
        while True:  # the FLAT answers are exact; the first inexact one comes from the new index
            dt, r = timed(e, xq[:1], 10)
            if r[0]["items"] != probe["items"]:
                res["add_to_first_new_answer_s"] = round(time.perf_counter() - t0, 3)
                break
            busy1.append(dt)
            dt, r = timed(e, xq, 10)
            if r[0]["items"] != probe["items"]:
                res["add_to_first_new_answer_s"] = round(time.perf_counter() - t0, 3)
                break
            busy512.append(dt)
        e.close()
        res["old_index_1q"] = {"idle": pct(idle1), "during_build": pct(busy1)}
        res["old_index_512q"] = {"idle": pct(idle512), "during_build": pct(busy512)}
        t0 = time.perf_counter()
        f = table(tmp + "/b", "IVFPQ", params, a.d)
        ingest(f, db)
        f.build_index()
        f.wait_indexed(a.n, timeout=3600)
        f.search(xq[:1], 10)
        res["create_and_reingest_to_first_answer_s"] = round(time.perf_counter() - t0, 3)
        f.close()
    res["card"], res["power_limit"], res["max_sm_clock"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
