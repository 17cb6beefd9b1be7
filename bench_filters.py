"""Filtered search through the engine C-ABI (include/gamma_api.h): per-call latency of searches with scalar filters,
the filter stage's device time, the bytes it reads and writes, and ingest rows/s with four indexed scalar fields.

  python bench_filters.py [--n 10000000] [--reps 20] [--out results.json]

Table: d = 128 sift-like rows (seeded), IVFPQ at the C3 shape (nlist 4096, nsubvector 16, nbits 8, nprobe 32, L2), and
four indexed scalar fields per document: price INT uniform in [0, 10000), ts LONG, score FLOAT, tag STRING (one of 100).
Requests of 1, 16 and 512 queries (k = 10) under each filter set:
  range1 / range10 / range50 / range90: price < 100 / 1000 / 5000 / 9000 (1, 10, 50, 90 % of the documents);
  term: tag in {t7} (1 %);  and / or: price < 5000 combined with tag in {t1 .. t10}.
Per call: the median host-clock time of `--reps` calls after two warm-up calls (Search returns after its results are on
the host).  Filter stage: filter_eval_kernel's device time in a separate torch.profiler pass (CUDA activities), averaged
over its launches; null when the build has no such kernel.  Filter bytes: what the kernel must move, the filtered
columns (value width plus a validity bit per document, or a 4-byte string code) plus N / 8 output bytes per filter.
Ingest: AddOrUpdateDoc calls per second over all N documents, each with the four scalar fields, until every vector is
indexed.  The result ids of every (request size, filter set) are hashed, so two builds can be compared with --compare.
Only the engine's C-ABI is used, so the script runs on any build of the engine.  Nothing is written to the tree.
"""
import argparse
import hashlib
import json
import os
import shutil
import statistics
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def filter_sets():
    i32 = lambda v: struct.pack("<i", v)
    tags10 = b"\x01".join(f"t{i}".encode() for i in range(1, 11))
    sets = {f"range{p}": dict(range_filters=[("price", b"", i32(p * 100), False, False)]) for p in (1, 10, 50, 90)}
    sets["term"] = dict(term_filters=[("tag", b"t7")])
    sets["and"] = dict(range_filters=[("price", b"", i32(5000), False, False)], term_filters=[("tag", tags10)])
    sets["or"] = dict(range_filters=[("price", b"", i32(5000), False, False)], term_filters=[("tag", tags10)], operator=1)
    return sets


def filter_bytes(name, n):
    per = {"price": n * 4 + n / 8, "tag": n * 4}
    cols = {"term": ["tag"], "and": ["price", "tag"], "or": ["price", "tag"]}.get(name, ["price"])
    return sum(per[c] + n / 8 for c in cols)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="compare the id hashes of two --out files")
    a = ap.parse_args()
    if a.compare:
        x, y = (json.load(open(p)) for p in a.compare)
        same = {k: x["ids"][k] == y["ids"].get(k) for k in x["ids"]}
        print(json.dumps({"ids_identical": all(same.values()), "differ": [k for k, v in same.items() if not v]}))
        return
    import torch
    from vearch_b200 import engine, synth, wire

    cond = gpu_conditions()
    n, d = a.n, 128
    rng = np.random.default_rng(11)
    price = rng.integers(0, 10000, n).astype(np.int32)
    tag = rng.integers(0, 100, n)
    xb = synth.sift_like(n, d, seed=1)
    xq = synth.sift_like(512, d, seed=2)
    tmp = tempfile.mkdtemp(prefix="bench_filters_")
    e = engine.GammaEngine(tmp, space_name="bf")
    e.create_table("bf", d, "IVFPQ", {"ncentroids": 4096, "nprobe": 32, "nsubvector": 16, "nbits_per_idx": 8,
                                      "metric_type": "L2", "training_threshold": 4096 * 100},
                   fields=(("_id", wire.DT_STRING, False), ("price", wire.DT_INT, True), ("ts", wire.DT_LONG, True),
                           ("score", wire.DT_FLOAT, True), ("tag", wire.DT_STRING, True)), refresh_interval=1000)
    tags = [f"t{i}".encode() for i in range(100)]
    t0 = time.perf_counter()
    for i in range(n):
        doc = wire.build_doc([("_id", b"d%d" % i, wire.DT_STRING), ("price", struct.pack("<i", int(price[i])), wire.DT_INT),
                              ("ts", struct.pack("<q", 1_700_000_000 + i), wire.DT_LONG),
                              ("score", struct.pack("<f", float(i % 1000) / 7), wire.DT_FLOAT),
                              ("tag", tags[tag[i]], wire.DT_STRING), ("emb", xb[i].tobytes(), wire.DT_VECTOR)])
        assert e.add_doc_raw(doc) == 0
    e.wait_indexed(n, timeout=3600)
    ingest_s = time.perf_counter() - t0
    print(json.dumps({"gpu": cond, "n": n, "ingest_rows_per_s": round(n / ingest_s, 1), "ingest_s": round(ingest_s, 2),
                      "memory": e.memory_info()}), flush=True)
    ids, rows = {}, []
    for nq in (1, 16, 512):
        q = xq[:nq]
        kw0 = dict(index_params={"nprobe": 32})
        for name, fk in [("none", {})] + list(filter_sets().items()):
            call = lambda: e.search(q, 10, **kw0, **fk)
            for _ in range(2):
                res = call()
            ts = []
            for _ in range(a.reps):
                t = time.perf_counter()
                res = call()
                ts.append(time.perf_counter() - t)
            keys = [[it["fields"]["_id"].decode() for it in r["items"]] for r in res]
            ids[f"{nq}/{name}"] = hashlib.sha1(json.dumps(keys).encode()).hexdigest()
            row = {"nq": nq, "filter": name, "call_ms": round(statistics.median(ts) * 1e3, 3)}
            if name != "none" and nq == 1:
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(10):
                        call()
                    torch.cuda.synchronize()
                ev = [k for k in prof.key_averages() if "filter_eval_kernel" in k.key]
                if ev:
                    us = ev[0].device_time_total / max(ev[0].count, 1) if hasattr(ev[0], "device_time_total") \
                        else ev[0].cuda_time_total / max(ev[0].count, 1)
                    b = filter_bytes(name, n)
                    row.update(filter_us=round(us, 2), filter_bytes=int(b),
                               filter_tb_per_s=round(b / (us * 1e-6) / 1e12, 3),
                               filter_share_of_3_35_tb_per_s=round(b / (us * 1e-6) / HBM_BYTES_PER_S, 3))
                else:
                    row.update(filter_us=None, filter_bytes=int(filter_bytes(name, n)))
            rows.append(row)
            print(json.dumps(row), flush=True)
    e.close()
    shutil.rmtree(tmp, ignore_errors=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": cond, "n": n, "ingest_rows_per_s": n / ingest_s, "rows": rows, "ids": ids}, f)


if __name__ == "__main__":
    main()
