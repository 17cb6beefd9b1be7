"""Host cost of the memory limit (SetMemoryLimitConfig): the time of AddOrUpdateDoc and of a 1-query Search with no
limit and with a limit that admits everything, alternated over several rounds in one process.  With a limit set, every
add asks the raw stores what they would grow by and every request reads the ledger and the pool attribute.

    python bench_memory_limit.py [--n 100000] [--d 128] [--ops 2000] [--rounds 3]

Prints the card, its power limit and SM clock, then one JSON line per round and mode (microseconds per call)."""
import argparse
import json
import subprocess
import tempfile
import time

import numpy as np

from vearch_b200 import engine as E, synth, wire


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        return f"unknown ({ex})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--ops", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print("gpu:", gpu_info(), flush=True)
    db = synth.sift_like(a.n + 2 * a.rounds * a.ops, a.d, seed=1)
    xq = synth.sift_like(a.ops, a.d, seed=2)
    with tempfile.TemporaryDirectory() as tmp:
        e = E.GammaEngine(tmp, space_name="bench")
        e.create_table("bench", a.d, "IVFPQ", {"ncentroids": 1024, "nprobe": 32, "metric_type": "L2", "nsubvector": 32,
                                               "training_threshold": 65536})
        for i in range(a.n):
            assert e.add_doc(f"d{i}", db[i]) == 0
        e.build_index()
        e.wait_indexed(a.n)
        reqs = [wire.encode_search_request("emb", xq[j:j + 1], 10) for j in range(a.ops)]
        docs = [wire.build_doc([("_id", f"d{i}".encode(), wire.DT_STRING), ("emb", db[i].tobytes(), wire.DT_VECTOR)])
                for i in range(a.n, len(db))]
        for r in reqs[:200]:  # warm every path the timed loops take
            e.search_raw(r)
        nxt = 0
        for rnd in range(a.rounds):
            for mode in ("off", "on"):
                E.set_memory_limit(90 if mode == "on" else 0)
                t0 = time.perf_counter()
                for k in range(a.ops):
                    assert e.add_doc_raw(docs[nxt + k]) == 0
                t_add = (time.perf_counter() - t0) / a.ops
                nxt += a.ops
                t0 = time.perf_counter()
                for r in reqs:
                    e.search_raw(r)
                t_search = (time.perf_counter() - t0) / a.ops
                print(json.dumps({"round": rnd, "limit": mode, "add_us": round(t_add * 1e6, 2),
                                  "search_1q_us": round(t_search * 1e6, 2)}), flush=True)
        E.set_memory_limit(0)
        e.close()


if __name__ == "__main__":
    main()
