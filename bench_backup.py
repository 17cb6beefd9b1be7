"""Backup and Dump at scale: how long the table lock is held (the capture), how long each call takes in all, and what a
backup costs the searches that keep running meanwhile.

    python bench_backup.py [--n 10000000] [--d 128] [--nlist 4096] [--m 16] [--rounds 3]

Defaults are the C3 shape (IVFPQ d 128, M 16, nlist 4096, N 10M, L2).  The table's rows are sift-like clusters from a
seed, ingested through the C API.  Timings are host clocks around calls that end in a device synchronise:
  - capture: from Backup's call until it waits at the test hold (gb_debug_backup_hold), i.e. the lock window plus the
    pending-row flush; the write then continues once the hold is released;
  - backup / dump: the whole call, without the hold, alternating the two for `rounds` rounds;
  - search: 1-query searches (k 10, nprobe 32) back to back, idle and while a backup runs; p50 and slowest call.
Files go to a temporary directory.  One JSON line, with the card's name, power limit and maximum SM clock."""
import argparse
import json
import shutil
import subprocess
import tempfile
import threading
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


def latencies(e, xq, stop=None, count=200):
    out, i = [], 0
    while (stop is None and i < count) or (stop is not None and not stop.is_set()):
        t0 = time.perf_counter()
        e.search(xq[i % len(xq)][None], 10, index_params={"nprobe": 32})
        out.append(time.perf_counter() - t0)
        i += 1
    return out


def summary(v):
    v = np.asarray(v) * 1e3
    return {"calls": int(v.size), "p50_ms": round(float(np.median(v)), 3), "max_ms": round(float(v.max()), 3)} if v.size else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--m", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    name, power, clock = card()
    tmp = tempfile.mkdtemp(prefix="bench_backup_")
    try:
        db = synth.sift_like(a.n, a.d, seed=1)
        xq = synth.sift_like(256, a.d, seed=2)
        e = E.GammaEngine(tmp, space_name="b")
        e.create_table("b", a.d, "IVFPQ", {"ncentroids": a.nlist, "nsubvector": a.m, "nprobe": 32, "metric_type": "L2"},
                       fields=(("_id", wire.DT_STRING, False),))
        t0 = time.perf_counter()
        for i in range(a.n):
            assert e.add_doc(f"d{i}", db[i]) == 0
        e.wait_indexed(a.n, timeout=3600)
        ingest_s = time.perf_counter() - t0
        latencies(e, xq, count=50)  # warm-up
        idle = latencies(e, xq)

        # the lock window: until the backup reaches its hold, right after the capture
        E.backup_hold(1)
        th = threading.Thread(target=e.backup)
        t0 = time.perf_counter()
        th.start()
        while E.backup_hold(-1) != 2:
            pass
        capture_s = time.perf_counter() - t0
        stage = E.backup_stage()
        E.backup_hold(0)
        th.join()

        backup_s, dump_s = [], []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            e.backup()
            backup_s.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            assert e.dump() == 0
            dump_s.append(time.perf_counter() - t0)

        stop = threading.Event()
        during = []
        th = threading.Thread(target=lambda: during.extend(latencies(e, xq, stop=stop)))
        th.start()
        t0 = time.perf_counter()
        e.backup()
        during_backup_s = time.perf_counter() - t0
        stop.set()
        th.join()
        e.close()
        print(json.dumps({
            "shape": {"type": "IVFPQ", "n": a.n, "d": a.d, "nlist": a.nlist, "M": a.m},
            "gpu": name, "power_limit": power, "max_sm_clock": clock, "ingest_s": round(ingest_s, 1),
            "capture_ms": round(capture_s * 1e3, 2), "stage_bytes": {"hbm": stage[0], "host": stage[1]},
            "backup_s": [round(v, 3) for v in backup_s], "dump_s": [round(v, 3) for v in dump_s],
            "search_idle": summary(idle), "search_during_backup": summary(during),
            "backup_with_searches_s": round(during_backup_s, 3)}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
