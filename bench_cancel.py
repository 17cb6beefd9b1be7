"""Search cancellation on one GPU: what an unset cancel token costs, and how soon a set one ends a search.

  python bench_cancel.py [--workloads c3,c3_host_rerank,flat] [--runs 3] [--steps 5] [--warmup 2] [--n-c3 10000000]

Workloads, each built once from seeded SIFT-shaped rows (d = 128, L2, k = 10):
  c3:             IVFPQ M = 16, nbits 8, nlist 4096, N = --n-c3, nprobe 32, nq = 10 000 per search
  c5:             the same index at N = --n-c5 (50M in bench.py's configs[4]); not in the default list
  c3_host_rerank: c3 with the raw rows in pinned host memory (store_type "RocksDB") at recall_num 400: every search
                  re-ranks 400 candidates per query over PCIe
  flat:           FLAT, N = 1M, nq = 10 000
Overhead (c3 only): the step time of a search without a token and with a token that is never set, the two arms
alternated, --runs runs of --steps timed searches each (host clock around Index.search, which ends in a device
synchronise).  Kill latency (every workload): a thread sets the token a fixed delay into the search; the time from the
set to the search's return is reported next to the uncancelled search's time.  The card's name, power limit and
maximum SM clock are read in the same process and printed with the numbers.  One JSON line per measurement; nothing is
written to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_ivfpqfs import gpu_conditions  # noqa: E402


def build(kind, a, torch, dev):
    from vearch_b200 import index as gi, synth
    d = 128
    if kind == "flat":
        idx = gi.GammaIndex("FLAT", d, {"metric_type": "L2"})
        idx.add_vectors(synth.sift_like_torch(1_000_000, d, seed=7, device=dev))
        return idx, {}
    n = a.n_c5 if kind == "c5" else a.n_c3
    idx = gi.GammaIndex("IVFPQ", d, {"ncentroids": 4096, "nprobe": 32, "nsubvector": 16, "metric_type": "L2"},
                        store_type="RocksDB" if kind == "c3_host_rerank" else None)
    step = 1 << 22
    for i0 in range(0, n, step):
        idx.add_vectors(synth.sift_like_torch(min(step, n - i0), d, seed=7 + i0, device=dev))
    idx.train()
    idx.add_pending()
    torch.cuda.synchronize()
    return idx, ({"recall_num": 400} if kind == "c3_host_rerank" else {})


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c3_host_rerank,flat")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n-c3", type=int, default=10_000_000)
    ap.add_argument("--n-c5", type=int, default=50_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--delay-ms", type=float, default=2.0, help="when the token is set, after the search starts")
    a = ap.parse_args()
    import torch
    from vearch_b200 import index as gi, synth
    if not torch.cuda.is_available():
        sys.exit("bench_cancel.py needs a CUDA device")
    dev = torch.device("cuda:0")
    card = gpu_conditions()
    xq = [synth.sift_like(a.nq, 128, seed=1000 + s) for s in range(a.warmup + a.steps)]
    for kind in a.workloads.split(","):
        idx, params = build(kind, a, torch, dev)
        for x in xq[:a.warmup]:
            idx.search(x, 10, params=params)
        if kind == "c3":
            # overhead: no token against a token that is never set, alternated
            arms = {"none": [], "unset_token": []}
            for _ in range(a.runs):
                for arm in arms:
                    tok = gi.CancelToken() if arm == "unset_token" else None
                    ms = [timed(lambda: idx.search(x, 10, params=params, cancel=tok)) for x in xq[a.warmup:]]
                    arms[arm].append(statistics.mean(ms))
            spread = max(max(v) - min(v) for v in arms.values())
            print(json.dumps({"measure": "overhead", "workload": kind, "nq": a.nq, "card": card,
                              "step_ms": {k: [round(t, 3) for t in v] for k, v in arms.items()},
                              "diff_ms": round(statistics.mean(arms["unset_token"]) - statistics.mean(arms["none"]), 3),
                              "run_spread_ms": round(spread, 3)}), flush=True)
        # kill latency
        full = [timed(lambda: idx.search(x, 10, params=params)) for x in xq[a.warmup:]]
        lat, total = [], []
        for x in xq[a.warmup:]:
            tok = gi.CancelToken()
            t_set = []

            def setter():
                time.sleep(a.delay_ms / 1e3)
                t_set.append(time.perf_counter())
                tok.set()

            th = threading.Thread(target=setter)
            t0 = time.perf_counter()
            th.start()
            killed = False
            try:
                idx.search(x, 10, params=params, cancel=tok)
            except gi.SearchKilled:
                killed = True
            t1 = time.perf_counter()
            th.join()
            if killed and t_set:
                lat.append((t1 - t_set[0]) * 1e3)
                total.append((t1 - t0) * 1e3)
        print(json.dumps({"measure": "kill_latency", "workload": kind, "nq": a.nq, "card": card,
                          "uncancelled_ms": round(statistics.median(full), 3), "set_delay_ms": a.delay_ms,
                          "set_to_return_ms": [round(t, 3) for t in lat],
                          "call_ms_when_killed": [round(t, 3) for t in total],
                          "killed": f"{len(lat)}/{a.steps}"}), flush=True)
        idx.close()


if __name__ == "__main__":
    main()
