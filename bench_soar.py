"""SOAR spilling (DESIGN.md §8): recall and throughput of spilled against unspilled lists on one GPU.

  python bench_soar.py [--n 10000000] [--types IVFPQFastScan,IVFRABITQ,VEARCH] [--lambdas 0,1.5] [--nprobes 8,16,32]
                       [--nq 10000] [--steps 5] [--warmup 2] [--repeats 2]

Per type and lambda: d = 128 rows from synth.sift_like_torch, L2, nlist = 4096, trained and filled on the device (the fill
-- assignment, the spilled list, encode and append -- is timed as add rows/s; list bytes = code + 8-byte id per entry).
Per nprobe: k = 10 through the host entry point, no re-rank; queries/s is the median step over `steps` distinct query
batches (host clock around a call that ends in a device synchronise), measured `repeats` times alternating the
nprobes, all steps printed for the spread; recall@10 against the exact top 10 (brute force over every row) on the first
`--recall-queries` queries; scanned entries per query from the coarse search and the list lengths.  Spilled lists are
about twice as long, so the comparison that matters is recall at equal scanned entries (spilled nprobe 16 against
unspilled nprobe 32).  The card's name, power limit and maximum SM clock go on every line.  Nothing is written to the
tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def make(typ, d, nlist, lam):
    from vearch_b200 import index as gidx
    p = {"ncentroids": nlist, "nprobe": 32, "metric_type": "L2"}
    if lam:
        p["soar_lambda"] = lam
    if typ == "IVFPQFastScan":
        return gidx.GammaIndex(typ, d, dict(p, nsubvector=64))
    if typ == "IVFRABITQ":
        return gidx.RaBitQIndex(d, dict(p, nb_bits=4, qb=4))
    return gidx.VearchIndex(d, dict(p, nsubvector=64))


def run(a, typ, lam, db, batches, exact, cond):
    import numpy as np
    idx = make(typ, a.d, a.nlist, lam)
    idx.add_vectors(db)
    t0 = time.perf_counter()
    idx.train()
    train_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    idx.add_pending()  # returns after its device work has finished
    fill_s = time.perf_counter() - t0
    lens = np.array([idx.list_len(l) for l in range(a.nlist)], np.int64)
    nprobes = [int(v) for v in a.nprobes.split(",")]
    times = {p: [] for p in nprobes}
    recall, scanned = {}, {}
    for rep in range(a.repeats):
        for p in nprobes:
            params = {"nprobe": p}
            for s, xq in enumerate(batches):
                t = time.perf_counter()
                _, ids = idx.search(xq, a.k, params=params)
                if s >= a.warmup:
                    times[p].append((time.perf_counter() - t) * 1e3)
                if rep == 0 and s == a.warmup:
                    got = ids[:a.recall_queries]
                    recall[p] = float(np.mean([len(set(got[q]) & set(exact[q])) / a.k for q in range(len(got))]))
                    _, probes = idx.coarse_search(xq, p)
                    scanned[p] = float(lens[probes].sum() / len(xq))
    for p in nprobes:
        ms = sorted(times[p])[len(times[p]) // 2]
        print(json.dumps({"workload": "soar", "type": typ, "soar_lambda": lam, "n": a.n, "d": a.d, "metric": "L2",
                          "nlist": a.nlist, "nq": a.nq, "nprobe": p, "k": a.k, "qps": a.nq / (ms / 1e3),
                          "step_ms_median": ms, "step_ms_all": times[p], "recall_at_10": recall[p],
                          "recall_queries": a.recall_queries, "scanned_entries_per_query": scanned[p],
                          "list_entries": int(lens.sum()), "list_bytes": int(lens.sum()) * (idx.code_size + 8),
                          "train_s": train_s, "add_rows_per_s": a.n / fill_s, "gpu": cond}), flush=True)
    idx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--types", default="IVFPQFastScan,IVFRABITQ,VEARCH")
    ap.add_argument("--lambdas", default="0,1.5")
    ap.add_argument("--nprobes", default="8,16,32")
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--recall-queries", type=int, default=1000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_soar.py needs a CUDA device")
    from vearch_b200 import index as gidx, synth
    cond = gpu_conditions()
    dev = torch.device("cuda:0")
    db = synth.sift_like_torch(a.n, a.d, seed=7, device=dev).cpu().numpy()
    batches = [synth.sift_like_torch(a.nq, a.d, seed=1000 + s, device=dev).cpu().numpy() for s in range(a.warmup + a.steps)]
    flat = gidx.GammaIndex("FLAT", a.d, {"metric_type": "L2"})
    flat.add_vectors(db)
    _, exact = flat.search(batches[a.warmup][:a.recall_queries], a.k)
    flat.close()
    for typ in a.types.split(","):
        for lam in [float(v) for v in a.lambdas.split(",")]:
            run(a, typ, lam, db, batches, exact, cond)


if __name__ == "__main__":
    main()
