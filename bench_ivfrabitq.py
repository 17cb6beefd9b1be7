"""IVFRABITQ throughput, scan roofline, encode rate and recall on one GPU.

  python bench_ivfrabitq.py [--n 10000000] [--shapes 128:L2,768:IP] [--bits 1,4,9] [--qbs 0,4] [--recall-nums 0,400]
                            [--nq 10000] [--steps 5] [--warmup 2]

Index per (d, metric, nb_bits): rows from the seeded generators (d 128 L2: synth.sift_like_torch; d 768 IP:
synth.embed_like_torch), nlist = 4096, trained and filled on the device; the fill (assignment + encode + append) is timed
as encode rows/s.  Search per (qb, recall_num): nprobe 32, k = 10, through the host entry point (end to end).  One JSON
line per search configuration:
  - queries/s: median step over `steps` distinct query batches, host clock around a call that ends in a device
    synchronise;
  - the list-scan kernel's device time (CUDA events around its launch) and its achieved bytes/s, counting the entry
    (code_size bytes) + its 8-byte id per scanned list entry, against the H100 SXM data-sheet HBM3 3.35 TB/s;
  - recall@10 against the exact top 10 (brute force over every stored row) on the first `--recall-queries` queries.
The card's name, power limit and maximum SM clock are printed with each line.  Nothing is written to the tree.
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

HBM_PEAK_GBS = 3350.0  # NVIDIA H100 SXM data sheet, not a measured peak


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def gen(d, n, seed, dev):
    from vearch_b200 import synth
    if d == 128:
        return synth.sift_like_torch(n, d, seed=seed, device=dev)
    return synth.embed_like_torch(n, d, seed=seed, device=dev)


def run(a, d, metric, bits, cond):
    import numpy as np
    import torch
    from vearch_b200 import index as gidx

    dev = torch.device("cuda:0")
    db = gen(d, a.n, 7, dev).float().cpu().numpy()
    batches = [gen(d, a.nq, 1000 + s, dev).float().cpu().numpy() for s in range(a.warmup + a.steps)]
    idx = gidx.RaBitQIndex(d, {"ncentroids": a.nlist, "nprobe": a.nprobe, "nb_bits": bits, "metric_type": metric})
    idx.add_vectors(db)
    t0 = time.perf_counter()
    idx.train()
    train_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    idx.add_pending()  # returns after its device work has finished
    fill_s = time.perf_counter() - t0
    del db
    exact_ids = None
    lens = np.array([idx.list_len(l) for l in range(a.nlist)], np.int64)
    entries = 0
    for xq in batches[a.warmup:]:
        _, probes = idx.coarse_search(xq, a.nprobe)
        entries += int(lens[probes].sum())
    entries //= a.steps
    for qb in [int(v) for v in a.qbs.split(",")]:
        for rn in [int(v) for v in a.recall_nums.split(",")]:
            params = {"nprobe": a.nprobe, "qb": qb}
            if rn:
                params["recall_num"] = rn
            times = []
            for s, xq in enumerate(batches):
                t = time.perf_counter()
                _, ids = idx.search(xq, a.k, params=params)
                if s >= a.warmup:
                    times.append((time.perf_counter() - t) * 1e3)
                if s == a.warmup:
                    got = ids[:a.recall_queries]
            if exact_ids is None:
                _, exact_ids = idx.search(batches[a.warmup][:a.recall_queries], a.k, brute_force=True)
            recall = float(np.mean([len(set(got[q]) & set(exact_ids[q])) / a.k for q in range(len(got))]))
            idx.set_scan_timing(True)
            _ = idx.last_scan_ms  # drop the events of the timed steps
            for xq in batches[a.warmup:]:
                idx.search(xq, a.k, params=params)
            scan_ms = idx.last_scan_ms / a.steps
            idx.set_scan_timing(False)
            bytes_per_step = entries * (idx.code_size + 8)
            gbs = bytes_per_step / (scan_ms / 1e3) / 1e9 if scan_ms > 0 else None
            ms = sorted(times)[len(times) // 2]
            print(json.dumps({"workload": "ivfrabitq", "n": a.n, "d": d, "metric": metric, "nb_bits": bits, "qb": qb,
                              "recall_num": rn, "nlist": a.nlist, "nq": a.nq, "nprobe": a.nprobe, "k": a.k,
                              "qps": a.nq / (ms / 1e3), "step_ms_median": ms, "step_ms_all": times,
                              "recall_at_10": recall, "recall_queries": len(got), "code_size": idx.code_size,
                              "scan_kernel": idx.last_scan_kernel, "scan_kernel_ms_per_step": scan_ms,
                              "scanned_entries_per_step": entries, "scan_bytes_per_step": bytes_per_step,
                              "scan_achieved_gbs": gbs, "hbm_peak_gbs_datasheet": HBM_PEAK_GBS,
                              "scan_frac_of_hbm_peak": gbs / HBM_PEAK_GBS if gbs else None, "train_s": train_s,
                              "encode_rows_per_s": a.n / fill_s, "gpu": cond}), flush=True)
    idx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--shapes", default="128:L2,768:InnerProduct")
    ap.add_argument("--bits", default="1,4,9")
    ap.add_argument("--qbs", default="0,4")
    ap.add_argument("--recall-nums", default="0,400")
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--recall-queries", type=int, default=1000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ivfrabitq.py needs a CUDA device")
    cond = gpu_conditions()
    for shape in a.shapes.split(","):
        d, metric = shape.split(":")
        for bits in [int(v) for v in a.bits.split(",")]:
            run(a, int(d), metric, bits, cond)


if __name__ == "__main__":
    main()
