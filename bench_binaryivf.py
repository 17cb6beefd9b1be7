"""BINARYIVF throughput, scan roofline and recall on one GPU.

  python bench_binaryivf.py [--n 10000000] [--dims 256,1024] [--nq 10000] [--steps 5] [--warmup 2]

Index: packed binary rows of d bits from the seeded clustered generator (synth.binary_clustered_torch: 4096 random
centres, 10 % of the bits flipped per row), nlist = 4096, trained and filled on the device; search: nprobe 32, k = 10,
through the host entry point (queries uploaded, results downloaded, so the time is end to end).  One JSON line per d:
  - queries/s: median step over `steps` distinct query batches, host clock around a call that ends in a device
    synchronise;
  - the list-scan kernel's device time (CUDA events around its launch, in a run of its own) and its achieved bytes/s,
    counting d / 8 + 8 bytes (code + id) per scanned list entry, against the H100 SXM data-sheet HBM3 3.35 TB/s;
  - recall@10: tie-aware, a result counts when its distance is within the exact 10th distance of its query (exact
    Hamming search over every row, on the first `--recall-queries` queries of the first timed batch).
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


def run(a, d_bits, cond):
    import numpy as np
    import torch
    from vearch_b200 import index as gidx, synth

    dev = torch.device("cuda:0")
    gen = dict(n_clusters=4096, flip=0.1)
    db = synth.binary_clustered_torch(a.n, d_bits, seed=7, device=dev, **gen).cpu().numpy()
    idx = gidx.BinaryIVFIndex(d_bits, {"ncentroids": a.nlist})
    t0 = time.perf_counter()
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()  # train and add_pending return after their device work has finished
    build_s = time.perf_counter() - t0
    del db
    batches = [synth.binary_clustered_torch(a.nq, d_bits, seed=1000 + s, device=dev, **gen).cpu().numpy()
               for s in range(a.warmup + a.steps)]
    params = {"nprobe": a.nprobe}
    times = []
    for s, xq in enumerate(batches):
        t = time.perf_counter()
        dis, _ = idx.search(xq, a.k, params=params)
        if s >= a.warmup:
            times.append((time.perf_counter() - t) * 1e3)
        if s == a.warmup:
            got = dis[:a.recall_queries]
    # exact 10th distances of the recall queries (brute force over every stored row)
    ex, _ = idx.search(batches[a.warmup][:a.recall_queries], a.k, brute_force=True)
    recall = float(np.mean(got <= ex[:, -1:]))
    # scan kernel time in runs of its own, and the entries it scanned
    idx.set_scan_timing(True)
    _ = idx.last_scan_ms  # drop the events of the timed steps
    entries = 0
    lens = np.array([idx.list_len(l) for l in range(a.nlist)], np.int64)
    for xq in batches[a.warmup:]:
        idx.search(xq, a.k, params=params)
        _, probes = idx.coarse_search(xq, a.nprobe)
        entries += int(lens[probes].sum())
    scan_ms = idx.last_scan_ms / a.steps
    idx.set_scan_timing(False)
    entries //= a.steps
    bytes_per_step = entries * (d_bits // 8 + 8)
    gbs = bytes_per_step / (scan_ms / 1e3) / 1e9 if scan_ms > 0 else None
    ms = sorted(times)[len(times) // 2]
    print(json.dumps({"workload": "binaryivf", "n": a.n, "d_bits": d_bits, "nlist": a.nlist, "nq": a.nq,
                      "nprobe": a.nprobe, "k": a.k, "qps": a.nq / (ms / 1e3), "step_ms_median": ms, "step_ms_all": times,
                      "recall_at_10_tie_aware": recall, "recall_queries": a.recall_queries,
                      "scan_kernel": idx.last_scan_kernel, "scan_kernel_ms_per_step": scan_ms,
                      "scanned_entries_per_step": entries, "scan_bytes_per_step": bytes_per_step,
                      "scan_achieved_gbs": gbs, "hbm_peak_gbs_datasheet": HBM_PEAK_GBS,
                      "scan_frac_of_hbm_peak": gbs / HBM_PEAK_GBS if gbs else None, "build_s": build_s, "gpu": cond}),
          flush=True)
    idx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dims", default="256,1024")
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
        raise SystemExit("bench_binaryivf.py needs a CUDA device")
    cond = gpu_conditions()
    for d_bits in [int(v) for v in a.dims.split(",")]:
        run(a, d_bits, cond)


if __name__ == "__main__":
    main()
