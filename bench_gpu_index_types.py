"""GPU_IVFPQ and GPU_IVFFLAT throughput and recall on one GPU, at the shapes vearch's GPU index classes are used with.

  python bench_gpu_index_types.py [--n-pq 10000000] [--n-flat 1000000] [--nq 512] [--steps 20] [--warmup 3]

  - GPU_IVFPQ at its SDK defaults (nsubvector 64, nbits 8), d 128 L2, nlist 4096, nprobe 32, next to IVFPQ at
    nsubvector 16 on the same rows (recall_num 0: ADC results, as GPU_IVFPQ always returns);
  - GPU_IVFFLAT at the C2 shape: d 128 L2, N 1M, nlist 1024, nprobe 32.
Rows from synth.sift_like_torch (seed 7), trained and filled on the device.  Searches go through the host entry point
in calls of `--nq` queries (512, the most a GPU-type call may carry), k = 10.  One JSON line per index:
  - queries/s: median step over `steps` distinct query batches, host clock around a call that ends in a device
    synchronise;
  - recall@10 against the exact top 10 (brute force over every stored row) on the first step's queries.
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


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def run(a, typ, params, db, batches, cond, n):
    import numpy as np
    from vearch_b200 import index as gidx

    idx = gidx.GammaIndex(typ, db.shape[1], params)
    idx.add_vectors(db)
    t0 = time.perf_counter()
    idx.train()
    idx.add_pending()  # returns after its device work has finished
    build_s = time.perf_counter() - t0
    times = []
    for s, xq in enumerate(batches):
        t = time.perf_counter()
        _, ids = idx.search(xq, a.k)
        if s >= a.warmup:
            times.append((time.perf_counter() - t) * 1e3)
        if s == a.warmup:
            got = ids
    kernel = idx.last_scan_kernel
    _, exact = idx.search(batches[a.warmup], a.k, brute_force=True)
    recall = float(np.mean([len(set(got[q]) & set(exact[q])) / a.k for q in range(len(got))]))
    ms = sorted(times)[len(times) // 2]
    print(json.dumps({"workload": "gpu_index_types", "type": typ, "params": params, "n": n, "d": db.shape[1],
                      "nq_per_call": a.nq, "k": a.k, "qps": a.nq / (ms / 1e3), "step_ms_median": ms,
                      "step_ms_all": times, "recall_at_10": recall, "scan_kernel": kernel,
                      "train_and_fill_s": build_s, "gpu": cond}), flush=True)
    idx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-pq", type=int, default=10_000_000)
    ap.add_argument("--n-flat", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=512)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from vearch_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_gpu_index_types.py needs a CUDA device")
    cond = gpu_conditions()
    dev = torch.device("cuda:0")
    batches = [synth.sift_like_torch(a.nq, 128, seed=1000 + s, device=dev).float().cpu().numpy()
               for s in range(a.warmup + a.steps)]
    common = {"ncentroids": 4096, "nprobe": 32, "metric_type": "L2"}
    db = synth.sift_like_torch(a.n_pq, 128, seed=7, device=dev).float()
    run(a, "GPU_IVFPQ", dict(common), db, batches, cond, a.n_pq)  # nsubvector 64, nbits_per_idx 8: the defaults
    run(a, "IVFPQ", dict(common, nsubvector=16), db, batches, cond, a.n_pq)
    del db
    db = synth.sift_like_torch(a.n_flat, 128, seed=7, device=dev).float()
    run(a, "GPU_IVFFLAT", {"ncentroids": 1024, "nprobe": 32, "metric_type": "L2"}, db, batches, cond, a.n_flat)


if __name__ == "__main__":
    main()
