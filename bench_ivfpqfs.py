"""IVFPQFastScan throughput and recall on one GPU.

  python bench_ivfpqfs.py [--n 10000000] [--nq 10000] [--steps 5] [--warmup 2] [--recall-nums 0,400]

Index: d = 128, M = 64 (32-byte codes), nlist = 4096, trained and filled on the device from seeded SIFT-shaped rows;
search: nprobe 32, k = 10.  Timing follows bench.py: CUDA events around each step, an L2 flush between steps, a
distinct query batch per step.  Prints one JSON line per recall_num with queries/s, recall@10 (the exact 1-NN among the
ten returned, exact neighbours from a FLAT search of the first batch) and the scan kernel's device time per step.
Nothing is written to the tree.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--m", type=int, default=64)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--recall-nums", default="0,400")
    a = ap.parse_args()

    import numpy as np
    import torch
    from vearch_b200 import index as gidx, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_ivfpqfs.py needs a CUDA device")
    dev = torch.device("cuda:0")
    db = synth.sift_like_torch(a.n, a.d, seed=7, device=dev)
    idx = gidx.GammaIndex("IVFPQFastScan", a.d, {"ncentroids": a.nlist, "nprobe": a.nprobe, "nsubvector": a.m,
                                                 "metric_type": "L2"})
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()  # train and add_pending return after their device work has finished
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    batches = [synth.sift_like_torch(a.nq, a.d, seed=1000 + s, device=dev) for s in range(a.warmup + a.steps)]
    # exact 1-NN of the first timed batch
    flat = gidx.GammaIndex("FLAT", a.d, {"metric_type": "L2"})
    flat.add_vectors(db)
    del db
    _, gt = flat.search_device(batches[a.warmup], 1)
    gt = gt.cpu().numpy()[:, 0]
    flat.close()
    torch.cuda.empty_cache()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    cond = gpu_conditions()
    for rn in [int(v) for v in a.recall_nums.split(",")]:
        params = {"nprobe": a.nprobe, "recall_num": rn} if rn > 0 else {"nprobe": a.nprobe}
        times, recall = [], None
        for s, xq in enumerate(batches):
            flush.fill_(s)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _, ids = idx.search_device(xq, a.k, params=params)
            e1.record()
            torch.cuda.synchronize()
            if s >= a.warmup:
                times.append(e0.elapsed_time(e1))
            if s == a.warmup:
                got = ids.cpu().numpy()
                recall = float(np.mean([gt[q] in got[q] for q in range(a.nq)]))
        # scan kernel time in a run of its own (the per-stage events stay out of the timed steps)
        idx.set_scan_timing(True)
        idx.stage_times()
        for xq in batches[a.warmup:]:
            idx.search_device(xq, a.k, params=params)
        torch.cuda.synchronize()
        stages = idx.stage_times()
        idx.set_scan_timing(False)
        ms = sorted(times)[len(times) // 2]
        print(json.dumps({"workload": "ivfpqfs", "n": a.n, "d": a.d, "M": a.m, "nlist": a.nlist, "nq": a.nq,
                          "nprobe": a.nprobe, "k": a.k, "recall_num": rn, "qps": a.nq / (ms / 1e3),
                          "step_ms_median": ms, "step_ms_all": times, "recall_at_10": recall,
                          "stages_ms_per_step": {k: v / a.steps for k, v in stages.items()},
                          "build_s": build_s, "gpu": cond}), flush=True)
    idx.close()


if __name__ == "__main__":
    main()
