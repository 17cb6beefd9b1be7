"""VEARCH throughput, scan bandwidth, encode rate and recall on one GPU, next to IVFPQFastScan on the same rows.

  python bench_vearch.py [--n 10000000] [--nq 10000] [--steps 5] [--warmup 2] [--thresholds 0.2,-1] [--reorder 0,1]

Rows: d = 128, inner product, N(0, 1/d) directions scaled by U(0.3, 1.5) norms (maximum inner product search data),
generated on the device from a seed.  VEARCH: nlist 4096, nsubvector 64 (32-byte codes), nprobe 32, k = 10, at each
ns_threshold (0.2: anisotropic codes; -1: plain nearest-centre codes) with reordering off and on (recall_num 100, the
reference's default).  IVFPQFastScan: M = 64, the same nlist and nprobe, recall_num 0 and 100.  Timing as bench.py:
CUDA events around each step, an L2 flush between steps, a distinct query batch per step.  One JSON line per
configuration: queries/s, the scan kernel's bytes/s (ceil(blocks / 2) + 8 bytes per scanned list entry, over its device
time), add rows/s (list assignment, encoding and append of the whole build's add_pending), recall@10 against an exact
FLAT search of the first timed batch, and the card's name, power limit and maximum SM clock.  Nothing is written to the
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nsub", type=int, default=64)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--thresholds", default="0.2,-1")
    ap.add_argument("--reorder", default="0,1")
    ap.add_argument("--fastscan", type=int, default=1)
    ap.add_argument("--gt-queries", type=int, default=1000)
    a = ap.parse_args()

    import numpy as np
    import torch
    from vearch_b200 import index as gidx

    if not torch.cuda.is_available():
        raise SystemExit("bench_vearch.py needs a CUDA device")
    dev = torch.device("cuda:0")

    def rows(n, seed):
        g = torch.Generator(device=dev).manual_seed(seed)
        x = torch.randn(n, a.d, device=dev, generator=g) / a.d ** 0.5
        return (x * (0.3 + 1.2 * torch.rand(n, 1, device=dev, generator=g))).contiguous()

    db = rows(a.n, 7)
    batches = [rows(a.nq, 1000 + s) for s in range(a.warmup + a.steps)]
    flat = gidx.GammaIndex("FLAT", a.d, {"metric_type": "InnerProduct"})
    flat.add_vectors(db)
    _, gt = flat.search_device(batches[a.warmup][: a.gt_queries], a.k)
    gt = gt.cpu().numpy()
    flat.close()
    torch.cuda.empty_cache()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    cond = gpu_conditions()
    xq_host = batches[a.warmup].cpu().numpy()

    def build(typ, params):
        idx = gidx.VearchIndex(a.d, params) if typ == "VEARCH" else gidx.GammaIndex(typ, a.d, params)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        idx.add_vectors(db)
        idx.train()
        t1 = time.perf_counter()
        idx.add_pending()  # train and add_pending return after their device work has finished
        t2 = time.perf_counter()
        return idx, t1 - t0, a.n / (t2 - t1)

    def scanned_entries(idx):
        lens = np.array([idx.list_len(l) for l in range(idx.nlist)], np.int64)
        _, probes = idx.coarse_search(xq_host, a.nprobe)
        return int(lens[probes].sum())

    def run(idx, workload, params, entry_bytes, scan_kernel, extra):
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
                got = ids.cpu().numpy()[: a.gt_queries]
                recall = float(np.mean([len(set(got[q]) & set(gt[q])) / a.k for q in range(len(gt))]))
        idx.set_scan_timing(True)
        idx.stage_times()
        for xq in batches[a.warmup:]:
            idx.search_device(xq, a.k, params=params)
        torch.cuda.synchronize()
        stages = {k: v / a.steps for k, v in idx.stage_times().items()}
        idx.set_scan_timing(False)
        ms = sorted(times)[len(times) // 2]
        scan_ms = stages.get(scan_kernel)
        ent = scanned_entries(idx)
        out = {"workload": workload, "n": a.n, "d": a.d, "nlist": a.nlist, "nq": a.nq, "nprobe": a.nprobe, "k": a.k,
               "params": params, "qps": a.nq / (ms / 1e3), "step_ms_median": ms, "step_ms_all": times,
               "recall_at_10": recall, "scanned_entries_per_step": ent,
               "scan_bytes_per_s": ent * entry_bytes / (scan_ms / 1e3) if scan_ms else None,
               "stages_ms_per_step": stages, "scan_kernel": idx.last_scan_kernel, "gpu": cond}
        out.update(extra)
        print(json.dumps(out), flush=True)

    for t in [float(v) for v in a.thresholds.split(",")]:
        for ro in [int(v) for v in a.reorder.split(",")]:
            idx, train_s, add_rps = build("VEARCH", {"ncentroids": a.nlist, "nsubvector": a.nsub, "ns_threshold": t,
                                                     "reordering": bool(ro)})
            run(idx, "vearch", {"nprobe": a.nprobe}, (idx.blocks + 1) // 2 + 8, "vearch_scan_kernel",
                {"ns_threshold": t, "reordering": bool(ro), "train_s": train_s, "add_rows_per_s": add_rps})
            idx.close()
    if a.fastscan:
        idx, train_s, add_rps = build("IVFPQFastScan", {"ncentroids": a.nlist, "nprobe": a.nprobe, "nsubvector": a.nsub,
                                                        "metric_type": "InnerProduct"})
        for rn in (0, 100):
            params = {"nprobe": a.nprobe, "recall_num": rn} if rn else {"nprobe": a.nprobe}
            run(idx, "ivfpqfs", params, (a.nsub + 1) // 2 + 8, "ivfpqfs_scan_kernel",
                {"train_s": train_s, "add_rows_per_s": add_rps})
        idx.close()


if __name__ == "__main__":
    main()
