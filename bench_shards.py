"""GPU_IVFPQ sharded over several devices against the unsharded index.

  python bench_shards.py [--n 10000000] [--nq 512] [--steps 5] [--warmup 2] [--same-device 2,4]

Workload: GPU_IVFPQ at its defaults (nsubvector 64, nlist 4096 here, nprobe 32, d = 128, L2, k = 10) over seeded
SIFT-shaped rows (synth.sift_like), searched in 512-query calls through the host entry point.  One JSON line per
placement: S = 1 (today's index), S shards over min(visible devices, 8) distinct devices when more than one is visible,
and S = 2 and 4 on device 0 alone, which isolates what the merge and the extra launches cost.  Each line gives queries/s
(host clock around the synchronous call with timing off, median over --steps after --warmup), the merge kernel's
device time per call (CUDA events around it, summed over --merge-calls calls in a separate pass), recall@10 overlap with the exact top 10 of the first 64 queries (brute force on the same
index), whether the results equal the unsharded index's, the HBM each device's default pool and the index hold after
the build, and the card's name, power limit and SM clock.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_ivfpqfs import gpu_conditions  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--nq", type=int, default=512)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--same-device", default="2,4")
    ap.add_argument("--merge-calls", type=int, default=50)
    a = ap.parse_args()
    import numpy as np
    import torch
    from vearch_b200 import index as gidx, synth

    d = 128
    ndev = torch.cuda.device_count()
    db = synth.sift_like(a.n, d, seed=1)
    xq = synth.sift_like(a.nq, d, seed=2)
    params = {"ncentroids": a.nlist, "nprobe": 32, "metric_type": "L2", "nsubvector": 64}
    placements = [None]
    if ndev > 1:
        placements.append(list(range(min(ndev, 8))))
    placements += [[0] * int(s) for s in a.same_device.split(",") if s]
    ref = None
    exact = None
    for devs in placements:
        idx = gidx.GammaIndex("GPU_IVFPQ", d, params, devices=devs)
        t0 = time.time()
        for i in range(0, a.n, 1 << 20):
            idx.add_vectors(db[i:i + (1 << 20)])
        idx.train()
        idx.add_pending()
        build_s = time.time() - t0
        torch.cuda.synchronize()
        hbm = {}
        for dv in sorted(set(devs or [0])):
            free, total = torch.cuda.mem_get_info(dv)
            hbm[f"cuda:{dv}"] = round((total - free) / 2**30, 3)
        times = []  # end to end, timing off
        for it in range(a.warmup + a.steps):
            t = time.perf_counter()
            got = idx.search(xq, 10)
            times.append(time.perf_counter() - t)
        # the merge kernel's device time: a separate pass with timing on, summed over --merge-calls calls
        idx.set_scan_timing(True)
        idx.stage_times()
        for it in range(a.merge_calls):
            idx.search(xq, 10)
        merge_ms = idx.stage_times().get("shard_merge", 0.0) / a.merge_calls
        idx.set_scan_timing(False)
        med = float(np.median(times[a.warmup:]))
        if exact is None:
            exact = idx.search(xq[:64], 10, brute_force=True)[1]
        rec = float(np.mean([len(set(got[1][q]) & set(exact[q])) / 10 for q in range(64)]))
        if ref is None:
            ref = got
        line = {"placement": "unsharded" if devs is None else devs, "shards": 1 if devs is None else len(devs),
                "n": a.n, "nq": a.nq, "qps": round(a.nq / med, 1), "call_ms": round(med * 1e3, 3),
                "merge_ms": round(merge_ms, 4), "recall_at_10": rec,
                "equal_to_unsharded": bool(np.array_equal(got[0].view(np.uint32), ref[0].view(np.uint32)) and
                                           np.array_equal(got[1], ref[1])),
                "index_hbm_GiB": round(idx.mem_bytes(0) / 2**30, 3), "device_used_GiB": hbm,
                "build_s": round(build_s, 1)}
        line["gpu"] = gpu_conditions()
        print(json.dumps(line), flush=True)
        idx.close()


if __name__ == "__main__":
    main()
