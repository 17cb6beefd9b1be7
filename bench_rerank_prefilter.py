"""What the two-pass exact re-rank reads on the flagship workload, and how fast it reads it.

  python bench_rerank_prefilter.py [--n 10000000] [--warmup 3] [--steps 5] [--recall-num 400] [--nprobe 32]

The exact re-rank (kernels_ivfpq.cu rerank_prefilter_kernel) first reads every candidate's int8 shadow row
(round_up(d, 16) + 16 bytes: the int8 values and their scale, error and norm) and bounds its fp32 score; only the
candidates whose bound can still reach the top k (the survivors) have their fp32 rows (4 d bytes) read and scored.
This script builds bench.py's default workload (C3: IVF-PQ d=128, M=16, nlist=4096, same builder and seeds), runs the
query batches bench.py times, and reports:

  survivors     per query (mean, p99, max), as counted by the kernel
  bytes         gathered in pass 1 (shadow rows of the live candidates) and pass 2 (fp32 rows of the survivors), plus
                the candidate keys, per step
  rerank_kernel its time per step from CUDA events (stage timing), and bytes over that time
  shadow        HBM bytes of the shadow rows (n rows x the shadow stride; the store's HBM figure includes them)

Prints one JSON line; nothing is written to the tree.
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
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--recall-num", type=int, default=400)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--k", type=int, default=10)
    a = ap.parse_args()

    import numpy as np
    import torch
    import bench

    if not torch.cuda.is_available():
        raise SystemExit("bench_rerank_prefilter.py needs a CUDA device")
    dev = torch.device("cuda:0")
    wl = dict(bench.WORKLOADS["ivfpq_10m"])
    t0 = time.time()
    idx, params, _ = bench.build_index(wl, a.n, 0, 0, "sift")
    nprobe = min(a.nprobe, params["ncentroids"])
    sp = {"nprobe": nprobe, "recall_num": a.recall_num}
    d, nq = wl["d"], wl["nq"]
    batches = [bench.generator("sift")(nq, d, seed=4321 + b, device=dev) for b in range(a.warmup + a.steps)]
    kk = max(a.k, a.recall_num)

    # survivors and live candidates of the timed batches (counted, not timed: the count waits for the kernel)
    idx.set_rerank_stats(True)
    surv, live = [], 0
    for b in range(a.warmup, a.warmup + a.steps):
        idx.search_device(batches[b], a.k, params=sp)
        torch.cuda.synchronize()
        s = idx.rerank_survivors()
        if len(s) != nq:
            raise SystemExit("the two-pass re-rank did not serve the search")
        surv.append(s)
        _, ids = idx.search(batches[b].cpu().numpy(), kk, params={"nprobe": nprobe})  # the candidates it was given
        live += int((ids >= 0).sum())
    idx.set_rerank_stats(False)
    surv = np.concatenate(surv).astype(np.float64)

    # stage times of the same batches
    for b in range(a.warmup):
        idx.search_device(batches[b], a.k, params=sp)
    torch.cuda.synchronize()
    idx.set_scan_timing(True)
    idx.stage_times()
    for b in range(a.warmup, a.warmup + a.steps):
        idx.search_device(batches[b], a.k, params=sp)
    torch.cuda.synchronize()
    stages = {kk_: v / a.steps for kk_, v in idx.stage_times().items()}
    idx.set_scan_timing(False)

    dpad = (d + 3) // 4 * 4
    shadow_stride = (dpad + 15) // 16 * 16 + 16
    pass1 = live / a.steps * shadow_stride
    pass2 = float(surv.sum()) / a.steps * 4 * dpad
    keys = nq * kk * 8.0
    ms = stages.get("rerank_kernel", 0.0)
    out = {"workload": "rerank_prefilter", "n": a.n, "nq": nq, "k": a.k, "recall_num": a.recall_num, "nprobe": nprobe,
           "survivors_per_query": {"mean": float(surv.mean()), "p99": float(np.percentile(surv, 99)),
                                   "max": float(surv.max())},
           "live_candidates_per_query": live / a.steps / nq,
           "bytes_per_step": {"pass1_shadow_rows": pass1, "pass2_fp32_rows": pass2, "candidate_keys": keys,
                              "one_pass_fp32_rows": live / a.steps * 4 * dpad},
           "rerank_kernel_ms": ms,
           "rerank_gbs": (pass1 + pass2 + keys) / (ms * 1e-3) / 1e9 if ms > 0 else None,
           "shadow_hbm_bytes": idx.ntotal * shadow_stride,
           "store_hbm_bytes": idx.mem_bytes(1),
           "stages_ms": stages, "gpu": gpu_conditions(), "setup_s": round(time.time() - t0, 1)}
    print(json.dumps(out), flush=True)
    idx.close()


if __name__ == "__main__":
    main()
