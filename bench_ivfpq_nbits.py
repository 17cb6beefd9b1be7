"""IVFPQ throughput and recall across code widths (nbits_per_idx) on one GPU.

  python bench_ivfpq_nbits.py [--configs 16x8,32x4,16x4,22x6] [--n 10000000] [--nq 10000] [--steps 5] [--warmup 2]
                              [--recall-nums 400,0]

Index: d = 128, nlist = 4096, M sub-quantisers of nbits bits each (a config "MxB"), trained and filled on the device
from seeded SIFT-shaped rows; search: nprobe 32, k = 10.  The default sweep holds 16-byte (16x8), 16-byte (32x4),
8-byte (16x4) and 17-byte (22x6, rows not word-aligned) codes.  A config whose M does not divide d runs on the same
rows zero-padded to the next multiple of M (22x6: d = 132), which leaves every L2 distance and so the exact neighbours
unchanged.  Timing follows bench.py: CUDA events around each step,
an L2 flush between steps, a distinct device-resident query batch per step.  Prints one JSON line per (config,
recall_num) with queries/s, recall@10 (the exact 1-NN among the ten returned; exact neighbours from a FLAT search of
the first timed batch), the bytes of list codes and the kernel that served the scan.

The 8-bit configuration runs the list-major tensor-core filter (pqtc_scan_kernel) on batches this large, the packed
ones the query-major packed-code kernel (ivfpq_packed_scan_kernel): the lines compare code widths, not kernels.
Nothing is written to the tree.
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
    ap.add_argument("--configs", default="16x8,32x4,16x4,22x6", help="comma-separated MxNBITS")
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--recall-nums", default="400,0")
    a = ap.parse_args()
    configs = [tuple(int(v) for v in c.split("x")) for c in a.configs.split(",")]
    for M, nbits in configs:
        if not 1 <= nbits <= 8:
            raise SystemExit(f"config {M}x{nbits}: nbits must be in 1..8")

    import numpy as np
    import torch
    from vearch_b200 import index as gidx, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_ivfpq_nbits.py needs a CUDA device")
    dev = torch.device("cuda:0")
    db = synth.sift_like_torch(a.n, a.d, seed=7, device=dev)
    batches = [synth.sift_like_torch(a.nq, a.d, seed=1000 + s, device=dev) for s in range(a.warmup + a.steps)]
    flat = gidx.GammaIndex("FLAT", a.d, {"metric_type": "L2"})
    flat.add_vectors(db)
    _, gt = flat.search_device(batches[a.warmup], 1)
    gt = gt.cpu().numpy()[:, 0]
    flat.close()
    torch.cuda.empty_cache()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    cond = gpu_conditions()
    print(json.dumps({"note": "nbits 8 runs pqtc_scan_kernel (list-major tensor-core filter) on these batches, nbits < 8 "
                              "the query-major ivfpq_packed_scan_kernel: the lines compare code widths, not kernels",
                      "gpu": cond}), flush=True)
    for M, nbits in configs:
        dm = -(-a.d // M) * M  # zero padding to a multiple of M
        pad = (lambda x: torch.nn.functional.pad(x, (0, dm - a.d))) if dm != a.d else (lambda x: x)
        qb = [pad(xq) for xq in batches]
        idx = gidx.GammaIndex("IVFPQ", dm, {"ncentroids": a.nlist, "nprobe": a.nprobe, "nsubvector": M,
                                            "nbits_per_idx": nbits, "metric_type": "L2"})
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        idx.add_vectors(pad(db))
        idx.train()
        idx.add_pending()  # train and add_pending return after their device work has finished
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        for rn in [int(v) for v in a.recall_nums.split(",")]:
            params = {"nprobe": a.nprobe, "recall_num": rn} if rn > 0 else {"nprobe": a.nprobe}
            times, recall, kernel = [], None, ""
            for s, xq in enumerate(qb):
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
                    kernel = idx.last_scan_kernel
            ms = sorted(times)[len(times) // 2]
            print(json.dumps({"workload": "ivfpq_nbits", "n": a.n, "d": dm, "M": M, "nbits": nbits,
                              "code_size": idx.code_size, "list_code_bytes": a.n * idx.code_size, "nlist": a.nlist,
                              "nq": a.nq, "nprobe": a.nprobe, "k": a.k, "recall_num": rn, "qps": a.nq / (ms / 1e3),
                              "step_ms_median": ms, "step_ms_all": times, "recall_at_10": recall,
                              "scan_kernel": kernel, "build_s": build_s, "gpu": cond}), flush=True)
        idx.close()
        del qb
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
