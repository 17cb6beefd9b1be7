"""Raw vectors in HBM against raw vectors in pinned host memory (store_type "RocksDB") on one GPU.

  python bench_host_store.py [--workloads c3,c2] [--runs 3] [--steps 5] [--warmup 2] [--n-c3 10000000] [--n-c2 1000000]

Workloads, each built once per placement from the same seeded SIFT-shaped rows (d = 128, L2, k = 10, nq = 10 000):
  c3: IVFPQ M = 16, nbits 8, nlist 4096, N = 10M, nprobe 32, at recall_num 0 and 400.  recall_num 400 re-ranks 400
      candidates per query from the raw rows: over PCIe for the host store (10k x 400 x 512 B = 2.05 GB per batch).
  c2: IVF-Flat nlist 1024, N = 1M, nprobe 32.  Its winner re-score reads the list rows in either placement.
The two placements run alternately, --runs times each.  Timing follows bench.py: CUDA events around each step, an L2
flush between steps, a distinct device-resident query batch per step.  Each run prints one JSON line: queries/s, recall@10
(the exact 1-NN among the ten returned; exact neighbours from a FLAT search of the first timed batch), whether its ids
equal those of the HBM placement's first run, the store's HBM and host bytes, the re-rank stage's device time per batch,
the pinned host-to-device bandwidth measured in the same process (events around a 1 GiB copy) and the card's name and
power limit.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_ivfpqfs import gpu_conditions  # noqa: E402

PLACEMENTS = (("hbm", None), ("host", "RocksDB"))


def pinned_h2d_gbps(torch, dev):
    src = torch.empty(1 << 30, dtype=torch.uint8).pin_memory()
    dst = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
    best = 0.0
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        best = max(best, (1 << 30) / (e0.elapsed_time(e1) / 1e3) / 1e9)
    del src, dst
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c2")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n-c3", type=int, default=10_000_000)
    ap.add_argument("--n-c2", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    a = ap.parse_args()

    import numpy as np
    import torch
    from vearch_b200 import index as gidx, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_host_store.py needs a CUDA device")
    dev = torch.device("cuda:0")
    d, k = 128, 10
    cond = gpu_conditions()
    h2d = pinned_h2d_gbps(torch, dev)
    print(json.dumps({"pinned_h2d_GBps": h2d, "gpu": cond}), flush=True)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    configs = {
        "c3": dict(type="IVFPQ", n=a.n_c3, params={"ncentroids": 4096, "nprobe": 32, "nsubvector": 16, "metric_type": "L2"},
                   recall_nums=[0, 400]),
        "c2": dict(type="IVFFLAT", n=a.n_c2, params={"ncentroids": 1024, "nprobe": 32, "metric_type": "L2"},
                   recall_nums=[0]),
    }
    for wl in a.workloads.split(","):
        cfg = configs[wl]
        db = synth.sift_like_torch(cfg["n"], d, seed=7, device=dev)
        batches = [synth.sift_like_torch(a.nq, d, seed=1000 + s, device=dev) for s in range(a.warmup + a.steps)]
        flat = gidx.GammaIndex("FLAT", d, {"metric_type": "L2"})
        flat.add_vectors(db)
        _, gt = flat.search_device(batches[a.warmup], 1)
        gt = gt.cpu().numpy()[:, 0]
        flat.close()
        idx = {}
        for name, st in PLACEMENTS:
            idx[name] = gidx.GammaIndex(cfg["type"], d, cfg["params"], store_type=st)
            idx[name].add_vectors(db)
            idx[name].train()
            idx[name].add_pending()
            idx[name].set_scan_timing(True)
        del db
        torch.cuda.empty_cache()
        for rn in cfg["recall_nums"]:
            params = {"nprobe": 32, "recall_num": rn} if rn > 0 else {"nprobe": 32}
            ref_ids = None
            for run in range(a.runs):
                for name, _ in PLACEMENTS:
                    ix = idx[name]
                    times, got = [], None
                    for s, xq in enumerate(batches):
                        flush.fill_(s)
                        torch.cuda.synchronize()
                        ix.stage_times()  # forget earlier stages
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        _, ids = ix.search_device(xq, k, params=params)
                        e1.record()
                        torch.cuda.synchronize()
                        if s >= a.warmup:
                            times.append(e0.elapsed_time(e1))
                        if s == a.warmup:
                            got = ids.cpu().numpy()
                            stages = ix.stage_times()
                    if ref_ids is None:
                        ref_ids = got
                    ms = sorted(times)[len(times) // 2]
                    rr_ms = stages.get("rerank_kernel")
                    rr_bytes = a.nq * rn * d * 4 if rn > 0 else 0
                    print(json.dumps({
                        "workload": wl, "placement": name, "run": run, "type": cfg["type"], "n": cfg["n"], "nq": a.nq,
                        "nprobe": 32, "k": k, "recall_num": rn, "qps": a.nq / (ms / 1e3), "step_ms_median": ms,
                        "step_ms_all": times, "recall_at_10": float(np.mean([gt[q] in got[q] for q in range(a.nq)])),
                        "ids_equal_hbm": bool(np.array_equal(got, ref_ids)), "store_hbm_bytes": ix.mem_bytes(1),
                        "store_host_bytes": ix.mem_bytes(2), "index_hbm_bytes": ix.mem_bytes(0),
                        "scan_kernel": ix.last_scan_kernel, "rerank_ms": rr_ms,
                        "rerank_GBps": rr_bytes / (rr_ms / 1e3) / 1e9 if rr_ms else None,
                        "rerank_share_of_pinned_h2d": (rr_bytes / (rr_ms / 1e3) / 1e9 / h2d
                                                       if rr_ms and name == "host" else None),
                        "pinned_h2d_GBps": h2d, "gpu": cond}), flush=True)
        for ix in idx.values():
            ix.close()
        del batches
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
