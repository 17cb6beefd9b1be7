"""What dead inverted-list entries cost a search, and what purging them costs, on one GPU.

  python bench_purge.py [--workloads c3,c2] [--n-c3 10000000] [--n-c2 1000000] [--nq 512] [--steps 5] [--warmup 2]

Workloads, built once from seeded SIFT-shaped rows (d = 128, L2, k = 10, nprobe 32):
  c3: IVFPQ M = 16, nbits 8, nlist 4096 (16-byte entries);  c2: IVF-Flat nlist 1024 (512-byte entries).
nq is small enough for the query-major scans, which stream every entry of the probed lists.  For each dead share (0, then
30 % and 50 % of the live entries then in the lists, deleted uniformly at random and hidden by the deletion bitmap; at 30 %
about half of the lists reach the 0.3 threshold and the rest keep their dead entries into the next round) one JSON line:
the search before the purge, the purge, the search after it, the list memory after the re-pack.  Search times are CUDA
events inside the library around the scan kernels (scan_ms) and a host clock around the synchronous search call (call_ms),
medians over --steps after --warmup, a 512 MiB fill between steps to empty L2.  purge_ms is a host clock around the purge
call, which returns after its device work is done and its host tables are refreshed: purge_GBps is the bytes the kernels
must move (ids read twice, live codes and ids read and written once) over that whole call, against the data sheet's
3.35 TB/s, so it is an end-to-end rate, not a kernel's.  Each line carries the card's name, power limit and SM clock.
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

HBM_PEAK_GBPS = 3350.0  # H100 SXM data sheet, at a 700 W limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c3,c2")
    ap.add_argument("--n-c3", type=int, default=10_000_000)
    ap.add_argument("--n-c2", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import numpy as np
    import torch
    from vearch_b200 import index as gidx, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_purge.py needs a CUDA device")
    dev = torch.device("cuda:0")
    d, k = 128, 10
    cond = gpu_conditions()
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    configs = {
        "c3": dict(type="IVFPQ", n=a.n_c3, params={"ncentroids": 4096, "nprobe": 32, "nsubvector": 16, "metric_type": "L2"}),
        "c2": dict(type="IVFFLAT", n=a.n_c2, params={"ncentroids": 1024, "nprobe": 32, "metric_type": "L2"}),
    }

    def timed_search(ix, batches, bm):
        call, scan, ids = [], [], None
        for s, xq in enumerate(batches):
            flush.fill_(s)
            torch.cuda.synchronize()
            ix.last_scan_ms  # forget earlier scans
            t0 = time.perf_counter()
            _, got = ix.search(xq, k, del_bitmap=bm)  # returns with the results on the host
            t1 = time.perf_counter()
            if s >= a.warmup:
                call.append((t1 - t0) * 1e3)
                scan.append(ix.last_scan_ms)
            if s == a.warmup:
                ids = got
        return sorted(call)[len(call) // 2], sorted(scan)[len(scan) // 2], ids

    for wl in a.workloads.split(","):
        cfg = configs[wl]
        db = synth.sift_like_torch(cfg["n"], d, seed=7, device=dev)
        batches = [synth.sift_like_torch(a.nq, d, seed=1000 + s, device=dev).cpu().numpy() for s in range(a.warmup + a.steps)]
        ix = gidx.GammaIndex(cfg["type"], d, cfg["params"])
        ix.add_vectors(db)
        ix.train()
        ix.add_pending()
        ix.compact()
        ix.set_scan_timing(True)
        del db
        torch.cuda.empty_cache()
        cb = ix.code_size
        rng = np.random.default_rng(11)
        alive = np.ones(cfg["n"], bool)
        for share in (0.0, 0.3, 0.5):
            live_vids = np.flatnonzero(alive)
            gone = rng.choice(live_vids, int(len(live_vids) * share), replace=False)
            alive[gone] = False
            ix.delete_vectors(gone)
            bm = np.packbits(~alive, bitorder="little")
            lens0 = np.array([ix.list_len(l) for l in range(ix.nlist)])
            entries = int(lens0.sum())
            mem_before = ix.mem_bytes(0)
            call0, scan0, ids0 = timed_search(ix, batches, bm)
            kern = ix.last_scan_kernel
            t0 = time.perf_counter()
            dropped = ix.purge(0.3, bm)
            purge_ms = (time.perf_counter() - t0) * 1e3
            lens1 = np.array([ix.list_len(l) for l in range(ix.nlist)])
            left = int(lens1.sum())
            call1, scan1, ids1 = timed_search(ix, batches, bm)
            ix.compact()
            hit = lens1 != lens0  # the lists the purge rewrote (uniform deletions leave some below the threshold)
            moved = 2 * 8 * int(lens0[hit].sum()) + 2 * (cb + 8) * int(lens1[hit].sum())
            print(json.dumps({
                "workload": wl, "type": cfg["type"], "n": cfg["n"], "nq": a.nq, "nprobe": 32, "k": k, "code_bytes": cb,
                "dead_share": share, "entries_before": entries, "entries_after": left, "dropped": dropped, "lists_purged": int(hit.sum()),
                "scan_kernel": kern, "scan_ms_before": scan0, "scan_ms_after": scan1, "call_ms_before": call0,
                "call_ms_after": call1, "ids_equal": bool(np.array_equal(ids0, ids1)),
                "index_mem_before": mem_before, "index_mem_after_repack": ix.mem_bytes(0),
                "purge_ms": purge_ms, "purge_moved_bytes": moved,
                "purge_GBps": moved / (purge_ms / 1e3) / 1e9 if dropped else None,
                "purge_share_of_hbm_datasheet": moved / (purge_ms / 1e3) / 1e9 / HBM_PEAK_GBPS if dropped else None,
                "gpu": cond}), flush=True)
        ix.close()
        del batches
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
