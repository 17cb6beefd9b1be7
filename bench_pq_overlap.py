"""Where the C3 step's time goes now that phase B's set-up runs beside phase A.

  python bench_pq_overlap.py [--n 10000000] [--steps 10] [--warmup 3] [--out DIR]

The list-major IVF-PQ search forks the pair grouping and operand staging (pq_group_and_stage_pairs) onto a side stream
while its own stream builds the inner-product table and runs phase A, and joins before binding the filter thresholds
(pq_bind_bounds).  This script builds bench.py's default workload (C3: IVF-PQ d=128, M=16, nlist=4096, nprobe=32,
re-rank 400, nq=10k; same builder, seeds and query batches) and reports, as one JSON line:

  step_ms          device time of a search step (CUDA events, stage timing off)
  stages_ms        per-stage device times (stage timing on, a separate pass); the side chain's stage overlaps others,
                   so the stages add up to more than the step
  main_chain_ms    the stages on the search stream alone: the step if the side chain were fully hidden
  hidden_side_ms   the part of the side chain hidden behind the search stream's work: stages - step, at most the side
                   chain; exposed_side_ms = the rest
  kernels_ms       per-kernel device time per step from torch.profiler, in a third pass (profiler on); its trace and
                   table go under --out
  gpu              the card's name, power limit and maximum SM clock, read in the same run
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_ivfpqfs import gpu_conditions  # noqa: E402

SIDE_STAGES = ("pq_group_and_stage_pairs",)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0, help="vectors (default: the workload's 10M)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default="", help="directory for the profiler's trace and table (default: a temporary one)")
    a = ap.parse_args()

    import numpy as np
    import torch
    import bench

    if not torch.cuda.is_available():
        raise SystemExit("bench_pq_overlap.py needs a CUDA device")
    out_dir = a.out or tempfile.mkdtemp(prefix="pq_overlap_")
    os.makedirs(out_dir, exist_ok=True)
    wl = bench.WORKLOADS["ivfpq_10m"]
    n = a.n or wl["n"]
    dev = "cuda:0"
    idx, params, _ = bench.build_index(wl, n, 0, 0, "sift")
    k, recall_num, nq = 10, 400, wl["nq"]
    sp = {"nprobe": min(wl["nprobe"], params["ncentroids"]), "recall_num": recall_num}
    gen = bench.generator("sift")
    nb = a.warmup + a.steps
    q = [gen(nq, wl["d"], seed=4321 + b, device=dev) for b in range(nb)]
    out_d = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2, between timed steps as in bench.py

    def step(b):
        idx.search_device(q[b], k, params=sp, out=(out_d, out_i))

    for b in range(a.warmup):
        step(b)
    torch.cuda.synchronize()
    kernel = idx.last_scan_kernel

    # pass 1: step time, nothing else recorded
    step_ms = []
    for s in range(a.steps):
        flush.fill_(s)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(a.warmup + s)
        e1.record()
        torch.cuda.synchronize()
        step_ms.append(e0.elapsed_time(e1))

    # pass 2: stage times
    idx.set_scan_timing(True)
    idx.stage_times()
    for s in range(a.steps):
        flush.fill_(s)
        torch.cuda.synchronize()
        step(a.warmup + s)
        torch.cuda.synchronize()
    stages = {name: v / a.steps for name, v in idx.stage_times().items()}
    idx.set_scan_timing(False)

    # pass 3: per-kernel times under torch.profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for s in range(a.profile_steps):
            flush.fill_(s)
            torch.cuda.synchronize()
            step(a.warmup + s)
            torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, "pq_overlap_trace.json"))
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t > 0 and ev.key != "fill_" and "elementwise" not in ev.key and "Memset" not in ev.key:
            kernels[ev.key] = round(t / 1000.0 / a.profile_steps, 4)
    kernels = dict(sorted(kernels.items(), key=lambda kv: -kv[1]))
    with open(os.path.join(out_dir, "pq_overlap_kernels.json"), "w") as f:
        json.dump(kernels, f, indent=1)
    idx.close()

    step_mean = float(np.mean(step_ms))
    side = sum(v for s_, v in stages.items() if s_ in SIDE_STAGES)
    main_chain = sum(v for s_, v in stages.items() if s_ not in SIDE_STAGES)
    hidden = min(side, max(0.0, main_chain + side - step_mean))
    print(json.dumps({
        "workload": "C3 " + wl["desc"], "scan_kernel": kernel, "n": n, "nq": nq, "nprobe": sp["nprobe"],
        "recall_num": recall_num, "steps": a.steps,
        "step_ms": round(step_mean, 4), "step_ms_min": round(min(step_ms), 4), "step_ms_max": round(max(step_ms), 4),
        "stages_ms": {s_: round(v, 4) for s_, v in stages.items()}, "stages_sum_ms": round(main_chain + side, 4),
        "main_chain_ms": round(main_chain, 4), "side_chain_ms": round(side, 4), "hidden_side_ms": round(hidden, 4),
        "exposed_side_ms": round(side - hidden, 4), "kernels_ms": kernels, "out_dir": out_dir,
        "gpu": gpu_conditions()}), flush=True)


if __name__ == "__main__":
    main()
