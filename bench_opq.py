"""OPQ training time (DESIGN.md §5, OPQ bar; §9 item 14): opq_train_device at embedding widths, and the share of it
each round's rotation solve (the SVD of X^T Y and R = V U^T) takes.

  python bench_opq.py [--dims 128,256,768,1024] [--n 65536] [--rounds 50] [--repeats 2]
                      [--parent DIR --parent-full-max-d 256 --parent-rounds 2]

Per d: n rows of synth.sift_like (float, seed 51), M = d / 8, one OPQ training of `rounds` rounds through
index.debug_opq_trace without detail (65 536 rows trained on at most).  The whole call is timed with a host clock (it
ends in a device synchronise); when the build reports it, the device time of each round's solve comes from CUDA events
around it, with the Jacobi sweeps the round took.  Each measurement runs in a fresh process after a one-round warm-up
at d = 64.

--parent DIR: the same measurement on another built tree of this project (DIR/vearch_b200/libgamma.so), alternating
with this one `repeats` times.  Above --parent-full-max-d both trees run --parent-rounds rounds only (a slow build
would spend most of an hour per training there) and this tree also runs the full count.  The card's name, power limit
and maximum SM clock go on every line.  Nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def worker(a):
    """one measurement in the tree this process imports from; prints one JSON object"""
    sys.path.insert(0, a.tree)
    import numpy as np
    from vearch_b200 import index as gidx, synth
    assert os.path.dirname(os.path.dirname(os.path.abspath(gidx.__file__))) == os.path.abspath(a.tree)
    d, M = a.d, a.d // 8
    x = synth.sift_like(a.n, d, seed=51, rounded=False)
    # module load and allocator at a small width: at the timed width a slow build's warm-up would cost a whole solve
    gidx.debug_opq_trace(synth.sift_like(4096, 64, seed=52, rounded=False), 8, niter=1, detail=False)
    t0 = time.perf_counter()
    tr = gidx.debug_opq_trace(x, M, niter=a.rounds, detail=False)
    total = time.perf_counter() - t0
    out = {"d": d, "M": M, "n": a.n, "rounds": a.rounds, "total_s": total, "per_round_ms": total / a.rounds * 1e3}
    if "solve_ms" in tr:
        out["solve_ms_total"] = float(np.sum(tr["solve_ms"]))
        out["solve_ms_per_round"] = float(np.mean(tr["solve_ms"]))
        out["solve_share"] = out["solve_ms_total"] / (total * 1e3)
        out["sweeps"] = [int(s) for s in tr["sweeps"]]
    print(json.dumps(out), flush=True)


def measure(tree, d, n, rounds, timeout):
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_opq.py"), "--worker", "--tree", tree, "--d", str(d),
                        "--n", str(n), "--rounds", str(rounds)], env=env, capture_output=True, text=True,
                       timeout=timeout)
    if r.returncode != 0:
        raise SystemExit(f"measurement in {tree} failed:\n{r.stdout}\n{r.stderr}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="128,256,768,1024")
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--parent", default=None)
    ap.add_argument("--parent-full-max-d", type=int, default=256)
    ap.add_argument("--parent-rounds", type=int, default=2)
    ap.add_argument("--timeout", type=float, default=3600)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--d", type=int, default=0)
    ap.add_argument("--tree", default=ROOT)
    a = ap.parse_args()
    if a.worker:
        worker(a)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_opq.py needs a CUDA device")
    cond = gpu_conditions()
    trees = [("this", ROOT)] + ([("parent", os.path.abspath(a.parent))] if a.parent else [])
    for d in [int(v) for v in a.dims.split(",")]:
        runs = []  # (label, tree, rounds, repeat)
        short = a.parent and d > a.parent_full_max_d
        for rep in range(a.repeats if not short else 1):
            order = trees if rep % 2 == 0 else trees[::-1]
            for label, tree in order:
                runs.append((label, tree, a.parent_rounds if short else a.rounds, rep))
        if short:
            runs.append(("this", ROOT, a.rounds, 0))
        for label, tree, rounds, rep in runs:
            res = measure(tree, d, a.n, rounds, a.timeout)
            res.update({"workload": "opq_train", "tree": label, "repeat": rep, "gpu": cond})
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
