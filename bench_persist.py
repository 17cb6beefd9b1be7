"""Restart cost of the quantised index types: the time from Load to the first answered search, from the index file and by
training again, and the index file's size.

  python bench_persist.py [--n 10000000] [--d 128] [--nlist 4096] [--types IVFPQFastScan,IVFRABITQ,VEARCH,BINARYIVF]

For each type an index over N rows (d = 128 floats, sift-like clusters generated on the device from a seed; BINARYIVF:
d = 256 bits, clustered bit vectors) is trained, filled and dumped to a temporary directory.  Then two fresh indexes get
the same raw rows (not timed: a table's Load restores them from its snapshot either way) and are timed, host clock
around work that ends in a device synchronise, from the start of:
  - file:    load_gamma (IndexModel::Load of the type's own file), then one search;
  - retrain: train (k-means and the codec's codebook on the first training_threshold rows), add_pending (every row
             assigned, encoded and appended), then one search;
until that search returns (nq = 100, k = 10, nprobe 32).  The loaded index must answer that batch exactly as the dumped
one did.  Parameters: IVFPQFastScan M = 64; IVFRABITQ nb_bits 4, qb 4; VEARCH nsubvector 64, reordering off; every type
nlist 4096 and its default training threshold.  One JSON line per type, with the card's name, power limit and maximum
SM clock read in the same run.  Nothing is written to the tree.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FILE = {"IVFPQFastScan": "gb_ivfpqfs.index", "IVFRABITQ": "gb_ivfrabitq.index", "VEARCH": "gb_vearch.index",
        "BINARYIVF": "gb_binaryivf.index"}


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else ""
    except (OSError, subprocess.SubprocessError):
        return ""


def make(gidx, kind, d, nlist):
    p = {"ncentroids": nlist, "nprobe": 32, "metric_type": "L2"}
    if kind == "IVFPQFastScan":
        return gidx.GammaIndex(kind, d, dict(p, nsubvector=64))
    if kind == "IVFRABITQ":
        return gidx.RaBitQIndex(d, dict(p, nb_bits=4, qb=4))
    if kind == "VEARCH":
        return gidx.VearchIndex(d, dict(p, nsubvector=64, reordering=False))
    return gidx.BinaryIVFIndex(d, {"ncentroids": nlist, "nprobe": 32})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--bits", type=int, default=256)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=100)
    ap.add_argument("--types", default="IVFPQFastScan,IVFRABITQ,VEARCH,BINARYIVF")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_persist.py measures on a CUDA device; none is visible")
    from vearch_b200 import index as gidx, synth
    dev = torch.device("cuda:0")
    cond = gpu_conditions()
    kinds = [t for t in a.types.split(",") if t]
    data = {}
    if any(k != "BINARYIVF" for k in kinds):
        data["float"] = (synth.sift_like_torch(a.n, a.d, 1, dev).cpu().numpy(),
                         synth.sift_like_torch(a.nq, a.d, 2, dev).cpu().numpy())
    if "BINARYIVF" in kinds:
        data["binary"] = (synth.binary_clustered_torch(a.n, a.bits, 1, dev).cpu().numpy(),
                          synth.binary_clustered_torch(a.nq, a.bits, 2, dev).cpu().numpy())
    torch.cuda.empty_cache()
    for kind in kinds:
        rows, xq = data["binary" if kind == "BINARYIVF" else "float"]
        d = a.bits if kind == "BINARYIVF" else a.d
        tmp = tempfile.mkdtemp(prefix="bench_persist_")
        try:
            src = make(gidx, kind, d, a.nlist)
            src.add_vectors(rows)
            src.train()
            src.add_pending()
            want = src.search(xq, 10)
            src.dump(tmp, "emb.000")
            src.close()
            size = os.path.getsize(os.path.join(tmp, "emb.000", FILE[kind]))

            ld = make(gidx, kind, d, a.nlist)
            ld.add_vectors(rows)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loaded = ld.load(tmp, "emb.000")
            got = ld.search(xq, 10)
            t_file = time.perf_counter() - t0
            ld.close()
            same = bool(np.array_equal(got[1], want[1]) and np.array_equal(got[0].view(np.uint32),
                                                                          want[0].view(np.uint32)))

            rt = make(gidx, kind, d, a.nlist)
            rt.add_vectors(rows)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rt.train()
            rt.add_pending()
            rt.search(xq, 10)
            t_retrain = time.perf_counter() - t0
            rt.close()
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        print(json.dumps({"type": kind, "n": a.n, "d": d, "nlist": a.nlist, "loaded_entries": loaded,
                          "load_to_first_search_s": {"file": round(t_file, 3), "retrain": round(t_retrain, 3)},
                          "file_bytes": size, "answers_equal": same, "gpu": cond}), flush=True)
        if not same:
            sys.exit(f"{kind}: the loaded index answers differently from the dumped one")


if __name__ == "__main__":
    main()
