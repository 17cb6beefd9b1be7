"""How many entries the IVF-PQ tensor-core filter passes per query, under the fp16 and the int8 error bounds.

  python bench_pqtc_int8.py [--n 10000000] [--nq 1000] [--warmup 3] [--kprime 400] [--nprobe 32] [--search-steps 3]

The list-major IVF-PQ search (kernels_pqtc.cu) scores each query's leading probes exactly (phase A), takes the k'-th
best score B_q as a bound, and lets the tensor core filter the other probes (phase B): an entry is a candidate when its
approximate score, widened by a rigorous error margin eps, can reach B_q.  Every candidate costs an epilogue slow
path, a queue record and an exact re-score, so the margin decides whether a cheaper operand type pays.  This script
restates the filter on bench.py's default workload (C3: IVF-PQ d=128, M=16, nlist=4096, same builder and seeds, the
first `--nq` queries of the first timed batch) in torch on the device and counts, per query, the phase-B entries
each bound passes:

  fp16       operands fp16(sa a), fp16(-2 sb r), sa / sb powers of two, eps = 2^-10 |a| R (the fp16 kernel)
  int8       qa = rn(a / s_a), s_a = amax / 127; qr = rn(r / s_b), one s_b for the codebook; exact integer
             products; eps = 2 * 1.05 (|da| R + (|a| + |da|) D) + the bias rounding (kernels_pqtc.cu, the int8 kernel)
  int8_per_m the same with one scale per sub-quantiser folded into the query rows (the alternative when the global
             scale is too coarse); eps = 2 * 1.05 (|a| D_m + |da'| Q)

plus `exact`: the phase-B entries whose exact score is <= B_q (what any filter must pass).  Each also gets the fp32
noise term 2^-17 Z of the reference evaluation.  Then it times `--search-steps` searches of the whole batch and reports
the stage times and recall@10 of the shipped kernel.  Prints JSON lines; nothing is written to the tree.
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


def stats(counts):
    import numpy as np
    c = np.asarray(counts, np.float64)
    return {"mean": float(c.mean()), "p99": float(np.percentile(c, 99)), "max": float(c.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=3, help="bench.py --warmup: its first timed batch is seed 4321 + warmup")
    ap.add_argument("--kprime", type=int, default=400)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--search-steps", type=int, default=3)
    a = ap.parse_args()

    import numpy as np
    import torch
    import bench
    from vearch_b200 import synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_pqtc_int8.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    wl = dict(bench.WORKLOADS["ivfpq_10m"])
    t0 = time.time()
    idx, params, _ = bench.build_index(wl, a.n, 0, 0, "sift")
    nprobe = min(a.nprobe, params["ncentroids"])
    xq_full = synth.sift_like_torch(wl["nq"], wl["d"], seed=4321 + a.warmup, device=dev)
    xq_host = xq_full[:a.nq].cpu().numpy()
    cdis, keys = idx.coarse_search(xq_host, nprobe)
    cent = torch.from_numpy(idx.get_centroids()).to(dev)
    pq = torch.from_numpy(idx.get_pq_centroids()).to(dev)  # [M][256][dsub]
    off, codes, _ = idx.export_lists()
    codes = torch.from_numpy(codes).to(dev)
    M, _, dsub = pq.shape
    d = M * dsub
    kp = a.kprime
    f64 = torch.float64
    xq = torch.from_numpy(xq_host).to(dev).double()
    cdis = torch.from_numpy(cdis).to(dev).double()
    keys_t = torch.from_numpy(keys).to(dev)
    lens = torch.from_numpy(np.diff(off)).to(dev)

    # ---- codebook-side tables ----
    pq64 = pq.double()
    nrm = (pq64 ** 2).sum(-1)                                # [M][256]
    R2 = float(nrm.max(1).values.sum())
    R = R2 ** 0.5
    cbmax = float(pq64.abs().max())
    # fp16: power-of-two scale into [2^13, 2^14), codebook pre-scaled by -2
    sb16 = 2.0 ** (13 - np.floor(np.log2(cbmax)))
    cb16 = (-2.0 * sb16 * pq64).half().double()
    # int8, one scale
    s_b = np.float32(cbmax) / np.float32(127.0)
    s_b = float(s_b)
    qr = torch.clamp(torch.round(pq64 / s_b), -127, 127)
    D = float(((pq64 - s_b * qr) ** 2).sum(-1).max(1).values.sum()) ** 0.5
    # int8, one scale per sub-quantiser
    s_m = pq64.abs().amax((1, 2)) / 127.0                    # [M]
    qr_m = torch.clamp(torch.round(pq64 / s_m[:, None, None]), -127, 127)
    D_m = float(((pq64 - s_m[:, None, None] * qr_m) ** 2).sum(-1).max(1).values.sum()) ** 0.5
    Q_m = float((qr_m ** 2).sum(-1).max(1).values.sum()) ** 0.5
    s_m_cols = s_m.repeat_interleave(dsub)                   # [d]

    def decode(l, tab):
        o0, o1 = int(off[l]), int(off[l + 1])
        c = codes[o0:o1].long()                              # [len][M]
        return tab[torch.arange(M, device=dev)[None, :], c].reshape(o1 - o0, d)

    # ---- phase A plan and bound B_q (bench's index: pa_max = min(nprobe - 1, 8), target 4 k') ----
    pa_max = min(nprobe - 1, 8)
    ll = torch.where(keys_t >= 0, lens[keys_t.clamp(min=0)], torch.zeros_like(keys_t))
    reached = torch.cumsum(ll[:, :pa_max], 1) >= 4 * kp
    P = torch.where(reached.any(1), reached.int().argmax(1) + 1, torch.full_like(reached[:, 0], pa_max, dtype=torch.long))
    in_a = torch.arange(nprobe, device=dev)[None, :] < P[:, None]
    flat_l = keys_t.reshape(-1)
    order = torch.argsort(flat_l)
    sorted_l = flat_l[order]
    uniq, counts = torch.unique_consecutive(sorted_l, return_counts=True)
    starts = torch.cumsum(counts, 0) - counts
    groups = [(int(l), order[int(s):int(s) + int(c)]) for l, s, c in zip(uniq.tolist(), starts.tolist(), counts.tolist())
              if l >= 0]
    a_scores = [[] for _ in range(a.nq)]
    for l, j in groups:
        q, p = j // nprobe, j % nprobe
        sel = in_a[q, p]
        if not bool(sel.any()):
            continue
        q = q[sel]
        r = decode(l, pq64)
        A = xq[q] - cent[l].double()
        sc = cdis[q, p[sel]][:, None] + (r * r).sum(1)[None, :] - 2.0 * A @ r.T
        for i, qq in enumerate(q.tolist()):
            a_scores[qq].append(sc[i])
    B = torch.empty(a.nq, dtype=f64, device=dev)
    for qq in range(a.nq):
        s = torch.cat(a_scores[qq]) if a_scores[qq] else torch.empty(0, dtype=f64, device=dev)
        B[qq] = torch.kthvalue(s, kp).values if s.numel() >= kp else float("inf")
    del a_scores

    # ---- phase B: entries each bound passes ----
    names = ("exact", "fp16", "int8", "int8_per_m")
    cnt = {k: torch.zeros(a.nq, dtype=torch.long, device=dev) for k in names}
    entries_b = torch.zeros(a.nq, dtype=torch.long, device=dev)
    for l, j in groups:
        q, p = j // nprobe, j % nprobe
        sel = ~in_a[q, p]
        if not bool(sel.any()):
            continue
        q, p = q[sel], p[sel]
        r = decode(l, pq64)
        ne = (r * r).sum(1)[None, :]
        c = cent[l].double()
        A = xq[q] - c
        dis0 = cdis[q, p][:, None]
        Bq = B[q][:, None]
        na = A.norm(dim=1, keepdim=True)
        nx = xq[q].norm(dim=1, keepdim=True)
        Z = dis0.abs() + R2 + 2.0 * (nx + float(c.norm())) * R
        noise = 2.0 ** -17 * Z
        amax = A.abs().amax(1, keepdim=True)
        exact = ne - 2.0 * A @ r.T
        thr0 = Bq - dis0
        entries_b.index_add_(0, q, torch.full_like(q, r.shape[0]))
        cnt["exact"].index_add_(0, q, (exact <= thr0).sum(1))
        # fp16
        sa16 = torch.exp2(13 - torch.floor(torch.log2(amax)))
        a16 = (sa16 * A).half().double()
        acc = a16 @ decode(l, cb16).T
        c16 = sa16 * sb16
        eps16 = 1.05 * 2.0 ** -10 * na * R + noise
        cnt["fp16"].index_add_(0, q, (acc + c16 * ne <= c16 * (thr0 + eps16)).sum(1))
        # int8, one scale
        s_a = amax / 127.0
        qa = torch.clamp(torch.round(A / s_a), -127, 127)
        da = (A - s_a * qa).norm(dim=1, keepdim=True)
        acc = qa @ decode(l, qr).T
        eps8 = 2.0 * 1.05 * (da * R + (na + da) * D) + noise + 2.0 * s_a * s_b + 2.0 ** -22 * R2
        cnt["int8"].index_add_(0, q, (ne - 2.0 * s_a * s_b * acc <= thr0 + eps8).sum(1))
        # int8, one scale per sub-quantiser folded into the rows
        Ap = A * s_m_cols[None, :]
        s_ap = Ap.abs().amax(1, keepdim=True) / 127.0
        qap = torch.clamp(torch.round(Ap / s_ap), -127, 127)
        dap = (Ap - s_ap * qap).norm(dim=1, keepdim=True)
        acc = qap @ decode(l, qr_m).T
        eps8m = 2.0 * 1.05 * (na * D_m + dap * Q_m) + noise + 2.0 * s_ap + 2.0 ** -22 * R2
        cnt["int8_per_m"].index_add_(0, q, (ne - 2.0 * s_ap * acc <= thr0 + eps8m).sum(1))
    out = {"workload": "pqtc_int8_bound", "n": a.n, "nq": a.nq, "kprime": kp, "nprobe": nprobe,
           "phase_b_entries_per_query": float(entries_b.double().mean()),
           "codebook": {"R": R, "cbmax": cbmax, "D_int8": D, "D_int8_per_m": D_m, "Q_per_m": Q_m},
           "candidate_cap": max(2048, min(8192, 1 << (8 * kp - 1).bit_length())),
           "passed_per_query": {k: stats(v.cpu().numpy()) for k, v in cnt.items()},
           "gpu": gpu_conditions(), "setup_s": round(time.time() - t0, 1)}
    print(json.dumps(out), flush=True)

    # ---- the shipped kernel on the whole batch: stage times and recall@10 ----
    k = 10
    sp = {"nprobe": nprobe, "recall_num": kp}
    _, gt = idx.search(xq_host, k, brute_force=True)
    for _ in range(2):
        idx.search_device(xq_full, k, params=sp)
    torch.cuda.synchronize()
    idx.set_scan_timing(True)
    idx.stage_times()
    for _ in range(a.search_steps):
        idx.search_device(xq_full, k, params=sp)
    torch.cuda.synchronize()
    stages = {kk: v / a.search_steps for kk, v in idx.stage_times().items()}
    idx.set_scan_timing(False)
    _, ids = idx.search(xq_host, k, params=sp)
    r1, r10 = bench.recall_stats(ids, gt)
    print(json.dumps({"workload": "pqtc_int8_search", "nq": int(xq_full.shape[0]), "stages_ms": stages,
                      "scan_kernel": idx.last_scan_kernel, "recall@10": r10, "recall@10_1nn": r1,
                      "gpu": gpu_conditions()}), flush=True)
    idx.close()


if __name__ == "__main__":
    main()
