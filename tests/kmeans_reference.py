"""Restatement of one device k-means iteration and the contract of its assignment (test infrastructure only).

The engine's k-means (DESIGN.md K6) trains every coarse quantiser and codebook.  index.debug_kmeans_trace records one
run: the sampled rows, the initial centroids and, per iteration t, each row's label and key score against C_t and the
centroids after the segmented mean, the empty-cluster split and the renormalisation (C_{t+1}).  This module states what
each of those must be, given the state the device itself reached, so that an iteration is checked alone:

  sample   rand_perm(n, seed)[:k mp] when n > k mp (mp = max_points_per_centroid > 0), else every row in order
  init     the sample's rows rand_perm(n_s, seed + 1)[:k], renormalised when spherical; a hot start keeps its own
  mean     orc.kmeans_update(x_s, k, labels_t)                       byte-equal* (members summed in row order)
  split    orc.kmeans_split(hassign, mean, n_s)                      byte-equal* (the same host code)
  norm     orc.kmeans_normalize(split) when spherical, else split    within RENORM_BOUND, else byte-equal
  labels   the assignment contract below, against C_t
(* any NaN equals any NaN: the CPU keeps a NaN's payload and sign through arithmetic, the GPU returns its own NaN.)

Renormalisation bound.  Both sides compute c_j / sqrt(sum c_i^2) in fp32 with correctly rounded sqrt and division; the
reference sums the squares in row order without FMA, normalize_rows_kernel with per-lane fmaf and a warp tree.  Either
sum of d squares is within d u (u = 2^-24, to first order) of the exact one, whatever the order; sqrt, the reciprocal and
the final product add u/2, u and u.  So each side is within (d/2 + 2.5) u of the exact c_j / |c|, and the two differ by at
most (d + 5) u relative; RENORM_BOUND takes 1.02 (d + 5) u |reference|.

Assignment contract of iteration t (rows x_s, centroids C_t, fp64 scores f and margins m of tests/float_contract.py):
  - the margin of the kernel that ran: k < 64 the exact CUDA-core kernel (direct form, direct_margin); k >= 64 the
    3xTF32 tensor-core kernel (expanded_l2_margin under L2, tc_dot_margin under IP);
  - no centroid certainly better than the label: f[l] - m[l] <= min_j (f[j] + m[j]) under L2, mirrored under IP;
  - the key's score is within m[l] of f[l];
  - a centroid identical to a lower one is never the label (identical inputs give identical scores, and ties go to the
    lowest id, as faiss's strict `dis < best` does);
  - a row holding a NaN or an infinity has only non-finite scores (+-inf or NaN, whatever the summation order), so it
    is held to faiss's rule exactly: the first centroid with the best score among those that beat the start value
    (FLT_MAX under L2, -FLT_MAX under IP; a NaN beats nothing), else cluster 0.  Under L2 every such score is +inf or
    NaN, so the row goes to cluster 0; under IP a +inf dot is a valid best score.  Its key score equals that score;
  - no finite row goes to a centroid that holds a NaN or an infinity (its score is NaN or infinite, and a finite
    centroid beats it).
"""
import numpy as np

import float_contract as fc
from oracle import oracle as orc

U = fc.U
TC_MIN_K = 64  # kmeans_device assigns on the tensor cores from k = 64 on


def sample_ids(n, k, mp, seed):
    """the rows a run trains on"""
    if mp > 0 and n > k * mp:
        return orc.rand_perm(n, seed)[:k * mp]
    return np.arange(n, dtype=np.int64)


def init_ids(ns, k, seed):
    """positions in the sample of the initial centroids"""
    return orc.rand_perm(ns, seed + 1)[:k]


def clamp_threshold(param, nlist, default):
    """IvfIndex::training_threshold: the parameter (0: the type's default) clamped as gamma's Indexing() does, a value
    below nlist raised to 39 nlist and one above 256 nlist lowered to it (in 64 bits: 256 nlist passes 2^31 at 2^23)"""
    t = param or default
    return 39 * nlist if t < nlist else min(t, 256 * nlist)


def assign_metric(spherical, l2_assign):
    return fc.METRIC_IP if spherical and not l2_assign else fc.METRIC_L2


def renorm_bound(ref, d):
    return 1.02 * (d + 5) * U * np.abs(np.asarray(ref, np.float64))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    """byte-equal, any NaN equal to any NaN (the CPU propagates a NaN's payload and sign, the GPU returns its own)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(bits(a)[~na], bits(b)[~nb])


def restated_step(xs, k, labels, spherical):
    """(mean, split, norm, splits) of one iteration from the labels the device gave the rows xs"""
    mean, h = orc.kmeans_update(xs, k, np.asarray(labels, np.int64))
    split, _, nsplit = orc.kmeans_split(h, mean, len(xs))
    norm = orc.kmeans_normalize(split) if spherical else split
    return mean, split, norm, nsplit


def check_norm(got, split, d):
    """None, or why the device's renormalisation of split is not within RENORM_BOUND of the reference's"""
    ref = orc.kmeans_normalize(split)
    fin = np.isfinite(ref)
    if not np.array_equal(np.isfinite(got), fin) or not same(got[~fin], ref[~fin]):
        return "renormalised centroids: non-finite entries differ"
    err = np.abs(got[fin].astype(np.float64) - ref[fin])
    bound = renorm_bound(ref[fin], d)
    if np.any(err > bound):
        j = int(np.argmax(err - bound))
        return f"renormalised centroid entry off by {err[j]:.3g} > bound {bound[j]:.3g}"
    return None


def margins(xs, cent, metric, k=None):
    """(f, m) fp64 scores and selection margins [n, len(cent)] of the kernel kmeans_device runs for k centroids
    (default len(cent); cent may be the finite subset of a run's centroids)"""
    k = len(cent) if k is None else k
    d = cent.shape[1]
    f, absdot = fc.scores64(xs, cent, metric)
    if k < TC_MIN_K:
        return f, fc.direct_margin(f, absdot, d, metric)
    if metric == fc.METRIC_IP:
        return f, fc.tc_dot_margin(absdot, d)
    x64, c64 = np.asarray(xs, np.float64), np.asarray(cent, np.float64)
    na, nb = (x64 * x64).sum(1)[:, None], (c64 * c64).sum(1)[None, :]
    return f, fc.expanded_l2_margin(absdot, na, nb, f, d)


def scores_exact(xs, cent, metric):
    """fp64 direct-form scores [n, k] of fp32 rows against fp32 centroids with IEEE infinities and NaN (no margin
    bookkeeping: for the rows holding a NaN or an infinity, whose every score is non-finite and so exact)"""
    x64, c64 = np.asarray(xs, np.float64)[:, None, :], np.asarray(cent, np.float64)[None, :, :]
    with np.errstate(all="ignore"):
        return ((c64 - x64) ** 2).sum(2) if metric == fc.METRIC_L2 else (c64 * x64).sum(2)


def restated_label(f, metric):
    """faiss's assignment of a row with scores f: the first centroid with the best score among those beating the start
    value FLT_MAX (-FLT_MAX under IP), else 0"""
    ok = f < fc.FLT_MAX if metric == fc.METRIC_L2 else f > -fc.FLT_MAX  # a NaN beats nothing
    if not ok.any():
        return 0
    best = f[ok].min() if metric == fc.METRIC_L2 else f[ok].max()
    return int(np.nonzero(ok & (f == best))[0][0])


def check_assignment(xs, cent, labels, scores, metric):
    """None if iteration's labels / key scores meet the contract against centroids cent, else the first reason"""
    xs, cent = np.asarray(xs, np.float32), np.asarray(cent, np.float32)
    labels, scores = np.asarray(labels, np.int64), np.asarray(scores, np.float32)
    n, k = len(xs), len(cent)
    if labels.min(initial=0) < 0 or labels.max(initial=0) >= k:
        return "label out of range"
    row_ok = np.isfinite(xs).all(1)
    cen_ok = np.isfinite(cent).all(1)
    bad_rows = np.nonzero(~row_ok)[0]
    if len(bad_rows):
        fb = scores_exact(xs[bad_rows], cent, metric)
        for r, f in zip(bad_rows, fb):
            want = restated_label(f, metric)
            if labels[r] != want:
                return f"non-finite row {int(r)}: label {int(labels[r])}, faiss's rule gives {want}"
            beats = f[want] < fc.FLT_MAX if metric == fc.METRIC_L2 else f[want] > -fc.FLT_MAX
            if beats and scores[r] != f[want]:
                return f"non-finite row {int(r)}: key score {scores[r]!r}, want {f[want]!r}"
    # a centroid identical to a lower one: the lowest of them takes the ties
    _, first = np.unique(bits(cent), axis=0, return_index=True)
    twin = np.ones(k, bool)
    twin[first] = False
    rows = np.nonzero(row_ok)[0]
    if len(rows) and np.any(twin[labels[rows]]):
        return f"row {int(rows[np.argmax(twin[labels[rows]])])} labelled with a duplicate of a lower centroid"
    if not cen_ok.any():
        return None if np.all(labels == 0) else "no finite centroid, yet a row left cluster 0"
    if len(rows) and np.any(~cen_ok[labels[rows]]):
        return f"finite row {int(rows[np.argmax(~cen_ok[labels[rows]])])} labelled with a non-finite centroid"
    cols = np.nonzero(cen_ok)[0]
    for r0 in range(0, len(rows), 4096):
        rr = rows[r0:r0 + 4096]
        f, m = margins(xs[rr], cent[cols], metric, k)
        pos = np.searchsorted(cols, labels[rr])
        fl, ml = f[np.arange(len(rr)), pos], m[np.arange(len(rr)), pos]
        if metric == fc.METRIC_L2:
            excess = (fl - ml) - (f + m).min(1)
        else:
            excess = (f - m).max(1) - (fl + ml)
        if np.any(excess > 0):
            i = int(np.argmax(excess))
            return (f"row {int(rr[i])}: label {int(labels[rr[i]])} while a centroid is better by {excess[i]:.4g} "
                    f"beyond the margins")
        err = np.abs(scores[rr].astype(np.float64) - fl)
        if np.any(err > ml):
            i = int(np.argmax(err - ml))
            return f"row {int(rr[i])}: key score {scores[rr[i]]!r} off by {err[i]:.3g} > margin {ml[i]:.3g}"
    return None


def check_trace(x, k, tr, seed=1234, spherical=False, l2_assign=False, mp=256, init=None):
    """Every step of a traced run (index.debug_kmeans_trace) against the restatement; raises AssertionError with the
    first iteration and step that breaks.  Returns the number of splits seen."""
    x = np.asarray(x, np.float32)
    n, d = x.shape
    metric = assign_metric(spherical, l2_assign)
    sid = sample_ids(n, k, mp, seed)
    assert np.array_equal(tr["sample"], sid), "sampled rows"
    xs = x[sid]
    if init is not None:
        assert same(tr["init"], init), "hot start did not keep its centroids"
    else:
        c0 = xs[init_ids(len(xs), k, seed)]
        if spherical:
            r = check_norm(tr["init"], c0, d)
            assert r is None, f"initial centroids: {r}"
        else:
            assert same(tr["init"], c0), "initial centroids"
    splits = 0
    cent = tr["init"]
    for t in range(len(tr["labels"])):
        r = check_assignment(xs, cent, tr["labels"][t], tr["scores"][t], metric)
        assert r is None, f"iteration {t}: {r}"
        mean, split, _, ns = restated_step(xs, k, tr["labels"][t], spherical)
        splits += ns
        assert same(tr["mean"][t], mean), f"iteration {t}: segmented mean"
        assert same(tr["split"][t], split), f"iteration {t}: split"
        if spherical:
            r = check_norm(tr["norm"][t], tr["split"][t], d)
            assert r is None, f"iteration {t}: {r}"
        else:
            assert same(tr["norm"][t], tr["split"][t]), f"iteration {t}: renormalised"
        cent = tr["norm"][t]
    return splits


def gap_excess(xs, cent, labels, metric):
    """how far the runner-up of each row is from being certainly worse than its label (> 0: an ambiguous row); the max
    over the rows.  Unambiguous data keeps this below 0 at every iteration."""
    f, m = margins(np.asarray(xs, np.float32), np.asarray(cent, np.float32), metric)
    idx = np.arange(len(f))
    fl, ml = f[idx, labels], m[idx, labels]
    f2, m2 = f.copy(), m.copy()
    f2[idx, labels] = np.inf if metric == fc.METRIC_L2 else -np.inf
    if metric == fc.METRIC_L2:
        return float(np.max((fl + ml) - (f2 - m2).min(1)))
    return float(np.max((f2 + m2).max(1) - (fl - ml)))
