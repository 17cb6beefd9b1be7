"""Float-accuracy contract of the search paths (test infrastructure only).

On float data no two evaluation orders agree bit for bit, so a kernel is checked against fp64 scores of its fp32
inputs within a rigorous bound on the error of its arithmetic form.  Let u = 2^-24.  Each margin bounds
|fp32 result - exact value| for one form, for any summation order:

  direct L2   t = fl(x_j - y_j), t^2 accumulated       1.01 (d + 3) u sum (x_j - y_j)^2
  direct IP   x_j y_j accumulated                      1.01 (d + 1) u sum |x_j y_j|
  3xTF32 dot  wgmma, hi*hi + hi*lo + lo*hi             (48 + C_TC (d + 4)) u sum |a_j b_j|
  expanded L2 |a|^2 + |b|^2 - 2 a.b over a, b          2 dot margin + (d + 2) u (|a|^2 + |b|^2) + u score

The 3xTF32 dot has two parts.  Representation: a = hi + lo exactly (hi keeps 10 explicit mantissa bits, so
|lo| <= 2^-10 |a|), but wgmma reads lo as TF32 too, dropping its low bits (|lo - lo'| <= 2^-10 |lo| <= 2^-20 |a|), and
lo*lo is never formed (|lo_a lo_b| <= 2^-20 |a b|): the three products miss a_j b_j by at most 3 * 2^-20 = 48 u of
|a_j b_j|, whatever d.  Accumulation: the products and their fp32 sums, C_TC (d + 4) u.  Below d ~ 8 the first part
dominates; without it dist_tc_kernel exceeded the margin at d = 1 by 1.5 %.
Hopper does not document its wgmma fp32 accumulation as round-to-nearest, so C_TC is a model constant, checked on the
GPU element-wise against the exact kernel's inputs (tests/test_gpu_float_accuracy.py,
tests/test_gpu_float_shape_limits.py from d = 1 to 4096).

The fp64 reference uses the direct form: fp32 differences and products are exact or within 2^-53 relative in fp64,
so its error is ~2^-29 of the fp32 margins; scores64 asserts it is below 1/1000 of them.

check_selection states what a returned top-k must satisfy, whatever kernel produced it, given fp64 scores f and
per-candidate selection margins m over the valid candidates:
  1. min(k, #valid) results, ordered by the returned score bits (L2 ascending, IP descending), ties by id as the
     engine's decoder lists them; empty slots last;
  2. every returned score within the direct-form margin of the fp64 score of its id (every path re-scores its
     winners in the direct form);
  3. no candidate left out is certainly better than one returned: max_K (f - m) <= min_notK (f + m) under L2,
     mirrored under IP;
  4. with a score window, a candidate whose f lies within m of an edge may fall on either side; every other one
     is on its correct side.
With every m = 0 this is the key-exact set check.
"""
import numpy as np

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)
U = 2.0 ** -24
U64 = 2.0 ** -53
C_TC = 4.0
METRIC_IP, METRIC_L2 = 0, 1


# ---- data regimes -----------------------------------------------------------------------------------------------------
def clustered(n, d, rng, centres, spread=0.35):
    return centres[rng.integers(0, len(centres), n)] + spread * rng.standard_normal((n, d))


def regime(name, n, d, nq, seed):
    """(db, xq) float32 of one ill-conditioned regime; seeded"""
    rng = np.random.default_rng(seed)
    if name.startswith("offset"):  # clustered N(0,1) mixture plus a common offset: offset100, offset1000
        off = float(name[6:])
        c = rng.standard_normal((64, d))
        db, xq = clustered(n, d, rng, c) + off, clustered(nq, d, rng, c) + off
    elif name == "sift_float":
        from vearch_b200 import synth
        db, xq = synth.sift_like(n, d, seed=seed, rounded=False), synth.sift_like(nq, d, seed=seed + 1, rounded=False)
    elif name in ("scaled_hi", "scaled_lo"):  # embed_like x 2^+-40
        from vearch_b200 import synth
        sc = 2.0 ** (40 if name == "scaled_hi" else -40)
        db = synth.embed_like(n, d, seed=seed).astype(np.float64) * sc
        xq = synth.embed_like(nq, d, seed=seed + 1).astype(np.float64) * sc
    elif name == "wide":  # per-dimension scale 2^U(-10, 10)
        c = rng.standard_normal((64, d))
        sc = 2.0 ** rng.uniform(-10, 10, d)
        db, xq = clustered(n, d, rng, c) * sc, clustered(nq, d, rng, c) * sc
    elif name == "near_dup":  # groups of 8 rows ~2^-20 apart (relative): ties within the margin are dense
        c = rng.standard_normal((64, d))
        base = clustered((n + 7) // 8, d, rng, c)
        db = np.repeat(base, 8, axis=0)[:n]
        db = db * (1 + 2.0 ** -20 * rng.standard_normal(db.shape))
        xq = base[rng.integers(0, len(base), nq)] * (1 + 2.0 ** -18 * rng.standard_normal((nq, d)))
    else:
        raise ValueError(name)
    return np.ascontiguousarray(db, F32), np.ascontiguousarray(xq, F32)


REGIMES = ["offset100", "offset1000", "sift_float", "scaled_hi", "scaled_lo", "wide", "near_dup"]


# ---- fp64 scores ------------------------------------------------------------------------------------------------------
def scores64(x, y, metric):
    """(f, absdot): fp64 direct-form scores of fp32 rows x [nq, d] against y [n, d], and sum_j |x_j y_j|"""
    x64, y64 = np.asarray(x, np.float64), np.asarray(y, np.float64)
    absdot = np.abs(x64) @ np.abs(y64).T
    if metric == METRIC_IP:
        f = x64 @ y64.T
        err = 1.01 * x.shape[1] * U64 * absdot
        assert np.all(err <= 1e-3 * ip_direct_margin(absdot, x.shape[1]))
        return f, absdot
    f = np.empty((len(x64), len(y64)))
    for q in range(len(x64)):
        t = y64 - x64[q]
        f[q] = np.einsum("ij,ij->i", t, t)
    err = 1.01 * (x.shape[1] + 3) * U64 * f
    assert np.all(err <= 1e-3 * l2_direct_margin(f, x.shape[1]))
    return f, absdot


# ---- margins ----------------------------------------------------------------------------------------------------------
def l2_direct_margin(f, d):
    return 1.01 * (d + 3) * U * np.asarray(f)


def ip_direct_margin(absdot, d):
    return 1.01 * (d + 1) * U * np.asarray(absdot)


def direct_margin(f, absdot, d, metric):
    return l2_direct_margin(f, d) if metric == METRIC_L2 else ip_direct_margin(absdot, d)


TF32_SPLIT = 3 * 2.0 ** -20  # the split's representation error per product, relative to |a_j b_j| (see above)


def tc_dot_margin(absdot, d, c_tc=C_TC):
    return (TF32_SPLIT + c_tc * (d + 4) * U) * np.asarray(absdot)


def expanded_l2_margin(absdot, na, nb, score, d, c_tc=C_TC):
    """|a|^2 + |b|^2 - 2 a.b over fp32 operands a, b (na, nb = |a|^2, |b|^2; absdot = sum |a_j b_j|)"""
    return 2 * tc_dot_margin(absdot, d, c_tc) + (d + 2) * U * (na + nb) + U * np.abs(score)


def shifted_l2_margin(absdot, na, nb, score, d, c_tc=C_TC):
    """the expanded form over a = fl(x - s), b = fl(y - s): the operands' own rounding (|a - a'| <= u |a|) adds at most
    u (f + 2 (|a|^2 + |b|^2)) to the score; the 1.01 covers the second-order terms"""
    return 1.01 * (expanded_l2_margin(absdot, na, nb, score, d, c_tc) + U * (np.abs(score) + 2 * (na + nb)))


def shifted_operands(x, y, s):
    """(|a|^2 [nx, 1], |b|^2 [1, ny], sum |a_j b_j| [nx, ny]) of a = x - s, b = y - s in fp64"""
    a = np.asarray(x, np.float64) - np.asarray(s, np.float64)
    b = np.asarray(y, np.float64) - np.asarray(s, np.float64)
    return (a * a).sum(1)[:, None], (b * b).sum(1)[None, :], np.abs(a) @ np.abs(b).T


# ---- selection --------------------------------------------------------------------------------------------------------
def f2ord(s):
    b = np.ascontiguousarray(s, F32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def check_selection(scores, ids, cand, f, m, md, k, metric, min_score=-FLT_MAX, max_score=FLT_MAX, ip_ties_desc=True):
    """One query's returned (scores, ids) against its valid candidates cand (ids), fp64 scores f, selection margins m
    and direct-form margins md (ip_ties_desc: equal IP scores list the larger id first, as the search decoder does;
    False for the raw key order of the coarse quantiser).  Returns None if the contract holds, else (reason, ids missing, excess) where ids
    missing counts the fp64 top-k ids (inside the window) not returned and excess is the worst amount by which rule 3
    is broken (0 if it holds)."""
    scores, ids = np.asarray(scores, F32), np.asarray(ids, np.int64)
    cand, f, m, md = (np.asarray(a) for a in (cand, f, m, md))
    l2 = metric == METRIC_L2
    live = ids >= 0
    n = int(live.sum())
    reasons = []
    if not np.all(live[:n]) or not np.all(scores[n:] == F32(FLT_MAX if l2 else -FLT_MAX)):
        reasons.append("empty slots not last")
    gs, gi = scores[:n], ids[:n]
    o = f2ord(gs).astype(np.int64)
    if l2:
        ok = np.all((o[1:] > o[:-1]) | ((o[1:] == o[:-1]) & (gi[1:] > gi[:-1])))
    else:
        tie = (gi[1:] < gi[:-1]) if ip_ties_desc else (gi[1:] > gi[:-1])
        ok = np.all((o[1:] < o[:-1]) | ((o[1:] == o[:-1]) & tie))
    if not ok:
        reasons.append("order")
    # the window: certainly inside, possibly inside
    sure = (f - m >= min_score) & (f + m <= max_score)
    maybe = (f + m >= min_score) & (f - m <= max_score)
    if not (min(k, int(sure.sum())) <= n <= min(k, int(maybe.sum()))):
        reasons.append(f"count {n}, want within [{min(k, int(sure.sum()))}, {min(k, int(maybe.sum()))}]")
    pos = {int(v): i for i, v in enumerate(cand)}
    idx = np.array([pos.get(int(v), -1) for v in gi], np.int64)
    if len(set(gi.tolist())) != n:
        reasons.append("duplicate id")
    if np.any(idx < 0):
        reasons.append(f"id {int(gi[np.argmax(idx < 0)])} is not a valid candidate")
        idx = idx[idx >= 0]
    if len(idx) and np.any(~maybe[idx]):
        reasons.append("a returned id is certainly outside the window")
    err = np.abs(gs[:len(idx)].astype(np.float64) - f[idx]) if len(idx) == n else np.zeros(0)
    if len(err) and np.any(err > md[idx]):
        j = int(np.argmax(err - md[idx]))
        reasons.append(f"score of id {int(gi[j])} off by {err[j]:.3g} > direct margin {md[idx][j]:.3g}")
    inK = np.zeros(len(cand), bool)
    inK[idx] = True
    out = ~inK & sure
    excess = 0.0
    if len(idx) and out.any():
        excess = (np.max(f[idx] - m[idx]) - np.min(f[out] + m[out])) if l2 else \
                 (np.max(f[out] - m[out]) - np.min(f[idx] + m[idx]))
        excess = max(0.0, float(excess))
        if excess > 0:
            reasons.append(f"a candidate left out is better than a returned one by {excess:.3g} beyond the margins")
    if n < k and out.any():
        reasons.append("fewer than k returned while a valid candidate inside the window was left out")
    if not reasons:
        return None
    inw = np.nonzero((f >= min_score) & (f <= max_score))[0]
    top = inw[np.argsort(f[inw] if l2 else -f[inw], kind="stable")[:k]]
    missing = len(set(cand[top].tolist()) - set(gi.tolist()))
    return "; ".join(reasons), missing, excess


def check_all(got, per_query, k, metric, what="", **window):
    """check_selection over every query; per_query(q) -> (cand, f, m, md).  Raises with the number of failing queries,
    fp64 top-k ids missing and the worst excess over the margins."""
    dis, ids = got
    bad, missing, worst, first = 0, 0, 0.0, None
    for q in range(len(ids)):
        r = check_selection(dis[q], ids[q], *per_query(q), k, metric, **window)
        if r is not None:
            bad += 1
            missing += r[1]
            worst = max(worst, r[2])
            first = first or f"query {q}: {r[0]}"
    assert bad == 0, (f"{what}: {bad}/{len(ids)} queries break the float contract; fp64 top-{k} ids missing "
                      f"{missing}/{len(ids) * k}, worst excess over the margins {worst:.4g}; {first}")
