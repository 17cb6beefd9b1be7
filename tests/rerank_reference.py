"""What the two-pass exact re-rank must show through its test hooks (index.debug_rerank, index.debug_shadow_rows),
derived from the numpy restatement of its bound (test_rerank_prefilter_cpu.py): rows padded as the raw store pads them,
both fp32 sums with each FMA rounded once, the shadow rows' rule, the fp32 brackets each pass-1 interval must fall in,
the k-th bound and survivor count pass 1 implies, and candidate sets whose survivor count is known in advance.
Self-checked without a GPU by test_rerank_reference_cpu.py."""
import numpy as np

import test_rerank_prefilter_cpu as P
import topk_reference as R

F32, F64 = np.float32, np.float64
INF = float("inf")
BOUNDED, WITHHELD, UNBOUNDED, DEAD = 0, 1, 2, 3  # index.GammaIndex.RR_*
ORD_DEAD, ORD_NOBOUND = 0xFFFFFFFF, 0xFFFFFFFE


def pad4(x):
    """rows as the raw store holds them: d fp32 values zero padded to dpad = round_up(d, 4)"""
    x = np.asarray(x, F32)
    out = np.zeros((len(x), (x.shape[1] + 3) // 4 * 4), F32)
    out[:, :x.shape[1]] = x
    return out


def f32_down(v):
    """the largest float32 <= v (fp64)"""
    v = np.asarray(v, F64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = v.astype(F32)
        return np.where(f.astype(F64) > v, np.nextafter(f, F32(-INF)), f)


def f32_up(v):
    """the smallest float32 >= v (fp64)"""
    v = np.asarray(v, F64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = v.astype(F32)
        return np.where(f.astype(F64) < v, np.nextafter(f, F32(INF)), f)


def fma32(a, b, c):
    """fmaf: a b + c rounded once to fp32.  The product is exact in fp64; the sum is rounded to odd there (an inexact
    fp64 sum with an even last bit moves one ulp towards the exact value), which makes the rounding to fp32 the single
    correct one.  A plain fp64 sum rounds twice and misses fmaf's result whenever a b lies on an fp32 midpoint and c is
    too small to show in fp64 (a query of 2^-64 against rows near 1): comparing the device's intervals end for end
    needs the single rounding, which test_rerank_prefilter_cpu.fma32 (a containment check) does without."""
    p, c = a.astype(F64) * b.astype(F64), np.asarray(c, F64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        fix = np.isfinite(s) & (err != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(err > 0, INF, -INF)), s)
    return s.astype(F32)


def pass1_sum(xq, qy, s, metric):
    """[nq, n] pass 1's fp32 sums, as test_rerank_prefilter_cpu.pass1_sum orders them, each FMA rounded once"""
    nq, n, cols16 = len(xq), len(qy), qy.shape[1]
    q = np.zeros((nq, cols16), F32)
    q[:, :xq.shape[1]] = xq
    qf = qy.astype(F32)
    lanes = np.zeros((8, nq, n), F32)
    for c in range(cols16 // 16):
        for i in range(16):
            col = 16 * c + i
            if metric == R.METRIC_L2:
                t = fma32(-s[None, :], qf[None, :, col], q[:, col][:, None])
                lanes[c % 8] = fma32(t, t, lanes[c % 8])
            else:
                lanes[c % 8] = fma32(q[:, col][:, None], qf[None, :, col], lanes[c % 8])
    for off in (1, 2, 4):
        lanes = (lanes + lanes[np.arange(8) ^ off]).astype(F32)
    return lanes[0]


def direct_fp32(xq, y, metric):
    """[nq, n] the one-pass kernel's scores (rr_exact_scores), as test_rerank_prefilter_cpu.direct_fp32 orders them,
    each FMA rounded once"""
    nq, n, d = len(xq), len(y), y.shape[1]
    acc = np.zeros((32, 4, nq, n), F32)
    for c in range(d // 4):
        for j in range(4):
            a, b = xq[:, 4 * c + j][:, None], y[None, :, 4 * c + j]
            if metric == R.METRIC_L2:
                t = (b - a).astype(F32)
                acc[c % 32, j] = fma32(t, t, acc[c % 32, j])
            else:
                acc[c % 32, j] = fma32(b, a, acc[c % 32, j])
    dis = ((acc[:, 0] + acc[:, 1]).astype(F32) + (acc[:, 2] + acc[:, 3]).astype(F32)).astype(F32)
    for off in (16, 8, 4, 2, 1):
        dis = (dis + dis[np.arange(32) ^ off]).astype(F32)
    return dis[0]


def shadow_mismatch(y, qy, s, e, nrm, ulps=4):
    """None if the shadow rows (qy, s, e, nrm) of the padded rows y follow the rule, else what breaks it: qy and s
    byte-equal to encode(); e and nrm at or above |y - s qy| and |s qy| in fp64 and within `ulps` fp32 ulps of them;
    a row whose scale is zero or not finite has e = nrm = inf"""
    wq, ws, _, _ = P.encode(y)
    if qy.shape != wq.shape:
        return f"shadow width {qy.shape[1]}, encode() gives {wq.shape[1]}"
    bad = np.nonzero((qy != wq).any(1) | (s.view(np.uint32) != ws.view(np.uint32)))[0]
    if len(bad):
        return f"rows {bad[:8].tolist()}: qy or s differ from encode()"
    ok = ws > 0
    y64, s64, q64 = y.astype(F64), ws.astype(F64)[:, None], wq[:, :y.shape[1]].astype(F64)
    e64 = np.sqrt(((y64 - s64 * q64) ** 2).sum(1))
    n64 = ws.astype(F64) * np.sqrt((q64 * q64).sum(1))
    if not (np.all(e[~ok] == INF) and np.all(nrm[~ok] == INF)):
        rows = np.nonzero(~ok & ((e != INF) | (nrm != INF)))[0][:8].tolist()
        return f"rows {rows}: unbounded rows need e = nrm = inf"
    for name, got, want in (("e", e, e64), ("nrm", nrm, n64)):
        g, w = got[ok].astype(F64), want[ok]
        top = f32_up(w)
        for _ in range(ulps - 1):
            top = np.nextafter(top, F32(INF))
        wrong = np.nonzero((g < w) | (g > top))[0]
        if len(wrong):
            i = np.nonzero(ok)[0][wrong[0]]
            return (f"{len(wrong)} rows' {name} not in [fp64, +{ulps} ulps]; first: row {i}, {g[wrong[0]]!r} vs "
                    f"{w[wrong[0]]!r}")
    return None


def brackets(xq, qy, s, e, nrm, metric, rel=2.0 ** -38):
    """[nq, n] the fp32 ends pass 1 must give for padded queries xq against shadow rows (qy, s, e, nrm): lo in
    [lo_min, lo_max] and hi in [hi_min, hi_max], the restated fp64 ends moved by rel times the larger end's magnitude
    (the device rounds every fp64 step outwards, the restatement to nearest) and rounded as the device rounds them,
    lo down and hi up; and `bounded` as pass 1 decides it"""
    st = pass1_sum(xq, qy, s, metric)
    lo, hi, bounded = P.interval(xq, st, s, e, nrm, xq.shape[1], metric)
    with np.errstate(invalid="ignore", over="ignore"):
        tol = rel * np.maximum(np.abs(lo), np.abs(hi))
        return f32_down(lo - tol), f32_down(lo + tol), f32_up(hi - tol), f32_up(hi + tol), bounded


def pass1_ords(lo, hi, state, metric):
    """the ordinals pass 1 ranks by, from debug_rerank's intervals [nq, n]: (best ordinal a candidate can have, worst
    ordinal of one that bounds the k-th result); dead: both ORD_DEAD; unbounded: 0 and ORD_DEAD; withheld: hi
    ORD_DEAD"""
    best, worst = (lo, hi) if metric == R.METRIC_L2 else (hi, lo)
    with np.errstate(invalid="ignore"):
        olo = np.where(state == BOUNDED, R.score2ord(np.where(state == BOUNDED, best, 0).astype(F32), metric), 0)
        olo = np.where(state == WITHHELD, R.score2ord(np.where(state == WITHHELD, best, 0).astype(F32), metric), olo)
        ohi = R.score2ord(np.where(state == BOUNDED, worst, 0).astype(F32), metric)
        ohi = np.where(state == BOUNDED, ohi, ORD_DEAD)
    olo = np.where(state == DEAD, ORD_DEAD, olo)
    return olo.astype(np.uint64), ohi.astype(np.uint64)


def expected_survivors(lo, hi, state, k, metric):
    """[nq] the candidates pass 2 must read: B = the k-th smallest worst ordinal (ORD_NOBOUND when fewer than k
    candidates bound it), then every candidate whose best ordinal is <= B"""
    olo, ohi = pass1_ords(lo, hi, state, metric)
    kk = min(k, ohi.shape[1])
    B = np.sort(ohi, axis=1)[:, kk - 1]
    B = np.where(B == ORD_DEAD, ORD_NOBOUND, B)
    return (olo <= B[:, None]).sum(1)


def copies_and_far(q, db, near, m, nfar, metric, rng):
    """candidate vids of one query: m copies of one row (vids `near`, all holding the same integer row next to the
    query) then nfar rows of db whose exact scores are far enough behind the copies' that their intervals cannot reach
    the copies' (L2: more than 16 times the copies' score plus 64; IP: below half of it), shuffled.  With k <= m the
    copies tie at the k-th score, so exactly the m copies survive pass 1."""
    s = R.exact_scores(q[None], db, metric)[0]
    s_near = s[near[0]]
    assert np.all(s[near] == s_near)
    far = np.nonzero(s > 16 * s_near + 64 if metric == R.METRIC_L2 else s < s_near / 2)[0]
    far = np.setdiff1d(far, near)
    cand = np.concatenate([near[:m], rng.choice(far, nfar, replace=False)])
    return rng.permutation(cand)
