"""The bound of the two-pass exact re-rank, restated in numpy (kernels_ivfpq.cu: shadow_encode_kernel,
rerank_prefilter_kernel pass 1).

A row y is stored as int8 qy = rn(y / s), s = fl(max|y| / 127), with e >= |y - s qy| and nrm >= |s qy|.  Pass 1 sums
the query against s qy in fp32 (8 lanes x 16 columns, then an xor tree) and widens that sum into an interval [lo, hi]
which must hold the score the one-pass kernel computes from the fp32 row: its direct form, lane l summing the float4
columns l, l + 32, ... into four FMA accumulators, then (a0 + a1) + (a2 + a3) and an xor-shuffle tree.  Both fp32 sums
are emulated here (each FMA exact in fp64, then rounded to fp32), on every float_contract regime, both metrics, and
rows that stress the encoder: zero rows, one dominant component, scales 2^30, 2^-30 and 2^-64.  The kernel rounds every
fp64 step of the interval outwards; the restatement widens its fp64 result by 2^-40 instead."""
import numpy as np
import pytest

import float_contract as FC

F32, F64 = np.float32, np.float64
U = 2.0 ** -24
INF = float("inf")


def fma32(a, b, c):
    return (a.astype(F64) * b.astype(F64) + c.astype(F64)).astype(F32)


def encode(y):
    """[n, cols] fp32 rows -> (qy int8 [n, cols16], s, e, nrm fp32 [n]); unbounded rows get e = nrm = inf"""
    y = np.asarray(y, F32)
    n, cols = y.shape
    cols16 = (cols + 15) // 16 * 16
    amax = np.abs(y).max(1)
    s = (amax / F32(127)).astype(F32)
    ok = np.isfinite(y).all(1) & (s > 0) & np.isfinite(s)
    ss = np.where(ok, s, F32(1))
    qy = np.clip(np.rint(y / ss[:, None]), -127, 127)
    qy[~ok] = 0
    with np.errstate(invalid="ignore", over="ignore"):  # the unbounded rows' values are replaced below
        diff = y.astype(F64) - s.astype(F64)[:, None] * qy
        e = (np.sqrt((diff * diff).sum(1)) * (1 + 2.0 ** -30))
        nrm = s.astype(F64) * np.sqrt((qy * qy).sum(1))
    e = np.where(ok, np.nextafter(e.astype(F32), F32(INF)), F32(INF))
    nrm = np.where(ok, np.nextafter(nrm.astype(F32), F32(INF)), F32(INF))
    s = np.where(ok, s, F32(0))
    out = np.zeros((n, cols16), np.int8)
    out[:, :cols] = qy
    return out, s, e, nrm


def pass1_sum(xq, qy, s, metric):
    """[nq, n] fp32 pass-1 sums: sub-lane j of 8 takes the 16-column chunks j, j + 8, ...; then xor 1, 2, 4"""
    nq, n, cols16 = len(xq), len(qy), qy.shape[1]
    q = np.zeros((nq, cols16), F32)
    q[:, :xq.shape[1]] = xq
    qf = qy.astype(F32)
    lanes = np.zeros((8, nq, n), F32)
    for c in range(cols16 // 16):
        j = c % 8
        for i in range(16):
            col = 16 * c + i
            if metric == FC.METRIC_L2:
                t = fma32(-s[None, :], qf[None, :, col], q[:, col][:, None])
                lanes[j] = fma32(t, t, lanes[j])
            else:
                lanes[j] = fma32(q[:, col][:, None], qf[None, :, col], lanes[j])
    for off in (1, 2, 4):
        lanes = (lanes + lanes[np.arange(8) ^ off]).astype(F32)
    return lanes[0]


def direct_fp32(xq, y, metric):
    """[nq, n] the one-pass kernel's scores: rr_exact_scores, lane by lane"""
    nq, n, d = len(xq), len(y), y.shape[1]
    acc = np.zeros((32, 4, nq, n), F32)
    for c in range(d // 4):
        l = c % 32
        for j in range(4):
            a, b = xq[:, 4 * c + j][:, None], y[None, :, 4 * c + j]
            if metric == FC.METRIC_L2:
                t = (b - a).astype(F32)
                acc[l, j] = fma32(t, t, acc[l, j])
            else:
                acc[l, j] = fma32(b, a, acc[l, j])
    dis = ((acc[:, 0] + acc[:, 1]).astype(F32) + (acc[:, 2] + acc[:, 3]).astype(F32)).astype(F32)
    for off in (16, 8, 4, 2, 1):
        dis = (dis + dis[np.arange(32) ^ off]).astype(F32)
    return dis[0]


def interval(xq, st, s, e, nrm, d, metric):
    """(lo, hi, bounded) [nq, n] as pass 1 computes them"""
    cols16 = (d + 15) // 16 * 16
    g1, gr = 1.01 * (cols16 + 3) * U, 1.01 * (d + 3) * U
    ab = (4.0 * cols16 + 64.0) * 2.0 ** -149
    qn = np.sqrt((xq.astype(F64) ** 2).sum(1))[:, None] * (1 + 2.0 ** -40)
    st, s, e, nrm = st.astype(F64), s.astype(F64)[None], e.astype(F64)[None], nrm.astype(F64)[None]
    with np.errstate(invalid="ignore", over="ignore"):
        if metric == FC.METRIC_L2:
            r2lo = np.maximum(0, (st - ab) * (1 - g1))
            r2hi = (st + ab) * (1 + 2 * g1)
            rlo = np.maximum(0, np.sqrt(r2lo) - e)
            rhi = np.sqrt(r2hi) + e
            lo = np.maximum(0, rlo * rlo * (1 - gr) - ab)
            hi = rhi * rhi * (1 + gr) + ab
            mag = hi
        else:
            c = s * st
            yb = qn * (nrm + e)
            r = g1 * qn * nrm + s * ab + qn * e + gr * yb + ab
            lo, hi = c - r, c + r
            mag = yb * (1 + gr) + ab
        lo = lo - np.abs(lo) * 2.0 ** -40
        hi = hi + np.abs(hi) * 2.0 ** -40
        bounded = mag <= 2.0 ** 126
    return lo, hi, bounded


def special_rows(d, rng):
    base = rng.standard_normal((12, d))
    rows = [np.zeros(d), np.eye(d)[3] * 7.0, np.eye(d)[0] * 1e3 + 1e-3 * rng.standard_normal(d)]
    rows += [base[0] * 2.0 ** 30, base[1] * 2.0 ** -30, base[2] * 2.0 ** -64, base[3] * 2.0 ** -64 + base[4] * 2.0 ** -100]
    return np.array(rows)


def check(xq, db, metric):
    d = db.shape[1]
    qy, s, e, nrm = encode(db)
    st = pass1_sum(xq, qy, s, metric)
    lo, hi, bounded = interval(xq, st, s, e, nrm, d, metric)
    ref = direct_fp32(xq, db, metric).astype(F64)
    inside = (lo <= ref) & (ref <= hi)
    bad = bounded & ~inside
    assert not bad.any(), (f"{int(bad.sum())} pairs outside their interval; first: ref {ref[bad][0]!r}, "
                           f"[{lo[bad][0]!r}, {hi[bad][0]!r}]")
    assert not bounded[:, ~np.isfinite(e)].any()
    return bounded


@pytest.mark.parametrize("metric", [FC.METRIC_L2, FC.METRIC_IP])
@pytest.mark.parametrize("d", [32, 128, 768])
@pytest.mark.parametrize("name", FC.REGIMES)
def test_interval_holds_the_direct_form(name, d, metric):
    n, nq = (160, 6) if d == 768 else (400, 8)
    db, xq = FC.regime(name, n, d, nq, seed=7)
    rng = np.random.default_rng(d)
    db = np.concatenate([db, special_rows(d, rng).astype(F32)])
    xq = np.concatenate([xq, db[-1:] * F32(1.5), db[:1]])  # a query in the 2^-64 range and one on a row
    bounded = check(xq, db, metric)
    # the zero row is unbounded (it always survives); ordinary rows are bounded
    assert not bounded[:, n].any() and bounded[:, :n].mean() > 0.9


def test_intervals_are_tight_enough_to_prune():
    """sift-like rows: the interval half-width is a small fraction of the 10-NN distance, as the pruning needs"""
    db, xq = FC.regime("sift_float", 2000, 128, 8, seed=3)
    qy, s, e, nrm = encode(db)
    st = pass1_sum(xq, qy, s, FC.METRIC_L2)
    lo, hi, _ = interval(xq, st, s, e, nrm, 128, FC.METRIC_L2)
    ref = direct_fp32(xq, db, FC.METRIC_L2).astype(F64)
    kth = np.sort(ref, 1)[:, 9]
    survivors = (lo <= np.sort(hi, 1)[:, 9][:, None]).sum(1)
    assert np.all(lo <= ref) and np.all(ref <= hi)
    assert np.all(np.sqrt(hi) - np.sqrt(lo) < 0.2 * np.sqrt(kth)[:, None])
    assert survivors.max() < 200  # of 2000


def test_encoder_rows():
    d = 64
    y = np.zeros((4, d), F32)
    y[1, 5] = -3.0
    y[2] = np.linspace(-1, 1, d)
    y[3, 0] = np.inf
    qy, s, e, nrm = encode(y)
    assert s[0] == 0 and e[0] == INF and not qy[0].any()
    assert s[1] == F32(3) / F32(127) and qy[1, 5] == -127 and e[1] >= abs(3.0 - float(s[1]) * 127)
    assert np.abs(qy[2]).max() == 127 and e[2] <= 0.5 * float(s[2]) * np.sqrt(d)
    assert e[3] == INF and nrm[3] == INF
