"""The helpers the device tests of the two-pass re-rank read it with (rerank_reference.py), checked without a GPU: the
shadow-row rule, the brackets of pass-1 intervals, the survivor count they imply, the sets with a known survivor count,
and the single-rounding FMA the restated sums need."""
import numpy as np
import pytest

import float_contract as FC
import rerank_reference as RR
from test_rerank_prefilter_cpu import encode, interval, special_rows
from vearch_b200 import synth

F32, F64 = np.float32, np.float64
INF = float("inf")


def test_shadow_rule_accepts_encode_and_rejects_loose_rows():
    rng = np.random.default_rng(2)
    y = RR.pad4(np.concatenate([special_rows(30, rng), rng.standard_normal((20, 30)) * 3]).astype(F32))
    y[3, 0] = 50 * 2.0 ** -149  # scale rounds to 0: unbounded
    y[3, 1:] = 0
    qy, s, e, nrm = encode(y)
    # the device's nrm: |s qy| in fp64, rounded up (encode() takes the root of the fp32 sum of squares)
    nrm = np.where(s > 0, RR.f32_up(s.astype(F64) * np.sqrt((qy.astype(F64) ** 2).sum(1))), F32(INF))
    assert y.shape[1] == 32 and qy.shape[1] == 32 and e[3] == INF and s[3] == 0
    assert RR.shadow_mismatch(y, qy, s, e, nrm) is None
    for what, change in (("e = 0", lambda a: a[2].__setitem__(9, 0)),
                         ("nrm loose", lambda a: a[3].__setitem__(9, a[3][9] * F32(1.001))),
                         ("qy", lambda a: a[0].__setitem__((9, 2), a[0][9, 2] + 1)),
                         ("s", lambda a: a[1].__setitem__(9, np.nextafter(a[1][9], F32(1)))),
                         ("bounded scale 0", lambda a: a[2].__setitem__(3, F32(1)))):
        arrs = [a.copy() for a in (qy, s, e, nrm)]
        change(arrs)
        assert RR.shadow_mismatch(y, *arrs) is not None, what


@pytest.mark.parametrize("metric", [FC.METRIC_L2, FC.METRIC_IP])
def test_brackets_are_a_few_ulps_wide_and_hold_the_rounded_interval(metric):
    db, xq = FC.regime("sift_float", 300, 48, 3, seed=9)
    qy, s, e, nrm = encode(db)
    lo_min, lo_max, hi_min, hi_max, bounded = RR.brackets(xq, qy, s, e, nrm, metric)
    lo, hi, _ = interval(xq, RR.pass1_sum(xq, qy, s, metric), s, e, nrm, 48, metric)
    assert bounded.all()
    assert np.all((lo_min <= RR.f32_down(lo)) & (RR.f32_down(lo) <= lo_max))
    assert np.all((hi_min <= RR.f32_up(hi)) & (RR.f32_up(hi) <= hi_max))
    ulps = lambda a, b: np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))  # noqa: E731
    assert ulps(lo_max, lo_min).max() <= 2 and ulps(hi_max, hi_min).max() <= 2


@pytest.mark.parametrize("metric", [FC.METRIC_L2, FC.METRIC_IP])
def test_expected_survivors_by_hand(metric):
    # L2 intervals; IP gets the mirrored scores, so the same candidates are the good ones
    lo = np.array([1, 1.5, 2, 3, 3.5, np.nan, np.nan, 0.5], F32)
    hi = np.array([2, 3, 4, 5, 6, np.nan, np.nan, 9], F32)
    state = np.array([RR.BOUNDED] * 5 + [RR.UNBOUNDED, RR.DEAD, RR.WITHHELD])
    if metric == FC.METRIC_IP:
        lo, hi = -hi, -lo
    # k = 2: the bound is the second-best worst end, 3 (a lo equal to it survives); the unbounded and the withheld
    # candidates survive, the dead one does not
    assert RR.expected_survivors(lo[None], hi[None], state[None], 2, metric)[0] == 6
    assert RR.expected_survivors(lo[None], hi[None], state[None], 1, metric)[0] == 5
    # fewer than k candidates bound it: every live one survives
    assert RR.expected_survivors(lo[None], hi[None], state[None], 6, metric)[0] == 7


@pytest.mark.parametrize("metric", [FC.METRIC_L2, FC.METRIC_IP])
@pytest.mark.parametrize("m", [32, 33])
def test_copies_and_far_survive_exactly_m(m, metric):
    rng = np.random.default_rng(m)
    d = 64
    db = np.rint(synth.sift_like(3000, d, seed=3) / 8)
    q = np.rint(synth.sift_like(1, d, seed=4) / 8)[0]
    if metric == FC.METRIC_IP:
        db, q = db - 16, q - 16
    near = q * (4 if metric == FC.METRIC_IP else 1)
    near[0] += 1
    db[2000:2040] = near
    db, q = db.astype(F32), q.astype(F32)
    cand = RR.copies_and_far(q, db, 2000 + np.arange(40), m, 300, metric, rng)
    assert len(cand) == m + 300 and len(np.unique(cand)) == len(cand)
    qy, s, e, nrm = encode(db[cand])
    lo_min, _, _, hi_max, bounded = RR.brackets(q[None], qy, s, e, nrm, metric)
    assert bounded.all()
    # the widest intervals the device may give these rows
    state = np.full(lo_min.shape, RR.BOUNDED)
    for k in (1, 10, m):
        assert RR.expected_survivors(lo_min, hi_max, state, k, metric)[0] == m


def test_fma32_rounds_once():
    a, b = np.array([1 + 2.0 ** -23], F32), np.array([1.5], F32)  # a b = 1.5 + 1.5 ulps: an fp32 midpoint
    assert RR.fma32(a, b, np.array([-(2.0 ** -64)], F32))[0] == F32(1.5 + 2.0 ** -23)  # fmaf rounds down, not to even
    assert RR.fma32(a, b, np.array([2.0 ** -64], F32))[0] == F32(1.5 + 2.0 ** -22)
    assert RR.fma32(a, b, np.array([0], F32))[0] == F32(1.5 + 2.0 ** -22)  # the tie itself goes to even
