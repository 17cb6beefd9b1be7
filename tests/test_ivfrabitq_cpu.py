"""The IVFRABITQ numpy twin (oracle_rabitq) against its own contract: the encoder's exact choice of t, the estimator's
identities, and the padding dimensions."""
import numpy as np
import pytest

from oracle_rabitq import rabitq as rq

F32 = np.float32


def brute_best_cos(r, B):
    """max cos(o, r) over a dense t grid, refined at every critical point and between consecutive ones"""
    a = np.abs(r.astype(np.float64))
    M = (1 << (B - 1)) - 1
    crit = np.unique(np.concatenate([[1e-30]] + [np.arange(1, M + 1) / x for x in a if x > 0]))
    mids = (crit[:-1] + crit[1:]) / 2 if len(crit) > 1 else crit
    grid = np.geomspace(crit[0] * 0.5 if crit[0] > 0 else 1e-3, crit[-1] * 2 + 1, 2000)
    ts = np.concatenate([crit, mids, grid, [crit[-1] * 4 + 1]])
    return max(rq.cos_at(r, B, rq.magnitudes_at(r, B, t)) for t in ts)


@pytest.mark.parametrize("B", range(1, 10))
def test_encoder_t_is_the_exact_argmax(B):
    rng = np.random.default_rng(B)
    for trial in range(12):
        d = int(rng.integers(1, 17))
        r = rng.standard_normal(d).astype(F32)
        if trial % 3 == 0:
            r = np.round(r * 2).astype(F32)  # ties between dimensions, zeros
        m, t, n2, nr2 = rq.choose_magnitudes(r, B)
        best = brute_best_cos(r, B)
        got = rq.cos_at(r, B, m)
        assert got >= best - 1e-12, (B, d, got, best)
        if t >= 0:  # the chosen state is m(t) at its critical t (nudged up: fl(j / a) * a may round below j)
            assert np.array_equal(m, rq.magnitudes_at(r, B, t * (1 + 1e-12)))
        assert abs(n2 - np.sum(np.abs(r.astype(np.float64)) * (2 * m + 1))) <= 1e-9 * max(1.0, n2)


@pytest.mark.parametrize("B", [1, 4, 9])
@pytest.mark.parametrize("d", [16, 30, 100, 128])
def test_estimate_of_the_residual_itself_is_its_norm(B, d):
    rng = np.random.default_rng(d + B)
    res = rng.standard_normal((20, d)).astype(F32)
    codes = rq.encode_residuals(res, B)
    u, nr2, f, S = rq.decode(codes, d, B)
    o = (u[:, :d] + 0.5 - (1 << (B - 1))).astype(np.float64)
    est = f.astype(np.float64) * np.sum(o * res.astype(np.float64), axis=1)  # f <o, r>
    assert np.allclose(est, np.sum(res.astype(np.float64) ** 2, axis=1), rtol=1e-6)
    assert np.allclose(nr2, np.sum(res.astype(np.float64) ** 2, axis=1), rtol=1e-6)
    assert np.array_equal(S, (o.sum(axis=1)).astype(F32))


@pytest.mark.parametrize("metric", [rq.METRIC_L2, rq.METRIC_IP])
@pytest.mark.parametrize("B", [1, 3, 4, 9])
def test_quantised_query_on_its_grid_equals_the_float_estimate(metric, B):
    """dyadic data: every fp32 sum of both paths is exact, so v on the qb grid gives equal scores"""
    rng = np.random.default_rng(B)
    d, qb = 64, 4
    c = np.zeros(d, F32) if metric == rq.METRIC_IP else (rng.integers(-4, 5, d) * 0.25).astype(F32)
    k = rng.integers(0, 16, d)
    k[0], k[1] = 0, 15  # lo and hi on the grid's ends
    v = (-2.0 + 0.25 * k).astype(F32)
    q = (v + c).astype(F32) if metric == rq.METRIC_L2 else v
    res = (rng.integers(-8, 9, (50, d)) * 0.5).astype(F32)
    codes = rq.encode_residuals(res, B)
    f0 = rq.estimate(codes, q, c, d, B, metric, 0)
    f4 = rq.estimate(codes, q, c, d, B, metric, qb)
    _, _, delta, lo, vbar = rq.list_tables(q, c, d, metric, qb)
    assert delta == F32(0.25) and lo == F32(-2.0) and np.array_equal(vbar[:d], k)
    u, nr2, f, S = rq.decode(codes, d, B)
    o = (u[:, :d] + 0.5 - (1 << (B - 1))).astype(np.float64)
    ipx = o @ v.astype(np.float64)
    assert np.array_equal(f0, f4)
    t = f.astype(np.float64) * ipx
    base = np.sum(v.astype(np.float64) ** 2) if metric == rq.METRIC_L2 else float(q.astype(np.float64) @ c)
    want = (nr2 + base - 2 * t) if metric == rq.METRIC_L2 else (base + t)
    assert np.allclose(f0, want, rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("d", [30, 100])
@pytest.mark.parametrize("B", [1, 4, 9])
def test_padding_dimensions_contribute_nothing(d, B):
    rng = np.random.default_rng(d * B)
    res = rng.standard_normal((40, d)).astype(F32)
    codes = rq.encode_residuals(res, B)
    assert codes.shape[1] == rq.code_bytes(d, B) == 4 * (B * rq.words(d) + 3)
    u, nr2, f, S = rq.decode(codes, d, B)
    assert np.all(u[:, d:] == 0)  # padding bits are 0 in every plane
    q = rng.standard_normal(d).astype(F32)
    c = np.zeros(d, F32)
    o = (u[:, :d] + 0.5 - (1 << (B - 1))).astype(np.float64)
    for metric in (rq.METRIC_L2, rq.METRIC_IP):
        est = rq.estimate(codes, q, c, d, B, metric, 0).astype(np.float64)
        t = f.astype(np.float64) * (o @ q.astype(np.float64))  # the real dimensions only
        base = float(q.astype(np.float64) @ q.astype(np.float64)) if metric == rq.METRIC_L2 else 0.0
        want = (nr2 + base - 2 * t) if metric == rq.METRIC_L2 else (base + t)
        assert np.allclose(est, want, rtol=1e-5, atol=1e-4)
        for qb in (1, 4, 8):
            _, _, _, _, vbar = rq.list_tables(q, c, d, metric, qb)
            assert np.all(vbar[d:] == 0)
