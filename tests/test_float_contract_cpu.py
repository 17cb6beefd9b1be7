"""The float-accuracy contract (tests/float_contract.py) on the CPU: numpy's own fp32 evaluations stay inside the
margins on every data regime, and check_selection accepts what the margins allow and nothing more."""
import numpy as np
import pytest

import float_contract as FC

L2, IP = FC.METRIC_L2, FC.METRIC_IP


@pytest.mark.parametrize("name", FC.REGIMES)
@pytest.mark.parametrize("d", [30, 128])
def test_numpy_fp32_forms_within_margins(name, d):
    db, xq = FC.regime(name, 3000, d, 16, seed=5)
    f, absdot = FC.scores64(xq, db, L2)
    t = db[None, :, :] - xq[:, None, :]  # fp32 differences
    direct = np.einsum("qnj,qnj->qn", t, t, dtype=np.float32)
    assert np.all(np.abs(direct - f) <= FC.l2_direct_margin(f, d)), name
    xn, yn = (xq * xq).sum(1, dtype=np.float32), (db * db).sum(1, dtype=np.float32)
    exp = np.maximum(np.float32(0), xn[:, None] + yn[None, :] - np.float32(2) * (xq @ db.T))
    na, nb = (xq.astype(np.float64) ** 2).sum(1)[:, None], (db.astype(np.float64) ** 2).sum(1)[None, :]
    assert np.all(np.abs(exp - f) <= FC.expanded_l2_margin(absdot, na, nb, f, d)), name
    # the same form over fp32 operands shifted by a point near the data (what the list-major scan evaluates)
    s = db[:64].mean(0).astype(np.float32)
    a, b = xq - s, db - s
    an, bn = (a * a).sum(1, dtype=np.float32), (b * b).sum(1, dtype=np.float32)
    sh = np.maximum(np.float32(0), an[:, None] + bn[None, :] - np.float32(2) * (a @ b.T))
    na, nb, ad = FC.shifted_operands(xq, db, s)
    assert np.all(np.abs(sh - f) <= FC.shifted_l2_margin(ad, na, nb, f, d)), name
    fi, absdot = FC.scores64(xq, db, IP)
    assert np.all(np.abs((xq @ db.T) - fi) <= FC.ip_direct_margin(absdot, d)), name


def test_offset_expanded_form_is_what_the_shift_is_for():
    # at offset 1000 the margin of the expanded form on raw vectors is far wider than the gaps between neighbours;
    # over operands shifted near the data it is not
    db, xq = FC.regime("offset1000", 2000, 128, 4, seed=1)
    f, absdot = FC.scores64(xq, db, L2)
    na, nb = (xq.astype(np.float64) ** 2).sum(1)[:, None], (db.astype(np.float64) ** 2).sum(1)[None, :]
    raw = FC.expanded_l2_margin(absdot, na, nb, f, 128)
    na, nb, ad = FC.shifted_operands(xq, db, db.mean(0))
    shifted = FC.shifted_l2_margin(ad, na, nb, f, 128)
    gap = np.diff(np.sort(f, axis=1)[:, :11], axis=1).mean()
    assert raw.min() > 10 * gap and shifted.max() < 0.1 * gap


# ---- check_selection ----------------------------------------------------------------------------------------------------
def case(metric, k=5, n=40, seed=0):
    rng = np.random.default_rng(seed)
    f = np.sort(rng.uniform(1, 100, n))
    if metric == IP:
        f = f[::-1].copy()
    cand = rng.permutation(1000)[:n].astype(np.int64)
    m = np.full(n, 1e-3)
    md = np.full(n, 1e-3)
    return cand, f, m, md


def result(cand, f, pick, metric, k, sc=None):
    pick = list(pick)
    s = (f[pick] if sc is None else sc).astype(np.float32)
    ids = cand[pick]
    o = np.argsort(s if metric == L2 else -s, kind="stable")
    s, ids = s[o], ids[o]
    pad = k - len(pick)
    fill = np.float32(FC.FLT_MAX if metric == L2 else -FC.FLT_MAX)
    return np.concatenate([s, np.full(pad, fill, np.float32)]), np.concatenate([ids, np.full(pad, -1, np.int64)])


@pytest.mark.parametrize("metric", [L2, IP])
def test_selection_exact_passes_and_swaps(metric):
    k = 5
    cand, f, m, md = case(metric, k)
    assert FC.check_selection(*result(cand, f, range(k), metric, k), cand, f, m, md, k, metric) is None
    # zero margins: the exact set check
    z = np.zeros_like(m)
    assert FC.check_selection(*result(cand, f, range(k), metric, k), cand, f, z, m, k, metric) is None
    # the k-th and (k+1)-th within the margin of each other: either may be returned
    f2 = f.copy()
    f2[k] = f2[k - 1] + (5e-4 if metric == L2 else -5e-4)
    s = f2[list(range(k - 1)) + [k]]
    assert FC.check_selection(*result(cand, f2, list(range(k - 1)) + [k], metric, k, s), cand, f2, m, md, k,
                              metric) is None
    # beyond the margin: refused, with the excess and the missing id reported
    r = FC.check_selection(*result(cand, f, list(range(k - 1)) + [k], metric, k), cand, f, m, md, k, metric)
    assert r is not None and r[1] == 1 and r[2] > 0
    with pytest.raises(AssertionError, match="1/1 queries"):
        g = result(cand, f, list(range(k - 1)) + [k], metric, k)
        FC.check_all((g[0][None], g[1][None]), lambda q: (cand, f, m, md), k, metric, "swap")


@pytest.mark.parametrize("metric", [L2, IP])
def test_selection_refusals(metric):
    k = 5
    cand, f, m, md = case(metric, k)
    # a score off by more than the direct margin
    s = f[:k].copy()
    s[k - 1] += 2e-3 if metric == L2 else -2e-3  # the last one: the order holds, only the score is off
    r = FC.check_selection(*result(cand, f, range(k), metric, k, s), cand, f, m, md, k, metric)
    assert r is not None and "off by" in r[0]
    # a missing id: k - 1 results while k are valid
    r = FC.check_selection(*result(cand, f, range(k - 1), metric, k), cand, f, m, md, k, metric)
    assert r is not None and "count" in r[0]
    # an id that is not a valid candidate
    sc, ids = result(cand, f, range(k), metric, k)
    ids[0] = 5000
    assert FC.check_selection(sc, ids, cand, f, m, md, k, metric) is not None
    # out of order
    sc, ids = result(cand, f, range(k), metric, k)
    assert FC.check_selection(sc[::-1].copy(), ids[::-1].copy(), cand, f, m, md, k, metric) is not None


@pytest.mark.parametrize("metric", [L2, IP])
def test_selection_window(metric):
    k = 5
    cand, f, m, md = case(metric, k)
    lo, hi = (f[3], FC.FLT_MAX) if metric == L2 else (-FC.FLT_MAX, f[3])
    win = {"min_score": lo, "max_score": hi}
    # f[3] sits on the edge: it may be in or out
    assert FC.check_selection(*result(cand, f, range(3, 3 + k), metric, k), cand, f, m, md, k, metric, **win) is None
    assert FC.check_selection(*result(cand, f, range(4, 4 + k), metric, k), cand, f, m, md, k, metric, **win) is None
    # f[2] is certainly outside: a window violation
    r = FC.check_selection(*result(cand, f, range(2, 2 + k), metric, k), cand, f, m, md, k, metric, **win)
    assert r is not None and "outside the window" in r[0]
    # a window that leaves fewer than k: all of them, no more
    lo2, hi2 = (f[-3] - 1e-2, FC.FLT_MAX) if metric == L2 else (-FC.FLT_MAX, f[-3] + 1e-2)
    w2 = {"min_score": lo2, "max_score": hi2}
    n = len(f)
    assert FC.check_selection(*result(cand, f, range(n - 3, n), metric, k), cand, f, m, md, k, metric, **w2) is None
    r = FC.check_selection(*result(cand, f, range(n - 2, n), metric, k), cand, f, m, md, k, metric, **w2)
    assert r is not None
