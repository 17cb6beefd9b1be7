"""The k-means restatement of tests/kmeans_reference.py, checked without a GPU: replaying orc.kmeans one iteration at a
time from its own labels reproduces it byte for byte (plain, spherical, spherical assigned by L2, with empty clusters),
a trace built from that replay passes check_trace, and the assignment contract accepts exact labels and rejects wrong
ones."""
import numpy as np
import pytest

import float_contract as fc
import kmeans_reference as kr
from oracle import oracle as orc

L2, IP = fc.METRIC_L2, fc.METRIC_IP


def replay(x, k, niter, seed, spherical, l2_assign, mp):
    """orc.kmeans restated step by step; returns (final centroids, a trace dict as index.debug_kmeans_trace gives)"""
    x = np.asarray(x, np.float32)
    sid = kr.sample_ids(len(x), k, mp, seed)
    xs = x[sid]
    cent = xs[kr.init_ids(len(xs), k, seed)]
    if spherical:
        cent = orc.kmeans_normalize(cent)
    metric = kr.assign_metric(spherical, l2_assign)
    tr = {"sample": sid, "init": cent, "labels": [], "scores": [], "mean": [], "split": [], "norm": []}
    for _ in range(niter):
        lab = orc.assign(cent, xs, metric)
        lab[lab < 0] = 0
        f = kr.scores_exact(xs, cent, metric)
        tr["labels"].append(lab)
        tr["scores"].append(f[np.arange(len(xs)), lab].astype(np.float32))
        mean, split, cent, _ = kr.restated_step(xs, k, lab, spherical)
        tr["mean"].append(mean)
        tr["split"].append(split)
        tr["norm"].append(cent)
    return cent, {key: np.asarray(v) for key, v in tr.items()}


def empty_cluster_data(n, d, seed):
    """few distinct rows, so that clusters empty out and split at every iteration"""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((5, d)).astype(np.float32)
    return base[rng.integers(0, 5, n)]


CASES = [  # (data, n, d, k, spherical, l2_assign, mp)
    ("gauss", 3000, 8, 16, False, False, 256),
    ("gauss", 3000, 8, 16, True, False, 256),
    ("gauss", 3000, 8, 16, True, True, 256),
    ("gauss", 5000, 5, 4, False, False, 1000),  # subsampled: 4 x 1000 of 5000 rows
    ("gauss", 700, 3, 64, False, False, 256),
    ("few", 400, 6, 16, False, False, 256),
    ("few", 400, 6, 16, True, False, 256),
    ("few", 200, 4, 64, False, False, 0),
    ("inf", 600, 6, 16, False, False, 256),
    ("inf", 600, 6, 16, True, False, 256),
    ("inf", 600, 6, 16, True, True, 256),
    ("inf", 900, 6, 64, True, False, 256),
]


@pytest.mark.parametrize("data,n,d,k,spherical,l2_assign,mp", CASES)
def test_replay_reproduces_oracle(data, n, d, k, spherical, l2_assign, mp):
    x = (empty_cluster_data(n, d, 7) if data == "few" else np.random.default_rng(7).standard_normal((n, d)).astype(np.float32))
    if data == "inf":  # rows holding +-inf (and one a NaN): under IP a +inf dot is a best score, under L2 cluster 0
        for j, r in enumerate(range(3, n, n // 7)):
            x[r, j % d] = (np.inf, -np.inf, np.nan)[j % 3] if j % 4 else np.inf
    niter, seed = 6, 1234
    want, _, _ = orc.kmeans(x, k, niter=niter, seed=seed, spherical=spherical, max_points_per_centroid=mp,
                            l2_assign=l2_assign)
    got, tr = replay(x, k, niter, seed, spherical, l2_assign, mp)
    assert kr.same(got, want)
    # the replay's own trace meets every check of the GPU tests (the margins are those of the kernel k selects)
    splits = kr.check_trace(x, k, tr, seed=seed, spherical=spherical, l2_assign=l2_assign, mp=mp)
    if data == "few":
        assert splits > 0


@pytest.mark.parametrize("spherical", [False, True])
def test_check_trace_catches_each_step(spherical):
    x = empty_cluster_data(400, 6, 9)
    _, tr = replay(x, 16, 4, 1234, spherical, False, 256)
    kr.check_trace(x, 16, tr, spherical=spherical)

    def broken(key, f):
        t = {k: v.copy() for k, v in tr.items()}
        f(t[key])
        with pytest.raises(AssertionError):
            kr.check_trace(x, 16, t, spherical=spherical)

    up = np.float32(9)
    broken("sample", lambda a: a.__setitem__(0, a[1]))
    # one ulp is within the renormalisation bound, so a spherical start is moved further
    broken("init", lambda a: a.__setitem__((0, 0), a[0, 0] * np.float32(1.001) if spherical else np.nextafter(a[0, 0], up)))
    broken("mean", lambda a: a.__setitem__((1, 2, 3), np.nextafter(a[1, 2, 3], up)))
    # one entry of a re-seeded (split) centroid
    t, c = next((t, c) for t in range(len(tr["labels"])) for c in range(16) if not np.any(tr["labels"][t] == c))
    broken("split", lambda a: a.__setitem__((t, c, 0), np.nextafter(a[t, c, 0], up)))
    broken("norm", lambda a: a.__setitem__((2, 1), a[2, 1] * np.float32(1.001) if spherical else np.nextafter(a[2, 1], up)))
    broken("labels", lambda a: a.__setitem__((1, 5), (a[1, 5] + 1) % 16))


@pytest.mark.parametrize("k", [16, 64])
@pytest.mark.parametrize("metric", [L2, IP])
def test_contract_accepts_exact_rejects_worse(k, metric):
    rng = np.random.default_rng(11)
    x = (rng.standard_normal((600, 12)) + 100).astype(np.float32)
    cent = (rng.standard_normal((k, 12)) + 100).astype(np.float32)
    if metric == IP:
        cent = orc.kmeans_normalize(cent)
    lab = orc.assign(cent, x, metric)
    f, _ = fc.scores64(x, cent, metric)
    sc = f[np.arange(len(x)), lab].astype(np.float32)
    assert kr.check_assignment(x, cent, lab, sc, metric) is None
    # a label moved to the row's worst centroid
    worst = np.argmax(f, 1) if metric == L2 else np.argmin(f, 1)
    bad = lab.copy()
    bad[17] = worst[17]
    assert "better" in kr.check_assignment(x, cent, bad, sc, metric)
    # the key's score moved far beyond the margin
    s2 = sc.copy()
    s2[3] = s2[3] * np.float32(2)
    assert "key score" in kr.check_assignment(x, cent, lab, s2, metric)
    # a duplicate of a lower centroid
    c2 = cent.copy()
    c2[k - 1] = c2[lab[0]]
    lab2 = orc.assign(c2, x, metric)
    lab2[0] = k - 1
    assert "duplicate" in kr.check_assignment(x, c2, lab2, sc, metric)


def test_contract_non_finite_rows_and_centroids():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((50, 4)).astype(np.float32)
    cent = rng.standard_normal((8, 4)).astype(np.float32)
    x[3, 1] = np.nan
    x[7, 0] = np.inf
    lab = orc.assign(cent, x, L2)
    lab[lab < 0] = 0
    lab[[3, 7]] = 0
    f = np.zeros(len(x))
    ok = np.isfinite(x).all(1)
    f[ok] = fc.scores64(x[ok], cent, L2)[0][np.arange(ok.sum()), lab[ok]]
    sc = f.astype(np.float32)
    assert kr.check_assignment(x, cent, lab, sc, L2) is None
    bad = lab.copy()
    bad[3] = 2
    assert "faiss's rule" in kr.check_assignment(x, cent, bad, sc, L2)
    # under IP an infinite row goes to the first centroid whose dot is +inf, not to cluster 0
    ci = kr.scores_exact(x[7:8], cent, IP)[0]
    first_inf = int(np.nonzero(ci == np.inf)[0][0])
    lab_ip = orc.assign(cent, x, IP)
    lab_ip[lab_ip < 0] = 0
    assert lab_ip[7] == first_inf
    sc_ip = np.zeros(len(x), np.float32)
    sc_ip[ok] = fc.scores64(x[ok], cent, IP)[0][np.arange(ok.sum()), lab_ip[ok]]
    sc_ip[7] = np.inf
    assert kr.check_assignment(x, cent, lab_ip, sc_ip, IP) is None
    bad = lab_ip.copy()
    bad[7] = 0 if first_inf else 1
    assert "faiss's rule" in kr.check_assignment(x, cent, bad, sc_ip, IP)
    c2 = cent.copy()
    c2[5, 2] = np.nan
    bad = orc.assign(c2, x, L2)
    bad[~ok] = 0
    bad[bad < 0] = 0
    bad[0] = 5
    assert "non-finite centroid" in kr.check_assignment(x, c2, bad, sc, L2)


def test_training_threshold_clamp_restated():
    """[39, 256] * nlist clamp of IvfIndex::training_threshold as the GPU tests restate it"""
    clamp_threshold = kr.clamp_threshold
    assert clamp_threshold(0, 32, 200 * 32) == 200 * 32
    assert clamp_threshold(31, 32, 0) == 39 * 32
    assert clamp_threshold(32, 32, 0) == 32
    assert clamp_threshold(300 * 32, 32, 0) == 256 * 32
    assert clamp_threshold(0, 2 ** 23, 256 * 2 ** 23) == 2 ** 31
