"""Training on the H100, held to the restatement of tests/kmeans_reference.py (DESIGN.md §5, training bar).

Every iteration of a traced device k-means run (index.debug_kmeans_trace) is checked from the state the device reached:
its labels meet the assignment contract against C_t, the segmented mean and the split are byte-equal to the oracle's
from those labels, the renormalisation is within the bound derived in the reference.  Around that: the sampled rows and
the initial centroids, hot start, degenerate data (splits at every iteration, identical rows, n = k and k + 1, zero
rows, NaN and infinite rows), whole runs byte-equal to orc.kmeans on data the trace proves unambiguous, and each index
type's trained state byte-equal to device k-means on its restated training set."""
import numpy as np
import pytest

import float_contract as fc
import kmeans_reference as kr
from oracle import oracle as orc
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = fc.METRIC_L2, fc.METRIC_IP
MODES = {"l2": (False, False), "ip": (True, False), "l2_assign": (True, True)}


def gi():
    from vearch_b200 import index as gidx
    return gidx


def traced(x, k, mode="l2", niter=4, seed=1234, mp=256, init=None):
    """a traced device run, checked step by step; returns (trace, splits)"""
    sph, l2a = MODES[mode]
    tr = gi().debug_kmeans_trace(x, k, niter=niter, seed=seed, spherical=sph, l2_assign=l2a, max_points_per_centroid=mp,
                                 init=init)
    return tr, kr.check_trace(x, k, tr, seed=seed, spherical=sph, l2_assign=l2a, mp=mp, init=init)


def regime_rows(name, n, d, seed=5):
    return fc.regime(name, n, d, 1, seed)[0]


# ---- the step contract, every iteration -------------------------------------------------------------------------------
@pytest.mark.parametrize("k,d", [(32, 16), (128, 8)])  # the exact CUDA-core argmin, the tensor-core one
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("regime", fc.REGIMES)
def test_step_contract_regimes(regime, mode, k, d):
    traced(regime_rows(regime, max(4 * k, 400), d), k, mode)


# the k and d ladders: both sides of the tensor-core switch at k = 64, dsub-like widths 1-5, 17 (one past a 16-column
# chunk), 768; the regime rotates along the ladder
LADDER = [(2, 1), (2, 768), (63, 3), (63, 17), (64, 1), (64, 768), (65, 2), (65, 5), (256, 4), (256, 16), (1024, 8),
          (64, 128)]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("i", range(len(LADDER)), ids=[f"k{k}-d{d}" for k, d in LADDER])
def test_step_contract_ladder(i, mode):
    k, d = LADDER[i]
    regime = fc.REGIMES[i % len(fc.REGIMES)]
    traced(regime_rows(regime, max(4 * k, 400), d, seed=11 + i), k, mode)


# ---- sampling and initialisation --------------------------------------------------------------------------------------
@pytest.mark.parametrize("delta", [-1, 0, 1])
@pytest.mark.parametrize("k,mp", [(5, 256), (5, 1000), (5, 0), (64, 256)])
def test_sampling_and_init(k, mp, delta):
    n = k * (mp or 300) + delta
    x = np.random.default_rng(3).standard_normal((n, 4)).astype(np.float32)
    tr, _ = traced(x, k, "l2", niter=2, seed=77, mp=mp)  # check_trace asserts the sample and the initial centroids
    assert len(tr["sample"]) == (k * mp if mp and n > k * mp else n)


@pytest.mark.parametrize("mode", ["l2", "ip"])
@pytest.mark.parametrize("k", [16, 64])
def test_hot_start_keeps_centroids(k, mode):
    rng = np.random.default_rng(4)
    x = rng.standard_normal((40 * k, 8)).astype(np.float32)
    init = rng.standard_normal((k, 8)).astype(np.float32)  # deliberately not normalised: a hot start takes it as given
    traced(x, k, mode, niter=3, init=init)


# ---- splits and degenerate data ---------------------------------------------------------------------------------------
def few_distinct(n, d, distinct, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((distinct, d)).astype(np.float32)[rng.integers(0, distinct, n)]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("k", [64, 256])
def test_splits_every_iteration(k, mode):
    x = few_distinct(4 * k, 6, 10, 8)
    tr, splits = traced(x, k, mode, niter=5)
    assert all(len(np.unique(lab)) < k for lab in tr["labels"]) and splits >= 5


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("k", [8, 64])
def test_identical_rows(k, mode):
    x = np.tile(np.arange(1, 6, dtype=np.float32) / 7, (4 * k, 1))
    tr, splits = traced(x, k, mode, niter=3)
    assert splits > 0


@pytest.mark.parametrize("extra", [0, 1])  # n = k (no split possible) and n = k + 1 (the split divides by n - k = 1)
@pytest.mark.parametrize("k", [16, 64])
def test_n_equals_k_and_k_plus_one(k, extra):
    x = few_distinct(k + extra, 5, k // 2, 9)
    traced(x, k, "l2", niter=4)
    traced(np.random.default_rng(9).standard_normal((k + extra, 5)).astype(np.float32), k, "l2", niter=4)


@pytest.mark.parametrize("mode", ["ip", "l2_assign"])
@pytest.mark.parametrize("k", [16, 64])
def test_zero_rows_spherical(k, mode):
    x = np.random.default_rng(6).standard_normal((20 * k, 8)).astype(np.float32)
    x[::3] = 0
    tr, _ = traced(x, k, mode, niter=4)


@pytest.mark.parametrize("bad", ["nan", "inf", "-inf", "mixed"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("k", [16, 64])
def test_non_finite_rows(k, mode, bad):
    """Rows holding a NaN or an infinity follow faiss's rule exactly on both argmin paths: NaN rows and, under L2
    assignment, infinite rows go to cluster 0; under IP an infinite row goes to the first centroid whose dot is +inf
    (at k >= 64 the tensor-core tiles cannot score it, the split of inf being NaN, so the exact kernel scores it again).
    The centroid that absorbs such a row turns non-finite, and no finite row may follow it there."""
    rng = np.random.default_rng(12)
    x = rng.standard_normal((30 * k, 8)).astype(np.float32)
    rows = rng.choice(len(x), 7, replace=False)
    val = {"nan": np.nan, "inf": np.inf, "-inf": -np.inf}
    for j, r in enumerate(rows):
        v = val[bad] if bad != "mixed" else list(val.values())[j % 3]
        x[r, j % 8] = v
    tr, _ = traced(x, k, mode, niter=4)
    # the finite rows went on clustering: not all of them in one cluster
    assert len(np.unique(tr["labels"][-1])) > k // 2
    if mode == "ip" and bad != "nan":  # some infinite row left cluster 0 (a +inf dot wins)
        assert np.any(tr["labels"][:, rows] != 0)


# ---- whole runs on unambiguous data -----------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [64, 256, 1024])
def test_whole_run_unambiguous_equals_oracle(k):
    """k well-separated points, rows near them, and the initial centroids one per point (the rows the seeded
    permutations pick are placed first): every row's label wins by more than the margin at every iteration, asserted
    from the trace, so the tensor-core run must equal orc.kmeans byte for byte."""
    d, mp, seed, niter = 16, 8, 1234, 6
    n = k * mp + 37
    rng = np.random.default_rng(k)
    pts = rng.uniform(-50, 50, (k, d)).astype(np.float32)
    sid = kr.sample_ids(n, k, mp, seed)
    first = sid[kr.init_ids(len(sid), k, seed)]
    which = rng.integers(0, k, n)
    which[first] = np.arange(k)
    x = (pts[which] + 0.05 * rng.standard_normal((n, d))).astype(np.float32)
    x[first] = pts  # the initial centroids are the points themselves
    tr, splits = traced(x, k, "l2", niter=niter, seed=seed, mp=mp)
    assert splits == 0
    cent = tr["init"]
    for t in range(niter):
        assert kr.gap_excess(x[sid], cent, tr["labels"][t], L2) < 0, f"iteration {t} is ambiguous"
        cent = tr["norm"][t]
    got, _ = gi().kmeans(x, k, niter=niter, seed=seed, max_points_per_centroid=mp)
    want, _, _ = orc.kmeans(x, k, niter=niter, seed=seed, max_points_per_centroid=mp)
    assert np.array_equal(kr.bits(got), kr.bits(want))
    assert np.array_equal(kr.bits(got), kr.bits(tr["norm"][-1]))


# ---- each index type's trained state ----------------------------------------------------------------------------------
NLIST = 16
# the training_threshold parameter: unset, below nlist (raised to 39 nlist), = nlist (k-means on n = k rows), between
# nlist and 39 nlist (kept as given), above 256 nlist (lowered to it)
THRESHOLDS = [None, NLIST - 1, NLIST, 20 * NLIST, 300 * NLIST]
N = 256 * NLIST + 100

# type -> (default threshold, niter, spherical under IP, l2_assign)
COARSE = {"IVFFLAT": (200 * NLIST, 25, False, False), "IVFPQ": (200 * NLIST, 10, True, False),
          "GPU_IVFPQ": (256 * NLIST, 10, True, False), "IVFPQFastScan": (39 * NLIST, 25, True, True),
          "IVFRABITQ": (200 * NLIST, 10, True, False), "VEARCH": (256 * NLIST, 12, True, True)}


def mt(metric):
    return "L2" if metric == L2 else "InnerProduct"


_open = []


@pytest.fixture(autouse=True)
def _close_indexes():
    """every index build() made is closed after its test, whether the test passed or not"""
    yield
    while _open:
        _open.pop().close()


def build(typ, d, metric, threshold, extra):
    x = synth.sift_like(N, d, seed=21, rounded=False)
    params = {"ncentroids": NLIST, "nprobe": 4, "metric_type": mt(metric)}
    if threshold is not None:
        params["training_threshold"] = threshold
    params.update(extra)
    idx = gi().GammaIndex(typ, d, params)
    _open.append(idx)
    idx.add_vectors(x)
    default, niter, sph, l2a = COARSE[typ]
    t = kr.clamp_threshold(threshold or 0, NLIST, default)
    assert idx.training_threshold == t
    return idx, x, x[:t], dict(niter=niter, spherical=sph and metric == IP, l2_assign=l2a)


def coarse_trace(xt, kp):
    return gi().debug_kmeans_trace(xt, NLIST, niter=kp["niter"], seed=1234, spherical=kp["spherical"],
                                   l2_assign=kp["l2_assign"], max_points_per_centroid=256)["norm"][-1]


def vid_lists(idx):
    off, _, ids = idx.export_lists()
    lst = np.empty(idx.ntotal, np.int64)
    for l in range(idx.nlist):
        lst[ids[off[l]:off[l + 1]]] = l
    return lst


def codebook_rows(t, npq):
    return orc.rand_perm(t, 1234)[:npq] if npq < t else np.arange(t)


def check_codebook(idx, x_rows, ksub):
    """each sub-quantiser's codebook = the traced k-means of its column slice (niter 25, seed 1234, mp 256)"""
    pq = idx.get_pq_centroids()
    M, _, dsub = pq.shape
    for m in range(M):
        want = gi().debug_kmeans_trace(x_rows[:, m * dsub:(m + 1) * dsub], ksub, niter=25, seed=1234,
                                       max_points_per_centroid=256)["norm"][-1]
        assert np.array_equal(kr.bits(pq[m]), kr.bits(want)), f"sub-quantiser {m}"


@pytest.mark.parametrize("ti", range(len(THRESHOLDS)))
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("typ", ["IVFFLAT", "IVFRABITQ", "VEARCH"])
def test_coarse_state_equals_trace(typ, metric, ti):
    extra = {"nsubvector": 4} if typ == "VEARCH" else {}
    idx, x, xt, kp = build(typ, 16, metric, THRESHOLDS[ti], extra)
    idx.train()
    assert np.array_equal(kr.bits(idx.get_centroids()), kr.bits(coarse_trace(xt, kp)))


# (nbits, dsub): every nbits the issue's ladder names, every dsub, crossed rather than multiplied; the thresholds rotate
IVFPQ_CASES = [(1, 3), (4, 1), (6, 2), (7, 8), (8, 4), (8, 1), (6, 3), (1, 8)]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("i", range(len(IVFPQ_CASES)), ids=[f"nbits{b}-dsub{s}" for b, s in IVFPQ_CASES])
def test_ivfpq_trained_state(i, metric):
    nbits, dsub = IVFPQ_CASES[i]
    M, ksub = 4, 1 << nbits
    threshold = THRESHOLDS[(i + metric) % len(THRESHOLDS)]
    idx, x, xt, kp = build("IVFPQ", M * dsub, metric, threshold, {"nsubvector": M, "nbits_per_idx": nbits})
    check_ivfpq(idx, x, xt, kp, ksub)


@pytest.mark.parametrize("ti", [0, 2, 4])
def test_gpu_ivfpq_trained_state(ti):
    idx, x, xt, kp = build("GPU_IVFPQ", 32, L2, THRESHOLDS[ti], {"nsubvector": 8})
    check_ivfpq(idx, x, xt, kp, 256)


def check_ivfpq(idx, x, xt, kp, ksub):
    t = len(xt)
    npq = min(t, 256 * ksub)
    if npq < ksub:  # faiss's k-means refuses fewer points than centroids: so must training
        with pytest.raises(gi().GammaError):
            idx.train()
        assert not idx.is_trained
        return
    idx.train()
    cent = idx.get_centroids()
    assert np.array_equal(kr.bits(cent), kr.bits(coarse_trace(xt, kp)))
    idx.add_pending()
    rows = codebook_rows(t, npq)
    lst = vid_lists(idx)[rows]  # add assigns with the exact argmin train_extra uses, on the same rows
    check_codebook(idx, (xt[rows] - cent[lst]).astype(np.float32), ksub)


@pytest.mark.parametrize("ti", range(len(THRESHOLDS)))
@pytest.mark.parametrize("metric", [L2, IP])
def test_ivfpqfs_trained_state(metric, ti):
    idx, x, xt, kp = build("IVFPQFastScan", 16, metric, THRESHOLDS[ti], {"nsubvector": 8})
    t = len(xt)
    npq = min(t, 256 * 16)  # t >= nlist = 16 = ksub in every case: the codebook always trains
    idx.train()
    assert np.array_equal(kr.bits(idx.get_centroids()), kr.bits(coarse_trace(xt, kp)))
    check_codebook(idx, xt[codebook_rows(t, npq)], 16)


def test_training_threshold_past_int32():
    """256 * nlist passes 2^31 at nlist = 2^23: the clamp is 64-bit, as gamma's size_t one"""
    nlist = 1 << 23
    idx = gi().GammaIndex("GPU_IVFFLAT", 4, {"ncentroids": nlist, "nprobe": 1, "metric_type": "InnerProduct"})
    _open.append(idx)
    assert idx.training_threshold == kr.clamp_threshold(0, nlist, 256 * nlist) == 1 << 31
