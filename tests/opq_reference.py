"""Restatement of one OPQ training round and the contract of each of its steps (test infrastructure only).

The OPQ rotation ("opq": {"nsubvector": M} on IVFPQ; DESIGN.md §5, OPQ bar) is trained by opq_train_device:
subsample at most 65536 rows (the first rows of rand_perm(n, 1234)), centre them, start from a random orthonormal
matrix, then per round project the centred rows X through the fp32 rotation, train a 256-centroid k-means per
subspace (40 iterations in round 0, 4 hot-started ones after it, mp = 1000), encode, decode to Y, form X^T Y on the
device and solve the orthogonal Procrustes problem on the host.  index.debug_opq_trace records every step; this module
states what each must be, given the state the device itself reached:

  sample     orc.rand_perm(n, 1234)[:65536] when n > 65536, else every row in order
  mean       within the fp64 accumulation bound of the exact column mean (col_mean_kernel sums in fp64, rounds once)
  centred    float32(x_s) - mean                                              byte-equal
  r0         std::mt19937(1234), libstdc++'s normal_distribution<double> and the row Gram-Schmidt, restated byte-equal
  rf[t]      float32(r0) in round 0, float32(r[t - 1]) after it               byte-equal
  proj[t]    centred @ rf[t]^T                                                ip_direct_margin of fp64, length d
  k-means    kmeans_reference.check_trace on each subspace's slice of proj[t], k = 256, mp = 1000; round t > 0 starts
             from round t - 1's final centroids
  codes[t]   orc.pq_compute_codes(the k-means' final centroids, proj[t])      byte-equal
  recon[t]   the codebook gathered at codes[t]                                byte-equal
  xty[t]     centred^T @ recon[t]                                             ip_direct_margin of fp64, length n_s
  r[t]       orthonormal (max |R R^T - I| <= 1e-12), Procrustes-optimal for float64(xty[t]): trace(R xty) equals the
             sum of its singular values within 1e-10 relative, and R equals numpy's V U^T within 1e-9 where the
             singular values are separated (otherwise the optimum is not unique)
"""
import math

import numpy as np

import float_contract as fc
import kmeans_reference as kr
from oracle import oracle as orc

U, U64 = fc.U, fc.U64
MAX_TRAIN = 65536
KSUB = 256
KM_MP = 1000
ORTHO_TOL = 1e-12
OBJ_RTOL = 1e-10
R_TOL = 1e-9
SEP = 1e-5  # relative gap between consecutive singular values (and to zero) below which R is not unique enough


def kmeans_iters(t):
    return 40 if t == 0 else 4


# ---- the random start ---------------------------------------------------------------------------------------------------
class MT19937:
    """std::mt19937 seeded with one 32-bit value (init_genrand), drawing 32-bit outputs"""

    def __init__(self, seed):
        mt = [0] * 624
        mt[0] = seed & 0xFFFFFFFF
        for i in range(1, 624):
            mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & 0xFFFFFFFF
        self.mt, self.i = mt, 624

    def _twist(self):
        mt = self.mt
        for i in range(624):
            y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7FFFFFFF)
            mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
        self.i = 0

    def __call__(self):
        if self.i >= 624:
            self._twist()
        y = self.mt[self.i]
        self.i += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return y


def canonical(g):
    """libstdc++ generate_canonical<double, 53> over a 32-bit engine: two draws, (a + b 2^32) / 2^64 in double"""
    s = float(g()) + float(g()) * 4294967296.0
    r = s / 18446744073709551616.0
    return r if r < 1.0 else math.nextafter(1.0, 0.0)


class Normal:
    """libstdc++ normal_distribution<double>(0, 1): Marsaglia's polar method, the second value saved for the next call"""

    def __init__(self):
        self.saved = None

    def __call__(self, g):
        if self.saved is not None:
            v, self.saved = self.saved, None
            return v
        while True:
            x = 2.0 * canonical(g) - 1.0
            y = 2.0 * canonical(g) - 1.0
            r2 = x * x + y * y
            if not (r2 > 1.0 or r2 == 0.0):
                break
        mult = math.sqrt(-2 * math.log(r2) / r2)
        self.saved = x * mult
        return y * mult


def seqdot(a, b):
    """sum_j a_j b_j accumulated in index order in fp64, each product rounded (no FMA, as the host code compiles)"""
    return float(np.cumsum(a * b)[-1])


def random_start(d, seed=1234):
    """the d x d fp64 start: Gaussian entries in row-major order, then Gram-Schmidt on the rows in the code's loop order"""
    g, nd = MT19937(seed), Normal()
    R = np.array([nd(g) for _ in range(d * d)], np.float64).reshape(d, d)
    for i in range(d):
        for p in range(i):
            R[i] -= seqdot(R[i], R[p]) * R[p]
        R[i] /= math.sqrt(seqdot(R[i], R[i]))
    return R


# ---- the steps --------------------------------------------------------------------------------------------------------
def sample_ids(n):
    return orc.rand_perm(n, 1234)[:MAX_TRAIN] if n > MAX_TRAIN else np.arange(n, dtype=np.int64)


def check_mean(got, xs):
    """None, or why the device's column means are not within the fp64 accumulation bound of the exact ones.  Any
    order of n - 1 fp64 additions is within (n - 1) 2^-53 sum|x| of the exact sum; the division adds 2^-53 and the
    rounding to fp32 u of the mean."""
    xs = np.asarray(xs, np.float64)
    n = len(xs)
    exact = np.array([math.fsum(xs[:, j]) for j in range(xs.shape[1])]) / n  # within 2^-53 relative
    mabs = np.abs(xs).sum(0) / n
    bound = 1.01 * (U * np.abs(exact) + (n + 1) * U64 * mabs)
    err = np.abs(np.asarray(got, np.float64) - exact)
    if np.any(err > bound):
        j = int(np.argmax(err - bound))
        return f"mean of column {j}: {got[j]!r} off the exact {exact[j]!r} by {err[j]:.3g} > bound {bound[j]:.3g}"
    return None


def check_ip_product(got, a, b, what):
    """None, or why got [p, q] is not within ip_direct_margin of the fp64 a @ b^T (contraction length a.shape[1])"""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    f = a64 @ b64.T
    m = fc.ip_direct_margin(np.abs(a64) @ np.abs(b64).T, a64.shape[1])
    err = np.abs(np.asarray(got, np.float64) - f)
    if np.any(err > m):
        i = np.unravel_index(int(np.argmax(err - m)), err.shape)
        return f"{what} {tuple(int(v) for v in i)}: off by {err[i]:.3g} > margin {m[i]:.3g}"
    return None


def separated(s):
    """the singular values (descending) are distinct and nonzero by more than SEP relative"""
    if s[0] == 0:
        return False
    gaps = np.append(s[:-1] - s[1:], s[-1]) / s[0]
    return bool(np.all(gaps > SEP))


def check_procrustes(R, xty):
    """None, or why R is not the orthonormal maximiser of trace(R A), A = float64(xty) (R = V U^T for A = U S V^T)"""
    R, A = np.asarray(R, np.float64), np.asarray(xty, np.float64)
    d = len(R)
    dev = float(np.abs(R @ R.T - np.eye(d)).max())
    if not dev <= ORTHO_TOL:
        return f"not orthonormal: max |R R^T - I| = {dev:.3g}"
    u, s, vt = np.linalg.svd(A)
    obj, best = float(np.trace(R @ A)), float(s.sum())
    if abs(obj - best) > OBJ_RTOL * max(best, np.finfo(float).tiny):
        return f"not Procrustes-optimal: trace(R A) = {obj!r}, sum of singular values {best!r}"
    if separated(s):
        e = float(np.abs(R - vt.T @ u.T).max())
        if e > R_TOL:
            return f"R differs from V U^T by {e:.3g}"
    return None


def subspace_codebook(km_round):
    """[M, 256, dsub]: each subspace's final centroids of one round"""
    return np.stack([np.asarray(t["norm"][-1], np.float32) for t in km_round])


def check_round(tr, t, M, check_kmeans=True):
    """every step of round t of a detailed trace; raises AssertionError naming the step"""
    xc, proj = tr["centred"], tr["proj"][t]
    d = xc.shape[1]
    ds = d // M
    want_rf = (tr["r0"] if t == 0 else tr["r"][t - 1]).astype(np.float32)
    assert kr.same(tr["rf"][t], want_rf), f"round {t}: the uploaded rotation is not float32 of the last one"
    r = check_ip_product(proj, xc, tr["rf"][t], "projection")
    assert r is None, f"round {t}: {r}"
    if check_kmeans:
        for m in range(M):
            init = None if t == 0 else tr["km"][t - 1][m]["norm"][-1]
            try:
                kr.check_trace(proj[:, m * ds:(m + 1) * ds], KSUB, tr["km"][t][m], mp=KM_MP, init=init)
            except AssertionError as e:
                raise AssertionError(f"round {t}, subspace {m}: {e}") from None
    pq = subspace_codebook(tr["km"][t])
    assert np.array_equal(tr["codes"][t], orc.pq_compute_codes(pq, proj)), f"round {t}: codes"
    rec = pq[np.arange(M)[None, :], tr["codes"][t]].reshape(len(proj), d)
    assert kr.same(tr["recon"][t], rec), f"round {t}: reconstruction"
    r = check_ip_product(tr["xty"][t], xc.T, tr["recon"][t].T, "X^T Y")
    assert r is None, f"round {t}: {r}"
    r = check_procrustes(tr["r"][t], tr["xty"][t])
    assert r is None, f"round {t}: {r}"


def check_trace(x, M, tr, check_kmeans=True):
    """the whole of a detailed trace of x's OPQ training; raises AssertionError with the first step that breaks"""
    x = np.asarray(x, np.float32)
    n, d = x.shape
    sid = sample_ids(n)
    assert np.array_equal(tr["sample"], sid), "sampled rows"
    xs = x[sid]
    r = check_mean(tr["mean"], xs)
    assert r is None, r
    assert kr.same(tr["centred"], xs - tr["mean"][None, :]), "centred rows"
    assert np.array_equal(tr["r0"].view(np.uint64), random_start(d).view(np.uint64)), "random orthonormal start"
    for t in range(len(tr["rf"])):
        check_round(tr, t, M, check_kmeans)


def check_rotations(tr):
    """the rotation chain of a trace without detail: float32 hand-over and every round's Procrustes solution.  Returns
    the worst max |R R^T - I| seen (for the record)"""
    worst = 0.0
    for t in range(len(tr["rf"])):
        want_rf = (tr["r0"] if t == 0 else tr["r"][t - 1]).astype(np.float32)
        assert kr.same(tr["rf"][t], want_rf), f"round {t}: the uploaded rotation is not float32 of the last one"
        R = tr["r"][t]
        worst = max(worst, float(np.abs(R @ R.T - np.eye(len(R))).max()))
        r = check_procrustes(R, tr["xty"][t])
        assert r is None, f"round {t}: {r}"
    return worst
