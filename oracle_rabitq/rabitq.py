"""numpy twin of this engine's IVFRABITQ codes and estimator (DESIGN.md section 3, K13; kernels_rabitq.cu).

This is the engine's own contract, not a restatement of faiss: the reference computes its codes and estimates inside
faiss v1.14.1 (RaBitQuantizer, RaBitQDistanceComputer, rabitq_utils), which is not available here, so nothing below
claims bit parity with faiss [faiss-restated statements are marked so and are not verifiable here].

Notation: B = nb_bits, W = ceil(d / 32) words per bit-plane, M = 2^(B-1) - 1, r = x - c_l the residual to the entry's list
centroid.

Grid.  u_i in [0, 2^B), o_i = u_i + 1/2 - 2^(B-1); u_i's top bit is r_i > 0, its magnitude m_i = min(floor(t |r_i|), M).
The encoder picks t > 0 maximising cos(o, r) exactly: the critical points t = j / |r_i| (fp64 quotients) are visited in
increasing (t, i) order; N2 = sum_i |r_i| (2 m_i + 1) is updated in fp64 in that order (starting from the fp64 sum of
|r_i| in index order), D4 = sum_i (2 m_i + 1)^2 exactly; at the end of every group of equal t the state scores
N2 * N2 / D4 (fp64) and the first maximum wins (a tie goes to the smaller t; the state before any event is first).

Entry: B bit-planes of W uint32 words (plane p = bit B-1-p of u, dim i at bit i & 31 of word i >> 5; sign plane first;
padding bits 0), then fp32 |r|^2 (fp64 sum in index order, rounded once), f = |r|^2 / (N2 / 2) (fp64, rounded once; 0
when r = 0), S = sum_i o_i over the real dimensions.

Estimate for query q in list l: v = q - c_l (L2) or q (IP).  base = |q - c_l|^2 (L2) or <q, c_l> (IP), summed as the
scan's CTA sums it: thread t (of 256) adds the products of dims t, t + 256, ... in order from 0, each warp of 32 adds its
partials by an xor butterfly (offsets 16, ..., 1), the 8 warp totals are added in order.  lo, hi = min, max of v over
the real dims; delta = (hi - lo) / (2^qb - 1) (0 when qb = 0 or hi = lo); vbar_i = rint((v_i - lo) / delta) clamped to
[0, 2^qb - 1], 0 on padding dims or when delta = 0.
  qb = 0:  <o, v> = an entry's L lanes (L = the largest power of two <= W, at most 8, and 32 once W >= 32) each add
           o_i * v_i (fp32,
           unfused) over words lane, lane + L, ... in order, dims 0..31 of a word in order, from 0; the L partials are
           added by an xor butterfly (offsets L/2, ..., 1).
  qb > 0:  A = sum u_i vbar_i, X = 2 A + (1 - 2^B) sum vbar_i (integers), <o, v> = delta * (f32(X) * 0.5) + lo * S.
Score: L2 (|r|^2 + base) - 2 (f <o, v>);  IP base + f <o, v>  (fp32, in that order).
"""
import numpy as np

F32 = np.float32
METRIC_IP, METRIC_L2 = 0, 1


def words(d):
    return (d + 31) // 32


def lanes(d):
    w = words(d)
    if w >= 32:
        return 32
    return 8 if w >= 8 else (4 if w >= 4 else (2 if w >= 2 else 1))


def code_bytes(d, nb_bits):
    return 4 * (nb_bits * words(d) + 3)


def _seq_sum(a):
    """fp64 sum in index order (a[0] + a[1] + ...)"""
    return float(np.add.accumulate(np.asarray(a, np.float64))[-1]) if len(a) else 0.0


def choose_magnitudes(r, nb_bits):
    """-> (m [d] int, t, N2, nr2): the magnitudes of the best state, its t (-1: before any event), fp64 N2 and |r|^2"""
    r = np.asarray(r, F32)
    d = len(r)
    a = np.abs(r).astype(np.float64)
    M = (1 << (nb_bits - 1)) - 1
    n20 = _seq_sum(a)
    nr2 = _seq_sum(r.astype(np.float64) * r.astype(np.float64))
    best, best_n2, best_t = (n20 * n20) / float(d), n20, -1.0
    nz = np.nonzero(a > 0)[0]
    if M > 0 and len(nz):
        j = np.tile(np.arange(1, M + 1, dtype=np.float64), len(nz))
        ii = np.repeat(nz, M)
        key = j / a[ii]
        o = np.lexsort((ii, key))
        key, ii, j = key[o], ii[o], j[o]
        n2 = np.add.accumulate(np.concatenate([[n20], 2.0 * a[ii]]))[1:]
        d4 = float(d) + np.cumsum(8 * j.astype(np.int64)).astype(np.float64)
        end = np.r_[key[1:] != key[:-1], True]
        obj = (n2[end] * n2[end]) / d4[end]
        cand = np.concatenate([[best], obj])
        b = int(np.argmax(cand))
        if b > 0 and cand[b] > best:
            best_n2, best_t = float(n2[end][b - 1]), float(key[end][b - 1])
    m = np.zeros(d, np.int64)
    if best_t >= 0:
        sel = key <= best_t
        m = np.bincount(ii[sel], minlength=d).astype(np.int64)
    return m, best_t, best_n2, nr2


def encode_residuals(res, nb_bits):
    """[n, d] fp32 residuals -> [n, code_bytes] uint8 entries"""
    res = np.asarray(res, F32)
    n, d = res.shape
    W, B = words(d), nb_bits
    half = 1 << (B - 1)
    out = np.zeros((n, B * W + 3), np.uint32)
    for row in range(n):
        r = res[row]
        m, _, n2, nr2 = choose_magnitudes(r, B)
        u = np.where(r > 0, half + m, half - 1 - m).astype(np.int64)
        up = np.zeros(32 * W, np.int64)
        up[:d] = u
        for p in range(B):
            bits = ((up >> (B - 1 - p)) & 1).astype(np.uint64).reshape(W, 32)
            out[row, p * W:(p + 1) * W] = (bits << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
        ssum = int(np.sum(2 * u + 1 - 2 * half))
        fac = np.array([np.float32(nr2), np.float32(nr2 / (n2 * 0.5)) if n2 > 0 else 0.0,
                        F32(F32(ssum) * F32(0.5))], F32)
        out[row, B * W:] = fac.view(np.uint32)
    return out.view(np.uint8).reshape(n, -1)


def encode(x, cents, assign, nb_bits):
    x, cents = np.asarray(x, F32), np.asarray(cents, F32)
    return encode_residuals(x - cents[np.asarray(assign)], nb_bits)


def decode(codes, d, nb_bits):
    """-> (u [n, 32 W] int64, nr2, f, S) of entries"""
    W, B = words(d), nb_bits
    w = np.ascontiguousarray(codes).view(np.uint32).reshape(len(codes), B * W + 3)
    u = np.zeros((len(codes), 32 * W), np.int64)
    for p in range(B):
        bits = (w[:, p * W:(p + 1) * W, None].astype(np.uint64) >> np.arange(32, dtype=np.uint64)) & 1
        u = (u << 1) | bits.reshape(len(codes), 32 * W).astype(np.int64)
    fac = w[:, B * W:].view(F32)
    return u, fac[:, 0], fac[:, 1], fac[:, 2]


def list_tables(q, c, d, metric, qb):
    """-> (v [32 W] fp32, base, delta, lo, vbar [32 W] int64) of a (query, list)"""
    W = words(d)
    q = np.asarray(q, F32)[:d]
    c = np.asarray(c, F32)[:d]
    if metric == METRIC_L2:
        v = q - c
        prod = v * v
    else:
        v = q.copy()
        prod = q * c
    nrow = -(-d // 256)
    p = np.zeros(nrow * 256, F32)
    p[:d] = prod
    s = np.zeros(256, F32)
    for rr in p.reshape(nrow, 256):
        s = s + rr
    s = s.reshape(8, 32)
    idx = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        s = s + s[:, idx ^ off]
    base = s[0, 0]
    for w in range(1, 8):
        base = F32(base + s[w, 0])
    lo, hi = F32(v.min()), F32(v.max())
    delta = F32(F32(hi - lo) / F32((1 << qb) - 1)) if (qb > 0 and hi > lo) else F32(0)
    vp = np.zeros(32 * W, F32)
    vp[:d] = v
    vbar = np.zeros(32 * W, np.int64)
    if delta > 0:
        vbar[:d] = np.clip(np.rint((v - lo) / delta), 0, (1 << qb) - 1).astype(np.int64)
    return vp, F32(base), delta, lo, vbar


def estimate(codes, q, c, d, nb_bits, metric, qb):
    """fp32 scores [n] of entries `codes` of the list with centroid c for query q"""
    B, W, L = nb_bits, words(d), lanes(d)
    u, nr2, f, S = decode(codes, d, B)
    v, base, delta, lo, vbar = list_tables(q, c, d, metric, qb)
    n = len(codes)
    if qb == 0:
        o = (2 * u + 1 - (1 << B)).astype(F32) * F32(0.5)
        prods = o * v[None, :]
        parts = np.zeros((n, L), F32)
        for ln in range(L):
            acc = np.zeros(n, F32)
            for w in range(ln, W, L):
                for k in range(32):
                    acc = acc + prods[:, 32 * w + k]
            parts[:, ln] = acc
        li = np.arange(L)
        off = L >> 1
        while off:
            parts = parts + parts[:, li ^ off]
            off >>= 1
        ip = parts[:, 0]
    else:
        A = (u * vbar[None, :]).sum(axis=1)
        X = 2 * A + (1 - (1 << B)) * int(vbar.sum())
        ip = (delta * (X.astype(F32) * F32(0.5))) + (lo * S)
    t = f * ip
    if metric == METRIC_L2:
        return ((nr2 + base) - F32(2) * t).astype(F32)
    return (base + t).astype(F32)


def cos_at(r, nb_bits, m):
    """cos(o, r) (fp64) of the magnitudes m"""
    r = np.asarray(r, np.float64)
    o = np.where(r > 0, m + 0.5, -(m + 0.5))
    nr = np.linalg.norm(r)
    return float(o @ r / (np.linalg.norm(o) * nr)) if nr > 0 else 0.0


def magnitudes_at(r, nb_bits, t):
    M = (1 << (nb_bits - 1)) - 1
    return np.minimum(np.floor(t * np.abs(np.asarray(r, np.float64))), M).astype(np.int64)
