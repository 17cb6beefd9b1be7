"""numpy twin of this engine's VEARCH codes, tables and scores (DESIGN.md section 3, K14; kernels_scann.cu).

The reference builds VEARCH on ScaNN 1.2.1 (third_party/scann-1.2.1), which needs bazel and TensorFlow and is not built
here, so this twin *is* the contract the device kernels are checked against, byte for byte and bit for bit.  Statements
about ScaNN's behaviour are read from its sources and marked [scann-source: <file>:<lines>]; they are not verified by
running it.

Blocks [scann-source: gamma_index_vearch.cc:128-186, VARIABLE_CHUNK projection].  nsub blocks of w = d // nsub dims, then,
when d % nsub > 0, one more block of the remaining dims.  Block b covers dims [b w, b w + width_b).  Each has 16 centres;
the codebook is 16 d floats: block b's centre c at floats [16 b w + c width_b, + width_b).

Codebook order [scann-source: asymmetric_hashing_impl.cc:220-243].  After each block's 16-centre k-means the centres are
ordered by cluster size, largest first, then rotated by ((b / 2) % max(1, 16 / 16)) * 16 = 0 places, then reversed in
every odd block b.  Equal sizes keep the k-means order here (std::sort leaves it open).

Encoder [scann-source: asymmetric_hashing_impl.cc:318-540, CoordinateDescentAHQuantize].  r = x - c_l (fp32) under
InnerProduct, r = x under L2.  In fp64, every operation rounded once, dims in index order:
  n2 = sum_i x_i^2 (also the squared norm of ComputeParallelCostMultiplier), inv = 1 / sqrt(n2)
  per (block, centre): rc_j = r_j - c_j;  rn = sum rc_j^2;  pr = sum (rc_j x_j) inv
  init: each block's first minimum of rn, as std::min_element with `<` finds it (a NaN never replaces the current
  minimum; a NaN first entry stays).  With noise shaping (IP and a threshold t that is not NaN):
  eta = (t^2 / n2) / ((1 - t^2 / n2) / (d - 1));  par = sum over blocks in order of pr[b][sel_b];
  blocks visited by decreasing rn[b][sel_b] (equal norms: lower block first; NaN norms last, lower block first), at
  most 10 rounds while a round moves;
  a visit of block b (current centre cur) tries every other centre c:
    npar = (par - pr[b][cur]) + pr[b][c];  pnd = npar^2 - par^2;  skipped when pnd > 0;
    cost = eta pnd + ((rn[b][c] - rn[b][cur]) - pnd);
  and moves to the lowest c of the smallest cost when that cost is < 0 (par = its npar).  NaN compares false, so a zero
  row (n2 = 0) or a row with a NaN coordinate keeps its initial codes.  Without noise shaping the initial codes are the
  codes.
Codes: block 2j in the low nibble of byte j, 2j + 1 in the high nibble.

Table [scann-source: asymmetric_hashing_impl.cc:553-665; hash.proto:81-92 for the defaults].  fp32, dims in order from 0:
  IP: t[b][c] = -(sum q_j c_j);  L2: t[b][c] = sum (q_j - c_j)^2
  m = 127 / max(sqrt(FLT_EPSILON), max |t|) (quantile 1.0);  lut = int(trunc(t m)) + 128 as uint8 (TRUNCATE, the proto
  default, and FixedPointBias<uint8_t> = 128).
Score of an entry: s = sum_b (lut[b][code_b] - 128) (integers);  v = f32(s) * f32(1 / m);
  L2: v;  IP: leaf - v with leaf = <q, c_l> (fp32, dims in order from 0).
"""
import numpy as np

F32, F64 = np.float32, np.float64
K = 16
METRIC_IP, METRIC_L2 = 0, 1


def blocks(d, nsub):
    """[(start, width)] of the VARIABLE_CHUNK split"""
    w = d // nsub
    out = [(b * w, w) for b in range(nsub)]
    if d % nsub:
        out.append((nsub * w, d - nsub * w))
    return out


def code_bytes(d, nsub):
    return (len(blocks(d, nsub)) + 1) // 2


def block_centres(cb, d, nsub):
    """the codebook (16 d floats) as a list of [16, width_b] arrays"""
    cb = np.asarray(cb, F32).reshape(-1)
    return [cb[K * s:K * s + K * w].reshape(K, w) for s, w in blocks(d, nsub)]


def flat_codebook(centres):
    return np.concatenate([np.asarray(c, F32).reshape(-1) for c in centres])


def order_centres(centres, sizes, b):
    """block b's 16 k-means centres in ScaNN's stored order: by size, largest first (stable), reversed for odd b"""
    perm = sorted(range(K), key=lambda c: -int(sizes[c]))
    if b & 1:
        perm = perm[::-1]
    return np.asarray(centres, F32)[perm]


def pack(sel):
    """[n, nb] codes < 16 -> [n, ceil(nb / 2)] bytes, block 2j in the low nibble of byte j"""
    sel = np.asarray(sel, np.uint8)
    n, nb = sel.shape
    if nb % 2:
        sel = np.concatenate([sel, np.zeros((n, 1), np.uint8)], axis=1)
    return (sel[:, 0::2] | (sel[:, 1::2] << 4)).astype(np.uint8)


def residual_stats(x, r, cb, d, nsub):
    """rn, pr [n, nb, 16] (fp64) and n2 [n] of rows x with residuals r (both fp32 [n, d])"""
    x64 = np.asarray(x, F32).astype(F64)
    r = np.asarray(r, F32)
    n = x64.shape[0]
    n2 = np.zeros(n, F64)
    for j in range(d):
        n2 = n2 + x64[:, j] * x64[:, j]
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = F64(1.0) / np.sqrt(n2)
    cents = block_centres(cb, d, nsub)
    nb = len(cents)
    rn = np.zeros((n, nb, K), F64)
    pr = np.zeros((n, nb, K), F64)
    with np.errstate(invalid="ignore", over="ignore"):
        for b, (s0, w) in enumerate(blocks(d, nsub)):
            c64 = cents[b].astype(F64)
            a = np.zeros((n, K), F64)
            p = np.zeros((n, K), F64)
            for j in range(w):
                rc = r[:, s0 + j].astype(F64)[:, None] - c64[None, :, j]
                a = a + rc * rc
                p = p + (rc * x64[:, s0 + j][:, None]) * inv[:, None]
            rn[:, b] = a
            pr[:, b] = p
    return rn, pr, n2


def eta_of(t, n2, d):
    """ComputeParallelCostMultiplier(t, n2, d) [scann-source: utils/noise_shaping_utils.h:27-34]"""
    with np.errstate(divide="ignore", invalid="ignore"):
        t2n = F64(t) * F64(t) / F64(n2)
        return t2n / ((F64(1.0) - t2n) / (F64(d) - F64(1.0)))


def first_min(rn):
    """InitializeToMinResidualNorm: the first minimum over the last axis (16 centres) under `<`, as std::min_element
    finds it: a NaN never becomes the minimum unless it is the first entry, which then stays"""
    best = np.zeros(rn.shape[:-1], np.int64)
    cur = rn[..., 0].copy()
    for c in range(1, rn.shape[-1]):
        better = rn[..., c] < cur
        best = np.where(better, c, best)
        cur = np.where(better, rn[..., c], cur)
    return best


def cd_codes(rn, pr, eta):
    """the coordinate-descent codes [nb] of one row from its statistics [nb, 16]"""
    nb = rn.shape[0]
    sel = first_min(rn)
    selnorm = rn[np.arange(nb), sel]
    par = F64(0.0)
    for b in range(nb):
        par = par + pr[b, sel[b]]
    order = np.argsort(-selnorm, kind="stable")  # NaN norms sort last, in block order
    idx = np.arange(K)
    with np.errstate(invalid="ignore", over="ignore"):
        for _ in range(10):
            changed = False
            for b in order:
                cur = sel[b]
                npar = (par - pr[b, cur]) + pr[b]
                pnd = npar * npar - par * par
                cost = eta * pnd + ((rn[b] - rn[b, cur]) - pnd)
                ok = ~(pnd > 0) & (cost < 0) & (idx != cur)
                if not ok.any():
                    continue
                cand = np.flatnonzero(ok)
                c = cand[np.argmin(cost[cand])]
                sel[b] = c
                par = npar[c]
                changed = True
            if not changed:
                break
    return sel


def encode(x, cb, d, nsub, metric, threshold, cents=None, assign=None):
    """packed codes [n, code_bytes] of rows x (IP: residuals to cents[assign]; L2: the rows).  threshold < 0 or NaN, or
    L2: nearest centres per block (the encoder's initial codes)"""
    x = np.asarray(x, F32)
    with np.errstate(invalid="ignore"):
        r = x - np.asarray(cents, F32)[np.asarray(assign)] if metric == METRIC_IP else x
    rn, pr, n2 = residual_stats(x, r, cb, d, nsub)
    shaped = metric == METRIC_IP and threshold is not None and not np.isnan(threshold) and threshold >= 0
    sel = first_min(rn)
    if shaped:
        for i in range(x.shape[0]):
            sel[i] = cd_codes(rn[i], pr[i], eta_of(threshold, n2[i], d))
    return pack(sel)


def anisotropic_cost(rn, pr, sel, eta):
    """eta |r_par|^2 + |r_perp|^2 of one row's codes sel [nb] (fp64)"""
    nb = rn.shape[0]
    par = sum(pr[b, sel[b]] for b in range(nb))
    tot = sum(rn[b, sel[b]] for b in range(nb))
    return eta * par * par + (tot - par * par)


def lut(q, cb, d, nsub, metric):
    """biased uint8 table [nb, 16] and multiplier (float32) of query q"""
    q = np.asarray(q, F32)
    tabs = []
    for c, (s0, w) in zip(block_centres(cb, d, nsub), blocks(d, nsub)):
        acc = np.zeros(K, F32)
        for j in range(w):
            if metric == METRIC_L2:
                u = q[s0 + j] - c[:, j]
                acc = acc + u * u
            else:
                acc = acc + q[s0 + j] * c[:, j]
        tabs.append(acc if metric == METRIC_L2 else -acc)
    t = np.stack(tabs).astype(F32)
    m = F32(np.abs(t).max())
    lim = np.sqrt(F32(np.finfo(F32).eps))
    mul = F32(127.0) / (m if lim < m else lim)
    return (np.trunc(t * mul).astype(np.int32) + 128).astype(np.uint8), F32(mul)


def unpack(codes, nb):
    codes = np.asarray(codes, np.uint8)
    lo, hi = codes & 15, codes >> 4
    sel = np.empty((codes.shape[0], 2 * codes.shape[1]), np.int64)
    sel[:, 0::2], sel[:, 1::2] = lo, hi
    return sel[:, :nb]


def leaf(q, c):
    """<q, c_l> in fp32, dims in order from 0"""
    q, c = np.asarray(q, F32), np.asarray(c, F32)
    acc = F32(0.0)
    for j in range(q.shape[0]):
        acc = F32(acc + q[j] * c[j])
    return acc


def scores(codes, table, mult, metric, leaf_term=F32(0.0)):
    """float32 scores of list entries `codes` under one query's (table, mult), plus the list's leaf term under IP"""
    nb = table.shape[0]
    sel = unpack(codes, nb)
    s = (table[np.arange(nb)[None, :], sel].astype(np.int64) - 128).sum(axis=1)
    v = s.astype(F32) * (F32(1.0) / F32(mult))
    return (F32(leaf_term) - v).astype(F32) if metric == METRIC_IP else v.astype(F32)
