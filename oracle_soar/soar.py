"""fp64 numpy restatement of SOAR spilling (DESIGN.md §8), the twin the GPU kernels are tested against.

Spilled list of a row x whose primary list is a (r = x - c_a, r' = x - c'), over every list c' != a:

    loss(c') = |r'|^2 + lambda <r, r'>^2 / |r|^2

the least loss, the lower list id among equal ones (Sun et al., NeurIPS 2023, eq. 7).  A row with |r| = 0, values that
are not finite, or no primary list, takes list gvid % nlist as an unassigned row does, or gvid + 1 when that is its
primary list.

Search over spilled lists selects 2 k' keys (score order, then vid) and keeps each vid's first: the k' distinct vids with
the best best-copy keys, since every vid has at most two live entries."""
import numpy as np

U32 = 2.0 ** -24  # unit roundoff of fp32
SENTINEL = np.uint64(0xFFFFFFFFFFFFFFFF)


def spill_terms(x, centroids, primary):
    """fp64 e [n][nlist] = |x - c'|^2, p = <r, x - c'>, pabs = sum |r_j| |x_j - c'_j|, rn [n] = |r|^2 (r = x - c_primary;
    rows without a primary list get rn = nan)"""
    x = np.asarray(x, np.float64)
    c = np.asarray(centroids, np.float64)
    primary = np.asarray(primary, np.int64)
    ok = (primary >= 0) & (primary < len(c))
    r = np.where(ok[:, None], x - c[np.where(ok, primary, 0)], np.nan)
    diff = x[:, None, :] - c[None, :, :]
    e = np.einsum("ncj,ncj->nc", diff, diff)
    p = np.einsum("nj,ncj->nc", r, diff)
    pabs = np.einsum("nj,ncj->nc", np.abs(r), np.abs(diff))
    rn = np.einsum("nj,nj->n", r, r)
    return e, p, pabs, rn


def spill_loss(x, centroids, primary, lam):
    """fp64 loss [n][nlist]; the primary list itself gets +inf"""
    e, p, _, rn = spill_terms(x, centroids, primary)
    with np.errstate(divide="ignore", invalid="ignore"):
        loss = e + lam * p * p / rn[:, None]
    primary = np.asarray(primary, np.int64)
    rows = np.nonzero((primary >= 0) & (primary < loss.shape[1]))[0]
    loss[rows, primary[rows]] = np.inf
    return loss


def fallback_list(gvid, primary, nlist):
    """the spilled list of a row the loss cannot place"""
    s = int(gvid) % nlist
    return (int(gvid) + 1) % nlist if s == primary else s


def spill_lists(x, centroids, primary, lam, vid0=0):
    """each row's spilled list: argmin of the loss (ties to the lower id), or the fallback rule"""
    loss = spill_loss(x, centroids, primary, lam)
    _, _, _, rn = spill_terms(x, centroids, primary)
    nlist = loss.shape[1]
    out = np.empty(len(loss), np.int64)
    for i in range(len(loss)):
        row = loss[i]
        good = np.isfinite(rn[i]) and rn[i] > 0 and np.isfinite(row).any()
        out[i] = int(np.argmin(np.where(np.isfinite(row), row, np.inf))) if good else fallback_list(vid0 + i, primary[i], nlist)
    return out


def spill_margin(x, centroids, primary, lam):
    """[n][nlist] bound on |fp32 loss - fp64 loss| of launch_soar_spill's arithmetic: e and p as fma chains over the
    fp32 differences (eta = (d + 3) u relative to sum (x - c)^2 and to sum |r| |x - c|), |r|^2 within eta, then three
    roundings (lambda p, p / |r|^2, the fma)"""
    d = np.asarray(x).shape[1]
    e, p, pabs, rn = spill_terms(x, centroids, primary)
    eta = 1.01 * (d + 3) * U32
    rn = rn[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        dp2 = 2 * np.abs(p) * eta * pabs + (eta * pabs) ** 2  # |p^2 - fl(p)^2|
        t = lam * p * p / rn
        m = eta * e + lam * dp2 / rn * (1 + eta + 3 * U32) + (eta + 3 * U32) * t + U32 * (e + t + lam * dp2 / rn)
    return 1.05 * m


def check_spill(x, centroids, primary, lam, got):
    """Each got[i] (not the primary) has a loss within the margin of the least one: loss(got) <= min_c (loss(c) +
    margin(c)) + margin(got).  Returns the rows that fail."""
    loss = spill_loss(x, centroids, primary, lam)
    m = spill_margin(x, centroids, primary, lam)
    bad = []
    for i, g in enumerate(np.asarray(got, np.int64)):
        if g == primary[i] or not (0 <= g < loss.shape[1]):
            bad.append(i)
            continue
        fin = np.isfinite(loss[i])
        if loss[i, g] > np.min((loss[i] + m[i])[fin]) + m[i, g]:
            bad.append(i)
    return bad


# ---- the duplicate-free selection ---------------------------------------------------------------------------------
def dedupe_first(keys, k):
    """launch_dedupe_keys: of a sorted uint64 key row, the first k keys whose vid (low 32 bits) has not occurred earlier,
    sentinel padded"""
    keys = np.asarray(keys, np.uint64)
    seen, out = set(), []
    for key in keys:
        if key == SENTINEL:
            out.append(key)
        else:
            v = int(key) & 0xFFFFFFFF
            if v in seen:
                continue
            seen.add(v)
            out.append(key)
        if len(out) == k:
            break
    out += [SENTINEL] * (k - len(out))
    return np.array(out, np.uint64)


def topk_best_copy(vids, keys, k):
    """the contract: the k distinct vids of best best-copy key, as their best keys in key order (sentinel padded)"""
    best = {}
    for v, key in zip(np.asarray(vids, np.int64), np.asarray(keys, np.uint64)):
        v = int(v)
        if v not in best or key < best[v]:
            best[v] = key
    out = sorted(best.values())[:k]
    return np.array(out + [SENTINEL] * (k - len(out)), np.uint64)


def make_keys(score_ord, vids):
    """(order-preserving score bits << 32) | vid, the scan's key layout"""
    return (np.asarray(score_ord, np.uint64) << np.uint64(32)) | np.asarray(vids, np.uint64)
