"""The VEARCH numpy twin (oracle_scann) against its own contract: the block split, the size order of the codebooks, the
coordinate-descent encoder (cost never above its initialisation, equal to a literal scalar replay of the reference's move
rule), plain codes for a zero row and a negative threshold, and a fixed-point table worked by hand."""
import math

import numpy as np
import pytest

from oracle_scann import ah

F32 = np.float32


def test_block_split_with_and_without_a_remainder():
    assert ah.blocks(128, 64) == [(2 * b, 2) for b in range(64)]
    assert ah.code_bytes(128, 64) == 32
    assert ah.blocks(10, 3) == [(0, 3), (3, 3), (6, 3), (9, 1)]
    assert ah.code_bytes(10, 3) == 2
    assert ah.blocks(7, 7) == [(j, 1) for j in range(7)] and ah.code_bytes(7, 7) == 4
    cb = np.arange(16 * 10, dtype=F32)
    cents = ah.block_centres(cb, 10, 3)
    assert [c.shape for c in cents] == [(16, 3), (16, 3), (16, 3), (16, 1)]
    assert cents[1][2, 0] == 48 + 2 * 3 and cents[3][5, 0] == 16 * 9 + 5
    assert np.array_equal(ah.flat_codebook(cents), cb)


def test_size_order_largest_first_stable_and_reversed_in_odd_blocks():
    c = np.arange(16, dtype=F32)[:, None] * np.ones((1, 2), F32)
    sizes = [5, 9, 9, 1, 0, 9, 3, 3, 2, 2, 2, 7, 7, 4, 6, 8]
    want = sorted(range(16), key=lambda i: (-sizes[i], i))
    assert np.array_equal(ah.order_centres(c, sizes, 0)[:, 0], np.array(want, F32))
    assert np.array_equal(ah.order_centres(c, sizes, 3)[:, 0], np.array(want[::-1], F32))


def test_packing():
    sel = np.array([[1, 2, 3], [15, 0, 7]])
    assert np.array_equal(ah.pack(sel), np.array([[0x21, 0x03], [0x0F, 0x07]], np.uint8))
    assert np.array_equal(ah.unpack(ah.pack(sel), 3), sel)


def replay(x, r, cb, d, nsub, t):
    """CoordinateDescentAHQuantize restated line by line with Python floats (IEEE fp64, one rounding per operation)"""
    cents = ah.block_centres(cb, d, nsub)
    bl = ah.blocks(d, nsub)
    chunked = 0.0
    for j in range(d):
        chunked += float(x[j]) * float(x[j])
    sq = chunked
    chunked = math.sqrt(chunked)
    inv = 1.0 / chunked if chunked else math.inf
    stats = []
    for (s0, w), c in zip(bl, cents):
        row = []
        for k in range(16):
            rn = pr = 0.0
            for j in range(w):
                rc = float(r[s0 + j]) - float(c[k, j])
                rn += rc * rc
                pr += rc * float(x[s0 + j]) * inv
            row.append((rn, pr))
        stats.append(row)
    t2 = t * t
    pc = t2 / sq if sq else math.inf
    mult = pc / ((1.0 - pc) / (d - 1.0))
    result = [min(range(16), key=lambda k: (stats[b][k][0], k)) for b in range(len(bl))]
    par = 0.0
    for b in range(len(bl)):
        par += stats[b][result[b]][1]
    # ZipSort by decreasing norm; equal norms in block order, NaN norms last (this engine's total order)
    def visit_key(b):
        v = stats[b][result[b]][0]
        return (1, 0.0, b) if math.isnan(v) else (0, -v, b)

    idx = sorted(range(len(bl)), key=visit_key)
    for _ in range(10):
        changed = False
        for b in idx:
            cur = result[b]
            best, best_cost, best_par = cur, 0.0, par
            for k in range(16):
                if k == cur:
                    continue
                npar = par - stats[b][cur][1] + stats[b][k][1]
                pnd = npar * npar - par * par
                if pnd > 0.0:
                    continue
                perp = (stats[b][k][0] - stats[b][cur][0]) - pnd
                cost = mult * pnd + perp
                if cost < best_cost:
                    best, best_cost, best_par = k, cost, npar
            if best != cur:
                result[b] = best
                par = best_par
                changed = True
        if not changed:
            break
    return result


def make_case(seed, d, nsub, n):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, d)) * rng.uniform(0.3, 1.5, (n, 1)) / np.sqrt(d)).astype(F32)
    cents = rng.standard_normal((3, d)).astype(F32)
    cents /= np.linalg.norm(cents, axis=1, keepdims=True)
    assign = rng.integers(0, 3, n)
    cb = (rng.standard_normal(16 * d) * 0.4).astype(F32)
    return x, cents, assign, cb


@pytest.mark.parametrize("d,nsub", [(8, 4), (10, 3), (12, 12), (16, 5)])
@pytest.mark.parametrize("t", [0.0, 0.2, 0.6])
def test_cd_encoder_equals_a_scalar_replay_and_never_raises_the_cost(d, nsub, t):
    x, cents, assign, cb = make_case(d * 100 + nsub, d, nsub, 40)
    codes = ah.encode(x, cb, d, nsub, ah.METRIC_IP, t, cents, assign)
    nb = len(ah.blocks(d, nsub))
    sel = ah.unpack(codes, nb)
    r = x - cents[assign]
    rn, pr, n2 = ah.residual_stats(x, r, cb, d, nsub)
    moved = 0
    for i in range(len(x)):
        assert list(sel[i]) == replay(x[i], r[i], cb, d, nsub, t), i
        eta = ah.eta_of(t, n2[i], d)
        init = np.argmin(rn[i], axis=1)
        moved += int((init != sel[i]).any())
        c0 = ah.anisotropic_cost(rn[i], pr[i], init, eta)
        assert ah.anisotropic_cost(rn[i], pr[i], sel[i], eta) <= c0 + 1e-12 * abs(c0) + 1e-15
    if t >= 0.6:
        assert moved > 0  # the cases exercise actual moves


def test_zero_row_and_negative_threshold_give_plain_codes():
    d, nsub = 12, 4
    x, cents, assign, cb = make_case(5, d, nsub, 30)
    x[3] = 0
    plain = ah.encode(x, cb, d, nsub, ah.METRIC_IP, -1.0, cents, assign)
    nan = ah.encode(x, cb, d, nsub, ah.METRIC_IP, float("nan"), cents, assign)
    shaped = ah.encode(x, cb, d, nsub, ah.METRIC_IP, 0.2, cents, assign)
    assert np.array_equal(plain, nan)
    rn, _, _ = ah.residual_stats(x, x - cents[assign], cb, d, nsub)
    assert np.array_equal(plain, ah.pack(np.argmin(rn, axis=2)))
    assert np.array_equal(shaped[3], plain[3])  # n2 = 0: NaN costs, no move
    assert not np.array_equal(shaped, plain)
    # L2: nearest centres of the raw rows, whatever the threshold
    l2 = ah.encode(x, cb, d, nsub, ah.METRIC_L2, 0.2)
    rn2, _, _ = ah.residual_stats(x, x, cb, d, nsub)
    assert np.array_equal(l2, ah.pack(np.argmin(rn2, axis=2)))


def test_fixed_point_table_by_hand():
    # d 2, one block of 2 dims: centres c_k = (k, 0) for k < 16; q = (2, 5)
    cb = np.zeros((16, 2), F32)
    cb[:, 0] = np.arange(16)
    q = np.array([2, 5], F32)
    lut, m = ah.lut(q, cb.reshape(-1), 2, 1, ah.METRIC_IP)
    # IP: t_k = -2k; max |t| = 30; m = 127 / 30; trunc(-2k * m) + 128
    assert m == F32(127) / F32(30)
    want = [int(np.trunc(F32(-2 * k) * m)) + 128 for k in range(16)]
    # fp32 127 / 30 rounds down, so -30 m = -126.99999 truncates to -126: the largest entry is not at the bound
    assert list(lut[0]) == want and want[0] == 128 and want[15] == 2
    assert want[1] == 128 - 8  # -2 * 4.2333 = -8.47 truncates toward zero
    lut2, m2 = ah.lut(q, cb.reshape(-1), 2, 1, ah.METRIC_L2)
    # L2: t_k = (2 - k)^2 + 25; max 194 at k = 15
    assert m2 == F32(127) / F32(194)
    assert lut2[0][15] == 127 + 128 and lut2[0][2] == int(np.trunc(F32(25) * m2)) + 128
    # scores: entries with codes 15 and 0 in list with leaf 1.5 under IP
    codes = ah.pack(np.array([[15], [0]]))
    s = ah.scores(codes, lut, m, ah.METRIC_IP, F32(1.5))
    inv = F32(1) / m
    assert s[0] == F32(F32(1.5) - F32(-126) * inv) and s[1] == F32(1.5)
    # an all-zero table: the multiplier comes from sqrt(FLT_EPSILON)
    lz, mz = ah.lut(np.zeros(2, F32), cb.reshape(-1), 2, 1, ah.METRIC_IP)
    assert mz == F32(127) / np.sqrt(F32(np.finfo(F32).eps)) and np.all(lz == 128)


def test_nan_rows_and_centres_follow_the_reference_comparisons():
    # std::min_element under `<`: a NaN never becomes the minimum, a NaN first entry stays
    rn = np.array([[3.0, np.nan, 1.0, 1.0] + [5.0] * 12, [np.nan, 0.5, 0.2] + [5.0] * 13, [np.nan] * 16])
    assert list(ah.first_min(rn)) == [2, 0, 0]
    # a row with a NaN coordinate: eta and every parallel component are NaN, so no move; its codes are the initial ones
    d, nsub = 12, 4
    x, cents, assign, cb = make_case(7, d, nsub, 20)
    x[2, 5] = np.nan
    shaped = ah.encode(x, cb, d, nsub, ah.METRIC_IP, 0.6, cents, assign)
    plain = ah.encode(x, cb, d, nsub, ah.METRIC_IP, -1.0, cents, assign)
    assert np.array_equal(shaped[2], plain[2])
    rn, _, _ = ah.residual_stats(x, x - cents[assign], cb, d, nsub)
    assert ah.unpack(plain, 4)[2][1] == 0  # block 1 holds dim 5: every norm NaN, the first centre stays
    # a NaN centre: blocks whose selected norm is NaN are visited last, and the move rule still equals the replay
    cb2 = cb.copy()
    cb2[16 * 3] = np.nan  # block 1, centre 0, first dim
    codes = ah.encode(x[:2], cb2, d, nsub, ah.METRIC_IP, 0.6, cents, assign[:2])
    sel = ah.unpack(codes, 4)
    r = x[:2] - cents[assign[:2]]
    for i in range(2):
        assert list(sel[i]) == replay(x[i], r[i], cb2, d, nsub, 0.6)
