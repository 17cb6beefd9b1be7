"""The fp32 restatements of the IVF-PQ filter caches (cache_reference.py) against their fp64 definitions, without a
GPU: they must be right before the device caches are held to them bit for bit."""
import numpy as np

import cache_reference as CR

F32, F64 = np.float32, np.float64


def codebook(M, dsub, seed, scale=1.0):
    return (np.random.default_rng(seed).normal(0, scale, (M, 256, dsub))).astype(F32)


def test_tables_follow_their_definitions():
    for M, dsub, seed, scale in ((16, 8, 1, 1.0), (8, 4, 2, 30.0), (4, 16, 3, 1e-3)):
        pq = codebook(M, dsub, seed, scale)
        cb8, nrm = CR.pq_tables(pq)
        p64 = pq.astype(F64)
        sb = np.abs(p64).max() / 127
        assert abs(nrm[-2] - sb) <= 1e-7 * sb
        assert np.all(np.abs(p64 / nrm[-2] - cb8) <= 0.5 + 1e-5) and np.abs(cb8).max() == 127
        n64 = (p64 * p64).sum(-1)
        assert np.allclose(nrm[:M * 256], n64.reshape(-1), rtol=dsub * 2.0 ** -23, atol=0)
        assert np.isclose(nrm[-3], n64.max(1).sum(), rtol=(M + dsub) * 2.0 ** -23)
        e64 = ((p64 - F64(nrm[-2]) * cb8) ** 2).sum(-1).max(1).sum()
        assert np.isclose(nrm[-1], np.sqrt(e64), rtol=(M + dsub) * 2.0 ** -22)
        assert nrm[-1] <= np.sqrt(M * dsub) * nrm[-2] / 2 * (1 + 1e-5)  # every element rounded to the nearest step


def test_tables_of_a_zero_codebook_disable_the_filter():
    pq = np.zeros((4, 256, 8), F32)
    pq[1, 7, 3] = 0.0  # all zero: no scale
    cb8, nrm = CR.pq_tables(pq)
    assert not cb8.any() and not nrm.any()


def test_fma_sums_differ_from_plain_fp32_sums():
    """the restatement rounds each product-sum once: on values with long mantissas that differs from the two roundings
    of a plain fp32 multiply-add for some entries, which is what makes a bitwise comparison meaningful"""
    pq = codebook(16, 8, 5, 1.0) * F32(1.0000001)
    _, nrm = CR.pq_tables(pq)
    plain = np.zeros((16, 256), F32)
    for j in range(8):
        plain = (plain + (pq[:, :, j] * pq[:, :, j]).astype(F32)).astype(F32)
    assert (plain.reshape(-1) != nrm[:16 * 256]).any()


def test_entry_norms_sum_in_subquantiser_order():
    M = 16
    rng = np.random.default_rng(7)
    _, nrm = CR.pq_tables(codebook(M, 8, 7))
    codes = rng.integers(0, 256, (500, M), dtype=np.uint8)
    got = CR.entry_norms(codes, nrm, M)
    want = sum(nrm[m * 256 + codes[:, m].astype(np.int64)].astype(F64) for m in range(M))
    assert np.allclose(got, want, rtol=M * 2.0 ** -23, atol=0)
    seq = np.zeros(len(codes), F32)
    for m in range(M):
        seq = seq + nrm[m * 256 + codes[:, m].astype(np.int64)]
    assert np.array_equal(got.view(np.uint32), seq.view(np.uint32))
    assert CR.entry_norms(np.zeros((0, M), np.uint8), nrm, M).shape == (0,)
