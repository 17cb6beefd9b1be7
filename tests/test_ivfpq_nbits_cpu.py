"""IVF-PQ at nbits_per_idx 1..8 without a GPU: faiss's bit packing (PQEncoderGeneric), the ksub-generic oracle
(oracle_pqnb) against the 8-bit oracle and against a numpy float32 restatement of the ADC scan, and the general-nbits
"IwPQ" index-file restatement (used by the GPU tests) against tests/gamma_index_file.py at nbits = 8."""
import struct

import numpy as np
import pytest

import gamma_index_file as gif
from oracle import oracle as orc
from oracle_pqnb import ivfpq_nbits as pqnb
from vearch_b200 import synth

L2, IP = orc.METRIC_L2, orc.METRIC_IP


def write_ivfpq_nbits(d, metric, nprobe, centroids, pq_centroids, list_off, codes, ids, ntotal, opq=None):
    """GammaIVFPQIndex::Dump (index/impl/gamma_index_ivfpq.cc:1019-1051) at any nbits: write_product_quantizer
    (index/index_io.cc:92-98) stores code_size = ceil(M nbits / 8), nbits and the [M][2^nbits][dsub] centroids, and the
    lists carry code_size-byte packed rows.  The ivf header and the list block are gamma_index_file's."""
    nlist = len(list_off) - 1
    pq = np.ascontiguousarray(pq_centroids, np.float32)
    M, ksub, dsub = pq.shape
    nbits = ksub.bit_length() - 1
    assert (1 << nbits) == ksub and dsub == d // M
    cs = pqnb.code_size(M, nbits)
    out = gif.fourcc("IwPQ") + gif._ivf_header(d, ntotal, metric, nlist, nprobe, centroids)
    out += struct.pack("<?QQQQQ", True, cs, d, M, nbits, pq.size) + pq.tobytes()
    if opq is not None:
        A = np.ascontiguousarray(opq, np.float32)
        assert A.shape == (d, d)
        out += gif.fourcc("LTra") + struct.pack("<?Q", False, A.size) + A.tobytes() + struct.pack("<Qii?", 0, d, d, True)
    out += gif._inverted_lists(list_off, codes, ids, cs)
    return out


def test_pack_codes_known_answers():
    # M = 3, nbits = 6: bits 0-5 = 0x2A, 6-11 = 0x15, 12-17 = 0x3F
    assert pqnb.pack_codes(np.array([[0x2A, 0x15, 0x3F]], np.uint8), 6).tobytes() == bytes([0x6A, 0xF5, 0x03])
    # M = 3, nbits = 4: code 2j in the low nibble of byte j, 2j + 1 in the high one (IVFPQFastScan's packing too)
    assert pqnb.pack_codes(np.array([[1, 2, 3]], np.uint8), 4).tobytes() == bytes([0x21, 0x03])
    # nbits = 8 is one byte per code
    assert pqnb.pack_codes(np.array([[7, 200, 255]], np.uint8), 8).tobytes() == bytes([7, 200, 255])


@pytest.mark.parametrize("nbits", range(1, 9))
@pytest.mark.parametrize("M", [1, 3, 8, 16, 17, 22])
def test_pack_round_trip(nbits, M):
    rng = np.random.default_rng(nbits * 100 + M)
    codes = rng.integers(0, 1 << nbits, (257, M)).astype(np.uint8)
    packed = pqnb.pack_codes(codes, nbits)
    assert packed.shape == (257, pqnb.code_size(M, nbits)) and pqnb.code_size(M, nbits) == -(-M * nbits // 8)
    assert np.array_equal(pqnb.unpack_codes(packed, M, nbits), codes)
    # unused high bits of the last byte are zero
    tail = M * nbits % 8
    if tail:
        assert not (packed[:, -1] >> tail).any()
    # the layout by definition: bit b of the row is bit b % nbits of code b // nbits
    bits = np.unpackbits(packed, axis=1, bitorder="little")
    b = np.arange(M * nbits)
    assert np.array_equal(bits[:, b], (codes[:, b // nbits] >> (b % nbits)) & 1)


def _state(d, M, nbits, n=3000, nlist=16, seed=0, rounded=False):
    db = synth.sift_like(n, d, seed=seed + 1, rounded=rounded)
    cent, _, _ = orc.kmeans(db[:2000], nlist, niter=4, seed=1234 + seed)
    a = orc.assign(cent, db, L2)
    pq = pqnb.pq_train(db[:2000] - cent[a[:2000]], M, 1 << nbits, niter=3)
    return db, cent, a, pq


def test_nbits8_entry_points_equal_the_8bit_oracle():
    d, M, nlist = 32, 8, 16
    db, cent, a, pq = _state(d, M, 8, nlist=nlist)
    assert pq.shape == (M, 256, d // M) and np.array_equal(pq, orc.pq_train(db[:2000] - cent[a[:2000]], M, niter=3))
    resid = db - cent[a]
    assert np.array_equal(pqnb.pq_compute_codes(pq, resid), orc.pq_compute_codes(pq, resid))
    codes = orc.ivfpq_encode(cent, pq, db, a)
    assert np.array_equal(pqnb.ivfpq_encode(cent, pq, db, a), codes)
    T = orc.ivfpq_precompute_table(cent, pq)
    assert np.array_equal(pqnb.ivfpq_precompute_table(cent, pq), T)
    off, order = orc.build_lists(a, nlist)
    xq = synth.sift_like(20, d, seed=9)
    for metric in (L2, IP):
        cd, keys = orc.coarse_search(cent, xq, 4, metric)
        Tm = T if metric == L2 else None
        for kw in ({}, {"recall_num": 30, "raw": db}):
            want = orc.ivfpq_search_preassigned(off, codes[order], order, cent, pq, Tm, xq, 10, keys, cd, metric, **kw)
            got = pqnb.ivfpq_search_preassigned(off, codes[order], order, cent, pq, Tm, xq, 10, keys, cd, metric, **kw)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def _numpy_adc(off, packed, ids, cent, pq, xq, k, keys, coarse_dis, metric):
    """search_preassigned restated in numpy float32: table entries added one at a time in code order, each add rounded
    to fp32 (scan_list_with_table, gamma_index_ivfpq.h:923-953).  L2 uses the precomputed table, dis0 = coarse
    distance; IP uses the inner-product table, dis0 = <x, centroid> (exact on integer data, whatever the order)."""
    M, ksub, dsub = pq.shape
    nbits = ksub.bit_length() - 1
    codes = pqnb.unpack_codes(packed, M, nbits)
    f32 = np.float32
    # ip[q][m][c] and T[l][m][c], each a sequential fp32 sum over the dsub coordinates
    ip = np.zeros((xq.shape[0], M, ksub), f32)
    nrm = np.zeros((M, ksub), f32)
    cip = np.zeros((cent.shape[0], M, ksub), f32)
    for j in range(dsub):
        xj = xq[:, j::dsub][:, :M].astype(f32)          # [nq][M]: coordinate m * dsub + j
        cj = cent[:, j::dsub][:, :M].astype(f32)        # [nlist][M]
        pj = pq[:, :, j]                                 # [M][ksub]
        ip = ip + xj[:, :, None] * pj[None]
        nrm = nrm + pj * pj
        cip = cip + cj[:, :, None] * pj[None]
    T = nrm[None] + f32(2) * cip
    out_d = np.full((xq.shape[0], k), np.inf if metric == L2 else -np.inf, f32)
    out_i = np.full((xq.shape[0], k), -1, np.int64)
    for q in range(xq.shape[0]):
        dis_all, id_all = [], []
        for p in range(keys.shape[1]):
            l = keys[q, p]
            b, e = off[l], off[l + 1]
            if b == e:
                continue
            if metric == L2:
                tab, dis0 = T[l] + f32(-2) * ip[q], coarse_dis[q, p]
            else:
                tab, dis0 = ip[q], f32(np.dot(xq[q].astype(np.float64), cent[l].astype(np.float64)))
            dis = np.full(e - b, dis0, f32)
            for m in range(M):
                dis = dis + tab[m][codes[b:e, m]]
            dis_all.append(dis)
            id_all.append(ids[b:e])
        dis, vid = np.concatenate(dis_all), np.concatenate(id_all)
        order = np.lexsort((vid, dis if metric == L2 else -dis))[:k]
        out_d[q, :len(order)], out_i[q, :len(order)] = dis[order], vid[order]
    return out_d, out_i


@pytest.mark.parametrize("nbits", range(1, 8))
@pytest.mark.parametrize("metric", [L2, IP])
def test_packed_adc_search_equals_numpy_restatement(nbits, metric):
    d, M, nlist, k = 30, 15, 16, 20
    rounded = metric == IP  # IP's dis0 is an 8-lane sum in the oracle: exact on integer data only
    db, cent, a, pq = _state(d, M, nbits, nlist=nlist, seed=nbits, rounded=rounded)
    if rounded:
        pq, cent = np.round(pq), np.round(cent)
    packed = pqnb.ivfpq_encode(cent, pq, db, a)
    assert packed.shape == (len(db), pqnb.code_size(M, nbits))
    off, order = orc.build_lists(a, nlist)
    codes, ids = packed[order], order
    xq = synth.sift_like(12, d, seed=50 + nbits, rounded=rounded)
    cd, keys = orc.coarse_search(cent, xq, 5, metric)
    T = pqnb.ivfpq_precompute_table(cent, pq) if metric == L2 else None
    do, io = pqnb.ivfpq_search_preassigned(off, codes, ids, cent, pq, T, xq, k, keys, cd, metric)
    dn, i_n = _numpy_adc(off, codes, ids, cent, pq, xq, k, keys, cd, metric)
    assert np.array_equal(do, dn)
    for q in range(len(xq)):  # ids equal up to the membership of the tie group at the k-th score
        inner = do[q] != do[q, -1]
        assert set(io[q][inner]) == set(i_n[q][inner])


def test_iwpq_restatement_matches_the_8bit_writer():
    d, M, nlist = 32, 8, 16
    db, cent, a, pq = _state(d, M, 8, nlist=nlist)
    off, order = orc.build_lists(a, nlist)
    codes = orc.ivfpq_encode(cent, pq, db, a)[order]
    ids = order.copy()
    ids[3] |= orc.DEL_MASK
    A = np.linalg.qr(np.random.default_rng(1).normal(size=(d, d)))[0].astype(np.float32)
    for metric in (L2, IP):
        for opq in (None, A):
            want = gif.write_ivfpq(d, metric, 8, cent, pq, off, codes, ids, len(db), opq=opq)
            assert write_ivfpq_nbits(d, metric, 8, cent, pq, off, codes, ids, len(db), opq=opq) == want
    # below 8 bits: code_size, nbits and the centroid count change, the rest of the layout does not
    pq4 = pqnb.pq_train(db[:2000] - cent[a[:2000]], M, 16, niter=2)
    packed = pqnb.ivfpq_encode(cent, pq4, db, a)[order]
    buf = write_ivfpq_nbits(d, L2, 8, cent, pq4, off, packed, ids, len(db))
    head = len(gif.fourcc("IwPQ") + gif._ivf_header(d, len(db), L2, nlist, 8, cent))
    assert struct.unpack_from("<?QQQQQ", buf, head) == (True, 4, d, M, 4, pq4.size)
    assert len(buf) == len(gif.write_ivfpq(d, L2, 8, cent, pq, off, codes, ids, len(db))) - (pq.size - pq4.size) * 4 - \
        len(db) * (M - 4)
