"""Every quantised codec of the shared list scan (list_scan.cuh) at the largest shapes its create rule accepts, and next
to them: the boundaries found from the engine, checked against a restatement of the scan's shared-memory formula and
pinned here as constants (DESIGN section 8); codes byte-equal to the CPU twins' encoders on rows the test supplies;
per-query tables and per-entry scores bit-equal to the twins; searched keys exact against tests/topk_reference.py at
k' in {1, 17, the largest k' the shape admits}; one k' past it refused by name.

The large shapes take the scan's generic (MW = 0) code layouts with 65-128-byte codes and 256-entry tiles, odd last
nibbles, wide remainder blocks and a shared-memory total close to the per-CTA limit."""
import re

import numpy as np
import pytest

import float_contract as fc
import topk_reference as R
from oracle_binary import binary_ivf as ob
from oracle_pqfs import twin
from oracle_pqfs.twin import assert_same_results
from oracle_pqnb import ivfpq_nbits as pqnb
from oracle_rabitq import rabitq as rq
from oracle_scann import ah
from test_gpu_topk_keys import PqState, assert_results, entries, make_data
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = R.METRIC_L2, R.METRIC_IP
MNAME = {L2: "L2", IP: "InnerProduct"}
F32 = np.float32


def gi():
    from vearch_b200 import index as gidx
    return gidx


# ---- the scan's shared memory, restated (list_scan.cuh list_scan_smem / list_scan_max_k and the codecs' tiles) ------
LS_NT, LS_NST = 256, 2
CTA_SMEM = 227 * 1024  # sm_90: shared memory of one CTA, static and dynamic
STATIC_RESERVE = 3 * 1024  # kListScanStaticSmem: the kernel's own static arrays
GPU_MAX_K = 2048  # Index::kGpuMaxK


def pow2(x):
    return 1 << max(0, (x - 1).bit_length())


def tile16(cb, group=LS_NT):
    """about 16 KiB of codes per tile, a multiple of `group` entries, between group and 1024 entries"""
    e = 16384 // cb // group * group
    return group if e < group else min(e, 1024)


def scan_smem(scan, k):
    table_bytes, cb, tile, code_sum = scan
    kp = pow2(max(k, 16))
    sortn = pow2(kp + tile + tile // 2)
    return table_bytes + sortn * 8 + LS_NST * tile * cb + (16 if code_sum else 0)


def scan_max_k(scan):
    k = 4096
    while k >= 16:
        if scan_smem(scan, k) <= CTA_SMEM - STATIC_RESERVE:
            return k
        k //= 2
    return 0


def ivfpq_scan(M, nbits):  # (table bytes, code bytes, tile entries, kCodeSum)
    if nbits == 8:
        return M * 256 * 4, M, {8: 1024, 16: 512, 32: 512, 64: 256}.get(M, tile16(M)), False
    cb = (M * nbits + 7) // 8
    return (((M << nbits) + 3) & ~3) * 4, cb, tile16(cb), True


def nibble_scan(nb):  # IVFPQFastScan (nb = M) and VEARCH (nb blocks): the uint16 / int16 byte-pair table
    cb = (nb + 1) // 2
    return cb * 256 * 2, cb, tile16(cb), False


def rabitq_scan(d, B, qb):
    W = (d + 31) // 32
    cb = 4 * (B * W + 3)
    return ((32 + 32 * W + qb * W + 3) & ~3) * 4, cb, tile16(cb, LS_NT // rq.lanes(d)), True


def binary_scan(cs):
    W = (cs + 3) // 4
    return ((W + 3) & ~3) * 4, cs, tile16(cs), True


def largest(pred, hi, step=1):
    x = hi
    while x > 0 and not pred(x):
        x -= step
    return x


# The boundaries, as the engine reports them on the H100 (each equal to the restatement, test_boundaries_*).  IVFPQ at
# 8 bits: every nsubvector <= 146 searches, at k' <= 128 from M = 145; packed codes: the largest M at each nbits, k' <= 128
# there; IVFPQFastScan and VEARCH: the type's own limit of 256, at k' = 4096; IVFRABITQ: d <= 4096 at every nb_bits;
# BINARYIVF: codes of at most 439 bytes (d = 3512 bits), k' <= 128 there.
PQ8_MAX_M = 146
PACKED_MAX_M = {1: 3128, 4: 703, 7: 234}
GPU_IVFPQ_MAX_M = 128
PQFS_MAX_M = 256
VEARCH_MAX_BLOCKS = 256
RABITQ_MAX_D = 4096
BINARY_MAX_CODE = 439
BOUNDARY_K = {"pq8": 128, "packed": 128, "binary": 128}


def restated_boundary(case):
    if case == "IVFPQ8":
        return largest(lambda M: scan_max_k(ivfpq_scan(M, 8)) >= 1, 400)
    if case.startswith("IVFPQ_nbits"):
        nb = int(case[11:])
        return largest(lambda M: scan_max_k(ivfpq_scan(M, nb)) >= 1, 8000)
    if case == "GPU_IVFPQ":
        return largest(lambda M: scan_max_k(ivfpq_scan(M, 8)) >= GPU_MAX_K, 400, 4)
    if case == "IVFPQFastScan":
        return largest(lambda M: scan_max_k(nibble_scan(M)) >= 4096, 256)
    if case == "VEARCH":
        return largest(lambda nb: scan_max_k(nibble_scan(nb)) >= 4096, 256)
    if case == "IVFRABITQ":
        return largest(lambda d: all(scan_max_k(rabitq_scan(d, B, 8)) >= 4096 for B in range(1, 10)), 4096)
    if case == "BINARYIVF":
        return largest(lambda cs: scan_max_k(binary_scan(cs)) >= 1, 2000)
    raise ValueError(case)


PINNED = {"IVFPQ8": PQ8_MAX_M, "IVFPQ_nbits1": PACKED_MAX_M[1], "IVFPQ_nbits4": PACKED_MAX_M[4],
          "IVFPQ_nbits7": PACKED_MAX_M[7], "GPU_IVFPQ": GPU_IVFPQ_MAX_M, "IVFPQFastScan": PQFS_MAX_M,
          "VEARCH": VEARCH_MAX_BLOCKS, "IVFRABITQ": RABITQ_MAX_D, "BINARYIVF": BINARY_MAX_CODE}


def creator(case):
    """(create(x), refusal pattern naming x and the engine's boundary, first x to try past the boundary)"""
    G = gi()
    if case == "IVFPQ8" or case.startswith("IVFPQ_nbits"):
        nb = 8 if case == "IVFPQ8" else int(case[11:])
        return (lambda M: G.GammaIndex("IVFPQ", M, {"ncentroids": 4, "nprobe": 4, "nsubvector": M, "nbits_per_idx": nb,
                                                    "metric_type": "L2"}),
                lambda M: rf"nsubvector \[{M}\] above (\d+) at nbits_per_idx {nb}", 8000)
    if case == "GPU_IVFPQ":  # x = M / 4: nsubvector must be a multiple of 4
        return (lambda j: G.GammaIndex("GPU_IVFPQ", 8 * j, {"ncentroids": 4, "nprobe": 4, "nsubvector": 4 * j}),
                lambda j: rf"GPU_IVFPQ: nsubvector \[{4 * j}\] above (\d+)", 100)
    if case == "IVFPQFastScan":
        return (lambda M: G.GammaIndex("IVFPQFastScan", M, {"ncentroids": 4, "nprobe": 4, "nsubvector": M}),
                lambda M: rf"nsubvector \[{M}\] above (\d+)", 1000)
    if case == "VEARCH":
        return (lambda nb: G.VearchIndex(nb, {"ncentroids": 4, "nsubvector": nb}),
                lambda nb: rf"VEARCH: {nb} blocks \(nsubvector {nb}\) above (\d+)", 1000)
    if case == "IVFRABITQ":
        return (lambda d: G.RaBitQIndex(d, {"ncentroids": 4, "nprobe": 4, "nb_bits": 9}),
                lambda d: rf"IVFRABITQ: dimension \[{d}\] above (\d+)", 8000)
    if case == "BINARYIVF":
        return (lambda cs: G.BinaryIVFIndex(8 * cs, {"ncentroids": 4}),
                lambda cs: rf"BINARYIVF: dimension \[{8 * cs}\] is too large for the list scan", 2000)
    raise ValueError(case)


def engine_boundary(case):
    """bisect create: the largest accepted x, and the boundary the refusal of x + 1 names (None if it names none)"""
    create, pattern, hi = creator(case)
    E = gi().GammaError

    def accepted(x):
        try:
            idx = create(x)
        except E as e:
            assert re.search(pattern(x), str(e)), str(e)
            return False
        idx.close()
        return True

    lo = 1
    assert accepted(lo) and not accepted(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if accepted(mid):
            lo = mid
        else:
            hi = mid
    with pytest.raises(E) as ei:
        create(lo + 1)
    m = re.search(pattern(lo + 1), str(ei.value))
    named = int(m.group(1)) if m.groups() else None
    return (4 * lo if case == "GPU_IVFPQ" else lo), named


@pytest.mark.parametrize("case", list(PINNED))
def test_boundaries_from_the_engine_equal_the_restated_scan(case):
    got, named = engine_boundary(case)
    assert got == PINNED[case] == restated_boundary(case), (got, PINNED[case], restated_boundary(case))
    assert named is None or named == got, named  # the refusal past the boundary names it


def test_restated_k_limits():
    """the k' each boundary shape admits, and the window's size at the tightest ones (no k' past a boundary fits)"""
    assert scan_max_k(ivfpq_scan(PQ8_MAX_M, 8)) == scan_max_k(ivfpq_scan(PQ8_MAX_M - 1, 8)) == BOUNDARY_K["pq8"]
    assert scan_max_k(ivfpq_scan(128, 8)) == GPU_MAX_K and scan_max_k(ivfpq_scan(96, 8)) == 4096
    for nb, M in PACKED_MAX_M.items():
        assert scan_max_k(ivfpq_scan(M, nb)) == BOUNDARY_K["packed"]
    for nb in (255, 256):
        assert scan_max_k(nibble_scan(nb)) == 4096
        assert scan_smem(nibble_scan(nb), 4096) == 192 * 1024  # 64 KiB table, 64 KiB queue, two 32 KiB stages
    assert scan_max_k(binary_scan(BINARY_MAX_CODE)) == BOUNDARY_K["binary"]
    assert scan_smem(rabitq_scan(4096, 9, 8), 4096) <= 157 * 1024


def sorted_keys(dis, ids, metric):
    return np.sort(R.keys(dis, np.where(ids >= 0, ids, 0), ids >= 0, metric), axis=1)


def refused_past(search, kmax, by_recall_num=True):
    """k' = kmax + 1 is refused, never a CUDA error: as topn by name below 4096 (every search entry refuses a topn above
    4096 itself), and as recall_num beside topn 10 by the scan's own limit.  search(k, params)"""
    E = gi().GammaError
    with pytest.raises(E, match=rf"\[{kmax + 1}\] above {kmax}" if kmax < 4096 else "topK or nprobe out of range"):
        search(kmax + 1, None)
    if by_recall_num:
        with pytest.raises(E, match=rf"recall_num / topn \[{kmax + 1}\] above {kmax}"):
            search(10, {"recall_num": kmax + 1})


def dead_bitmap(n, seed, frac=0.2):
    return np.packbits(np.random.default_rng(seed).random(n) < frac, bitorder="little")


def tombstone_second(idx, off, ids, nlist):
    """tombstone the second entry of every list that has one; marks it in the raw ids (in place), as the scan sees it"""
    for l in range(nlist):
        if off[l + 1] - off[l] > 1:
            idx.tombstone(l, 1)
            ids[off[l] + 1] |= np.iinfo(np.int64).min


# ---- IVFPQ, 8-bit codes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M", [(PQ8_MAX_M, PQ8_MAX_M), (2 * (PQ8_MAX_M - 1), PQ8_MAX_M - 1), (192, 96)])
def test_ivfpq_8bit_largest_m(d, M, metric):
    """M = 146 (the largest accepted), 145 and the generic layout at 96: codes, keys at k' up to the shape's limit"""
    kmax = scan_max_k(ivfpq_scan(M, 8))
    n, nq, nlist = 3000, 4, 8
    db, xq = make_data("pool", n, d, nq, metric, seed=M)
    st = PqState("IVFPQ", d, M, 8, nlist, metric, db, xq, seed=M)
    _, codes, _ = st.idx.export_lists()
    vid = st.ids & 0xFFFFFFFF
    assert np.array_equal(codes, pqnb.ivfpq_encode(st.cent, st.pq, db[vid], st.el))
    probes = st.probes(nlist)
    for k in (1, 17, kmax):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQ M={M} k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_scan_kernel"
    dele = dead_bitmap(n, M)
    assert_results(st.search(probes, kmax, del_bitmap=dele), st.ref(probes, kmax, del_bitmap=dele), metric, "deleted")
    refused_past(lambda k, p: st.search(probes, k, params=p), kmax)
    st.idx.close()


# ---- IVFPQ, bit-packed codes --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nbits", [1, 4, 7])
@pytest.mark.parametrize("below", [0, 1])
def test_ivfpq_packed_largest_m(nbits, below, metric):
    """the largest M at nbits 1, 4 and 7 (391-, 352- and 205-byte codes) and one below: codes byte-equal to the twin's
    packing, scores bit-equal to ivfpq_nbits.ivfpq_search_preassigned, keys exact at the shape's largest k'"""
    M = PACKED_MAX_M[nbits] - below
    d, n, nq, nlist = M, 2000, 3, 4
    kmax = scan_max_k(ivfpq_scan(M, nbits))
    assert kmax == BOUNDARY_K["packed"]
    db, xq = make_data("pool", n, d, nq, metric, seed=nbits + below)
    st = PqState("IVFPQ", d, M, nbits, nlist, metric, db, xq, seed=nbits)
    assert st.idx.code_size == pqnb.code_size(M, nbits)
    off, codes, _ = st.idx.export_lists()
    vid = st.ids & 0xFFFFFFFF
    assert np.array_equal(codes, pqnb.ivfpq_encode(st.cent, st.pq, db[vid], st.el))
    probes = st.probes(nlist)
    for k in (1, 17, kmax):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQ nbits={nbits} M={M} k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_packed_scan_kernel"
    T = pqnb.ivfpq_precompute_table(st.cent, st.pq) if metric == L2 else None
    cd = np.take_along_axis(st.coarse, probes, 1).astype(F32)
    dele = dead_bitmap(n, nbits)
    dg, ig = st.search(probes, kmax, del_bitmap=dele)
    do, io = pqnb.ivfpq_search_preassigned(off, codes, st.ids, st.cent, st.pq, T, xq, kmax, probes, cd, metric,
                                           del_bitmap=dele)
    assert_same_results(dg, ig, do, io)
    assert_results((dg, ig), st.ref(probes, kmax, del_bitmap=dele), metric, "deleted")
    refused_past(lambda k, p: st.search(probes, k, params=p), kmax)
    st.idx.close()


# ---- GPU_IVFPQ ----------------------------------------------------------------------------------------------------------
def test_gpu_ivfpq_largest_m():
    d, M, n, nq, nlist = 256, GPU_IVFPQ_MAX_M, 4000, 4, 8
    db, xq = make_data("pool", n, d, nq, L2, seed=7)
    st = PqState("GPU_IVFPQ", d, M, 8, nlist, L2, db, xq, seed=7)
    probes = st.probes(nlist)
    for k in (1, 17, GPU_MAX_K):
        assert_results(st.search(probes, k), st.ref(probes, k), L2, f"GPU_IVFPQ M=128 k'={k}")
        assert st.idx.last_scan_kernel == "ivfpq_scan_kernel"
    with pytest.raises(gi().GammaError, match=rf"\[{GPU_MAX_K + 1}\]"):
        st.search(probes, GPU_MAX_K + 1)
    st.idx.close()
    M1 = GPU_IVFPQ_MAX_M + 4
    with pytest.raises(gi().GammaError, match=rf"nsubvector \[{M1}\] above {GPU_IVFPQ_MAX_M}"):
        gi().GammaIndex("GPU_IVFPQ", 2 * M1, {"ncentroids": 4, "nprobe": 4, "nsubvector": M1})


# ---- IVFPQFastScan ------------------------------------------------------------------------------------------------------
PQFS_SHAPES = [(256, 256), (512, 256), (510, 255), (258, 129)]  # 128-byte codes; an odd nibble; 65 bytes


def float_codebook(db, M, ksub, seed):
    """[M][ksub][dsub]: each sub-quantiser's centres drawn from the rows' sub-vectors"""
    dsub = db.shape[1] // M
    rng = np.random.default_rng(seed)
    rows = db[rng.integers(0, len(db), (M, ksub))]
    return np.stack([rows[m, :, m * dsub:(m + 1) * dsub] for m in range(M)]).astype(F32)


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("regime", ["sift_float", "offset1000"])
@pytest.mark.parametrize("d,M", PQFS_SHAPES)
def test_ivfpqfs_tables_codes_and_scores_bit_equal(d, M, regime, metric):
    n, nq, nlist = 3000, 4, 4
    db, xq = fc.regime(regime, n, d, nq, seed=M)
    pq = float_codebook(db, M, 16, seed=M)
    idx = gi().GammaIndex("IVFPQFastScan", d, {"ncentroids": nlist, "nprobe": nlist, "nsubvector": M,
                                               "metric_type": MNAME[metric]})
    idx.set_centroids(db[:nlist])
    idx.set_pq_centroids(pq)
    idx.add(db)
    off, codes, ids = idx.export_lists()
    want = twin.pack(twin.encode(pq, db))
    assert codes.shape[1] == (M + 1) // 2 and np.array_equal(codes, want[ids])
    lut8, ab = idx.pqfs_lut(xq)
    olut, oab = twin.lut(pq, xq, metric)
    assert np.array_equal(lut8, olut) and np.array_equal(ab.view(np.uint32), oab.view(np.uint32))
    probes = np.tile(np.arange(nlist), (nq, 1))
    dis, got = idx.search_preassigned(xq, n, probes, np.zeros(probes.shape, F32))  # every entry
    assert idx.last_scan_kernel == "ivfpqfs_scan_kernel"
    cu = twin.unpack(codes, M)
    for q in range(nq):
        sc = dict(zip(ids.tolist(), twin.scores(olut[q], oab[q], cu).tolist()))
        assert sorted(got[q].tolist()) == sorted(sc)
        assert np.array_equal(dis[q].view(np.uint32), np.array([sc[v] for v in got[q]], F32).view(np.uint32))
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("d,M", PQFS_SHAPES)
def test_ivfpqfs_keys_exact_at_kprime_4096(d, M, metric):
    n, nq, nlist = 6000, 4, 6
    db, xq = make_data("pool", n, d, nq, metric, seed=M + 1)
    st = PqState("IVFPQFastScan", d, M, 4, nlist, metric, db, xq, seed=M)
    probes = st.probes(nlist)
    for k in (1, 17, 4096):
        assert_results(st.search(probes, k), st.ref(probes, k), metric, f"IVFPQFastScan M={M} k'={k}")
        assert st.idx.last_scan_kernel == "ivfpqfs_scan_kernel"
    dele = dead_bitmap(n, M)
    assert_results(st.search(probes, 4096, del_bitmap=dele), st.ref(probes, 4096, del_bitmap=dele), metric, "deleted")
    for k in (10, 4096):  # recall_num = 4096: the exact re-rank of the 4096 best codes
        want = R.rerank_keys(st.ref(probes, 4096), xq, db, k, metric)
        assert_results(st.search(probes, k, params={"recall_num": 4096}), want, metric, f"re-rank k={k}")
    refused_past(lambda k, p: st.search(probes, k, params=p), 4096)
    st.idx.close()


# ---- VEARCH -------------------------------------------------------------------------------------------------------------
def mips_rows(n, d, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)) / np.sqrt(d)
    return (x * rng.uniform(0.3, 1.5, (n, 1))).astype(F32)


def vearch_index(d, nsub, metric, t, db, cent, cb, **extra):
    p = {"ncentroids": len(cent), "nsubvector": nsub, "metric_type": MNAME[metric], **extra}
    if t is not None:
        p["ns_threshold"] = t
    idx = gi().VearchIndex(d, p)
    idx.set_codebook(cb)
    idx.set_centroids(cent)
    idx.add(db)
    return idx


def vearch_twin_scores(codes, el, cent, cb, xq, d, nsub, metric):
    out = []
    for q in xq:
        tab, m = ah.lut(q, cb, d, nsub, metric)
        s = np.zeros(len(codes), F32)
        for l in np.unique(el):
            sel = el == l
            s[sel] = ah.scores(codes[sel], tab, m, metric, ah.leaf(q, cent[l]) if metric == IP else F32(0))
        out.append(s)
    return np.stack(out)


# (d, nsub, metric, ns_threshold): 256 blocks of 1 and 6 dims; 255 blocks of 3 dims and a 235-dim remainder block; 255
# blocks (an odd last nibble) under IP and L2
VEARCH_SHAPES = [(256, 256, IP, 0.2), (1536, 256, IP, 0.2), (1000, 255, IP, 0.2), (255, 255, IP, 0.2),
                 (255, 255, L2, None)]


@pytest.mark.parametrize("d,nsub,metric,t", VEARCH_SHAPES)
def test_vearch_largest_block_counts(d, nsub, metric, t):
    nlist, nq = 2, 4
    n = 520 if metric == IP else 2000  # the twin's noise-shaped encoder is slow at 256 blocks
    db = mips_rows(n, d, d + nsub)
    cent = (db[:nlist] / np.linalg.norm(db[:nlist], axis=1, keepdims=True)).astype(F32) if metric == IP else db[:nlist]
    cb = (np.random.default_rng(d).standard_normal(16 * d) * 0.3).astype(F32)
    idx = vearch_index(d, nsub, metric, t, db, cent, cb)
    nb = len(ah.blocks(d, nsub))
    assert idx.blocks == nb and idx.code_size == (nb + 1) // 2
    off, codes, ids, el = entries(idx, nlist)
    for l in range(nlist):
        rows = ids[el == l]
        assert np.array_equal(codes[el == l], ah.encode(db[rows], cb, d, nsub, metric, t if t is not None else -1.0,
                                                        cent, np.full(len(rows), l)))
    xq = mips_rows(nq, d, 99)
    lut, mult = idx.lut(xq)
    for j, q in enumerate(xq):
        tab, m = ah.lut(q, cb, d, nsub, metric)
        assert np.array_equal(lut[j], tab) and mult[j].view(np.uint32) == m.view(np.uint32)
    scores = vearch_twin_scores(codes, el, cent, cb, xq, d, nsub, metric)
    probes = np.tile(np.arange(nlist), (nq, 1))
    cd = np.zeros(probes.shape, F32)
    dis, got = idx.search_preassigned(xq, n, probes, cd)  # every entry
    for q in range(nq):
        want = dict(zip(ids.tolist(), scores[q].tolist()))
        assert sorted(got[q].tolist()) == sorted(want)
        assert np.array_equal(dis[q].view(np.uint32), np.array([want[v] for v in got[q]], F32).view(np.uint32))
    for k in (1, 17, 4096):
        dis, got = idx.search_preassigned(xq, k, probes, cd)
        assert np.array_equal(sorted_keys(dis, got, metric), R.search_entries(scores, el, ids, probes, k, metric))
        assert idx.last_scan_kernel == "vearch_scan_kernel"
    tombstone_second(idx, off, ids, nlist)
    dele = dead_bitmap(n, d)
    dis, got = idx.search_preassigned(xq, 4096, probes, cd, del_bitmap=dele)
    assert np.array_equal(sorted_keys(dis, got, metric),
                          R.search_entries(scores, el, ids, probes, 4096, metric, del_bitmap=dele))
    refused_past(lambda k, p: idx.search_preassigned(xq, k, probes, cd, params=p), 4096, by_recall_num=False)
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
def test_vearch_reordering_at_recall_num_4096(metric):
    """256 blocks, reordering: the k best by exact score of the twin's 4096 best codes (integer rows)"""
    d, nsub, nlist, n, nq = 256, 256, 3, 6000, 3
    rng = np.random.default_rng(31)
    db = rng.integers(-6, 7, (n, d)).astype(F32)
    xq = rng.integers(-6, 7, (nq, d)).astype(F32)
    cent = db[:nlist] / np.linalg.norm(db[:nlist], axis=1, keepdims=True) if metric == IP else db[:nlist]
    cent = cent.astype(F32)
    cb = (rng.standard_normal(16 * d) * 3).astype(F32)
    idx = vearch_index(d, nsub, metric, -1.0 if metric == IP else None, db, cent, cb, reordering=True)
    _, codes, ids, el = entries(idx, nlist)
    scores = vearch_twin_scores(codes, el, cent, cb, xq, d, nsub, metric)
    probes = np.tile(np.arange(nlist), (nq, 1))
    cand = R.search_entries(scores, el, ids, probes, 4096, metric)
    for k in (10, 4096):
        dis, got = idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, F32), params={"recall_num": 4096})
        assert idx.last_scan_kernel == "vearch_scan_kernel"
        assert np.array_equal(sorted_keys(dis, got, metric), R.rerank_keys(cand, xq, db, k, metric))
    refused_past(lambda k, p: idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, F32), params=p), 4096)
    idx.close()


def test_vearch_257_blocks_refused():
    with pytest.raises(gi().GammaError, match=r"257 blocks \(nsubvector 257\) above 256"):
        gi().VearchIndex(257, {"ncentroids": 4, "nsubvector": 257})
    with pytest.raises(gi().GammaError, match=r"257 blocks \(nsubvector 256\) above 256"):
        gi().VearchIndex(1000, {"ncentroids": 4, "nsubvector": 256})  # 256 blocks of 3 dims and one of 232


# ---- IVFRABITQ ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", ["normal", "offset1000"])
@pytest.mark.parametrize("B", [1, 9])
@pytest.mark.parametrize("d", [1024, 3000, 4095, 4096])
def test_rabitq_encoder_byte_equal_above_768(d, B, regime):
    n = 8 if B == 9 else 48
    if regime == "normal":
        x = np.random.default_rng(d + B).standard_normal((n, d)).astype(F32)
    else:
        x, _ = fc.regime(regime, n, d, 1, seed=d + B)
    cent = (x[:4] * F32(0.5)).astype(F32)
    idx = gi().RaBitQIndex(d, {"ncentroids": 4, "nprobe": 4, "nb_bits": B})
    idx.set_centroids(cent)
    assign = np.arange(n) % 4
    got = idx.encode(x, assign)
    assert got.shape == (n, rq.code_bytes(d, B)) == (n, idx.code_size)
    assert np.array_equal(got, rq.encode(x, cent, assign, B))
    idx.close()


@pytest.mark.parametrize("metric", [L2, IP])
def test_rabitq_scan_at_d_4096(metric):
    """d = 4096, nb_bits 9: list entries are the encoder's, estimates bit-equal to the twin at qb 0 and 8, keys exact at
    k' in {1, 17, 4096}, d = 4097 refused"""
    d, B, nlist, n, nq = RABITQ_MAX_D, 9, 2, 400, 3
    db = np.random.default_rng(41).standard_normal((n, d)).astype(F32)
    cent = db[:nlist].copy()
    idx = gi().RaBitQIndex(d, {"ncentroids": nlist, "nprobe": nlist, "nb_bits": B, "metric_type": MNAME[metric]})
    idx.set_centroids(cent)
    idx.add(db)
    off, codes, ids, el = entries(idx, nlist)
    assert np.array_equal(codes, idx.encode(db[ids], el))
    xq = np.random.default_rng(42).standard_normal((nq, d)).astype(F32)
    probes = np.tile(np.arange(nlist), (nq, 1))
    cd = np.zeros(probes.shape, F32)
    tombstone_second(idx, off, ids, nlist)
    dele = dead_bitmap(n, 43)
    for qb in (0, 8):
        scores = np.stack([np.concatenate([rq.estimate(codes[el == l], xq[j], cent[l], d, B, metric, qb)
                                           for l in range(nlist)]) for j in range(nq)])
        est = idx.estimate(np.repeat(xq, nlist, 0), np.tile(np.arange(nlist), nq), qb=qb)
        for j in range(nq):
            got = np.concatenate(est[j * nlist:(j + 1) * nlist])
            assert np.array_equal(got.view(np.uint32), scores[j].view(np.uint32)), qb
        for k, kw in ((1, {}), (17, {}), (4096, {}), (4096, {"del_bitmap": dele})):
            dis, got = idx.search_preassigned(xq, k, probes, cd, params={"qb": qb}, **kw)
            assert idx.last_scan_kernel == "rabitq_scan_kernel"
            assert np.array_equal(sorted_keys(dis, got, metric), R.search_entries(scores, el, ids, probes, k, metric, **kw))
    refused_past(lambda k, p: idx.search_preassigned(xq, k, probes, cd, params=p), 4096)
    idx.close()
    with pytest.raises(gi().GammaError, match=r"dimension \[4097\] above 4096"):
        gi().RaBitQIndex(4097, {"ncentroids": 4, "nprobe": 4})


def test_rabitq_rerank_at_d_4096():
    d, B, nlist, n, nq, metric = RABITQ_MAX_D, 9, 2, 4200, 2, L2
    rng = np.random.default_rng(51)
    db = rng.integers(-6, 7, (n, d)).astype(F32)
    xq = rng.integers(-6, 7, (nq, d)).astype(F32)
    cent = db[:nlist].copy()
    idx = gi().RaBitQIndex(d, {"ncentroids": nlist, "nprobe": nlist, "nb_bits": B, "metric_type": "L2"})
    idx.set_centroids(cent)
    idx.add(db)
    _, codes, ids, el = entries(idx, nlist)
    qb = idx.qb
    scores = np.stack([np.concatenate([rq.estimate(codes[el == l], xq[j], cent[l], d, B, metric, qb)
                                       for l in range(nlist)]) for j in range(nq)])
    probes = np.tile(np.arange(nlist), (nq, 1))
    cand = R.search_entries(scores, el, ids, probes, 4096, metric)
    for k in (10, 4096):
        dis, got = idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, F32), params={"recall_num": 4096})
        assert idx.last_scan_kernel == "rabitq_scan_kernel"
        assert np.array_equal(sorted_keys(dis, got, metric), R.rerank_keys(cand, xq, db, k, metric))
    idx.close()


# ---- BINARYIVF ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cs", [BINARY_MAX_CODE, BINARY_MAX_CODE - 4])
def test_binaryivf_largest_code_size(cs):
    kmax = scan_max_k(binary_scan(cs))
    n, nq, nlist = 3000, 4, 4
    db = synth.binary_clustered(n, cs * 8, seed=cs, n_clusters=16, flip=0.2)
    xq = synth.binary_clustered(nq, cs * 8, seed=cs + 1, n_clusters=16, flip=0.2)
    idx = gi().BinaryIVFIndex(cs * 8, {"ncentroids": nlist})
    idx.set_centroids(db[np.random.default_rng(cs).choice(n, nlist, replace=False)])
    idx.add_vectors(db)
    idx.add_pending()
    off, codes, ids, el = entries(idx, nlist)
    assert np.array_equal(codes, db[ids])  # list entries are the raw bytes
    probes = np.tile(np.arange(nlist), (nq, 1))
    scores = ob.hamming(xq, codes)
    for k in (1, 17, kmax):
        dis, got = idx.search_preassigned(xq, k, probes)
        assert idx.last_scan_kernel == "binary_ivf_scan_kernel"
        assert np.array_equal(sorted_keys(dis, got, L2), R.search_entries(scores, el, ids, probes, k, L2))
    tombstone_second(idx, off, ids, nlist)
    dele = dead_bitmap(n, cs)
    dis, got = idx.search_preassigned(xq, kmax, probes, del_bitmap=dele)
    assert np.array_equal(sorted_keys(dis, got, L2), R.search_entries(scores, el, ids, probes, kmax, L2, del_bitmap=dele))
    with pytest.raises(gi().GammaError, match=rf"topK \[{kmax + 1}\] above {kmax}"):
        idx.search_preassigned(xq, kmax + 1, probes)
    idx.close()
