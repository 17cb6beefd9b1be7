"""IVF-PQ at nbits_per_idx 1..8: the oracle of oracle/oracle.py made ksub-generic, plus faiss's bit packing.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py.  The reference's IVFPQ takes any nbits (pq.nbits = nbits_per_idx,
internal/engine/index/impl/gamma_index_ivfpq.cc:182; the "!= 8" check is commented out in IVFPQModelParams::Validate,
gamma_index_ivfpq.h:1223-1224) and stores codes the way faiss's PQEncoderGeneric writes them; its scanner reads them
back through PQDecoder (gamma_index_ivfpq.h:284-285, 398, 532-536): code m sits at bits [m nbits, (m + 1) nbits) of
the entry, bits counted LSB-first (bit b = bit b % 8 of byte b / 8), unused high bits of the last byte zero.

The arithmetic is the 8-bit oracle's own (oracle/gamma_oracle.c, compiled with -ffp-contract=off), reached by padding
the codebook to 256 centroids per sub-quantiser:
  - encode: padding centroids at +inf are never strictly nearer than a real one, so the argmin (first minimum wins)
    over the 256 is the argmin over the ksub real centroids, each distance summed in the same order;
  - precomputed table T[l][m][c] = |pq_m[c]|^2 + 2 <centroid_l|m, pq_m[c]>: entries c < ksub are computed exactly as
    at ksub = 256 and the padding columns are dropped;
  - search_preassigned: codes < ksub never index a padding column, so every score is dis0 + tab[m][code_m] added for
    m = 0..M-1 one fp32 add at a time (scan_list_with_table, gamma_index_ivfpq.h:923-953), with the same heaps,
    filters, score window and exact re-rank.
At nbits = 8 every entry point returns what the oracle/oracle.py function of the same name returns, byte for byte.
"""
import numpy as np

from oracle import oracle as orc

ORC_KSUB = 256  # the 8-bit oracle's ksub


def code_size(M, nbits):
    """faiss ProductQuantizer::code_size = ceil(M nbits / 8)."""
    return (M * nbits + 7) // 8


def pack_codes(codes, nbits):
    """[n][M] codes (each < 2^nbits) -> [n][code_size(M, nbits)] bytes in PQEncoderGeneric's layout."""
    codes = np.ascontiguousarray(codes, np.uint8)
    n, M = codes.shape
    assert 1 <= nbits <= 8 and int(codes.max(initial=0)) < (1 << nbits)
    # bit b of the entry = bit (b % nbits) of code b // nbits, for b < M nbits; zero above
    bits = ((codes[:, :, None] >> np.arange(nbits, dtype=np.uint8)) & 1).reshape(n, M * nbits)
    cs = code_size(M, nbits)
    padded = np.zeros((n, cs * 8), np.uint8)
    padded[:, :M * nbits] = bits
    return np.packbits(padded, axis=1, bitorder="little")


def unpack_codes(packed, M, nbits):
    """The inverse of pack_codes: [n][code_size] bytes -> [n][M] codes."""
    packed = np.ascontiguousarray(packed, np.uint8)
    n = packed.shape[0]
    assert packed.shape[1] == code_size(M, nbits)
    bits = np.unpackbits(packed, axis=1, bitorder="little")[:, :M * nbits].reshape(n, M, nbits)
    return (bits << np.arange(nbits, dtype=np.uint8)).sum(axis=2, dtype=np.uint32).astype(np.uint8)


def _nbits_of(ksub):
    nbits = int(ksub).bit_length() - 1
    assert 1 <= nbits <= 8 and (1 << nbits) == ksub, f"ksub {ksub} is not 2^nbits with nbits in 1..8"
    return nbits


def _pad_codebook(pq, fill):
    """[M][ksub][dsub] -> [M][256][dsub], columns ksub.. filled with `fill`."""
    pq = np.ascontiguousarray(pq, np.float32)
    M, ksub, dsub = pq.shape
    if ksub == ORC_KSUB:
        return pq
    out = np.full((M, ORC_KSUB, dsub), fill, np.float32)
    out[:, :ksub] = pq
    return out


def pq_train(x, M, ksub, niter=25, seed=1234):
    """ProductQuantizer::train with ksub = 2^nbits: M independent ksub-means (ClusteringParameters defaults, at most
    256 points per centroid) on the dsub-wide slices, as orc.pq_train does for 256."""
    x = np.ascontiguousarray(x, np.float32)
    if ksub == ORC_KSUB:
        return orc.pq_train(x, M, niter=niter, seed=seed)
    dsub = x.shape[1] // M
    out = np.empty((M, ksub, dsub), np.float32)
    for m in range(M):
        out[m], _, _ = orc.kmeans(x[:, m * dsub:(m + 1) * dsub], ksub, niter=niter, seed=seed)
    return out


def pq_compute_codes(pq, x):
    """pq.compute_codes before packing (gamma_index_ivfpq.cc:494): [n][M] codes, argmin over ksub, first minimum."""
    _nbits_of(pq.shape[1])
    return orc.pq_compute_codes(_pad_codebook(pq, np.inf), x)


def ivfpq_encode(coarse_centroids, pq, x, assign_ids):
    """GammaIVFPQIndex::Add (gamma_index_ivfpq.cc:455-540): residual codes, packed at nbits = log2(ksub)."""
    nbits = _nbits_of(pq.shape[1])
    codes = orc.ivfpq_encode(coarse_centroids, _pad_codebook(pq, np.inf), x, assign_ids)
    return codes if nbits == 8 else pack_codes(codes, nbits)


def ivfpq_precompute_table(coarse_centroids, pq):
    """IndexIVFPQ::precompute_table: [nlist][M][ksub]."""
    ksub = pq.shape[1]
    _nbits_of(ksub)
    T = orc.ivfpq_precompute_table(coarse_centroids, _pad_codebook(pq, 0.0))
    return T if ksub == ORC_KSUB else np.ascontiguousarray(T[:, :, :ksub])


def ivfpq_search_preassigned(list_off, list_codes, list_ids, coarse_centroids, pq, precomputed_table, xq, k, keys,
                             coarse_dis, metric, **kw):
    """GammaIVFPQIndex::search_preassigned over packed list codes ([n][code_size] bytes); keyword arguments as
    orc.ivfpq_search_preassigned (recall_num, raw, del_bitmap, filter_bitmap, min_score, max_score)."""
    M, ksub, _ = pq.shape
    nbits = _nbits_of(ksub)
    codes = np.ascontiguousarray(list_codes, np.uint8)
    T = precomputed_table
    if nbits != 8:
        codes = unpack_codes(codes.reshape(-1, code_size(M, nbits)), M, nbits)
        if T is not None:
            T = np.zeros((T.shape[0], M, ORC_KSUB), np.float32)
            T[:, :, :ksub] = precomputed_table
    return orc.ivfpq_search_preassigned(list_off, codes, list_ids, coarse_centroids, _pad_codebook(pq, 0.0), T, xq, k,
                                        keys, coarse_dis, metric, **kw)
