"""BINARYIVF restated in numpy: faiss IndexBinaryIVF as gamma's GammaIndexBinaryIVF drives it.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py.  Each rule cites the reference line it restates:
  - packing: bit i of a vector is bit (i & 7) of byte i >> 3 (faiss binary_to_real, utils/hamming.cpp), i.e.
    numpy.packbits(..., bitorder="little");
  - training (gamma_index_binary_ivf.cc:212-267): the first `sample_size` stored rows, expanded to +-1 floats, clustered
    by faiss Clustering (niter 10, gamma_index_binary_ivf.cc:97) under an IndexFlatL2; centroids packed back by sign
    (real_to_binary: a component > 0 is bit 1);
  - coarse search (gamma_index_binary_ivf.cc:309-312): IndexBinaryFlat, the nprobe Hamming-nearest centroids, the
    smaller list id first among equal distances;
  - list scan (search_knn_hamming_heap, faiss IndexBinaryIVF.cpp): lists in probe order, entries in list order; an entry
    counts when it is live (tombstone, deletion and filter bitmaps: RetrievalContext::IsValid), inside the score window
    (IsSimilarScoreValid), and strictly below the heap's worst (dis < simi[0]): the first-seen entry wins a tie at the
    boundary;
  - Hamming distance over every byte of the code.  The reference's scanner (select_IVFBinaryScannerL2) hands a code size
    outside {4, 8, 16, 20, 32, 64} to HammingComputer8 / HammingComputer4, which read only the first 8 / 4 bytes;
    `reference_scanner_distance` restates that truncation, and this engine deliberately counts every bit instead.
"""
import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def binary_to_real(x, d):
    """[n, d / 8] uint8 -> [n, d] float32 of +-1 (gamma_index_binary_ivf.cc:257-267 -> faiss binary_to_real)"""
    bits = np.unpackbits(np.asarray(x, np.uint8), axis=1, bitorder="little")[:, :d]
    return np.where(bits == 1, np.float32(1), np.float32(-1)).astype(np.float32)


def real_to_binary(xf):
    """[n, d] float -> [n, d / 8] uint8, bit = component > 0 (faiss real_to_binary)"""
    return np.packbits(np.asarray(xf) > 0, axis=1, bitorder="little")


def hamming(a, b):
    """[na, nb] int64 Hamming distances of packed rows, every byte counted"""
    a = np.asarray(a, np.uint8)
    b = np.asarray(b, np.uint8)
    x = a[:, None, :] ^ b[None, :, :]
    return np.unpackbits(x, axis=2).sum(2).astype(np.int64)


def reference_scanner_distance(a, b):
    """the distance the reference's list scanner computes (select_IVFBinaryScannerL2): full for code sizes 4, 8, 16, 20,
    32 and 64; otherwise only the first 8 bytes (a multiple of 8) or the first 4 (a multiple of 4)"""
    cs = np.asarray(a).shape[1]
    if cs in (4, 8, 16, 20, 32, 64):
        return hamming(a, b)
    if cs % 8 == 0:
        return hamming(np.asarray(a)[:, :8], np.asarray(b)[:, :8])
    if cs % 4 == 0:
        return hamming(np.asarray(a)[:, :4], np.asarray(b)[:, :4])
    return hamming(a, b)  # HammingComputerDefault


def sample_size(nlist, training_threshold):
    """rows Indexing trains on (gamma_index_binary_ivf.cc:220-240)"""
    if training_threshold < nlist:
        return nlist * 39
    if training_threshold <= nlist * 256:
        return training_threshold
    return nlist * 256


def default_training_threshold(nlist):
    """Init without a table threshold: nlist * min_points_per_centroid (gamma_index_binary_ivf.cc:89-93)"""
    return nlist * 39


def coarse_search(xq, centroids, nprobe):
    """(distances int64, list ids) of the nprobe nearest centroids, ties to the smaller id (IndexBinaryFlat)"""
    d = hamming(xq, centroids)
    order = np.lexsort((np.broadcast_to(np.arange(d.shape[1]), d.shape), d), axis=1)[:, :nprobe]
    return np.take_along_axis(d, order, 1), order


def assign(x, centroids):
    return coarse_search(x, centroids, 1)[1][:, 0]


def _bit(bitmap, vid):
    return (int(bitmap[vid >> 3]) >> (vid & 7)) & 1


def search_knn_hamming_heap(xq, lists, probes, k, del_bitmap=None, filter_bitmap=None, min_score=-FLT_MAX,
                            max_score=FLT_MAX):
    """lists: {list id: (codes [n, cs] uint8, raw ids [n] int64, top bit set = tombstone)}; probes [nq, nprobe].
    -> (dis [nq, k] float32 ascending, ids [nq, k], -1 / FLT_MAX for empty slots)"""
    nq = len(xq)
    out_d = np.full((nq, k), np.float32(FLT_MAX), np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    for q in range(nq):
        heap = []  # (dis, seen order, vid): a CMax heap, the worst at the end after sorting
        seen = 0
        for l in probes[q]:
            if l < 0 or l not in lists:
                continue
            codes, ids = lists[l]
            if len(codes) == 0:
                continue
            dis = hamming(xq[q:q + 1], codes)[0]
            for j in range(len(codes)):
                raw = int(ids[j])
                if raw < 0:
                    continue
                vid = raw & 0xFFFFFFFF
                if filter_bitmap is not None and not _bit(filter_bitmap, vid):
                    continue
                if del_bitmap is not None and _bit(del_bitmap, vid):
                    continue
                s = float(np.float32(dis[j]))
                if not (min_score <= s <= max_score):
                    continue
                if len(heap) < k:
                    heap.append((s, seen, vid))
                else:
                    worst = max(heap, key=lambda t: (t[0], t[1]))
                    if s < worst[0]:  # strict: an equal distance never displaces an entry already kept
                        heap.remove(worst)
                        heap.append((s, seen, vid))
                seen += 1
        heap.sort(key=lambda t: (t[0], t[2]))
        for i, (s, _, vid) in enumerate(heap):
            out_d[q, i] = s
            out_i[q, i] = vid
    return out_d, out_i
