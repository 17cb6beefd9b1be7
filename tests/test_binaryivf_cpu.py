"""BINARYIVF oracle (oracle_binary) on the CPU: packing, Hamming distance, the heap's tie rule, the training sample
size, and the one distance this engine computes differently from the reference (every bit, at every code size)."""
import numpy as np
import pytest

from oracle_binary import binary_ivf as ob
from vearch_b200 import synth

CODE_SIZES = [1, 3, 4, 8, 12, 16, 20, 24, 32, 64, 128]


def test_binary_to_real_and_back_match_unpackbits():
    rng = np.random.default_rng(0)
    x = rng.integers(0, 256, size=(17, 5), dtype=np.uint8)
    xf = ob.binary_to_real(x, 40)
    bits = np.unpackbits(x, axis=1, bitorder="little")
    assert np.array_equal(xf, np.where(bits == 1, 1.0, -1.0).astype(np.float32))
    assert np.array_equal(ob.real_to_binary(xf), x)
    # a component must be strictly positive to become a 1 bit
    z = np.zeros((1, 8), np.float32)
    z[0, 3] = 0.5
    assert ob.real_to_binary(z)[0, 0] == 8


@pytest.mark.parametrize("cs", CODE_SIZES)
def test_hamming_matches_numpy(cs):
    rng = np.random.default_rng(cs)
    a = rng.integers(0, 256, size=(7, cs), dtype=np.uint8)
    b = rng.integers(0, 256, size=(9, cs), dtype=np.uint8)
    want = np.array([[int(np.unpackbits(a[i] ^ b[j]).sum()) for j in range(9)] for i in range(7)])
    assert np.array_equal(ob.hamming(a, b), want)


def test_heap_keeps_first_seen_at_a_boundary_tie():
    q = np.zeros((1, 1), np.uint8)
    # three entries at distance 1, k = 2: the two seen first stay (strict <), whatever their ids
    codes = np.array([[1], [2], [4]], np.uint8)
    lists = {0: (codes[:1], np.array([9])), 1: (codes[1:], np.array([5, 1]))}
    d, i = ob.search_knn_hamming_heap(q, lists, np.array([[0, 1]]), 2)
    assert d.tolist() == [[1.0, 1.0]] and sorted(i[0].tolist()) == [5, 9]


def test_heap_applies_bitmaps_tombstones_and_window():
    q = np.zeros((1, 1), np.uint8)
    codes = np.array([[0], [1], [3], [7]], np.uint8)
    ids = np.array([0, 1, 2, -(1 << 63) + 3])
    dele = np.array([0b0001], np.uint8)
    d, i = ob.search_knn_hamming_heap(q, {0: (codes, ids)}, np.array([[0]]), 4, del_bitmap=dele, min_score=1, max_score=2)
    assert i[0].tolist() == [1, 2, -1, -1] and d[0, :2].tolist() == [1.0, 2.0]


@pytest.mark.parametrize("nlist,tt,want", [(100, 50, 3900), (100, 2000, 2000), (100, 25600, 25600), (100, 30000, 25600)])
def test_sample_size_rule(nlist, tt, want):
    assert ob.sample_size(nlist, tt) == want


def test_default_training_threshold():
    assert ob.default_training_threshold(256) == 256 * 39


def test_full_distance_deviation_at_128_bytes():
    a = np.zeros((1, 128), np.uint8)
    b = a.copy()
    b[0, 100] = 0xFF  # differs only after byte 8
    assert ob.hamming(a, b)[0, 0] == 8
    assert ob.reference_scanner_distance(a, b)[0, 0] == 0  # the reference's HammingComputer8 sees no difference
    assert ob.reference_scanner_distance(a[:, :32], b[:, :32])[0, 0] == 0  # 32 bytes: full in both
    c = b[:, :32].copy()
    c[0, 20] = 1
    assert ob.reference_scanner_distance(a[:, :32], c)[0, 0] == 1


def test_coarse_ties_go_to_the_smaller_list():
    cent = np.array([[3], [5], [0]], np.uint8)  # distances 2, 2, 0 to the query 0
    d, l = ob.coarse_search(np.zeros((1, 1), np.uint8), cent, 3)
    assert l[0].tolist() == [2, 0, 1] and d[0].tolist() == [0, 2, 2]


def test_clustered_generator_is_seeded_and_clustered():
    x = synth.binary_clustered(2000, 64, seed=3, n_clusters=8, flip=0.05)
    assert x.shape == (2000, 8) and x.dtype == np.uint8
    assert np.array_equal(x, synth.binary_clustered(2000, 64, seed=3, n_clusters=8, flip=0.05))
    d = ob.hamming(x[:50], x)
    d[np.arange(50), np.arange(50)] = 999
    assert np.median(d.min(1)) < 16  # a same-centre neighbour is close; random rows sit near 32
