"""The index files of IVFPQFastScan, IVFRABITQ, VEARCH and BINARYIVF as tests/quantised_index_file.py restates them:
every layout round-trips, and the reader refuses what the engine's loader refuses (a truncated file, a wrong magic, a
wrong dimension, and a wrong nb_bits, M, metric or other codec parameter).  tests/test_gpu_persist_quantised.py holds
the engine's files to the same restatement byte for byte."""
import struct

import numpy as np
import pytest

import quantised_index_file as qf

IP, L2 = qf.METRIC_IP, qf.METRIC_L2


def case(kind, metric=L2):
    """a small file of `kind` and the table it belongs to, lists with empty ones and tombstones"""
    rng = np.random.default_rng(len(kind))
    nlist, n = 5, 23
    d = 64 if kind == "BINARYIVF" else 24
    lens = np.array([7, 0, 9, 0, 7])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = rng.permutation(40)[:n].astype(np.int64)
    ids[[2, 10]] |= np.int64(-(1 << 63))  # tombstones
    table = dict(d=d, nlist=nlist, metric=metric)
    codec = {}
    if kind == "IVFPQFastScan":
        table["M"] = 6
        codec["pq_centroids"] = rng.standard_normal((6, 16, d // 6)).astype(np.float32)
        code_size = 3
    elif kind == "IVFRABITQ":
        table.update(nb_bits=4, qb=3)
        codec.update(nb_bits=4, qb=3)
        code_size = 4 * (4 * 1 + 3)
    elif kind == "VEARCH":
        table.update(nsub=5, blocks=6, ns_threshold=0.2 if metric == IP else float("nan"), reordering=True)
        codec.update(nsub=5, blocks=6, ns_threshold=table["ns_threshold"], reordering=True,
                     codebook=rng.standard_normal(16 * d).astype(np.float32))
        code_size = 3
    else:
        codec["binary_centroids"] = rng.integers(0, 256, (nlist, d // 8), dtype=np.uint8)
        code_size = d // 8
    codes = rng.integers(0, 256, (n, code_size), dtype=np.uint8)
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    buf = qf.write_quantised(kind, d, metric, 3, cent, off, codes, ids, 31, code_size, **codec)
    return buf, table, dict(centroids=cent, list_off=off, codes=codes, ids=ids, code_size=code_size, **codec)


KINDS = [("IVFPQFastScan", L2), ("IVFPQFastScan", IP), ("IVFRABITQ", L2), ("IVFRABITQ", IP), ("VEARCH", L2),
         ("VEARCH", IP), ("BINARYIVF", L2)]


@pytest.mark.parametrize("kind,metric", KINDS)
def test_round_trip(kind, metric):
    buf, table, want = case(kind, metric)
    got = qf.read_quantised(buf, kind, table)
    assert got["indexed_count"] == 31 and got["ntotal"] == 31 and got["metric"] == metric
    for key, v in want.items():
        if key == "ns_threshold":
            assert (np.isnan(v) and np.isnan(got[key])) or v == got[key]
        else:
            assert np.array_equal(np.asarray(got[key]), np.asarray(v)), key
    # written again from what was read: the same bytes
    codec = {k: got[k] for k in ("pq_centroids", "nb_bits", "qb", "nsub", "blocks", "ns_threshold", "reordering",
                                 "codebook", "binary_centroids") if k in got}
    again = qf.write_quantised(kind, got["d"], got["metric"], got["nprobe"], got["centroids"], got["list_off"],
                               got["codes"], got["ids"], got["indexed_count"], got["code_size"], **codec)
    assert again == buf


@pytest.mark.parametrize("kind,metric", KINDS)
def test_truncated_files_are_refused(kind, metric):
    buf, table, _ = case(kind, metric)
    for cut in sorted(set(np.linspace(0, len(buf) - 1, 97).astype(int).tolist()) | {len(buf) - 1, len(buf) - 4}):
        with pytest.raises(ValueError):
            qf.read_quantised(buf[:cut], kind, table)


@pytest.mark.parametrize("kind,metric", KINDS)
def test_wrong_magic_dimension_and_metric_are_refused(kind, metric):
    buf, table, _ = case(kind, metric)
    with pytest.raises(ValueError, match="magic"):
        qf.read_quantised(b"IwPQ" + buf[4:], kind, table)
    other = [k for k in qf.MAGIC if k != kind][0]  # another quantised type's file under this name
    with pytest.raises(ValueError, match="magic"):
        qf.read_quantised(buf, other, table)
    with pytest.raises(ValueError, match="d or nlist"):
        qf.read_quantised(buf, kind, dict(table, d=table["d"] + 8))
    with pytest.raises(ValueError, match="d or nlist"):
        qf.read_quantised(buf, kind, dict(table, nlist=table["nlist"] + 1))
    with pytest.raises(ValueError, match="metric"):
        qf.read_quantised(buf, kind, dict(table, metric=IP if metric == L2 else L2))
    # the header's d patched: the quantiser no longer matches either
    with pytest.raises(ValueError):
        qf.read_quantised(buf[:4] + struct.pack("<i", table["d"] + 8) + buf[8:], kind, table)


@pytest.mark.parametrize("kind,key,value", [
    ("IVFPQFastScan", "M", 4), ("IVFPQFastScan", "M", 12),
    ("IVFRABITQ", "nb_bits", 5), ("IVFRABITQ", "qb", 4),
    ("VEARCH", "nsub", 6), ("VEARCH", "blocks", 5), ("VEARCH", "reordering", False), ("VEARCH", "ns_threshold", 0.3),
])
def test_wrong_codec_parameter_is_refused(kind, key, value):
    buf, table, _ = case(kind, IP)
    with pytest.raises(ValueError, match="differs from the table"):
        qf.read_quantised(buf, kind, dict(table, **{key: value}))


def test_vearch_threshold_nan_matches_only_nan():
    buf, table, _ = case("VEARCH", L2)  # L2: no noise shaping, written as NaN
    assert np.isnan(qf.read_quantised(buf, "VEARCH", table)["ns_threshold"])
    with pytest.raises(ValueError):
        qf.read_quantised(buf, "VEARCH", dict(table, ns_threshold=0.2))


def test_file_names_are_not_the_references():
    # gamma reads ivfflat.index, ivfpq.index and ivfrabitq.index (faiss IndexIVFRaBitQ); none of ours may collide
    assert not set(qf.FILE.values()) & {"ivfflat.index", "ivfpq.index", "ivfrabitq.index"}
    assert len(set(qf.MAGIC.values())) == 4 and not set(qf.MAGIC.values()) & {"IvFl", "IwPQ", "Iwrq", "Iwrr"}
