"""Independent restatement (struct.pack, no shared code with csrc/index_io.cu) of this engine's own index files of the
quantised types, used by the tests as the golden writer / reader:

  IVFPQFastScan   "GbFS"  <field>.000/gb_ivfpqfs.index
  IVFRABITQ       "GbRQ"  <field>.000/gb_ivfrabitq.index
  VEARCH          "GbVR"  <field>.000/gb_vearch.index
  BINARYIVF       "GbBI"  <field>.000/gb_binaryivf.index

Each is gamma's IVF skeleton (tests/gamma_index_file.py: fourcc, ivf header with an IndexFlat quantiser, direct map,
"ilar" lists, the trailing i32 indexed_count of ivfflat.index) with the type's codec block between the direct map and the
lists.  read_quantised refuses a file the engine must refuse: a wrong magic, a truncated file, or a d,
nlist, metric or codec parameter other than the table's.
"""
import math
import struct

import numpy as np

from gamma_index_file import METRIC_IP, METRIC_L2, _Reader, _inverted_lists, _ivf_header, fourcc

MAGIC = {"IVFPQFastScan": "GbFS", "IVFRABITQ": "GbRQ", "VEARCH": "GbVR", "BINARYIVF": "GbBI"}
FILE = {"IVFPQFastScan": "gb_ivfpqfs.index", "IVFRABITQ": "gb_ivfrabitq.index", "VEARCH": "gb_vearch.index",
        "BINARYIVF": "gb_binaryivf.index"}


def _codec_block(kind, code_size, d, nlist, codec):
    if kind == "IVFPQFastScan":
        pq = np.ascontiguousarray(codec["pq_centroids"], np.float32)
        M = pq.shape[0]
        assert pq.shape == (M, 16, d // M)
        return struct.pack("<QQQQQ", code_size, d, M, 4, pq.size) + pq.tobytes()
    if kind == "IVFRABITQ":
        return struct.pack("<Qii", code_size, codec["nb_bits"], codec["qb"])
    if kind == "VEARCH":
        cb = np.ascontiguousarray(codec["codebook"], np.float32).reshape(-1)
        assert cb.size == 16 * d
        return (struct.pack("<QiidBQ", code_size, codec["nsub"], codec["blocks"], codec["ns_threshold"],
                            int(bool(codec["reordering"])), cb.size) + cb.tobytes())
    if kind == "BINARYIVF":
        bc = np.ascontiguousarray(codec["binary_centroids"], np.uint8)
        assert bc.shape == (nlist, d // 8)
        return struct.pack("<QQ", code_size, bc.size) + bc.tobytes()
    raise ValueError(kind)


def write_quantised(kind, d, metric, nprobe, centroids, list_off, codes, ids, indexed_count, code_size, **codec):
    """centroids: [nlist, d] fp32 (BINARYIVF: the float k-means centroids, d in bits, metric L2); codes: [n, code_size]
    uint8 in list order; ids: int64 with the tombstone top bit."""
    nlist = len(list_off) - 1
    out = fourcc(MAGIC[kind]) + _ivf_header(d, indexed_count, metric, nlist, nprobe, centroids)
    out += _codec_block(kind, code_size, d, nlist, codec)
    out += _inverted_lists(list_off, np.ascontiguousarray(codes, np.uint8).reshape(-1, code_size), ids, code_size)
    out += struct.pack("<i", indexed_count)
    return out


def read_quantised(buf, kind, table):
    """Parse a file of `kind` for a table {d, nlist, metric, and the codec parameters: M (IVFPQFastScan); nb_bits, qb
    (IVFRABITQ); nsub, blocks, ns_threshold, reordering (VEARCH)}; ValueError where the engine refuses the file."""
    try:
        return _read(buf, kind, table)
    except struct.error as e:
        raise ValueError(f"truncated: {e}") from None


def _read(buf, kind, t):
    r = _Reader(buf)

    def arr(dtype, n):
        if r.p + np.dtype(dtype).itemsize * n > len(buf):
            raise ValueError("truncated array")
        return r.arr(dtype, n)

    if r.take("4s").decode(errors="replace") != MAGIC[kind]:
        raise ValueError("bad magic")
    d, ntotal, _, _, _, metric = r.take("iqqq?i")
    nlist, nprobe = r.take("QQ")
    if d != t["d"] or nlist != t["nlist"]:
        raise ValueError("d or nlist differs from the table's")
    if metric != t["metric"]:
        raise ValueError("metric differs from the table's")
    if r.take("4s") not in (b"IxF2", b"IxFI"):
        raise ValueError("bad quantizer")
    qd, qn, _, _, _, _ = r.take("iqqq?i")
    n = r.take("Q")
    if (qd, qn, n) != (d, nlist, nlist * d):
        raise ValueError("bad quantizer")
    out = dict(d=d, ntotal=ntotal, metric=metric, nlist=nlist, nprobe=nprobe,
               centroids=arr(np.float32, n).reshape(nlist, d))
    if r.take("bQ") != (0, 0):
        raise ValueError("direct map")
    if kind == "IVFPQFastScan":
        code_size, pd, M, nbits, n = r.take("QQQQQ")
        if (pd, M, nbits, code_size) != (d, t["M"], 4, (t["M"] + 1) // 2) or n != M * 16 * (d // M):
            raise ValueError("codebook differs from the table's")
        out["pq_centroids"] = arr(np.float32, n).reshape(M, 16, d // M)
    elif kind == "IVFRABITQ":
        code_size, nb_bits, qb = r.take("Qii")
        if (nb_bits, qb) != (t["nb_bits"], t["qb"]):
            raise ValueError("nb_bits or qb differs from the table's")
        out.update(nb_bits=nb_bits, qb=qb)
    elif kind == "VEARCH":
        code_size, nsub, blocks, ns, reo, n = r.take("QiidBQ")
        same_ns = (math.isnan(ns) and math.isnan(t["ns_threshold"])) or ns == t["ns_threshold"]
        if (nsub, blocks, bool(reo)) != (t["nsub"], t["blocks"], bool(t["reordering"])) or not same_ns or n != 16 * d:
            raise ValueError("codebook differs from the table's")
        out.update(nsub=nsub, blocks=blocks, ns_threshold=ns, reordering=bool(reo), codebook=arr(np.float32, n))
    else:
        code_size, n = r.take("QQ")
        if code_size != d // 8 or n != nlist * code_size:
            raise ValueError("binary centroids differ from the table's")
        out["binary_centroids"] = arr(np.uint8, n).reshape(nlist, code_size)
    if r.take("4s") != b"ilar":
        raise ValueError("bad inverted lists")
    nb, cb = r.take("QQ")
    if r.take("4s") != b"full" or nb != nlist or cb != code_size or r.take("Q") != nlist:
        raise ValueError("bad inverted lists")
    sizes = arr(np.uint64, nlist).astype(np.int64)
    off = np.zeros(nlist + 1, np.int64)
    np.cumsum(sizes, out=off[1:])
    codes = np.empty((int(off[-1]), cb), np.uint8)
    ids = np.empty(int(off[-1]), np.int64)
    for l in range(nlist):
        if sizes[l]:
            codes[off[l]:off[l + 1]] = arr(np.uint8, int(sizes[l]) * cb).reshape(-1, cb)
            ids[off[l]:off[l + 1]] = arr(np.int64, int(sizes[l]))
    out.update(code_size=code_size, list_off=off, codes=codes, ids=ids)
    out["indexed_count"] = r.take("i")
    if out["indexed_count"] < 0:
        raise ValueError("invalid indexed count")
    assert r.p == len(buf), "trailing bytes"
    return out
