"""Independent restatement (struct.pack) of the index files of a spilled IVFPQFastScan, IVFRABITQ or VEARCH index
(model parameter "soar_lambda" > 0, DESIGN.md §8, SOAR spilling): the unspilled layout of tests/quantised_index_file.py with

  * the variant fourcc "GsFS" / "GsRQ" / "GsVR" in place of "GbFS" / "GbRQ" / "GbVR", and
  * f64 soar_lambda right after the codec block, before the "ilar" lists,

the lists holding both entries of every spilled row.  read_spilled refuses an unspilled file (its magic) and a lambda
other than the table's; the unspilled reader refuses a spilled file the same way."""
import struct

from gamma_index_file import _inverted_lists, _ivf_header, fourcc
import numpy as np
import quantised_index_file as qf

MAGIC = {"IVFPQFastScan": "GsFS", "IVFRABITQ": "GsRQ", "VEARCH": "GsVR"}
FILE = {k: qf.FILE[k] for k in MAGIC}  # the same file names: a table finds the file and refuses the other kind's


def write_spilled(kind, d, metric, nprobe, centroids, list_off, codes, ids, indexed_count, code_size, soar_lambda, **codec):
    nlist = len(list_off) - 1
    out = fourcc(MAGIC[kind]) + _ivf_header(d, indexed_count, metric, nlist, nprobe, centroids)
    out += qf._codec_block(kind, code_size, d, nlist, codec)
    out += struct.pack("<d", soar_lambda)
    out += _inverted_lists(list_off, np.ascontiguousarray(codes, np.uint8).reshape(-1, code_size), ids, code_size)
    out += struct.pack("<i", indexed_count)
    return out


def read_spilled(buf, kind, table):
    """table as qf.read_quantised takes it, plus soar_lambda; ValueError where the engine refuses the file"""
    if buf[:4].decode(errors="replace") != MAGIC[kind]:
        raise ValueError("bad magic")
    unspilled_magic = qf.MAGIC[kind].encode()
    # the same fields with the lambda cut out: find the end of the codec block by reading the unspilled form's prefix
    head = unspilled_magic + buf[4:]
    probe = _codec_end(head, kind, table)
    if len(head) < probe + 8:
        raise ValueError("truncated: soar_lambda")
    (lam,) = struct.unpack_from("<d", head, probe)
    if lam != table["soar_lambda"]:
        raise ValueError("soar_lambda differs from the table's")
    out = qf.read_quantised(head[:probe] + head[probe + 8:], kind, table)
    out["soar_lambda"] = lam
    return out


def _codec_end(buf, kind, t):
    """byte offset of the end of the codec block (where the lists' "ilar" starts in an unspilled file)"""
    p = 4 + struct.calcsize("<iqqq?i") + 16 + 4 + struct.calcsize("<iqqq?i") + 8 + 4 * t["nlist"] * t["d"] + 9
    if kind == "IVFPQFastScan":
        n = struct.unpack_from("<QQQQQ", buf, p)[4]
        return p + 40 + 4 * n
    if kind == "IVFRABITQ":
        return p + 16
    n = struct.unpack_from("<QiidBQ", buf, p)[5]
    return p + struct.calcsize("<QiidBQ") + 4 * n
