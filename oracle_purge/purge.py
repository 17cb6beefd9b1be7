"""Numpy restatement of the inverted-list purge (RealTimeMemData::CompactIfNeed / CompactBucket,
index/realtime/realtime_mem_data.cc:94-146, 347-373), the twin the GPU purge is tested against.

Lists are the CSR view GammaIndex.export_lists() returns: off [nlist + 1], codes [n, code_size] uint8, ids [n] int64 with
the tombstone in the top bit.  A deletion bitmap is dense and LSB first (bit vid & 7 of byte vid >> 3), as every search
takes it."""
import numpy as np

TOMBSTONE = np.int64(-2 ** 63)


def bitmap_of(vids, nbits):
    """The deletion bitmap with the bits `vids` set, covering nbits documents."""
    b = np.zeros(nbits, bool)
    b[np.asarray(vids, np.int64)] = True
    return np.packbits(b, bitorder="little")


def live(ids, del_bitmap=None):
    """An entry is live iff it is not tombstoned and its bit in the deletion bitmap (if any) is clear; ids beyond the
    bitmap are not deleted."""
    ids = np.asarray(ids, np.int64)
    ok = ids >= 0
    if del_bitmap is not None:
        bm = np.asarray(del_bitmap, np.uint8)
        v = np.where(ok, ids, 0)
        inside = ok & ((v >> 3) < bm.size)
        bit = np.zeros(ids.shape, bool)
        bit[inside] = (bm[v[inside] >> 3] >> (v[inside] & 7).astype(np.uint8)) & 1
        ok &= ~bit
    return ok


def select_lists(dead, lens, threshold=0.3):
    """Compactable(): the lists whose counted dead share is >= threshold in float32 arithmetic; a list without a dead
    entry is never selected, so threshold 0 means "every list with a dead entry"."""
    dead, lens = np.asarray(dead, np.int64), np.asarray(lens, np.int64)
    share = np.zeros(len(lens), np.float32)
    nz = lens > 0
    share[nz] = dead[nz].astype(np.float32) / lens[nz].astype(np.float32)
    return np.flatnonzero((dead > 0) & nz & (share >= np.float32(threshold)))


def vid_positions(off, ids, nvid):
    """vid -> list << 32 | pos of its entry that is not tombstoned, -1 if it has none."""
    off, ids = np.asarray(off, np.int64), np.asarray(ids, np.int64)
    out = np.full(nvid, -1, np.int64)
    lst = np.repeat(np.arange(len(off) - 1, dtype=np.int64), np.diff(off))
    pos = np.arange(len(ids), dtype=np.int64) - off[lst]
    keep = ids >= 0
    out[ids[keep]] = (lst[keep] << 32) | pos[keep]
    return out


def purge(off, codes, ids, lists, del_bitmap=None):
    """Rewrite `lists` with their live entries only, in their old order; every other list is untouched, tombstones
    included.  Returns (off, codes, ids, dropped)."""
    off, ids = np.asarray(off, np.int64), np.asarray(ids, np.int64)
    codes = np.asarray(codes)
    nlist = len(off) - 1
    lst = np.repeat(np.arange(nlist, dtype=np.int64), np.diff(off))
    sel = np.zeros(nlist, bool)
    sel[np.asarray(lists, np.int64)] = True
    keep = ~sel[lst] | live(ids, del_bitmap)
    new_off = np.zeros(nlist + 1, np.int64)
    np.cumsum(np.bincount(lst[keep], minlength=nlist), out=new_off[1:])
    return new_off, codes[keep], ids[keep], int((~keep).sum())
