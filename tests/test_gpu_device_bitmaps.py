"""search_device with deletion and filter bitmaps in HBM (gb_index_search_device_filtered): for every float index type
it returns exactly what the host search returns with the same bitmaps, including bitmaps shorter than the store and
bitmaps at an odd address."""
import numpy as np
import pytest

from vearch_b200 import synth

pytestmark = pytest.mark.gpu
D, N, NQ, K, NLIST = 32, 3000, 24, 10, 16

TYPES = [
    ("FLAT", {}),
    ("IVFFLAT", {}),
    ("IVFPQ", {"nsubvector": 8}),
    ("IVFPQFastScan", {"nsubvector": 8}),
    ("IVFRABITQ", {"nb_bits": 4, "qb": 4}),
    ("VEARCH", {"nsubvector": 8, "reordering": True}),
    ("GPU_IVFPQ", {"nsubvector": 8}),
    ("GPU_IVFFLAT", {}),
    ("GPU_IVFPQ/2", {"nsubvector": 8}),  # sharded S = 2 on one device
]


def build(typ, extra):
    from vearch_b200 import index as gidx
    name, _, shards = typ.partition("/")
    p = {"metric_type": "L2"}
    if name != "FLAT":
        p.update(ncentroids=NLIST, nprobe=8, training_threshold=1000)
    p.update(extra)
    devices = [0] * int(shards) if shards else None
    cls = {"IVFRABITQ": gidx.RaBitQIndex, "VEARCH": gidx.VearchIndex}.get(name)
    idx = cls(D, p) if cls else gidx.GammaIndex(name, D, p, devices=devices)
    db = synth.sift_like(N, D, seed=31, n_clusters=32)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    return idx, db


def on_device(bm, odd):
    import torch
    t = torch.from_numpy(bm)
    if not odd:
        return t.cuda()
    buf = torch.zeros(bm.size + 1, dtype=torch.uint8, device="cuda")
    buf[1:].copy_(t)
    return buf[1:]  # one byte past an allocation boundary


@pytest.mark.parametrize("typ,extra", TYPES, ids=[t for t, _ in TYPES])
def test_search_device_bitmaps_match_host(typ, extra):
    import torch
    idx, db = build(typ, extra)
    rng = np.random.default_rng(7)
    xq = synth.sift_like(NQ, D, seed=32, n_clusters=32)
    xd = torch.from_numpy(xq).cuda()
    dele = np.packbits(rng.random(N) < 0.1, bitorder="little")
    filt = np.packbits(rng.random(N) < 0.5, bitorder="little")
    short_f, short_d = filt[:100], dele[:100]  # ids past 800: not allowed, not deleted
    cases = [
        dict(del_bitmap=dele),
        dict(filter_bitmap=filt),
        dict(del_bitmap=dele, filter_bitmap=filt),
        dict(del_bitmap=short_d, filter_bitmap=short_f),
        dict(filter_bitmap=short_f[:37]),
        dict(del_bitmap=short_d[:37]),
        dict(filter_bitmap=np.zeros(0, np.uint8)),
        dict(filter_bitmap=filt, min_score=2.0e4, max_score=2.0e5),
    ]
    params = None if typ == "FLAT" else {"nprobe": 8}
    for odd in (False, True):
        for case in cases:
            for brute in ((False, True) if typ != "FLAT" else (False,)):
                want = idx.search(xq, K, params=params, brute_force=brute, **case)
                dev = {k: (on_device(v, odd) if k.endswith("bitmap") else v) for k, v in case.items()}
                got = idx.search_device(xd, K, params=params, brute_force=brute, **dev)
                torch.cuda.synchronize()
                gd, gi_ = got[0].cpu().numpy(), got[1].cpu().numpy()
                what = f"{typ} {sorted(case)} brute={brute} odd={odd}"
                assert np.array_equal(gi_, want[1]), what
                assert np.array_equal(gd.view(np.uint32), want[0].view(np.uint32)), what
    idx.close()
