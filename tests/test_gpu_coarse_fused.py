"""The fused coarse quantiser (coarse_topk_kernel: scores and top-nprobe in one tensor-core kernel) against the
score-matrix path it replaces (GB_COARSE_FUSED=0).  Both evaluate the same 3xTF32 scores and the same total key
order, so distances and list ids must be byte-identical, on float data too."""
import numpy as np
import pytest

from oracle import oracle as orc
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = orc.METRIC_L2, orc.METRIC_IP
FUSED_MAX_NPROBE = 64  # kCoarseMaxK: one above it exercises the fallback


def gi():
    from vearch_b200 import index as gidx
    return gidx


def launches():
    from vearch_b200 import _lib
    return _lib.lib().gb_launch_count()


def data(kind, n, d, seed):
    if kind == "embed":
        return synth.embed_like(n, d, seed=seed)
    return synth.sift_like(n, d, seed=seed, rounded=False)


@pytest.mark.parametrize("kind", ["embed", "sift"])
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nlist", [1000, 4096])
@pytest.mark.parametrize("d", [100, 128, 768])
def test_coarse_fused_bytes_equal(monkeypatch, kind, metric, nlist, d):
    cent = data(kind, nlist, d, seed=11)
    xq = data(kind, 1000, d, seed=12)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 8,
                                         "metric_type": "L2" if metric == L2 else "InnerProduct"})
    try:
        idx.set_centroids(cent)
        for nq in (33, 300, 1000):
            for nprobe in (1, 8, 32, FUSED_MAX_NPROBE, FUSED_MAX_NPROBE + 1):
                monkeypatch.setenv("GB_COARSE_FUSED", "0")
                n0 = launches()
                do, io = idx.coarse_search(xq[:nq], nprobe)
                ref_launches = launches() - n0
                monkeypatch.delenv("GB_COARSE_FUSED")
                n0 = launches()
                dg, ig = idx.coarse_search(xq[:nq], nprobe)
                # the fused path stages the queries, runs the fused kernel, merges the segments and splits the keys;
                # the matrix path computes, selects and splits
                want = ref_launches + 1 if nprobe <= FUSED_MAX_NPROBE else ref_launches
                assert launches() - n0 == want, f"nq={nq} nprobe={nprobe}: unexpected path"
                assert (io >= 0).all()
                assert dg.tobytes() == do.tobytes(), f"nq={nq} nprobe={nprobe}: distances differ"
                assert ig.tobytes() == io.tobytes(), f"nq={nq} nprobe={nprobe}: ids differ"
    finally:
        idx.close()


def test_coarse_fused_after_train(monkeypatch):
    # train() rebuilds the centroid tiles from the k-means result
    d, nlist = 64, 128
    db = synth.embed_like(20000, d, seed=3)
    xq = synth.embed_like(500, d, seed=4)
    idx = gi().GammaIndex("IVFFLAT", d, {"ncentroids": nlist, "nprobe": 8, "metric_type": "L2",
                                         "training_threshold": 10000})
    try:
        idx.add_vectors(db)
        idx.train()
        monkeypatch.setenv("GB_COARSE_FUSED", "0")
        do, io = idx.coarse_search(xq, 16)
        monkeypatch.delenv("GB_COARSE_FUSED")
        dg, ig = idx.coarse_search(xq, 16)
        assert dg.tobytes() == do.tobytes() and ig.tobytes() == io.tobytes()
    finally:
        idx.close()
