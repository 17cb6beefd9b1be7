"""The fused coarse quantiser's selection (coarse_topk_kernel: selection warps apart from the MMA warpgroup, a query
tile's partial key sets merged inside the kernel) at the limits it must keep, against the score-matrix path
(GB_COARSE_FUSED=0): nprobe up to kCoarseMaxK, nlist not a multiple of the 128-centroid tile, nq not a multiple of
the 128-query tile, both metrics, tied centroids and non-finite query rows.  Both paths evaluate the same 3xTF32
scores under the same total key order, so distances and list ids must be byte-identical."""
import numpy as np
import pytest

from oracle import oracle as orc
from vearch_b200 import synth

pytestmark = pytest.mark.gpu
L2, IP = orc.METRIC_L2, orc.METRIC_IP
D = 128


def queries(nq, seed):
    xq = synth.embed_like(nq, D, seed=seed)
    xq[min(5, nq - 1), 3] = np.inf
    if nq > 17:
        xq[17, 0] = np.nan
        xq[nq - 1, 100] = -np.inf
    return xq


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nlist", [1000, 4096])
def test_coarse_select_limits(monkeypatch, metric, nlist):
    from vearch_b200 import index as gidx
    cent = synth.embed_like(nlist, D, seed=21)
    # a third of the centroids repeat earlier ones: their scores tie, and ties resolve by centroid id
    ndup = nlist // 3
    cent[nlist - ndup:] = cent[:ndup]
    idx = gidx.GammaIndex("IVFFLAT", D, {"ncentroids": nlist, "nprobe": 8,
                                         "metric_type": "L2" if metric == L2 else "InnerProduct"})
    try:
        idx.set_centroids(cent)
        for nq, path in ((10000, "coarse_topk_kernel"), (1, "dist_tile_kernel+select_rows_kernel")):
            xq = queries(nq, seed=22)
            finite = np.isfinite(xq).all(axis=1)
            for nprobe in (1, 32, 64):
                monkeypatch.setenv("GB_COARSE_FUSED", "0")
                do, io = idx.coarse_search(xq, nprobe)
                monkeypatch.delenv("GB_COARSE_FUSED")
                dg, ig = idx.coarse_search(xq, nprobe)
                assert idx.last_coarse_kernel == path, (nq, idx.last_coarse_kernel)
                assert (io[finite] >= 0).all()
                assert dg.tobytes() == do.tobytes(), f"nq={nq} nprobe={nprobe}: distances differ"
                assert ig.tobytes() == io.tobytes(), f"nq={nq} nprobe={nprobe}: ids differ"
            if nq > 1:
                # the duplicated centroids do tie inside the selected sets, so the id order is exercised
                _, ids = idx.coarse_search(xq[finite][:200], 64)
                assert np.isin(ids, np.arange(nlist - ndup, nlist)).any()
    finally:
        idx.close()
