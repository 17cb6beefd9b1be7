"""The int8 error bound of the IVF-PQ tensor-core filter (kernels_pqtc.cu, pq_stage_pairs_kernel / pqtc_tables_kernel).

The filter multiplies int8 rows qa = rn(a / sa), sa = max|a| / 127, with an int8 codebook qr = rn(pq / sb), sb = max|pq| / 127,
and accumulates exactly in s32.  It passes an entry when the approximate score, widened by
    eps = f * 1.05 * (|da| R + (|a| + |da|) D),   da = a - sa qa,  R^2 = sum_m max_c |pq_m,c|^2,
                                                   D^2 = sum_m max_c |pq_m,c - sb qr_m,c|^2,  f = 2 (L2) / 1 (IP),
can reach the query's bound, so eps must cover |f <a, r> - f sa sb <qa, qr>| for every row and every entry.

CPU: a numpy restatement of the quantisation (fp32 where the kernels compute in fp32) checked against fp64 on random,
heavy-tailed and single-dominant-component rows and codebooks -- the last is int8's worst case, every other component
rounds to 0.  GPU: the same dominant-component regime end to end, the list-major search key-equal to the LUT kernel on
every shape the filter takes, under both metrics.
"""
import numpy as np
import pytest

F32 = np.float32


def quantise_rows(a):
    """(qa, sa, |da|) per row, as pq_stage_pairs_kernel computes them"""
    a = a.astype(F32)
    amax = np.abs(a).max(1)
    sa = amax / F32(127)
    inv = F32(127) / amax
    qa = np.clip(np.rint(a * inv[:, None]), -127, 127).astype(F32)
    da = a - sa[:, None] * qa
    return qa, sa, np.sqrt((da.astype(np.float64) ** 2).sum(1))


def quantise_codebook(pq):
    """(qr, sb, R, D) as pqtc_tables_kernel computes them; pq is [M][256][dsub]"""
    pq = pq.astype(F32)
    cbmax = np.abs(pq).max()
    sb, inv = cbmax / F32(127), F32(127) / cbmax
    qr = np.clip(np.rint(pq * inv), -127, 127).astype(F32)
    dr = pq - sb * qr
    R = np.sqrt((pq.astype(np.float64) ** 2).sum(-1).max(1).sum())
    D = np.sqrt((dr.astype(np.float64) ** 2).sum(-1).max(1).sum())
    return qr, sb, R, D


def draw(kind, shape, rng):
    if kind == "random":
        return rng.standard_normal(shape)
    if kind == "heavy":  # Student t with 1.5 degrees of freedom: a few components dwarf the rest
        return rng.standard_t(1.5, shape)
    # one component per row (per sub-vector of the codebook) 2^12 times the others
    x = rng.standard_normal(shape) * 2.0 ** -12
    idx = rng.integers(0, shape[-1], shape[:-1])
    np.put_along_axis(x, idx[..., None], rng.choice([-1.0, 1.0], shape[:-1])[..., None] * rng.uniform(0.5, 1, shape[:-1])[..., None], -1)
    return x


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("rows", ["random", "heavy", "dominant"])
@pytest.mark.parametrize("book", ["random", "heavy", "dominant"])
def test_int8_bound_covers_the_quantisation_error(d, rows, book):
    rng = np.random.default_rng(d * 7 + len(rows) * 3 + len(book))
    for M in [m for m in (4, 8, 16) if d % m == 0 and d // m in (4, 8, 16, 32)]:
        dsub = d // M
        a = draw(rows, (64, d), rng).astype(F32)
        pq = draw(book, (M, 256, dsub), rng).astype(F32)
        qa, sa, da = quantise_rows(a)
        qr, sb, R, D = quantise_codebook(pq)
        codes = rng.integers(0, 256, (512, M))
        # the codebook's extreme centroids too: the entries that reach R and D
        codes[:M] = np.argmax((pq.astype(np.float64) ** 2).sum(-1), 1)[None, :]
        r = pq[np.arange(M)[None, :], codes].reshape(len(codes), d).astype(np.float64)
        rq = qr[np.arange(M)[None, :], codes].reshape(len(codes), d).astype(np.float64)
        exact = -2.0 * a.astype(np.float64) @ r.T
        acc = qa.astype(np.float64) @ rq.T
        assert np.abs(acc).max() < 2 ** 22  # the biased accumulator stays exact
        approx = -2.0 * (sa.astype(np.float64) * float(sb))[:, None] * acc
        na = np.sqrt((a.astype(np.float64) ** 2).sum(1))
        eps = 2.0 * 1.05 * (da * R + (na + da) * D)
        err = np.abs(exact - approx)
        worst = (err / eps[:, None]).max()
        assert worst <= 1.0, f"d={d} M={M} rows={rows} book={book}: error reaches {worst:.3f} of eps"


# ---- GPU: the dominant-component regime end to end ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("M,dsub", [(16, 8), (8, 16), (8, 8), (16, 4), (4, 16), (4, 32), (4, 8), (8, 4)])
def test_ivfpq_filter_dominant_components(M, dsub, metric):
    from test_gpu_float_accuracy import IP, L2, best, gi, mt
    import float_contract as FC
    metric = [L2, IP][metric]
    d, n, nq, nlist, nprobe = M * dsub, 20000, 128, 16, 6
    rng = np.random.default_rng(M * 10 + dsub)
    db = (draw("dominant", (n, d), rng) * 100).astype(F32)
    xq = (draw("dominant", (nq, d), rng) * 100).astype(F32)
    cent = db[rng.choice(n, nlist, replace=False)]
    pq = (draw("dominant", (M, 256, dsub), rng) * 100).astype(F32)
    idx = gi().GammaIndex("IVFPQ", d, {"ncentroids": nlist, "nprobe": nprobe, "nsubvector": M, "metric_type": mt(metric)})
    try:
        idx.set_centroids(cent)
        idx.set_pq_centroids(pq)
        idx.add(db)
        fq, _ = FC.scores64(xq, cent, metric)
        probes = best(fq, nprobe, metric).astype(np.int64)
        cd = np.take_along_axis(fq, probes, 1).astype(F32)
        for k in (10, 100):
            dg, ig = idx.search_preassigned(xq, k, probes, cd)
            assert idx.last_scan_kernel == "pqtc_scan_kernel", idx.last_scan_kernel
            parts = []
            for q0 in range(0, nq, 3):
                parts.append(idx.search_preassigned(xq[q0:q0 + 3], k, probes[q0:q0 + 3], cd[q0:q0 + 3]))
                assert idx.last_scan_kernel == "ivfpq_scan_kernel", idx.last_scan_kernel
            ds, is_ = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
            bad = np.nonzero(np.any(dg.view(np.uint32) != ds.view(np.uint32), 1) | np.any(ig != is_, 1))[0]
            assert len(bad) == 0, (f"M={M} dsub={dsub} k={k}: {len(bad)}/{nq} queries differ from the LUT kernel; "
                                   f"query {bad[0]}: {ig[bad[0]][:5]} vs {is_[bad[0]][:5]}")
    finally:
        idx.close()
