"""SOAR spilling on the GPU (DESIGN.md §8, SOAR spilling), for IVFPQFastScan, IVFRABITQ and VEARCH under L2 and InnerProduct:

1. the spilled list of every row against the fp64 twin (oracle_soar) within a rigorous margin, exact on exact ties and
   zero residuals, and every live vid in exactly two lists;
2. searches key-exact against the twins' scores deduplicated by best copy, at k' = 1, 10, 100 and 2048, with deletions,
   filters and split probe groups, and k' = 2049 refused;
3. the exact re-rank over distinct candidates;
4. updates, deletes and a purge: both slots live, no stale copy, the purge changes no answer;
5. the spilled file: round trip, layout, and each kind refusing the other's file;
6. the engine: a spilled table searched; the admission charge of two entries a row, and a memory limit refusing spilled
   rows at twice the entry cost; Backup and a table restored from it; AddFieldIndexWithParams on a second field;
7. bad values refused, and the key ignored by every other type."""
import os

import numpy as np
import pytest

import quantised_index_file as qf
import soar_index_file as sf
import topk_reference as R
from oracle_rabitq import rabitq as rq
from oracle_pqfs import twin
from oracle_soar import soar
from test_gpu_persist_quantised import BITS, D, NLIST, N, gi, make, params_of, rows, table_of
from test_gpu_shape_limits import vearch_twin_scores
from test_gpu_topk_keys import entries

pytestmark = pytest.mark.gpu
L2, IP = qf.METRIC_L2, qf.METRIC_IP
LAM = 1.5
KINDS = [(k, m) for k in ("IVFPQFastScan", "IVFRABITQ", "VEARCH") for m in (L2, IP)]
MASK = np.int64(0x7FFFFFFFFFFFFFFF)


def spilled(kind, metric, reordering=False, **over):
    over.setdefault("soar_lambda", LAM)
    if kind == "VEARCH":
        over["reordering"] = reordering
    return make(kind, metric, **over)


def built(kind, metric, n=N, seed=1, **over):
    idx = spilled(kind, metric, **over)
    db = rows(kind, n, seed)
    idx.add_vectors(db)
    idx.train()
    idx.add_pending()
    return idx, db


def entry_scores(kind, idx, xq, metric):
    """every list entry's scan score for every query, from the codes and the scan's own hooks / twins"""
    off, codes, ids, el = entries(idx, idx.nlist)
    if kind == "IVFPQFastScan":
        lut8, ab = idx.pqfs_lut(xq, metric)
        cu = twin.unpack(codes, idx.pq_m)
        s = np.stack([twin.scores(lut8[q], ab[q], cu) for q in range(len(xq))])
    elif kind == "IVFRABITQ":
        cent = idx.get_centroids()
        s = np.zeros((len(xq), len(ids)), np.float32)
        for l in np.unique(el):
            sel = el == l
            for j in range(len(xq)):
                s[j, sel] = rq.estimate(codes[sel], xq[j], cent[l], idx.d, idx.nb_bits, metric, idx.qb)
    else:
        s = vearch_twin_scores(codes, el, idx.get_centroids(), idx.get_codebook(), xq, idx.d, idx.nsub, metric)
    return off, ids, el, s


def ref_keys(scores, el, ids, probes, k, metric, **bm):
    """the contract: the k distinct vids of best best-copy key among the probed live entries"""
    allk = R.search_entries(scores, el, ids, probes, len(ids), metric, **bm)
    return np.stack([soar.dedupe_first(row, k) for row in allk])


def probe_order(xq, cent, metric):
    """every list, nearest first (fp64): the probes of a search_preassigned that reads all or the leading few"""
    x, c = np.asarray(xq, np.float64), np.asarray(cent, np.float64)
    s = ((x[:, None, :] - c[None]) ** 2).sum(-1) if metric == L2 else -(x @ c.T)
    return np.argsort(s, axis=1, kind="stable").astype(np.int64)


def assert_keys(got, want_keys, metric, what):
    dw, iw = R.decode(want_keys, metric)
    dg, ig = got
    assert np.array_equal(ig, iw), what
    assert np.array_equal(dg.view(np.uint32), dw.view(np.uint32)), what


def assert_two_entries(idx, deleted=()):
    """every vid not deleted has exactly two live entries, in two lists, where its slots say"""
    off, _, ids, el = entries(idx, idx.nlist)
    live = ids >= 0
    vid = ids & MASK
    cnt = np.bincount(vid[live], minlength=idx.ntotal)
    want = np.full(idx.ntotal, 2)
    want[list(deleted)] = cnt[list(deleted)]
    assert np.array_equal(cnt, want)
    for v in np.random.default_rng(0).choice(idx.ntotal, 200, replace=False):
        slots = idx.vid_slots(int(v))
        if v in deleted and len(slots) < 2:
            continue
        assert len(slots) == 2 and slots[0][0] != slots[1][0], (v, slots)
        for l, p in slots:
            assert ids[off[l] + p] == v, (v, l, p)


# ---- 1. the spilled list ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,metric", KINDS)
def test_spilled_list_against_fp64(kind, metric):
    idx, db = built(kind, metric)
    cent = idx.get_centroids()
    slots = [idx.vid_slots(v) for v in range(N)]
    prim = np.array([s[0][0] for s in slots])
    got = np.array([s[1][0] for s in slots])
    assert soar.check_spill(db, cent, prim, LAM, got) == []
    assert_two_entries(idx)
    idx.close()


@pytest.mark.parametrize("kind,metric", KINDS)
def test_spilled_list_exact_ties_and_zero_residuals(kind, metric):
    """integer rows and centroids: every fp32 term is exact, so equal (|r'|^2, <r, r'>) give equal losses and the lower
    list id must win; rows equal to a centroid have |r| = 0 and take the fallback list"""
    rng = np.random.default_rng(7)
    nl, d = 24, D
    cent = rng.integers(-1, 2, (nl, d)).astype(np.float32)
    x = rng.integers(-1, 2, (2000, d)).astype(np.float32)
    x[:40] = cent[rng.integers(0, nl, 40)]  # zero residuals
    idx = spilled(kind, metric, ncentroids=nl)
    idx.set_centroids(cent)
    idx.add_vectors(x)
    idx.add_pending()
    slots = [idx.vid_slots(v) for v in range(len(x))]
    prim = np.array([s[0][0] for s in slots])
    got = np.array([s[1][0] for s in slots])
    e, p, _, rn = soar.spill_terms(x, cent, prim)
    loss = soar.spill_loss(x, cent, prim, LAM)
    ties = 0
    for i in range(len(x)):
        if rn[i] == 0:
            assert got[i] == soar.fallback_list(i, prim[i], nl), i
            continue
        at = np.nonzero(loss[i] == loss[i].min())[0]
        if len(at) > 1 and len({(e[i, c], p[i, c] ** 2) for c in at}) == 1:
            ties += 1
            assert got[i] == at[0], (i, at, got[i])
    assert ties > 10
    good = rn > 0
    assert soar.check_spill(x[good], cent, prim[good], LAM, got[good]) == []
    assert_two_entries(idx)
    idx.close()


def test_one_list_is_refused():
    for kind in ("IVFPQFastScan", "IVFRABITQ", "VEARCH"):
        with pytest.raises(Exception, match="ncentroids >= 2"):
            spilled(kind, L2, ncentroids=1, nprobe=1)


@pytest.mark.parametrize("kind,metric", KINDS)
def test_spilled_entries_are_coded_against_their_list(kind, metric):
    """each entry's code is the codec's encoding of its row for the list it is in: a residual code against the spilled
    centroid (IVFRABITQ, VEARCH under IP), the raw row's code, equal in both lists, otherwise"""
    idx, db = built(kind, metric)
    off, codes, ids, _ = entries(idx, idx.nlist)
    slots = [idx.vid_slots(v) for v in range(N)]
    got = [codes[[off[s[j][0]] + s[j][1] for s in slots]] for j in (0, 1)]
    lists = [np.array([s[j][0] for s in slots], np.int64) for j in (0, 1)]
    if kind == "IVFRABITQ" or (kind == "VEARCH" and metric == IP):
        for j in (0, 1):
            assert np.array_equal(got[j], idx.encode(db, lists[j])), j
        assert not np.array_equal(got[0], got[1])
    else:
        assert np.array_equal(got[0], got[1])
        if kind == "VEARCH":
            assert np.array_equal(got[0], idx.encode(db))
    idx.close()


# ---- 2. search, key-exact -----------------------------------------------------------------------------------------
def nq_for_split(pg, nprobe):
    import torch
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    return -(-pg * nsm * 32 // nprobe)


@pytest.mark.parametrize("kind,metric", KINDS)
def test_search_key_exact(kind, metric):
    idx, db = built(kind, metric)
    Q = 6
    xq = rows(kind, Q, 9)
    off, ids, el, scores = entry_scores(kind, idx, xq, metric)
    probes = probe_order(xq, idx.get_centroids(), metric)
    zeros = np.zeros(probes.shape, np.float32)
    rng = np.random.default_rng(3)
    dele = np.packbits(rng.random(N) < 0.3, bitorder="little")
    filt = np.packbits(rng.random(N) < 0.5, bitorder="little")
    for k in (1, 10, 100, 2048):
        for bm in ({}, {"del_bitmap": dele}, {"del_bitmap": dele, "filter_bitmap": filt}):
            got = idx.search_preassigned(xq, k, probes, zeros, **bm)
            assert_keys(got, ref_keys(scores, el, ids, probes, k, metric, **bm), metric, (k, list(bm)))
            ig = got[1]
            for r in ig:
                v = r[r >= 0]
                assert len(np.unique(v)) == len(v)
    # fewer probes: some vids' second copy is not probed
    got = idx.search_preassigned(xq, 100, probes[:, :3], zeros[:, :3])
    assert_keys(got, ref_keys(scores, el, ids, probes[:, :3], 100, metric), metric, "nprobe 3")
    # probe groups: a batch large enough for several probes per CTA, each row a distinct query's probes reordered
    nq = nq_for_split(3, NLIST)
    rows_ = np.arange(nq) % Q
    pr = np.stack([np.random.default_rng(r).permutation(probes[q]) for r, q in enumerate(rows_)])
    got = idx.search_preassigned(xq[rows_], 100, pr, np.zeros(pr.shape, np.float32), del_bitmap=dele)
    assert idx.last_scan_info.get("probes_per_cta", 1) >= 3
    want = ref_keys(scores, el, ids, probes, 100, metric, del_bitmap=dele)
    assert_keys(got, want[rows_], metric, "probe groups")
    with pytest.raises(Exception, match="2048"):
        idx.search_preassigned(xq, 2049, probes, zeros)
    idx.close()


# ---- 3. exact re-rank ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,metric", KINDS)
def test_rerank_distinct_exact(kind, metric):
    idx, db = built(kind, metric, reordering=True)
    xq = rows(kind, 5, 11)
    off, ids, el, scores = entry_scores(kind, idx, xq, metric)
    probes = probe_order(xq, idx.get_centroids(), metric)
    kk, k = 64, 10
    adc = ref_keys(scores, el, ids, probes, kk, metric)
    got = idx.search_preassigned(xq, k, probes, np.zeros(probes.shape, np.float32), params={"recall_num": kk})
    assert_keys(got, R.rerank_keys(adc, xq, db, k, metric), metric, "rerank")
    for r in got[1]:
        assert len(np.unique(r)) == k
    idx.close()


# ---- 4. mutations -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,metric", KINDS)
def test_update_delete_purge(kind, metric):
    idx, db = built(kind, metric)
    new = rows(kind, 40, 5)
    for v, x in zip(range(40), new):
        idx.update_vector(v, x)
    dead = list(range(100, 130))
    idx.delete_vectors(np.array(dead, np.int64))
    dc = idx.dead_counts()
    assert dc.sum() == 2 * 40 + 2 * len(dead)  # both entries of every updated and deleted row
    del_bm = np.packbits(np.isin(np.arange(N), dead), bitorder="little")
    xq = rows(kind, 4, 12)
    probes = probe_order(xq, idx.get_centroids(), metric)
    zeros = np.zeros(probes.shape, np.float32)

    def check():
        off, ids, el, scores = entry_scores(kind, idx, xq, metric)
        got = idx.search_preassigned(xq, 200, probes, zeros, del_bitmap=del_bm)
        assert_keys(got, ref_keys(scores, el, ids, probes, 200, metric, del_bitmap=del_bm), metric, "after churn")
        assert not np.isin(got[1], dead).any()
        return got

    before = check()
    assert_two_entries(idx, deleted=dead)
    assert idx.purge(0.0, del_bitmap=del_bm) == 2 * 40 + 2 * len(dead)
    after = check()
    assert np.array_equal(before[1], after[1]) and np.array_equal(before[0].view(np.uint32), after[0].view(np.uint32))
    assert_two_entries(idx, deleted=dead)
    for v in dead:
        assert idx.vid_slots(v) == []
    assert idx.dead_counts().sum() == 0
    idx.close()


# ---- 5. files -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,metric", KINDS)
def test_file_round_trip_and_refusals(tmp_path, kind, metric):
    idx, db = built(kind, metric)
    idx.update_vector(3, rows(kind, 1, 77)[0])  # a tombstone in two lists
    xq = rows(kind, 5, 13)
    ans = [idx.search(xq, k, params={"nprobe": NLIST}) for k in (10, 500)]
    idx.dump(tmp_path, "s.000")
    buf = (tmp_path / "s.000" / sf.FILE[kind]).read_bytes()
    table = dict(table_of(kind, idx, metric), soar_lambda=LAM, reordering=False)
    parsed = sf.read_spilled(buf, kind, table)
    off, codes, ids = idx.export_lists()
    assert np.array_equal(parsed["list_off"], off) and np.array_equal(parsed["ids"], ids)
    assert np.array_equal(parsed["codes"], codes[:, :parsed["code_size"]])
    with pytest.raises(ValueError, match="magic"):
        qf.read_quantised(buf, kind, table)

    idx2 = spilled(kind, metric)
    idx2.add_vectors(idx.get_vectors(0, N))
    assert idx2.load(tmp_path, "s.000") == N
    for a, k in zip(ans, (10, 500)):
        b = idx2.search(xq, k, params={"nprobe": NLIST})
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))
    assert_two_entries(idx2)
    idx2.dump(tmp_path, "again.000")
    assert (tmp_path / "again.000" / sf.FILE[kind]).read_bytes() == buf

    # an unspilled table refuses the spilled file, a spilled one the unspilled file and another lambda: untrained again
    plain = make(kind, metric, **({"reordering": False} if kind == "VEARCH" else {}))
    plain.add_vectors(db)
    with pytest.raises(Exception):
        plain.load(tmp_path, "s.000")
    assert not plain.is_trained
    plain.train()
    plain.add_pending()
    plain.dump(tmp_path, "p.000")
    pbuf = (tmp_path / "p.000" / qf.FILE[kind]).read_bytes()
    qf.read_quantised(pbuf, kind, dict(table_of(kind, plain, metric), reordering=False))
    for other, name in ((spilled(kind, metric), "p.000"), (spilled(kind, metric, soar_lambda=2.0), "s.000")):
        other.add_vectors(db)
        with pytest.raises(Exception):
            other.load(tmp_path, name)
        assert not other.is_trained
        other.close()
    for i in (idx, idx2, plain):
        i.close()


# ---- 6. the engine ------------------------------------------------------------------------------------------------
def eng_mod():
    from vearch_b200 import engine
    return engine


def engine_with(path, kind, lam, name="t"):
    from vearch_b200 import wire
    e = eng_mod().GammaEngine(str(path), space_name=name)
    p = params_of(kind, IP, training_threshold=2000, **({"reordering": False} if kind == "VEARCH" else {}))
    if lam:
        p["soar_lambda"] = lam
    e.create_table(name, D, kind, p, fields=(("_id", wire.DT_STRING, False),))
    return e


ENGINE_KINDS = ["IVFPQFastScan", "IVFRABITQ", "VEARCH"]


def engine_ids(res):
    return [[it["fields"]["_id"] for it in r["items"]] for r in res]


def engine_answers(e, xq, topn=100):
    res = e.search(xq, topn, index_params={"nprobe": NLIST})
    return engine_ids(res), [[it["score"] for it in r["items"]] for r in res]


def feed(e, db, extra=None):
    from vearch_b200 import wire
    for i, v in enumerate(db):
        ex = [] if extra is None else [("f1", extra[i].tobytes(), wire.DT_VECTOR)]
        assert e.add_doc(f"doc{i}", v, extra_fields=ex) == 0


@pytest.mark.parametrize("kind", ENGINE_KINDS)
def test_engine_spilled_table(tmp_path, kind):
    n = 2500
    db, xq = rows(kind, n, 31), rows(kind, 4, 32)
    e = engine_with(tmp_path, kind, LAM)
    feed(e, db)
    e.wait_indexed(n)
    assert e.add_doc("doc5", db[6]) == 0 and e.delete_doc("doc7") == 0
    e.wait_indexed(n)
    for ids in engine_ids(e.search(xq, 100, index_params={"nprobe": NLIST})):
        assert len(ids) == 100 and len(set(ids)) == 100 and b"doc7" not in ids
    e.close()


@pytest.mark.parametrize("kind,metric", KINDS)
def test_memory_charge_counts_two_entries(kind, metric):
    """the admission charge of a spilled index: the same store growth, twice the index entries of the rows it holds"""
    plain, sp = spilled(kind, metric, soar_lambda=0), spilled(kind, metric)
    for n_total in (1, N, 5 * N):
        g0, r0, i0 = plain.memory_charge(n_total)
        g1, r1, i1 = sp.memory_charge(n_total)
        assert (g0, r0) == (g1, r1) and r0 > 0
        assert i0 == r0 * (plain.code_size + 8) and i1 == 2 * i0
    plain.close()
    sp.close()


@pytest.fixture
def no_limit_after():
    yield
    eng_mod().set_memory_limit(0)
    eng_mod().set_memory_total(0, 0)


def limit_to(nbytes):
    """a device limit of nbytes: 50 % of a total of 2 nbytes"""
    eng_mod().set_memory_total(0, 2 * nbytes)
    eng_mod().set_memory_limit(50)
    assert eng_mod().memory_ledger(0)[2] == nbytes


@pytest.mark.parametrize("kind", ENGINE_KINDS)
def test_memory_limit_refuses_spilled_rows_at_twice_the_entry_cost(tmp_path, kind, no_limit_after):
    """a limit with room for the first document's store growth and 1.5 times its rows' unspilled entries: the unspilled
    table takes the document, the spilled one (two entries a row) is refused"""
    ref = {lam: spilled(kind, IP, soar_lambda=lam) for lam in (0, LAM)}  # an engine's index of the same parameters
    (g0, r0, i0), (g1, r1, i1) = ref[0].memory_charge(1), ref[LAM].memory_charge(1)
    for x in ref.values():
        x.close()
    assert (g0, r0) == (g1, r1) and i1 == 2 * i0 > 0
    x = rows(kind, 4, 51)
    for lam in (0, LAM):
        e = engine_with(tmp_path / f"m{lam}", kind, lam)
        limit_to(1)
        assert e.add_doc("doc0", x[0]) != 0  # refused; the pools are trimmed before refusing
        usage = eng_mod().memory_ledger(0)[0]
        limit_to(usage + g0 + i0 + i0 // 2)
        rc = e.add_doc("doc0", x[0])
        if lam:
            assert rc != 0 and e.status()["doc_num"] == 0
        else:
            assert rc == 0 and e.status()["doc_num"] == 1
        limit_to(usage + g0 + 2 * i0 + (1 << 20))
        assert e.add_doc("doc1", x[1]) == 0
        eng_mod().set_memory_limit(0)
        e.close()


@pytest.mark.parametrize("kind", ENGINE_KINDS)
def test_backup_of_a_spilled_table(tmp_path, kind):
    """Backup writes the spilled file Dump writes, two live entries per document, and a table restored from it answers
    as the leader did"""
    import shutil
    n = 2500
    leader, follower = tmp_path / "leader", tmp_path / "follower"
    db, xq = rows(kind, n, 61), rows(kind, 4, 62)
    e = engine_with(leader, kind, LAM)
    feed(e, db)
    e.wait_indexed(n)
    assert e.add_doc("doc5", db[6]) == 0 and e.delete_doc("doc7") == 0
    e.wait_indexed(n)
    before = engine_answers(e, xq)
    assert e.dump() == 0
    e.backup()
    rel = "retrieval_model_index/emb.000/" + sf.FILE[kind]
    buf = (leader / "backup" / rel).read_bytes()
    assert buf == (leader / rel).read_bytes()
    t = spilled(kind, IP)
    table = dict(table_of(kind, t, IP), soar_lambda=LAM, reordering=False)
    t.close()
    parsed = sf.read_spilled(buf, kind, table)
    live = parsed["ids"][parsed["ids"] >= 0]
    assert np.array_equal(np.bincount(live, minlength=n), np.full(n, 2))
    lists = np.repeat(np.arange(NLIST), np.diff(parsed["list_off"]))[parsed["ids"] >= 0]
    for v in range(0, n, 97):  # the two entries of a document are in two lists
        assert len(set(lists[live == v])) == 2
    e.close()
    for name in os.listdir(leader / "backup"):  # the follower takes the backup as a snapshot
        shutil.copytree(leader / "backup" / name, follower / name)
    f = engine_with(follower, kind, LAM)
    assert f.load() == 0
    assert f.status()["index_status"] == 2
    assert engine_answers(f, xq) == before
    f.close()


@pytest.mark.parametrize("kind", ENGINE_KINDS)
def test_add_field_index_with_soar_on_a_second_field(tmp_path, kind):
    """AddFieldIndexWithParams puts a spilled index on a second vector field; a search on that field answers as a table
    created with the same spilled index on those rows"""
    from vearch_b200 import wire
    n = 2500
    db, f1, xq = rows(kind, n, 71), rows(kind, n, 72), rows(kind, 4, 73)
    p = params_of(kind, IP, training_threshold=2000, **({"reordering": False} if kind == "VEARCH" else {}))
    e = eng_mod().GammaEngine(str(tmp_path / "a"), space_name="mv")
    e.create_table("mv", D, kind, p, fields=(("_id", wire.DT_STRING, False),),
                   extra_vectors=[("f1", D, "FLAT", {"metric_type": "InnerProduct"})])
    feed(e, db, extra=f1)
    e.wait_indexed(n)
    e.add_field_index("f1", kind, dict(p, soar_lambda=LAM))
    assert e.dump() == 0  # waits for the run-time build to swap in
    e.wait_indexed(n)
    e.vec_name = "f1"
    got = engine_answers(e, xq)
    g = engine_with(tmp_path / "b", kind, LAM)
    feed(g, f1)
    g.wait_indexed(n)
    want = engine_answers(g, xq)
    assert got == want
    for ids in got[0]:
        assert len(ids) == 100 and len(set(ids)) == 100
    e.close()
    g.close()


# ---- 7. bad values and the other types ----------------------------------------------------------------------------
@pytest.mark.parametrize("value", [-1.0, -1e-9, float("nan"), float("inf")])
def test_bad_lambda_is_refused(value):
    for kind in ("IVFPQFastScan", "IVFRABITQ", "VEARCH"):
        with pytest.raises(Exception, match="invalid soar_lambda"):
            make(kind, L2, soar_lambda=value)


def test_engine_bad_lambda_is_code_4(tmp_path):
    from vearch_b200 import wire
    for kind in ("IVFRABITQ", "VEARCH"):
        e = eng_mod().GammaEngine(str(tmp_path / kind), space_name="b")
        p = params_of(kind, IP, soar_lambda=float("nan"))
        with pytest.raises(eng_mod().GammaStatusError) as ex:
            e.create_table("b", D, kind, p, fields=(("_id", wire.DT_STRING, False),))
        assert ex.value.code == 4 and "invalid soar_lambda" in str(ex.value)
        e.close()


@pytest.mark.parametrize("kind", ["IVFPQ", "IVFFLAT", "GPU_IVFPQ", "GPU_IVFFLAT", "FLAT", "BINARYIVF"])
def test_other_types_ignore_the_key(kind):
    def one(extra):
        p = {"ncentroids": NLIST, "nprobe": 8, "training_threshold": 1000, "metric_type": "L2"}
        if kind in ("IVFPQ", "GPU_IVFPQ"):
            p["nsubvector"] = 8
        p.update(extra)
        if kind == "BINARYIVF":
            idx = gi().BinaryIVFIndex(BITS, p)
            db, xq = rows(kind, N, 1), rows(kind, 6, 2)
        else:
            idx = gi().GammaIndex(kind, D, p)
            db, xq = rows("IVFPQ", N, 1), rows("IVFPQ", 6, 2)
        idx.add_vectors(db)
        idx.train()
        idx.add_pending()
        out = idx.search(xq, 20, params={"nprobe": 8})
        idx.close()
        return out

    a, b, c = one({}), one({"soar_lambda": LAM}), one({"soar_lambda": -1})
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[1], c[1])
