"""The query-major split the probe-group tests size their batches by (tests/test_gpu_probe_groups.py), restated and
checked at the SM counts of the H100 SXM (132) and PCIe (114): every case reaches its pg, one query fewer does not,
the last group is shorter at pg 3 and 7, the GPU types' 512-query cap holds and the partial keys stay small."""
import pytest

from test_gpu_probe_groups import MAX_PG, NPROBE, PG, QUERY_BLOCK, nq_for, ngroups, probes_per_cta

NSM = {"H100 SXM": 132, "H100 PCIe": 114}


def test_split_formula():
    assert probes_per_cta(64, 1, 132) == 1 and probes_per_cta(64, 10000, 132) == MAX_PG
    assert probes_per_cta(32, 10000, 132) == 32  # the issue's batch shape: nq = 10000, nprobe = 32
    assert probes_per_cta(1, 8447, 132) == 1 and probes_per_cta(1, 8448, 132) == 2  # pg = floor(nprobe nq / 4224)
    assert probes_per_cta(64, 131, 132) == 1 and probes_per_cta(64, 132, 132) == 2


@pytest.mark.parametrize("card", list(NSM))
@pytest.mark.parametrize("fam", list(NPROBE))
def test_case_table(fam, card):
    nsm = NSM[card]
    nprobe, cap = NPROBE[fam]
    assert nprobe < nsm * 32  # nq_for is then exact: nprobe * nq crosses a multiple of nsm * 32 at most once a step
    for pg in PG:
        nq = nq_for(pg, nprobe, nsm)
        assert probes_per_cta(nprobe, nq, nsm) == pg
        assert pg == 1 or probes_per_cta(nprobe, nq - 1, nsm) == pg - 1
        assert cap is None or nq <= cap, (fam, pg, nq)
        g = ngroups(nprobe, pg)
        last = nprobe - (g - 1) * pg
        if pg in (3, 7):
            assert 0 < last < pg  # the last group is shorter than the others
        assert g * nq <= 2 * nsm * 32  # the partial keys (nq * ngroups * k') stay within twice one per SM warp
        assert nq < QUERY_BLOCK


def test_case_table_values_at_132_sms():
    """pinned: a change to the restatement shows here before it reaches the GPU tests"""
    assert [nq_for(pg, 64, 132) for pg in PG] == [66, 132, 198, 462, 2112]
    assert [nq_for(pg, 50, 132) for pg in PG] == [85, 169, 254, 592, 2704]
    assert [nq_for(pg, 265, 132) for pg in PG] == [16, 32, 48, 112, 511]
    assert [nq_for(pg, 64, 114) for pg in PG] == [57, 114, 171, 399, 1824]
