"""The shared memory of the generic IVF-Flat query-major scan (kernels_ivfflat.cu ivfflat_scan_kernel), restated: the
largest k the parent's fixed 4-stage ring served at each large d, the dimension bound IVFFLAT and GPU_IVFFLAT pin at
create with the launch-time ring depth (4, 3 or 2 stages), and the 4-stage ring kept at every shape it served before.
tests/test_gpu_float_shape_limits.py checks the same numbers against the engine."""

CTA_SMEM = 227 * 1024  # sm_90: shared memory of one CTA, static and dynamic
STATIC_SMEM = 1152  # ivfflat_scan_kernel's own __shared__ arrays (mbarriers, the queue's count, tau, radix histogram)
NT, STAGE_BYTES = 128, 16 * 1024
IVFFLAT_MAX_DIM = 4604  # the pinned bound: the largest padded d served at k = 4096 (two stages there)


def pow2(x):
    return 1 << max(0, (x - 1).bit_length())


def geom(d):
    """ivf_geom: (rows per tile T, bytes per stage) at padded width d"""
    s = d >> 2
    lpr = 1
    while lpr < 32 and s // (lpr * 2) >= 8:
        lpr <<= 1
    g = NT // lpr
    t = g * max(1, STAGE_BYTES // (g * d * 4))
    return t, t * d * 4


def scan_smem(d, k, nst):
    """dynamic shared memory: nst stages, the query, the candidate queue (KP + 2 T keys, a power of two)"""
    t, stage = geom(d)
    return nst * stage + 4 * d + pow2(pow2(max(k, 16)) + 2 * t) * 8


def stages(d, k):
    """ivfflat_scan_stages: the deepest ring of 4, 3 or 2 stages that fits beside the static arrays, 0 if none"""
    for nst in (4, 3, 2):
        if scan_smem(d, k, nst) + STATIC_SMEM <= CTA_SMEM:
            return nst
    return 0


def parent_fits(d, k):
    """the parent's rule: 4 stages, launched whenever the dynamic window alone was <= 227 KiB"""
    return scan_smem(d, k, 4) <= CTA_SMEM


def parent_max_k(d):
    return max((k for k in (16 << i for i in range(9)) if parent_fits(d, k)), default=0)


def max_dim():
    """ivfflat_scan_max_dim: the largest padded width served at k = 4096"""
    d = 4
    while stages(d + 4, 4096):
        d += 4
    return d


def pad(d):
    return (d + 3) // 4 * 4


KP_LADDER = [16 << i for i in range(9)]  # every queue size: k in (KP / 2, KP] share it


def test_parent_table():
    """the largest k the parent's query-major scan served; none from d = 3456: every small-batch search failed"""
    assert {d: parent_max_k(d) for d in (2304, 2560, 3072, 3328, 3456, 4096)} == \
        {2304: 4096, 2560: 2048, 3072: 1024, 3328: 256, 3456: 0, 4096: 0}


def test_pinned_dimension_bound():
    assert max_dim() == IVFFLAT_MAX_DIM >= 4096
    assert stages(IVFFLAT_MAX_DIM, 4096) == 2 and stages(IVFFLAT_MAX_DIM + 4, 4096) == 0
    assert stages(pad(IVFFLAT_MAX_DIM + 1), 4096) == 0  # d = N + 1 pads to N + 4: refused at create
    # every accepted d is served at every k
    for d in range(4, IVFFLAT_MAX_DIM + 1, 4):
        assert all(stages(d, k) >= 2 for k in KP_LADDER), d
    # at k = 4096: 4 stages to d = 2436, 3 to 3184, then 2
    assert [stages(d, 4096) for d in (2048, 2436, 2440, 3184, 3188, 4096)] == [4, 4, 3, 3, 2, 2]


def test_four_stages_wherever_the_parent_launched():
    """the ring stays 4 deep at every (d, k) the parent could launch (its window plus the static arrays fit), so those
    searches run exactly as before; shapes the parent accepted but could not launch now take a shallower ring"""
    changed = []
    for d in range(4, IVFFLAT_MAX_DIM + 1, 4):
        for k in KP_LADDER:
            launched = scan_smem(d, k, 4) + STATIC_SMEM <= CTA_SMEM
            assert (stages(d, k) == 4) == launched, (d, k)
            if parent_fits(d, k) and not launched:
                changed.append((d, k))
    assert changed and all(d > 2048 for d, _ in changed)


def test_bench_shapes_keep_four_stages():
    """bench.py's IVF-Flat workloads (d = 128 and 768) and the warp kernel's largest width, at every k"""
    for d in (128, 768, 1536):
        for k in range(1, 4097):
            assert stages(d, k) == 4, (d, k)
