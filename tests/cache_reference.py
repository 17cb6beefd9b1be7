"""fp32 restatements of the IVF-PQ caches the tensor-core filter reads (kernels_pqtc.cu, DESIGN.md section 3 K5
list-major): the tables pqtc_tables_kernel derives from the codebook, and the per-entry |r_e|^2 pq_entry_norms_kernel
derives from the list codes.  Each sum is taken in the kernel's order with every FMA rounded once, so a device cache
must equal them bit for bit.  Self-checked without a GPU by test_cache_reference_cpu.py."""
import numpy as np

from rerank_reference import fma32

F32, F64 = np.float32, np.float64


def pq_tables(pq):
    """pq [M][256][dsub] fp32 -> (cb8 int8 [M][256][dsub], cbnrm fp32 [M * 256 + 3]): the int8 codebook rn(pq / sb),
    |pq[m][c]|^2, then R^2 = sum_m max_c |pq[m][c]|^2, sb = max |pq| / 127 (0 when that is 0 or not finite) and
    D = sqrt(sum_m max_c |pq[m][c] - sb cb8[m][c]|^2)"""
    pq = np.asarray(pq, F32)
    M, ksub, dsub = pq.shape
    assert ksub == 256
    cbmax = F32(np.max(np.abs(pq))) if pq.size else F32(0)
    ok = bool(cbmax > 0 and np.isfinite(cbmax))
    sb = F32(cbmax / F32(127)) if ok else F32(0)
    inv = F32(F32(127) / cbmax) if ok else F32(0)
    q = np.clip(np.rint((pq * inv).astype(F32)), -127, 127).astype(F32)
    n2 = np.zeros((M, ksub), F32)
    e2 = np.zeros((M, ksub), F32)
    for j in range(dsub):  # per (m, c): n2 = fmaf(v, v, n2); dv = v - sb qv (contracted to one FMA); e2 = fmaf(dv, dv, e2)
        v = pq[:, :, j]
        n2 = fma32(v, v, n2)
        dv = fma32(np.full_like(v, -sb), q[:, :, j], v)
        e2 = fma32(dv, dv, e2)
    total, err = F32(0), F32(0)
    for m in range(M):  # the per-subquantiser maxima summed in m order
        total = F32(total + n2[m].max())
        err = F32(err + e2[m].max())
    cbnrm = np.concatenate([n2.reshape(-1), np.array([total, sb, np.sqrt(err)], F32)])
    return q.astype(np.int8), cbnrm


def entry_norms(codes, cbnrm, M):
    """|r_e|^2 of list entries with 8-bit codes [n][M]: sum_m cbnrm[m * 256 + code_m], summed in m order in fp32"""
    codes = np.asarray(codes, np.uint8).reshape(-1, M)
    out = np.zeros(len(codes), F32)
    for m in range(M):
        out = (out + cbnrm[m * 256 + codes[:, m].astype(np.int64)]).astype(F32)
    return out
