// K5 / K11 query-major list scan: the pipeline the IVF-PQ (kernels_ivfpq.cu) and IVFPQFastScan (kernels_pqfs.cu) codecs
// share.
//
// One CTA (LS_NT threads) per (query, group of <= pg probes).  Thread 0 streams the codes of the group's lists through a
// TMA bulk ring over the flat (list, tile) sequence, so the next list's first tiles are in flight while the CTA prepares
// that list.  Each thread scores LS_NT-strided entries of a tile from a [code byte][256] table in shared memory; an entry
// inside the score window and the queue's bound has its id read (tombstone, deletion / filter bitmaps) and enters the
// CandQueue.
//
// A codec supplies what differs:
//   Entry                             element type of the [code_bytes()][256] table
//   kDis0                             the score starts from the probe's coarse distance (coarse_dis is read only then)
//   kMinCtasPerSm                     CTAs per SM the register allocation must admit (0: ptxas chooses)
//   pt(MW)                            entries per thread per tile of the vector-load instantiations (MW = code bytes / 4)
//   code_bytes(), tile_entries()      bytes per entry, entries per tile (a multiple of LS_NT; pt(MW) * LS_NT when MW > 0)
//   cta_begin(tab, q, METRIC)         once per CTA, while the first tiles are in flight
//   list_begin(tab, list, METRIC)     when a list starts
//   Acc, start(dis0), finish(acc)     an entry's score is finish(start(dis0) + its table entries, added in code order)
// A hook that writes the table ends with the barrier that publishes it.
//
// A codec whose codes are not one per byte (bit-packed IVF-PQ) also declares kCodeSum = true and supplies
//   table_entries()                   Entry elements of its table (a multiple of 4: the code stages behind it stay
//                                     16-byte aligned)
//   code_sum(code, tab, acc)          acc + the entry's table entries in code order; `code` is the entry's first byte in
//                                     the stage, not 4-byte aligned in general; it may read the aligned 32-bit word
//                                     holding the entry's last byte (the launcher pads the window by 16 bytes)
// and is launched with MW = 0 only.  The other codecs keep the [code_bytes()][256] table and table_sum.
//
// A kCodeSum codec whose entries are too wide for one thread each (IVFRABITQ) also declares kLanes = true and supplies
//   lanes()                           L, a power of two <= 32: L consecutive threads score one entry together
//   score_lanes(code, tab, lane)      the entry's score, returned in each of its L lanes (lane = tid % L); every thread
//                                     of the CTA calls it the same number of times, so it may shuffle within its group
// Its tile_entries() is then a multiple of LS_NT / L; start / finish / code_sum are not called.
#pragma once
#include "common.cuh"

namespace gb {

constexpr int LS_NT = 256;
constexpr int LS_NST = 2;
constexpr int LS_MAX_PG = 32;  // probes per CTA

// w[0, MW) = the first MW 32-bit words of code, by the widest vector loads its alignment allows (codes are 4 MW bytes)
template <int MW>
__device__ __forceinline__ void load_code_words(const unsigned char* __restrict__ code, uint32_t* w) {
  if (MW % 4 == 0) {
#pragma unroll
    for (int i = 0; i < MW / 4; i++) {
      const uint4 v = reinterpret_cast<const uint4*>(code)[i];
      w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
    }
  } else if (MW % 2 == 0) {
#pragma unroll
    for (int i = 0; i < MW / 2; i++) {
      const uint2 v = reinterpret_cast<const uint2*>(code)[i];
      w[2 * i] = v.x, w[2 * i + 1] = v.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < MW; i++) w[i] = reinterpret_cast<const uint32_t*>(code)[i];
  }
}

// acc += tab[j][code[j]] for j = 0, 1, ... in order: 4 MW code bytes read as words, or (MW = 0) nbytes bytes one by one
template <int MW, class Acc, class Entry>
__device__ __forceinline__ Acc table_sum(const unsigned char* __restrict__ code, const Entry* __restrict__ tab, Acc acc,
                                         int nbytes) {
  if (MW > 0) {
    uint32_t w[MW > 0 ? MW : 1];
    load_code_words<MW>(code, w);
#pragma unroll
    for (int i = 0; i < MW; i++) {
      const uint32_t x = w[i];
      acc += tab[(4 * i + 0) * 256 + (x & 0xffu)];
      acc += tab[(4 * i + 1) * 256 + ((x >> 8) & 0xffu)];
      acc += tab[(4 * i + 2) * 256 + ((x >> 16) & 0xffu)];
      acc += tab[(4 * i + 3) * 256 + (x >> 24)];
    }
  } else {
    for (int j = 0; j < nbytes; j++) acc += tab[j * 256 + code[j]];
  }
  return acc;
}

// LsCodeSum<Codec>::value: the codec declares kCodeSum (and then supplies table_entries / code_sum)
template <class Codec, class = void>
struct LsCodeSum {
  static constexpr bool value = false;
};
template <class Codec>
struct LsCodeSum<Codec, decltype(void(Codec::kCodeSum))> {
  static constexpr bool value = Codec::kCodeSum;
};

// LsLanes<Codec>::value: the codec scores an entry with lanes() threads (and supplies score_lanes)
template <class Codec, class = void>
struct LsLanes {
  static constexpr bool value = false;
};
template <class Codec>
struct LsLanes<Codec, decltype(void(Codec::kLanes))> {
  static constexpr bool value = Codec::kLanes;
};

// threads that score one entry
template <class Codec>
__host__ __device__ __forceinline__ int ls_lanes(const Codec& c) {
  if constexpr (LsLanes<Codec>::value) {
    return c.lanes();
  } else {
    return 1;
  }
}

// Entry elements of the codec's table
template <class Codec>
__host__ __device__ __forceinline__ int ls_table_entries(const Codec& c) {
  if constexpr (LsCodeSum<Codec>::value) {
    return c.table_entries();
  } else {
    return c.code_bytes() * 256;
  }
}

// an entry's sum over the table: the codec's own for kCodeSum codecs, table_sum otherwise
template <int MW, class Codec, class Acc, class Entry>
__device__ __forceinline__ Acc ls_entry_sum(const Codec& c, const unsigned char* code, const Entry* tab, Acc acc,
                                            int nbytes) {
  if constexpr (LsCodeSum<Codec>::value) {
    return c.code_sum(code, tab, acc);
  } else {
    return table_sum<MW>(code, tab, acc, nbytes);
  }
}

// the launcher's arguments; the kernel takes them one by one, with its pointers __restrict__ (passed as this struct,
// two IVF-PQ instantiations spilled)
struct ListScanArgs {
  const int32_t* probe_ids;  // [nq][ld_probe]; the first nprobe of a row are scanned, < 0 = no list
  const float* coarse_dis;   // [nq][ld_probe]
  int nprobe, ld_probe, pg;
  ListDirectory dir;
  int k;
  FilterArgs f;
  const int* gate_cnt;  // non-null: only queries with gate_cnt[q] > gate_cap are scanned
  int gate_cap;
  const int* row_limit;  // non-null: [nq][ld_probe] rows scanned of each probed list
  bool sorted_out;       // false: partial[..][k - 1] = the largest key, the others in any order
  unsigned long long* partial;  // [nq][ceil(nprobe / pg)][k]
};

template <class Codec, int METRIC, int MW>
__global__ void __launch_bounds__(LS_NT, Codec::kMinCtasPerSm)
    list_scan_kernel(Codec c, const int32_t* __restrict__ probe_ids, const float* __restrict__ coarse_dis, int nprobe,
                     int ld_probe, int pg, ListDirectory dir, int k, FilterArgs f, const int* __restrict__ gate_cnt,
                     int gate_cap, const int* __restrict__ row_limit, bool sorted_out,
                     unsigned long long* __restrict__ partial, int tile_e, int KP, int SORTN) {
  using Entry = typename Codec::Entry;
  static_assert(!LsCodeSum<Codec>::value || MW == 0, "a kCodeSum codec runs the generic layout only");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int cb = c.code_bytes();
  const int tile_bytes = tile_e * cb;
  // the table sits at the start of the dynamic window: its shared address is a link-time constant, so every gather is
  // LDS [byte_offset + imm]  with no base add
  Entry* tab = reinterpret_cast<Entry*>(smem_raw);
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(tab + ls_table_entries(c));
  unsigned char* stages = reinterpret_cast<unsigned char*>(buf + SORTN);
  __shared__ __align__(8) uint64_t full_bar[LS_NST];
  __shared__ int s_cnt;
  __shared__ unsigned long long s_tau;
  __shared__ int g_list[LS_MAX_PG], g_len[LS_MAX_PG], g_tile0[LS_MAX_PG + 1];
  __shared__ float g_dis0[Codec::kDis0 ? LS_MAX_PG : 1];

  const int tid = threadIdx.x;
  const int q = blockIdx.y, grp = blockIdx.x;
  // flag-gated launch (safety net of the tensor-core filter, kernels_pqtc.cu): only queries whose candidate list
  // overflowed are scanned
  if (gate_cnt && gate_cnt[q] <= gate_cap) return;
  if (cta_cancelled(f.cancel, kCsListScan)) return;
  unsigned long long* out = partial + ((int64_t)q * gridDim.x + grp) * k;
  const int p0 = grp * pg;
  const int np = min(pg, nprobe - p0);

  if (tid == 0) {
    int acc = 0;
    for (int i = 0; i < np; i++) {
      const int64_t qp = (int64_t)q * ld_probe + p0 + i;
      const int l = probe_ids[qp];
      int len = (l >= 0 && l < dir.nlist) ? dir.len[l] : 0;  // key < 0: "not enough centroids" (ivfpq.cc:640)
      // phase A of the tensor-core filter scans only a prefix of its lists (kernels_pqtc.cu)
      if (row_limit) len = min(len, row_limit[qp]);
      g_list[i] = l;
      g_len[i] = len;
      if (Codec::kDis0) g_dis0[i] = coarse_dis[qp];
      g_tile0[i] = acc;
      acc += (len + tile_e - 1) / tile_e;
    }
    g_tile0[np > 0 ? np : 0] = acc;
    for (int s = 0; s < LS_NST; s++) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  CandQueue cq{buf, &s_cnt, &s_tau, k, KP, SORTN};
  cq.init();  // __syncthreads inside: g_* and barriers visible
  const int total_tiles = np > 0 ? g_tile0[np] : 0;
  if (total_tiles == 0) {
    for (int i = tid; i < k; i += LS_NT) out[i] = kKeySentinel;
    return;
  }

  // producer cursor (thread 0 only)
  int pr_pi = 0;
  auto issue = [&](int gt) {
    while (gt >= g_tile0[pr_pi + 1]) pr_pi++;
    const int ti = gt - g_tile0[pr_pi];
    const int n_e = min(tile_e, g_len[pr_pi] - ti * tile_e);
    const uint32_t bytes = ((uint32_t)n_e * cb + 15u) & ~15u;
    const int s = gt % LS_NST;
    mbar_arrive_expect_tx(&full_bar[s], bytes);
    bulk_g2s(stages + (size_t)s * tile_bytes, dir.codes[g_list[pr_pi]] + (int64_t)ti * tile_e * cb, bytes,
             &full_bar[s]);
  };
  if (tid == 0)
    for (int gt = 0; gt < LS_NST && gt < total_tiles; gt++) issue(gt);

  c.cta_begin(tab, q, METRIC);

  int pi = -1;  // consumer cursor
  float dis0 = 0.f;
  const int64_t* __restrict__ lids = nullptr;
  // entries per thread per tile: compile-time for the vector-load code layouts (gives the compiler PT independent
  // chains to interleave), runtime for the generic layout
  constexpr int PT = MW > 0 ? Codec::pt(MW) : 1;
  const int per_thread = MW > 0 ? PT : tile_e / (LS_NT / ls_lanes(c));
  int est = 0;  // upper bound of the queue fill, identical in every thread

  for (int gt = 0; gt < total_tiles; gt++) {
    int npi = pi < 0 ? 0 : pi;
    while (gt >= g_tile0[npi + 1]) npi++;
    if (npi != pi) {  // first tile of a new list
      pi = npi;
      if (Codec::kDis0) dis0 = g_dis0[pi];
      lids = dir.ids[g_list[pi]];
      c.list_begin(tab, g_list[pi], METRIC);
    }
    const int ti = gt - g_tile0[pi];
    const int n_e = min(tile_e, g_len[pi] - ti * tile_e);
    const int s = gt % LS_NST;
    mbar_wait(&full_bar[s], (gt / LS_NST) & 1);
    const unsigned long long tau = s_tau;
    // score window and the queue's bound folded into one float interval: two compares per entry, the
    // order-preserving key is only built for entries inside it
    const float tb = key_bound<METRIC>(tau);
    const float lo_b = METRIC == kMetricL2 ? f.min_score : fmaxf(tb, f.min_score);
    const float hi_b = METRIC == kMetricL2 ? fminf(tb, f.max_score) : f.max_score;
    const unsigned char* st = stages + (size_t)s * tile_bytes;
    int pushed = 0;

    auto consider = [&](int e, float dis) {
      bool pred = e < n_e && dis <= hi_b && dis >= lo_b;
      unsigned long long key = kKeySentinel;
      if (pred) {
        const int64_t raw = lids[(int64_t)ti * tile_e + e];
        pred = raw >= 0;  // tombstone (gamma_index_ivfpq.h:930)
        const uint32_t vid = (uint32_t)raw;
        if (pred) pred = ctx_is_valid(f.del_bits, f.filter_bits, vid);
        key = make_key(score2ord<METRIC>(dis), vid);
        pred = pred && key < tau;
      }
      cq.push_warp(pred, key);
      pushed |= pred ? 1 : 0;
    };
    if (MW > 0) {
      typename Codec::Acc acc[PT];
#pragma unroll
      for (int u = 0; u < PT; u++) {
        // entries past n_e read stale-but-in-bounds stage bytes; they are masked in consider()
        acc[u] = table_sum<MW>(st + (size_t)(u * LS_NT + tid) * cb, tab, c.start(dis0), cb);
      }
#pragma unroll
      for (int u = 0; u < PT; u++) consider(u * LS_NT + tid, c.finish(acc[u]));
    } else {
      if constexpr (LsLanes<Codec>::value) {
        // L threads per entry; only the group's first lane offers it to the queue (e = tile_e masks the others)
        const int L = c.lanes();
        const int lane = tid & (L - 1);
        for (int u = 0; u < per_thread; u++) {
          const int e = u * (LS_NT / L) + tid / L;
          const float dis = c.score_lanes(st + (size_t)e * cb, tab, lane);
          consider(lane == 0 ? e : tile_e, dis);
        }
      } else {
        for (int u = 0; u < per_thread; u++) {
          const int e = u * LS_NT + tid;
          consider(e, e < n_e ? c.finish(ls_entry_sum<MW>(c, st + (size_t)e * cb, tab, c.start(dis0), cb)) : 0.f);
        }
      }
    }
    // stage consumed + pushes done; the count is identical in every thread (no 2nd barrier needed)
    est += __syncthreads_count(pushed) * per_thread;
    if (tid == 0 && gt + LS_NST < total_tiles) issue(gt + LS_NST);
    if (gt + 1 < total_tiles && est + tile_e > cq.cap()) {
      cq.flush();
      est = 0;
    }
  }
  __syncthreads();
  if (sorted_out) {
    cq.flush(true);
  } else {
    // The caller wants the k best and their bound, not their order (phase A of the tensor-core filter): exact radix
    // select, no sort; the largest key -- the sentinel when fewer than k entries qualified -- goes to slot k - 1.
    cq.flush(false, true);
    __shared__ unsigned long long s_wmax[LS_NT / 32];
    __shared__ int s_wpos[LS_NT / 32];
    unsigned long long mx = 0;
    int pos = -1;
    for (int i = tid; i < k; i += LS_NT) {
      const unsigned long long v = buf[i];
      if (pos < 0 || v > mx) mx = v, pos = i;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned long long om = __shfl_xor_sync(0xffffffffu, mx, off);
      const int op = __shfl_xor_sync(0xffffffffu, pos, off);
      if (op >= 0 && (pos < 0 || om > mx || (om == mx && op > pos))) mx = om, pos = op;
    }
    if ((tid & 31) == 0) s_wmax[tid >> 5] = mx, s_wpos[tid >> 5] = pos;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < LS_NT / 32; w++)
        if (s_wpos[w] >= 0 && (pos < 0 || s_wmax[w] > mx || (s_wmax[w] == mx && s_wpos[w] > pos))) mx = s_wmax[w], pos = s_wpos[w];
      if (pos >= 0 && pos != k - 1) {
        buf[pos] = buf[k - 1];
        buf[k - 1] = mx;
      }
    }
    __syncthreads();
  }
  for (int i = tid; i < k; i += LS_NT) out[i] = buf[i];
}

// queue geometry of a scan for k and the dynamic shared memory it needs: table, queue, code stages
template <class Codec>
size_t list_scan_smem(const Codec& c, int k, int* KP_out = nullptr, int* SORTN_out = nullptr) {
  const int tile_e = c.tile_entries();
  const int KP = next_pow2(k < 16 ? 16 : k);
  const int SORTN = next_pow2(KP + tile_e + tile_e / 2);  // cap >= tile_e: one tile always fits after a flush
  if (KP_out) *KP_out = KP;
  if (SORTN_out) *SORTN_out = SORTN;
  return (size_t)ls_table_entries(c) * sizeof(typename Codec::Entry) + (size_t)SORTN * 8 +
         (size_t)LS_NST * tile_e * c.code_bytes() + (LsCodeSum<Codec>::value ? 16 : 0);
}
// A CTA's shared memory, static and dynamic together, is at most 227 KiB on sm_90.  The kernel's own static arrays
// (CandQueue's histogram, the probe group's tables, the barriers) take 2688 to 2816 bytes depending on the codec, so
// the dynamic window gets what is left after a 3 KiB reserve; without it a scan within ~3 KiB of the cap was accepted
// here and refused by cudaFuncSetAttribute.  GPU_IVFPQ at M = 128, k' = 2048 needs exactly this window.
constexpr size_t kListScanStaticSmem = 3 * 1024;
constexpr size_t kListScanMaxSmem = 227 * 1024 - kListScanStaticSmem;

// the largest k (<= 4096) a codec's scan can select, 0 if none: the shared memory grows with k only through KP
template <class Codec>
int list_scan_max_k(const Codec& c) {
  for (int k = 4096; k >= 16; k >>= 1)
    if (list_scan_smem(c, k) <= kListScanMaxSmem) return k;
  return 0;
}

// partial[q][group][k], one CTA per (query, group of pg probes); nq <= 65535, 1 <= k <= 4096, 1 <= pg <= LS_MAX_PG
template <class Codec, int METRIC, int MW>
cudaError_t launch_list_scan(const Codec& c, int nq, const ListScanArgs& a, cudaStream_t st) {
  if (nq <= 0 || a.nprobe <= 0) return cudaSuccess;
  if (a.k <= 0 || a.k > 4096 || nq > 65535 || a.pg < 1 || a.pg > LS_MAX_PG) return cudaErrorInvalidValue;
  const int tile_e = c.tile_entries();
  int KP, SORTN;
  const size_t smem = list_scan_smem(c, a.k, &KP, &SORTN);
  if (smem > kListScanMaxSmem) return cudaErrorInvalidValue;
  cudaError_t e =
      cudaFuncSetAttribute(list_scan_kernel<Codec, METRIC, MW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  dim3 grid((a.nprobe + a.pg - 1) / a.pg, nq);
  list_scan_kernel<Codec, METRIC, MW><<<grid, LS_NT, smem, st>>>(c, a.probe_ids, a.coarse_dis, a.nprobe, a.ld_probe, a.pg, a.dir,
                                                                  a.k, a.f, a.gate_cnt, a.gate_cap, a.row_limit,
                                                                  a.sorted_out, a.partial, tile_e, KP, SORTN);
  note_launch();
  return cudaGetLastError();
}

}  // namespace gb
