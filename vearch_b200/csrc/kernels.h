// Host-callable launchers of the sm_90a kernels (one per row of SURVEY.md 8a).
// Plain pointers + stream, no torch types.  All device matrices are row-major fp32 with a row
// stride ("ld") that is a multiple of 4 floats so rows are 16-byte aligned.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gb {

constexpr int kMetricIP = 0;  // DistanceComputeType::INNER_PRODUCT (gamma default, gamma_index_ivfflat.cc:55)
constexpr int kMetricL2 = 1;

// number of kernels launched by this library so far (bench.py's gpu_launches evidence)
void note_launch(int n = 1);
long long launch_count();

// A search's cancel word as its kernels poll it (DESIGN.md section 8, cancellation).  word: mapped host memory that only
// ever goes from 0 to 1 (RequestContext::is_killed); seen: 4 bytes of device memory, zeroed when the search starts, on
// the device the kernel runs on.  Every CTA reads `seen`; one CTA in kCancelPollStride also reads `word` and, finding it
// set, sets `seen`, so most CTAs never cross PCIe.  Every CTA that skips has found `seen` or `word` set and leaves
// `seen` set, so the kernels after it in stream order skip too.  word == nullptr: never cancelled.
struct CancelPoll {
  const uint32_t* word = nullptr;
  uint32_t* seen = nullptr;
};
constexpr int kCancelPollStride = 32;

struct FilterArgs {            // RetrievalContext (index/index_model.h:86-110)
  const uint32_t* del_bits;    // bit set => docid deleted            (nullable)
  const uint32_t* filter_bits; // bit set => docid passes the filter  (nullable = no filter)
  float min_score, max_score;  // IsSimilarScoreValid window
  // the search's cancel word: a CTA of a polling kernel that finds it set leaves its outputs unwritten
  CancelPoll cancel;
};

// Kernels that poll the cancel word; a CTA that skips its work adds 1 to its kernel's counter (device memory, per
// device).  cancel_skips_take adds the counters of `device` to acc[kCancelSites] and clears them.
enum CancelSite {
  kCsDistTile,        // dist_tile_kernel (FLAT distance tiles)
  kCsSelectRows,      // select_rows_kernel (FLAT selection; scored inputs only)
  kCsHammingTile,     // hamming_tile_kernel (BINARYIVF brute force)
  kCsIvfflatScan,     // ivfflat_scan_kernel (IVF-Flat query-major)
  kCsIvfflatScanWarp, // ivfflat_scan_warp_kernel (IVF-Flat query-major, short rows)
  kCsListmajorTma,    // ivf_listmajor_tma_kernel
  kCsListmajorPipe,   // ivf_listmajor_pipe_kernel
  kCsSegSelect,       // seg_select_kernel (IVF-Flat list-major, large k)
  kCsListScan,        // list_scan_kernel (IVF-PQ, IVFPQFastScan, IVFRABITQ, VEARCH, BINARYIVF query-major)
  kCsPqtcScan,        // pqtc_scan_kernel
  kCsPqRescore,       // pq_rescore_kernel
  kCsRerank,          // rerank_kernel
  kCsRerankPrefilter, // rerank_prefilter_kernel
  kCancelSites
};
const char* cancel_site_name(int site);
int register_cancel_skips(cudaError_t (*take)(int device, unsigned long long* acc));
cudaError_t cancel_skips_take(int device, unsigned long long* acc);

// ---- K1/K2/K6/K8: tiled exact distance kernel ------------------------------------------
// out[i][j] = |X_i - C_j|^2 (L2) or <X_i, C_j> (IP), i<n, j<m.  d multiple of 4.
// cancel: the search's cancel word, polled by every CTA (none by default)
cudaError_t launch_dist_matrix(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                               int metric, float* out, int64_t ldo, cudaStream_t st, CancelPoll cancel = {});
// best[i] = min over j of key(score(X_i,C_j), j + col_base) via atomicMin; caller pre-fills
// best with 0xFF.. .  Lowest j wins ties (faiss IndexFlat::assign, "first minimum wins").
cudaError_t launch_dist_argmin(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                               int metric, unsigned long long* best, int col_base, cudaStream_t st);

// tensor-core (wgmma, 3xTF32) variants of the two calls above (norms accumulated in-kernel).
// Scores agree with the exact kernel to ~1e-6 relative and are bit-equal on integer-valued
// operands below 2^11.
cudaError_t launch_dist_matrix_tc(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                                  int metric, float* out, int64_t ldo, cudaStream_t st);
cudaError_t launch_dist_argmin_tc(const float* X, int64_t ldx, int n, const float* C, int64_t ldc, int m, int d,
                                  int metric, unsigned long long* best, cudaStream_t st);
// rows of x (n x d, stride ldx) -> 128-row operand tiles in the canonical tensor-core layout (per K = 16 chunk a
// TF32 head and an fp32 remainder, tc_mirror_tile_floats(k16) floats per tile) and norms[row] = |x_row|^2; rows
// past n are zero
cudaError_t launch_tc_stage_rows(const float* x, int64_t ldx, int64_t n, int d, int k16, float* tiles, float* norms,
                                 cudaStream_t st);
// fused coarse quantiser (3xTF32 scores, bit-equal to launch_dist_matrix_tc): every query's k best keys, sorted
// ascending, sentinel padded: out[q * k + i].  a_* / c_*: launch_tc_stage_rows of the queries and the centroids;
// nsm: the device's SM count (one CTA each); ws: coarse_topk_workspace_bytes of device memory.
constexpr int kCoarseMaxK = 64;
size_t coarse_topk_workspace_bytes(int nq, int nlist, int k, int nsm);
cudaError_t launch_coarse_topk(const float* a_tiles, const float* a_norms, int nq, const float* c_tiles, const float* c_norms,
                               int nlist, int k16, int metric, int k, int nsm, void* ws, unsigned long long* out,
                               cudaStream_t st);

// ---- K7: top-k selection / merge ----------------------------------------------------------
// Per row r: select the k best of m candidates.  Input is either scores (fp32, vid = id_base+col)
// or ready-made keys.  Output keys sorted ascending (sentinel padded) in out_keys[r*k..].
cudaError_t launch_select_scores(const float* scores, int64_t ld, int nrows, int m, int64_t id_base, int k, int metric,
                                 FilterArgs f, unsigned long long* out_keys, int64_t out_stride, cudaStream_t st);
cudaError_t launch_select_keys(const unsigned long long* keys, int64_t ld, int nrows, int m, int k,
                               unsigned long long* out_keys, int64_t out_stride, cudaStream_t st);
// keys -> (score, id) in the reference's output order (heap_reorder): L2 (score, id) ascending;
// IP score descending, larger id first among equal scores.  Sentinels -> id -1, score +-FLT_MAX.
cudaError_t launch_decode_keys(const unsigned long long* keys, int64_t ld, int nrows, int k, int metric, float* out_dis,
                               int64_t* out_ids, int64_t id_or /* OR-ed into valid ids */, cudaStream_t st);
// keys -> int32 ids / float scores only (coarse quantiser output)
cudaError_t launch_split_keys(const unsigned long long* keys, int64_t n, int metric, float* out_scores, int32_t* out_ids,
                              cudaStream_t st);

// ---- K3: IVF-Flat list scan ---------------------------------------------------------------
struct ListDirectory {            // device-resident mirror of RTInvertIndex (T1)
  const float* const* vecs;       // [nlist] -> len x dpad fp32 rows (codes_array_)
  const uint8_t* const* codes;    // [nlist] -> len x M bytes (IVFPQ)
  const int64_t* const* ids;      // [nlist] -> len int64, top bit = tombstone (idx_array_)
  const int* len;                 // [nlist] published length
  int nlist;
};
// partial[q][part][k]; *nparts_out (<= ivfflat_scan_nparts) = parts actually written per query.
// One CTA per (query, group of (probe, split) work items).  *kernel_out = the name of the kernel launched.
cudaError_t launch_ivfflat_scan(const float* xq, int64_t ldq, int nq, int d, const int32_t* probe_ids, int nprobe,
                                ListDirectory dir, int max_list_len, int avg_list_len, int k, int metric, FilterArgs f,
                                unsigned long long* partial, int* nparts_out, const char** kernel_out, cudaStream_t st);
int ivfflat_scan_nparts(int nprobe, int max_list_len);
// *nst = ring depth (4, 3 or 2) of the generic query-major scan at row width d (a multiple of 4) and k, 0 if none fits
// (on the current device; an error if its image of the kernel cannot be queried)
cudaError_t ivfflat_scan_stages(int d, int k, int* nst);
// *max_d = the largest row width (a multiple of 4) the generic scan serves at k = 4096: IVFFLAT and GPU_IVFFLAT refuse
// any d whose padded width is above it (4604 on sm_90; pinned, and restated from the shared-memory formula, in the tests)
cudaError_t ivfflat_scan_max_dim(int* max_d);

// K3 list-major (tensor cores): (query, probe) pairs grouped by list; tile = 128 pairs x 128 rows.
struct LmTile {
  int list, pair0, npairs, row0, nrows, seg;
  int grp;  // ordinal of this (list, pair group): its slot in the staged-query scratch
};
// List shifts (L2 only): every list-major operand is staged as x - s_l, s_l the row of its list in shifts [nlist][ldq]
// (the pair's list for queries), so the expanded form |x - s|^2 + |y - s|^2 - 2 (x - s).(y - s) works on residual-sized
// norms; nullptr = unshifted.  launch_list_shifts writes s_l = round(c_l / g_l) * g_l, g_l the largest power of two
// <= rho_l / sqrt(d), rho_l half the distance from c_l to its nearest other centroid (s_l = c_l when rho_l = 0).
cudaError_t launch_list_shifts(const float* cent, int64_t ldc, int nlist, int d, float* shifts, cudaStream_t st);
// scores[pair_off[j] + r] = score(query pair_q[j], row r of its list)
cudaError_t launch_ivf_listmajor_tc(const float* xq, int64_t ldq, int d, const LmTile* tiles, int ntiles,
                                    const int32_t* pair_q, const int64_t* pair_off, ListDirectory dir,
                                    const float* shifts, int metric, float* scores, cudaStream_t st);
// device-side grouping of the (query, probe) pairs by list: histogram + scans (totals[0..2] = score
// floats, tiles, valid pairs), then slot assignment and the tile table
cudaError_t launch_lm_count_scan(const int32_t* probe_ids, int64_t npairs, ListDirectory dir, int32_t* cnt,
                                 int32_t* start, int64_t* base_off, int32_t* tile_start, int64_t* totals,
                                 cudaStream_t st);
cudaError_t launch_lm_assign_tiles(const int32_t* probe_ids, int64_t npairs, int nprobe, ListDirectory dir,
                                   const int32_t* cnt, const int32_t* start, int32_t* cursor, const int64_t* base_off,
                                   const int32_t* tile_start, int32_t* pair_q, int64_t* pair_off, int64_t* seg_off,
                                   LmTile* tiles, cudaStream_t st);
// per query: stream its nprobe score segments (seg_off[q*nprobe+p], -1 = none), filter, top-k -> out_keys[q][k]
cudaError_t launch_seg_select(const float* scores, const int64_t* seg_off, const int32_t* probe_ids, int nq, int nprobe,
                              ListDirectory dir, int k, int metric, FilterArgs f, unsigned long long* out_keys,
                              cudaStream_t st);

// K3 list-major with a fused top-k epilogue (k <= kLmkMaxK): work item = (list, 128 pairs, row segment);
// the CTA walks the segment's 128-row tiles, every thread keeps the k best keys of its (query, list)
// pair in shared memory and admits candidates against a per-query bound shared through tau_g.
// out[(j * nseg_max + seg) * k + i], j = q * nprobe + p; unused slots must be pre-set to the sentinel.
constexpr int kLmkMaxK = 64;
constexpr int kLmkSegRows = 2048;
// grouping: cnt/start/cursor/item_start/grp_start: [nlist] ints; totals = {groups, items, pairs} (device side);
// a list's pairs are split evenly over ceil(pairs / gsize) groups
cudaError_t launch_lmk_group(const int32_t* probe_ids, int64_t npairs, ListDirectory dir, int nseg_max, int gsize, int32_t* cnt,
                             int32_t* start, int32_t* cursor, int32_t* item_start, int32_t* grp_start, int64_t* totals,
                             int64_t* pair_j, LmTile* items, cudaStream_t st);
// TMA-fed variant (kernels_tc.cu, "mirror"): the lists are kept a second time pre-split (TF32 head +
// fp32 remainder) and pre-tiled in the exact shared-memory operand layout, so a K chunk of a 128-row
// tile is one contiguous 16 KiB block a single cp.async.bulk brings in; row norms are precomputed.
struct TcMirrorView {
  const float* base;     // tile t of the index at base + t * tile_floats(k16)
  const int64_t* tile0;  // [nlist + 1] first tile of every list
  const float* norms;    // [total_tiles * 128] |y|^2, 0 for padding rows
  int k16;               // row length rounded up to the K chunk (16)
};
inline int64_t tc_mirror_tile_floats(int k16) { return (int64_t)128 * k16 * 2; }
// rows just appended to the lists (row i of x -> position pos[i] of list list[i], list < 0: skipped)
cudaError_t launch_tc_mirror_append(const float* x, int64_t ldx, int64_t n, int d, int k16, const int32_t* list,
                                    const int32_t* pos, const int64_t* tile0, const float* shifts, float* mirror,
                                    float* norms, cudaStream_t st);
cudaError_t launch_tc_mirror_build(ListDirectory dir, int d, int k16, const int64_t* tile0, int64_t total_tiles,
                                   const float* shifts, float* mirror, float* norms, cudaStream_t st);
// a_scratch: per pair group nk chunks of 16 KiB (hi, lo) of the group's 128 queries; a_norms: [group][128]
cudaError_t launch_lm_stage_queries(const float* xq, int64_t ldq, int d, int k16, const LmTile* items, int max_items,
                                    const int64_t* totals, const int64_t* pair_j, int nprobe, const float* shifts,
                                    float* a_scratch, float* a_norms, cudaStream_t st);
cudaError_t launch_ivf_listmajor_tma(const float* a_scratch, const float* a_norms, TcMirrorView mv, const LmTile* items,
                                     int max_items, const int64_t* totals, const int64_t* pair_j, int nprobe,
                                     ListDirectory dir, int k, int nseg_max, int metric, FilterArgs f,
                                     unsigned long long* tau_g, unsigned long long* out, cudaStream_t st);
// register-staged variant: reads the lists themselves (no mirror), any d
cudaError_t launch_ivf_listmajor_pipe(const float* xq, int64_t ldq, int d, const LmTile* items, int max_items,
                                      const int64_t* totals, const int64_t* pair_j, int nprobe, ListDirectory dir,
                                      const float* shifts, int k, int nseg_max, int metric, FilterArgs f,
                                      unsigned long long* tau_g, unsigned long long* out, cudaStream_t st);

// ---- OPQ training helpers (kernels_build.cu) ---------------------------------------------------
// mean[j] = the column means of x (fp64 sums, rounded once); out[i][j] = x[i][j] - mean_j (columns >= d zeroed up to
// ldo).  mean: d floats of device memory
cudaError_t launch_center_rows(const float* x, int64_t ldx, int64_t n, int d, float* mean, float* out, int64_t ldo,
                               cudaStream_t st);
// out[j][i] = x[i][j]  (n x d -> d x n, row stride ldo >= n)
cudaError_t launch_transpose(const float* x, int64_t ldx, int64_t n, int d, float* out, int64_t ldo, cudaStream_t st);
// recon[i][m * dsub + j] = pq[m][codes[i][m]][j]
cudaError_t launch_pq_decode(const uint8_t* codes, int64_t n, const float* pq_centroids, int M, int dsub, float* recon,
                             int64_t ldr, cudaStream_t st);
// The rotation of one OPQ round (kernels_opq.cu): R = V U^T for xty = X^T Y = U S V^T (d x d fp32, row stride ldx),
// the SVD a one-sided Jacobi in fp64 with jacobi_svd.h's rules.  float(R) goes to r32 (row stride ld32, columns >= d
// untouched); R itself to r64 (d x d) when it is not null.  ws: opq_procrustes_ws_bytes(d) bytes of device memory.
// Synchronises st once, to read which singular values vanished; *sweeps (when not null): the Jacobi sweeps run.
size_t opq_procrustes_ws_bytes(int d);
cudaError_t opq_procrustes_device(const float* xty, int64_t ldx, int d, void* ws, float* r32, int64_t ld32,
                                  double* r64, int* sweeps, cudaStream_t st);

// ---- K4/K5: IVF-PQ look-up tables + ADC scan --------------------------------------------
// ip[q][m][c] = <x_q|m, pq_m[c]>   (pq.compute_inner_prod_table); ksub = 2^nbits centroids per sub-quantiser
cudaError_t launch_pq_ip_table(const float* xq, int64_t ldq, int nq, const float* pq_centroids, int M, int dsub,
                               float* ip, cudaStream_t st, int ksub = 256);
// T[l][m][c] = |pq_m[c]|^2 + 2 <centroid_l|m, pq_m[c]>  (IndexIVFPQ::precompute_table), [nlist][M][ksub]
cudaError_t launch_pq_precompute_table(const float* coarse, int64_t ldc, int nlist, const float* pq_centroids, int M,
                                       int dsub, float* T, cudaStream_t st, int ksub = 256);
// partial[q][group][k], group = ceil(nprobe/pg) CTAs per query, each scanning pg (<= 32) probed lists.
// coarse_dis = dis0 per (q, probe).  T nullable for IP.
// ld_probe: row stride of probe_ids / coarse_dis (0 = nprobe; > nprobe scans the first nprobe probes of
// every row).  gate_cnt: when non-null only queries with gate_cnt[q] > gate_cap are scanned.
cudaError_t launch_ivfpq_scan(const float* ip_table, int nq, const int32_t* probe_ids, const float* coarse_dis,
                              int nprobe, int pg, ListDirectory dir, int M, const float* T, int k, int metric,
                              FilterArgs f, unsigned long long* partial, cudaStream_t st, int ld_probe = 0,
                              const int* gate_cnt = nullptr, int gate_cap = 0, const int* row_limit = nullptr,
                              bool sorted_out = true);  // false: partial[..][k - 1] = the largest key, the others in any order
// the largest k (<= 4096) launch_ivfpq_scan (nbits 8) / launch_ivfpq_packed_scan (1..7) can select for M sub-quantisers,
// 0 if none: the [M][2^nbits] fp32 table, the queue and the code stages share one CTA's shared memory
int ivfpq_scan_max_k(int M, int nbits);
// the same scan over bit-packed codes, nbits_per_idx 1..7 (ceil(M nbits / 8) bytes per entry, code m at bits
// [m nbits, (m + 1) nbits), LSB-first); ip_table [nq][M][2^nbits], T [nlist][M][2^nbits]; sorted partials
cudaError_t launch_ivfpq_packed_scan(const float* ip_table, int nq, const int32_t* probe_ids, const float* coarse_dis,
                                     int nprobe, int pg, ListDirectory dir, int M, int nbits, const float* T, int k,
                                     int metric, FilterArgs f, unsigned long long* partial, cudaStream_t st);

// ---- K5 list-major: tensor-core filter + exact re-score (kernels_pqtc.cu) ---------------------------
bool pqtc_supported(int M, int dsub);
// bytes per pair slot of `meta` below: the filter's per-pair record, then (after all max_groups x 256 of those) the
// doubles that its threshold needs besides the bound
size_t pqtc_pair_meta_bytes();
// cb[m][c][.] = int8 rn(pq / sb), sb = rmax2[1] = max |pq| / 127; nrm[m][c] = |pq[m][c]|^2; rmax2[0] = sum_m max_c nrm;
// rmax2[2] = sqrt(sum_m max_c |pq[m][c] - sb cb[m][c]|^2)
cudaError_t launch_pqtc_tables(const float* pq, int M, int dsub, int8_t* cb, float* nrm, float* rmax2, cudaStream_t st);
// phase A's plan: per query its first P_q probes in full (fewest with >= target entries together, at most pa_max);
// probes_a / probes_b = probe_ids with the other phase's probes set to -1, row_limit[q][p] = rows phase A scores exactly
cudaError_t launch_pqtc_plan_phase_a(const int32_t* probe_ids, int64_t npairs, int nprobe, int pa_max, long long target,
                                     const int* list_len, int32_t* probes_a, int32_t* probes_b, int* row_limit,
                                     cudaStream_t st);
// per pair group: int8 operand tile (each row rn(a / sa), sa = max |a| / 127) of a = x - centroid (L2) / x (IP) + the
// pairs' filter records except the bound-dependent threshold; independent of phase A.  Queries whose rows cannot be
// bounded get cand_cnt = cap + 1
cudaError_t launch_pq_stage_pairs(const float* xq, int64_t ldq, int d, const float* coarse, int64_t ldc, const LmTile* items,
                                  int max_items, const int64_t* totals, const int64_t* pair_j, int nprobe,
                                  const float* coarse_dis, const float* rmax2, FilterArgs f, int metric,
                                  unsigned char* a_scratch, void* meta, int64_t max_groups, int* cand_cnt, int cap,
                                  const int* row_limit, cudaStream_t st);
// after phase A and the staging: every staged pair's threshold from bound_keys[q][kprime - 1] (phase A's k'-th key);
// queries without a bound get cand_cnt = cap + 1
cudaError_t launch_pq_bind_bounds(const int64_t* totals, int64_t max_groups, int nprobe, const float* coarse_dis,
                                  const unsigned long long* bound_keys, int64_t bound_stride, int kprime, FilterArgs f,
                                  int metric, void* meta, int* cand_cnt, int cap, cudaStream_t st);
// persistent kernel, one CTA per SM: candidates (probe << 32 | position) appended to cand[q][cap]
cudaError_t launch_pqtc_scan(const unsigned char* a_scratch, const void* meta, const int8_t* cb, const float* pqnorm, const int64_t* pqnorm_off,
                             const LmTile* items, int max_items, const int64_t* totals, ListDirectory dir, int M, int dsub,
                             FilterArgs f, int metric, int* cand_cnt, unsigned long long* cand, int cap, int num_sms,
                             cudaStream_t st);
// |r_e|^2 of every list entry: out[off[l] + pos] (L2; cached beside the lists, streamed to the filter kernel with the codes)
cudaError_t launch_pq_entry_norms(ListDirectory dir, int nlist, int max_len, int M, const float* nrm, const int64_t* off,
                                  float* out, cudaStream_t st);
// out[q][kprime] = best kprime of keys_a[q] + the re-scored candidates (queries with cand_cnt > cap untouched)
cudaError_t launch_pq_rescore(const float* ip_table, int nq, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                              ListDirectory dir, int M, const float* T, const int* cand_cnt, const unsigned long long* cand,
                              int cap, const unsigned long long* keys_a, int64_t keys_a_stride, int kprime, int metric,
                              const int* row_limit, FilterArgs f, bool sorted_out, unsigned long long* out, cudaStream_t st);
// queries with cand_cnt > cap: out[q] = best kprime of partial[q][ngroups][kprime]
cudaError_t launch_pq_fallback_merge(const int* cand_cnt, int cap, int nq, const unsigned long long* partial, int ngroups,
                                     int kprime, unsigned long long* out, cudaStream_t st);
// K5r exact re-rank of ADC candidates (gamma_index_ivfpq.cc:675-726).  Row of vid: raw_segments[vid >> seg_shift] +
// (vid & (2^seg_shift - 1)) * ld_raw; seg_shift 0 makes raw_segments a per-vid row-pointer table.  host_rows: the rows
// are in mapped host memory (a variant with more rows in flight per warp for PCIe latency).
cudaError_t launch_rerank(const unsigned long long* cand_keys, int ncand, int nq, const float* xq, int64_t ldq, int d,
                          const float* const* raw_segments, int seg_shift, int64_t ld_raw, bool host_rows, int k,
                          int metric, FilterArgs f, unsigned long long* out_keys, cudaStream_t st);
// The same re-rank in two passes (rows in HBM with an int8 shadow, RawStore): candidates are bounded from their shadow
// rows (shadow_segs, the same segments as raw_segments, shadow_stride = round_up(d, 16) + 16 bytes apart) and only
// those that can still reach the top k have their fp32 rows read and scored.  The output keys equal launch_rerank's.
// survivors (nullable): per query, the candidates whose fp32 row was read.  intervals (nullable, tests only):
// [nq][ncand] pass-1 results {lo, hi, flo, fhi}: the two ordinals pass 1 keeps (kOrdDead / 0 markers included) and the
// interval's fp32 ends as float bits (NaN for a dead or unbounded candidate).
cudaError_t launch_rerank_prefilter(const unsigned long long* cand_keys, int ncand, int nq, const float* xq, int64_t ldq,
                                    int d, const float* const* raw_segments, int seg_shift, int64_t ld_raw,
                                    const unsigned char* const* shadow_segs, int64_t shadow_stride, int k, int metric,
                                    FilterArgs f, unsigned long long* out_keys, int* survivors, cudaStream_t st,
                                    uint4* intervals = nullptr);
// n fp32 rows (cols values, ld floats apart) -> their shadow rows, out_stride = round_up(cols, 16) + 16 bytes apart:
// int8 qy = rn(y / s), s = max|y| / 127, zero padded, then float4 {s, e >= |y - s qy|, nrm >= |s qy|, 0}; a row with a
// zero or non-finite scale gets {0, inf, inf, 0}
cudaError_t launch_shadow_encode(const float* rows, int64_t ld, int64_t n, int cols, unsigned char* out,
                                 int64_t out_stride, cudaStream_t st);
// IVF-Flat row pointers: rowptr[vid] = the list row holding vid, for every live (not tombstoned) list entry
cudaError_t launch_ivf_rowptrs(ListDirectory dir, int ld, const float** rowptr, cudaStream_t st);

// ---- K11: IVFPQFastScan (kernels_pqfs.cu): 16-centroid PQ on raw vectors, 4-bit codes, uint8 tables -------------
// codes[i][j] = code(2j) | code(2j + 1) << 4, code(m) = argmin_c |x_i|m - pq_m[c]|^2; pq_centroids [M][16][dsub]
cudaError_t launch_pqfs_encode(const float* x, int64_t ldx, int64_t n, const float* pq_centroids, int M, int dsub, uint8_t* codes,
                               cudaStream_t st);
// per query the M x 16 float table (L2 distance / inner product per sub-vector), quantised per sub-quantiser:
// lut8[q][m][c] = floor((v - min_m) a + 0.5), a = 255 / max_m span_m (1 if every span is 0), ab[q] = (a, sum_m min_m)
cudaError_t launch_pqfs_lut(const float* xq, int64_t ldq, int nq, const float* pq_centroids, int M, int dsub, int metric,
                            uint8_t* lut8, float* ab, cudaStream_t st);
// partial[q][group][k] sorted, group = ceil(nprobe / pg) CTAs per query; score = accu * (1 / a) + b
cudaError_t launch_ivfpqfs_scan(const uint8_t* lut8, const float* ab, int nq, const int32_t* probe_ids, int nprobe, int pg,
                                ListDirectory dir, int M, int k, int metric, FilterArgs f, unsigned long long* partial,
                                cudaStream_t st);

// ---- K12: BINARYIVF (kernels_binary.cu): packed binary rows, Hamming distance on the CUDA cores ---------------------
// out[q][r] = popcount(Q_q ^ R_r) over `words` 32-bit words (rows zero padded to whole words; strides in words), exact
// integers as fp32.  Used for every query x rows job: coarse search (rows = centroids), add-time assignment, brute force.
constexpr int kHammingTileMaxQueries = 65535 * 16;  // queries of one launch: grid.y of 16-query tiles
cudaError_t launch_hamming_tile(const uint32_t* Q, int64_t ldq, int nq, const uint32_t* R, int64_t ldr, int m, int words,
                                float* out, int64_t ldo, cudaStream_t st, CancelPoll cancel = {});
// faiss binary_to_real / real_to_binary: bit j of a packed row (byte j >> 3, bit j & 7) <-> +1 / -1 (a float > 0 is 1)
cudaError_t launch_binary_to_real(const uint8_t* x, int64_t ldx, int64_t n, int d, float* out, int64_t ldo, cudaStream_t st);
cudaError_t launch_real_to_binary(const float* x, int64_t ldx, int64_t n, int d, uint8_t* out, int64_t ldo, cudaStream_t st);
// query-major Hamming scan of the probed lists (code_size bytes per entry): partial[q][group][k] sorted, as
// launch_ivfpq_scan; queries [nq][ldq] words, zero padded past code_size bytes
cudaError_t launch_binary_ivf_scan(const uint32_t* queries, int64_t ldq, int nq, const int32_t* probe_ids, int nprobe, int pg,
                                   ListDirectory dir, int code_size, int k, FilterArgs f, unsigned long long* partial,
                                   cudaStream_t st);
int binary_scan_max_k(int code_size);  // the largest k (<= 4096) the scan can select at this code size, 0 if none

// ---- K13: IVFRABITQ (kernels_rabitq.cu): multi-bit RaBitQ codes of residuals, estimator scan ------------------------
// dimensions above this are refused: the encoder keeps 16 bytes per dimension of a vector in shared memory, and the
// scan's integer sums stay below 2^31
constexpr int kRabitqMaxDim = 4096;
int rabitq_code_bytes(int d, int nb_bits);  // 4 (nb_bits ceil(d / 32) + 3): bit-planes, then |r|^2, f, S
// codes[i] of the residual x_i - cents[lists[i]] (rows of x and cents zero padded, strides in floats)
cudaError_t launch_rabitq_encode(const float* x, int64_t ldx, int64_t n, const int32_t* lists, const float* cents, int64_t ldc,
                                 int d, int nb_bits, uint8_t* codes, cudaStream_t st);
// query-major estimator scan of the probed lists: partial[q][group][k] sorted, as launch_ivfpq_scan; qb in [0, 8]
cudaError_t launch_rabitq_scan(const float* xq, int64_t ldq, int nq, const float* cents, int64_t ldc, int d, int nb_bits, int qb,
                               const int32_t* probe_ids, int nprobe, int pg, ListDirectory dir, int k, int metric, FilterArgs f,
                               unsigned long long* partial, cudaStream_t st);
int rabitq_scan_max_k(int d, int nb_bits, int qb);  // the largest k (<= 4096) the scan can select, 0 if none
// test hook: out[out_off[j] + e] = the scan's estimate of entry e of list l_of[j] for query q_of[j], every entry
cudaError_t launch_rabitq_estimate(const float* xq, int64_t ldq, const float* cents, int64_t ldc, int d, int nb_bits, int qb,
                                   int metric, ListDirectory dir, const int32_t* q_of, const int32_t* l_of,
                                   const int64_t* out_off, int npairs, float* out, cudaStream_t st);

// ---- K14: VEARCH (kernels_scann.cu): anisotropic 4-bit codes, fixed-point tables, scan ------------------------------
// blocks of a d-dimensional vector split into nsub: nsub of d / nsub dims, plus one of d % nsub dims when that is > 0.
// The codebook is [16 d] floats: block b's 16 centres of width_b floats each, from float 16 * b * (d / nsub).
int scann_blocks(int d, int nsub);
// codes[i] ((nb + 1) / 2 bytes, block 2j in the low nibble of byte j): lists non-null (IP) codes the residual
// x_i - cents[lists[i]], by CoordinateDescentAHQuantize when ns_threshold is not NaN, else the nearest centre per block;
// lists null (L2): the nearest centre per block of the raw row
cudaError_t launch_scann_encode(const float* x, int64_t ldx, int64_t n, const int32_t* lists, const float* cents, int64_t ldc,
                                int d, int nsub, const float* codebook, double ns_threshold, uint8_t* codes, cudaStream_t st);
// per query: the [nb][16] float table (IP -<q_b, c>, L2 |q_b - c|^2) as biased uint8 lut, and its multiplier mult[q]
cudaError_t launch_scann_lut(const float* xq, int64_t ldq, int nq, int d, int nsub, const float* codebook, int metric,
                             uint8_t* lut, float* mult, cudaStream_t st);
// leaf[q][p] = <q, cents[probe_ids[q][p]]> (fp32, dims in order; 0 for a probe < 0)
cudaError_t launch_scann_leaf(const float* xq, int64_t ldq, int nq, const int32_t* probe_ids, int nprobe, const float* cents,
                              int64_t ldc, int nlist, int d, float* leaf, cudaStream_t st);
// query-major scan of the probed lists: partial[q][group][k] sorted, as launch_ivfpq_scan; leaf [nq][nprobe] read under IP
cudaError_t launch_vearch_scan(const uint8_t* lut, const float* mult, const float* leaf, int nq, const int32_t* probe_ids,
                               int nprobe, int pg, ListDirectory dir, int nb, int k, int metric, FilterArgs f,
                               unsigned long long* partial, cudaStream_t st);
int vearch_scan_max_k(int nb);  // the largest k (<= 4096) the scan can select at nb blocks, 0 if none

// ---- K6/K8: build-side kernels ------------------------------------------------------------
// centroids[c] = (sum of x[perm[off[c]..off[c+1])] in that order) * (1/count); empty => zeros
cudaError_t launch_segment_mean(const float* x, int64_t ldx, int d, const int32_t* perm, const int32_t* off, int k,
                                float* centroids, int64_t ldc, cudaStream_t st);
// out = x - centroids[assign]
cudaError_t launch_residual(const float* x, int64_t ldx, int64_t n, int d, const float* centroids, int64_t ldc,
                            const int32_t* assign, float* out, int64_t ldo, cudaStream_t st);
// codes[i][m] = argmin_c |(x_i - coarse[assign_i])|m - pq_m[c]|^2 over c < ksub, first minimum (coarse nullable =>
// no residual); one byte per code
cudaError_t launch_pq_encode(const float* x, int64_t ldx, int64_t n, const float* coarse, int64_t ldc,
                             const int32_t* assign, const float* pq_centroids, int M, int dsub, uint8_t* codes,
                             cudaStream_t st, int ksub = 256);
// [n][M] codes < 2^nbits -> [n][ceil(M nbits / 8)] rows, code m at bits [m nbits, (m + 1) nbits) LSB-first, high bits 0
cudaError_t launch_pq_pack_codes(const uint8_t* codes, int64_t n, int M, int nbits, uint8_t* packed, cudaStream_t st);
// copy a column slice [col0, col0+w) of x into a dense n x ldo buffer (zero padded to ldo)
cudaError_t launch_slice_cols(const float* x, int64_t ldx, int64_t n, int col0, int w, float* out, int64_t ldo,
                              cudaStream_t st);
// gather rows: out[i] = x[idx[i]]
cudaError_t launch_gather_rows(const float* x, int64_t ldx, const int32_t* idx, int64_t n, int d, float* out,
                               int64_t ldo, cudaStream_t st);
// scale rows to unit L2 norm in place (spherical k-means)
cudaError_t launch_normalize_rows(float* x, int64_t ldx, int64_t n, int d, cudaStream_t st);
// IVF append (RTInvertIndex::AddKeys): row i -> list[i] at pos[i]
cudaError_t launch_ivf_append_vecs(const float* x, int64_t ldx, int64_t n, int d, const int32_t* list, const int32_t* pos,
                                   float* const* list_vecs, int64_t* const* list_ids, int64_t vid0, cudaStream_t st);
cudaError_t launch_ivf_append_codes(const uint8_t* codes, int64_t n, int M, const int32_t* list, const int32_t* pos,
                                    uint8_t* const* list_codes, int64_t* const* list_ids, int64_t vid0,
                                    cudaStream_t st);
// IVF purge (RealTimeMemData::CompactBucket): stable compaction of the nsel lists sel_list[] into fresh regions, keeping
// the entries that are neither tombstoned nor set in del_bits (nullable), in their old order.  The lists are cut into
// chunks of kPurgeChunk entries (chunks[], list by list; sel_chunk0[s] = the first chunk of sel_list[s], [nsel] = nchunks).
constexpr int kPurgeChunk = 1024;
constexpr int kPurgeMaxCodeBytes = 1 << 20;  // keeps a chunk's copy units inside an int
struct PurgeChunk {
  int sel, first;  // ordinal in sel_list, first entry
};
// chunk_off[c] = live entries of the list before chunk c, sel_live[s] = live entries of sel_list[s], vid_range = the
// smallest and largest vid among all entries of the selected lists, dead ones included ({~0, 0}: no entries)
cudaError_t launch_purge_count(ListDirectory dir, const int* sel_list, const int* sel_chunk0, int nsel,
                               const PurgeChunk* chunks, int nchunks, const uint32_t* del_bits, int* chunk_off,
                               int* sel_live, unsigned long long* vid_range, cudaStream_t st);
// live entry with rank r of sel_list[s]: code -> dst_data[s] + r code_bytes, id -> dst_ids[s][r], and
// newpos[vid - vid_min] = list << 32 | r (the caller pre-fills newpos with ~0, so a dropped vid reads ~0).  align: the
// widest power of two <= 16 that divides code_bytes and every source and destination base.  copies = 2 (spilled lists,
// where a vid may have two live entries): newpos holds two slots per vid, [2 (vid - vid_min) + {0, 1}], filled in
// whichever order the entries are met
cudaError_t launch_purge_scatter(ListDirectory dir, const int* sel_list, const PurgeChunk* chunks, int nchunks,
                                 const uint32_t* del_bits, const int* chunk_off, int code_bytes, int align,
                                 void* const* dst_data, int64_t* const* dst_ids, unsigned long long* newpos,
                                 int64_t vid_min, cudaStream_t st, int copies = 1);

// ---- SOAR spilling (kernels_soar.cu, DESIGN.md §8, SOAR spilling) -------------------------------------------
// out[i] = the spilled list of row i (rows x, ldx floats apart, d dims) whose primary list is primary[i]: the list
// c' != primary[i] of least |x - c'|^2 + lambda <r, x - c'>^2 / |r|^2 (r = x - c_primary), the lower id among equal
// losses; -1 when primary[i] is no list, |r|^2 is 0 or not finite, or no loss is finite
cudaError_t launch_soar_spill(const float* x, int64_t ldx, int64_t n, int d, const float* centroids, int64_t ldc, int nlist,
                              const int32_t* primary, float lambda, int32_t* out, cudaStream_t st);
// Per row of m sorted keys (ld apart): the first k whose vid (low 32 bits) has not occurred earlier in the row, in key
// order, sentinel padded; m <= kDedupeMaxKeys
constexpr int kDedupeMaxKeys = 4096;
cudaError_t launch_dedupe_keys(const unsigned long long* keys, int64_t ld, int nrows, int m, int k, unsigned long long* out,
                               int64_t out_stride, cudaStream_t st);
// List pack (the capture of a backup or dump, stage.h): n entries of one list from its slab region into a stage, in the
// index file's order.  Each code keeps the first dst_cb of its src_cb bytes (IVF-Flat rows drop their padding); the
// ids are copied as stored, tombstone bits included, to dst_ids, which may sit at any byte offset.  A list is cut into
// chunks of about kPackChunkBytes of codes, one CTA each, so a long list spreads over the device.
constexpr int kPackChunkBytes = 64 << 10;
struct PackChunk {
  const uint8_t* src_codes;
  const int64_t* src_ids;
  uint8_t* dst_codes;
  uint8_t* dst_ids;
  int n;
};
// align: the widest power of two <= 16 that divides src_cb, dst_cb and every pointer of every chunk
cudaError_t launch_list_pack(const PackChunk* chunks, int nchunks, int src_cb, int dst_cb, int align, cudaStream_t st);
cudaError_t launch_fill_u64(unsigned long long* p, int64_t n, unsigned long long v, cudaStream_t st);
cudaError_t launch_pad_rows(const float* src, int64_t n, int d, float* dst, int64_t ldd, cudaStream_t st);

// ---- scalar filters (kernels_filter.cu) ------------------------------------------------------
// One evaluated filter of a request, on the device columns of its field.  A document d < ncol has a value; d >= ncol
// has none.  Numeric columns are `width` bytes per document (1: uint8, 4: int32 / float, 8: int64 / double) with a
// validity bit each, compared in int64 (is_float 0) or double (is_float 1).  String columns hold an int32 dictionary
// code per document; string-array columns an (offset, count) run of codes in `pool`.
enum FilterKind { kFilterNumeric = 0, kFilterString = 1, kFilterStringArray = 2 };
struct FilterDesc {
  int kind, width, is_float;
  int equal, neg;  // numeric: Equal (NotEqual when neg); string: NotIn when neg
  int has_lo, has_hi, lo_ok, hi_ok, inc_lo, inc_hi;
  int nterms;                    // string: sorted codes in terms[]
  int64_t lo_i, hi_i;
  double lo_f, hi_f;
  int64_t ncol;
  const void* col;               // numeric values
  const uint32_t* valid;         // numeric validity bits
  const int32_t* codes;          // string codes
  const int64_t* arr_off;        // string-array runs
  const int32_t* arr_cnt;
  const int32_t* pool;
  const int32_t* terms;
};
// out[w], w < words: bit b = the request's filters, combined in order (op 0 And, 1 Or, else the first one's set), on
// document 32 w + b; zero at and above n.  *card (zeroed by the caller) += the set bits.
cudaError_t launch_filter_eval(const FilterDesc* fd, int nf, int op, int64_t n, int64_t words, uint32_t* out,
                               unsigned long long* card, cudaStream_t st);
// col[docs[i]] = the low `width` bytes of vals[i], i < m (docids distinct); valid (nullable): bit docs[i] = ok[i]
cudaError_t launch_scatter_column(const int32_t* docs, const uint64_t* vals, const uint8_t* ok, int64_t m, int width,
                                  void* col, uint32_t* valid, cudaStream_t st);

}  // namespace gb
