/*
 * gamma_b200_index.h -- C-ABI of the index-model seam of the gamma hot path on H100.
 *
 * This is the secondary drop-in seam of SURVEY.md 8(b): the shape of the reference's IndexModel
 * plug-in interface (internal/engine/index/index_model.h:229-335) and of its faiss-like wrappers
 * vearch::IndexIVFFlat / IndexIVFPQ / index_factory (internal/engine/index/index.h), flattened to
 * extern "C" with plain pointers and sizes.  The primary seam (the 23 gamma symbols the Go
 * partition server binds through cgo) is include/gamma_api.h and is implemented on top of this
 * one.  Every entry point runs CUDA kernels on the chosen device; there is no CPU path, and
 * creation fails if no CUDA device is present.
 *
 * Conventions: int-returning calls give 0 on success, -1 on error (gb_last_error() has the
 * message, thread-local), -2 when the request was killed.  Metric ids: 0 = InnerProduct,
 * 1 = L2 (squared).  Results are nq x k row-major, best first; unfilled slots have id -1 and
 * score +FLT_MAX (L2) / -FLT_MAX (IP), exactly what faiss heap_reorder leaves behind.
 */
#ifndef GAMMA_B200_INDEX_H_
#define GAMMA_B200_INDEX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gb_index gb_index;

const char *gb_last_error(void);
int gb_device_count(void);
/* kernels launched by this library since load (bench.py's gpu_launches evidence) */
long long gb_launch_count(void);

/* reflector().GetNewIndex(type) + IndexModel::Init(model_parameters, training_threshold)
 * (index/reflector.h:68-80, vector/vector_manager.cc:171; gamma_index_ivfflat.cc:215-291,
 * gamma_index_ivfpq.cc:112-231).  index_type: "FLAT" | "IVFFLAT" | "IVFPQ" | "GPU_IVFFLAT" | "GPU_IVFPQ" | ...
 * (GPU_IVFFLAT / GPU_IVFPQ: IVFFLAT / IVFPQ under gamma's GPU parameter and request contracts, DESIGN.md section 8).
 * model_params_json keys: ncentroids, nprobe, metric_type ("L2"|"InnerProduct"), nsubvector,
 * nbits_per_idx (IVFPQ: 1..8), training_threshold, bucket_init_size, bucket_max_size, store_type ("RocksDB", any
 * case: raw vectors in pinned host memory; anything else: in HBM) (may be NULL/""). */
gb_index *gb_index_create(const char *index_type, int dimension, const char *model_params_json, int device);
/* A GPU_IVFPQ or GPU_IVFFLAT index sharded over devices[0..ndevices) (an ordinal may repeat): global vid v is held by
 * shard v % ndevices, on devices[v % ndevices]; the raw vectors, training, brute force and the cross-shard merge stay on
 * devices[0].  One device, or any other type: gb_index_create on devices[0]. */
gb_index *gb_index_create_sharded(const char *index_type, int dimension, const char *model_params_json,
                                  const int *devices, int ndevices);
/* shards of the index (1 unless sharded), and a handle on shard i's index structures (its lists, centroids, codebook
 * and tables; its own raw store is empty), valid while the index lives: gb_index_destroy frees only the handle */
int gb_index_shard_count(gb_index *index);
gb_index *gb_index_shard(gb_index *index, int shard);
void gb_index_destroy(gb_index *index);
/* the registered type name the index was created under (Index::type) */
const char *gb_index_type(gb_index *index);

/* VectorManager::AddToStore (vector_manager.cc:455): append n raw vectors (n x d fp32). */
int gb_index_add_vectors(gb_index *index, int64_t n, const float *x);
int gb_index_add_vectors_device(gb_index *index, int64_t n, const float *x_dev, int64_t ld);
/* Engine::Update (search/engine.cc:774-850): RawVector update in place + IndexModel::Update (old list
 * entry tombstoned, vector re-appended to its new list; realtime_mem_data.cc:298-320) */
int gb_index_update_vector(gb_index *index, int64_t vid, const float *x);
int gb_index_get_vector(gb_index *index, int64_t vid, float *out);
int gb_index_get_vectors(gb_index *index, int64_t start, int64_t n, float *out); /* n x d */

/* IndexModel::Indexing(): train on the first training_threshold stored vectors
 * (gamma_index_ivfflat.cc:342-411, gamma_index_ivfpq.cc:296-376). */
int gb_index_train(gb_index *index);
/* VectorManager::AddRTVecsToIndex (vector_manager.cc:572-702) -> IndexModel::Add: index every
 * stored vector that is not indexed yet.  del_bitmap (host, may be NULL): docids deleted before
 * they were indexed are skipped (gamma_index_ivfflat.cc:436). */
int gb_index_add_pending(gb_index *index, const uint8_t *del_bitmap);

int64_t gb_index_ntotal(gb_index *index);        /* stored vectors */
int64_t gb_index_indexed_count(gb_index *index); /* vectors present in the index */
int gb_index_is_trained(gb_index *index);
int64_t gb_index_training_threshold(gb_index *index);
int64_t gb_index_mem_bytes(gb_index *index, int which /* 0 = index, 1 = raw vectors in HBM, 2 = raw vectors in host memory */);

/* IndexModel::Search (index_model.h:296-298) with the RetrievalContext flattened:
 * retrieval_params_json = the request's index_params (nprobe, metric_type, recall_num,
 * parallel_on_queries; gamma_index_ivfpq.cc:233-294), brute_force => FLAT scan,
 * del_bitmap / filter_bitmap = docids_bitmap / scalar filter as dense LSB-first bitmaps of
 * bitmap_bits bits (NULL = none), [min_score, max_score] = IsSimilarScoreValid window. */
int gb_index_search(gb_index *index, int nq, const float *x, int k, const char *retrieval_params_json,
                    int brute_force, const uint8_t *del_bitmap, const uint8_t *filter_bitmap, int64_t bitmap_bits,
                    float min_score, float max_score, float *out_scores, int64_t *out_ids);
/* Same with queries and results resident in HBM (x_dev: nq rows, stride ld floats) on `stream`
 * (a cudaStream_t, may be NULL).  Asynchronous: results are ready when the stream is. */
int gb_index_search_device(gb_index *index, int nq, const float *x_dev, int64_t ld, int k,
                           const char *retrieval_params_json, int brute_force, float *out_scores_dev,
                           int64_t *out_ids_dev, void *stream);
/* Same, additionally (or only: out_scores_dev / out_ids_dev may be NULL) writing the nq x k result KEYS,
 * (order-preserving score bits << 32) | local doc id, best first, 0xFF..FF padded: what one partition
 * contributes to the cross-partition merge (one all-gather instead of scores + ids). */
int gb_index_search_device_keys(gb_index *index, int nq, const float *x_dev, int64_t ld, int k,
                                const char *retrieval_params_json, int brute_force, unsigned long long *out_keys_dev,
                                float *out_scores_dev, int64_t *out_ids_dev, void *stream);
/* gb_index_search_device with a deletion and a filter bitmap in device memory on the index's device (either NULL),
 * in gb_index_search's layout: ceil(bitmap_bits / 8) LSB-first bytes, bit set => deleted / allowed, ids at or above
 * bitmap_bits neither; any alignment.  They are read on `stream`; the score window is [min_score, max_score]. */
int gb_index_search_device_filtered(gb_index *index, int nq, const float *x_dev, int64_t ld, int k,
                                    const char *retrieval_params_json, int brute_force, const uint8_t *del_bits_dev,
                                    const uint8_t *filter_bits_dev, int64_t bitmap_bits, float min_score,
                                    float max_score, float *out_scores_dev, int64_t *out_ids_dev, void *stream);
/* Cancellation (RequestContext::is_killed; DESIGN.md section 8, cancellation).  A token is one cancel word in pinned host
 * memory that every device reads; it only ever goes from unset to set.  A search given a token polls it in its scan and
 * re-rank kernels and its host loops, stops early once it is set, and returns -2 when it was set at any time before
 * the search's final synchronise (gb_index_search_device_cancellable: before it returns; a token set later leaves the
 * outputs undefined).  NULL = never cancelled; an unset token changes no result.  A token may serve one search at a
 * time; free it after that search has returned.  create: NULL on failure (gb_last_error). */
typedef struct gb_cancel_token gb_cancel_token;
gb_cancel_token *gb_cancel_token_create(void);
void gb_cancel_token_set(gb_cancel_token *token);
int gb_cancel_token_is_set(gb_cancel_token *token);
void gb_cancel_token_free(gb_cancel_token *token);
/* gb_index_search with the enable_realtime tail (search_unindexed_tail, as gb_index_search_binary) and a cancel token */
int gb_index_search_cancellable(gb_index *index, int nq, const float *x, int k, const char *retrieval_params_json,
                                int brute_force, const uint8_t *del_bitmap, const uint8_t *filter_bitmap,
                                int64_t bitmap_bits, float min_score, float max_score, int search_unindexed_tail,
                                gb_cancel_token *cancel, float *out_scores, int64_t *out_ids);
int gb_index_search_device_cancellable(gb_index *index, int nq, const float *x_dev, int64_t ld, int k,
                                       const char *retrieval_params_json, int brute_force, gb_cancel_token *cancel,
                                       float *out_scores_dev, int64_t *out_ids_dev, void *stream);
/* Test hooks.  cancel_stats: {"kernel": CTAs that skipped their work, ...} for every kernel that polls, on `device`,
 * since the last call (which clears them); *json_out is malloc'd, the caller frees it.  cancel_register: the kill
 * registry behind SetKillStatus with `token` in place of a running search's word (op 1 register under (request_id,
 * partition_id), op 0 remove); no device is involved. */
int gb_debug_cancel_stats(int device, char **json_out, int *out_len);
int gb_debug_cancel_register(const char *request_id, int partition_id, gb_cancel_token *token, int op);
/* {"stage": ms, ...}: device time per stage of the searches run since the last call with timing enabled
 * (CUDA events on the launching stream); *json_out is malloc'd, the caller frees it */
int gb_index_stage_times(gb_index *index, char **json_out, int *out_len);
/* while on, searches that re-rank through the two-pass kernel record per query the candidates whose fp32 rows they
 * read (and wait for the count); gb_index_rerank_survivors hands them over (*out malloc'd, the caller frees it) and
 * clears them */
void gb_index_set_rerank_stats(gb_index *index, int on);
int gb_index_rerank_survivors(gb_index *index, int **out, int64_t *n);
/* device time of the dominant scan kernel(s) of the last search, ms (0 unless timing enabled) */
void gb_index_set_scan_timing(gb_index *index, int on);
float gb_index_last_scan_ms(gb_index *index);
/* name of the scan kernel(s) that served the last search (bench roofline label) */
const char *gb_index_last_scan_kernel(gb_index *index);
/* JSON details of the path that served the last search (e.g. probes scanned exactly before the tensor-core filter) */
const char *gb_index_last_scan_info(gb_index *index);

/* ---- index-state exchange (parity tests share centroids / codebooks / lists with the oracle,
 * SURVEY.md 8c; also the substrate for Dump/Load) ---- */
int gb_index_nlist(gb_index *index);
int gb_index_set_centroids(gb_index *index, const float *centroids, int nlist); /* marks trained */
int gb_index_get_centroids(gb_index *index, float *centroids);
int gb_index_pq_m(gb_index *index);
int gb_index_pq_ksub(gb_index *index); /* centroids per sub-quantiser: 2^nbits_per_idx (IVFPQ), 16 (IVFPQFastScan) */
int gb_index_set_pq_centroids(gb_index *index, const float *pq); /* [M][ksub][dsub] */
int gb_index_get_pq_centroids(gb_index *index, float *pq);
int gb_index_get_precomputed_table(gb_index *index, float *table); /* [nlist][M][ksub] */
/* OPQ rotation of an IVFPQ index created with "opq": {"nsubvector": M} (gamma_index_ivfpq.cc:168-178):
 * A is d x d row-major, y = A x; apply runs the device path the index itself uses */
int gb_index_has_opq(gb_index *index);
int gb_index_set_opq(gb_index *index, const float *A);
int gb_index_get_opq(gb_index *index, float *A);
int gb_index_apply_opq(gb_index *index, int64_t n, const float *x, float *out);
int gb_index_list_len(gb_index *index, int list);
int gb_index_code_size(gb_index *index);
/* copy one inverted list to the host: codes = len x code_size bytes, ids = len int64 */
int gb_index_get_list(gb_index *index, int list, uint8_t *codes, int64_t *ids);
/* test hook: tombstone one entry where it is (and count it dead); never purges by itself */
int gb_index_tombstone(gb_index *index, int list, int pos);
/* The other half of gamma's realtime list container (RTInvertIndex::Delete, RealTimeMemData::CompactIfNeed,
 * index/realtime/realtime_mem_data.cc:186-196, 347-373).  delete: the documents vids[0..n) were deleted; their entries
 * stay in the lists, hidden by the deletion bitmap of each search, and are counted dead (a vid that is in no list, or
 * already counted, is ignored).  purge: every list whose counted dead share (deleted + tombstoned by updates) is
 * >= threshold (the reference: 0.3; 0: every list with a dead entry) is rewritten on the GPU without its tombstoned
 * entries and without the entries whose bit is set in del_bitmap (bitmap_bytes bytes, bit vid & 7 of byte vid >> 3;
 * may be NULL), the survivors in their old order; *dropped (may be NULL) = entries removed.  No search result changes:
 * a dead entry was never returned.  dead_counts: out[nlist], the dead entries counted per list since its last purge.
 * delete and purge are no-ops on a FLAT index. */
int gb_index_delete(gb_index *index, const int64_t *vids, int64_t n);
int gb_index_purge(gb_index *index, float threshold, const uint8_t *del_bitmap, int64_t bitmap_bytes, int64_t *dropped);
int gb_index_dead_counts(gb_index *index, int *out);
/* Test hook: the list entries of vid as (list << 32 | position), out[2], ~0 for none.  An index with SOAR spilling
 * (model parameter "soar_lambda" > 0) holds every indexed vid in two lists; a fresh build puts its primary entry in
 * out[0] and its spilled one in out[1], a loaded index either way round.  An unspilled index leaves out[1] = ~0. */
int gb_index_vid_slots(gb_index *index, int64_t vid, uint64_t *out);
/* Test hook: what admission under SetMemoryLimitConfig charges for storing rows up to n_total -- *store_bytes, the raw
 * store's growth, making room for *rows rows, and *index_bytes, the list entries those rows will take once indexed (two
 * per row with SOAR spilling). */
int gb_index_memory_charge(gb_index *index, int64_t n_total, int64_t *store_bytes, int64_t *rows, int64_t *index_bytes);
/* IndexModel::Dump / Load (index/index_model.h) in gamma's own file formats -- "IvFl" / "IwPQ" header,
 * IndexFlat quantizer, "ilar" inverted lists (index/impl/gamma_index_ivfflat.cc:807-892,
 * gamma_index_ivfpq.cc:1019-1116, index/index_io.cc:108-194): <dir>/<abs_name>/{ivfflat,ivfpq}.index.
 * dump: 0 on success (also when untrained: nothing written, like the reference).  load: the vectors
 * the file indexes must already be in the store (gb_index_add); *load_num = vectors covered, 0 if
 * there is no file.  FLAT indexes: both are no-ops. */
int gb_index_dump(gb_index *index, const char *dir, const char *abs_name);
/* re-pack the inverted lists into one tight allocation (the growable lists of
 * realtime_mem_data.cc never give memory back; neither do ours until this runs).  Also done
 * automatically after a bulk add when more than half of the list memory is dead. */
int gb_index_compact(gb_index *index);
/* test hook: how often the tensor-core mirror of the lists (DESIGN.md section 2) was built in full; appends
 * that fit the reserved tiles update it in place and do not count */
int gb_index_mirror_builds(gb_index *index);
/* test hook (IVFFLAT): the list shifts s_l of the list-major L2 scan, nlist x d floats; its tensor-core operands are
 * x - s_l and y - s_l.  s_l = round(c_l / g_l) * g_l with g_l the largest power of two <= rho_l / sqrt(d) and rho_l half
 * the distance from centroid c_l to its nearest other centroid; s_l = c_l when rho_l = 0 */
int gb_index_get_list_shifts(gb_index *index, float *out);
/* Test hooks over the caches the list-major scans keep beside the lists (DESIGN.md section 3, cache freshness).  None
 * changes index state: each holds the index locks shared and writes only scratch and the caller's buffers.  They take an
 * unsharded index or a shard handle (gb_index_shard).
 * gb_debug_mirror (IVFFLAT, GPU_IVFFLAT): list `list`'s first ceil(len / 128) tensor-core mirror tiles, *tile_floats
 * floats each (the hi then the lo operand of 128 rows), into tiles, and their 128 row norms each into norms, from the
 * live mirror; gb_debug_mirror_rebuilt: the same tiles as a build from the lists into scratch writes them, the live
 * mirror left as it is.  *ntiles = tiles written (at most max_tiles; none when tiles is NULL, or the live mirror does
 * not exist); *state (both) bit 0: the live mirror is current, bit 1: it is disabled (HBM too full).
 * gb_debug_rowptr_rows (IVFFLAT on a "RocksDB" store, or a shard of GPU_IVFFLAT): the rows the winner re-score's
 * row-pointer table points at for vids [v0, v0 + n) (a shard's local vids), rows [n][d]; state[i] 0: an entry of a
 * list, 1: null, 2: points at no list entry (row zeroed where state != 0).
 * gb_debug_pq_norms (IVFPQ at 8 bits): list `list`'s cached |r_e|^2 segment (live, the first min(*len, cached length)
 * entries) and the same segment recomputed from the lists and codebook into scratch (recomputed, *len entries; *len =
 * the list's length); *current: the cache's key matches the lists and the codebook.  live / recomputed may be NULL.
 * gb_debug_pq_tables (IVFPQ at 8 bits): the tensor-core filter's int8 codebook cb8 [M][256][dsub] and cbnrm
 * [M * 256 + 4]: |pq[m][c]|^2, then R^2, sb, D and one unused float. */
int gb_debug_mirror(gb_index *index, int list, int64_t max_tiles, float *tiles, float *norms, int64_t *ntiles,
                    int64_t *tile_floats, int *state);
int gb_debug_mirror_rebuilt(gb_index *index, int list, int64_t max_tiles, float *tiles, float *norms, int64_t *ntiles,
                            int64_t *tile_floats, int *state);
int gb_debug_rowptr_rows(gb_index *index, int64_t v0, int64_t n, float *rows, int *state);
int gb_debug_pq_norms(gb_index *index, int list, float *live, float *recomputed, int64_t *len, int *current);
int gb_debug_pq_tables(gb_index *index, int8_t *cb8, float *cbnrm);
/* test hook (IVF types): the kernel(s) of the last coarse search: "coarse_topk_kernel" (fused), or the score matrix of
 * "dist_tc_kernel+select_rows_kernel" (>= 32 queries) or "dist_tile_kernel+select_rows_kernel" (exact) */
const char *gb_index_last_coarse_kernel(gb_index *index);
int gb_index_load(gb_index *index, const char *dir, const char *abs_name, int64_t *load_num);
/* quantizer->search (gamma_index_ivfflat.cc:568); refuses an untrained index and nprobe outside [1, min(nlist, 4096)] */
int gb_index_coarse_search(gb_index *index, int nq, const float *x, int nprobe, float *out_dis, int64_t *out_ids);
/* search_preassigned (gamma_index_ivfflat.cc:579, gamma_index_ivfpq.cc:730) with caller-given
 * probe lists and coarse distances; refuses an untrained index, topK or nprobe outside [1, 4096] */
int gb_index_search_preassigned(gb_index *index, int nq, const float *x, int k, const int64_t *keys,
                                const float *coarse_dis, int nprobe, const char *retrieval_params_json,
                                const uint8_t *del_bitmap, const uint8_t *filter_bitmap, int64_t bitmap_bits,
                                float min_score, float max_score, float *out_scores, int64_t *out_ids);
/* BINARYIVF (create with index_type "BINARYIVF" and the dimension in bits, a positive multiple of 8): rows, queries
 * and centroids are packed binary vectors of d / 8 bytes, bit i at bit (i & 7) of byte i >> 3.  Scores are Hamming
 * distances (integers as floats, smaller first).  The float entry points that take or return rows, queries or
 * centroids (gb_index_add_vectors*, gb_index_update_vector, gb_index_get_vector(s), gb_index_search*,
 * gb_index_coarse_search, gb_index_search_preassigned, gb_index_set/get_centroids) refuse it. */
int gb_index_add_binary(gb_index *index, int64_t n, const uint8_t *x);
int gb_index_update_binary(gb_index *index, int64_t vid, const uint8_t *x);
int gb_index_get_binary(gb_index *index, int64_t start, int64_t n, uint8_t *out);
int gb_index_search_binary(gb_index *index, int nq, const uint8_t *x, int k, const char *retrieval_params_json,
                           int brute_force, const uint8_t *del_bitmap, const uint8_t *filter_bitmap, int64_t bitmap_bits,
                           float min_score, float max_score, int search_unindexed_tail, float *out_scores, int64_t *out_ids);
int gb_index_search_binary_cancellable(gb_index *index, int nq, const uint8_t *x, int k, const char *retrieval_params_json,
                                       int brute_force, const uint8_t *del_bitmap, const uint8_t *filter_bitmap,
                                       int64_t bitmap_bits, float min_score, float max_score, int search_unindexed_tail,
                                       gb_cancel_token *cancel, float *out_scores, int64_t *out_ids);
int gb_index_set_binary_centroids(gb_index *index, const uint8_t *centroids, int nlist);
int gb_index_get_binary_centroids(gb_index *index, uint8_t *centroids);
/* the float centroids of the +-1 k-means the packed centroids were taken from: nlist x d floats */
int gb_index_get_real_centroids(gb_index *index, float *centroids);
int gb_index_coarse_search_binary(gb_index *index, int nq, const uint8_t *x, int nprobe, float *out_dis, int64_t *out_ids);
int gb_index_search_preassigned_binary(gb_index *index, int nq, const uint8_t *x, int k, const int64_t *keys, int nprobe,
                                       const uint8_t *del_bitmap, const uint8_t *filter_bitmap, int64_t bitmap_bits,
                                       float min_score, float max_score, float *out_scores, int64_t *out_ids);
/* pq.compute_codes on residuals (gamma_index_ivfpq.cc:489-494): codes = n x code_size bytes, bit-packed below
   nbits_per_idx = 8 (code m at bits [m nbits, (m + 1) nbits) of the row, LSB-first) */
int gb_index_pq_encode(gb_index *index, int64_t n, const float *x, const int64_t *assign, uint8_t *codes);
/* IVFPQFastScan encodes raw vectors (assign is ignored, may be NULL): codes = n x ceil(M/2) bytes, sub-quantiser 2j in
   the low nibble of byte j.  The uint8 look-up tables of a query batch: lut8 = nq x M x 16, ab = nq x (a, b), the
   score of an entry being accu * (1/a) + b; metric -1 = the index metric. */
int gb_index_pqfs_lut(gb_index *index, int nq, const float *x, int metric, uint8_t *lut8, float *ab);
/* IVFRABITQ (DESIGN.md section 3, K13): the model's nb_bits and qb; list entries of n rows assigned to lists `assign`
   (n x code_size bytes: nb_bits bit-planes of ceil(d / 32) words, sign plane first, then the fp32 factors |r|^2, f, S);
   the scan's estimate of every entry of list lists[j] for query j, the lists' entries one after another in out, under
   qb in [0, 8] and metric (-1 = the index metric) */
int gb_index_rabitq_nb_bits(gb_index *index);
int gb_index_rabitq_qb(gb_index *index);
int gb_index_rabitq_encode(gb_index *index, int64_t n, const float *x, const int64_t *assign, uint8_t *codes);
int gb_index_rabitq_estimate(gb_index *index, int nq, const float *x, const int64_t *lists, int qb, int metric, float *out);
/* VEARCH (DESIGN.md section 3, K14): nsubvector and the block count (one more than nsubvector when d % nsubvector != 0);
   the codebook, 16 d floats (block b's 16 centres of its width each, from float 16 b (d / nsubvector)); the list codes
   of n rows ((blocks + 1) / 2 bytes, block 2j in the low nibble of byte j) of the residuals to the lists `assign` under
   InnerProduct (assign ignored, may be NULL, under L2); the biased uint8 tables of a query batch, lut = nq x blocks x 16,
   and their multipliers mult = nq floats */
int gb_index_vearch_nsub(gb_index *index);
int gb_index_vearch_blocks(gb_index *index);
int gb_index_vearch_set_codebook(gb_index *index, const float *codebook);
int gb_index_vearch_get_codebook(gb_index *index, float *codebook);
int gb_index_vearch_encode(gb_index *index, int64_t n, const float *x, const int64_t *assign, uint8_t *codes);
int gb_index_vearch_lut(gb_index *index, int nq, const float *x, uint8_t *lut, float *mult);

/* ---- standalone kernels exposed for tests / bench ---- */
/* faiss Clustering restated (k-means), host in/out; obj (niter floats) may be NULL */
int gb_kmeans(int device, const float *x, int64_t n, int d, int k, int niter, int64_t seed, int spherical,
              int max_points_per_centroid, float *centroids, float *obj);
/* The same k-means run, traced step by step (a debug surface for the tests; DESIGN.md §5, training bar).  x: n x d;
 * l2_assign: spherical, assigned by L2; init: NULL, or k x d centroids to start from (hot start).  n_s = the rows
 * trained on: min(n, k * max_points_per_centroid), or n when max_points_per_centroid is 0.  Outputs (all required):
 * sample [n_s] (the rows of x trained on), init_out [k][d], labels [niter][n_s], scores [niter][n_s] (the score each
 * row's key carried), and the centroids [niter][k][d] after the segmented mean (mean), the empty-cluster split (split)
 * and the spherical renormalisation (norm; = split when not spherical). */
int gb_debug_kmeans_trace(int device, const float *x, int64_t n, int d, int k, int niter, int64_t seed, int spherical,
                          int l2_assign, int max_points_per_centroid, const float *init, int64_t *sample,
                          float *init_out, int32_t *labels, float *scores, float *mean, float *split, float *norm);
/* One OPQ training run (the rotation "opq": {"nsubvector": M} learns in front of IVFPQ) over the n x d rows x, for
 * niter rounds, traced (a debug surface for the tests; DESIGN.md §5, OPQ bar).  n_s = min(n, 65536) rows are trained
 * on; T = niter.  Always written: sample [n_s], mean [d], r0 [d][d] (fp64 start), rf [T][d][d] (the fp32 rotation of
 * each round), xty [T][d][d] (X^T Y read back), r [T][d][d] (fp64 rotation each round solves for), sweeps [T] (the
 * Jacobi sweeps of each round's SVD), solve_ms [T] (device time of each round's SVD and R = V U^T).  With detail set
 * also: centred [n_s][d], proj [T][n_s][d], codes [T][n_s][M], recon [T][n_s][d], and per round and subspace (round
 * major) the subspace k-means of gb_debug_kmeans_trace (k = 256, width d / M, no sampling below 256 000 rows; I
 * iterations: 40 in round 0, 4 after it): km_init [256][d / M], km_labels and km_scores [I][n_s], km_mean, km_split
 * and km_norm [I][256][d / M]. */
int gb_debug_opq_trace(int device, const float *x, int64_t n, int d, int M, int niter, int detail, int64_t *sample,
                       float *mean, float *centred, double *r0, float *rf, float *proj, uint8_t *codes, float *recon,
                       float *xty, double *r, float *km_init, int32_t *km_labels, float *km_scores, float *km_mean,
                       float *km_split, float *km_norm, int32_t *sweeps, float *solve_ms);
/* centroid update only: centroids[c] = mean of x[assign == c] in point order */
int gb_kmeans_update(int device, const float *x, int64_t n, int d, int k, const int64_t *assign, float *centroids);
/* router merge (internal/client/client.go:1530-1609) on device memory: dis/ids are
 * nparts x nq x k, outputs nq x k with ids = (partition << 32) | local id */
int gb_merge_partitions_device(int device, const float *dis_dev, const int64_t *ids_dev, int nparts, int nq, int k,
                               int metric, float *out_dis_dev, int64_t *out_ids_dev, void *stream);
/* the same merge from the partitions' result keys [nparts][nq][k] (gb_index_search_device_keys) */
int gb_merge_partition_keys_device(int device, const unsigned long long *keys_dev, int nparts, int nq, int k, int metric,
                                   float *out_dis_dev, int64_t *out_ids_dev, void *stream);

/* exact (CUDA-core fp32) or tensor-core (wgmma 3xTF32) score matrix, host in/out: out[n][m] */
int gb_debug_dist_matrix(int device, const float *x, int n, const float *c, int m, int d, int metric, int use_tc,
                         float *out);

/* The exact re-rank over the index's HBM rows, for tests: nq queries [nq][d], each with ncand candidate vids
 * cand[nq][ncand] (-1: no candidate, at any position), re-ranked to k by the two-pass kernel (two_pass != 0) or the
 * one-pass kernel under the score window of gb_index_search.  The bitmaps (gb_index_search's) screen the candidates as
 * the list scans do before a re-rank: a deleted or filtered-out vid is no candidate.  Results out_dis / out_ids
 * [nq][k].  Two-pass only: out_survivors[nq], the candidates whose fp32 rows were read, and per candidate [nq][ncand] its pass-1 interval
 * [out_lo, out_hi] as scores and out_state: 0 bounded, 1 bounded but withheld from the k-th bound (the interval
 * crosses the score window), 2 unbounded (lo, hi NaN), 3 dead (no candidate; lo, hi NaN). */
int gb_debug_rerank(gb_index *index, int nq, const float *xq, int ncand, const int64_t *cand, int k,
                    const uint8_t *del_bitmap, const uint8_t *filter_bitmap, int64_t bitmap_bits, float min_score,
                    float max_score, int two_pass, float *out_dis, int64_t *out_ids, int *out_survivors, float *out_lo,
                    float *out_hi, int *out_state);
/* the raw store's int8 shadow rows [start, start + n), *row_bytes = round_up(dpad, 16) + 16 bytes each: the int8
 * values, then float {s, e, nrm, 0}.  out == NULL: only *row_bytes. */
int gb_debug_shadow_rows(gb_index *index, int64_t start, int64_t n, uint8_t *out, int64_t *row_bytes);

/* the device's default memory pool, which every search's scratch comes from: bytes in use and the high-water mark
 * since the last reset (after the device's pending work); reset_peak != 0 then restarts the mark at the current use */
int gb_device_pool_usage(int device, int reset_peak, int64_t *used, int64_t *peak);

/* the memory ledger behind SetMemoryLimitConfig (DESIGN.md section 8), device >= 0 or -1 for the host: *usage = the bytes
 * this library holds there (on a device: tracked allocations + the reserved bytes of its default pool),
 * *pool_reserved = that pool's part, *limit = the limit in bytes (0: none); any pointer may be NULL */
int gb_memory_ledger(int device, int64_t *usage, int64_t *pool_reserved, int64_t *limit);
/* test hook: the total memory SetMemoryLimitConfig's percentage applies to on a device (-1: the host) becomes `bytes`;
 * 0 restores the real one (cudaDeviceProp::totalGlobalMem; the host's MemTotal or cgroup v1 limit) */
void gb_memory_set_total(int device, int64_t bytes);

/* Backup (include/gamma_api.h, DESIGN.md section 8) test hooks.  hold: op 1 makes the next Backup wait after its capture
 * and before it writes, op 0 lets it go on, op -1 only reads; returns 0 (off), 1 (set) or 2 (a Backup is waiting).  It
 * never blocks a Backup unless set.  stage: the bytes the last finished capture (Dump or Backup) staged in HBM and in
 * pinned host memory. */
int gb_debug_backup_hold(int op);
int gb_debug_backup_stage(int64_t *device_bytes, int64_t *host_bytes);
/* A capture of an index's file as Dump and Backup take it (index lists packed on the device into a stage, in the
 * file's order: per list its codes of code_size bytes on disk, then its ids as stored).  out (may be NULL) receives
 * min(cap, *bytes) of the staged lists; *on_host = 1 when the device could not hold the stage.  An unsharded index
 * only; an untrained one or FLAT stages nothing. */
int gb_index_capture_lists(gb_index *index, uint8_t *out, int64_t cap, int64_t *bytes, int *on_host);

/* ---- host-logic test hooks: run the C++ wire codecs of the gamma boundary without a GPU ---- */
/* an engine over `path` (may be "") made without looking for a device, for the checks that need none; Close frees it */
void *gb_debug_engine_create(const char *path);
/* RequestConcurrentController (search/engine.cc:47-119): op 0 threshold, 1 in-flight, 2 set threshold (<= 0: system value),
 * 3 Acquire(value) -> 1/0, 4 Release(value) */
int gb_debug_concurrency(int op, int value);
int gb_debug_parse_search_request(const char *buf, int len, char **json_out, int *out_len);
int gb_debug_roundtrip_doc(const char *buf, int len, char **out, int *out_len);
int gb_debug_parse_table(const char *buf, int len, char **json_out, int *out_len);
int gb_debug_encode_response(int nq, int k, const double *scores, const char *const *keys, int total, char **out,
                             int *out_len);
/* the run-time index records (AddFieldIndexWithParams / RemoveFieldIndex) at the end of a snapshot's last len bytes,
 * as JSON {"bytes": n, "records": [[field, has_index, type, params], ...]}; -1 if a record does not parse */
int gb_debug_index_records(const char *tail, int64_t len, char **json_out, int *out_len);

#ifdef __cplusplus
}
#endif
#endif /* GAMMA_B200_INDEX_H_ */
