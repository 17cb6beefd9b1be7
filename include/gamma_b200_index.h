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

/* ---- host-logic test hooks: run the C++ wire codecs of the gamma boundary without a GPU ---- */
/* RequestConcurrentController (search/engine.cc:47-119): op 0 threshold, 1 in-flight, 2 set threshold (<= 0: system value),
 * 3 Acquire(value) -> 1/0, 4 Release(value) */
int gb_debug_concurrency(int op, int value);
int gb_debug_parse_search_request(const char *buf, int len, char **json_out, int *out_len);
int gb_debug_roundtrip_doc(const char *buf, int len, char **out, int *out_len);
int gb_debug_parse_table(const char *buf, int len, char **json_out, int *out_len);
int gb_debug_encode_response(int nq, int k, const double *scores, const char *const *keys, int total, char **out,
                             int *out_len);

#ifdef __cplusplus
}
#endif
#endif /* GAMMA_B200_INDEX_H_ */
