/*
 * gamma_oracle.c -- CPU restatement of the gamma FLAT / IVF-Flat / IVF-PQ hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (vearch_b200/, libgamma.so)
 * may include, link or call this file.  Legitimate users: tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs.
 *
 * PARITY STATUS: "parity unpinned" at the faiss boundary.  gamma's arithmetic lives in
 * faiss v1.14.1 (cloud/env/install-dependencies.sh:37-55), which is not vendored in the
 * reference tree and not installable here, and the reference ships no golden vectors
 * for this path (SURVEY.md 8c).  Everything that gamma itself decides (loop structure,
 * filters, tombstones, score window, re-rank, parameter defaults, list layout) follows the
 * cited gamma file:line.  Everything faiss decides (heap tie-break, k-means, PQ) is
 * restated from faiss's published algorithm and is marked [faiss-restated].
 *
 * Build: see oracle/Makefile (gcc -O3 -mavx2 -ffp-contract=off -fopenmp).
 * -ffp-contract=off keeps every a*b+c as two roundings so results do not depend on the
 * compiler's FMA choices.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef int64_t idx_t;

#define ORC_METRIC_IP 0 /* DistanceComputeType::INNER_PRODUCT, the gamma default (gamma_index_ivfflat.cc:55) */
#define ORC_METRIC_L2 1

/* realtime_mem_data.h:26-27 : top bit of a list id marks a tombstoned entry */
#define ORC_DEL_MASK ((idx_t)1 << 63)
#define ORC_RECOVER_MASK (~ORC_DEL_MASK)

/* ------------------------------------------------------------------------------------------
 * Heaps [faiss-restated: faiss/utils/Heap.h + ordered_key_value.h, >= v1.7.3]
 * CMax (used for L2): root = largest (value, id); CMin (IP): root = smallest (value, id).
 * cmp2 breaks value ties on the id.  is_max selects the comparator.
 * ---------------------------------------------------------------------------------------- */
static inline int h_cmp(int is_max, float a, float b) { return is_max ? (a > b) : (a < b); }
static inline int h_cmp2(int is_max, float a1, float b1, idx_t a2, idx_t b2) {
  return is_max ? ((a1 > b1) || (a1 == b1 && a2 > b2)) : ((a1 < b1) || (a1 == b1 && a2 < b2));
}
static inline float h_neutral(int is_max) { return is_max ? FLT_MAX : -FLT_MAX; }

static void heap_heapify(int is_max, size_t k, float *val, idx_t *ids) {
  for (size_t i = 0; i < k; i++) {
    val[i] = h_neutral(is_max);
    ids[i] = -1;
  }
}

static void heap_pop(int is_max, size_t k, float *bh_val, idx_t *bh_ids) {
  bh_val--; /* 1-based indexing */
  bh_ids--;
  float val = bh_val[k];
  idx_t id = bh_ids[k];
  size_t i = 1, i1, i2;
  while (1) {
    i1 = i << 1;
    i2 = i1 + 1;
    if (i1 > k) break;
    if (i2 == k + 1 || h_cmp2(is_max, bh_val[i1], bh_val[i2], bh_ids[i1], bh_ids[i2])) {
      if (h_cmp2(is_max, val, bh_val[i1], id, bh_ids[i1])) break;
      bh_val[i] = bh_val[i1];
      bh_ids[i] = bh_ids[i1];
      i = i1;
    } else {
      if (h_cmp2(is_max, val, bh_val[i2], id, bh_ids[i2])) break;
      bh_val[i] = bh_val[i2];
      bh_ids[i] = bh_ids[i2];
      i = i2;
    }
  }
  bh_val[i] = bh_val[k];
  bh_ids[i] = bh_ids[k];
}

static void heap_push(int is_max, size_t k, float *bh_val, idx_t *bh_ids, float val, idx_t id) {
  bh_val--;
  bh_ids--;
  size_t i = k, i_father;
  while (i > 1) {
    i_father = i >> 1;
    if (!h_cmp2(is_max, val, bh_val[i_father], id, bh_ids[i_father])) break;
    bh_val[i] = bh_val[i_father];
    bh_ids[i] = bh_ids[i_father];
    i = i_father;
  }
  bh_val[i] = val;
  bh_ids[i] = id;
}

static void heap_replace_top(int is_max, size_t k, float *bh_val, idx_t *bh_ids, float val, idx_t id) {
  bh_val--;
  bh_ids--;
  size_t i = 1, i1, i2;
  while (1) {
    i1 = i << 1;
    i2 = i1 + 1;
    if (i1 > k) break;
    if (i2 == k + 1 || h_cmp2(is_max, bh_val[i1], bh_val[i2], bh_ids[i1], bh_ids[i2])) {
      if (h_cmp2(is_max, val, bh_val[i1], id, bh_ids[i1])) break;
      bh_val[i] = bh_val[i1];
      bh_ids[i] = bh_ids[i1];
      i = i1;
    } else {
      if (h_cmp2(is_max, val, bh_val[i2], id, bh_ids[i2])) break;
      bh_val[i] = bh_val[i2];
      bh_ids[i] = bh_ids[i2];
      i = i2;
    }
  }
  bh_val[i] = val;
  bh_ids[i] = id;
}

/* sorts the heap in place (best first), drops id==-1 slots to the tail; returns #valid */
static size_t heap_reorder(int is_max, size_t k, float *bh_val, idx_t *bh_ids) {
  size_t i, ii;
  for (i = 0, ii = 0; i < k; i++) {
    float val = bh_val[0];
    idx_t id = bh_ids[0];
    heap_pop(is_max, k - i, bh_val, bh_ids);
    bh_val[k - ii - 1] = val;
    bh_ids[k - ii - 1] = id;
    if (id != -1) ii++;
  }
  size_t nel = ii;
  memmove(bh_val, bh_val + k - ii, ii * sizeof(*bh_val));
  memmove(bh_ids, bh_ids + k - ii, ii * sizeof(*bh_ids));
  for (; ii < k; ii++) {
    bh_val[ii] = h_neutral(is_max);
    bh_ids[ii] = -1;
  }
  return nel;
}

/* ------------------------------------------------------------------------------------------
 * Distances [faiss-restated: fvec_L2sqr / fvec_inner_product].  faiss's SIMD kernels keep
 * 8 running partial sums (one AVX register) and reduce them at the end; we restate that
 * order explicitly so gcc vectorises it without -ffast-math.
 * ---------------------------------------------------------------------------------------- */
static inline float hsum8(const float *a) {
  return ((a[0] + a[4]) + (a[2] + a[6])) + ((a[1] + a[5]) + (a[3] + a[7]));
}

static float fvec_L2sqr(const float *x, const float *y, size_t d) {
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  size_t i = 0;
  for (; i + 8 <= d; i += 8)
    for (int j = 0; j < 8; j++) {
      float t = x[i + j] - y[i + j];
      acc[j] += t * t;
    }
  float s = hsum8(acc);
  for (; i < d; i++) {
    float t = x[i] - y[i];
    s += t * t;
  }
  return s;
}

static float fvec_inner_product(const float *x, const float *y, size_t d) {
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  size_t i = 0;
  for (; i + 8 <= d; i += 8)
    for (int j = 0; j < 8; j++) acc[j] += x[i + j] * y[i + j];
  float s = hsum8(acc);
  for (; i < d; i++) s += x[i] * y[i];
  return s;
}

float orc_l2sqr(const float *x, const float *y, int d) { return fvec_L2sqr(x, y, (size_t)d); }
float orc_inner_product(const float *x, const float *y, int d) { return fvec_inner_product(x, y, (size_t)d); }

/* ------------------------------------------------------------------------------------------
 * RetrievalContext (common/gamma_common_data.h:94-106, index/index_model.h:86-110)
 *   IsValid(id)            : !(filter && !filter.Has(id)) && !docids_bitmap.Test(id)
 *   IsSimilarScoreValid(s) : min_score <= s <= max_score
 * Bitmaps are dense, LSB-first: bit id lives in byte id>>3, mask 1<<(id&7).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  const uint8_t *del_bitmap;    /* bit set => docid deleted (may be NULL) */
  const uint8_t *filter_bitmap; /* bit set => docid passes the scalar filter (may be NULL = no filter) */
  float min_score, max_score;
} orc_ctx;

static inline int bit_test(const uint8_t *bm, idx_t id) { return (bm[id >> 3] >> (id & 7)) & 1; }
static inline int ctx_is_valid(const orc_ctx *c, idx_t id) {
  if (c->filter_bitmap && !bit_test(c->filter_bitmap, id)) return 0;
  if (c->del_bitmap && bit_test(c->del_bitmap, id)) return 0;
  return 1;
}
static inline int ctx_score_ok(const orc_ctx *c, float s) { return s <= c->max_score && s >= c->min_score; }

/* ------------------------------------------------------------------------------------------
 * K1  GammaFLATIndex::Search  (index/impl/gamma_index_flat.cc:130-370, query-parallel mode
 * :286-302, inner loop search_impl :224-281).  db is n rows of d floats, row stride ld.
 * Output: nq*k row-major, sorted best-first, unfilled slots id -1 / neutral value.
 * ---------------------------------------------------------------------------------------- */
int orc_flat_search(const float *db, int64_t ld, int64_t n, int d, const float *xq, int nq, int k, int metric,
                    const uint8_t *del_bitmap, const uint8_t *filter_bitmap, float min_score, float max_score,
                    float *out_dis, int64_t *out_ids) {
  if (k <= 0 || d <= 0) return -1;
  orc_ctx ctx = {del_bitmap, filter_bitmap, min_score, max_score};
  const int is_max = (metric == ORC_METRIC_L2);
#pragma omp parallel for schedule(dynamic)
  for (int i = 0; i < nq; i++) {
    const float *xi = xq + (size_t)i * d;
    float *simi = out_dis + (size_t)i * k;
    idx_t *idxi = out_ids + (size_t)i * k;
    heap_heapify(is_max, k, simi, idxi);
    for (int64_t vid = 0; vid < n; vid++) {
      if (!ctx_is_valid(&ctx, vid)) continue;
      const float *yi = db + vid * ld;
      float dis = is_max ? fvec_L2sqr(xi, yi, d) : fvec_inner_product(xi, yi, d);
      if (!ctx_score_ok(&ctx, dis)) continue;
      if (h_cmp(is_max, simi[0], dis)) {
        heap_pop(is_max, k, simi, idxi);
        heap_push(is_max, k, simi, idxi, dis, vid);
      }
    }
    heap_reorder(is_max, k, simi, idxi);
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * K2  coarse quantiser: quantizer->search / quantizer->assign on a faiss::IndexFlat
 * (gamma_index_ivfflat.cc:253,427,568; gamma_index_ivfpq.cc:156,478,595).
 * [faiss-restated] IndexFlat is an exact search; for >= 20 queries faiss evaluates L2 as
 * |x|^2+|y|^2-2x.y through BLAS, which changes low-order bits only.  We restate it with the
 * direct form, i.e. FLAT search without filters.
 * ---------------------------------------------------------------------------------------- */
int orc_coarse_search(const float *centroids, int nlist, int d, const float *xq, int nq, int nprobe, int metric,
                      float *out_dis, int64_t *out_ids) {
  return orc_flat_search(centroids, d, nlist, d, xq, nq, nprobe, metric, NULL, NULL, -FLT_MAX, FLT_MAX, out_dis,
                         out_ids);
}

/* assign = search with k=1 (first minimum wins) */
int orc_assign(const float *centroids, int nlist, int d, const float *x, int64_t n, int metric, int64_t *out_ids) {
  const int is_max = (metric == ORC_METRIC_L2);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; i++) {
    const float *xi = x + (size_t)i * d;
    float best = h_neutral(is_max);
    idx_t bi = -1;
    for (int c = 0; c < nlist; c++) {
      const float *yc = centroids + (size_t)c * d;
      float dis = is_max ? fvec_L2sqr(xi, yc, d) : fvec_inner_product(xi, yc, d);
      if (h_cmp(is_max, best, dis)) {
        best = dis;
        bi = c;
      }
    }
    out_ids[i] = bi;
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * K3  GammaIVFFlatIndex::search_preassigned (gamma_index_ivfflat.cc:579-787, pmode 0 loop
 * :695-733) + GammaIVFFlatScanner::scan_codes (gamma_index_ivfflat.h:63-91).
 * Inverted lists are given in CSR form: list l = entries [list_off[l], list_off[l+1]) of
 * list_vecs (d floats each, insertion order) and list_ids (int64, top bit = tombstone,
 * realtime_mem_data.h:26-27).
 * ---------------------------------------------------------------------------------------- */
int orc_ivfflat_search_preassigned(const int64_t *list_off, const float *list_vecs, const int64_t *list_ids, int nlist,
                                   int d, const float *xq, int nq, int k, const int64_t *keys, int nprobe, int metric,
                                   const uint8_t *del_bitmap, const uint8_t *filter_bitmap, float min_score,
                                   float max_score, float *out_dis, int64_t *out_ids) {
  if (k <= 0) return -1;
  orc_ctx ctx = {del_bitmap, filter_bitmap, min_score, max_score};
  const int is_max = (metric == ORC_METRIC_L2);
#pragma omp parallel for schedule(dynamic)
  for (int i = 0; i < nq; i++) {
    const float *xi = xq + (size_t)i * d;
    float *simi = out_dis + (size_t)i * k;
    idx_t *idxi = out_ids + (size_t)i * k;
    heap_heapify(is_max, k, simi, idxi);
    for (int ik = 0; ik < nprobe; ik++) {
      idx_t key = keys[(size_t)i * nprobe + ik];
      if (key < 0 || key >= nlist) continue; /* ivfflat.cc:653-659 */
      int64_t b = list_off[key], e = list_off[key + 1];
      for (int64_t j = b; j < e; j++) { /* scan_codes, ivfflat.h:66-89 */
        if (list_ids[j] & ORC_DEL_MASK) continue;
        idx_t vid = list_ids[j] & ORC_RECOVER_MASK;
        if (!ctx_is_valid(&ctx, vid)) continue;
        const float *yj = list_vecs + (size_t)j * d;
        float dis = is_max ? fvec_L2sqr(xi, yj, d) : fvec_inner_product(xi, yj, d);
        if (ctx_score_ok(&ctx, dis) && h_cmp(is_max, simi[0], dis)) heap_replace_top(is_max, k, simi, idxi, dis, list_ids[j]);
      }
    }
    heap_reorder(is_max, k, simi, idxi);
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * Product quantiser [faiss-restated: ProductQuantizer, nbits = 8 => ksub = 256]
 * centroids layout: [M][ksub][dsub] (faiss ProductQuantizer::centroids).
 * ---------------------------------------------------------------------------------------- */
#define ORC_KSUB 256

/* pq.compute_codes (gamma_index_ivfpq.cc:442,494): per sub-space argmin of squared L2, lowest
 * index wins ties. */
int orc_pq_compute_codes(const float *pq_centroids, int M, int dsub, const float *x, int64_t n, uint8_t *codes) {
  const int d = M * dsub;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; i++) {
    for (int m = 0; m < M; m++) {
      const float *xs = x + (size_t)i * d + (size_t)m * dsub;
      const float *cm = pq_centroids + (size_t)m * ORC_KSUB * dsub;
      float best = FLT_MAX;
      int bi = 0;
      for (int c = 0; c < ORC_KSUB; c++) {
        float dis = 0;
        for (int j = 0; j < dsub; j++) {
          float t = xs[j] - cm[(size_t)c * dsub + j];
          dis += t * t;
        }
        if (dis < best) {
          best = dis;
          bi = c;
        }
      }
      codes[(size_t)i * M + m] = (uint8_t)bi;
    }
  }
  return 0;
}

/* residual encode of the add path: GammaIVFPQIndex::Add (gamma_index_ivfpq.cc:455-540):
 * assign -> compute_residuals (:378-391,489: r = x - centroid[list]) -> pq.compute_codes (:494) */
int orc_ivfpq_encode(const float *coarse_centroids, int d, const float *pq_centroids, int M, const float *x, int64_t n,
                     const int64_t *assign, uint8_t *codes) {
  const int dsub = d / M;
  float *res = (float *)malloc(sizeof(float) * (size_t)n * d);
  if (!res) return -1;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; i++) {
    const float *c = coarse_centroids + (size_t)assign[i] * d;
    for (int j = 0; j < d; j++) res[(size_t)i * d + j] = x[(size_t)i * d + j] - c[j];
  }
  int r = orc_pq_compute_codes(pq_centroids, M, dsub, res, n, codes);
  free(res);
  return r;
}

/* [faiss-restated: IndexIVFPQ::precompute_table, use_precomputed_table = 1]
 * T[l][m][c] = |pq_m[c]|^2 + 2 <centroid_l|_m , pq_m[c]>   (SURVEY Appendix A) */
int orc_ivfpq_precompute_table(const float *coarse_centroids, int nlist, int d, const float *pq_centroids, int M,
                               float *table) {
  const int dsub = d / M;
#pragma omp parallel for schedule(static)
  for (int l = 0; l < nlist; l++) {
    for (int m = 0; m < M; m++) {
      const float *cl = coarse_centroids + (size_t)l * d + (size_t)m * dsub;
      for (int c = 0; c < ORC_KSUB; c++) {
        const float *p = pq_centroids + ((size_t)m * ORC_KSUB + c) * dsub;
        float nrm = 0, ip = 0;
        for (int j = 0; j < dsub; j++) {
          nrm += p[j] * p[j];
          ip += cl[j] * p[j];
        }
        table[((size_t)l * M + m) * ORC_KSUB + c] = nrm + 2.0f * ip;
      }
    }
  }
  return 0;
}

/* pq.compute_inner_prod_table (gamma_index_ivfpq.h:166,173): tab[m][c] = <x_m, pq_m[c]> */
static void pq_inner_prod_table(const float *pq_centroids, int M, int dsub, const float *x, float *tab) {
  for (int m = 0; m < M; m++)
    for (int c = 0; c < ORC_KSUB; c++) {
      const float *p = pq_centroids + ((size_t)m * ORC_KSUB + c) * dsub;
      float ip = 0;
      for (int j = 0; j < dsub; j++) ip += x[m * dsub + j] * p[j];
      tab[m * ORC_KSUB + c] = ip;
    }
}

/* pq.compute_distance_table (gamma_index_ivfpq.h:171,248): tab[m][c] = |x_m - pq_m[c]|^2 */
static void pq_distance_table(const float *pq_centroids, int M, int dsub, const float *x, float *tab) {
  for (int m = 0; m < M; m++)
    for (int c = 0; c < ORC_KSUB; c++) {
      const float *p = pq_centroids + ((size_t)m * ORC_KSUB + c) * dsub;
      float dis = 0;
      for (int j = 0; j < dsub; j++) {
        float t = x[m * dsub + j] - p[j];
        dis += t * t;
      }
      tab[m * ORC_KSUB + c] = dis;
    }
}

/* ------------------------------------------------------------------------------------------
 * K4 + K5 + K5r  GammaIVFPQIndex::search_preassigned (gamma_index_ivfpq.cc:730-947, pmode 0
 * :811-848), QueryTables (gamma_index_ivfpq.h:154-309), scan_list_with_table (:923-953),
 * compute_dis re-rank (gamma_index_ivfpq.cc:675-726).
 *
 *  precomputed_table != NULL  => use_precomputed_table = 1 (L2 only):
 *        tab = T[list] + (-2) * ip_table(x),   dis0 = coarse_dis            (ivfpq.h:254-262)
 *  precomputed_table == NULL  => L2: residual = x - centroid, tab = distance_table(residual),
 *        dis0 = 0 (ivfpq.h:246-252);  IP: tab = ip_table(x), dis0 = <x, centroid> (:223-237)
 *  recall_num_param > 0       => ADC heap of max(k, recall_num_param), then exact re-rank from
 *        raw vectors (raw, stride raw_ld); else plain reorder of the ADC heap.
 * List ids carry the tombstone bit; the value returned as label is ids[j] (ivfpq.h:364).
 * ---------------------------------------------------------------------------------------- */
int orc_ivfpq_search_preassigned(const int64_t *list_off, const uint8_t *list_codes, const int64_t *list_ids, int nlist,
                                 int d, int M, const float *coarse_centroids, const float *pq_centroids,
                                 const float *precomputed_table, const float *xq, int nq, int k, const int64_t *keys,
                                 const float *coarse_dis, int nprobe, int metric, int recall_num_param,
                                 const float *raw, int64_t raw_ld, const uint8_t *del_bitmap,
                                 const uint8_t *filter_bitmap, float min_score, float max_score, float *out_dis,
                                 int64_t *out_ids) {
  if (k <= 0) return -1;
  const int dsub = d / M;
  orc_ctx ctx = {del_bitmap, filter_bitmap, min_score, max_score};
  const int is_max = (metric == ORC_METRIC_L2);
  int recall_num = k;
  const int rerank = recall_num_param > 0; /* ivfpq.cc:765 */
  if (recall_num_param > k) recall_num = recall_num_param;
  int err = 0;
#pragma omp parallel
  {
    float *tab = (float *)malloc(sizeof(float) * M * ORC_KSUB);
    float *tab2 = (float *)malloc(sizeof(float) * M * ORC_KSUB);
    float *resid = (float *)malloc(sizeof(float) * d);
    float *rsimi = (float *)malloc(sizeof(float) * recall_num);
    idx_t *ridx = (idx_t *)malloc(sizeof(idx_t) * recall_num);
#pragma omp for schedule(dynamic)
    for (int i = 0; i < nq; i++) {
      const float *xi = xq + (size_t)i * d;
      float *simi = out_dis + (size_t)i * k;
      idx_t *idxi = out_ids + (size_t)i * k;
      heap_heapify(is_max, k, simi, idxi);
      float *recall_simi = simi;
      idx_t *recall_idxi = idxi;
      if (rerank) {
        recall_simi = rsimi;
        recall_idxi = ridx;
        heap_heapify(is_max, recall_num, recall_simi, recall_idxi);
      }
      /* init_query (ivfpq.h:154-175) */
      if (!is_max)
        pq_inner_prod_table(pq_centroids, M, dsub, xi, tab);
      else if (precomputed_table)
        pq_inner_prod_table(pq_centroids, M, dsub, xi, tab2);

      for (int ik = 0; ik < nprobe; ik++) {
        idx_t key = keys[(size_t)i * nprobe + ik];
        if (key < 0 || key >= nlist) continue; /* ivfpq.cc:640-647 */
        int64_t b = list_off[key], e = list_off[key + 1];
        if (b == e) continue;
        /* precompute_list_tables (ivfpq.h:188-309) */
        float dis0 = 0;
        const float *cl = coarse_centroids + (size_t)key * d;
        if (!is_max) {
          dis0 = fvec_inner_product(xi, cl, d);
        } else if (precomputed_table) {
          dis0 = coarse_dis[(size_t)i * nprobe + ik];
          const float *T = precomputed_table + (size_t)key * M * ORC_KSUB;
          for (int t = 0; t < M * ORC_KSUB; t++) tab[t] = T[t] + (-2.0f) * tab2[t]; /* fvec_madd */
        } else {
          for (int j = 0; j < d; j++) resid[j] = xi[j] - cl[j];
          pq_distance_table(pq_centroids, M, dsub, resid, tab);
        }
        /* scan_list_with_table (ivfpq.h:923-953) */
        const uint8_t *codes = list_codes + (size_t)b * M;
        for (int64_t j = b; j < e; j++, codes += M) {
          if (list_ids[j] & ORC_DEL_MASK) continue;
          if (!ctx_is_valid(&ctx, list_ids[j] & ORC_RECOVER_MASK)) continue;
          float dis = dis0;
          const float *t = tab;
          for (int m = 0; m < M; m++) {
            dis += t[codes[m]];
            t += ORC_KSUB;
          }
          if (ctx_score_ok(&ctx, dis) && h_cmp(is_max, recall_simi[0], dis))
            heap_replace_top(is_max, recall_num, recall_simi, recall_idxi, dis, list_ids[j]);
        }
      }
      /* compute_dis (ivfpq.cc:675-726) */
      if (rerank) {
        if (!raw) {
          err = -1;
          continue;
        }
        for (int j = 0; j < recall_num; j++) {
          if (recall_idxi[j] < 0) continue;
          const float *v = raw + (size_t)recall_idxi[j] * raw_ld;
          float dis = is_max ? fvec_L2sqr(xi, v, d) : fvec_inner_product(xi, v, d);
          if (ctx_score_ok(&ctx, dis) && h_cmp(is_max, simi[0], dis)) {
            heap_pop(is_max, k, simi, idxi);
            heap_push(is_max, k, simi, idxi, dis, recall_idxi[j]);
          }
        }
        heap_reorder(is_max, k, simi, idxi);
      } else {
        heap_reorder(is_max, recall_num, recall_simi, recall_idxi);
      }
    }
    free(tab);
    free(tab2);
    free(resid);
    free(rsimi);
    free(ridx);
  }
  return err;
}

/* ------------------------------------------------------------------------------------------
 * mt19937 [faiss-restated: faiss::RandomGenerator wraps std::mt19937; rand_int(max) =
 * mt() % max; rand_float() = mt() / float(mt.max())]
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  uint32_t mt[624];
  int idx;
} orc_mt;

static void mt_seed(orc_mt *g, uint32_t seed) {
  g->mt[0] = seed;
  for (int i = 1; i < 624; i++) g->mt[i] = 1812433253u * (g->mt[i - 1] ^ (g->mt[i - 1] >> 30)) + (uint32_t)i;
  g->idx = 624;
}
static uint32_t mt_next(orc_mt *g) {
  if (g->idx >= 624) {
    for (int i = 0; i < 624; i++) {
      uint32_t y = (g->mt[i] & 0x80000000u) | (g->mt[(i + 1) % 624] & 0x7fffffffu);
      g->mt[i] = g->mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    g->idx = 0;
  }
  uint32_t y = g->mt[g->idx++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

/* [faiss-restated: rand_perm(perm, n, seed)] */
void orc_rand_perm(int64_t *perm, int64_t n, int64_t seed) {
  orc_mt g;
  mt_seed(&g, (uint32_t)seed);
  for (int64_t i = 0; i < n; i++) perm[i] = i;
  for (int64_t i = 0; i + 1 < n; i++) {
    int64_t i2 = i + (int64_t)(mt_next(&g) % (uint32_t)(n - i));
    int64_t t = perm[i];
    perm[i] = perm[i2];
    perm[i2] = t;
  }
}

/* ------------------------------------------------------------------------------------------
 * K6  k-means [faiss-restated: faiss::Clustering::train, ClusteringParameters defaults
 * niter=25 seed=1234 max_points_per_centroid=256; gamma overrides in gamma_index_ivfpq.cc:188-191
 * (niter=10, spherical for IP); gamma's training-set choice is the caller's job
 * (gamma_index_ivfflat.cc:350-405)].
 *   - subsample to k*max_points when n is larger (seeded permutation, seed)
 *   - initial centroids = first k entries of rand_perm(n, seed+1)
 *   - each iteration: exact assign; centroid = sum(members in point order) * (1/count);
 *     empty clusters re-seeded by splitting (split_clusters, EPS = 1/1024, rng(1234));
 *     spherical => renormalise
 * l2_assign: spherical, but assigned by L2 (faiss's default IndexFlatL2 clustering index, which IVFPQFastScan and VEARCH
 * keep under IP).
 * centroids_out: k*d.  If assign_out != NULL it receives the last assignment (n entries, only
 * meaningful when no subsampling happened).  obj_out (may be NULL): niter objective values.
 * ---------------------------------------------------------------------------------------- */
static void km_assign(const float *x, int64_t n, int d, const float *cent, int k, int64_t *assign, float *dis,
                      int use_ip) {
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; i++) {
    const float *xi = x + (size_t)i * d;
    float best = use_ip ? -FLT_MAX : FLT_MAX;
    int64_t bi = 0;
    for (int c = 0; c < k; c++) {
      float v = use_ip ? fvec_inner_product(xi, cent + (size_t)c * d, d) : fvec_L2sqr(xi, cent + (size_t)c * d, d);
      if (use_ip ? (v > best) : (v < best)) {
        best = v;
        bi = c;
      }
    }
    assign[i] = bi;
    dis[i] = best;
  }
}

/* one Lloyd update given an assignment; exported so the GPU update step can be checked alone */
int orc_kmeans_update(const float *x, int64_t n, int d, int k, const int64_t *assign, float *centroids,
                      float *hassign /* k */) {
  memset(centroids, 0, sizeof(float) * (size_t)k * d);
  for (int c = 0; c < k; c++) hassign[c] = 0;
  for (int64_t i = 0; i < n; i++) {
    int64_t c = assign[i];
    hassign[c] += 1.0f;
    float *cc = centroids + (size_t)c * d;
    const float *xi = x + (size_t)i * d;
    for (int j = 0; j < d; j++) cc[j] += xi[j];
  }
  for (int c = 0; c < k; c++) {
    if (hassign[c] == 0) continue;
    float norm = 1.0f / hassign[c];
    float *cc = centroids + (size_t)c * d;
    for (int j = 0; j < d; j++) cc[j] *= norm;
  }
  return 0;
}

int orc_kmeans_split(int d, int k, int64_t n, float *hassign, float *centroids) {
  const float EPS = 1.0f / 1024.0f;
  int nsplit = 0;
  orc_mt g;
  mt_seed(&g, 1234u);
  for (int ci = 0; ci < k; ci++) {
    if (hassign[ci] != 0) continue;
    int cj;
    for (cj = 0;; cj = (cj + 1) % k) {
      float p = (hassign[cj] - 1.0f) / (float)(n - k);
      float r = (float)mt_next(&g) / (float)4294967295u;
      if (r < p) break;
    }
    memcpy(centroids + (size_t)ci * d, centroids + (size_t)cj * d, sizeof(float) * d);
    for (int j = 0; j < d; j++) {
      if (j % 2 == 0) {
        centroids[(size_t)ci * d + j] *= 1 + EPS;
        centroids[(size_t)cj * d + j] *= 1 - EPS;
      } else {
        centroids[(size_t)ci * d + j] *= 1 - EPS;
        centroids[(size_t)cj * d + j] *= 1 + EPS;
      }
    }
    hassign[ci] = hassign[cj] / 2;
    hassign[cj] -= hassign[ci];
    nsplit++;
  }
  return nsplit;
}

/* spherical k-means' renormalisation of the k x d centroids (a zero row stays zero) */
void orc_kmeans_normalize(float *cent, int k, int d) {
  for (int c = 0; c < k; c++) {
    float *cc = cent + (size_t)c * d;
    float nr = 0;
    for (int j = 0; j < d; j++) nr += cc[j] * cc[j];
    if (nr > 0) {
      float s = 1.0f / sqrtf(nr);
      for (int j = 0; j < d; j++) cc[j] *= s;
    }
  }
}

int orc_kmeans(const float *x_in, int64_t n_in, int d, int k, int niter, int64_t seed, int spherical, int l2_assign,
               int max_points_per_centroid, float *centroids_out, int64_t *assign_out, float *obj_out) {
  if (n_in < k) return -1;
  const float *x = x_in;
  int64_t n = n_in;
  float *xsub = NULL;
  if (max_points_per_centroid > 0 && n_in > (int64_t)k * max_points_per_centroid) {
    n = (int64_t)k * max_points_per_centroid;
    int64_t *perm = (int64_t *)malloc(sizeof(int64_t) * n_in);
    orc_rand_perm(perm, n_in, seed);
    xsub = (float *)malloc(sizeof(float) * (size_t)n * d);
    for (int64_t i = 0; i < n; i++) memcpy(xsub + (size_t)i * d, x_in + (size_t)perm[i] * d, sizeof(float) * d);
    free(perm);
    x = xsub;
  }
  int64_t *perm = (int64_t *)malloc(sizeof(int64_t) * n);
  orc_rand_perm(perm, n, seed + 1);
  for (int c = 0; c < k; c++) memcpy(centroids_out + (size_t)c * d, x + (size_t)perm[c] * d, sizeof(float) * d);
  free(perm);
  if (spherical) orc_kmeans_normalize(centroids_out, k, d);

  int64_t *assign = (int64_t *)malloc(sizeof(int64_t) * n);
  float *dis = (float *)malloc(sizeof(float) * n);
  float *hassign = (float *)malloc(sizeof(float) * k);
  for (int it = 0; it < niter; it++) {
    /* faiss's clustering index is an IndexFlatL2 even for spherical k-means unless the caller
       passes an IP index; gamma passes its quantizer, which is IndexFlat(d, metric)
       (gamma_index_ivfpq.cc:156) => IP assign when spherical, unless l2_assign. */
    km_assign(x, n, d, centroids_out, k, assign, dis, spherical && !l2_assign);
    if (obj_out) {
      double obj = 0;
      for (int64_t i = 0; i < n; i++) obj += dis[i];
      obj_out[it] = (float)obj;
    }
    orc_kmeans_update(x, n, d, k, assign, centroids_out, hassign);
    orc_kmeans_split(d, k, n, hassign, centroids_out);
    if (spherical) orc_kmeans_normalize(centroids_out, k, d);
  }
  if (assign_out && !xsub) memcpy(assign_out, assign, sizeof(int64_t) * n);
  free(assign);
  free(dis);
  free(hassign);
  free(xsub);
  return 0;
}

/* ------------------------------------------------------------------------------------------
 * K8  PQ training [faiss-restated: ProductQuantizer::train = M independent k-means, k = 256,
 * on the dsub-wide slices; ClusteringParameters defaults (niter 25, seed 1234, max 256 pts)].
 * x: n x d (already residuals for IVFPQ).  out: [M][256][dsub]
 * ---------------------------------------------------------------------------------------- */
int orc_pq_train(const float *x, int64_t n, int d, int M, int niter, int64_t seed, float *pq_centroids_out) {
  const int dsub = d / M;
  float *slice = (float *)malloc(sizeof(float) * (size_t)n * dsub);
  int rc = 0;
  for (int m = 0; m < M && rc == 0; m++) {
    for (int64_t i = 0; i < n; i++) memcpy(slice + (size_t)i * dsub, x + (size_t)i * d + (size_t)m * dsub, sizeof(float) * dsub);
    rc = orc_kmeans(slice, n, dsub, ORC_KSUB, niter, seed, 0, 0, 256, pq_centroids_out + (size_t)m * ORC_KSUB * dsub, NULL,
                    NULL);
  }
  free(slice);
  return rc;
}

/* ------------------------------------------------------------------------------------------
 * K7  cross-partition merge (router semantics, internal/client/client.go:1530-1609): merge
 * nparts sorted lists of k (score,id) into one sorted top-k.  Ascending for L2, descending for
 * IP; on equal scores the entry from the LATER partition is preferred (client.go:1553-1573).
 * ids out are (partition << 32) | local id.  id -1 slots are skipped.
 * ---------------------------------------------------------------------------------------- */
int orc_merge_partitions(const float *dis, const int64_t *ids, int nparts, int nq, int k, int metric, float *out_dis,
                         int64_t *out_ids) {
  const int asc = (metric == ORC_METRIC_L2);
  int *pos = (int *)malloc(sizeof(int) * nparts);
  for (int q = 0; q < nq; q++) {
    for (int p = 0; p < nparts; p++) pos[p] = 0;
    for (int o = 0; o < k; o++) {
      int best = -1;
      float bv = 0;
      for (int p = 0; p < nparts; p++) {
        while (pos[p] < k && ids[((size_t)p * nq + q) * k + pos[p]] < 0) pos[p] = k;
        if (pos[p] >= k) continue;
        float v = dis[((size_t)p * nq + q) * k + pos[p]];
        if (best < 0 || (asc ? (v <= bv) : (v >= bv))) {
          best = p;
          bv = v;
        }
      }
      if (best < 0) {
        out_dis[(size_t)q * k + o] = asc ? FLT_MAX : -FLT_MAX;
        out_ids[(size_t)q * k + o] = -1;
      } else {
        out_dis[(size_t)q * k + o] = bv;
        out_ids[(size_t)q * k + o] = ((int64_t)best << 32) | ids[((size_t)best * nq + q) * k + pos[best]];
        pos[best]++;
      }
    }
  }
  free(pos);
  return 0;
}

int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
