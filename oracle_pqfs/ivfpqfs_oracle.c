/* CPU restatement of the IVFPQFastScan index (TEST INFRASTRUCTURE ONLY): faiss IndexIVFPQFastScan with
 * by_residual = false, as gamma's index/impl/gamma_index_ivfpqfs.cc builds it.  Restated from upstream faiss v1.14.1
 * (ProductQuantizer::compute_codes, BitstringWriter, quantize_lut::round_uint8_per_column, the fast-scan
 * accumulation of IndexIVFFastScan::search); SURVEY.md Appendix A lists the assumptions.
 *
 * Build: see oracle_pqfs/Makefile (gcc -O2 -ffp-contract=off): every a*b+c stays two roundings, and every sum runs
 * sequentially in the order the device kernels use, so the uint8 tables, (a, b), codes and scores are bit-equal to
 * theirs.  PQ training (16-means per sub-quantiser) is oracle/gamma_oracle.c's k-means, called from ivfpqfs.py.
 *
 * Selection uses the engine's total order -- score, then the smaller id -- through a bounded heap of 64-bit keys, and
 * the output follows faiss heap_reorder: L2 ascending (score, id), IP descending score with the larger id first among
 * equal scores.  faiss admits a candidate on its value alone, so which of several candidates tied at the k-th score
 * survive depends on scan order there (DESIGN.md §4 tie rule). */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define KSUB 16
#define METRIC_L2 1

static uint32_t f2ord(float f) {
  uint32_t b;
  memcpy(&b, &f, 4);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
static float ord2f(uint32_t o) {
  uint32_t b = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
  float f;
  memcpy(&f, &b, 4);
  return f;
}
static uint64_t make_key(float s, int metric, uint32_t vid) {
  uint32_t o = metric == METRIC_L2 ? f2ord(s) : ~f2ord(s);
  return ((uint64_t)o << 32) | vid;
}
static float key_score(uint64_t key, int metric) {
  uint32_t o = (uint32_t)(key >> 32);
  return metric == METRIC_L2 ? ord2f(o) : ord2f(~o);
}

/* ---- bounded max-heap of keys: keeps the k smallest ---------------------------------------------------------- */
static void kheap_push(uint64_t *h, int *n, int k, uint64_t key) {
  if (*n == k) {
    if (key >= h[0]) return;
    int i = 0;
    for (;;) {  /* replace the root (the largest kept key), sift down */
      int l = 2 * i + 1, r = l + 1, m = i;
      uint64_t big = key;
      if (l < k && h[l] > big) m = l, big = h[l];
      if (r < k && h[r] > big) m = r, big = h[r];
      if (m == i) break;
      h[i] = h[m];
      i = m;
    }
    h[i] = key;
    return;
  }
  int i = (*n)++;
  h[i] = key;
  while (i > 0 && h[(i - 1) / 2] < h[i]) {
    uint64_t t = h[i];
    h[i] = h[(i - 1) / 2];
    h[(i - 1) / 2] = t;
    i = (i - 1) / 2;
  }
}
static int cmp_u64(const void *a, const void *b) {
  uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
  return x < y ? -1 : x > y;
}
/* sorted keys -> (score, id) in the decoder's order, padded with the heap's neutral value and id -1 */
static void write_out(uint64_t *h, int n, int k, int metric, float *dis, int64_t *ids) {
  qsort(h, (size_t)n, 8, cmp_u64);
  for (int i = 0; i < n; i++) {
    int s = i, e = i + 1;
    if (metric != METRIC_L2) {  /* equal scores: larger id first */
      while (s > 0 && (h[s - 1] >> 32) == (h[i] >> 32)) s--;
      while (e < n && (h[e] >> 32) == (h[i] >> 32)) e++;
    }
    int j = metric != METRIC_L2 ? s + (e - 1 - i) : i;
    dis[j] = key_score(h[i], metric);
    ids[j] = (int64_t)(uint32_t)h[i];
  }
  for (int i = n; i < k; i++) {
    dis[i] = metric == METRIC_L2 ? FLT_MAX : -FLT_MAX;
    ids[i] = -1;
  }
}

/* ---- encode: per sub-vector argmin over 16 centroids (lowest index on ties), two codes per byte ---------------- */
int orcfs_encode(const float *pq, int M, int dsub, const float *x, int64_t n, uint8_t *codes) {
  const int d = M * dsub, mb = (M + 1) / 2;
  for (int64_t i = 0; i < n; i++) {
    uint8_t *out = codes + i * mb;
    memset(out, 0, (size_t)mb);
    for (int m = 0; m < M; m++) {
      const float *xm = x + i * d + (int64_t)m * dsub;
      float best = FLT_MAX;
      int bi = 0;
      for (int c = 0; c < KSUB; c++) {
        const float *cc = pq + ((int64_t)m * KSUB + c) * dsub;
        float dis = 0.f;
        for (int j = 0; j < dsub; j++) {
          float t = xm[j] - cc[j];
          dis = dis + t * t;
        }
        if (dis < best) {
          best = dis;
          bi = c;
        }
      }
      out[m / 2] |= (uint8_t)(bi << (4 * (m & 1)));
    }
  }
  return 0;
}

/* ---- float table and its uint8 quantisation (round_uint8_per_column) ------------------------------------------- */
int orcfs_lut(const float *pq, int M, int dsub, const float *xq, int nq, int metric, uint8_t *lut8, float *ab) {
  const int d = M * dsub;
  float *tab = malloc(sizeof(float) * M * KSUB), *mins = malloc(sizeof(float) * M);
  if (!tab || !mins) return -1;
  for (int q = 0; q < nq; q++) {
    float max_span = 0.f, b = 0.f;
    for (int m = 0; m < M; m++) {
      const float *xm = xq + (int64_t)q * d + (int64_t)m * dsub;
      float mn = FLT_MAX, mx = -FLT_MAX;
      for (int c = 0; c < KSUB; c++) {
        const float *cc = pq + ((int64_t)m * KSUB + c) * dsub;
        float acc = 0.f;
        for (int j = 0; j < dsub; j++) {
          if (metric == METRIC_L2) {
            float t = xm[j] - cc[j];
            acc = acc + t * t;
          } else {
            acc = acc + xm[j] * cc[j];
          }
        }
        tab[m * KSUB + c] = acc;
        if (acc < mn) mn = acc;
        if (acc > mx) mx = acc;
      }
      mins[m] = mn;
      float span = mx - mn;
      if (span > max_span) max_span = span;
    }
    /* every span 0: faiss would divide by zero; a = 1 leaves the table 0 */
    const float a = max_span > 0.f ? 255.f / max_span : 1.f;
    for (int m = 0; m < M; m++) {
      b = b + mins[m];
      for (int c = 0; c < KSUB; c++)
        lut8[((int64_t)q * M + m) * KSUB + c] = (uint8_t)floorf((tab[m * KSUB + c] - mins[m]) * a + 0.5f);
    }
    ab[2 * q] = a;
    ab[2 * q + 1] = b;
  }
  free(tab);
  free(mins);
  return 0;
}

static int bit(const uint8_t *bm, int64_t id) { return (bm[id >> 3] >> (id & 7)) & 1; }

/* ---- search over given probes: keys[q][p] = list (-1 = none).  Tombstones (negative ids), deletion bitmap, filter
 * bitmap and the score window [min_score, max_score] apply to every entry before selection.  recall_num > 0: the
 * max(k, recall_num) best by quantised score are re-ranked by the exact distance to their raw row (raw[vid * ld_raw],
 * summed sequentially over d), the window applied again. -------------------------------------------------------- */
int orcfs_search_preassigned(const int64_t *list_off, const uint8_t *list_codes, const int64_t *list_ids, int nlist,
                             int M, const uint8_t *lut8, const float *ab, const float *xq, int d, int nq, int k,
                             const int64_t *keys, int nprobe, int metric, int recall_num, const float *raw, int64_t ld_raw,
                             const uint8_t *del_bitmap, const uint8_t *filter_bitmap, float min_score, float max_score,
                             float *out_dis, int64_t *out_ids) {
  const int mb = (M + 1) / 2;
  const int kk = recall_num > 0 && recall_num > k ? recall_num : k;
  uint64_t *h = malloc(sizeof(uint64_t) * kk), *h2 = malloc(sizeof(uint64_t) * k);
  if (!h || !h2) return -1;
  for (int q = 0; q < nq; q++) {
    const uint8_t *lq = lut8 + (int64_t)q * M * KSUB;
    const float one_a = 1.f / ab[2 * q], b = ab[2 * q + 1];
    int n = 0;
    for (int p = 0; p < nprobe; p++) {
      int64_t l = keys[(int64_t)q * nprobe + p];
      if (l < 0 || l >= nlist) continue;
      for (int64_t e = list_off[l]; e < list_off[l + 1]; e++) {
        int64_t id = list_ids[e];
        if (id < 0) continue;
        if (del_bitmap && bit(del_bitmap, id)) continue;
        if (filter_bitmap && !bit(filter_bitmap, id)) continue;
        const uint8_t *c = list_codes + e * mb;
        uint32_t accu = 0;
        for (int m = 0; m < M; m++) accu += lq[m * KSUB + ((c[m / 2] >> (4 * (m & 1))) & 15)];
        float s = (float)accu * one_a + b;
        if (s < min_score || s > max_score) continue;
        kheap_push(h, &n, kk, make_key(s, metric, (uint32_t)id));
      }
    }
    if (recall_num <= 0) {
      write_out(h, n, k, metric, out_dis + (int64_t)q * k, out_ids + (int64_t)q * k);
      continue;
    }
    int n2 = 0;
    for (int i = 0; i < n; i++) {
      uint32_t vid = (uint32_t)h[i];
      const float *y = raw + (int64_t)vid * ld_raw, *x = xq + (int64_t)q * d;
      float s = 0.f;
      for (int j = 0; j < d; j++) {
        if (metric == METRIC_L2) {
          float t = y[j] - x[j];
          s = s + t * t;
        } else {
          s = s + y[j] * x[j];
        }
      }
      if (s < min_score || s > max_score) continue;
      kheap_push(h2, &n2, k, make_key(s, metric, vid));
    }
    write_out(h2, n2, k, metric, out_dis + (int64_t)q * k, out_ids + (int64_t)q * k);
  }
  free(h);
  free(h2);
  return 0;
}
