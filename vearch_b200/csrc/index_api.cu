// extern "C" surface of include/gamma_b200_index.h.
#include <strings.h>

#include <algorithm>
#include <vector>

#include "../../include/gamma_b200_index.h"
#include "common.cuh"
#include "index.h"
#include "json.h"
#include "params.h"

using namespace gb;

struct gb_index {
  Index* impl;
  bool view = false;  // a shard of a sharded index (gb_index_shard): destroying the handle leaves the index alone
};

namespace gb {

// IVFFlatModelParams::Parse / IVFPQModelParams::Parse (gamma_index_ivfflat.cc:64-196,
// gamma_index_ivfpq.h:1031-1257)
// VearchModelParams::Parse (gamma_index_vearch.cc:40-126): ncentroids and nsubvector are required, ns_threshold < 0 means
// no noise shaping, metric_type defaults to InnerProduct; thread_num has no effect here
static bool parse_vearch_params(const std::string& text, ModelParams* mp, std::string* err) {
  JsonValue jv;
  if (!JsonParser::parse(text, &jv) || jv.type != JsonValue::Object) {
    *err = "parse vearch retrieval parameters error: " + text;
    return false;
  }
  int v;
  mp->ncentroids = VearchIndex::kDefaultNlist;
  mp->nsubvector = VearchIndex::kDefaultNsub;
  mp->metric = kMetricIP;
  const char* required[2] = {"ncentroids", "nsubvector"};
  int* target[2] = {&mp->ncentroids, &mp->nsubvector};
  for (int i = 0; i < 2; i++) {
    if (!jv.get_int(required[i], &v)) {
      *err = std::string("cannot get ") + required[i] + " for vearch, set it when create space";
      return false;
    }
    if (v < -1) {
      *err = std::string("invalid ") + required[i] + " =" + std::to_string(v);
      return false;
    }
    if (v > 0) *target[i] = v;
  }
  mp->has_ncentroids = true;
  mp->ncentroids_arg = mp->ncentroids;
  double t;
  if (jv.get_double("ns_threshold", &t)) mp->ns_threshold = t;
  std::string mt;
  if (jv.get_string("metric_type", &mt)) {
    if (strcasecmp("L2", mt.c_str()) && strcasecmp("InnerProduct", mt.c_str())) {
      *err = "invalid metric_type = " + mt;
      return false;
    }
    mp->metric = !strcasecmp("L2", mt.c_str()) ? kMetricL2 : kMetricIP;
  }
  bool b;
  if (jv.get_bool("reordering", &b)) mp->reordering = b;
  // this engine's own keys, as for every type
  if (jv.get_int("training_threshold", &v) && v > 0) mp->training_threshold = v;
  std::string stt;
  if (jv.get_string("store_type", &stt)) mp->host_store = !strcasecmp("RocksDB", stt.c_str());
  return true;
}

bool parse_model_params(const std::string& text, const std::string& type, ModelParams* mp, std::string* err) {
  if (type == "VEARCH") return parse_vearch_params(text, mp, err);
  if (text.empty()) return true;
  const bool gpu = is_gpu_index_type(type);
  JsonValue jv;
  if (!JsonParser::parse(text, &jv) || jv.type != JsonValue::Object) {
    // IVFPQGPUModelParams::Parse / IVFFlatGPUModelParams::Parse (gamma_index_ivfpq_gpu.cc:63-69, ivfflat_gpu.h:67-73)
    *err = type == "GPU_IVFPQ"     ? "failed to parse IVFPQ retrieval parameters"
           : type == "GPU_IVFFLAT" ? "Parse model parameters error"
                                   : "parse model parameters error: " + text;
    return false;
  }
  int v;
  if (jv.get("ncentroids")) {
    if (!jv.get_int("ncentroids", &v)) {
      *err = "parse ncentroids error";
      return false;
    }
    if (v > 0) mp->ncentroids = v;
    mp->ncentroids_arg = v;
    mp->has_ncentroids = true;
  }
  if (jv.get_int("nprobe", &v)) {
    mp->has_nprobe = true;
    mp->nprobe_arg = v;
    if (v < -1 && !gpu) {
      *err = "invalid nprobe =" + std::to_string(v);
      return false;
    }
    if (v > 0) mp->nprobe = v;
    if (mp->nprobe > mp->ncentroids && !gpu) {
      *err = "nprobe should less than ncentroids";
      return false;
    }
  }
  if (jv.get_int("nsubvector", &v)) {
    mp->has_nsubvector = true;
    mp->nsubvector_arg = v;
    if (v < -1 && !gpu) {
      *err = "invalid nsubvector =" + std::to_string(v);
      return false;
    }
    if (v > 0) mp->nsubvector = v;
  }
  if (const JsonValue* opq = jv.get("opq")) {  // gamma_index_ivfpq.h:1202-1216
    mp->has_opq = opq->type == JsonValue::Object;
    if (opq->type == JsonValue::Object && opq->get_int("nsubvector", &v)) {
      if (v < -1) {
        *err = "invalid opq_nsubvector = " + std::to_string(v);
        return false;
      }
      if (v > 0) mp->opq_nsubvector = v;
    }
  }
  if (jv.get_int("nbits_per_idx", &v)) {
    mp->has_nbits = true;
    mp->nbits_arg = v;
    if (v < -1 && !gpu) {
      *err = "invalid nbits_per_idx =" + std::to_string(v);
      return false;
    }
    if (v > 0) mp->nbits = v;
  }
  if (jv.get_int("bucket_init_size", &v)) {
    mp->bucket_init_arg = v;
    if (v < -1 && !gpu) {
      *err = "invalid bucket_init_size =" + std::to_string(v);
      return false;
    }
    if (v > 0) mp->bucket_init_size = v;
  }
  if (jv.get_int("bucket_max_size", &v)) {
    mp->bucket_max_arg = v;
    if (v < -1 && !gpu) {
      *err = "invalid bucket_max_size =" + std::to_string(v);
      return false;
    }
    if (v > 0) mp->bucket_max_size = v;
  }
  // IVFPQFastScan only (validated by create_index): the reference's bbs-blocked list layout never leaves its process, so
  // the block size has no effect here beyond being checked
  if (jv.get_int("bbs", &v)) mp->bbs = v;
  // IVFRABITQ only (validated by create_index, gamma_index_ivfrabitq.h:392-410)
  if (jv.get_int("nb_bits", &v)) mp->nb_bits = v;
  if (jv.get_int("qb", &v)) mp->qb = v;
  if (jv.get_int("training_threshold", &v) && v > 0) mp->training_threshold = v;
  // placement of the raw vectors (VectorManager::DetermineVectorStorageType, vector_manager.cc:50-89): "RocksDB" keeps
  // them out of HBM, in pinned host memory; every other value, and none, keeps them in HBM
  std::string stt;
  if (jv.get_string("store_type", &stt)) mp->host_store = !strcasecmp("RocksDB", stt.c_str());
  std::string mt;
  if (jv.get_string("metric_type", &mt)) {
    if (strcasecmp("L2", mt.c_str()) && strcasecmp("InnerProduct", mt.c_str())) {
      if (gpu) {  // GPU_IVFPQ refuses it in create_index; GPU_IVFFLAT ignores it and keeps InnerProduct
        mp->metric_unknown = mt;
        return true;
      }
      *err = "invalid metric_type = " + mt;
      return false;
    }
    mp->metric = !strcasecmp("L2", mt.c_str()) ? kMetricL2 : kMetricIP;
  }
  return true;
}

// GammaIVFPQIndex::Parse / GammaIVFFlatIndex::Parse (gamma_index_ivfpq.cc:233-294,
// gamma_index_ivfflat.cc:293-340): invalid values fall back to the index defaults.
bool parse_retrieval_params(const std::string& text, RetrievalParams* rp, std::string* err) {
  if (text.empty()) return true;
  JsonValue jv;
  if (!JsonParser::parse(text, &jv) || jv.type != JsonValue::Object) {
    *err = "parse retrieval parameters error: " + text;
    return false;
  }
  rp->given = true;
  std::string mt;
  if (jv.get_string("metric_type", &mt)) rp->metric = !strcasecmp("L2", mt.c_str()) ? kMetricL2 : kMetricIP;
  int v;
  if (jv.get_int("recall_num", &v) && v > 0) rp->recall_num = v;
  if (jv.get_int("nprobe", &v) && v > 0) rp->nprobe = v;
  if (jv.get_int("parallel_on_queries", &v)) rp->parallel_on_queries = v != 0;
  // IVFRABITQ (gamma_index_ivfrabitq.cc:215-229): a qb outside [0, 8] falls back to the index's
  if (jv.get_int("qb", &v) && v >= 0 && v <= 8) rp->qb = v;
  bool b;
  if (jv.get_bool("centered", &b)) rp->centered = b;
  return true;
}

}  // namespace gb

static int fill_ctx(SearchContext* ctx, const char* rp_json, int brute_force, const uint8_t* del_bitmap,
                    const uint8_t* filter_bitmap, int64_t bitmap_bits, float min_score, float max_score) {
  std::string err;
  if (!parse_retrieval_params(rp_json ? rp_json : "", &ctx->params, &err)) {
    set_last_error(err);
    return -1;
  }
  ctx->params.brute_force = brute_force != 0;
  ctx->del_bitmap = del_bitmap;
  ctx->filter_bitmap = filter_bitmap;
  ctx->bitmap_bits = bitmap_bits;
  ctx->min_score = min_score;
  ctx->max_score = max_score;
  return 0;
}

#define IDX_OR_FAIL(idx)                 \
  if (!(idx) || !(idx)->impl) {          \
    set_last_error("null index handle"); \
    return -1;                           \
  }

template <class T>
static T* as(gb_index* index) {
  return index && index->impl ? dynamic_cast<T*>(index->impl) : nullptr;
}

// A BINARYIVF index stores and searches packed binary rows: every entry point taking or returning float rows, queries or
// centroids refuses it (the _binary ones serve it)
static bool packed_binary(gb_index* index) {
  if (!as<BinaryIvfIndex>(index)) return false;
  set_last_error("BINARYIVF: rows, queries and centroids are packed binary; use the _binary entry points");
  return true;
}

// A shard handle (gb_index_shard) reads a shard's structures; changing them goes through the sharded index, which keeps
// the shards consistent with each other and with its raw store
static bool shard_view(gb_index* index) {
  if (!index || !index->view) return false;
  set_last_error("a shard handle is read-only: change the sharded index instead");
  return true;
}

// the IVF index whose trained state (centroids, codebook, tables, coarse quantiser) a handle answers for: the index, or
// a sharded index's first shard (every shard holds the same state)
template <class T>
static T* state_of(gb_index* index) {
  if (ShardedIndex* sh = index && index->impl ? dynamic_cast<ShardedIndex*>(index->impl) : nullptr)
    return dynamic_cast<T*>(sh->shard(0));
  return as<T>(index);
}
static ShardedIndex* sharded(gb_index* index) {
  return index && index->impl ? dynamic_cast<ShardedIndex*>(index->impl) : nullptr;
}

extern "C" {

const char* gb_last_error(void) { return last_error(); }

long long gb_launch_count(void) { return launch_count(); }

int gb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

gb_index* gb_index_create(const char* index_type, int dimension, const char* model_params_json, int device) {
  ModelParams mp;
  std::string err;
  if (!parse_model_params(model_params_json ? model_params_json : "", index_type ? index_type : "", &mp, &err)) {
    set_last_error(err);
    return nullptr;
  }
  Index* impl = create_index(index_type ? index_type : "", dimension, mp, device, 20);
  if (!impl) return nullptr;
  gb_index* h = new gb_index;
  h->impl = impl;
  return h;
}

gb_index* gb_index_create_sharded(const char* index_type, int dimension, const char* model_params_json, const int* devices,
                                  int ndevices) {
  if (!devices || ndevices < 1) {
    set_last_error("gb_index_create_sharded: at least one device");
    return nullptr;
  }
  const std::string type = index_type ? index_type : "";
  // one device, or a type that is not sharded: the index lives on the first device, as gb_index_create places it
  if (ndevices == 1 || !is_gpu_index_type(type)) return gb_index_create(index_type, dimension, model_params_json, devices[0]);
  ModelParams mp;
  std::string err;
  if (!parse_model_params(model_params_json ? model_params_json : "", type, &mp, &err)) {
    set_last_error(err);
    return nullptr;
  }
  Index* impl = create_sharded_index(type, dimension, mp, std::vector<int>(devices, devices + ndevices), 20);
  if (!impl) return nullptr;
  gb_index* h = new gb_index;
  h->impl = impl;
  return h;
}

int gb_index_shard_count(gb_index* index) {
  if (!index || !index->impl) return 0;
  ShardedIndex* sh = dynamic_cast<ShardedIndex*>(index->impl);
  return sh ? sh->nshards() : 1;
}

gb_index* gb_index_shard(gb_index* index, int shard) {
  ShardedIndex* sh = index && index->impl ? dynamic_cast<ShardedIndex*>(index->impl) : nullptr;
  if (!sh || shard < 0 || shard >= sh->nshards()) {
    set_last_error("gb_index_shard: not a sharded index, or no such shard");
    return nullptr;
  }
  gb_index* h = new gb_index;
  h->impl = sh->shard(shard);
  h->view = true;
  return h;
}

const char* gb_index_type(gb_index* index) { return index && index->impl ? index->impl->type().c_str() : ""; }

void gb_index_destroy(gb_index* index) {
  if (!index) return;
  if (index->impl && !index->view) {
    cudaSetDevice(index->impl->device());
    delete index->impl;
  }
  delete index;
}

int gb_index_add_vectors(gb_index* index, int64_t n, const float* x) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  return index->impl->add_vectors(x, n);
}
int gb_index_add_vectors_device(gb_index* index, int64_t n, const float* x_dev, int64_t ld) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  return index->impl->add_vectors_device(x_dev, ld, n);
}
int gb_index_update_vector(gb_index* index, int64_t vid, const float* x) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  cudaSetDevice(index->impl->device());
  return index->impl->update_vector(vid, x);  // RawVector update + IndexModel::Update
}
int gb_index_get_vector(gb_index* index, int64_t vid, float* out) {
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  cudaSetDevice(index->impl->device());
  return index->impl->store().get_host(vid, out);
}
int gb_index_get_vectors(gb_index* index, int64_t start, int64_t n, float* out) {
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  cudaSetDevice(index->impl->device());
  return index->impl->store().get_rows_host(start, n, out);
}
int gb_index_train(gb_index* index) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  return index->impl->train();
}
int gb_index_add_pending(gb_index* index, const uint8_t* del_bitmap) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  return index->impl->add_pending(del_bitmap);
}
int64_t gb_index_ntotal(gb_index* index) { return index && index->impl ? index->impl->store().size() : -1; }
int64_t gb_index_indexed_count(gb_index* index) { return index && index->impl ? index->impl->indexed_count() : -1; }
int gb_index_is_trained(gb_index* index) { return index && index->impl ? (int)index->impl->trained() : 0; }
int64_t gb_index_training_threshold(gb_index* index) {
  return index && index->impl ? index->impl->training_threshold() : -1;
}
int64_t gb_index_mem_bytes(gb_index* index, int which) {
  if (!index || !index->impl) return -1;
  if (which == 0) return index->impl->index_mem_bytes();
  return which == 2 ? index->impl->store().host_bytes() : index->impl->store().mem_bytes();
}

int gb_index_search(gb_index* index, int nq, const float* x, int k, const char* retrieval_params_json, int brute_force,
                    const uint8_t* del_bitmap, const uint8_t* filter_bitmap, int64_t bitmap_bits, float min_score,
                    float max_score, float* out_scores, int64_t* out_ids) {
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  SearchContext ctx;
  if (fill_ctx(&ctx, retrieval_params_json, brute_force, del_bitmap, filter_bitmap, bitmap_bits, min_score, max_score))
    return -1;
  return index->impl->search(ctx, nq, x, k, out_scores, out_ids);
}

int gb_index_search_device(gb_index* index, int nq, const float* x_dev, int64_t ld, int k,
                           const char* retrieval_params_json, int brute_force, float* out_scores_dev,
                           int64_t* out_ids_dev, void* stream) {
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  SearchContext ctx;
  if (fill_ctx(&ctx, retrieval_params_json, brute_force, nullptr, nullptr, 0, -3.4028235e38f, 3.4028235e38f)) return -1;
  return index->impl->search_device(ctx, nq, x_dev, ld, k, out_scores_dev, out_ids_dev,
                                    static_cast<cudaStream_t>(stream));
}

int gb_index_search_device_filtered(gb_index* index, int nq, const float* x_dev, int64_t ld, int k,
                                    const char* retrieval_params_json, int brute_force, const uint8_t* del_bits_dev,
                                    const uint8_t* filter_bits_dev, int64_t bitmap_bits, float min_score,
                                    float max_score, float* out_scores_dev, int64_t* out_ids_dev, void* stream) {
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  if (bitmap_bits < 0) {
    set_last_error("bitmap_bits must not be negative");
    return -1;
  }
  SearchContext ctx;
  if (fill_ctx(&ctx, retrieval_params_json, brute_force, nullptr, nullptr, bitmap_bits, min_score, max_score)) return -1;
  // byte bitmaps of any alignment: search_device copies them into word-aligned, padded scratch on `stream`
  ctx.del_bits_dev = reinterpret_cast<const uint32_t*>(del_bits_dev);
  ctx.filter_bits_dev = reinterpret_cast<const uint32_t*>(filter_bits_dev);
  ctx.bits_dev_words = 0;
  return index->impl->search_device(ctx, nq, x_dev, ld, k, out_scores_dev, out_ids_dev,
                                    static_cast<cudaStream_t>(stream));
}

int gb_index_search_device_keys(gb_index* index, int nq, const float* x_dev, int64_t ld, int k,
                                const char* retrieval_params_json, int brute_force, unsigned long long* out_keys_dev,
                                float* out_scores_dev, int64_t* out_ids_dev, void* stream) {
  IDX_OR_FAIL(index);
  if (packed_binary(index)) return -1;
  SearchContext ctx;
  if (fill_ctx(&ctx, retrieval_params_json, brute_force, nullptr, nullptr, 0, -3.4028235e38f, 3.4028235e38f)) return -1;
  return index->impl->search_device(ctx, nq, x_dev, ld, k, out_scores_dev, out_ids_dev, static_cast<cudaStream_t>(stream),
                                    out_keys_dev);
}

// {"stage": ms, ...} of the searches run since the last call while scan timing was on (malloc'd, caller frees)
int gb_index_stage_times(gb_index* index, char** json_out, int* out_len) {
  IDX_OR_FAIL(index);
  std::string js = "{";
  bool first = true;
  for (auto& kv : index->impl->stage_times()) {
    char buf[64];
    snprintf(buf, sizeof(buf), "%.6f", kv.second);
    js += std::string(first ? "" : ", ") + "\"" + kv.first + "\": " + buf;
    first = false;
  }
  js += "}";
  char* p = static_cast<char*>(malloc(js.size() + 1));
  if (!p) return -1;
  memcpy(p, js.c_str(), js.size() + 1);
  *json_out = p;
  *out_len = (int)js.size();
  return 0;
}

void gb_index_set_rerank_stats(gb_index* index, int on) {
  if (index && index->impl) index->impl->set_rerank_stats(on != 0);
}
int gb_index_rerank_survivors(gb_index* index, int** out, int64_t* n) {
  IDX_OR_FAIL(index);
  const std::vector<int> v = index->impl->take_rerank_survivors();
  int* p = static_cast<int*>(malloc(std::max<size_t>(1, v.size()) * sizeof(int)));
  if (!p) return -1;
  if (!v.empty()) memcpy(p, v.data(), v.size() * sizeof(int));
  *out = p;
  *n = (int64_t)v.size();
  return 0;
}

void gb_index_set_scan_timing(gb_index* index, int on) {
  if (index && index->impl) index->impl->set_time_scan(on != 0);
}
const char* gb_index_last_scan_kernel(gb_index* index) {
  return index && index->impl ? index->impl->last_scan_kernel() : "";
}
const char* gb_index_last_scan_info(gb_index* index) { return index && index->impl ? index->impl->last_scan_info() : "{}"; }
float gb_index_last_scan_ms(gb_index* index) { return index && index->impl ? index->impl->last_scan_ms() : 0.f; }

#define AS_OR_FAIL(T, v, index, what)          \
  T* v = as<T>(index);                         \
  if (!v) {                                    \
    set_last_error("not an " what " index");   \
    return -1;                                 \
  }
#define IVF_OR_FAIL(v, index) AS_OR_FAIL(IvfIndex, v, index, "IVF")
#define STATE_OR_FAIL(T, v, index, what)      \
  T* v = state_of<T>(index);                   \
  if (!v) {                                    \
    set_last_error("not an " what " index");   \
    return -1;                                 \
  }
#define PQ_OR_FAIL(v, index) AS_OR_FAIL(IvfPqBase, v, index, "IVFPQ")

int gb_index_nlist(gb_index* index) {
  STATE_OR_FAIL(IvfIndex, ivf, index, "IVF");
  return ivf->nlist();
}
int gb_index_set_centroids(gb_index* index, const float* centroids, int nlist) {
  if (shard_view(index)) return -1;
  IVF_OR_FAIL(ivf, index);
  if (packed_binary(index)) return -1;
  return ivf->set_centroids(centroids, nlist);
}
int gb_index_get_centroids(gb_index* index, float* centroids) {
  STATE_OR_FAIL(IvfIndex, ivf, index, "IVF");
  if (packed_binary(index)) return -1;
  return ivf->get_centroids(centroids);
}
int gb_index_pq_m(gb_index* index) {
  STATE_OR_FAIL(IvfPqBase, pq, index, "IVFPQ");
  return pq->M();
}
int gb_index_pq_ksub(gb_index* index) {
  STATE_OR_FAIL(IvfPqBase, pq, index, "IVFPQ");
  return pq->ksub();
}
int gb_index_set_pq_centroids(gb_index* index, const float* pqc) {
  if (shard_view(index)) return -1;
  PQ_OR_FAIL(pq, index);
  return pq->set_pq_centroids(pqc);
}
int gb_index_get_pq_centroids(gb_index* index, float* pqc) {
  STATE_OR_FAIL(IvfPqBase, pq, index, "IVFPQ");
  return pq->get_pq_centroids(pqc);
}
int gb_index_pqfs_lut(gb_index* index, int nq, const float* x, int metric, uint8_t* lut8, float* ab) {
  AS_OR_FAIL(IVFPQFastScanIndex, fs, index, "IVFPQFastScan");
  return fs->lut_host(nq, x, metric, lut8, ab);
}
int gb_index_get_precomputed_table(gb_index* index, float* table) {
  STATE_OR_FAIL(IVFPQIndex, pq, index, "IVFPQ");
  return pq->get_precomputed_table(table);
}
int gb_index_has_opq(gb_index* index) {
  IVFPQIndex* pq = state_of<IVFPQIndex>(index);
  return pq && pq->has_opq() ? 1 : 0;
}
int gb_index_set_opq(gb_index* index, const float* A) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  IVFPQIndex* pq = as<IVFPQIndex>(index);
  return pq ? pq->set_opq(A) : -1;
}
int gb_index_get_opq(gb_index* index, float* A) {
  IDX_OR_FAIL(index);
  IVFPQIndex* pq = state_of<IVFPQIndex>(index);
  return pq ? pq->get_opq(A) : -1;
}
int gb_index_apply_opq(gb_index* index, int64_t n, const float* x, float* out) {
  IDX_OR_FAIL(index);
  IVFPQIndex* pq = as<IVFPQIndex>(index);
  return pq ? pq->apply_opq_host(x, n, out) : -1;
}
int gb_index_mirror_builds(gb_index* index) {
  if (!index || !index->impl) return -1;
  IVFFlatIndex* ivf = as<IVFFlatIndex>(index);
  return ivf ? ivf->mirror_builds() : 0;
}
int gb_index_get_list_shifts(gb_index* index, float* out) {
  STATE_OR_FAIL(IVFFlatIndex, ivf, index, "IVFFLAT");
  return ivf->get_list_shifts(out);
}
const char* gb_index_last_coarse_kernel(gb_index* index) {
  IvfIndex* ivf = state_of<IvfIndex>(index);
  return ivf ? ivf->last_coarse_kernel() : "";
}
int gb_index_compact(gb_index* index) {
  IDX_OR_FAIL(index);
  if (shard_view(index)) return -1;
  if (ShardedIndex* sh = sharded(index)) {  // every shard's lists
    for (int s = 0; s < sh->nshards(); s++)
      if (sh->shard(s)->compact_lists()) return -1;
    cudaSetDevice(sh->device());
    return 0;
  }
  IvfIndex* ivf = as<IvfIndex>(index);
  return ivf ? ivf->compact_lists() : 0;
}
int gb_index_dump(gb_index* index, const char* dir, const char* abs_name) {
  IDX_OR_FAIL(index);
  if (!dir || !abs_name) return -1;
  cudaSetDevice(index->impl->device());
  return index->impl->dump_gamma(dir, abs_name);
}
int gb_index_load(gb_index* index, const char* dir, const char* abs_name, int64_t* load_num) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  if (!dir || !abs_name || !load_num) return -1;
  cudaSetDevice(index->impl->device());
  return index->impl->load_gamma(dir, abs_name, load_num);
}
static int gb_index_list_len_of(IvfIndex* ivf, int list) {
  if (!ivf->lists() || list < 0 || list >= ivf->nlist()) return 0;
  return ivf->lists()->lens()[list];
}
int gb_index_list_len(gb_index* index, int list) {
  if (ShardedIndex* sh = sharded(index)) {  // the list's entries over every shard
    int n = 0;
    for (int s = 0; s < sh->nshards(); s++) n += gb_index_list_len_of(sh->shard(s), list);
    return n;
  }
  IVF_OR_FAIL(ivf, index);
  if (!ivf->lists() || list < 0 || list >= ivf->nlist()) return 0;
  return ivf->lists()->lens()[list];
}
int gb_index_code_size(gb_index* index) {
  STATE_OR_FAIL(IvfIndex, ivf, index, "IVF");
  return ivf->code_bytes();
}
int gb_index_get_list(gb_index* index, int list, uint8_t* codes, int64_t* ids) {
  IVF_OR_FAIL(ivf, index);
  if (!ivf->lists()) return -1;
  cudaSetDevice(ivf->device());
  std::vector<uint8_t> c;
  std::vector<int64_t> i;
  if (ivf->lists()->download_list(list, &c, &i)) return -1;
  if (codes && !c.empty()) memcpy(codes, c.data(), c.size());
  if (ids && !i.empty()) memcpy(ids, i.data(), i.size() * 8);
  return 0;
}
int gb_index_tombstone(gb_index* index, int list, int pos) {
  if (shard_view(index)) return -1;
  IVF_OR_FAIL(ivf, index);
  if (!ivf->lists()) return -1;
  cudaSetDevice(ivf->device());
  return ivf->lists()->tombstone(list, pos, nullptr);
}
int gb_index_delete(gb_index* index, const int64_t* vids, int64_t n) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  if (n < 0 || (n > 0 && !vids)) return -1;
  return index->impl->delete_vectors(vids, n);
}
int gb_index_purge(gb_index* index, float threshold, const uint8_t* del_bitmap, int64_t bitmap_bytes, int64_t* dropped) {
  if (shard_view(index)) return -1;
  IDX_OR_FAIL(index);
  if (!(threshold >= 0.f) || bitmap_bytes < 0) {
    set_last_error("purge: threshold must be >= 0 and bitmap_bytes >= 0");
    return -1;
  }
  return index->impl->purge_lists(threshold, del_bitmap, bitmap_bytes, dropped);
}
int gb_index_dead_counts(gb_index* index, int* out) {
  if (!out) return -1;
  if (ShardedIndex* sh = sharded(index)) {  // per list, summed over the shards
    std::vector<int> part(sh->shard(0)->nlist());
    for (int l = 0; l < (int)part.size(); l++) out[l] = 0;
    for (int s = 0; s < sh->nshards(); s++) {
      if (sh->shard(s)->dead_counts(part.data())) return -1;
      for (int l = 0; l < (int)part.size(); l++) out[l] += part[l];
    }
    return 0;
  }
  IVF_OR_FAIL(ivf, index);
  return ivf->dead_counts(out);
}
int gb_index_coarse_search(gb_index* index, int nq, const float* x, int nprobe, float* out_dis, int64_t* out_ids) {
  STATE_OR_FAIL(IvfIndex, ivf, index, "IVF");
  if (packed_binary(index)) return -1;
  return ivf->coarse_search_host(nq, x, nprobe, out_dis, out_ids);
}
int gb_index_search_preassigned(gb_index* index, int nq, const float* x, int k, const int64_t* keys,
                                const float* coarse_dis, int nprobe, const char* retrieval_params_json,
                                const uint8_t* del_bitmap, const uint8_t* filter_bitmap, int64_t bitmap_bits,
                                float min_score, float max_score, float* out_scores, int64_t* out_ids) {
  IVF_OR_FAIL(ivf, index);
  if (packed_binary(index)) return -1;
  SearchContext ctx;
  if (fill_ctx(&ctx, retrieval_params_json, 0, del_bitmap, filter_bitmap, bitmap_bits, min_score, max_score)) return -1;
  return ivf->search_preassigned_host(ctx, nq, x, k, keys, coarse_dis, nprobe, out_scores, out_ids);
}
int gb_index_pq_encode(gb_index* index, int64_t n, const float* x, const int64_t* assign, uint8_t* codes) {
  PQ_OR_FAIL(pq, index);
  return pq->encode_host(x, n, assign, codes);
}

#define BIN_OR_FAIL(v, index) AS_OR_FAIL(BinaryIvfIndex, v, index, "BINARYIVF")
int gb_index_add_binary(gb_index* index, int64_t n, const uint8_t* x) {
  BIN_OR_FAIL(b, index);
  return b->add_vectors(x, n);
}
int gb_index_update_binary(gb_index* index, int64_t vid, const uint8_t* x) {
  BIN_OR_FAIL(b, index);
  cudaSetDevice(b->device());
  return b->update_vector(vid, x);
}
int gb_index_get_binary(gb_index* index, int64_t start, int64_t n, uint8_t* out) {
  BIN_OR_FAIL(b, index);
  cudaSetDevice(b->device());
  return b->store().get_rows_host(start, n, out);
}
int gb_index_search_binary(gb_index* index, int nq, const uint8_t* x, int k, const char* retrieval_params_json,
                           int brute_force, const uint8_t* del_bitmap, const uint8_t* filter_bitmap, int64_t bitmap_bits,
                           float min_score, float max_score, int search_unindexed_tail, float* out_scores, int64_t* out_ids) {
  BIN_OR_FAIL(b, index);
  SearchContext ctx;
  if (fill_ctx(&ctx, retrieval_params_json, brute_force, del_bitmap, filter_bitmap, bitmap_bits, min_score, max_score))
    return -1;
  ctx.search_unindexed_tail = search_unindexed_tail != 0;
  return b->search(ctx, nq, x, k, out_scores, out_ids);
}
int gb_index_set_binary_centroids(gb_index* index, const uint8_t* centroids, int nlist) {
  BIN_OR_FAIL(b, index);
  return b->set_binary_centroids(centroids, nlist);
}
int gb_index_get_binary_centroids(gb_index* index, uint8_t* centroids) {
  BIN_OR_FAIL(b, index);
  return b->get_binary_centroids(centroids);
}
int gb_index_get_real_centroids(gb_index* index, float* centroids) {
  BIN_OR_FAIL(b, index);
  return b->get_centroids(centroids);
}
int gb_index_coarse_search_binary(gb_index* index, int nq, const uint8_t* x, int nprobe, float* out_dis, int64_t* out_ids) {
  BIN_OR_FAIL(b, index);
  return b->coarse_search_host(nq, x, nprobe, out_dis, out_ids);
}
int gb_index_search_preassigned_binary(gb_index* index, int nq, const uint8_t* x, int k, const int64_t* keys, int nprobe,
                                       const uint8_t* del_bitmap, const uint8_t* filter_bitmap, int64_t bitmap_bits,
                                       float min_score, float max_score, float* out_scores, int64_t* out_ids) {
  BIN_OR_FAIL(b, index);
  SearchContext ctx;
  if (fill_ctx(&ctx, "", 0, del_bitmap, filter_bitmap, bitmap_bits, min_score, max_score)) return -1;
  return b->search_preassigned_host(ctx, nq, x, k, keys, nullptr, nprobe, out_scores, out_ids);
}

#define RQ_OR_FAIL(v, index) AS_OR_FAIL(RaBitQIndex, v, index, "IVFRABITQ")
int gb_index_rabitq_nb_bits(gb_index* index) {
  RQ_OR_FAIL(rq, index);
  return rq->nb_bits();
}
int gb_index_rabitq_qb(gb_index* index) {
  RQ_OR_FAIL(rq, index);
  return rq->qb();
}
int gb_index_rabitq_encode(gb_index* index, int64_t n, const float* x, const int64_t* assign, uint8_t* codes) {
  RQ_OR_FAIL(rq, index);
  return rq->encode_host(x, n, assign, codes);
}
int gb_index_rabitq_estimate(gb_index* index, int nq, const float* x, const int64_t* lists, int qb, int metric, float* out) {
  RQ_OR_FAIL(rq, index);
  return rq->estimate_host(nq, x, lists, qb, metric >= 0 ? metric : rq->metric(), out);
}

#define VR_OR_FAIL(v, index) AS_OR_FAIL(VearchIndex, v, index, "VEARCH")
int gb_index_vearch_nsub(gb_index* index) {
  VR_OR_FAIL(vr, index);
  return vr->nsub();
}
int gb_index_vearch_blocks(gb_index* index) {
  VR_OR_FAIL(vr, index);
  return vr->nblocks();
}
int gb_index_vearch_set_codebook(gb_index* index, const float* codebook) {
  VR_OR_FAIL(vr, index);
  return vr->set_codebook(codebook);
}
int gb_index_vearch_get_codebook(gb_index* index, float* codebook) {
  VR_OR_FAIL(vr, index);
  return vr->get_codebook(codebook);
}
int gb_index_vearch_encode(gb_index* index, int64_t n, const float* x, const int64_t* assign, uint8_t* codes) {
  VR_OR_FAIL(vr, index);
  return vr->encode_host(x, n, assign, codes);
}
int gb_index_vearch_lut(gb_index* index, int nq, const float* x, uint8_t* lut, float* mult) {
  VR_OR_FAIL(vr, index);
  return vr->lut_host(nq, x, lut, mult);
}

}  // extern "C"

// kmeans_device on host rows: gb_kmeans and its trace.  init: nullptr, or k x d starting centroids (hot start)
static int kmeans_host(int device, const float* x, int64_t n, int d, int k, KMeansParams kp, const float* init,
                       float* centroids, std::vector<float>* obj, KMeansTrace* trace) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_last_error("no CUDA device");
    return -1;
  }
  cudaStream_t st;
  GB_CUDA(cudaStreamCreate(&st));
  int rc = -1;
  {
    Scratch s(st);
    const int dpad = (d + 3) / 4 * 4;
    float* dx = s.alloc_n<float>((size_t)n * dpad);
    float* dc = s.alloc_n<float>((size_t)k * dpad);
    if (dx && dc && cudaMemsetAsync(dc, 0, (size_t)k * dpad * 4, st) == cudaSuccess &&
        upload_rows_padded(dx, x, n, d, dpad, st) == cudaSuccess &&
        (!init || cudaMemcpy2DAsync(dc, (size_t)dpad * 4, init, (size_t)d * 4, (size_t)d * 4, k, cudaMemcpyHostToDevice,
                                    st) == cudaSuccess)) {
      kp.hot_start = init != nullptr;
      rc = kmeans_device(dx, dpad, n, d, k, kp, dc, dpad, st, obj, trace);
      if (rc == 0 && (cudaMemcpy2DAsync(centroids, (size_t)d * 4, dc, (size_t)dpad * 4, (size_t)d * 4, k,
                                        cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                      cudaStreamSynchronize(st) != cudaSuccess))
        rc = -1;
    }
  }
  cudaStreamSynchronize(st);
  cudaStreamDestroy(st);
  return rc;
}

extern "C" {

int gb_kmeans(int device, const float* x, int64_t n, int d, int k, int niter, int64_t seed, int spherical,
              int max_points_per_centroid, float* centroids, float* obj) {
  KMeansParams kp;
  kp.niter = niter;
  kp.seed = seed;
  kp.spherical = spherical != 0;
  kp.max_points_per_centroid = max_points_per_centroid;
  std::vector<float> o;
  const int rc = kmeans_host(device, x, n, d, k, kp, nullptr, centroids, obj ? &o : nullptr, nullptr);
  if (rc == 0 && obj)
    for (size_t i = 0; i < o.size(); i++) obj[i] = o[i];
  return rc;
}

int gb_debug_kmeans_trace(int device, const float* x, int64_t n, int d, int k, int niter, int64_t seed, int spherical,
                          int l2_assign, int max_points_per_centroid, const float* init, int64_t* sample,
                          float* init_out, int32_t* labels, float* scores, float* mean, float* split, float* norm) {
  KMeansParams kp;
  kp.niter = niter;
  kp.seed = seed;
  kp.spherical = spherical != 0;
  kp.l2_assign = l2_assign != 0;
  kp.max_points_per_centroid = max_points_per_centroid;
  KMeansTrace t;
  std::vector<float> cent((size_t)k * d);
  if (kmeans_host(device, x, n, d, k, kp, init, cent.data(), nullptr, &t)) return -1;
  const int64_t ns = t.sample.empty() ? n : (int64_t)t.sample.size();
  for (int64_t i = 0; i < ns; i++) sample[i] = t.sample.empty() ? i : t.sample[i];
  std::copy(t.init.begin(), t.init.end(), init_out);
  std::copy(t.labels.begin(), t.labels.end(), labels);
  std::copy(t.scores.begin(), t.scores.end(), scores);
  std::copy(t.mean.begin(), t.mean.end(), mean);
  std::copy(t.split.begin(), t.split.end(), split);
  std::copy(t.norm.begin(), t.norm.end(), norm);
  return 0;
}

int gb_kmeans_update(int device, const float* x, int64_t n, int d, int k, const int64_t* assign, float* centroids) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_last_error("no CUDA device");
    return -1;
  }
  cudaStream_t st = nullptr;
  Scratch s(st);
  const int dpad = (d + 3) / 4 * 4;
  float* dx = s.alloc_n<float>((size_t)n * dpad);
  float* dc = s.alloc_n<float>((size_t)k * dpad);
  int32_t* dperm = s.alloc_n<int32_t>(n);
  int32_t* doff = s.alloc_n<int32_t>(k + 1);
  if (!dx || !dc || !dperm || !doff) return -1;
  std::vector<int32_t> off(k + 1, 0), perm(n), cur(k);
  for (int64_t i = 0; i < n; i++) off[assign[i] + 1]++;
  for (int c = 0; c < k; c++) {
    off[c + 1] += off[c];
    cur[c] = off[c];
  }
  for (int64_t i = 0; i < n; i++) perm[cur[assign[i]]++] = (int32_t)i;
  GB_CUDA(upload_rows_padded(dx, x, n, d, dpad, st));
  GB_CUDA(cudaMemcpyAsync(dperm, perm.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(doff, off.data(), (size_t)(k + 1) * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(launch_segment_mean(dx, dpad, d, dperm, doff, k, dc, dpad, st));
  GB_CUDA(cudaMemcpy2DAsync(centroids, (size_t)d * 4, dc, (size_t)dpad * 4, (size_t)d * 4, k, cudaMemcpyDeviceToHost,
                            st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int gb_debug_dist_matrix(int device, const float* x, int n, const float* c, int m, int d, int metric, int use_tc,
                         float* out) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_last_error("no CUDA device");
    return -1;
  }
  cudaStream_t st = nullptr;
  Scratch s(st);
  const int dpad = (d + 3) / 4 * 4;
  const int64_t ldo = (m + 3) / 4 * 4;
  float* dx = s.alloc_n<float>((size_t)n * dpad);
  float* dc = s.alloc_n<float>((size_t)m * dpad);
  float* dout = s.alloc_n<float>((size_t)n * ldo);
  if (!dx || !dc || !dout) return -1;
  GB_CUDA(upload_rows_padded(dx, x, n, d, dpad, st));
  GB_CUDA(upload_rows_padded(dc, c, m, d, dpad, st));
  if (use_tc) {
    GB_CUDA(launch_dist_matrix_tc(dx, dpad, n, dc, dpad, m, dpad, metric, dout, ldo, st));
  } else {
    GB_CUDA(launch_dist_matrix(dx, dpad, n, dc, dpad, m, dpad, metric, dout, ldo, st));
  }
  GB_CUDA(cudaMemcpy2DAsync(out, (size_t)m * 4, dout, (size_t)ldo * 4, (size_t)m * 4, n, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int gb_device_pool_usage(int device, int reset_peak, int64_t* used, int64_t* peak) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_last_error("no CUDA device");
    return -1;
  }
  cudaMemPool_t pool;
  uint64_t u = 0, h = 0;
  GB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
  GB_CUDA(cudaDeviceSynchronize());  // stream-ordered frees of finished searches are returned to the pool
  GB_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &u));
  GB_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &h));
  if (used) *used = (int64_t)u;
  if (peak) *peak = (int64_t)h;
  if (reset_peak) {
    uint64_t zero = 0;  // the only value accepted: the high-water mark restarts at the current use
    GB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &zero));
  }
  return 0;
}

int gb_merge_partitions_device(int device, const float* dis_dev, const int64_t* ids_dev, int nparts, int nq, int k,
                               int metric, float* out_dis_dev, int64_t* out_ids_dev, void* stream) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_last_error("no CUDA device");
    return -1;
  }
  return merge_partitions_device(dis_dev, ids_dev, nparts, nq, k, metric, out_dis_dev, out_ids_dev,
                                 static_cast<cudaStream_t>(stream));
}

int gb_merge_partition_keys_device(int device, const unsigned long long* keys_dev, int nparts, int nq, int k, int metric,
                                   float* out_dis_dev, int64_t* out_ids_dev, void* stream) {
  if (cudaSetDevice(device) != cudaSuccess) {
    set_last_error("no CUDA device");
    return -1;
  }
  return merge_partition_keys_device(keys_dev, nparts, nq, k, metric, out_dis_dev, out_ids_dev,
                                     static_cast<cudaStream_t>(stream));
}

}  // extern "C"
