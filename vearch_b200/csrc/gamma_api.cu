// The gamma C-ABI (include/gamma_api.h): the symbols the Go partition server binds through cgo
// (internal/engine/sdk/go/gamma/gamma.go), implemented over gb::Engine.
// Mirrors internal/engine/c_api/gamma_api.cc:35-374; every output buffer is malloc()'d.
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <string>
#include <vector>

#include "../../include/gamma_api.h"
#include "engine.h"
#include "json.h"

using gb::Engine;

static void to_cstatus(const gb::Status& s, struct CStatus* c) {
  c->code = s.code;
  c->msg = nullptr;
  if (s.code != 0) {
    std::string m = s.ToString();
    // the reference allocates with new[] while Go frees with C.free (gamma_api.cc:149 vs
    // gamma.go:47-53); the drop-in must malloc
    c->msg = static_cast<char*>(malloc(m.size() + 1));
    if (c->msg) memcpy(c->msg, m.c_str(), m.size() + 1);
  }
}

static void out_buffer(const std::string& s, char** out, int* len) {
  *len = (int)s.size();
  *out = static_cast<char*>(malloc(s.size() ? s.size() : 1));
  if (*out && !s.empty()) memcpy(*out, s.data(), s.size());
}

static std::atomic<int> g_log_dir_flag{0};

// Init's device list: a JSON array of ordinals or "all", or the environment's "0,1,2,3" / "all" in its place.  false:
// malformed, empty, or an ordinal outside [0, ndev)
static bool parse_devices(const gb::JsonValue* jv, const char* env, int ndev, std::vector<int>* out) {
  out->clear();
  std::string all;
  if (env) {
    all = env;
    if (all != "all") {
      size_t at = 0;
      for (;;) {  // every comma-separated token an integer: "0,", ",1" and "0,,1" are malformed
        const size_t comma = all.find(',', at);
        const std::string tok = all.substr(at, comma == std::string::npos ? std::string::npos : comma - at);
        char* end = nullptr;
        const long v = strtol(tok.c_str(), &end, 10);
        if (tok.empty() || *end) return false;
        out->push_back((int)v);
        if (comma == std::string::npos) break;
        at = comma + 1;
      }
    }
  } else if (jv) {
    if (jv->type == gb::JsonValue::String) {
      if (jv->str != "all") return false;
      all = "all";
    } else if (jv->type == gb::JsonValue::Array && !jv->arr.empty()) {
      for (const gb::JsonValue& v : jv->arr) {
        if (v.type != gb::JsonValue::Number || v.num != (double)(int)v.num) return false;
        out->push_back((int)v.num);
      }
    } else {
      return false;
    }
  }
  if (all == "all")
    for (int d = 0; d < ndev; d++) out->push_back(d);
  for (int d : *out)
    if (d < 0 || d >= ndev) return false;
  return true;
}

extern "C" {

void* Init(const char* config_str, int len) {
  gb::JsonValue j;
  if (!config_str || len <= 0 || !gb::JsonParser::parse(std::string(config_str, (size_t)len), &j) ||
      j.type != gb::JsonValue::Object)
    return nullptr;
  std::string log_dir, path, space = "default";
  int flag = g_log_dir_flag.fetch_add(1);
  if (flag == 0 && !j.get_string("log_dir", &log_dir)) return nullptr;  // mandatory on first call (gamma_api.cc:40-47)
  if (!j.get_string("path", &path)) return nullptr;                     // gamma_api.cc:49-53
  j.get_string("space_name", &space);
  int device = 0;
  j.get_int("device", &device);
  if (const char* env = getenv("GAMMA_B200_DEVICE")) device = atoi(env);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return nullptr;  // no CPU path
  if (device < 0 || device >= ndev) device = ((device % ndev) + ndev) % ndev;
  // "devices": the GPU_IVFPQ / GPU_IVFFLAT fields shard over them (IndexShards), devices[0] is the partition's device;
  // GAMMA_B200_DEVICES ("0,1,2,3" or "all") overrides it as GAMMA_B200_DEVICE overrides "device"
  std::vector<int> devices;
  const char* env_devices = getenv("GAMMA_B200_DEVICES");
  if (env_devices && !*env_devices) env_devices = nullptr;  // set but empty: as if unset
  if (!parse_devices(j.get("devices"), env_devices, ndev, &devices)) return nullptr;
  return static_cast<void*>(new Engine(path, space, device, devices));
}

int Close(void* engine) {
  delete static_cast<Engine*>(engine);
  return 0;
}

struct CStatus CreateTable(void* engine, const char* table_str, int len) {
  struct CStatus c;
  if (!engine) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "null engine"), &c);
    return c;
  }
  to_cstatus(static_cast<Engine*>(engine)->CreateTable(reinterpret_cast<const uint8_t*>(table_str), (size_t)len), &c);
  return c;
}

int AddOrUpdateDoc(void* engine, const char* doc_str, int len) {
  if (!engine) return -1;
  return static_cast<Engine*>(engine)->AddOrUpdate(reinterpret_cast<const uint8_t*>(doc_str), (size_t)len);
}

int DeleteDoc(void* engine, const char* docid, int docid_len) {
  if (!engine) return -1;
  return static_cast<Engine*>(engine)->Delete(std::string(docid, (size_t)docid_len));
}

void GetEngineStatus(void* engine, char** status, int* len) {
  out_buffer(engine ? static_cast<Engine*>(engine)->EngineStatus() : std::string("{}"), status, len);
}

void GetMemoryInfo(void* engine, char** memory_info, int* len) {
  out_buffer(engine ? static_cast<Engine*>(engine)->MemoryInfo() : std::string("{}"), memory_info, len);
}

int GetDocByID(void* engine, const char* docid, int docid_len, char** doc_str, int* len) {
  if (!engine) return -1;
  std::string fb;
  int ret = static_cast<Engine*>(engine)->GetDocByKey(std::string(docid, (size_t)docid_len), &fb);
  out_buffer(fb, doc_str, len);
  return ret;
}

int GetDocByDocID(void* engine, int docid, char next, char** doc_str, int* len) {
  if (!engine) return -1;
  std::string fb;
  int ret = static_cast<Engine*>(engine)->GetDocByDocid(docid, next != 0, &fb);
  out_buffer(fb, doc_str, len);
  return ret;
}

int BuildIndex(void* engine) { return engine ? static_cast<Engine*>(engine)->BuildIndex() : -1; }

int RebuildIndex(void* engine, int drop_before_rebuild, int limit_cpu, int describe) {
  return engine ? static_cast<Engine*>(engine)->RebuildIndex(drop_before_rebuild, limit_cpu, describe) : -1;
}

int Dump(void* engine) { return engine ? static_cast<Engine*>(engine)->Dump() : -1; }
int Load(void* engine) { return engine ? static_cast<Engine*>(engine)->Load() : -1; }

struct CStatus Search(void* engine, const char* request_str, int req_len, char** response_str, int* res_len) {
  struct CStatus c;
  if (!engine) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "null engine"), &c);
    return c;
  }
  // gamma_api.cc:179-185: refused while usage + the request passes the memory limit, before admission control
  if (!static_cast<Engine*>(engine)->request_admitted(req_len)) {
    to_cstatus(gb::Status::Make(gb::kMemoryExceeded, ""), &c);
    return c;
  }
  gb::SearchRequestPB req;
  if (!req.parse(reinterpret_cast<const uint8_t*>(request_str), (size_t)req_len)) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "parse search request failed"), &c);
    return c;
  }
  std::string resp;
  gb::Status st = static_cast<Engine*>(engine)->Search(req, &resp);
  to_cstatus(st, &c);
  if (st.ok()) out_buffer(resp, response_str, res_len);
  return c;
}

struct CStatus Query(void* engine, const char* request_str, int req_len, char** response_str, int* res_len) {
  struct CStatus c;
  if (!engine) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "null engine"), &c);
    return c;
  }
  if (!static_cast<Engine*>(engine)->request_admitted(req_len)) {  // gamma_api.cc:205-211
    to_cstatus(gb::Status::Make(gb::kMemoryExceeded, ""), &c);
    return c;
  }
  gb::QueryRequestPB req;
  if (!req.parse(reinterpret_cast<const uint8_t*>(request_str), (size_t)req_len)) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "parse query request failed"), &c);
    return c;
  }
  std::string resp;
  gb::Status st = static_cast<Engine*>(engine)->Query(req, &resp);
  to_cstatus(st, &c);
  if (st.ok()) out_buffer(resp, response_str, res_len);
  return c;
}

int SetConfig(void* engine, const char* config_str, int len) {
  return engine ? static_cast<Engine*>(engine)->SetConfig(std::string(config_str, (size_t)len)) : -1;
}

int GetConfig(void* engine, char** config_str, int* len) {
  if (!engine) return -1;
  out_buffer(static_cast<Engine*>(engine)->GetConfig(), config_str, len);
  return 0;
}

// gamma_api.cc:312-318; the engine's Backup (engine.h) says what each command does
struct CStatus Backup(void* engine, int command) {
  struct CStatus c;
  if (!engine) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "null engine"), &c);
    return c;
  }
  to_cstatus(static_cast<Engine*>(engine)->Backup(command), &c);
  return c;
}

// a vector field's index type and params (gammacb/gamma.go:538-572); a scalar field ignores them
struct CStatus AddFieldIndexWithParams(void* engine, const char* field_name, int field_name_len, const char* index_type,
                                       int index_type_len, const char* index_params, int index_params_len) {
  struct CStatus c;
  if (!engine || !field_name) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "null engine"), &c);
    return c;
  }
  const std::string type = index_type && index_type_len > 0 ? std::string(index_type, (size_t)index_type_len) : "";
  const std::string params =
      index_params && index_params_len > 0 ? std::string(index_params, (size_t)index_params_len) : "";
  to_cstatus(static_cast<Engine*>(engine)->SetFieldIndexed(std::string(field_name, (size_t)field_name_len), true, type,
                                                           params),
             &c);
  return c;
}

struct CStatus RemoveFieldIndex(void* engine, const char* field_name, int field_name_len) {
  struct CStatus c;
  if (!engine || !field_name) {
    to_cstatus(gb::Status::Make(gb::kInvalidArgument, "null engine"), &c);
    return c;
  }
  to_cstatus(static_cast<Engine*>(engine)->SetFieldIndexed(std::string(field_name, (size_t)field_name_len), false), &c);
  return c;
}

// MemoryManager's limit (memory/memoryManager.cc:17-26): memory_limit % of each device's HBM and of host memory, over
// what this library holds (mem_ledger.h); 0 removes it
void SetMemoryLimitConfig(int memory_limit) { gb::mem::set_limit_percent(memory_limit); }

void SetKillStatus(const char* request_id, int partition_id, int reason) {
  if (request_id) Engine::SetKill(request_id, partition_id, reason);
}

void DeleteKillStatus(const char* request_id, int partition_id) {
  if (request_id) Engine::ClearKill(request_id, partition_id);
}

}  // extern "C"

// ---- host-logic test hooks (declared in include/gamma_b200_index.h): exercise the wire codecs
// without a GPU so the CPU test suite can pin them against golden bytes -------------------------
#include "wire.h"

static std::string hex_escape(const std::string& s) { return gb::json_escape(s); }
static std::string to_hex(const std::string& s) {
  static const char* d = "0123456789abcdef";
  std::string o;
  for (unsigned char c : s) o += d[c >> 4], o += d[c & 15];
  return o;
}

extern "C" {

// the kill registry (SetKillStatus) with a caller's token in place of a running search's word: op 1 registers it under
// (request_id, partition_id), op 0 removes it
int gb_debug_cancel_register(const char* request_id, int partition_id, gb_cancel_token* token, int op) {
  if (!request_id || !token) return -1;
  if (op)
    Engine::RegisterCancel(request_id, partition_id, token->c);
  else
    Engine::UnregisterCancel(request_id, partition_id, token->c);
  return 0;
}

// admission controller introspection: op 0 = threshold, 1 = in-flight count, 2 = set threshold to `value`
// (<= 0 restores the system-derived one), 3 = Acquire(value) -> 1 admitted / 0 refused, 4 = Release(value)
int gb_debug_concurrency(int op, int value) {
  auto& c = gb::RequestConcurrentController::GetInstance();
  switch (op) {
    case 0: return c.threshold();
    case 1: return c.in_flight();
    case 2: c.set_threshold(value); return c.threshold();
    case 3: return c.Acquire(value) ? 1 : 0;
    case 4: c.Release(value); return c.in_flight();
  }
  return -1;
}

int gb_memory_ledger(int device, int64_t* usage, int64_t* pool_reserved, int64_t* limit) {
  if (usage) *usage = gb::mem::usage(device);
  if (pool_reserved) *pool_reserved = device >= 0 ? gb::mem::pool_reserved(device) : 0;
  if (limit) *limit = gb::mem::limit(device);
  return 0;
}

void gb_memory_set_total(int device, int64_t bytes) { gb::mem::set_total(device, bytes); }

int gb_debug_backup_hold(int op) { return gb::backup_hold(op); }

int gb_debug_backup_stage(int64_t* device_bytes, int64_t* host_bytes) {
  gb::last_capture_stage(device_bytes, host_bytes);
  return 0;
}

void* gb_debug_engine_create(const char* path) { return path ? static_cast<void*>(new Engine(path, "default", 0)) : nullptr; }

// the run-time index records at the end of a snapshot's last `len` bytes, as Load reads them:
// {"bytes": <record part>, "records": [[field, has_index, type, params], ...]}; -1 if a record does not parse
int gb_debug_index_records(const char* tail, int64_t len, char** json_out, int* out_len) {
  std::vector<gb::IndexRecord> recs;
  size_t bytes = 0;
  if (gb::decode_index_records(std::string(tail, (size_t)len), &recs, &bytes)) return -1;
  std::string j = "{\"bytes\":" + std::to_string(bytes) + ",\"records\":[";
  for (size_t i = 0; i < recs.size(); i++)
    j += std::string(i ? "," : "") + "[\"" + hex_escape(recs[i].field) + "\"," + (recs[i].has_index ? "true" : "false") +
         ",\"" + hex_escape(recs[i].type) + "\",\"" + hex_escape(recs[i].params) + "\"]";
  out_buffer(j + "]}", json_out, out_len);
  return 0;
}

int gb_debug_parse_search_request(const char* buf, int len, char** json_out, int* out_len) {
  gb::SearchRequestPB r;
  bool ok = r.parse(reinterpret_cast<const uint8_t*>(buf), (size_t)len);
  std::string j = "{";
  j += "\"ok\":" + std::string(ok ? "true" : "false");
  j += ",\"request_id\":\"" + hex_escape(r.request_id) + "\"";
  j += ",\"partition_id\":" + std::to_string(r.partition_id);
  j += ",\"req_num\":" + std::to_string(r.req_num);
  j += ",\"topn\":" + std::to_string(r.topn);
  j += ",\"brute_force_search\":" + std::to_string(r.brute_force_search);
  j += ",\"index_params\":\"" + hex_escape(r.index_params) + "\"";
  j += ",\"multi_vector_rank\":" + std::to_string(r.multi_vector_rank);
  j += ",\"l2_sqrt\":" + std::string(r.l2_sqrt ? "true" : "false");
  j += ",\"trace\":" + std::string(r.trace ? "true" : "false");
  j += ",\"offset\":" + std::to_string(r.offset);
  j += ",\"n_range_filters\":" + std::to_string(r.n_range_filters);
  j += ",\"n_term_filters\":" + std::to_string(r.n_term_filters);
  j += ",\"filter_operator\":" + std::to_string(r.filter_operator);
  j += ",\"filters\":[";
  for (size_t i = 0; i < r.filters.size(); i++) {
    auto& fl = r.filters[i];
    j += std::string(i ? "," : "") + "{\"field\":\"" + hex_escape(fl.field) + "\",\"lower\":\"" + to_hex(fl.lower) +
         "\",\"upper\":\"" + to_hex(fl.upper) + "\",\"include_lower\":" + (fl.include_lower ? "true" : "false") +
         ",\"include_upper\":" + (fl.include_upper ? "true" : "false") + ",\"is_term\":" + (fl.is_term ? "true" : "false") +
         ",\"is_union\":" + std::to_string(fl.is_union) + "}";
  }
  j += "]";
  j += ",\"fields\":[";
  for (size_t i = 0; i < r.fields.size(); i++) j += (i ? ",\"" : "\"") + hex_escape(r.fields[i]) + "\"";
  j += "],\"vec_fields\":[";
  for (size_t i = 0; i < r.vec_fields.size(); i++) {
    auto& v = r.vec_fields[i];
    char nb[128];
    snprintf(nb, sizeof nb, "%.17g,\"max_score\":%.17g", v.has_min ? v.min_score : 0.0, v.has_max ? v.max_score : 0.0);
    j += std::string(i ? "," : "") + "{\"name\":\"" + hex_escape(v.name) + "\",\"value_len\":" +
         std::to_string(v.value.size()) + ",\"index_type\":\"" + hex_escape(v.index_type) + "\",\"min_score\":" + nb + "}";
  }
  j += "]}";
  out_buffer(j, json_out, out_len);
  return ok ? 0 : -1;
}

// flatbuffers Doc -> re-serialised with the C++ builder (reader + builder round trip)
int gb_debug_roundtrip_doc(const char* buf, int len, char** out, int* out_len) {
  gb::FbTable d = gb::FbTable::root(reinterpret_cast<const uint8_t*>(buf), (size_t)len);
  if (!d.ok()) return -1;
  gb::FbBuilder b;
  std::vector<gb::FbBuilder::Off> offs;
  for (size_t i = 0; i < d.vec_len(0); i++) {
    gb::FbTable f = d.vec_table(0, i);
    const uint8_t* p = nullptr;
    size_t n = 0;
    f.bytes(1, &p, &n);
    gb::FbBuilder::Off v = b.create_bytes(p, n, false);
    gb::FbBuilder::Off nm = b.create_string(f.str(0));
    b.start_table(3);
    b.add_offset(0, nm);
    b.add_offset(1, v);
    int8_t dt = f.scalar<int8_t>(2, 0);
    if (dt) b.add_scalar<int8_t>(2, dt);
    offs.push_back(b.end_table());
  }
  gb::FbBuilder::Off fv = b.create_offset_vector(offs);
  b.start_table(1);
  b.add_offset(0, fv);
  b.finish(b.end_table());
  out_buffer(std::string(reinterpret_cast<const char*>(b.data()), b.size()), out, out_len);
  return 0;
}

// flatbuffers Table -> JSON summary of what CreateTable would see
int gb_debug_parse_table(const char* buf, int len, char** json_out, int* out_len) {
  gb::FbTable t = gb::FbTable::root(reinterpret_cast<const uint8_t*>(buf), (size_t)len);
  if (!t.ok()) return -1;
  std::string j = "{\"name\":\"" + hex_escape(t.str(0)) + "\",\"fields\":[";
  for (size_t i = 0; i < t.vec_len(1); i++) {
    gb::FbTable f = t.vec_table(1, i);
    j += std::string(i ? "," : "") + "{\"name\":\"" + hex_escape(f.str(0)) + "\",\"data_type\":" +
         std::to_string((int)f.scalar<int8_t>(1, 0)) + ",\"is_index\":" + std::to_string((int)f.scalar<uint8_t>(2, 0)) + "}";
  }
  j += "],\"vectors\":[";
  for (size_t i = 0; i < t.vec_len(2); i++) {
    gb::FbTable v = t.vec_table(2, i);
    j += std::string(i ? "," : "") + "{\"name\":\"" + hex_escape(v.str(0)) + "\",\"dimension\":" +
         std::to_string(v.scalar<int32_t>(3, 0)) + ",\"store_type\":\"" + hex_escape(v.str(4)) + "\"}";
  }
  j += "],\"refresh_interval\":" + std::to_string(t.scalar<int32_t>(5, 1000));
  j += ",\"enable_id_cache\":" + std::to_string((int)t.scalar<uint8_t>(6, 0));
  j += ",\"enable_realtime\":" + std::to_string((int)t.scalar<uint8_t>(7, 0));
  j += ",\"indexes\":[";
  for (size_t i = 0; i < t.vec_len(8); i++) {
    gb::FbTable ix = t.vec_table(8, i);
    j += std::string(i ? "," : "") + "{\"name\":\"" + hex_escape(ix.str(0)) + "\",\"type\":\"" + hex_escape(ix.str(1)) +
         "\",\"field_name\":\"" + hex_escape(ix.str(2)) + "\",\"params\":\"" + hex_escape(ix.str(4)) + "\"}";
  }
  j += "]}";
  out_buffer(j, json_out, out_len);
  return 0;
}

// SearchResponse encoder check: one result with the given scores/keys
int gb_debug_encode_response(int nq, int k, const double* scores, const char* const* keys, int total, char** out,
                             int* out_len) {
  gb::PbWriter resp;
  for (int i = 0; i < nq; i++) {
    gb::PbWriter sr, items;
    double mx = -1.7976931348623157e308;
    for (int j = 0; j < k; j++) {
      gb::PbWriter item, fld;
      double s = scores[i * k + j];
      if (s > mx) mx = s;
      item.put_double(1, s);
      fld.put_string(1, "_id");
      fld.put_bytes(3, keys[i * k + j], strlen(keys[i * k + j]));
      item.put_message(2, fld.out);
      items.put_message(7, item.out);
    }
    sr.put_double(2, mx);
    gb::PbWriter st;
    st.put_int32(1, total);
    st.put_int32(3, total);
    sr.put_message(5, st.out);
    sr.put_string(6, "OK");
    sr.out += items.out;
    resp.put_message(2, sr.out);
  }
  out_buffer(resp.out, out, out_len);
  return 0;
}

}  // extern "C"
