// Engine (see engine.h).  Reference call sites cited inline.
#include "engine.h"

#include <float.h>
#include <stdio.h>
#include <string.h>
#include <dirent.h>
#include <errno.h>
#include <fcntl.h>
#include <ftw.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <thread>
#include <fstream>
#include <map>

#include "json.h"
#include "params.h"
#include "wire.h"

namespace gb {

std::string Status::ToString() const {  // util/status.cc:43-100
  const char* type = "";
  switch (code) {
    case kOk: return "OK";
    case kNotFound: type = "NotFound: "; break;
    case kIndexError: type = "IndexError: "; break;
    case kNotSupported: type = "Not implemented: "; break;
    case kInvalidArgument: type = "Invalid argument: "; break;
    case kIOError: type = "IO error: "; break;
    case kBusy: type = "Resource busy: "; break;
    case kTimedOut: type = "Operation timed out: "; break;
    case kCanceled: type = "Operation canceled: "; break;
    case kMemoryExceeded: type = "Memory exceed limit: "; break;
    default: type = "Unknown code: "; break;
  }
  return std::string(type) + msg;
}

// ---- vearchpb.SearchRequest (router_grpc.proto:168-191; request.cc:17-91) --------------------
static bool parse_filter(const PbField& f, bool is_term, SearchRequestPB::Filter* fl) {
  fl->is_term = is_term;
  PbReader v(f.data, f.len);
  PbField vf;
  while (v.next(&vf)) {
    if (vf.num == 1 && vf.wire == 2) fl->field.assign(reinterpret_cast<const char*>(vf.data), vf.len);
    if (vf.num == 2 && vf.wire == 2) fl->lower.assign(reinterpret_cast<const char*>(vf.data), vf.len);
    if (is_term) {
      if (vf.num == 3 && vf.wire == 0) fl->is_union = (int)vf.val;
    } else {
      if (vf.num == 3 && vf.wire == 2) fl->upper.assign(reinterpret_cast<const char*>(vf.data), vf.len);
      if (vf.num == 4 && vf.wire == 0) fl->include_lower = vf.val != 0;
      if (vf.num == 5 && vf.wire == 0) fl->include_upper = vf.val != 0;
      if (vf.num == 6 && vf.wire == 0) fl->is_union = (int)vf.val;
    }
  }
  return !v.error();
}

bool QueryRequestPB::parse(const uint8_t* data, size_t len) {
  PbReader r(data, len);
  PbField f;
  while (r.next(&f)) {
    switch (f.num) {
      case 2:
        if (f.wire == 2) document_ids.emplace_back(reinterpret_cast<const char*>(f.data), f.len);
        break;
      case 3: partition_id = (int)f.val; break;
      case 5:
      case 6: {
        if (f.wire != 2) break;
        SearchRequestPB::Filter fl;
        if (!parse_filter(f, f.num == 6, &fl)) return false;
        filters.push_back(std::move(fl));
        break;
      }
      case 7:
        if (f.wire == 2) fields.emplace_back(reinterpret_cast<const char*>(f.data), f.len);
        break;
      case 9: limit = (int)f.val; break;
      case 15: filter_operator = (int)f.val; break;
      case 17: offset = (int)f.val; break;
      default: break;
    }
  }
  return !r.error();
}

bool SearchRequestPB::parse(const uint8_t* data, size_t len) {
  PbReader r(data, len);
  PbField f;
  while (r.next(&f)) {
    switch (f.num) {
      case 1: {  // RequestHead: only params (field 7, map<string,string>) matter
        if (f.wire != 2) break;
        PbReader h(f.data, f.len);
        PbField hf;
        while (h.next(&hf)) {
          if (hf.num != 7 || hf.wire != 2) continue;
          PbReader e(hf.data, hf.len);
          PbField ef;
          std::string k, v;
          while (e.next(&ef)) {
            if (ef.wire != 2) continue;
            if (ef.num == 1) k.assign(reinterpret_cast<const char*>(ef.data), ef.len);
            if (ef.num == 2) v.assign(reinterpret_cast<const char*>(ef.data), ef.len);
          }
          if (k == "request_id") request_id = v;
          if (k == "partition_id") partition_id = atoi(v.c_str());
        }
        if (h.error()) return false;
        break;
      }
      case 2: req_num = (int)f.val; break;
      case 3: topn = (int)f.val; break;
      case 4: brute_force_search = (int)f.val; break;
      case 5: {  // VectorQuery
        if (f.wire != 2) break;
        VecQuery q;
        PbReader v(f.data, f.len);
        PbField vf;
        while (v.next(&vf)) {
          if (vf.num == 1 && vf.wire == 2) q.name.assign(reinterpret_cast<const char*>(vf.data), vf.len);
          if (vf.num == 2 && vf.wire == 2) q.value.assign(reinterpret_cast<const char*>(vf.data), vf.len);
          if (vf.num == 3 && vf.wire == 1) q.min_score = pb_double(vf.val), q.has_min = true;
          if (vf.num == 4 && vf.wire == 1) q.max_score = pb_double(vf.val), q.has_max = true;
          if (vf.num == 6 && vf.wire == 2) q.index_type.assign(reinterpret_cast<const char*>(vf.data), vf.len);
        }
        if (v.error()) return false;
        vec_fields.push_back(std::move(q));
        break;
      }
      case 6:
        if (f.wire == 2) fields.emplace_back(reinterpret_cast<const char*>(f.data), f.len);
        break;
      case 7:
      case 8: {
        if (f.wire != 2) break;
        Filter fl;
        if (!parse_filter(f, f.num == 8, &fl)) return false;
        (fl.is_term ? n_term_filters : n_range_filters)++;
        filters.push_back(std::move(fl));
        break;
      }
      case 9:
        if (f.wire == 2) index_params.assign(reinterpret_cast<const char*>(f.data), f.len);
        break;
      case 10: multi_vector_rank = (int)f.val; break;
      case 15:
        if (f.wire == 2) ranker.assign(reinterpret_cast<const char*>(f.data), f.len);
        break;
      case 11: l2_sqrt = f.val != 0; break;
      case 16: trace = f.val != 0; break;
      case 17: filter_operator = (int)f.val; break;
      case 20: offset = (int)f.val; break;
      default: break;  // unknown / unused fields are skipped
    }
  }
  return !r.error();
}

// ---- kill switch ---------------------------------------------------------------------------
// g_killed: the kills recorded (checked before and after a search); g_inflight: the cancel word of every running search
// by (request id, partition id), which SetKill sets so the search's kernels and host loops stop early (DESIGN.md
// section 8, cancellation).  A word only ever goes from 0 to 1 while its search runs: ClearKill does not reset it.
static std::mutex g_kill_mu;
static std::map<std::pair<std::string, int>, int> g_killed;
static std::multimap<std::pair<std::string, int>, CancelWord*> g_inflight;
static std::vector<CancelWord*> g_idle_words;  // words of finished searches, reset to 0, for the next ones
void Engine::SetKill(const std::string& request_id, int partition_id, int reason) {
  std::lock_guard<std::mutex> g(g_kill_mu);
  g_killed[{request_id, partition_id}] = reason;
  auto r = g_inflight.equal_range({request_id, partition_id});
  for (auto it = r.first; it != r.second; ++it) cancel_set(it->second->w);
}
void Engine::ClearKill(const std::string& request_id, int partition_id) {
  std::lock_guard<std::mutex> g(g_kill_mu);
  g_killed.erase({request_id, partition_id});
}
void Engine::RegisterCancel(const std::string& request_id, int partition_id, CancelWord* c) {
  std::lock_guard<std::mutex> g(g_kill_mu);
  g_inflight.insert({{request_id, partition_id}, c});
  if (g_killed.count({request_id, partition_id})) cancel_set(c->w);
}
void Engine::UnregisterCancel(const std::string& request_id, int partition_id, CancelWord* c) {
  std::lock_guard<std::mutex> g(g_kill_mu);
  auto r = g_inflight.equal_range({request_id, partition_id});
  for (auto it = r.first; it != r.second; ++it)
    if (it->second == c) {
      g_inflight.erase(it);
      return;
    }
}
Engine::KillScope::KillScope(const std::string& request_id, int partition_id) : rid(request_id), pid(partition_id) {
  if (request_id.empty()) return;  // a request without an id cannot be killed (IsKilled)
  {
    std::lock_guard<std::mutex> g(g_kill_mu);
    if (!g_idle_words.empty()) {
      c = g_idle_words.back();
      g_idle_words.pop_back();
    }
  }
  if (!c) c = cancel_word_create();
  if (!c) return;  // no word: the search runs to its end, and the kill is still seen after it
  RegisterCancel(rid, pid, c);
}
Engine::KillScope::~KillScope() {
  if (!c) return;
  UnregisterCancel(rid, pid, c);
  *c->w = 0;  // the search has returned: nothing reads the word until the next search takes it
  std::lock_guard<std::mutex> g(g_kill_mu);
  g_idle_words.push_back(c);
}
bool Engine::IsKilled(const std::string& request_id, int partition_id) {
  if (request_id.empty()) return false;
  std::lock_guard<std::mutex> g(g_kill_mu);
  return g_killed.count({request_id, partition_id}) != 0;
}

// ---- admission control (search/engine.cc:47-119) ----------------------------------------------
static int read_proc_int(const char* path) {  // the reference popen()s `cat <path>`; same number, no shell
  int v = -1;
  if (FILE* fp = fopen(path, "r")) {
    if (fscanf(fp, "%d", &v) != 1) v = -1;
    fclose(fp);
  }
  return v;
}
RequestConcurrentController& RequestConcurrentController::GetInstance() {
  static RequestConcurrentController instance;
  return instance;
}
RequestConcurrentController::RequestConcurrentController() {
  const int threads_max = read_proc_int("/proc/sys/kernel/threads-max");
  const int max_map_count = read_proc_int("/proc/sys/vm/max_map_count");
  const int pid_max = read_proc_int("/proc/sys/kernel/pid_max");
  max_threads_ = std::min(std::min(threads_max, pid_max), max_map_count / 2);
  const int host_threads = std::max(1u, std::thread::hardware_concurrency());
  system_threshold_ = (int)((max_threads_ * 0.5) / (host_threads + 1));
  if (system_threshold_ <= 0) system_threshold_ = 1;  // the reference aborts (LOG(FATAL)); a library must not
  concurrent_threshold_ = system_threshold_;
  if (const char* e = getenv("GAMMA_CONCURRENT_THRESHOLD")) set_threshold(atoi(e));
}
void RequestConcurrentController::set_threshold(int t) { concurrent_threshold_ = t > 0 ? t : system_threshold_; }
bool RequestConcurrentController::Acquire(int req_num) {
  const int num = cur_concurrent_num_.fetch_add(req_num);
  return num < concurrent_threshold_;
}
void RequestConcurrentController::Release(int req_num) { cur_concurrent_num_.fetch_sub(req_num); }
namespace {
struct AdmissionGuard {  // every return path of Engine::Search releases what it acquired
  int n;
  bool permit;
  explicit AdmissionGuard(int req_num) : n(req_num), permit(RequestConcurrentController::GetInstance().Acquire(req_num)) {}
  ~AdmissionGuard() { RequestConcurrentController::GetInstance().Release(n); }
};
}  // namespace

// ---------------------------------------------------------------------------------------------
Engine::Engine(const std::string& path, const std::string& space_name, int device, const std::vector<int>& devices)
    : path_(path), space_name_(space_name), device_(devices.empty() ? device : devices[0]), devices_(devices) {}

// the GPU types shard over a device list of two entries or more (IndexShards); everything else lives on device_
Index* Engine::make_index(const std::string& type, int dim, const ModelParams& mp) const {
  if (devices_.size() > 1 && is_gpu_index_type(type)) return create_sharded_index(type, dim, mp, devices_, 20);
  return create_index(type, dim, mp, device_, 20);
}

namespace {
// the trained state a Dump writes beside the rows and a Load restores: the IVF index, or a sharded index's first shard
// (every shard holds the same; ShardedIndex::train copies shard 0's to the others)
IvfIndex* trained_state_of(Index* ix) {
  if (ShardedIndex* sh = dynamic_cast<ShardedIndex*>(ix)) return sh->shard(0);
  return dynamic_cast<IvfIndex*>(ix);
}
}  // namespace

namespace {
struct LiveEngines {
  std::mutex mu;
  std::vector<Engine*> all;
};
LiveEngines& live_engines() {
  static LiveEngines* s = new LiveEngines;  // leaked on purpose
  return *s;
}
void quiesce_all_engines() {
  std::vector<Engine*> v;
  {
    std::lock_guard<std::mutex> g(live_engines().mu);
    v = live_engines().all;
  }
  for (Engine* e : v) e->quiesce();
}
}  // namespace

void Engine::quiesce() {
  field_build_stop_.store(true);
  join_field_build();
  stop_indexing();
}
void Engine::stop_indexing() {
  int st = indexing_state_.load();
  if (st != 0) indexing_state_.store(3);
  idx_cv_.notify_all();
  std::lock_guard<std::mutex> g(indexing_thread_mu_);
  if (indexing_thread_.joinable()) indexing_thread_.join();
}

Engine::~Engine() {
  // Close: stop the indexing thread (search/engine.cc Engine::~Engine / Close)
  {
    std::lock_guard<std::mutex> g(live_engines().mu);
    auto& a = live_engines().all;
    a.erase(std::remove(a.begin(), a.end(), this), a.end());
  }
  quiesce();
  cudaSetDevice(device_);
  index_.reset();
}

// Engine::CreateTable (search/engine.cc:582-690) + TableInfo::Deserialize (table.cc:30-157) +
// VectorManager::CreateVectorTable (vector_manager.cc:343-453)
Status Engine::CreateTable(const uint8_t* fb, size_t len) {
  std::unique_lock<std::shared_mutex> lk(mu_);
  if (created_table_) return Status::Make(kInvalidArgument, "table is created");
  FbTable t = FbTable::root(fb, len);
  if (!t.ok()) return Status::Make(kInvalidArgument, "table deserialize error");
  table_name_ = t.str(0);
  fields_.clear();
  field_idx_.clear();
  bool has_id = false;
  for (size_t i = 0; i < t.vec_len(1); i++) {
    FbTable f = t.vec_table(1, i);
    FieldDef fd{f.str(0), (int)f.scalar<int8_t>(1, 0), f.scalar<uint8_t>(2, 0) != 0};
    if (fd.name == "_id") has_id = true;
    field_idx_[fd.name] = (int)fields_.size();
    fields_.push_back(fd);
  }
  if (!has_id) {  // the key field always exists (table/table.cc)
    field_idx_["_id"] = (int)fields_.size();
    fields_.push_back({"_id", DT_STRING, false});
  }
  values_.assign(fields_.size(), {});
  sidx_.clear();
  sidx_.resize(fields_.size());
  size_t nvec = t.vec_len(2);
  if (nvec == 0) return Status::Make(kInvalidArgument, space_name_ + " table has no vector field");
  FbTable v = t.vec_table(2, 0);
  vec_name_ = v.str(0);
  dim_ = v.scalar<int32_t>(3, 0);
  if (dim_ <= 0) return Status::Make(kInvalidArgument, "invalid vector dimension");
  std::string table_index_params = t.str(4);
  refresh_interval_ = t.scalar<int32_t>(5, 1000);
  enable_id_cache_ = t.scalar<uint8_t>(6, 0) != 0;
  enable_realtime_ = t.scalar<uint8_t>(7, 0) != 0;
  training_threshold_ = 0;
  {
    JsonValue jv;
    int tt = 0;
    if (!table_index_params.empty() && JsonParser::parse(table_index_params, &jv) && jv.get_int("training_threshold", &tt) &&
        tt > 0)
      training_threshold_ = tt;
  }
  table_training_threshold_ = training_threshold_;
  // index type of the vector field: first entry of `indexes` with a matching field_name
  // (vector_manager.cc:365-373)
  index_type_.clear();
  for (size_t i = 0; i < t.vec_len(8); i++) {
    FbTable ix = t.vec_table(8, i);
    if (ix.str(2) == vec_name_ && !ix.str(1).empty()) {
      index_type_ = ix.str(1);
      index_params_ = ix.str(4);
      break;
    }
  }
  if (index_type_.empty()) return Status::Make(kInvalidArgument, vec_name_ + " index type is empty");
  table_params_given_ = !table_index_params.empty();
  Index* idx = nullptr;
  Status ist = create_field_index(vec_name_, dim_, index_type_, index_params_, true,
                                  !strcasecmp(v.str(4).c_str(), "RocksDB"),  // VectorInfo.store_type
                                  nvec, &training_threshold_, &idx);
  if (!ist.ok()) return ist;
  index_.reset(idx);
  vbytes_ = (size_t)idx->store().row_bytes();
  extra_.clear();
  for (size_t vi = 1; vi < nvec; vi++) {  // the other vector fields: same rules, their own index each
    FbTable ev = t.vec_table(2, vi);
    VecField vf;
    vf.name = ev.str(0);
    vf.dim = ev.scalar<int32_t>(3, 0);
    if (vf.dim <= 0 || vf.name.empty() || vf.name == vec_name_) return Status::Make(kInvalidArgument, "invalid vector field");
    for (size_t i = 0; i < t.vec_len(8); i++) {
      FbTable ix = t.vec_table(8, i);
      if (ix.str(2) == vf.name && !ix.str(1).empty()) {
        vf.index_type = ix.str(1);
        vf.index_params = ix.str(4);
        break;
      }
    }
    if (vf.index_type.empty()) return Status::Make(kInvalidArgument, vf.name + " index type is empty");
    int64_t ett = training_threshold_;
    Index* eidx = nullptr;
    Status est = create_field_index(vf.name, vf.dim, vf.index_type, vf.index_params, false,
                                    !strcasecmp(ev.str(4).c_str(), "RocksDB"), nvec, &ett, &eidx);
    if (!est.ok()) return est;
    vf.index.reset(eidx);
    extra_.push_back(std::move(vf));
  }
  {  // registered after the index (and so after CUDA start-up): at exit the engine's thread stops first
    std::lock_guard<std::mutex> g(live_engines().mu);
    static bool hooked = (atexit(quiesce_all_engines), true);
    (void)hooked;
    live_engines().all.push_back(this);
  }
  if (training_threshold_ <= 0) training_threshold_ = index_->training_threshold();
  for (size_t fi = 0; fi < fields_.size(); fi++)
    if (fields_[fi].indexed && scalar_index_rebuild((int)fi)) return Status::Make(kIndexError, last_error());
  fidx_.assign(nvec, FieldIndex());
  created_table_ = true;
  // <path>/<table>.schema, as the reference writes it (engine.cc:676-684)
  if (!path_.empty()) {
    mkdir(path_.c_str(), 0755);
    std::ofstream f(path_ + "/" + table_name_ + ".schema", std::ios::binary);
    if (f) f.write(reinterpret_cast<const char*>(fb), (std::streamsize)len);
  }
  return Status::OK();
}

int Engine::vec_field(const std::string& name) const {
  if (name == vec_name_) return 0;
  for (size_t i = 0; i < extra_.size(); i++)
    if (extra_[i].name == name) return (int)i + 1;
  return -1;
}
std::shared_ptr<Index> Engine::index_ref(const std::string& vec_name, int* dim) {
  const int vi = vec_field(vec_name);
  if (vi < 0) return nullptr;
  *dim = vdim(vi);
  return std::atomic_load(&vslot(vi));
}

Index* Engine::index_of(const std::string& vec_name, int* dim) {
  if (vec_name == vec_name_) {
    *dim = dim_;
    return index_.get();
  }
  for (auto& e : extra_)
    if (e.name == vec_name) {
      *dim = e.dim;
      return e.index.get();
    }
  return nullptr;
}

int Engine::flush_pending_locked() {
  if (scalar_flush_locked()) return -1;
  if (pending_n_ == 0) return 0;
  // Row i of every vector field must stay document i: a field is appended only while its store is as long as the
  // primary one was when this flush began, so a retry after a partial failure appends exactly the missing fields,
  // and the pending buffers are dropped only when every field has taken its rows.
  const int64_t base = index_->store().size();
  for (auto& e : extra_) {
    if (e.index->store().size() == base + pending_n_) continue;  // taken by an earlier, partially failed flush
    if (e.index->store().size() != base || (int64_t)e.pending.size() != (int64_t)pending_n_ * e.dim) {
      set_last_error("vector fields out of step (field " + e.name + ")");
      return -1;
    }
    if (e.index->add_vectors(e.pending.data(), pending_n_)) return -1;
  }
  int rc = index_->add_vectors(pending_.data(), pending_n_);
  if (rc) return rc;
  for (auto& e : extra_) e.pending.clear();
  pending_.clear();
  pending_n_ = 0;
  return 0;
}

void Engine::memory_places(std::vector<mem::Charge>* out, int64_t bytes) const {
  out->push_back({device_, bytes});
  for (int d : devices_)
    if (d != device_) out->push_back({d, bytes});
  bool host = index_ && index_->store().on_host();
  for (auto& e : extra_) host = host || e.index->store().on_host();
  if (host) out->push_back({mem::kHost, bytes});
}
bool Engine::rows_admitted(int64_t n_total) {
  if (!mem::limited()) return true;
  std::vector<mem::Charge> c;
  memory_places(&c, 0);  // nothing to grow still needs usage within the limit
  index_->memory_charges(n_total, &c);
  for (auto& e : extra_) e.index->memory_charges(n_total, &c);
  return mem::admit(c);
}
bool Engine::request_admitted(int64_t bytes) const {
  if (!mem::limited()) return true;
  std::vector<mem::Charge> c;
  memory_places(&c, bytes);
  return mem::admit(c);
}

// Engine::AddOrUpdate (search/engine.cc:691-772) + Doc::Deserialize (doc.cc:43-76)
int Engine::AddOrUpdate(const uint8_t* fb, size_t len) {
  if (!created_table_) return -1;
  FbTable d = FbTable::root(fb, len);
  if (!d.ok()) return -3;
  std::string key;
  std::vector<DocField> table_fields;
  const uint8_t* vec = nullptr;
  size_t vec_len = 0;
  bool has_vec = false;
  std::vector<std::pair<const uint8_t*, size_t>> evec(extra_.size(), {nullptr, 0});
  for (size_t i = 0; i < d.vec_len(0); i++) {
    FbTable f = d.vec_table(0, i);
    DocField df;
    df.name = f.str(0);
    const uint8_t* p = nullptr;
    size_t n = 0;
    f.bytes(1, &p, &n);
    df.data_type = f.scalar<int8_t>(2, 0);
    if (df.name == "_id") key.assign(reinterpret_cast<const char*>(p), n);
    if (df.data_type == DT_VECTOR) {
      if (df.name == vec_name_) {
        vec = p;
        vec_len = n;
        has_vec = true;
      }
      for (size_t ei = 0; ei < extra_.size(); ei++)
        if (df.name == extra_[ei].name) evec[ei] = {p, n};
    } else {
      if (!field_idx_.count(df.name)) continue;  // "Unknown field" (doc.cc:66-69)
      df.value.assign(reinterpret_cast<const char*>(p), n);
      table_fields.push_back(std::move(df));
    }
  }
  std::unique_lock<std::shared_mutex> lk(mu_);
  auto it = key2docid_.find(key);
  int docid = it == key2docid_.end() ? -1 : it->second;
  if (docid != -1 && docid < max_docid_) {  // Update (engine.cc:703-710, 774-850)
    for (auto& f : table_fields) {
      const int fi = field_idx_[f.name];
      scalar_index_put(fi, docid, f.value, &values_[fi][docid]);
      values_[fi][docid] = f.value;
    }
    if (scalar_staged() >= kScalarFlushRows && scalar_flush_locked()) return -1;
    if (has_vec) {
      if (vec_len != vbytes_) return -1;
      std::vector<unsigned char> x(vec, vec + vec_len);
      if (flush_pending_locked()) return -1;
      if (index_->update_vector(docid, x.data())) return -1;
      if (fidx_[0].building) fidx_[0].updated.push_back(docid);
    }
    for (size_t ei = 0; ei < extra_.size(); ei++) {
      if (!evec[ei].first) continue;
      if (evec[ei].second != (size_t)extra_[ei].dim * 4) return -1;
      std::vector<float> x(extra_[ei].dim);
      memcpy(x.data(), evec[ei].first, evec[ei].second);
      if (flush_pending_locked()) return -1;
      if (extra_[ei].index->update_vector(docid, x.data())) return -1;
      if (fidx_[ei + 1].building) fidx_[ei + 1].updated.push_back(docid);
    }
    purge_indexes(delete_num_ > 0 ? del_bitmap_.data() : nullptr, (size_t)(max_docid_ >> 3) + 1);
    return 0;
  } else if (docid >= max_docid_) {
    return -2;
  }
  // CheckDoc (engine.cc:802-813): every vector field present with d*4 bytes (BINARYIVF: d / 8)
  if (!has_vec || vec_len != vbytes_) return -3;
  for (size_t ei = 0; ei < extra_.size(); ei++)
    if (!evec[ei].first || evec[ei].second != (size_t)extra_[ei].dim * 4) return -3;
  if (key.empty()) return -3;
  // VectorManager::AddToStore fails when the raw vectors' next segment would pass the memory limit
  // (memory_raw_vector.cc:165-185): the document is refused before anything of it is stored
  if (!rows_admitted((int64_t)max_docid_ + 1)) return -5;
  for (size_t fi = 0; fi < fields_.size(); fi++) values_[fi].emplace_back();
  for (auto& f : table_fields) values_[field_idx_[f.name]][max_docid_] = f.value;
  values_[field_idx_["_id"]][max_docid_] = key;
  for (size_t fi = 0; fi < fields_.size(); fi++)
    if (fields_[fi].indexed) scalar_index_put((int)fi, max_docid_, values_[fi][max_docid_], nullptr);
  keys_.push_back(key);
  key2docid_[key] = max_docid_;
  pending_.resize((size_t)(pending_n_ + 1) * vbytes_);
  memcpy(pending_.data() + (size_t)pending_n_ * vbytes_, vec, vec_len);
  for (size_t ei = 0; ei < extra_.size(); ei++) {
    auto& e = extra_[ei];
    e.pending.resize((size_t)(pending_n_ + 1) * e.dim);
    memcpy(e.pending.data() + (size_t)pending_n_ * e.dim, evec[ei].first, evec[ei].second);
  }
  pending_n_++;
  ++max_docid_;
  if ((size_t)(max_docid_ >> 3) + 1 > del_bitmap_.size()) del_bitmap_.resize((size_t)(max_docid_ >> 3) + 4096, 0);
  if ((pending_n_ >= 8192 || scalar_staged() >= kScalarFlushRows) && flush_pending_locked()) return -5;
  // auto-start indexing (engine.cc:753-761)
  if (refresh_interval_ >= 0 && indexing_state_.load() == 0 && index_status_.load() == 0 &&
      max_docid_ - delete_num_ >= training_threshold_ &&
      now_ms() - last_train_failure_ms_.load() >= kTrainRetryMs) {  // a failed training is retried after a back-off
    lk.unlock();
    BuildIndex();
  }
  return 0;
}

// Engine::Delete (search/engine.cc:852-879)
int Engine::Delete(const std::string& key) {
  std::unique_lock<std::shared_mutex> lk(mu_);
  auto it = key2docid_.find(key);
  if (it == key2docid_.end() || it->second < 0) return -1;
  int docid = it->second;
  if ((del_bitmap_[docid >> 3] >> (docid & 7)) & 1) return 0;
  del_bitmap_[docid >> 3] |= (uint8_t)(1u << (docid & 7));
  ++delete_num_;
  key2docid_.erase(it);  // table_->Delete(key)
  // vec_manager_->Delete(docid) (engine.cc:868): the lists count the entry dead; the bitmap keeps hiding it
  const int64_t vid = docid;
  if (index_) index_->delete_vectors(&vid, 1);
  for (auto& e : extra_) e.index->delete_vectors(&vid, 1);
  for (auto& fx : fidx_)
    if (fx.building) fx.deleted.push_back(vid);
  return 0;
}

void Engine::purge_indexes(const uint8_t* bitmap, size_t bytes) {
  auto purge = [&](Index* ix, const std::string& field) {
    if (ix && ix->purge_lists(0.3f, bitmap, (int64_t)bytes, nullptr))
      fprintf(stderr, "gamma: purge of the dead list entries of field %s failed: %s\n", field.c_str(), last_error());
  };
  purge(index_.get(), vec_name_);
  for (auto& e : extra_) purge(e.index.get(), e.name);
}

void Engine::serialize_doc(int docid, bool with_docid, std::string* out) {
  FbBuilder b;
  std::vector<FbBuilder::Off> offs;
  auto add_field = [&](const std::string& name, const std::string& value, int dt) {
    FbBuilder::Off v = b.create_bytes(value.data(), value.size(), false);
    FbBuilder::Off n = b.create_string(name);
    b.start_table(3);
    b.add_offset(0, n);
    b.add_offset(1, v);
    if (dt) b.add_scalar<int8_t>(2, (int8_t)dt);
    offs.push_back(b.end_table());
  };
  if (docid >= 0) {
    for (size_t fi = 0; fi < fields_.size(); fi++) add_field(fields_[fi].name, values_[fi][docid], fields_[fi].data_type);
    if (with_docid) add_field("_docid", std::string(reinterpret_cast<const char*>(&docid), 4), DT_INT);
    std::string x(vbytes_, '\0');
    bool got = false;
    int64_t stored = index_->store().size();
    if (docid < stored) {
      got = index_->store().get_host(docid, &x[0]) == 0;
    } else if (docid - stored < pending_n_) {
      memcpy(&x[0], pending_.data() + (size_t)(docid - stored) * vbytes_, vbytes_);
      got = true;
    }
    if (got) add_field(vec_name_, x, DT_VECTOR);
    for (auto& e : extra_) {
      std::vector<float> ex(e.dim);
      bool egot = false;
      if (docid < stored) {
        egot = e.index->store().get_host(docid, ex.data()) == 0;
      } else if (docid - stored < pending_n_) {
        memcpy(ex.data(), e.pending.data() + (size_t)(docid - stored) * e.dim, (size_t)e.dim * 4);
        egot = true;
      }
      if (egot) add_field(e.name, std::string(reinterpret_cast<const char*>(ex.data()), (size_t)e.dim * 4), DT_VECTOR);
    }
  }
  FbBuilder::Off fv = b.create_offset_vector(offs);
  b.start_table(1);
  b.add_offset(0, fv);
  b.finish(b.end_table());
  out->assign(reinterpret_cast<const char*>(b.data()), b.size());
}

// Engine::GetDoc (search/engine.cc:881-948)
int Engine::GetDocByKey(const std::string& key, std::string* fb_out) {
  std::shared_lock<std::shared_mutex> lk(mu_);
  cudaSetDevice(device_);
  auto it = key2docid_.find(key);
  if (it == key2docid_.end() || it->second < 0) {
    serialize_doc(-1, false, fb_out);
    return -1;
  }
  int docid = it->second;
  if ((del_bitmap_[docid >> 3] >> (docid & 7)) & 1) {
    serialize_doc(-1, false, fb_out);
    return -1;
  }
  serialize_doc(docid, false, fb_out);
  return 0;
}
int Engine::GetDocByDocid(int docid, bool next, std::string* fb_out) {
  std::shared_lock<std::shared_mutex> lk(mu_);
  cudaSetDevice(device_);
  auto deleted = [&](int id) { return ((del_bitmap_[id >> 3] >> (id & 7)) & 1) != 0; };
  if ((next ? docid < -1 : docid < 0) || docid >= max_docid_) {
    serialize_doc(-1, false, fb_out);
    return -1;
  }
  if (next) {
    while (++docid < max_docid_)
      if (!deleted(docid)) break;
    if (docid >= max_docid_) {
      serialize_doc(-1, false, fb_out);
      return -1;
    }
  } else if (deleted(docid)) {
    serialize_doc(-1, false, fb_out);
    return -1;
  }
  serialize_doc(docid, next, fb_out);
  return 0;
}

// ---- scalar filters ------------------------------------------------------------------------------
// Filter() semantics per field type (table/scalar_index_manager.cc:294-345):
//   numeric: lower == upper -> Equal (NotEqual when is_union == Not); only one bound -> <, <=, >, >=;
//            both -> Range with the include flags.  Values are the field type's raw little-endian bytes.
//   string / string array: lower_value split at \001 -> In (NotIn when is_union == Not); a string-array
//            document matches when any of its \001-separated elements does.
// Search(): the per-filter sets are intersected (operator And) or united (Or).  A filter on a field
// without a scalar index, or an empty result, means "no result" (scalar_index_manager.cc:598-610).
namespace {
std::vector<std::string> split001(const std::string& s) {
  std::vector<std::string> out;
  size_t a = 0;
  while (true) {
    size_t b = s.find('\001', a);
    out.push_back(s.substr(a, b == std::string::npos ? std::string::npos : b - a));
    if (b == std::string::npos) break;
    a = b + 1;
  }
  return out;
}
}  // namespace

static bool is_float_type(int dt) { return dt == DT_FLOAT || dt == DT_DOUBLE; }
static bool is_string_type(int dt) { return dt == DT_STRING || dt == DT_STRINGARRAY; }
// raw little-endian field bytes -> (int64 | double); false: wrong width for the type
static bool decode_num(int dt, const std::string& v, int64_t* iv, double* fv) {
  const size_t w = (dt == DT_INT || dt == DT_FLOAT) ? 4 : (dt == DT_BOOL ? 1 : 8);
  if (v.size() != w) return false;
  switch (dt) {
    case DT_INT: {
      int32_t x;
      memcpy(&x, v.data(), 4);
      *iv = x;
      return true;
    }
    case DT_FLOAT: {
      float x;
      memcpy(&x, v.data(), 4);
      *fv = x;
      return true;
    }
    case DT_DOUBLE: memcpy(fv, v.data(), 8); return true;
    case DT_BOOL: *iv = (uint8_t)v[0]; return true;
    default: memcpy(iv, v.data(), 8); return true;  // DT_LONG, DT_DATE
  }
}

void Engine::scalar_index_put(int fi, int docid, const std::string& value, const std::string* old) {
  if (fi < (int)sidx_.size() && sidx_[fi].built()) sidx_[fi].stage(docid, value, old);
}

int Engine::scalar_index_rebuild(int fi) {
  if (fi >= (int)sidx_.size()) sidx_.resize(fields_.size());
  cudaSetDevice(device_);
  if (sidx_[fi].build(fields_[fi].data_type, values_[fi]) == 0) return 0;
  sidx_[fi].release();
  return -1;
}

int64_t Engine::scalar_staged() const {
  int64_t n = 0;
  for (const auto& c : sidx_) n = std::max(n, c.staged());
  return n;
}

int Engine::scalar_flush_locked() {
  if (scalar_staged() == 0) return 0;
  cudaSetDevice(device_);
  for (size_t fi = 0; fi < sidx_.size(); fi++) {
    ScalarColumn& c = sidx_[fi];
    if (c.flush(cudaStreamPerThread)) return -1;
    if (c.wants_repack() && c.build(fields_[fi].data_type, values_[fi])) return -1;  // the live runs, packed
  }
  return 0;
}

// A request's filter bitmap on device_: ceil(n / 32) + 1 words, zero at and above n, so every scan reads it in place.
// Allocated on the calling thread's stream of device_ and freed there when the request ends.
struct Engine::FilterBits {
  int device;
  Scratch s;
  uint32_t* bits = nullptr;
  int64_t words = 0;
  explicit FilterBits(int dev) : device(dev), s(cudaStreamPerThread) {}
  ~FilterBits() { cudaSetDevice(device); }  // before s frees on the stream of that device
};

int64_t Engine::eval_filters(const std::vector<SearchRequestPB::Filter>& filters, int op, FilterBits* out) const {
  const int64_t n = max_docid_;
  std::vector<FilterDesc> fd;
  std::vector<int32_t> terms, codes;
  std::vector<size_t> term_at;  // fd[i]'s first term in `terms`
  for (const auto& fl : filters) {
    auto it = field_idx_.find(fl.field);
    if (it == field_idx_.end() || !fields_[it->second].indexed) return 0;
    const int fi = it->second, dt = fields_[fi].data_type;
    const bool is_str = is_string_type(dt);
    if (fl.lower.empty() && (is_str || fl.upper.empty())) continue;  // Filter() returns an untouched result
    if (fi >= (int)sidx_.size() || !sidx_[fi].built()) return 0;
    FilterDesc d;
    memset(&d, 0, sizeof d);
    sidx_[fi].describe(&d);
    d.neg = fl.is_union == 2;
    if (is_str) {
      sidx_[fi].codes_of(split001(fl.lower), &codes);  // terms the dictionary does not know match no document
      d.nterms = (int)codes.size();
      term_at.push_back(terms.size());
      terms.insert(terms.end(), codes.begin(), codes.end());
    } else {
      term_at.push_back(terms.size());
      d.has_lo = !fl.lower.empty(), d.has_hi = !fl.upper.empty();
      d.lo_ok = d.has_lo && decode_num(dt, fl.lower, &d.lo_i, &d.lo_f);
      d.hi_ok = d.has_hi && decode_num(dt, fl.upper, &d.hi_i, &d.hi_f);
      d.inc_lo = fl.include_lower, d.inc_hi = fl.include_upper;
      d.equal = fl.lower == fl.upper;
      d.neg = d.equal && d.neg;  // is_union means nothing else to a numeric field
      d.is_float = is_float_type(dt);
    }
    fd.push_back(d);
  }
  if (fd.empty()) return 0;
  cudaSetDevice(device_);
  cudaStream_t st = out->s.stream();
  // one upload: the cardinality counter (zero), the descriptors, the term codes
  const size_t desc_at = 16, codes_at = desc_at + fd.size() * sizeof(FilterDesc);
  std::vector<uint8_t> blob(codes_at + terms.size() * 4, 0);
  out->words = (n + 31) / 32 + 1;
  out->bits = out->s.alloc_n<uint32_t>((size_t)out->words);
  uint8_t* dblob = out->s.alloc_n<uint8_t>(blob.size());
  if (!out->bits || !dblob) return -1;
  for (size_t i = 0; i < fd.size(); i++) fd[i].terms = reinterpret_cast<const int32_t*>(dblob + codes_at) + term_at[i];
  memcpy(blob.data() + desc_at, fd.data(), fd.size() * sizeof(FilterDesc));
  if (!terms.empty()) memcpy(blob.data() + codes_at, terms.data(), terms.size() * 4);
  unsigned long long card = 0;
  auto* dcard = reinterpret_cast<unsigned long long*>(dblob);
  GB_CUDA(cudaMemcpyAsync(dblob, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
  GB_CUDA(launch_filter_eval(reinterpret_cast<const FilterDesc*>(dblob + desc_at), (int)fd.size(), op, n, out->words,
                             out->bits, dcard, st));
  GB_CUDA(cudaMemcpyAsync(&card, dcard, 8, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));  // the columns may change once the shared lock is released
  return (int64_t)card;
}

// Engine::Search (search/engine.cc:242-402) + VectorManager::Search (vector_manager.cc:739-1079)
// + Response::Serialize (response.cc:46-185)
Status Engine::Search(const SearchRequestPB& req, std::string* pb_out) {
  if (!created_table_) return Status::Make(kInvalidArgument, space_name_ + " table not created");
  if (req.req_num <= 0) return Status::Make(kInvalidArgument, space_name_ + " req_num should not less than 0");
  // engine.cc:252-260: Status::ResourceExhausted() = kBusy + "Resource temporarily unavailable"
  AdmissionGuard admission(req.req_num);
  if (!admission.permit) return Status::Make(kBusy, "Resource temporarily unavailable");
  if (req.topn <= 0) return Status::Make(kInvalidArgument, "limit[topN] is zero");
  if (req.vec_fields.empty()) return Status::Make(kInvalidArgument, "no vector query");
  if (req.vec_fields.size() > 1) return SearchMulti(req, pb_out);
  const auto& vq = req.vec_fields[0];
  int qdim = 0;
  std::shared_ptr<Index> qindex = index_ref(vq.name, &qdim);
  if (!qindex) return Status::Make(kInvalidArgument, "Query name " + vq.name + " not exist in created vector table");
  int brute = req.brute_force_search;
  if (brute == 2 && index_status_.load() != 2) brute = 1;
  if (brute == 0 && index_status_.load() != 2 && max_docid_ > 100 && !enable_realtime_ && !awaiting_training_.load())
    return Status::Make(kIndexError, space_name_ + " index not trained, brute_force_search is 0, max_docid_ = " +
                                         std::to_string(max_docid_) + ", threshold = 100");
  const size_t qbytes = (size_t)qindex->store().row_bytes();  // d * 4, or BINARYIVF's d / 8
  int n = (int)(vq.value.size() / qbytes);
  if (n <= 0) return Status::Make(kInvalidArgument, "Search n shouldn't less than 0!");
  if (IsKilled(req.request_id, req.partition_id)) return Status::Make(kMemoryExceeded, "");
  KillScope kill(req.request_id, req.partition_id);
  SearchContext ctx;
  ctx.cancel = kill.word();
  std::string err;
  if (!parse_retrieval_params(req.index_params, &ctx.params, &err)) return Status::Make(kInvalidArgument, err);
  ctx.params.brute_force = brute != 0;
  ctx.search_unindexed_tail = enable_realtime_;
  // proto3 drops zero-valued doubles; the router always sends a window (doc_query.go:1220-1226)
  ctx.min_score = vq.has_min ? (float)std::max(vq.min_score, -(double)FLT_MAX) : (vq.has_max ? 0.f : -FLT_MAX);
  ctx.max_score = vq.has_max ? (float)std::min(vq.max_score, (double)FLT_MAX) : (vq.has_min ? 0.f : FLT_MAX);
  if (!vq.has_min && !vq.has_max) {
    ctx.min_score = -FLT_MAX;
    ctx.max_score = FLT_MAX;
  }
  const int topN = req.topn + req.offset;
  std::vector<float> dis((size_t)n * topN);
  std::vector<int64_t> ids((size_t)n * topN);
  std::vector<uint8_t> bm;
  FilterBits fbits(device_);
  int total_docs;
  {
    std::unique_lock<std::shared_mutex> wl(mu_, std::defer_lock);
    std::shared_lock<std::shared_mutex> rl(mu_);
    bool need_flush = pending_n_ > 0 || scalar_staged() > 0;
    rl.unlock();
    if (need_flush) {
      wl.lock();
      if (flush_pending_locked()) return Status::Make(kIndexError, last_error());
      wl.unlock();
    }
    rl.lock();
    const int vi = vec_field(vq.name);
    qindex = vslot(vi);  // the index a swap left, held until the results are read
    if (!fidx_[vi].has_index) ctx.params.brute_force = true;  // a field without an index is searched exactly
    if (delete_num_ > 0) {
      bm.assign(del_bitmap_.begin(), del_bitmap_.begin() + (max_docid_ >> 3) + 1);
      ctx.del_bitmap = bm.data();
      ctx.bitmap_bits = max_docid_;
    }
    total_docs = doc_num();
    if (!req.filters.empty()) {  // ScalarIndexQuery (search/engine.cc:349-366, 525-580)
      const int64_t card = eval_filters(req.filters, req.filter_operator, &fbits);
      if (card < 0) return Status::Make(kIndexError, last_error());
      if (card == 0) {
        PbWriter resp;
        for (int i = 0; i < req.req_num; i++) {
          PbWriter sr, st;
          st.put_int32(1, 0);
          st.put_int32(3, 0);
          sr.put_message(5, st.out);
          sr.put_string(6, space_name_ + " no result: numeric filter return 0 result");
          resp.put_message(2, sr.out);
        }
        *pb_out = resp.out;
        return Status::OK();
      }
      ctx.filter_bits_dev = fbits.bits;
      ctx.bits_dev_words = fbits.words;
      ctx.bitmap_bits = max_docid_;
    }
  }
  const int rc = qindex->search(ctx, n, vq.value.data(), topN, dis.data(), ids.data());
  if (rc == -2 || IsKilled(req.request_id, req.partition_id)) return Status::Make(kMemoryExceeded, "");
  if (rc != 0) return Status::Make(kInvalidArgument, "faild search of query " + vq.name + ": " + last_error());

  serialize_results(req, n, topN, dis.data(), ids.data(), total_docs, pb_out);
  return Status::OK();
}

Engine::FieldSel Engine::select_fields(const std::vector<std::string>& names) {
  FieldSel sel;
  if (!names.empty()) {
    int dim;
    for (auto& nme : names) {
      if (index_of(nme, &dim))
        sel.vecs.push_back(nme);
      else if (field_idx_.count(nme))
        sel.attr.push_back(field_idx_[nme]);
    }
  } else {
    for (size_t fi = 0; fi < fields_.size(); fi++) sel.attr.push_back((int)fi);
  }
  std::sort(sel.attr.begin(), sel.attr.end(), [&](int a, int b) { return fields_[a].name < fields_[b].name; });
  return sel;
}

void Engine::serialize_results(const SearchRequestPB& req, int n, int topN, const float* dis, const int64_t* ids,
                               int total_docs, std::string* pb_out) {
  std::shared_lock<std::shared_mutex> rl(mu_);
  const FieldSel sel = select_fields(req.fields);
  PbWriter resp;
  Status okst;
  for (int i = 0; i < req.req_num && i < n; i++) {
    PbWriter sr;
    // field order on the wire follows the field numbers, like the C++ serializer
    double max_score = -DBL_MAX;
    PbWriter items;
    for (int j = req.offset; j < topN; j++) {
      int64_t docid = ids[(size_t)i * topN + j];
      if (docid < 0) continue;  // vector_manager.cc:1059
      double score = dis[(size_t)i * topN + j];
      max_score = std::max(max_score, score);
      PbWriter item;
      item.put_double(1, score);
      put_doc_fields((int)docid, sel, &item);
      items.put_message(7, item.out);
    }
    sr.put_double(2, max_score);
    PbWriter st;
    st.put_int32(1, total_docs);
    st.put_int32(3, total_docs);
    sr.put_message(5, st.out);
    sr.put_string(6, okst.ToString());
    sr.out += items.out;
    resp.put_message(2, sr.out);
  }
  *pb_out = resp.out;
}

// WeightedRanker::Parse (common/common_query_data.h:257-300)
static bool parse_ranker(const std::string& raw, size_t nvec, std::vector<double>* w, std::string* err) {
  w->assign(nvec, 1.0 / (double)nvec);
  if (raw.empty()) return true;
  *err = "weighted ranker params err: " + raw;
  JsonValue jv;
  if (!JsonParser::parse(raw, &jv) || !jv.get("type") || !jv.get("params")) return false;
  const JsonValue* arr = jv.get("params");
  if (arr->type != JsonValue::Array) return false;
  if (arr->arr.size() != nvec) {
    *err = "weighted ranker params: " + raw + ", length don't equal to " + std::to_string(nvec);
    return false;
  }
  for (size_t i = 0; i < nvec; i++) {
    if (arr->arr[i].type != JsonValue::Number) return false;
    (*w)[i] = arr->arr[i].num;
  }
  return true;
}

Status Engine::SearchMulti(const SearchRequestPB& req, std::string* pb_out) {
  const size_t nvec = req.vec_fields.size();
  std::vector<std::shared_ptr<Index>> idx(nvec);
  std::vector<int> dims(nvec);
  std::vector<char> exact(nvec, 0);  // fields without an index are searched exactly
  int n = -1;
  for (size_t j = 0; j < nvec; j++) {
    const auto& vq = req.vec_fields[j];
    idx[j] = index_ref(vq.name, &dims[j]);
    if (!idx[j]) return Status::Make(kInvalidArgument, "Query name " + vq.name + " not exist in created vector table");
    const int nj = (int)(vq.value.size() / ((size_t)dims[j] * 4));
    if (nj <= 0 || (n >= 0 && nj != n)) return Status::Make(kInvalidArgument, "Search n shouldn't less than 0!");
    n = nj;
  }
  std::vector<double> weights;
  std::string err;
  if (!parse_ranker(req.ranker, nvec, &weights, &err)) return Status::Make(kInvalidArgument, err);
  int brute = req.brute_force_search;
  if (brute == 2 && index_status_.load() != 2) brute = 1;
  if (brute == 0 && index_status_.load() != 2 && max_docid_ > 100 && !enable_realtime_ && !awaiting_training_.load())
    return Status::Make(kIndexError, space_name_ + " index not trained, brute_force_search is 0, max_docid_ = " +
                                         std::to_string(max_docid_) + ", threshold = 100");
  if (IsKilled(req.request_id, req.partition_id)) return Status::Make(kMemoryExceeded, "");
  KillScope kill(req.request_id, req.partition_id);
  SearchContext base;
  base.cancel = kill.word();
  if (!parse_retrieval_params(req.index_params, &base.params, &err)) return Status::Make(kInvalidArgument, err);
  base.params.brute_force = brute != 0;
  base.search_unindexed_tail = enable_realtime_;
  const int topN = req.topn + req.offset;
  std::vector<uint8_t> bm;
  FilterBits fbits(device_);
  int total_docs;
  {
    std::unique_lock<std::shared_mutex> wl(mu_, std::defer_lock);
    std::shared_lock<std::shared_mutex> rl(mu_);
    bool need_flush = pending_n_ > 0 || scalar_staged() > 0;
    rl.unlock();
    if (need_flush) {
      wl.lock();
      if (flush_pending_locked()) return Status::Make(kIndexError, last_error());
      wl.unlock();
    }
    rl.lock();
    for (size_t j = 0; j < nvec; j++) {
      const int vi = vec_field(req.vec_fields[j].name);
      idx[j] = vslot(vi);
      exact[j] = !fidx_[vi].has_index;
    }
    if (delete_num_ > 0) {
      bm.assign(del_bitmap_.begin(), del_bitmap_.begin() + (max_docid_ >> 3) + 1);
      base.del_bitmap = bm.data();
      base.bitmap_bits = max_docid_;
    }
    total_docs = doc_num();
    if (!req.filters.empty()) {
      const int64_t card = eval_filters(req.filters, req.filter_operator, &fbits);
      if (card < 0) return Status::Make(kIndexError, last_error());
      if (card == 0) {
        PbWriter resp;
        for (int i = 0; i < req.req_num; i++) {
          PbWriter sr, st;
          st.put_int32(1, 0);
          st.put_int32(3, 0);
          sr.put_message(5, st.out);
          sr.put_string(6, space_name_ + " no result: numeric filter return 0 result");
          resp.put_message(2, sr.out);
        }
        *pb_out = resp.out;
        return Status::OK();
      }
      base.filter_bits_dev = fbits.bits;
      base.bits_dev_words = fbits.words;
      base.bitmap_bits = max_docid_;
    }
  }
  // every field on its own, topN each (vector_manager.cc:790-852)
  std::vector<std::vector<float>> dis(nvec, std::vector<float>((size_t)n * topN));
  std::vector<std::vector<int64_t>> ids(nvec, std::vector<int64_t>((size_t)n * topN));
  for (size_t j = 0; j < nvec; j++) {
    const auto& vq = req.vec_fields[j];
    SearchContext ctx = base;
    if (exact[j]) ctx.params.brute_force = true;
    ctx.min_score = vq.has_min ? (float)std::max(vq.min_score, -(double)FLT_MAX) : (vq.has_max ? 0.f : -FLT_MAX);
    ctx.max_score = vq.has_max ? (float)std::min(vq.max_score, (double)FLT_MAX) : (vq.has_min ? 0.f : FLT_MAX);
    if (!vq.has_min && !vq.has_max) ctx.min_score = -FLT_MAX, ctx.max_score = FLT_MAX;
    std::vector<float> x((size_t)n * dims[j]);
    memcpy(x.data(), vq.value.data(), x.size() * 4);
    int rc = idx[j]->search(ctx, n, x.data(), topN, dis[j].data(), ids[j].data());
    if (rc == -2 || IsKilled(req.request_id, req.partition_id)) return Status::Make(kMemoryExceeded, "");
    if (rc != 0) return Status::Make(kInvalidArgument, "faild search of query " + vq.name + ": " + last_error());
  }
  // docid join (vector_manager.cc:900-964): a document survives when EVERY field returned it; its score is
  // the weighted sum of the per-field scores; docid order unless multi_vector_rank asks for score order
  std::vector<float> out_dis((size_t)n * topN, 0.f);
  std::vector<int64_t> out_ids((size_t)n * topN, -1);
  const bool l2 = std::atomic_load(&index_)->metric() == kMetricL2;
  for (int i = 0; i < n; i++) {
    std::map<int64_t, std::pair<int, double>> acc;  // docid -> (fields seen, score)
    for (size_t j = 0; j < nvec; j++)
      for (int r = 0; r < topN; r++) {
        const int64_t d = ids[j][(size_t)i * topN + r];
        if (d < 0) continue;
        auto& e = acc[d];
        e.first++;
        e.second += (double)((float)dis[j][(size_t)i * topN + r] * (float)weights[j]);  // float product, as the reference
      }
    std::vector<std::pair<int64_t, double>> common;
    for (auto& kv : acc)
      if (kv.second.first == (int)nvec) common.push_back({kv.first, kv.second.second});
    if (req.multi_vector_rank == 1)
      std::sort(common.begin(), common.end(), [l2](const std::pair<int64_t, double>& a, const std::pair<int64_t, double>& b) {
        return l2 ? a.second < b.second : a.second > b.second;
      });
    for (size_t r = 0; r < common.size() && r < (size_t)topN; r++) {
      out_ids[(size_t)i * topN + r] = common[r].first;
      out_dis[(size_t)i * topN + r] = (float)common[r].second;
    }
  }
  serialize_results(req, n, topN, out_dis.data(), out_ids.data(), total_docs, pb_out);
  return Status::OK();
}

void Engine::put_doc_fields(int docid, const FieldSel& sel, PbWriter* item) {
  for (int fi : sel.attr) {
    PbWriter fld;
    fld.put_string(1, fields_[fi].name);
    const std::string& val = values_[fi][docid];
    fld.put_bytes(3, val.data(), val.size());
    item->put_message(2, fld.out);
  }
  for (const auto& vn : sel.vecs) {
    int dim = 0;
    Index* ix = index_of(vn, &dim);
    std::vector<unsigned char> vbuf(ix ? ix->store().row_bytes() : 0);
    if (ix && ix->store().get_host(docid, vbuf.data()) == 0) {
      PbWriter fld;
      fld.put_string(1, vn);
      fld.put_bytes(3, vbuf.data(), vbuf.size());
      item->put_message(2, fld.out);
    }
  }
}

// Engine::Query (search/engine.cc:404-523): documents by key (by docid when partition_id > 0), or the
// first `limit` live documents that pass the scalar filters, as one SearchResult with score-less items
Status Engine::Query(const QueryRequestPB& req, std::string* pb_out) {
  if (!created_table_) return Status::Make(kInvalidArgument, space_name_ + " table not created");
  {
    // documents accepted but not yet uploaded must be visible to GetDoc-style reads: flush under the exclusive
    // lock, then serve the query under the shared one (filters, field reads and the per-document device reads
    // of put_doc_fields do not block ingest or other searches)
    std::unique_lock<std::shared_mutex> wl(mu_);
    if ((pending_n_ > 0 || scalar_staged() > 0) && flush_pending_locked()) return Status::Make(kIndexError, last_error());
  }
  std::shared_lock<std::shared_mutex> rl(mu_);
  std::vector<int> docids;
  auto deleted = [&](int d) { return ((del_bitmap_[d >> 3] >> (d & 7)) & 1) != 0; };
  if (!req.document_ids.empty()) {
    for (const auto& id : req.document_ids) {
      int docid = -1;
      if (req.partition_id > 0) {
        char* end = nullptr;
        long v = strtol(id.c_str(), &end, 10);
        if (id.empty() || *end != '\0' || v < 0 || v >= max_docid_) continue;
        docid = (int)v;
      } else {
        auto it = key2docid_.find(id);
        if (it == key2docid_.end()) continue;
        docid = it->second;
      }
      if (!deleted(docid)) docids.push_back(docid);
    }
  } else {
    const int topn = req.limit;
    if (!req.filters.empty()) {
      FilterBits fbits(device_);
      const int64_t card = eval_filters(req.filters, req.filter_operator, &fbits);
      if (card < 0) return Status::Make(kIndexError, last_error());
      if (card == 0) {
        PbWriter resp, sr, st;
        st.put_int32(1, 0);
        st.put_int32(3, 0);
        sr.put_message(5, st.out);
        sr.put_string(6, space_name_ + " no result: numeric filter return 0 result");
        resp.put_message(2, sr.out);
        *pb_out = resp.out;
        return Status::OK();
      }
      std::vector<uint8_t> fbm((size_t)fbits.words * 4);  // the words, LSB-first, are the bytes of the host layout
      if (cudaMemcpyAsync(fbm.data(), fbits.bits, fbm.size(), cudaMemcpyDeviceToHost, fbits.s.stream()) != cudaSuccess ||
          cudaStreamSynchronize(fbits.s.stream()) != cudaSuccess)
        return Status::Make(kIndexError, "filter bitmap download failed");
      int skipped = 0;
      for (int d = 0; d < max_docid_ && (int)docids.size() < topn; d++) {
        if (!((fbm[d >> 3] >> (d & 7)) & 1)) continue;
        if (skipped++ < req.offset) continue;  // ScalarIndexManager::Query drops `offset` hits first
        if (!deleted(d)) docids.push_back(d);
      }
    }
  }
  const FieldSel sel = select_fields(req.fields);
  PbWriter resp, sr, st, items;
  for (int d : docids) {
    PbWriter item;  // score 0.0: proto3 leaves it off the wire
    put_doc_fields(d, sel, &item);
    items.put_message(7, item.out);
  }
  sr.put_double(2, docids.empty() ? -DBL_MAX : 0.0);
  st.put_int32(1, (int)docids.size());
  st.put_int32(3, (int)docids.size());
  sr.put_message(5, st.out);
  sr.put_string(6, Status::OK().ToString());
  sr.out += items.out;
  resp.put_message(2, sr.out);
  *pb_out = resp.out;
  return Status::OK();
}

Status Engine::SetFieldIndexed(const std::string& field, bool indexed, const std::string& index_type,
                               const std::string& index_params) {
  if (!created_table_) return Status::Make(kIOError, "table not initialized");
  if (vec_field(field) >= 0) return indexed ? AddFieldIndex(field, index_type, index_params) : RemoveFieldIndex(field);
  std::unique_lock<std::shared_mutex> lk(mu_);
  auto it = field_idx_.find(field);
  if (it == field_idx_.end()) return Status::Make(kInvalidArgument, "field " + field + " not found");
  cudaSetDevice(device_);
  if (indexed) {  // AddFieldIndex builds the index over the documents already stored
    fields_[it->second].indexed = true;
    if (scalar_index_rebuild(it->second)) {
      fields_[it->second].indexed = false;
      return Status::Make(kIndexError, last_error());
    }
  } else {
    fields_[it->second].indexed = false;
    if (it->second < (int)sidx_.size()) sidx_[it->second].release();
  }
  return Status::OK();
}

// CreateTable's rules for the index of one vector field (vector_manager.cc:343-453), for CreateTable and for
// AddFieldIndex alike
Status Engine::create_field_index(const std::string& name, int dim, const std::string& type, const std::string& params,
                                  bool first, bool host, size_t nvec, int64_t* tt, Index** out) const {
  ModelParams mp;
  std::string err;
  if (!parse_model_params(params, type, &mp, &err)) return Status::Make(kInvalidArgument, err);
  if (first && !table_params_given_ && mp.training_threshold > *tt) *tt = mp.training_threshold;  // table.cc:143-150
  if (*tt > 0) mp.training_threshold = (int)*tt;
  mp.host_store = host;
  // BINARYIVF: the field's values are packed bits, dimension / 8 bytes (vector_manager.cc:100-130); a table with more
  // than one vector field cannot join Hamming and float scores here
  if (type == "BINARYIVF" && nvec > 1)
    return Status::Make(kNotSupported, name + ": BINARYIVF is not supported in a multi-vector table");
  Index* idx = make_index(type, dim, mp);
  if (!idx) {
    const bool known = type == "FLAT" || type == "IVFFLAT" || type == "IVFPQ" || type == "IVFPQFastScan" ||
                       type == "BINARYIVF" || type == "IVFRABITQ" || type == "VEARCH" || is_gpu_index_type(type);
    return Status::Make(!first || known ? kInvalidArgument : kNotSupported, last_error());
  }
  *out = idx;
  return Status::OK();
}

// ---- a vector field's index at run time ---------------------------------------------------------
// CreateTable's rules for the field, and the raw rows it already stores: the new index must read them as they are
Status Engine::make_field_index(int vi, const std::string& type, const std::string& params, std::shared_ptr<Index>* out,
                                int64_t* tt) {
  const std::string& name = vname(vi);
  if (type.empty()) return Status::Make(kNotSupported, name + " index type is empty");
  RawStore& st = vslot(vi)->store();
  const int row_bytes = type == "BINARYIVF" ? vdim(vi) / 8 : vdim(vi) * 4;
  if (row_bytes != st.row_bytes())
    return Status::Make(kInvalidArgument, name + ": a " + type + " index reads rows of " + std::to_string(row_bytes) +
                                              " bytes, the field stores rows of " + std::to_string(st.row_bytes()));
  // the first field follows the table's threshold as CreateTable gave it; the others take the engine's
  int64_t t = vi == 0 ? table_training_threshold_ : training_threshold_;
  Index* idx = nullptr;
  Status s = create_field_index(name, vdim(vi), type, params, vi == 0, st.on_host(), fidx_.size(), &t, &idx);
  if (!s.ok()) return s;
  out->reset(idx);
  *tt = t > 0 ? t : idx->training_threshold();
  return Status::OK();
}

void Engine::swap_field_index(int vi, std::shared_ptr<Index> nidx, const std::string& type, const std::string& params,
                              bool has_index, int64_t tt) {
  std::atomic_store(&vslot(vi), std::move(nidx));  // a search still in the old index keeps it until it returns
  FieldIndex& fx = fidx_[vi];
  fx.has_index = has_index;
  fx.changed = true;
  vtype(vi) = type;
  vparams(vi) = params;
  if (vi == 0) training_threshold_ = tt;
  bool ready = true;  // every field is trained or has no index
  for (size_t v = 0; v < fidx_.size(); v++) ready = ready && (!fidx_[v].has_index || vslot((int)v)->trained());
  // an index swapped in before the field reaches its training threshold is left as CreateTable leaves one: the
  // indexing thread trains it once the table has enough rows (BuildIndex's rule); until then its searches are exact
  if (ready) {
    index_status_.store(2);
    awaiting_training_.store(false);
  } else if (has_index && !vslot(vi)->trained()) {
    index_status_.store(0);
    awaiting_training_.store(true);
  }
}

// the build thread and RemoveFieldIndex call this; field_build_mu_ makes them one pauser at a time
bool Engine::pause_indexing() {
  bool was_running = false;
  for (;;) {
    int st = indexing_state_.load();
    if (st == 0) {
      if (indexing_state_.compare_exchange_strong(st, 4)) break;
      continue;
    }
    was_running = was_running || st == 1 || st == 2;
    indexing_state_.store(3);
    idx_cv_.notify_all();
    std::lock_guard<std::mutex> g(indexing_thread_mu_);
    if (indexing_thread_.joinable()) indexing_thread_.join();
  }
  return was_running;
}
void Engine::resume_indexing(bool was_running) {
  indexing_state_.store(0);
  if (was_running || index_status_.load() == 2) BuildIndex();
}

void Engine::join_field_build() {
  std::lock_guard<std::mutex> g(field_build_mu_);
  join_field_build_locked();
}
void Engine::join_field_build_locked() {
  if (field_build_thread_.joinable()) field_build_thread_.join();
}

Status Engine::AddFieldIndex(const std::string& field, const std::string& type, const std::string& params) {
  const int vi = vec_field(field);
  if (vi < 0) return Status::Make(kInvalidArgument, "field " + field + " not found");
  std::lock_guard<std::mutex> g(field_build_mu_);  // join, validate and spawn as one step
  join_field_build_locked();  // one build at a time
  cudaSetDevice(device_);
  std::shared_ptr<Index> nidx;
  int64_t tt = 0;
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    Status st = make_field_index(vi, type, params, &nidx, &tt);
    if (!st.ok()) return st;
    // the new index's bytes for every row stored or accepted, beside the old index's until the swap frees them
    const int64_t rows = vslot(vi)->store().size() + pending_n_;
    if (mem::limited()) {
      std::vector<mem::Charge> c;
      memory_places(&c, 0);
      nidx->charge_index_rows(rows, &c);
      if (!mem::admit(c))
        return Status::Make(kMemoryExceeded, field + ": a " + type + " index of " + std::to_string(rows) + " rows");
    }
    nidx->adopt_store(vslot(vi)->share_store());
    FieldIndex& fx = fidx_[vi];
    fx.building = nidx;
    fx.building_type = type;
    fx.building_params = params;
    fx.updated.clear();
    fx.deleted.clear();
  }
  field_build_stop_.store(false);
  field_build_thread_ = std::thread(&Engine::field_build, this, vi, nidx, tt);
  return Status::OK();
}

// Train the successor on the field's first stored rows (BuildIndex's rule), index every stored row while the field's
// current index serves searches, then, with the indexing thread stopped and the table held exclusively, index the rows
// added since, apply the updates and deletions made meanwhile and swap.
void Engine::field_build(int vi, std::shared_ptr<Index> nidx, int64_t tt) {
  cudaSetDevice(device_);
  FieldIndex& fx = fidx_[vi];
  const std::string name = vname(vi), type = fx.building_type;
  auto give_up = [&](bool log) {  // mu_ held exclusively
    if (log)
      fprintf(stderr, "gamma: building the %s index of vector field %s failed, the field keeps its index: %s\n",
              type.c_str(), name.c_str(), last_error());
    fx.building.reset();
    fx.updated.clear();
    fx.deleted.clear();
  };
  auto del_bitmap = [&](std::vector<uint8_t>* bm) {  // mu_ held
    if (delete_num_ > 0) bm->assign(del_bitmap_.begin(), del_bitmap_.begin() + (max_docid_ >> 3) + 1);
  };
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (flush_pending_locked()) return give_up(true);
  }
  // fewer rows than the training threshold: the successor replaces the index untrained, as CreateTable would leave it
  const bool train_now = nidx->store().size() >= nidx->training_threshold();
  bool failed = train_now && nidx->train() != 0;
  // rows stored while a pass runs are indexed by the next one; the last few are indexed under the exclusive lock
  for (int pass = 0; train_now && !failed && !field_build_stop_.load() && pass < 8; pass++) {
    std::vector<uint8_t> bm;
    int64_t stored;
    {
      std::shared_lock<std::shared_mutex> lk(mu_);
      del_bitmap(&bm);
      stored = nidx->store().size();
    }
    // only the rows the bitmap covers: the store grows while the pass runs
    failed = nidx->add_pending(bm.empty() ? nullptr : bm.data(), stored) != 0;
    if (nidx->store().size() - stored < 65536) break;
  }
  if (failed || field_build_stop_.load()) {
    std::unique_lock<std::shared_mutex> lk(mu_);
    return give_up(failed);
  }
  const bool was_running = pause_indexing();
  std::shared_ptr<Index> old;
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    std::vector<uint8_t> bm;
    failed = flush_pending_locked() != 0;
    if (train_now) {
      del_bitmap(&bm);
      failed = failed || nidx->add_pending(bm.empty() ? nullptr : bm.data()) != 0;
      std::vector<unsigned char> row((size_t)nidx->store().row_bytes());
      for (int64_t vid : fx.updated)  // the store holds the new row; the successor re-lists it
        failed = failed || nidx->store().get_host(vid, row.data()) || nidx->update_vector(vid, row.data());
      if (!failed && !fx.deleted.empty())
        failed = nidx->delete_vectors(fx.deleted.data(), (int64_t)fx.deleted.size()) != 0;
    }
    if (failed) {
      give_up(true);
    } else {
      old = vslot(vi);
      swap_field_index(vi, nidx, type, fx.building_params, true, tt);
      give_up(false);
    }
  }
  old.reset();  // freed here unless a search still holds it
  if (!failed) remove_index_files(name);  // the old type's file; Dump writes the new one
  resume_indexing(was_running);
}

void Engine::remove_index_files(const std::string& field) const {  // <path>/retrieval_model_index/<field>.000/
  if (path_.empty()) return;
  const std::string dir = path_ + "/retrieval_model_index/" + field + ".000";
  if (DIR* d = opendir(dir.c_str())) {
    while (dirent* e = readdir(d))
      if (strcmp(e->d_name, ".") && strcmp(e->d_name, "..")) unlink((dir + "/" + e->d_name).c_str());
    closedir(d);
  }
  rmdir(dir.c_str());
}

// The field keeps its raw store; what serves it is an index that is never trained and that every search of the field
// scans exactly (the brute-force path): FLAT under the old index's metric, or for packed binary rows a BINARYIVF index
// with the old parameters, whose brute-force path is the Hamming scan.
Status Engine::RemoveFieldIndex(const std::string& field) {
  const int vi = vec_field(field);
  if (vi < 0) return Status::Make(kInvalidArgument, "field " + field + " not found");
  std::lock_guard<std::mutex> g(field_build_mu_);  // no build starts while the index is removed
  join_field_build_locked();
  if (!fidx_[vi].has_index) return Status::OK();
  cudaSetDevice(device_);
  const bool was_running = pause_indexing();
  std::shared_ptr<Index> old;
  Status st;
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    std::shared_ptr<Index> cur = vslot(vi);
    const bool binary = cur->type() == "BINARYIVF";
    const std::string type = binary ? cur->type() : "FLAT";
    const std::string params =
        binary ? vparams(vi) : std::string("{\"metric_type\": \"") + (cur->metric() == kMetricL2 ? "L2" : "InnerProduct") + "\"}";
    ModelParams mp;
    std::string err;
    if (flush_pending_locked()) {
      st = Status::Make(kIndexError, last_error());
    } else if (!parse_model_params(params, type, &mp, &err)) {
      st = Status::Make(kInvalidArgument, err);
    } else {
      mp.host_store = cur->store().on_host();
      std::shared_ptr<Index> none(create_index(type, vdim(vi), mp, device_, 20));
      if (!none) {
        st = Status::Make(kInvalidArgument, last_error());
      } else {
        none->adopt_store(cur->share_store());
        old = cur;
        swap_field_index(vi, none, type, params, false, training_threshold_);
      }
    }
  }
  old.reset();
  if (st.ok()) remove_index_files(field);
  resume_indexing(was_running);
  return st;
}

int64_t Engine::now_ms() {
  return std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Engine::BuildIndex / Engine::Indexing (search/engine.cc:951-988, 1091-1142)
int Engine::BuildIndex() {
  if (!created_table_) return -1;
  int expected = 0;
  if (!indexing_state_.compare_exchange_strong(expected, 1)) return 0;  // already in progress
  std::lock_guard<std::mutex> g(indexing_thread_mu_);
  if (indexing_thread_.joinable()) indexing_thread_.join();
  indexing_thread_ = std::thread(&Engine::indexing_loop, this);
  return 0;
}

// Engine::RebuildIndex: only acts on a running, indexed engine; stops the indexing thread, drops the index
// structures of every vector field (the raw vectors stay) and starts over: train on the current first
// training_threshold vectors, re-add everything.  Both reference variants (build the new indexes aside, or
// drop first) end in the same state; here the old index is dropped first, so searches in between see the
// "index not trained" / brute-force rules of an un-indexed table.
int Engine::RebuildIndex(int drop_before_rebuild, int limit_cpu, int describe) {
  (void)drop_before_rebuild;
  (void)limit_cpu;
  if (!created_table_) return -1;
  std::lock_guard<std::mutex> g(field_build_mu_);  // a run-time index build ends in its swap or its failure first
  join_field_build_locked();
  if (indexing_state_.load() != 2 || index_status_.load() == 0) return 0;  // "index not running, no need to rebuild!"
  stop_indexing();
  indexing_state_.store(0);
  if (describe) return 0;
  cudaSetDevice(device_);
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (flush_pending_locked()) return -1;
  }
  for (size_t vi = 0; vi < fidx_.size(); vi++)
    if (fidx_[vi].has_index && vslot((int)vi)->reset_index()) return -1;
  index_status_.store(0);
  if (refresh_interval_ >= 0 && max_docid_ - delete_num_ >= training_threshold_) return BuildIndex();
  return 0;
}

void Engine::indexing_loop() {
  cudaSetDevice(device_);
  int expected = 1;
  if (!indexing_state_.compare_exchange_strong(expected, 2)) {
    indexing_state_.store(0);
    return;
  }
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    flush_pending_locked();
  }
  bool train_failed = false;  // e.g. fewer vectors than training_threshold; a field without an index is not trained
  for (size_t vi = 0; vi < fidx_.size(); vi++)
    train_failed = train_failed || (fidx_[vi].has_index && vslot((int)vi)->train() != 0);
  if (train_failed) {
    // e.g. fewer vectors than training_threshold: remember when, so AddOrUpdate does not spawn and join a new
    // indexing thread for every document until the threshold is reached (BuildIndex retries after a back-off)
    last_train_failure_ms_.store(now_ms());
    indexing_state_.store(0);
    idx_cv_.notify_all();
    return;
  }
  bool has_error = false;
  while (indexing_state_.load() == 2) {
    if (has_error) {
      std::this_thread::sleep_for(std::chrono::milliseconds(200));
      continue;
    }
    std::vector<uint8_t> bm;
    {
      std::unique_lock<std::shared_mutex> lk(mu_);
      if (flush_pending_locked()) has_error = true;
      if (delete_num_ > 0) bm.assign(del_bitmap_.begin(), del_bitmap_.begin() + (max_docid_ >> 3) + 1);
    }
    for (size_t vi = 0; vi < fidx_.size(); vi++)
      if (!has_error && fidx_[vi].has_index && vslot((int)vi)->add_pending(bm.empty() ? nullptr : bm.data()) != 0)
        has_error = true;
    if (!has_error) purge_indexes(bm.empty() ? nullptr : bm.data(), bm.size());
    if (!has_error) {
      index_status_.store(2);
      awaiting_training_.store(false);
    }
    // sleep refresh_interval ms, waking early on Close
    std::unique_lock<std::mutex> lk(idx_mu_);
    idx_cv_.wait_for(lk, std::chrono::milliseconds(refresh_interval_ > 0 ? refresh_interval_ : 1),
                     [this] { return indexing_state_.load() != 2; });
  }
  indexing_state_.store(0);
  idx_cv_.notify_all();
}

std::string Engine::EngineStatus() {  // search/engine.cc:1164-1176
  std::shared_lock<std::shared_mutex> lk(mu_);
  // min over the vector fields that have an index; with none, the rows every field stores
  int64_t min_indexed = -1;
  for (size_t vi = 0; vi < fidx_.size(); vi++)
    if (fidx_[vi].has_index) {
      const int64_t c = vslot((int)vi)->indexed_count();
      min_indexed = min_indexed < 0 ? c : std::min(min_indexed, c);
    }
  if (min_indexed < 0) min_indexed = created_table_ && index_ ? index_->store().size() : 0;
  char buf[256];
  snprintf(buf, sizeof buf,
           "{\"backup_status\":%d,\"doc_num\":%d,\"index_status\":%d,\"max_docid\":%d,\"min_indexed_num\":%lld}",
           backup_status_.load(), doc_num(), index_status_.load(), max_docid_ - 1, (long long)min_indexed);
  return buf;
}

std::string Engine::MemoryInfo() {  // search/engine.cc:1178-1200
  std::shared_lock<std::shared_mutex> lk(mu_);
  long long table_mem = 0;
  for (auto& col : values_)
    for (auto& v : col) table_mem += (long long)v.size() + (long long)sizeof(std::string);
  long long index_mem = index_ ? index_->index_mem_bytes() : 0;
  // raw vectors wherever they are placed: HBM, or pinned host memory (store_type "RocksDB")
  long long vec_mem = index_ ? index_->store().mem_bytes() + index_->store().host_bytes() : 0;
  for (auto& e : extra_)
    index_mem += e.index->index_mem_bytes(), vec_mem += e.index->store().mem_bytes() + e.index->store().host_bytes();
  for (auto& fx : fidx_)  // a successor being built shares the store: only its index counts
    if (fx.building) index_mem += fx.building->index_mem_bytes();
  long long field_range_mem = 0;  // the scalar indexes: device columns, string-array pools, dictionaries
  for (auto& c : sidx_) field_range_mem += c.mem_bytes();
  char buf[256];
  snprintf(buf, sizeof buf,
           "{\"bitmap_mem\":%lld,\"field_range_mem\":%lld,\"index_mem\":%lld,\"table_mem\":%lld,\"vector_mem\":%lld}",
           (long long)del_bitmap_.size(), field_range_mem, index_mem, table_mem, vec_mem);
  return buf;
}

int Engine::SetConfig(const std::string& json) {  // search/engine.cc:1764-1790
  JsonValue jv;
  if (!JsonParser::parse(json, &jv)) return -1;
  int v;
  if (jv.get_int("refresh_interval", &v)) refresh_interval_ = v;
  if (jv.get_int("slow_search_time", &v)) slow_search_time_ = v;
  bool b;
  if (jv.get_bool("enable_id_cache", &b)) enable_id_cache_ = b;
  return 0;
}
std::string Engine::GetConfig() {  // search/engine.cc:1792-1807
  char buf[256];
  snprintf(buf, sizeof buf,
           "{\"enable_id_cache\":%s,\"engine_cache_size\":0,\"refresh_interval\":%d,\"slow_search_time\":%d}",
           enable_id_cache_ ? "true" : "false", refresh_interval_, slow_search_time_);
  return buf;
}

// ---- Dump / Load (own snapshot format; byte-compatible gamma dumps are a "next" row) --------
namespace {
template <typename T>
bool rdv(std::ifstream& f, T* v) {
  return (bool)f.read(reinterpret_cast<char*>(v), sizeof(T));
}
bool rd_str(std::ifstream& f, std::string* s) {
  uint64_t n;
  if (!rdv(f, &n) || n > ((uint64_t)1 << 40)) return false;
  s->resize(n);
  return n == 0 || (bool)f.read(&(*s)[0], (std::streamsize)n);
}
// The snapshot's optional last part: the vector fields whose index AddFieldIndex / RemoveFieldIndex changed, each as
// (name, has index, type, params), then the part's byte length and kIndexRecordMagic.  A snapshot without it ends with
// the trained state, as snapshots written before the record existed do.
const char kIndexRecordMagic[8] = {'G', 'B', 'F', 'I', 'D', 'X', '0', '1'};
}  // namespace

std::string encode_index_records(const std::vector<IndexRecord>& recs) {
  std::string out;
  auto put = [&](const void* p, size_t n) { out.append(static_cast<const char*>(p), n); };
  auto put_str = [&](const std::string& v) {
    const uint64_t n = v.size();
    put(&n, 8);
    put(v.data(), v.size());
  };
  const uint32_t n = (uint32_t)recs.size();
  put(&n, 4);
  for (const IndexRecord& r : recs) {
    put_str(r.field);
    const int32_t has = r.has_index ? 1 : 0;
    put(&has, 4);
    put_str(r.type);
    put_str(r.params);
  }
  const uint64_t len = out.size();
  put(&len, 8);
  put(kIndexRecordMagic, 8);
  return out;
}

int decode_index_records(const std::string& tail, std::vector<IndexRecord>* recs, size_t* bytes) {
  recs->clear();
  *bytes = 0;
  if (tail.size() < 16 || memcmp(tail.data() + tail.size() - 8, kIndexRecordMagic, 8)) return 0;
  uint64_t len;
  memcpy(&len, tail.data() + tail.size() - 16, 8);
  if (len > tail.size() - 16) return -1;
  const char* p = tail.data() + tail.size() - 16 - len;
  const char* end = p + len;
  auto get = [&](void* v, size_t n) {
    if ((size_t)(end - p) < n) return false;
    memcpy(v, p, n);
    p += n;
    return true;
  };
  auto get_str = [&](std::string* v) {
    uint64_t n;
    if (!get(&n, 8) || n > (uint64_t)(end - p)) return false;
    v->assign(p, (size_t)n);
    p += n;
    return true;
  };
  uint32_t n;
  if (!get(&n, 4)) return -1;
  for (uint32_t i = 0; i < n; i++) {
    IndexRecord r;
    int32_t has;
    if (!get_str(&r.field) || !get(&has, 4) || !get_str(&r.type) || !get_str(&r.params)) return -1;
    r.has_index = has != 0;
    recs->push_back(std::move(r));
  }
  if (p != end) return -1;
  *bytes = (size_t)len + 16;
  return 0;
}

struct Engine::Image {
  std::string table_name;
  int32_t max_docid = 0;
  std::string head, tail;  // the .gbdump before and after the first vector field's rows
  struct Field {
    std::string name;
    int32_t dim = 0;
    Stage rows;          // rows [0, max_docid), packed
    GammaImage index;    // its index file (none when untrained or FLAT)
  };
  std::vector<Field> fields;  // the first vector field (its rows in the .gbdump), then extra_ (<table>.<field>.gbvec)
};

// mu_ held exclusively, pending rows flushed: every device copy has finished when it returns
int Engine::capture_locked(Image* img) {
  img->table_name = table_name_;
  img->max_docid = max_docid_;
  std::string& h = img->head;
  auto put = [](std::string& o, const void* p, size_t n) { o.append(static_cast<const char*>(p), n); };
  auto put_str = [&](std::string& o, const std::string& v) {
    const uint64_t n = v.size();
    put(o, &n, 8);
    o += v;
  };
  size_t bytes = 36 + del_bitmap_.size() + 8;
  for (size_t fi = 0; fi < fields_.size(); fi++)
    for (int d = 0; d < max_docid_; d++) bytes += 8 + values_[fi][d].size();
  h.reserve(bytes);
  const char magic[8] = {'G', 'B', '2', '0', '0', 'D', 'M', 'P'};
  const int32_t hdr[4] = {1, max_docid_, delete_num_, dim_};
  const uint64_t nf = fields_.size();
  put(h, magic, 8);
  put(h, hdr, sizeof hdr);
  put(h, &nf, 8);
  for (size_t fi = 0; fi < fields_.size(); fi++)
    for (int d = 0; d < max_docid_; d++) put_str(h, values_[fi][d]);
  put_str(h, std::string(del_bitmap_.begin(), del_bitmap_.end()));
  const int32_t trained = index_->trained() ? 1 : 0;
  put(img->tail, &trained, 4);
  // an index whose trained state does not persist (IVFPQFastScan) is trained again by Load
  IvfIndex* ivf = index_->persists_trained_state() ? trained_state_of(index_.get()) : nullptr;
  IVFPQIndex* pq = dynamic_cast<IVFPQIndex*>(ivf);
  if (trained && ivf) {
    std::vector<float> c((size_t)ivf->nlist() * dim_);
    if (ivf->get_centroids(c.data())) return -1;
    put(img->tail, c.data(), c.size() * 4);
    if (pq) {
      std::vector<float> p((size_t)pq->M() * pq->ksub() * pq->dsub());
      if (pq->get_pq_centroids(p.data())) return -1;
      put(img->tail, p.data(), p.size() * 4);
    }
  }
  std::vector<IndexRecord> recs;
  for (size_t vi = 0; vi < fidx_.size(); vi++)
    if (fidx_[vi].changed) recs.push_back({vname((int)vi), fidx_[vi].has_index, vtype((int)vi), vparams((int)vi)});
  if (!recs.empty()) img->tail += encode_index_records(recs);
  // the raw rows, device to device (or host to host), and every index's trained state and lists
  cudaSetDevice(device_);
  cudaStream_t st = nullptr;
  GB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  int rc = 0;
  img->fields.resize(1 + extra_.size());
  for (size_t vi = 0; rc == 0 && vi < img->fields.size(); vi++) {
    Image::Field& f = img->fields[vi];
    Index* idx = vslot((int)vi).get();
    f.name = vname((int)vi);
    f.dim = vdim((int)vi);
    rc = idx->store().capture_rows(max_docid_, &f.rows, st);
    if (rc == 0 && idx->trained()) rc = idx->capture_gamma(&f.index);
    cudaSetDevice(device_);
  }
  const cudaError_t e = cudaStreamSynchronize(st);
  cudaStreamDestroy(st);
  if (rc) return -1;
  if (e != cudaSuccess) {
    set_last_error(std::string("capture of the raw rows: ") + cudaGetErrorString(e));
    return -1;
  }
  int64_t dev = 0, host = 0;
  for (const Image::Field& f : img->fields) {
    (f.rows.on_host() ? host : dev) += (int64_t)f.rows.size();
    for (const GammaImage::Part& p : f.index.parts) (p.stage.on_host() ? host : dev) += (int64_t)p.stage.size();
  }
  note_capture_stage(dev, host);
  return 0;
}

namespace {
bool write_file(const std::string& path, const std::function<bool(FILE*)>& body) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) {
    set_last_error("cannot open " + path + ": " + strerror(errno));
    return false;
  }
  bool ok = body(f);
  ok = fclose(f) == 0 && ok;
  if (!ok) set_last_error("write error in " + path);
  return ok;
}
}  // namespace

// Engine::Dump's files (search/engine.cc:1202-1247): <dir>/<table>.gbdump, <dir>/<table>.<field>.gbvec for every further
// vector field, each index in gamma's format (IndexModel::Dump via VectorManager::Dump, vector_manager.cc:1155-1170):
// <dir>/<vector name>.000/{ivfflat,ivfpq}.index, or this engine's own file of a quantised type (gb_ivfpqfs,
// gb_ivfrabitq, gb_vearch, gb_binaryivf.index), none for FLAT; dump.done last
int Engine::write_image(const Image& img, const std::string& dir) {
  if (mkdir(dir.c_str(), 0755) && errno != EEXIST) {
    set_last_error("cannot create " + dir + ": " + strerror(errno));
    return -1;
  }
  const Image::Field& first = img.fields[0];
  if (!write_file(dir + "/" + img.table_name + ".gbdump", [&](FILE* f) {
        return fwrite(img.head.data(), 1, img.head.size(), f) == img.head.size() &&
               first.rows.write(f, 0, first.rows.size()) && fwrite(img.tail.data(), 1, img.tail.size(), f) == img.tail.size();
      }))
    return -1;
  if (write_gamma_image(first.index, dir, first.name + ".000")) return -1;
  for (size_t vi = 1; vi < img.fields.size(); vi++) {
    const Image::Field& e = img.fields[vi];
    if (!write_file(dir + "/" + img.table_name + "." + e.name + ".gbvec", [&](FILE* f) {
          const int32_t hdr[2] = {img.max_docid, e.dim};
          return fwrite(hdr, sizeof hdr, 1, f) == 1 && e.rows.write(f, 0, e.rows.size());
        }))
      return -1;
    if (write_gamma_image(e.index, dir, e.name + ".000")) return -1;
  }
  return write_file(dir + "/dump.done", [](FILE* f) { return fputs("ok", f) >= 0; }) ? 0 : -1;
}

// Engine::Dump (search/engine.cc:1202-1247) into <path>/retrieval_model_index: searches and writes wait for the capture
// only, not for the files
int Engine::Dump() {
  if (!created_table_) return -1;
  join_field_build();  // a run-time index build ends in its swap or its failure first
  std::lock_guard<std::mutex> dg(dump_mu_);
  cudaSetDevice(device_);
  Image img;
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (flush_pending_locked() || capture_locked(&img)) return -1;
  }
  mkdir(path_.c_str(), 0755);
  return write_image(img, path_ + "/retrieval_model_index");
}

namespace {
std::atomic<int> g_backup_hold{0};

int remove_tree(const std::string& dir) {
  return nftw(
      dir.c_str(), [](const char* p, const struct stat*, int, struct FTW*) { return remove(p); }, 16, FTW_DEPTH | FTW_PHYS);
}
// the finished backup at tmp takes dst's place: swapped in one step where the file system can, else by two renames;
// either way dst is never a partial backup
int replace_dir(const std::string& tmp, const std::string& dst) {
  struct stat sb;
  if (stat(dst.c_str(), &sb) != 0) return rename(tmp.c_str(), dst.c_str());  // the first backup
  if (renameat2(AT_FDCWD, tmp.c_str(), AT_FDCWD, dst.c_str(), RENAME_EXCHANGE) == 0) return remove_tree(tmp) ? -1 : 0;
  const std::string old = dst + ".old";
  remove_tree(old);
  if (rename(dst.c_str(), old.c_str())) return -1;
  if (rename(tmp.c_str(), dst.c_str())) {
    const int why = errno;
    rename(old.c_str(), dst.c_str());
    errno = why;
    return -1;
  }
  return remove_tree(old) ? -1 : 0;
}
}  // namespace

int backup_hold(int op) {
  if (op == 1) g_backup_hold = 1;
  if (op == 0) g_backup_hold = 0;
  return g_backup_hold.load();
}

Status Engine::Backup(int command) {
  int idle = 0;
  if (!backup_status_.compare_exchange_strong(idle, 1)) return Status::Make(kIOError, "backup is in progress, wait done");
  struct Idle {
    std::atomic<int>& s;
    ~Idle() { s = 0; }
  } idle_at_exit{backup_status_};
  if (command != 0) return Status::OK();  // BackupThread acts on "create" only
  if (path_.empty()) return Status::Make(kInvalidArgument, "backup needs the engine's path, and Init was given none");
  if (!created_table_) return Status::Make(kInvalidArgument, "backup of an engine without a table");
  join_field_build();
  cudaSetDevice(device_);
  Image img;
  {
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (flush_pending_locked() || capture_locked(&img)) return Status::Make(kIOError, std::string("backup capture: ") + last_error());
  }
  int armed = 1;
  if (g_backup_hold.compare_exchange_strong(armed, 2))
    while (g_backup_hold.load() == 2) std::this_thread::sleep_for(std::chrono::milliseconds(1));
  const std::string root = path_ + "/backup", dst = root + "/retrieval_model_index", tmp = dst + ".tmp";
  mkdir(path_.c_str(), 0755);
  mkdir(root.c_str(), 0755);
  remove_tree(tmp);  // left by a process that died during a backup
  if (mkdir(tmp.c_str(), 0755)) return Status::Make(kIOError, "backup: cannot create " + tmp + ": " + strerror(errno));
  if (write_image(img, tmp)) {
    const std::string why = last_error();
    remove_tree(tmp);
    return Status::Make(kIOError, "backup: " + why);
  }
  if (replace_dir(tmp, dst)) {
    const std::string why = strerror(errno);
    remove_tree(tmp);
    return Status::Make(kIOError, "backup: cannot move " + tmp + " to " + dst + ": " + why);
  }
  return Status::OK();
}

// Engine::Load (search/engine.cc:1278-1400): restore the newest complete dump, then let the
// indexing thread re-add the vectors (the lists are a deterministic function of the stored
// vectors and the trained state).
int Engine::Load() {
  if (!created_table_) return -1;
  cudaSetDevice(device_);
  std::string dir = path_ + "/retrieval_model_index";
  std::ifstream done(dir + "/dump.done");
  if (!done) return 0;  // nothing to load
  std::ifstream f(dir + "/" + table_name_ + ".gbdump", std::ios::binary);
  if (!f) return -1;
  char magic[8];
  int32_t ver, maxd, deln, dim;
  uint64_t nf;
  if (!f.read(magic, 8) || memcmp(magic, "GB200DMP", 8) || !rdv(f, &ver) || ver != 1 || !rdv(f, &maxd) || !rdv(f, &deln) ||
      !rdv(f, &dim) || dim != dim_ || !rdv(f, &nf) || nf != fields_.size())
    return -1;
  std::unique_lock<std::shared_mutex> lk(mu_);
  if (max_docid_ != 0) return -1;
  {  // the indexes AddFieldIndex / RemoveFieldIndex left, re-created before their rows and trained state are read
    const std::streampos at = f.tellg();
    f.seekg(0, std::ios::end);
    const int64_t size = (int64_t)f.tellg();
    std::string tail((size_t)std::min<int64_t>(size, 1 << 20), '\0');
    f.seekg(size - (int64_t)tail.size());
    std::vector<IndexRecord> recs;
    size_t rec_bytes = 0;
    if (!f.read(&tail[0], (std::streamsize)tail.size()) || decode_index_records(tail, &recs, &rec_bytes)) return -1;
    for (const IndexRecord& r : recs) {
      const int vi = vec_field(r.field);
      if (vi < 0) return -1;
      std::shared_ptr<Index> idx;
      int64_t tt = training_threshold_;
      if (r.has_index) {
        Status st = make_field_index(vi, r.type, r.params, &idx, &tt);
        if (!st.ok()) {
          fprintf(stderr, "gamma: the recorded index of vector field %s is refused: %s\n", r.field.c_str(), st.msg.c_str());
          return -1;
        }
      } else {
        ModelParams mp;
        std::string err;
        if (!parse_model_params(r.params, r.type, &mp, &err)) return -1;
        mp.host_store = vslot(vi)->store().on_host();
        idx.reset(create_index(r.type, vdim(vi), mp, device_, 20));
        if (!idx) return -1;
      }
      swap_field_index(vi, idx, r.type, r.params, r.has_index, tt);
    }
    index_status_.store(0);  // set by the indexing thread once the rows are indexed, as for a table never changed
    awaiting_training_.store(false);
    f.clear();
    f.seekg(at);
  }
  for (size_t fi = 0; fi < fields_.size(); fi++) {
    values_[fi].resize(maxd);
    for (int d = 0; d < maxd; d++)
      if (!rd_str(f, &values_[fi][d])) return -1;
  }
  std::string bm;
  if (!rd_str(f, &bm)) return -1;
  del_bitmap_.assign(bm.begin(), bm.end());
  del_bitmap_.resize(std::max<size_t>(del_bitmap_.size(), (size_t)(maxd >> 3) + 4096), 0);
  std::vector<unsigned char> rows((size_t)maxd * vbytes_);
  if (maxd && !f.read(reinterpret_cast<char*>(rows.data()), (std::streamsize)rows.size())) return -1;
  int32_t trained;
  if (!rdv(f, &trained)) return -1;
  for (size_t fi = 0; fi < fields_.size(); fi++)
    if (fields_[fi].indexed && scalar_index_rebuild((int)fi)) return -1;
  keys_.resize(maxd);
  int idf = field_idx_["_id"];
  for (int d = 0; d < maxd; d++) {
    keys_[d] = values_[idf][d];
    if (!((del_bitmap_[d >> 3] >> (d & 7)) & 1)) key2docid_[keys_[d]] = d;
  }
  max_docid_ = maxd;
  delete_num_ = deln;
  if (maxd && index_->add_vectors(rows.data(), maxd)) return -1;
  for (auto& e : extra_) {
    std::ifstream ef(dir + "/" + table_name_ + "." + e.name + ".gbvec", std::ios::binary);
    int32_t en = 0, ed = 0;
    if (!ef || !rdv(ef, &en) || !rdv(ef, &ed) || en != maxd || ed != e.dim) return -1;
    std::vector<float> erows((size_t)maxd * e.dim);
    if (maxd && !ef.read(reinterpret_cast<char*>(erows.data()), (std::streamsize)(erows.size() * 4))) return -1;
    if (maxd && e.index->add_vectors(erows.data(), maxd)) return -1;
    int64_t eload = 0;
    if (e.index->load_gamma(dir, e.name + ".000", &eload))  // trained state + lists; absent or refused: trained again later
      fprintf(stderr, "gamma: index file of vector field %s not loaded, the index is built again: %s\n", e.name.c_str(),
              last_error());
  }
  IvfIndex* ivf = index_->persists_trained_state() ? trained_state_of(index_.get()) : nullptr;
  IVFPQIndex* pq = dynamic_cast<IVFPQIndex*>(ivf);
  if (trained && ivf) {
    std::vector<float> c((size_t)ivf->nlist() * dim_);
    if (!f.read(reinterpret_cast<char*>(c.data()), (std::streamsize)(c.size() * 4))) return -1;
    if (ivf->set_centroids(c.data(), ivf->nlist())) return -1;
    if (pq) {
      std::vector<float> p((size_t)pq->M() * pq->ksub() * pq->dsub());
      if (!f.read(reinterpret_cast<char*>(p.data()), (std::streamsize)(p.size() * 4))) return -1;
      if (pq->set_pq_centroids(p.data())) return -1;
    }
  }
  if (trained && ivf) {
    // IndexModel::Load: take the inverted lists from the index file when it matches this table; a
    // missing or refused file only means the indexing thread re-adds the vectors itself
    int64_t load_num = 0;
    if (index_->load_gamma(dir, vec_name_ + ".000", &load_num) == 0 && load_num > 0) index_status_.store(2);
  } else if (trained && !index_->persists_trained_state()) {
    // the quantised types keep their trained state in their own index file only: a file that loads leaves the index
    // trained and searchable at once; without one, the indexing thread trains it again from the raw rows
    int64_t load_num = 0;
    if (index_->load_gamma(dir, vec_name_ + ".000", &load_num))
      fprintf(stderr, "gamma: index file of vector field %s refused, the index is trained again: %s\n", vec_name_.c_str(),
              last_error());
    else if (!index_->trained())
      fprintf(stderr, "gamma: no index file for vector field %s, the index is trained again\n", vec_name_.c_str());
    else if (load_num > 0)
      index_status_.store(2);
  }
  bool changed = false;
  for (auto& fx : fidx_) changed = changed || fx.changed;
  lk.unlock();
  if (trained || changed) BuildIndex();  // train() is a no-op on a trained index; the loop adds what the file did not cover
  return 0;
}

}  // namespace gb
