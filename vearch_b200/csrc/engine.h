// vearch::Engine re-implemented for the GPU hot path (search/engine.{h,cc} +
// vector/vector_manager.{h,cc} reduced to what the vector path needs): docid allocation,
// `_id` <-> docid map, in-memory field table, deletion bitmap, indexing state machine and
// thread, status JSON.  One vector field per table (multi-vector ranking is a "next" row).
#pragma once
#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "index.h"
#include "mem_ledger.h"
#include "scalar_index.h"

namespace gb {
struct PbWriter;

struct Status {  // util/status.h
  int code = 0;  // vearch::status::Code (idl/fbs/status.fbs)
  std::string msg;
  bool ok() const { return code == 0; }
  std::string ToString() const;
  static Status OK() { return Status(); }
  static Status Make(int code, const std::string& msg) {
    Status s;
    s.code = code;
    s.msg = msg;
    return s;
  }
};
enum StatusCode {
  kOk = 0, kNotFound = 1, kIndexError = 2, kNotSupported = 3, kInvalidArgument = 4, kIOError = 5, kBusy = 6,
  kTimedOut = 7, kMemoryExceeded = 8, kCanceled = 9
};

// RequestConcurrentController (search/engine.h:197-222, search/engine.cc:47-119): process-wide admission of
// Search requests.  Acquire adds req_num to the in-flight count and admits the request while the count BEFORE the
// add is below the threshold ((min(threads-max, pid_max, max_map_count/2) * 0.5) / (host threads + 1), the
// reference's rule with omp_get_max_threads() read as the host's hardware threads); a refused request still holds
// its count until Release, exactly as the reference's call sites do (engine.cc:253-258).
class RequestConcurrentController {
 public:
  static RequestConcurrentController& GetInstance();
  bool Acquire(int req_num);
  void Release(int req_num);
  int threshold() const { return concurrent_threshold_; }
  int in_flight() const { return cur_concurrent_num_.load(); }
  void set_threshold(int t);  // test hook (gb_debug_concurrency); <= 0 restores the system-derived value

 private:
  RequestConcurrentController();
  int system_threshold_ = 0, concurrent_threshold_ = 0, max_threads_ = 0;
  std::atomic<int> cur_concurrent_num_{0};
};

enum DataType { DT_INT = 0, DT_LONG, DT_FLOAT, DT_DOUBLE, DT_STRING, DT_VECTOR, DT_BOOL, DT_DATE, DT_STRINGARRAY };

struct DocField {
  std::string name;
  std::string value;
  int data_type = DT_STRING;
};

struct SearchRequestPB {  // c_api/api_data/request.{h,cc}
  std::string request_id;
  int partition_id = 0;
  int req_num = 0;
  int topn = 0;
  int brute_force_search = 0;
  struct VecQuery {
    std::string name, value, index_type;
    double min_score = 0, max_score = 0;
    bool has_min = false, has_max = false;
  };
  std::vector<VecQuery> vec_fields;
  std::vector<std::string> fields;
  // RangeFilter / TermFilter (router_grpc.proto:109-122): a term filter is a range filter that only
  // carries lower_value (search/engine.cc:551-559)
  struct Filter {
    std::string field, lower, upper;
    bool include_lower = false, include_upper = false, is_term = false;
    int is_union = 0;  // FilterOperator: 0 And, 1 Or, 2 Not (table/scalar_index_utils.h:31)
  };
  std::vector<Filter> filters;
  int filter_operator = 0;  // SearchRequest.operator: how the filters combine
  int n_range_filters = 0, n_term_filters = 0;
  std::string index_params;
  int multi_vector_rank = 0;
  std::string ranker;  // WeightedRanker JSON {"type": ..., "params": [w0, w1, ...]} (common_query_data.h:251-300)
  bool l2_sqrt = false;
  bool trace = false;
  int offset = 0;
  bool parse(const uint8_t* data, size_t len);
};

struct QueryRequestPB {  // vearchpb.QueryRequest (router_grpc.proto:147-166), c_api/api_data/query_request.cc
  std::vector<std::string> document_ids;
  int partition_id = 0;
  std::vector<SearchRequestPB::Filter> filters;
  int filter_operator = 0;
  std::vector<std::string> fields;
  int limit = 0, offset = 0;
  bool parse(const uint8_t* data, size_t len);
};

// One vector field's index as AddFieldIndex / RemoveFieldIndex left it, as Dump records it at the end of the snapshot
struct IndexRecord {
  std::string field;
  bool has_index = true;
  std::string type, params;
};
std::string encode_index_records(const std::vector<IndexRecord>& recs);
// the records at the end of a snapshot's last bytes `tail` (none when it does not end with them), and in *bytes their
// length; -1: a record that does not parse
int decode_index_records(const std::string& tail, std::vector<IndexRecord>* recs, size_t* bytes);
// test hook (gb_debug_backup_hold): op 1 makes the next Backup wait between its capture and its write, 0 lets it go
// on; returns the state, 0 off, 1 set, 2 a Backup is waiting (op -1 only reads it)
int backup_hold(int op);

class Engine {
 public:
  // devices: Init's "devices" (empty: one device); a GPU_IVFPQ / GPU_IVFFLAT field is sharded over two or more, every
  // other index lives on device, which is devices[0] when they are given
  Engine(const std::string& path, const std::string& space_name, int device, const std::vector<int>& devices = {});
  ~Engine();

  Status CreateTable(const uint8_t* fb, size_t len);
  int AddOrUpdate(const uint8_t* fb, size_t len);
  int Delete(const std::string& key);
  int GetDocByKey(const std::string& key, std::string* fb_out);
  int GetDocByDocid(int docid, bool next, std::string* fb_out);
  Status Search(const SearchRequestPB& req, std::string* pb_out);
  Status Query(const QueryRequestPB& req, std::string* pb_out);  // search/engine.cc:404-523
  int BuildIndex();
  int RebuildIndex(int drop_before_rebuild, int limit_cpu, int describe);  // search/engine.cc:991-1089
  std::string EngineStatus();
  std::string MemoryInfo();
  int SetConfig(const std::string& json);
  std::string GetConfig();
  int Dump();
  int Load();
  // Engine::Backup (search/engine.cc:1431-1470).  0 ("create"): the state captured as Dump captures it, written into
  // <path>/backup/retrieval_model_index, which a backup replaces only once complete.  1 ("restore"): nothing to do (the
  // server places the files and calls Load).  A second Backup while one runs: kIOError.
  Status Backup(int command);
  const std::string& space_name() const { return space_name_; }
  void quiesce();  // stop the indexing thread (also from an atexit hook for engines never Closed)
  // Engine::AddFieldIndex / RemoveFieldIndex (search/engine.cc:1471-1600): for a scalar field, build the field's device
  // columns over the documents already stored, or free them; for a vector field, AddFieldIndex / RemoveFieldIndex below
  Status SetFieldIndexed(const std::string& field, bool indexed, const std::string& index_type = "",
                         const std::string& index_params = "");
  // A vector field's index at run time (vector_manager.cc:217-317).  AddFieldIndex validates `type` and `params` as
  // CreateTable does, creates the index over the field's raw store and returns; a build thread trains and fills it from
  // the stored rows while searches keep using the field's current index, then swaps it in.  RemoveFieldIndex drops the
  // field's index and its files; the field is then searched exactly, as brute-force searches are.
  Status AddFieldIndex(const std::string& field, const std::string& type, const std::string& params);
  Status RemoveFieldIndex(const std::string& field);
  // whether a Search / Query request of `bytes` fits the memory limit (mem_ledger.h) on every place the table uses
  bool request_admitted(int64_t bytes) const;

  // cooperative cancellation (c_api/api_data/request_context.h:51-88)
  static void SetKill(const std::string& request_id, int partition_id, int reason);
  static void ClearKill(const std::string& request_id, int partition_id);
  static bool IsKilled(const std::string& request_id, int partition_id);
  // the registry of running searches' cancel words (SetKill sets the words registered under its pair)
  static void RegisterCancel(const std::string& request_id, int partition_id, CancelWord* c);
  static void UnregisterCancel(const std::string& request_id, int partition_id, CancelWord* c);
  // a search's cancel word, registered for its lifetime (none for a request without an id); taken from a pool of
  // words of finished searches
  struct KillScope {
    std::string rid;
    int pid;
    CancelWord* c = nullptr;
    KillScope(const std::string& request_id, int partition_id);
    ~KillScope();
    const uint32_t* word() const { return c && c->device_readable ? c->w : nullptr; }
  };

 private:
  int flush_pending_locked();
  // Dump and Backup (DESIGN.md §8, backup and snapshots): the table's state is captured under the exclusive lock into
  // an image, device copies into a stage (stage.h) plus the host table, and written to `dir` after the lock is released
  struct Image;
  int capture_locked(Image* img);
  static int write_image(const Image& img, const std::string& dir);
  std::mutex dump_mu_;                  // one Dump writes retrieval_model_index at a time
  std::atomic<int> backup_status_{0};  // 1 while a Backup runs (GetEngineStatus's backup_status)
  void indexing_loop();
  void serialize_doc(int docid, bool with_docid, std::string* out);
  int doc_num() const { return max_docid_ - delete_num_; }
  // whether the vector fields may grow to n_total rows under the memory limit: the stores' growth and the index bytes
  // of the rows it makes room for
  bool rows_admitted(int64_t n_total);
  // a charge of `bytes` on every place the table keeps memory: its devices, and the host when a field is stored there
  void memory_places(std::vector<mem::Charge>* out, int64_t bytes) const;

  std::string path_, space_name_;
  int device_;
  std::vector<int> devices_;
  Index* make_index(const std::string& type, int dim, const ModelParams& mp) const;
  bool created_table_ = false;

  // table (table/table.{h,cc} reduced to an in-memory column store)
  std::string table_name_;
  struct FieldDef {
    std::string name;
    int data_type;
    bool indexed = false;  // FieldInfo.is_index: only indexed fields can be filtered on
  };
  // ScalarIndexManager::Search (table/scalar_index_manager.cc:294-345, 588-651) on the device columns, with the table
  // held shared: the LSB-first bitmap of the docids that pass, as uint32 words on device_ in `bits` (the request owns
  // it); returns the cardinality (0: "no result"), -1 on a CUDA error (last_error)
  struct FilterBits;
  int64_t eval_filters(const std::vector<SearchRequestPB::Filter>& filters, int op, FilterBits* bits) const;
  struct FieldSel {
    std::vector<int> attr;           // table fields, in name order (std::map order of the reference)
    std::vector<std::string> vecs;   // vector fields asked for by name
  };
  FieldSel select_fields(const std::vector<std::string>& names);  // requested ones, or every table field
  void put_doc_fields(int docid, const FieldSel& sel, PbWriter* item);
  // Response::Serialize (response.cc:89-162) for n queries x topN (score, docid) slots, -1 = empty
  void serialize_results(const SearchRequestPB& req, int n, int topN, const float* dis, const int64_t* ids, int total_docs,
                         std::string* pb_out);
  // VectorManager::Search with several vector fields (vector_manager.cc:747, 900-964)
  Status SearchMulti(const SearchRequestPB& req, std::string* pb_out);
  std::vector<FieldDef> fields_;
  std::unordered_map<std::string, int> field_idx_;
  std::vector<std::vector<std::string>> values_;  // [field][docid]
  // Scalar indexes of the fields created with is_index (table/scalar_index_manager.cc: one index per field): device
  // columns on device_ (scalar_index.h).  AddOrUpdate stages values; flush_pending_locked applies them; Load and
  // AddFieldIndex build a field in bulk.  Changed only under the EXCLUSIVE table lock, evaluated under the SHARED one.
  std::vector<ScalarColumn> sidx_;  // [field]
  // docid's value of field fi is now `value` (old: the value it replaces, nullptr for a new document)
  void scalar_index_put(int fi, int docid, const std::string& value, const std::string* old);
  int scalar_index_rebuild(int fi);
  int scalar_flush_locked();  // apply what AddOrUpdate staged; re-pack string-array pools that are half dead
  int64_t scalar_staged() const;  // the most values any field has staged
  static constexpr int kScalarFlushRows = 8192;  // staged values of one field that trigger a flush from AddOrUpdate
  std::unordered_map<std::string, int> key2docid_;
  std::vector<std::string> keys_;  // docid -> _id

  // vector field
  std::string vec_name_, index_type_, index_params_;
  int dim_ = 0;
  // Searches take the index they search by atomic load (index_ref) and hold it until their results are read, so a swap
  // under the exclusive lock never frees an index a search is in; every other use holds mu_
  std::shared_ptr<Index> index_;
  // rows accepted by AddOrUpdate, not yet uploaded to HBM: vbytes_ bytes each (d fp32 values, or BINARYIVF's d / 8 bytes)
  std::vector<unsigned char> pending_;
  size_t vbytes_ = 0;
  int pending_n_ = 0;
  // further vector fields of a multi-vector table (vector_manager.cc:343-453: one raw vector + one index
  // per field).  The first field keeps the members above; every document carries all of them.
  struct VecField {
    std::string name, index_type, index_params;
    int dim = 0;
    std::shared_ptr<Index> index;
    std::vector<float> pending;
  };
  std::vector<VecField> extra_;
  Index* index_of(const std::string& vec_name, int* dim);  // nullptr: no such vector field
  std::shared_ptr<Index> index_ref(const std::string& vec_name, int* dim);  // index_of for a search, without mu_

  // Run-time index changes (AddFieldIndex / RemoveFieldIndex) of vector field vi: 0 the first, 1 + i extra_[i]
  struct FieldIndex {
    bool has_index = true;  // false after RemoveFieldIndex: a FLAT index over the raw store serves the field
    bool changed = false;   // type or params differ from CreateTable's: the snapshot records them
    std::shared_ptr<Index> building;  // the successor being trained and filled, sharing the field's raw store
    std::string building_type, building_params;
    std::vector<int64_t> updated, deleted;  // docids updated or deleted during the build, applied to it before the swap
  };
  std::vector<FieldIndex> fidx_;
  int vec_field(const std::string& name) const;  // vi, -1: not a vector field
  std::shared_ptr<Index>& vslot(int vi) { return vi == 0 ? index_ : extra_[vi - 1].index; }
  std::string& vtype(int vi) { return vi == 0 ? index_type_ : extra_[vi - 1].index_type; }
  std::string& vparams(int vi) { return vi == 0 ? index_params_ : extra_[vi - 1].index_params; }
  const std::string& vname(int vi) const { return vi == 0 ? vec_name_ : extra_[vi - 1].name; }
  int vdim(int vi) const { return vi == 0 ? dim_ : extra_[vi - 1].dim; }
  // CreateTable's rules for the index of one vector field: parse, training threshold, store placement, BINARYIVF only
  // alone, creation.  first: the table's first vector field, whose threshold follows its type when the table gave none
  // (*tt in: the threshold so far, out: the one the field keeps); every other field takes *tt as it is
  Status create_field_index(const std::string& name, int dim, const std::string& type, const std::string& params,
                            bool first, bool host, size_t nvec, int64_t* tt, Index** out) const;
  // an index of `type` / `params` for vector field vi, validated as CreateTable validates the field's; *tt: the
  // training threshold the engine keeps for it
  Status make_field_index(int vi, const std::string& type, const std::string& params, std::shared_ptr<Index>* out,
                          int64_t* tt);
  // put `nidx` in vector field vi's slot (mu_ held exclusively); the old index is freed once no search holds it
  void swap_field_index(int vi, std::shared_ptr<Index> nidx, const std::string& type, const std::string& params,
                        bool has_index, int64_t tt);
  void field_build(int vi, std::shared_ptr<Index> nidx, int64_t tt);  // the build thread's work
  void join_field_build();
  void join_field_build_locked();  // field_build_mu_ held
  void remove_index_files(const std::string& field) const;
  // stop the indexing thread and keep it from being started until resume_indexing
  bool pause_indexing();
  void resume_indexing(bool was_running);
  void stop_indexing();
  // guards field_build_thread_; AddFieldIndex, RemoveFieldIndex and RebuildIndex hold it throughout
  std::mutex field_build_mu_;
  std::thread field_build_thread_;
  // a field's index was swapped in untrained (below its training threshold): searches are exact until it trains
  std::atomic<bool> awaiting_training_{false};
  std::atomic<bool> field_build_stop_{false};
  int64_t table_training_threshold_ = 0;  // the table's own training_threshold, 0 if it has none

  std::vector<uint8_t> del_bitmap_;
  // RealTimeMemData::CompactIfNeed for every vector field's index: lists that are 30 % dead are rewritten without the
  // entries that updates tombstoned and `bitmap` marks deleted.  A failure is logged and leaves the index as it was.
  void purge_indexes(const uint8_t* bitmap, size_t bytes);
  int max_docid_ = 0, delete_num_ = 0;
  int64_t training_threshold_ = 0;  // the index's clamp can pass 2^31 rows (256 * nlist)
  bool table_params_given_ = false;  // the table carried index params (table.cc:143-150)
  int refresh_interval_ = 1000;
  bool enable_id_cache_ = false, enable_realtime_ = false;
  int slow_search_time_ = 0;

  static int64_t now_ms();
  static constexpr int64_t kTrainRetryMs = 1000;
  std::atomic<int64_t> last_train_failure_ms_{-(int64_t)1 << 40};
  std::atomic<int> index_status_{0};    // IndexStatus: 0 UNINDEXED, 1 INDEXING, 2 INDEXED
  std::atomic<int> indexing_state_{0};  // IndexingState: 0 IDLE, 1 STARTING, 2 RUNNING, 3 STOPPING, 4 PAUSED
  std::mutex indexing_thread_mu_;  // guards indexing_thread_ (started by BuildIndex, joined by whoever stops it)
  std::thread indexing_thread_;
  std::mutex idx_mu_;
  std::condition_variable idx_cv_;
  mutable std::shared_mutex mu_;  // table state: searches shared, writes exclusive
};

}  // namespace gb
