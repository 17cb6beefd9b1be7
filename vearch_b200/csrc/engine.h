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
  const std::string& space_name() const { return space_name_; }
  void quiesce();  // stop the indexing thread (also from an atexit hook for engines never Closed)
  // Engine::AddFieldIndex / RemoveFieldIndex (search/engine.cc:1471-1600): build the field's device columns over the
  // documents already stored, or free them
  Status SetFieldIndexed(const std::string& field, bool indexed);
  // whether a Search / Query request of `bytes` fits the memory limit (mem_ledger.h) on every place the table uses
  bool request_admitted(int64_t bytes) const;

  // cooperative cancellation (c_api/api_data/request_context.h:51-88)
  static void SetKill(const std::string& request_id, int partition_id, int reason);
  static void ClearKill(const std::string& request_id, int partition_id);
  static bool IsKilled(const std::string& request_id, int partition_id);

 private:
  int flush_pending_locked();
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
  std::unique_ptr<Index> index_;
  // rows accepted by AddOrUpdate, not yet uploaded to HBM: vbytes_ bytes each (d fp32 values, or BINARYIVF's d / 8 bytes)
  std::vector<unsigned char> pending_;
  size_t vbytes_ = 0;
  int pending_n_ = 0;
  // further vector fields of a multi-vector table (vector_manager.cc:343-453: one raw vector + one index
  // per field).  The first field keeps the members above; every document carries all of them.
  struct VecField {
    std::string name, index_type, index_params;
    int dim = 0;
    std::unique_ptr<Index> index;
    std::vector<float> pending;
  };
  std::vector<VecField> extra_;
  Index* index_of(const std::string& vec_name, int* dim);  // nullptr: no such vector field

  std::vector<uint8_t> del_bitmap_;
  // RealTimeMemData::CompactIfNeed for every vector field's index: lists that are 30 % dead are rewritten without the
  // entries that updates tombstoned and `bitmap` marks deleted.  A failure is logged and leaves the index as it was.
  void purge_indexes(const uint8_t* bitmap, size_t bytes);
  int max_docid_ = 0, delete_num_ = 0;
  int64_t training_threshold_ = 0;  // the index's clamp can pass 2^31 rows (256 * nlist)
  int refresh_interval_ = 1000;
  bool enable_id_cache_ = false, enable_realtime_ = false;
  int slow_search_time_ = 0;

  static int64_t now_ms();
  static constexpr int64_t kTrainRetryMs = 1000;
  std::atomic<int64_t> last_train_failure_ms_{-(int64_t)1 << 40};
  std::atomic<int> index_status_{0};    // IndexStatus: 0 UNINDEXED, 1 INDEXING, 2 INDEXED
  std::atomic<int> indexing_state_{0};  // IndexingState: 0 IDLE, 1 STARTING, 2 RUNNING, 3 STOPPING
  std::thread indexing_thread_;
  std::mutex idx_mu_;
  std::condition_variable idx_cv_;
  mutable std::shared_mutex mu_;  // table state: searches shared, writes exclusive
};

}  // namespace gb
