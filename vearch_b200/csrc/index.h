// Host side of the hot path: device-resident raw vectors, inverted lists, and the three index
// models, mirroring the reference's IndexModel plug-in interface
// (index/index_model.h:229-335: Init / Indexing / Add / Search, RetrievalContext,
// RetrievalParameters) so that the engine above it (engine.cc) reads like search/engine.cc +
// vector/vector_manager.cc.  No CPU compute path exists here: every Search/Train/Add call runs
// CUDA kernels and fails if the device is unavailable.
#pragma once
#include <stdio.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <memory>
#include <atomic>
#include <mutex>
#include <thread>
#include <shared_mutex>
#include <string>
#include <vector>

#include "kernels.h"
#include "mem_ledger.h"

namespace gb {

void set_last_error(const std::string& msg);
const char* last_error();
#define GB_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess) {                                                                      \
      ::gb::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(e__) + " @" __FILE__ ":" + \
                           std::to_string(__LINE__));                                              \
      return -1;                                                                                   \
    }                                                                                              \
  } while (0)

// Stream-ordered scratch allocations released when the object dies.
class Scratch {
 public:
  explicit Scratch(cudaStream_t st) : st_(st) {}
  ~Scratch();
  void* alloc(size_t bytes);  // nullptr on failure (last_error set)
  template <typename T>
  T* alloc_n(size_t n) {
    return static_cast<T*>(alloc(n * sizeof(T)));
  }
  cudaStream_t stream() const { return st_; }

 private:
  cudaStream_t st_;
  std::vector<void*> ptrs_;
};

// MemoryRawVector on device (vector/memory_raw_vector.cc:152-240): append-only rows of row_bytes bytes kept in
// fixed-size segments, row stride row_bytes rounded up to 16 bytes, zero padded.  A row is d fp32 values (4 d bytes,
// stride 4 dpad) for the float index types and d / 8 packed bytes for BINARYIVF: the store knows only its byte size.  The segments are in HBM, or, for a
// field whose store_type is "RocksDB" (host placement), in pinned host memory mapped into the device's address space:
// kernels then read rows over PCIe through the same segment table, and the partition's HBM holds only its index.
class RawStore {
 public:
  // host placement: segments of 2^kHostSegShift rows (32 MiB at d = 128), so a small partition pins little memory;
  // kMaxSegs of them still cover 2^32 rows
  static constexpr int kHostSegShift = 16;
  RawStore(int row_bytes, int seg_shift, bool host);
  ~RawStore();
  int row_bytes() const { return (int)row_bytes_; }
  int64_t stride() const { return stride_; }  // bytes between rows
  int64_t size() const { return n_; }
  bool on_host() const { return host_; }
  int seg_shift() const { return seg_shift_; }
  int64_t seg_rows() const { return (int64_t)1 << seg_shift_; }
  int nsegs() const { return (int)segs_.size(); }
  // a segment's base: device memory, or (host placement) the pinned host rows, for copies
  const unsigned char* seg_bytes(int i) const { return segs_[i].base; }
  const float* seg(int i) const { return reinterpret_cast<const float*>(segs_[i].base); }  // float index types
  // device-visible segment bases [kMaxSegs], what kernels index rows through
  const float* const* d_segs() const { return reinterpret_cast<const float* const*>(d_segs_); }
  // rows: n x row_bytes, packed, on host, or n rows ld_bytes apart on device
  int append_host(const void* x, int64_t n, cudaStream_t st);
  int append_device(const void* x, int64_t ld_bytes, int64_t n, cudaStream_t st);
  int update_host(int64_t vid, const void* x, cudaStream_t st);
  int get_host(int64_t vid, void* out) const;
  int get_rows_host(int64_t start, int64_t n, void* out) const;  // n x row_bytes, packed
  // the rows [0, n) contiguous in device memory, stride() bytes apart (training slab, GetVectorHeader): the segment
  // itself or a copy owned by `s`
  const float* contiguous(int64_t n, Scratch& s);
  // rows [start, start + n) (stride() bytes apart) into device memory at dst, ordered on st
  cudaError_t copy_rows_to_device(int64_t start, int64_t n, void* dst, cudaStream_t st) const;
  // bytes ensure(n_total) would newly obtain (its granules and segments, the shadow's included), and in *rows the rows
  // of this store they make room for: what the memory limit admits before documents are accepted
  int64_t growth_bytes(int64_t n_total, int64_t* rows) const;
  // physical HBM behind the store, its int8 shadow included (0 for host placement)
  int64_t mem_bytes() const { return phys_bytes_ + (shadow_ ? shadow_->phys_bytes_ : 0); }
  int64_t host_bytes() const { return host_bytes_; }  // pinned host memory behind the store
  // The int8 shadow of fp32 rows that the two-pass exact re-rank screens candidates with (launch_rerank_prefilter):
  // row vid at shadow_segs()[vid >> seg_shift()] + (vid & (seg_rows() - 1)) * shadow_stride().  Written with the fp32
  // rows in the same stream-ordered step, so whatever sees a row sees its shadow.  Only an HBM store of fp32 rows gets
  // one, and only while it is empty (enable_shadow is a no-op otherwise).
  void enable_shadow();
  bool has_shadow() const { return shadow_ != nullptr; }
  const unsigned char* const* shadow_segs() const { return shadow_->d_segs_; }
  int64_t shadow_stride() const { return shadow_->stride_; }

 private:
  int encode_shadow(int64_t si, int64_t off, int64_t cnt, cudaStream_t st);
  std::unique_ptr<RawStore> shadow_;
  int ensure(int64_t n_total);
  int new_segment();
  int map_rows(int si, int64_t rows);
  struct Seg {
    unsigned char* base = nullptr;
    bool vmm = false;
    size_t va_bytes = 0, mapped = 0, gran = 0;
    std::vector<std::pair<unsigned long long, size_t>> chunks;  // (CUmemGenericAllocationHandle, bytes), in address order
  };
  size_t row_bytes_;
  int64_t stride_;
  int seg_shift_, device_ = 0;
  bool host_;
  int64_t n_ = 0, phys_bytes_ = 0, host_bytes_ = 0;
  std::vector<Seg> segs_;
  unsigned char** d_segs_ = nullptr;  // device array [kMaxSegs]
  static constexpr int kMaxSegs = 65536;
};

// RTInvertIndex / RealTimeMemData on device (index/realtime/realtime_mem_data.{h,cc}): per-list
// growable arrays of fixed-size codes + int64 ids (top bit = tombstone), entries in insertion
// order, length published after the data.
class IvfLists {
 public:
  IvfLists(int nlist, int code_bytes);
  ~IvfLists();
  int nlist() const { return nlist_; }
  int max_len() const { return max_len_; }
  int64_t total() const { return total_; }
  const std::vector<int>& lens() const { return h_len_; }
  uint64_t uid() const { return uid_; }  // distinguishes list sets (reset_index builds a new one)
  ListDirectory directory() const;
  // make room for add[l] more entries in every list; grows by copy (x1.5) when needed
  int reserve(const std::vector<int>& add, cudaStream_t st);
  // device arrays of per-list base pointers (valid after reserve)
  void* const* d_data() const { return d_data_; }
  int64_t* const* d_ids() const { return d_ids_; }
  // account for appended entries and publish the new lengths (after the scatter kernel, same stream)
  int commit(const std::vector<int>& add, cudaStream_t st);
  // tombstone one entry (Update path, realtime_mem_data.cc:298-320)
  int tombstone(int list, int pos, cudaStream_t st);
  // host copies for dump / parity tests
  int download_list(int l, std::vector<uint8_t>* codes, std::vector<int64_t>* ids) const;
  // append position of list l (valid after reserve): where the next entry's code / id goes
  void* list_data(int l) const { return static_cast<char*>(h_data_[l]) + (size_t)h_len_[l] * code_bytes_; }
  int64_t* list_ids(int l) const { return h_ids_[l] + h_len_[l]; }
  int64_t mem_bytes() const { return bytes_; }
  // bytes the lists would occupy packed tightly; compact() re-packs them into one fresh slab and
  // frees every old one (copy-on-grow never reuses the regions it leaves behind).  The caller must
  // exclude concurrent searches; in-flight kernels are drained before the old slabs go.
  int64_t packed_bytes() const;
  int compact(cudaStream_t st);
  // whether the slab space the lists have left behind is worth a re-pack: more than half of the live bytes and more
  // than 1 GiB
  bool compact_due() const { return bytes_ - packed_bytes() > std::max<int64_t>((int64_t)1 << 30, packed_bytes() / 2); }
  // Dead entries reported per list (deleted_nums_ of the reference): tombstone() counts the entry it marks,
  // add_dead() the deletions and loaded tombstones the owner knows of.  They choose the lists to purge; what a purge
  // drops is decided entry by entry on the device.
  const std::vector<int>& dead_counts() const { return h_dead_; }
  void add_dead(int list, int n) { h_dead_[list] += n; }
  // Bumped by purge(): entries moved inside their lists, so "same list set + same lengths" no longer means "same
  // content".  Whatever caches per-entry data beside the lists keys on it.
  uint64_t content_gen() const { return content_gen_; }
  // Drop the dead entries (tombstoned, or set in the device bitmap d_del_bits, nullable) of `lists`, in one pass over
  // the device (RealTimeMemData::CompactBucket, realtime_mem_data.cc:94-146).  Survivors keep their order and move to
  // fresh regions, as copy-on-grow does, so a kernel still reading an old region reads valid memory; pointers are
  // published before lengths.  The caller holds the index lock exclusively with earlier searches drained.
  // newpos[vid - vid_min] = (list << 32 | pos) of every surviving vid, ~0 for vids no longer in these lists.
  struct Purged {
    int64_t dropped = 0, vid_min = 0;
    std::vector<uint64_t> newpos;
  };
  int purge(const std::vector<int>& lists, const uint32_t* d_del_bits, cudaStream_t st, Purged* out);

 private:
  void* slab_alloc(size_t bytes);
  int slab_reserve(size_t need_bytes);  // a new slab unless the current one has need_bytes left
  int nlist_, code_bytes_;
  uint64_t uid_, content_gen_ = 0;
  std::vector<int> h_dead_;
  std::vector<void*> h_data_;
  std::vector<int64_t*> h_ids_;
  std::vector<int> h_len_, h_cap_;
  void** d_data_ = nullptr;
  int64_t** d_ids_ = nullptr;
  int* d_len_ = nullptr;
  int max_len_ = 0;
  int64_t total_ = 0, bytes_ = 0;
  std::vector<void*> slabs_;
  char* slab_cur_ = nullptr;
  size_t slab_left_ = 0;
};

struct ModelParams {  // index/impl/gamma_index_ivfpq.h:1031-1257, gamma_index_ivfflat.cc:40-196
  int ncentroids = 2048;
  int nprobe = 80;
  int metric = kMetricIP;       // gamma default: InnerProduct
  int nsubvector = 0;           // 0 => d/2 ... see IVFPQIndex::init (gamma_index_ivfpq.cc:122-124)
  int nbits = 8;
  int training_threshold = 0;   // 0 => engine default
  int bucket_init_size = 1000;
  int bucket_max_size = 1280000;
  int opq_nsubvector = 0;       // > 0: OPQ rotation in front of the IVFPQ index (gamma_index_ivfpq.h:1202-1216)
  bool has_opq = false;         // an "opq" object was given (IVFPQFastScan refuses it)
  int bbs = 32;                 // IVFPQFastScan block size as given (gamma_index_ivfpqfs.h:126-133; <= 0 => 32)
  bool host_store = false;      // raw vectors in pinned host memory (store_type "RocksDB"); otherwise in HBM
  int ncentroids_arg = 0;       // "ncentroids" as given, 0 if absent (BINARYIVF has its own default and range check)
  int nb_bits = 4;              // IVFRABITQ bits per dimension as given (validated by create_index: [1, 9])
  int qb = 4;                   // IVFRABITQ query bits as given (validated by create_index: [0, 8])
  // The GPU_* types check the values as given, in their own order and with their own messages (create_index): whether
  // each key was present, its value even when <= 0, and a metric_type that is neither L2 nor InnerProduct
  bool has_ncentroids = false, has_nprobe = false, has_nsubvector = false, has_nbits = false;
  int nprobe_arg = 0, nsubvector_arg = 0, nbits_arg = 0;
  int bucket_init_arg = 1000, bucket_max_arg = 1000000;  // GPU_IVFFLAT's defaults (IVFFlatGPUModelParams)
  std::string metric_unknown;
  double ns_threshold = 0.2;  // VEARCH noise-shaping threshold (VearchModelParams); NaN: no noise shaping
  bool reordering = false;    // VEARCH exact re-rank of the k' best codes
};

// gamma's two GPU index types (index/impl/gpu/): GPU_IVFPQ is an IVFPQIndex and GPU_IVFFLAT an IVFFlatIndex, created
// under the reference's GPU parameter contract and searched under its GPU request contract (Index::gpu_contract)
inline bool is_gpu_index_type(const std::string& type) { return type == "GPU_IVFPQ" || type == "GPU_IVFFLAT"; }

struct RetrievalParams {  // gamma_index_ivfpq.cc:233-294, gamma_index_ivfflat.cc:293-340
  int nprobe = -1;
  int metric = -1;  // -1 => index metric
  int recall_num = -1;
  int parallel_on_queries = 1;
  bool brute_force = false;
  int qb = -1;            // IVFRABITQ query bits, -1 => the index's (a value outside [0, 8] falls back to it)
  bool centered = false;  // IVFRABITQ: parsed, no effect (the estimate already centres the query on the list)
  bool given = false;     // the parameter string was not empty (VEARCH's defaults depend on it)
};

struct SearchContext {  // RetrievalContext / SearchCondition (common/gamma_common_data.h:33-121)
  const uint8_t* del_bitmap = nullptr;     // host, bit set => deleted
  const uint8_t* filter_bitmap = nullptr;  // host, bit set => allowed (nullptr => no filter)
  // the same bitmaps as uint32 words on the index's device, used in place of the host ones; they must be readable
  // when the search starts (written on its stream, or waited for)
  const uint32_t* del_bits_dev = nullptr;
  const uint32_t* filter_bits_dev = nullptr;
  // words readable at each device bitmap, zero past bitmap_bits; 0: only its ceil(bitmap_bits / 8) bytes.  A bitmap
  // that covers what the scan reads (upload_bitmaps) is used as it is, any other is copied into padded scratch.
  int64_t bits_dev_words = 0;
  int64_t bitmap_bits = 0;
  float min_score = -3.4028235e38f, max_score = 3.4028235e38f;
  bool search_unindexed_tail = false;  // table.enable_realtime: brute-force the not-yet-indexed vectors too
  RetrievalParams params;
};

class Index {
 public:
  // row_bytes: bytes of a stored row (0: 4 d, d fp32 values)
  Index(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift, int row_bytes = 0);
  virtual ~Index();
  const std::string& type() const { return type_; }
  // The GPU_* types' request contract (CommonSearch, gamma_gpu_search_base.h:40-112): at most kGpuMaxReq queries per
  // call and k' = max(k, recall_num) at most kGpuMaxK, refused before request coalescing; no exact re-rank; a request
  // nprobe outside (0, min(nlist, kGpuMaxK)] falls back to the model's (resolve_nprobe)
  static constexpr int kGpuMaxReq = 512, kGpuMaxK = 2048;
  // bytes of per-(query, part) partial keys one scan step may hold (FLAT chunks, IVF-Flat query-major splits); larger
  // batches are cut into query blocks
  static constexpr int64_t kScanPartialBudget = (int64_t)1 << 30;
  bool gpu_contract() const { return gpu_contract_; }
  int d() const { return d_; }
  int device() const { return device_; }
  int metric() const { return mp_.metric; }
  const ModelParams& model_params() const { return mp_; }
  RawStore& store() { return *store_; }
  int64_t indexed_count() const { return indexed_count_; }
  bool trained() const { return trained_; }
  virtual int64_t training_threshold() const { return 0; }
  // whether Engine::Dump saves the trained state (centroids, codebook) beside the rows for Load to restore; false: the
  // trained state lives only in the type's index file (dump_gamma), and Load trains again when that file is missing or
  // refused
  virtual bool persists_trained_state() const { return true; }

  // AddToStore (vector_manager.cc:455): append raw vectors, host rows n x store().row_bytes() bytes
  int add_vectors(const void* x, int64_t n);
  int add_vectors_device(const float* x, int64_t ld, int64_t n);
  // IndexModel::Indexing(): train on the first `num` stored vectors
  virtual int train() { trained_ = true; return 0; }
  // VectorManager::AddRTVecsToIndex (vector_manager.cc:572-702): index all not-yet-indexed rows
  virtual int add_pending(const uint8_t* del_bitmap) { indexed_count_ = store_->size(); return 0; }
  // Engine::Update -> RawVector update + IndexModel::Update (search/engine.cc:774-850;
  // realtime_mem_data.cc:298-320: old entry tombstoned, vector re-appended to its new list)
  virtual int update_vector(int64_t vid, const void* x);  // x: one row of store().row_bytes() bytes
  // IndexModel::Delete (RTInvertIndex::Delete, realtime_mem_data.cc:186-196): the documents were deleted.  Their
  // entries stay where they are, hidden by the deletion bitmap at search time; the lists only count them.
  virtual int delete_vectors(const int64_t* vids, int64_t n) { (void)vids; (void)n; return 0; }
  // RealTimeMemData::CompactIfNeed (realtime_mem_data.cc:347-370): rewrite every list whose counted dead share is at
  // least `threshold` (the reference: 0.3f; 0 = every list with a dead entry) without its tombstoned entries and the
  // entries set in del_bitmap (host, bitmap_bytes bytes, nullable).  *dropped (optional) = entries removed.
  virtual int purge_lists(float threshold, const uint8_t* del_bitmap, int64_t bitmap_bytes, int64_t* dropped) {
    (void)threshold; (void)del_bitmap; (void)bitmap_bytes;
    if (dropped) *dropped = 0;
    return 0;
  }
  // IndexModel::Search (index_model.h:296): x = nq host rows of store().row_bytes() bytes (d floats; BINARYIVF: d / 8
  // packed bytes); out = nq x k, unfilled id -1.  Returns 0, -1 on error (last_error), -2 if killed.
  int search(const SearchContext& ctx, int nq, const void* x, int k, float* out_dis, int64_t* out_ids);
  // one H2D -> kernels -> D2H round trip on the calling thread's stream
  int search_direct(const SearchContext& ctx, int nq, const void* x, int k, float* out_dis, int64_t* out_ids);
  // float queries already in device memory (nq rows of d floats, ldx floats apart), results left there, ordered on st.
  // out_keys_dev (optional): the nq x k result keys, (order-preserving score bits << 32) | vid, best first,
  // sentinel padded -- what the multi-GPU merge exchanges (one all-gather instead of scores + ids)
  int search_device(const SearchContext& ctx, int nq, const float* x_dev, int64_t ldx, int k, float* out_dis_dev,
                    int64_t* out_ids_dev, cudaStream_t st, unsigned long long* out_keys_dev = nullptr);
  // forget the trained state and the index structures, keep the raw vectors (Engine::RebuildIndex ->
  // VectorManager::ReCreateVectorIndexes, search/engine.cc:991-1089): the next train() starts over
  virtual int reset_index() { return 0; }
  virtual int64_t index_mem_bytes() const { return 0; }
  // Admission under the memory limit (mem_ledger.h): what storing rows up to n_total costs -- the store's growth where
  // the store lives, and for every row that growth makes room for, the index bytes it will take once indexed
  void memory_charges(int64_t n_total, std::vector<mem::Charge>* out);
  // the index bytes `rows` new rows will take once indexed, on the devices that will hold them (none for FLAT)
  virtual void charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) { (void)rows; (void)out; }
  // free the scan scratch buffers no search is using (the memory limit's trim)
  void release_idle_scratch();
  // gamma's own index file of the type (IvfIndex::dump_gamma / load_gamma); the types without one write and read nothing
  virtual int dump_gamma(const std::string& dir, const std::string& abs_name) { (void)dir; (void)abs_name; return 0; }
  virtual int load_gamma(const std::string& dir, const std::string& abs_name, int64_t* load_num) {
    (void)dir; (void)abs_name;
    *load_num = 0;
    return 0;
  }
  // stop the background worker (request coalescer); also run from an atexit hook for objects the host
  // never closed, so no thread of ours is inside the CUDA runtime while it is being torn down
  void quiesce();
  // device time spent in the dominant scan kernel(s) since the last call (ms), for the bench
  // roofline: CUDA events recorded on the launching stream around the scan launches, read here.
  float last_scan_ms();
  std::vector<std::pair<std::string, float>> stage_times();
  void set_time_scan(bool on) { time_scan_ = on; }
  const char* last_scan_kernel() const { return last_scan_kernel_; }
  const char* last_scan_info() const { return last_scan_info_; }  // JSON details of the last scan path (bench)
  // While on, every search that re-ranks through the two-pass kernel records, per query, how many candidates' fp32
  // rows it read (and waits for the count); take_rerank_survivors() returns and clears them.  Off by default.
  void set_rerank_stats(bool on) { rr_stats_ = on; }
  std::vector<int> take_rerank_survivors() {
    std::lock_guard<std::mutex> g(ev_mu_);
    return std::move(rr_survivors_);
  }

 protected:
  // Device queries, here and below: nq rows store().stride() bytes apart, zero padded (dpad floats; BINARYIVF: words).
  // nq host rows of store().row_bytes() bytes as device queries in `s`; nullptr on failure (last_error set)
  const void* upload_queries(int nq, const void* x, Scratch& s);
  // the search behind every query entry point, with mu_ held shared: bitmaps, brute force or the index, the realtime
  // tail; the nq x k result keys into *keys (allocated in s)
  int search_keys(const SearchContext& ctx, int nq, const void* xq, int k, unsigned long long** keys, Scratch& s);
  // the nq x k result keys decoded under `metric` into the host arrays; returns once they are there
  int download_results(const unsigned long long* keys, int nq, int k, int metric, float* out_dis, int64_t* out_ids,
                       Scratch& s);
  // the metric a search ranks by: the retrieval parameters' metric_type, else the index's
  virtual int search_metric(const SearchContext& ctx) const { return ctx.params.metric >= 0 ? ctx.params.metric : mp_.metric; }
  // GammaFLATIndex::Search (gamma_index_flat.cc:130-370) over rows [row_begin, nrows)
  int flat_search_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                      int64_t nrows, unsigned long long* out_keys, Scratch& s, int64_t row_begin = 0);
  // flat_search_dev's distance tile: scores [nq][ldo] of queries xq against m device rows (both store().stride() bytes
  // apart), exact; names the scan's kernels in last_scan_kernel_
  virtual cudaError_t flat_tile(const void* xq, int nq, const void* rows, int m, int metric, float* scores, int64_t ldo,
                                cudaStream_t st);
  virtual int search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                              unsigned long long* out_keys, Scratch& s) = 0;
  int upload_bitmaps(const SearchContext& ctx, FilterArgs* f, Scratch& s);
  // rows [vid0, vid0 + n) as device rows (store().stride() bytes apart): in HBM the segment itself (the rows must lie in
  // one segment), for host placement a copy in `s`, ordered on its stream (any rows)
  const void* store_rows_dev(int64_t vid0, int64_t n, Scratch& s);
  // A copy stream and its events for the staged FLAT scan of a host store (flat_search_dev).  Created on first use and
  // pooled: a search holds a lane while it enqueues its copies; what it enqueued keeps the events' records it waited on.
  struct CopyLane {
    cudaStream_t cs = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr}, reusable[2] = {nullptr, nullptr};
    ~CopyLane();
  };
  CopyLane* lane_acquire();  // nullptr on failure (last_error set)
  void lane_release(CopyLane* l);
  std::mutex lane_mu_;
  std::vector<std::unique_ptr<CopyLane>> lanes_;
  std::vector<CopyLane*> free_lanes_;

  // the GPU_* request limits above, for a search of nq queries at top k; 0 or -1 (last_error set)
  int check_gpu_request(const SearchContext& ctx, int nq, int k) const;

  std::string type_;
  bool gpu_contract_;
  int d_, dpad_, device_;
  ModelParams mp_;
  std::unique_ptr<RawStore> store_;
  int64_t indexed_count_ = 0;
  bool trained_ = false;
  mutable std::shared_mutex mu_;  // searches shared, index mutation exclusive
  // Kernels of a search keep reading the list directory (lengths, base pointers), the centroids and the raw-store
  // segments AFTER the search call released mu_ (device-resident searches are asynchronous).  Every search leaves an
  // event on its stream; whoever mutates those structures takes mu_ exclusively (no new search can enqueue) and then
  // drains the events, so no kernel of an earlier search observes a directory that changes under it.
  void note_search_enqueued(cudaStream_t st);
  void drain_searches();
  std::mutex inflight_mu_;
  std::vector<cudaEvent_t> inflight_;
  std::mutex build_mu_;           // serialises train / add_pending / update_vector (one writer at a time)

  // Request coalescing (SURVEY 8f N-3; reference: the batching thread of its GPU index,
  // index/impl/gpu/gamma_index_ivfflat_gpu.cc:302-396): concurrent small Search calls with the
  // same (k, retrieval params, score window, no bitmaps) are merged into one device batch by a
  // worker thread; callers block until their slice of the result is ready.
  struct CoReq {
    const SearchContext* ctx;
    int nq, k;
    const void* x;
    float* out_dis;
    int64_t* out_ids;
    int rc = 0;
    bool done = false;
    std::string err;
  };
  void coalesce_loop();
  bool coalescable(const SearchContext& ctx, int nq) const;
  std::mutex co_mu_;
  std::condition_variable co_cv_, co_done_cv_;
  std::vector<CoReq*> co_queue_;
  std::thread co_thread_;
  bool co_stop_ = false, co_started_ = false;
  cudaStream_t build_stream_ = nullptr;
  // grow-only cache of multi-GB scratch (list-major score segments): stream-ordered pools re-map
  // such blocks on every search when the caller's stream is the legacy default stream
  void* big_acquire(size_t bytes, cudaStream_t st);
  void big_release(void* p, cudaStream_t st);
  void free_idle_big_locked();  // big_mu_ held
  struct BigBuf {
    void* p;
    size_t cap;
    bool busy;
    cudaEvent_t done;
  };
  std::mutex big_mu_;
  std::vector<BigBuf> big_;
  struct BigScope {  // a big_acquire'd buffer (p, nullptr on failure), released event-stamped on every exit path
    Index* ix;
    cudaStream_t st;
    void* p;
    BigScope(Index* i, size_t bytes, cudaStream_t s) : ix(i), st(s), p(i->big_acquire(bytes, s)) {}
    ~BigScope() {
      if (p) ix->big_release(p, st);
    }
  };
  void scan_timer_begin(cudaStream_t st);
  void scan_timer_end(cudaStream_t st);
  // per-stage device times (bench breakdown): CUDA events on the launching stream around each stage of a
  // search while set_time_scan(true); stage_times() sums them per name since the last call
  void stage_begin(const char* name, cudaStream_t st);
  void stage_end(cudaStream_t st);
  struct StageEv {
    const char* name;
    cudaEvent_t e0, e1;
  };
  std::vector<StageEv> stage_events_;
  struct StageScope {
    Index* ix;
    cudaStream_t st;
    StageScope(Index* i, const char* name, cudaStream_t s) : ix(i), st(s) { ix->stage_begin(name, st); }
    ~StageScope() { ix->stage_end(st); }
  };
  std::mutex ev_mu_;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> scan_events_;
  bool time_scan_ = false;
  bool rr_stats_ = false;
  std::vector<int> rr_survivors_;  // under ev_mu_
  const char* last_scan_kernel_ = "";  // which scan path served the last search (bench roofline label)
  char last_scan_info_[160] = "{}";
};

class FlatIndex : public Index {
 public:
  FlatIndex(int d, const ModelParams& mp, int device, int seg_shift) : Index("FLAT", d, mp, device, seg_shift) {
    trained_ = true;
  }

 protected:
  int search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                      unsigned long long* out_keys, Scratch& s) override;
};

// k-means on device (faiss Clustering restated; DESIGN.md K6)
struct KMeansParams {
  int niter = 25;
  int64_t seed = 1234;
  bool spherical = false;
  int max_points_per_centroid = 256;
  bool hot_start = false;  // keep the centroids passed in as the initial state (ProductQuantizer::Train_hot_start)
  bool l2_assign = false;  // spherical, but assign by L2 (quantiser IndexFlatL2, as IVFPQFastScan has under IP)
};
// What one kmeans_device run did, step by step (gb_debug_kmeans_trace; DESIGN.md §5, training bar).  n_s = the rows
// trained on, k x d centroid snapshots.
struct KMeansTrace {
  std::vector<int32_t> sample;            // [n_s] the rows of x sampled (empty: all of them, in order)
  std::vector<float> init;                // [k][d] the initial centroids
  std::vector<int32_t> labels;            // [niter][n_s] each row's cluster
  std::vector<float> scores;              // [niter][n_s] the score its key carried
  std::vector<float> mean, split, norm;   // [niter][k][d] after the segmented mean, the split, the renormalisation
};
// trace: nullptr on every production path
int kmeans_device(const float* x, int64_t ldx, int64_t n, int d, int k, const KMeansParams& kp, float* centroids,
                  int64_t ldc, cudaStream_t st, std::vector<float>* obj, KMeansTrace* trace = nullptr);

// What an IVF index's codec puts into gamma's index file (index_io.cu)
struct GammaFileFormat {
  const char* file = nullptr;  // <dir>/<abs_name>/<file>; nullptr: no index file for this type
  uint32_t magic = 0;          // fourcc of the index: faiss's, or this engine's own for the types gamma writes no file of
  uint64_t code_size = 0;      // bytes per list entry on disk (in memory: code_bytes(), rows padded when they differ)
  bool indexed_count = false;  // an i32 indexed_count follows the lists
};

// The inverted-file skeleton shared by every IVF type: coarse centroids, inverted lists, train / add / update / reset /
// compact, coarse search, and the gamma index-file skeleton.  A codec derived from it says how vectors become list
// entries (append_batch, code_bytes) and how a query scans the probed lists (scan_dev).
class IvfIndex : public Index {
 public:
  IvfIndex(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift, int row_bytes = 0);
  ~IvfIndex() override;
  int64_t training_threshold() const override;
  int train() override;
  int add_pending(const uint8_t* del_bitmap) override;
  int update_vector(int64_t vid, const void* x) override;
  int delete_vectors(const int64_t* vids, int64_t n) override;  // a vid not in a list, or already counted, is ignored
  int purge_lists(float threshold, const uint8_t* del_bitmap, int64_t bitmap_bytes, int64_t* dropped) override;
  int dead_counts(int* out);  // [nlist] dead entries counted per list since its last purge
  int reset_index() override;
  int64_t index_mem_bytes() const override;
  int nlist() const { return nlist_; }
  virtual int code_bytes() const = 0;  // bytes per list entry
  void charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) override;  // a list entry and its id
  // parity hooks: exchange index state with the oracle
  int set_centroids(const float* host, int nlist);  // marks trained
  int get_centroids(float* host) const;
  const char* last_coarse_kernel() const { return last_coarse_kernel_; }  // test hook: which coarse path ran last
  IvfLists* lists() { return lists_.get(); }
  // quantizer->search (ivfflat.cc:568): top-nprobe lists per query; x: host rows as Index::search takes them
  int coarse_search_host(int nq, const void* x, int nprobe, float* out_dis, int64_t* out_ids);
  // search_preassigned with caller-provided (keys, coarse_dis): host in/out; coarse_dis may be null (zeros)
  int search_preassigned_host(const SearchContext& ctx, int nq, const void* x, int k, const int64_t* keys,
                              const float* coarse_dis, int nprobe, float* out_dis, int64_t* out_ids);
  // re-pack the inverted lists into one tight slab (IvfLists::compact); also done automatically after
  // a bulk add_pending when more than half of the slab space is dead
  int compact_lists();
  // gamma's own index files (index_io.cu): <dir>/<abs_name>/<gamma_format().file>.  load: the vector
  // store must already hold the vectors the file indexes; *load_num = IndexModel::Load's load_num
  int dump_gamma(const std::string& dir, const std::string& abs_name) override;
  int load_gamma(const std::string& dir, const std::string& abs_name, int64_t* load_num) override;

 protected:
  friend class ShardedIndex;
  // One shard of a ShardedIndex holds the global vids v with v % shard_count_ == shard_id_ as local vid v / shard_count_;
  // the deletion bitmap of add_pending and the list fallback of a row without a nearest list take the global vid
  int64_t shard_count_ = 1, shard_id_ = 0;
  int64_t global_vid(int64_t local) const { return local * shard_count_ + shard_id_; }
  // train() on the first training_threshold() rows of `src` (a sharded index trains its first shard on its own store)
  int train_on(RawStore& src);
  // Update's list part: tombstone vid's entry, append the row x_dev (device, store().stride() bytes) to its new list;
  // build_mu_ held
  int reindex_vector(int64_t vid, const void* x_dev);
  // empty lists, the trained state kept (a sharded Load that failed part way)
  void clear_lists();
  // the lists whose counted dead share is at least threshold, and their purge with the device bitmap d_del_bits (by
  // vid, nullable), ordered on build_stream_; build_mu_ and mu_ held exclusively
  std::vector<int> purge_candidates(float threshold) const;
  int purge_locked(const std::vector<int>& sel, const uint32_t* d_del_bits, int64_t* dropped);
  // the gamma index file with this index's header and trained state, `lens` and the list contents `fetch` gives
  // (codes of code_bytes() bytes and ids per list); build_mu_ held
  int write_gamma(const std::string& dir, const std::string& abs_name, int64_t indexed, const std::vector<int>& lens,
                  const std::function<int(int, std::vector<uint8_t>*, std::vector<int64_t>*)>& fetch);
  // load_gamma keeping only the file's entries of this shard (global vid % shard_count_ == shard_id_, as local vids);
  // store_rows: the rows of the (global) vector store; *file_indexed = the file's indexed count (IvFl) or this shard's
  // live entries (IwPQ)
  int load_gamma_part(const std::string& dir, const std::string& abs_name, int64_t store_rows, int64_t* load_num,
                      int64_t* file_indexed);
  virtual GammaFileFormat gamma_format() const = 0;
  // codec blocks after the coarse quantiser (product quantizer, OPQ)
  virtual int dump_gamma_extra(FILE* f) { (void)f; return 0; }
  virtual int load_gamma_extra(FILE* f) { (void)f; return 0; }
  // the reference's default training_threshold of the type; training_threshold() clamps it to [39, 256] * nlist
  virtual int64_t default_training_threshold() const = 0;
  // k-means of the coarse centroids (default: faiss ClusteringParameters)
  virtual KMeansParams coarse_kmeans_params() const { return KMeansParams(); }
  int search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                      unsigned long long* out_keys, Scratch& s) override;
  // the nprobe nearest lists of each query (after transform_dev)
  virtual int coarse_dev(int nq, const void* xq, int nprobe, int metric, int32_t* probe_ids, float* coarse_dis, Scratch& s);
  // xq: the queries after transform_dev; xq_raw: the same queries untransformed (the exact re-rank reads the raw store)
  virtual int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq,
                       const void* xq_raw, int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                       unsigned long long* out_keys, Scratch& s) = 0;
  // scan_dev of the estimating codecs (IVFPQ, IVFPQFastScan, IVFRABITQ) through the query-major list scan, with the
  // recall_num / re-rank semantics of gamma_index_ivfpq.cc:764-770: the k' = max(k, recall_num) best estimates, re-ranked
  // exactly from the raw vectors (rerank_xq) when recall_num > 0.  `prepare(kk, keys, need_sorted)` builds the per-query
  // tables and may serve the scan another way (0 = served, 1 = not, < 0 = error); `launch(kk, pg, partial)` launches the
  // scan kernel, named `kernel`, over pg probes per CTA; max_kk: the largest k' it selects, `limit_at` names what bounds
  // it in the error ("nsubvector 16")
  int scan_query_major_dev(const char* kernel, const SearchContext& ctx, const FilterArgs& f, int metric, int nq,
                           const float* rerank_xq, int k, int nprobe, int max_kk, const std::string& limit_at,
                           unsigned long long* out_keys, Scratch& s,
                           const std::function<int(int, unsigned long long*, bool)>& prepare,
                           const std::function<cudaError_t(int, int, unsigned long long*)>& launch);
  // List-major pair grouping (launch_lmk_group): the (query, probe) pairs grouped by list, `group` pairs per group, each
  // group cut into nseg row segments.  Items, pair order and totals are left in `s` for the list-major kernels.  The
  // scratch is allocated first (alloc_pair_grouping, stream-ordered on s), so the grouping may run on a stream forked
  // from s's after it.
  struct LmGrouping {
    int32_t *cnt, *start, *cursor, *item_start, *grp_start;
    int64_t* totals;
    int64_t* pair_j;
    LmTile* items;
  };
  int alloc_pair_grouping(int64_t npairs, int64_t max_items, LmGrouping* g, Scratch& s);
  cudaError_t group_pairs_by_list(const int32_t* probe_ids, int64_t npairs, int nseg, int group, const LmGrouping& g,
                                  cudaStream_t st);
  int assign_dev(const float* x, int64_t ldx, int64_t n, int32_t* assign_dev_out, Scratch& s);
  // the rows of a batch as the codec takes them (*xc) and each row's nearest list (out): fp32 rows (stride dpad) through
  // transform_dev and assign_dev; BINARYIVF: the packed rows as they are, by Hamming distance
  virtual int assign_batch(const void* x, int64_t n, const void** xc, int32_t* out, Scratch& s);
  virtual int resolve_nprobe(const SearchContext& ctx) const;
  // metric of the coarse quantiser (list assignment and probe choice) for a search under `metric`
  virtual int coarse_metric(int metric) const { return metric; }
  // write rows x [vid0, vid0+n) (as assign_batch left them) into the lists at (d_list, d_pos), after reserve and before
  // commit; add[l] = rows for list l
  virtual int append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                           const std::vector<int>& add, Scratch& s) = 0;
  virtual int train_extra(const float* xtrain, int64_t n, Scratch& s) { (void)xtrain; (void)n; (void)s; return 0; }
  // codec state dropped by reset_index, with build_mu_ and mu_ held exclusively
  virtual void reset_codec() {}
  // vector transform in front of the index (OPQ, gamma_index_ivfpq.cc:362-364, 422, 470, 585-590): applied to the
  // training slab (which also trains it), to vectors on their way into the lists and to queries; the raw store
  // and the exact re-rank keep the original vectors.  Default: identity (returns x).
  virtual const float* train_transform(const float* xt, int64_t n, Scratch& s) { (void)n; (void)s; return xt; }
  virtual const float* transform_dev(const float* x, int64_t n, Scratch& s) { (void)n; (void)s; return x; }

  // index rows [vid0, vid0+n) (device pointer x, store().stride() bytes apart) into the lists
  int index_batch(const void* x, int64_t n, int64_t vid0, const uint8_t* del_bitmap);
  // after every change of the lists (append, compaction), with mu_ held exclusively, ordered on st
  virtual int lists_changed(cudaStream_t st) { (void)st; return 0; }
  int compact_locked();  // lists_->compact + lists_changed, with mu_ held exclusively

  int nlist_;
  const char* last_coarse_kernel_ = "";
  float* d_centroids_ = nullptr;  // [nlist][dpad]
  // the centroids once more as tensor-core operand tiles (launch_tc_stage_rows) for the fused coarse quantiser, and
  // |c|^2 per row; rebuilt by every change of d_centroids_ (rebuild_centroid_tiles)
  float* d_cent_tiles_ = nullptr;
  float* d_cent_norms_ = nullptr;
  int rebuild_centroid_tiles(cudaStream_t st);
  // after every change of d_centroids_ (the end of rebuild_centroid_tiles), with mu_ held exclusively, ordered on st
  virtual int centroids_changed(cudaStream_t st) { (void)st; return 0; }
  std::unique_ptr<IvfLists> lists_;
  std::vector<uint64_t> vid2pos_;  // vid -> (list << 32 | pos), ~0 = not in a list (vid_bucket_no_pos_)
  std::vector<bool> del_counted_;  // vid's entry is counted dead by delete_vectors (so it is counted once)
};

// GammaIVFFlatIndex (index/impl/gamma_index_ivfflat.{h,cc}): the lists hold the raw fp32 rows.  type: "IVFFLAT", or
// "GPU_IVFFLAT" (GammaIVFFlatGPUIndex, the same index under the GPU contract)
class IVFFlatIndex : public IvfIndex {
 public:
  IVFFlatIndex(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift);
  ~IVFFlatIndex() override;
  int64_t index_mem_bytes() const override;
  int code_bytes() const override { return dpad_ * 4; }
  void charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) override;  // and its mirror row, while kept
  int mirror_builds() const { return mirror_.builds; }  // test hook
  int get_list_shifts(float* host) const;               // test hook: d_shifts_ as [nlist][d] (L2 indexes only)

 protected:
  GammaFileFormat gamma_format() const override;
  // gamma_index_ivfflat.cc:239; GPU_IVFFLAT: ncentroids * max_points_per_centroid (gamma_index_ivfflat_gpu.cc)
  int64_t default_training_threshold() const override { return (int64_t)nlist_ * (gpu_contract_ ? 256 : 200); }
  int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, const void* xq_raw, int k,
               const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
               Scratch& s) override;
  // list-major IVF-Flat scan on the tensor cores (kernels_tc.cu); returns 1 if not applicable
  int scan_listmajor_dev(const FilterArgs& f, int metric, int nq, const float* xq, int k, const int32_t* probe_ids,
                         int nprobe, unsigned long long* out_keys, Scratch& s);
  int append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                   const std::vector<int>& add, Scratch& s) override;
  void reset_codec() override;
  int lists_changed(cudaStream_t st) override;
  int centroids_changed(cudaStream_t st) override;  // new list shifts; the mirror goes stale
  // The list shifts s_l [nlist][dpad] of the list-major scan of an L2 index (nullptr under IP) (launch_list_shifts): its tensor-core operands are
  // x - s_l and y - s_l, so the rounding of the expanded form scales with the residual norms, not the raw ones.
  float* d_shifts_ = nullptr;
  // host placement, and every shard of a ShardedIndex (whose raw rows live with the sharded index): rowptr[vid] = the
  // list row holding vid, for the winner re-score (lists_changed)
  bool rescore_from_lists() const { return store_->on_host() || shard_count_ > 1; }
  const float** d_rowptr_ = nullptr;
  int64_t rowptr_cap_ = 0;

  // Tensor-core mirror of the lists (kernels_tc.cu): every list once more, pre-split and
  // pre-tiled in the shared-memory operand layout so the list-major kernel is fed by cp.async.bulk.
  // Built by the first list-major search, kept current in place by appends that fit its reserve,
  // rebuilt when a list outgrows it; users hold mirror_rw_ shared from the freshness check until their
  // kernels are enqueued, the rebuilder takes it exclusively and drains the device first.  Skipped
  // (register-staged kernel instead) when HBM is too full for it.
  struct TcMirror {
    float* base = nullptr;
    float* norms = nullptr;
    int64_t* d_tile0 = nullptr;
    int64_t tiles = 0, cap_tiles = 0;
    std::vector<int> lens;        // rows mirrored per list
    uint64_t content_gen = 0;     // IvfLists::content_gen() they were mirrored at: a purge moves rows inside lists
    std::vector<int> list_tiles;  // tiles reserved per list (a little slack, so appends go in place)
    bool disabled = false;
    int builds = 0;  // full (re)builds so far
  } mirror_;
  // appends keep the mirror current in place while the reserved tiles last; otherwise it goes stale and the
  // next list-major search rebuilds it
  int mirror_append(const float* x, int64_t n, const int32_t* d_list, const int32_t* d_pos, const std::vector<int>& add,
                    cudaStream_t st);
  std::shared_mutex mirror_rw_;  // taken after mu_
  int ensure_mirror(std::shared_lock<std::shared_mutex>& lk, cudaStream_t st);  // 0 = usable and current
  bool mirror_current() const {
    return mirror_.base && mirror_.lens == lists_->lens() && mirror_.content_gen == lists_->content_gen();
  }
};

// Product-quantiser base of IVFPQ and IVFPQFastScan: M sub-quantisers of ksub centroids each over dsub-wide slices, the
// codebook [M][ksub][dsub], its training, the encode path into the lists and the query-major list-scan search path.
class IvfPqBase : public IvfIndex {
 public:
  IvfPqBase(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift, int M, int ksub);
  ~IvfPqBase() override;
  int64_t index_mem_bytes() const override;
  int M() const { return M_; }
  int dsub() const { return dsub_; }
  int ksub() const { return ksub_; }
  int set_pq_centroids(const float* host);  // [M][ksub][dsub]; runs codebook_changed
  int get_pq_centroids(float* host) const;
  // list codes of n host rows; assign: each row's list (residual codecs), may be null otherwise
  int encode_host(const float* x, int64_t n, const int64_t* assign, uint8_t* codes_out);

 protected:
  // codes of n device rows (stride dpad) into codes [n][code_bytes()]; lists: each row's list (residual codecs)
  virtual cudaError_t encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st) = 0;
  // tables derived from the codebook, rebuilt after every change of it
  virtual int codebook_changed(cudaStream_t st) { (void)st; return 0; }
  int append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                   const std::vector<int>& add, Scratch& s) override;
  // faiss ProductQuantizer::train on n rows (stride dpad): M independent ksub-means on the dsub-wide slices
  int train_codebook(const float* x, int64_t n, Scratch& s);
  int M_, dsub_, ksub_;
  float* d_pq_ = nullptr;  // [M][ksub][dsub]
};

// GammaIVFPQIndex (index/impl/gamma_index_ivfpq.{h,cc}) at nbits_per_idx 1..8: ksub = 2^nbits centroids per
// sub-quantiser; list entries hold the residual codes bit-packed in ceil(M nbits / 8) bytes (faiss PQEncoderGeneric:
// code m at bits [m nbits, (m + 1) nbits), LSB-first), one byte per code at nbits = 8.  type: "IVFPQ", or "GPU_IVFPQ"
// (GammaIVFPQGPUIndex, the same index at nbits 8 under the GPU contract)
class IVFPQIndex : public IvfPqBase {
 public:
  // nbits_per_idx above this: faiss's 16-bit codes (PQDecoder16), whose [M][65536] fp32 table no scan keeps in shared memory
  static constexpr int kMaxNbits = 8;
  static constexpr int kGpuDefaultM = 64;  // GPU_IVFPQ's nsubvector default (IVFPQGPUModelParams)
  IVFPQIndex(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift);
  ~IVFPQIndex() override;
  int64_t index_mem_bytes() const override;
  int nbits() const { return nbits_; }
  int code_bytes() const override { return (M_ * nbits_ + 7) / 8; }
  int get_precomputed_table(float* host) const;  // [nlist][M][ksub]

 protected:
  GammaFileFormat gamma_format() const override;
  int64_t default_training_threshold() const override;
  KMeansParams coarse_kmeans_params() const override;
  int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, const void* xq_raw, int k,
               const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
               Scratch& s) override;
  void reset_codec() override { opq_trained_ = false; }
  int dump_gamma_extra(FILE* f) override;
  int load_gamma_extra(FILE* f) override;
  cudaError_t encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st) override;
  int train_extra(const float* xtrain, int64_t n, Scratch& s) override;
  int codebook_changed(cudaStream_t st) override;
  // list-major scan through the tensor-core filter (kernels_pqtc.cu); 1 = not applicable
  int scan_listmajor_pq(const FilterArgs& f, int metric, int nq, const float* xq, int kk, float* ip,
                        const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* adc_out,
                        bool need_sorted, Scratch& s);

  const float* train_transform(const float* xt, int64_t n, Scratch& s) override;
  const float* transform_dev(const float* x, int64_t n, Scratch& s) override;

  int nbits_;
  float* d_table_ = nullptr;  // [nlist][M][ksub] (L2 only)
  // the tensor-core filter and its tables exist at nbits = 8 only; packed codes are scanned query-major
  int8_t* d_cb8_ = nullptr;     // [M][256][dsub] int8 codebook (tensor-core filter)
  float* d_cbnrm_ = nullptr;    // [M][256] |pq|^2, then R^2, sb, D
  // |r_e|^2 of every list entry (L2), flat with 32-entry aligned list segments: built by the first list-major search
  // after the lists or the codebook changed (between purges lists are append-only: same list set + same content
  // generation + same lengths = same content)
  struct PqNormCache {
    float* base = nullptr;
    int64_t* d_off = nullptr;
    size_t cap = 0;
    std::vector<int> lens;
    uint64_t lists_uid = 0, content_gen = 0, pq_gen = 0;
  } pqn_;
  std::mutex pqn_mu_;
  uint64_t pq_gen_ = 1;
  int ensure_pq_norms(cudaStream_t st);
  float* d_opq_ = nullptr;    // [d][dpad] rows of the OPQ rotation A (y = A x); nullptr: no OPQ
  bool opq_trained_ = false;

 public:
  bool has_opq() const { return d_opq_ != nullptr; }
  int set_opq(const float* host_A);        // d x d row-major; marks the rotation trained
  int get_opq(float* host_A) const;
  int apply_opq_host(const float* x, int64_t n, float* out);  // test hook: y = A x through the device path
};

// GammaIVFPQFastScanIndex (index/impl/gamma_index_ivfpqfs.{h,cc}): faiss::IndexIVFPQFastScan with by_residual = false.
// The lists hold 4-bit codes of the raw vectors (16-centroid PQ, two codes per byte); a search quantises each query's
// M x 16 table to uint8 and sums it in integers.  The coarse quantiser is IndexFlatL2 under either metric.
class IVFPQFastScanIndex : public IvfPqBase {
 public:
  static constexpr int kKsub = 16;
  IVFPQFastScanIndex(int d, const ModelParams& mp, int device, int seg_shift)
      : IvfPqBase("IVFPQFastScan", d, mp, device, seg_shift, mp.nsubvector, kKsub) {
    store_->enable_shadow();
  }
  int code_bytes() const override { return (M_ + 1) / 2; }
  // M above this: faiss's 16-bit table sums could wrap (255 * 257 < 2^16), and the byte-pair table grows past what
  // the scan's shared memory holds beside its stages and queue
  static constexpr int kMaxM = 256;
  bool persists_trained_state() const override { return false; }
  // uint8 tables [nq][M][16] and (a, b) [nq][2] of a query batch under `metric` (-1: the index metric)
  int lut_host(int nq, const float* x, int metric, uint8_t* lut8_out, float* ab_out);

 protected:
  // the reference dumps no index file for this type; this engine writes its own (index_io.cu), which only it reads
  GammaFileFormat gamma_format() const override;
  int dump_gamma_extra(FILE* f) override;
  int load_gamma_extra(FILE* f) override;
  int64_t default_training_threshold() const override { return (int64_t)nlist_ * 39; }  // gamma_index_ivfpqfs.cc
  KMeansParams coarse_kmeans_params() const override;
  int coarse_metric(int metric) const override { (void)metric; return kMetricL2; }
  cudaError_t encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st) override;
  int train_extra(const float* xtrain, int64_t n, Scratch& s) override;
  int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, const void* xq_raw, int k,
               const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
               Scratch& s) override;
};

// GammaIndexBinaryIVF (index/impl/gamma_index_binary_ivf.{h,cc}): faiss::IndexBinaryIVF over packed binary rows of
// d / 8 bytes (d in bits), compared by Hamming distance, smaller first.  The coarse centroids are trained by faiss
// Clustering on the rows expanded to +-1 floats (binary_to_real), kept as floats in d_centroids_ and packed again
// (real_to_binary) for the coarse quantiser; list entries are the raw d / 8 bytes.  Rows and queries are packed bytes
// (store().row_bytes()), searched through the shared entry points: Index::search, coarse_search_host,
// search_preassigned_host.
class BinaryIvfIndex : public IvfIndex {
 public:
  static constexpr int kDefaultNlist = 256;   // BinaryModelParams() (gamma_index_binary_ivf.cc:23)
  static constexpr int kDefaultNprobe = 20;   // GammaIndexBinaryIVF::Init (gamma_index_binary_ivf.cc:114)
  BinaryIvfIndex(int d_bits, const ModelParams& mp, int device, int seg_shift);
  ~BinaryIvfIndex() override;
  int code_bytes() const override { return cb_; }
  bool persists_trained_state() const override { return false; }
  int64_t index_mem_bytes() const override;
  // packed centroids [nlist][d / 8] (set_binary_centroids marks the index trained)
  int set_binary_centroids(const uint8_t* host, int nlist);
  int get_binary_centroids(uint8_t* host) const;

 protected:
  // this engine's own index file (index_io.cu): the float centroids as the coarse quantiser, the packed ones after it
  GammaFileFormat gamma_format() const override;
  int dump_gamma_extra(FILE* f) override;
  int load_gamma_extra(FILE* f) override;
  int64_t default_training_threshold() const override { return (int64_t)nlist_ * 39; }  // nlist * min_points_per_centroid
  KMeansParams coarse_kmeans_params() const override;
  const float* train_transform(const float* xt, int64_t n, Scratch& s) override;
  int centroids_changed(cudaStream_t st) override;
  // Hamming distances rank like L2, whatever metric_type the retrieval parameters carry
  int search_metric(const SearchContext& ctx) const override { (void)ctx; return kMetricL2; }
  cudaError_t flat_tile(const void* xq, int nq, const void* rows, int m, int metric, float* scores, int64_t ldo,
                        cudaStream_t st) override;
  int coarse_dev(int nq, const void* xq, int nprobe, int metric, int32_t* probe_ids, float* coarse_dis, Scratch& s) override;
  int assign_batch(const void* x, int64_t n, const void** xc, int32_t* out, Scratch& s) override;
  int append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                   const std::vector<int>& add, Scratch& s) override;
  int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, const void* xq_raw, int k,
               const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
               Scratch& s) override;

 private:
  // the k Hamming-nearest lists of nq device rows (ldw_ words apart), the smaller list id among equals: keys [nq][k], sorted
  int hamming_topk(const uint32_t* xq, int nq, int k, unsigned long long* keys, Scratch& s);
  int cb_;             // bytes per row, d / 8
  int64_t ldw_;        // words between device rows (the raw store's stride)
  uint8_t* d_bcent_ = nullptr;  // [nlist][4 ldw_] packed centroids
};

// GammaIVFRABITQIndex (index/impl/gamma_index_ivfrabitq.{h,cc}): IVF with by_residual = true and a multi-bit RaBitQ code
// of each residual (kernels_rabitq.cu, DESIGN.md §3 K13).  The coarse quantiser is exact under the index metric (an
// "hnsw" object is accepted and ignored).  recall_num > 0 re-ranks the estimated candidates exactly from the raw vectors.
class RaBitQIndex : public IvfIndex {
 public:
  RaBitQIndex(int d, const ModelParams& mp, int device, int seg_shift)
      : IvfIndex("IVFRABITQ", d, mp, device, seg_shift), nb_bits_(mp.nb_bits), qb_(mp.qb) {
    store_->enable_shadow();
  }
  int code_bytes() const override { return rabitq_code_bytes(d_, nb_bits_); }
  bool persists_trained_state() const override { return false; }
  int nb_bits() const { return nb_bits_; }
  int qb() const { return qb_; }
  // test hooks: list entries of n host rows assigned to lists `assign`; the scan's estimates of every entry of list
  // lists[j] for query j (out: the lists' entries one after another), under `metric` and `qb`
  int encode_host(const float* x, int64_t n, const int64_t* assign, uint8_t* codes_out);
  int estimate_host(int nq, const float* x, const int64_t* lists, int qb, int metric, float* out);

 protected:
  // the reference's ivfrabitq.index is faiss's IndexIVFRaBitQ, which this engine neither reads nor writes; it writes its
  // own file under another name (index_io.cu)
  GammaFileFormat gamma_format() const override;
  int dump_gamma_extra(FILE* f) override;
  int load_gamma_extra(FILE* f) override;
  int64_t default_training_threshold() const override;
  KMeansParams coarse_kmeans_params() const override;
  int append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                   const std::vector<int>& add, Scratch& s) override;
  int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, const void* xq_raw, int k,
               const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
               Scratch& s) override;

 private:
  int nb_bits_, qb_;
};

// GammaVearchIndex (index/impl/scann/gamma_index_vearch.{h,cc}) over ScaNN's asymmetric hashing, restated: IVF lists of
// 4-bit codes, one per block of the VARIABLE_CHUNK split (kernels_scann.cu, DESIGN.md §3 K14).  Under IP the lists hold
// anisotropic (noise-shaped) codes of the residuals to spherical centroids and a search adds <q, c_l> to the table sum;
// under L2 they hold the nearest-centre codes of the raw rows.  reordering re-ranks k' = max(k, recall_num) candidates
// exactly from the raw vectors.
class VearchIndex : public IvfIndex {
 public:
  static constexpr int kDefaultNlist = 2048, kDefaultNsub = 64;  // VearchModelParams()
  // blocks above this: the byte-pair table, two code stages and a k' = 4096 queue no longer fit the scan's shared memory
  // with room to spare
  static constexpr int kMaxBlocks = 256;
  static constexpr int kDefaultLeaves = 512;  // GammaVearchIndex::leaves_
  VearchIndex(int d, const ModelParams& mp, int device, int seg_shift);
  ~VearchIndex() override;
  int code_bytes() const override { return (nb_ + 1) / 2; }
  bool persists_trained_state() const override { return false; }
  int64_t index_mem_bytes() const override;
  int nsub() const { return mp_.nsubvector; }
  int nblocks() const { return nb_; }
  double ns_threshold() const { return mp_.ns_threshold; }
  bool reordering() const { return mp_.reordering; }
  // test hooks: the codebook [16 d] floats (set marks nothing trained by itself), the list codes of n host rows assigned
  // to `assign` (IP; ignored under L2), the biased uint8 tables [nq][nblocks][16] and multipliers [nq] of a query batch
  int set_codebook(const float* host);
  int get_codebook(float* host) const;
  int encode_host(const float* x, int64_t n, const int64_t* assign, uint8_t* codes_out);
  int lut_host(int nq, const float* x, uint8_t* lut_out, float* mult_out);

 protected:
  GammaFileFormat gamma_format() const override;  // this engine's own index file (index_io.cu)
  int dump_gamma_extra(FILE* f) override;
  int load_gamma_extra(FILE* f) override;
  int64_t default_training_threshold() const override { return (int64_t)nlist_ * 256; }
  KMeansParams coarse_kmeans_params() const override;
  // the codes are built for the index metric: a request's metric_type does not change the ranking
  int search_metric(const SearchContext& ctx) const override { (void)ctx; return mp_.metric; }
  int resolve_nprobe(const SearchContext& ctx) const override;
  int train_extra(const float* xtrain, int64_t n, Scratch& s) override;
  int append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                   const std::vector<int>& add, Scratch& s) override;
  int scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, const void* xq_raw, int k,
               const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
               Scratch& s) override;

 private:
  cudaError_t encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st);
  int nb_;
  float* d_cb_ = nullptr;  // [16 d]
};

// host rows n x d (stride d) -> device rows n x dpad, the padding columns zeroed
cudaError_t upload_rows_padded(float* dst, const float* src, int64_t n, int d, int dpad, cudaStream_t st);

// gamma's GPU types over several devices (faiss::IndexShards, gamma_index_ivfpq_gpu.cc:269-298,
// gamma_index_ivfflat_gpu.cc:140-173): S shards of one IVF type, shard s on devices[s], holding the global vids
// v % S == s as local vids v / S (so a shard's (score, local vid) order is the (score, global vid) order).  The raw
// vectors stay in this index's store on devices[0], the primary device; shards hold only index structures.  Training
// runs once, on the primary device, and its state is copied to every shard.  A search runs the request checks, the
// coalescer, brute force and the realtime tail here, each shard's coarse search and scan on its own device and stream
// (bitmaps cut per shard on the device), and merges the S sorted key rows of every query on the primary device
// (index_shards.cu, DESIGN.md §7).
class ShardedIndex : public Index {
 public:
  ShardedIndex(const std::string& type, int d, const ModelParams& mp, const std::vector<int>& devices, int seg_shift,
               std::vector<std::unique_ptr<IvfIndex>> shards);
  ~ShardedIndex() override;
  int nshards() const { return (int)shards_.size(); }
  IvfIndex* shard(int s) { return shards_[s].get(); }
  int64_t training_threshold() const override { return shards_[0]->training_threshold(); }
  int train() override;
  int add_pending(const uint8_t* del_bitmap) override;
  int update_vector(int64_t vid, const void* x) override;
  int delete_vectors(const int64_t* vids, int64_t n) override;
  int purge_lists(float threshold, const uint8_t* del_bitmap, int64_t bitmap_bytes, int64_t* dropped) override;
  int reset_index() override;
  int64_t index_mem_bytes() const override;
  void charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) override;  // each shard its share
  // the unsharded type's file: list l is the merge of the shards' lists l by global vid, ids written as global vids
  int dump_gamma(const std::string& dir, const std::string& abs_name) override;
  // every shard reads the file and keeps its own entries
  int load_gamma(const std::string& dir, const std::string& abs_name, int64_t* load_num) override;

 protected:
  int search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                      unsigned long long* out_keys, Scratch& s) override;

 private:
  // shard 0's trained state (centroids, OPQ, PQ codebook and with it the precomputed table) to every other shard
  int sync_trained_state();
  // f's bitmaps (covering `bits` vids) cut into S per-shard bitmaps of shard_words(bits) words each, in s
  int64_t shard_words(int64_t bits) const;
  int split_bitmap(const uint32_t* src, int64_t bits, uint32_t** out, Scratch& s);
  // a stream per shard and their events, for one search at a time; pooled
  struct ShardLane {
    cudaEvent_t start = nullptr;        // primary device: queries and bitmaps are ready
    std::vector<cudaStream_t> st;       // shard s's device
    std::vector<cudaEvent_t> done;      // shard s's keys are on the primary device
  };
  ShardLane* shard_lane_acquire();
  void shard_lane_release(ShardLane* l);
  void shard_lane_free(ShardLane* l);
  std::vector<int> devices_;
  std::vector<std::unique_ptr<IvfIndex>> shards_;
  cudaEvent_t build_ev_ = nullptr;  // primary device: rows staged for a shard on build_stream_
  std::mutex shard_lane_mu_;
  std::vector<ShardLane*> shard_lanes_, free_shard_lanes_;
};

// reflector (index/reflector.h:68-80): type name -> index object
Index* create_index(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift);
// a GPU_IVFPQ / GPU_IVFFLAT index sharded over `devices` (at least two entries; an entry may repeat)
Index* create_sharded_index(const std::string& type, int d, const ModelParams& mp, const std::vector<int>& devices,
                            int seg_shift);

// cross-partition merge (router semantics, internal/client/client.go:1530-1609) on device:
// in: nparts x nq x k (dis, ids) sorted per partition; out: nq x k, ids = (part << 32) | local id
int merge_partitions_device(const float* dis, const int64_t* ids, int nparts, int nq, int k, int metric, float* out_dis,
                            int64_t* out_ids, cudaStream_t st);
// the same merge straight from the partitions' result keys [nparts][nq][k] (Index::search_device out_keys_dev)
int merge_partition_keys_device(const unsigned long long* keys, int nparts, int nq, int k, int metric, float* out_dis,
                                int64_t* out_ids, cudaStream_t st);

}  // namespace gb
