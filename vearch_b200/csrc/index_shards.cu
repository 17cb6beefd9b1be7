// ShardedIndex (index.h): gamma's GPU types over several devices, as faiss::IndexShards places them
// (gamma_index_ivfpq_gpu.cc:269-298, gamma_index_ivfflat_gpu.cc:140-173, gamma_gpu_index_base.h:145-155).
// Global vid v lives in shard v % S as local vid v / S.  Two kernels of its own: the per-shard cut of a vid bitmap and
// the S-way merge of the shards' sorted result keys.
#include "common.cuh"
#include "index.h"

#include <algorithm>

namespace gb {

#define GB_ALLOC(var, T, n, s)          \
  T* var = (s).alloc_n<T>((size_t)(n)); \
  if (!var) return -1

// ---- kernels ----------------------------------------------------------------------------------
// dst[s][w] bit b = src bit (32 w + b) S + s, for the global bits [0, bits); zero beyond them
__global__ void split_bitmap_kernel(const uint32_t* __restrict__ src, int64_t bits, int S, int64_t words,
                                    uint32_t* __restrict__ dst) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)S * words) return;
  const int s = (int)(i / words);
  const int64_t w = i - (int64_t)s * words;
  uint32_t out = 0;
  for (int b = 0; b < 32; b++) {
    const int64_t g = (w * 32 + b) * S + s;
    if (g < bits && ((src[g >> 5] >> (g & 31)) & 1u)) out |= 1u << b;
  }
  dst[i] = out;
}

// the key with its local vid rewritten to the global vid local * S + s; the sentinel stays the sentinel
__device__ __forceinline__ unsigned long long shard_key(unsigned long long key, int S, int s) {
  if (key == kKeySentinel) return key;
  const uint32_t local = (uint32_t)key;
  return (key & 0xFFFFFFFF00000000ull) | (uint32_t)(local * (uint32_t)S + (uint32_t)s);
}

// keys [S][nq][k]: per shard and query k keys sorted ascending (best first), sentinel padded.  out [nq][k] (prefilled
// with the sentinel) = the k smallest global keys of the S rows.  Global keys are distinct (a global vid lives in one
// shard), so a key's place in the merged row is its place in its own row plus, in every other row, the number of
// keys below it (a binary search); one thread per key, the ones placed at k or later write nothing.
__global__ void merge_shard_keys_kernel(const unsigned long long* __restrict__ keys, int S, int nq, int k,
                                        unsigned long long* __restrict__ out) {
  const int q = blockIdx.x, s = blockIdx.y;
  const unsigned long long* row = keys + ((int64_t)s * nq + q) * k;
  for (int p = threadIdx.x; p < k; p += blockDim.x) {
    const unsigned long long key = row[p];
    if (key == kKeySentinel) break;  // the rest of the row is padding
    const unsigned long long g = shard_key(key, S, s);
    int rank = p;
    for (int r = 0; r < S && rank < k; r++) {
      if (r == s) continue;
      const unsigned long long* o = keys + ((int64_t)r * nq + q) * k;
      int lo = 0, hi = k;  // first position whose key is not below g
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (shard_key(o[mid], S, r) < g)
          lo = mid + 1;
        else
          hi = mid;
      }
      rank += lo;
    }
    if (rank < k) out[(int64_t)q * k + rank] = g;
  }
}

static cudaError_t launch_split_bitmap(const uint32_t* src, int64_t bits, int S, int64_t words, uint32_t* dst,
                                       cudaStream_t st) {
  const int64_t n = (int64_t)S * words;
  if (n <= 0) return cudaSuccess;
  split_bitmap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, bits, S, words, dst);
  note_launch();
  return cudaGetLastError();
}

static cudaError_t launch_merge_shard_keys(const unsigned long long* keys, int S, int nq, int k, unsigned long long* out,
                                           cudaStream_t st) {
  if (nq <= 0) return cudaSuccess;
  cudaError_t e = launch_fill_u64(out, (int64_t)nq * k, kKeySentinel, st);
  if (e != cudaSuccess) return e;
  merge_shard_keys_kernel<<<dim3((unsigned)nq, (unsigned)S), std::min(256, (k + 31) / 32 * 32), 0, st>>>(keys, S, nq, k,
                                                                                                        out);
  note_launch();
  return cudaGetLastError();
}

// ---- construction ----------------------------------------------------------------------------
Index* create_sharded_index(const std::string& type, int d, const ModelParams& mp, const std::vector<int>& devices,
                            int seg_shift) {
  if (!is_gpu_index_type(type) || devices.size() < 2) {
    set_last_error("a sharded index is a GPU_IVFPQ or GPU_IVFFLAT index over two devices or more");
    return nullptr;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess) ndev = 0;
  for (int dev : devices)
    if (dev < 0 || dev >= ndev) {
      set_last_error("no CUDA device " + std::to_string(dev) + " (visible devices: " + std::to_string(ndev) + ")");
      return nullptr;
    }
  ModelParams smp = mp;
  smp.host_store = false;  // a shard's own store stays empty: the rows live in the sharded index's
  std::vector<std::unique_ptr<IvfIndex>> shards;
  for (size_t s = 0; s < devices.size(); s++) {
    Index* ix = create_index(type, d, smp, devices[s], seg_shift);  // the type's own parameter checks and messages
    if (!ix) return nullptr;
    shards.emplace_back(static_cast<IvfIndex*>(ix));
  }
  // peer access where the devices offer it: the copies between shards then go device to device
  for (int a : devices)
    for (int b : devices) {
      int can = 0;
      if (a == b || cudaDeviceCanAccessPeer(&can, a, b) != cudaSuccess || !can) continue;
      cudaSetDevice(a);
      if (cudaDeviceEnablePeerAccess(b, 0) != cudaSuccess) cudaGetLastError();  // already enabled is fine
    }
  return new ShardedIndex(type, d, mp, devices, seg_shift, std::move(shards));
}

ShardedIndex::ShardedIndex(const std::string& type, int d, const ModelParams& mp, const std::vector<int>& devices,
                           int seg_shift, std::vector<std::unique_ptr<IvfIndex>> shards)
    : Index(type, d, mp, devices[0], seg_shift), devices_(devices), shards_(std::move(shards)) {
  for (size_t s = 0; s < shards_.size(); s++) {  // before any row reaches a shard
    shards_[s]->shard_count_ = (int64_t)shards_.size();
    shards_[s]->shard_id_ = (int64_t)s;
  }
  cudaSetDevice(device_);
  cudaEventCreateWithFlags(&build_ev_, cudaEventDisableTiming);
}

ShardedIndex::~ShardedIndex() {
  drain_searches();
  quiesce();
  for (ShardLane* l : shard_lanes_) shard_lane_free(l);
  cudaSetDevice(device_);
  if (build_ev_) cudaEventDestroy(build_ev_);
  for (auto& sh : shards_) {
    cudaSetDevice(sh->device());
    sh.reset();
  }
  cudaSetDevice(device_);
}

ShardedIndex::ShardLane* ShardedIndex::shard_lane_acquire() {
  {
    std::lock_guard<std::mutex> g(shard_lane_mu_);
    if (!free_shard_lanes_.empty()) {
      ShardLane* l = free_shard_lanes_.back();
      free_shard_lanes_.pop_back();
      return l;
    }
  }
  ShardLane* l = new ShardLane;
  cudaError_t e = cudaSetDevice(device_);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&l->start, cudaEventDisableTiming);
  for (size_t s = 0; s < shards_.size() && e == cudaSuccess; s++) {
    l->st.push_back(nullptr);
    l->done.push_back(nullptr);
    e = cudaSetDevice(devices_[s]);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&l->st[s], cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&l->done[s], cudaEventDisableTiming);
  }
  cudaSetDevice(device_);
  if (e != cudaSuccess) {
    set_last_error(std::string("shard streams: ") + cudaGetErrorString(e));
    shard_lane_free(l);
    return nullptr;
  }
  std::lock_guard<std::mutex> g(shard_lane_mu_);
  shard_lanes_.push_back(l);
  return l;
}
void ShardedIndex::shard_lane_release(ShardLane* l) {
  std::lock_guard<std::mutex> g(shard_lane_mu_);
  free_shard_lanes_.push_back(l);
}
void ShardedIndex::shard_lane_free(ShardLane* l) {
  for (size_t s = 0; s < l->st.size(); s++) {
    cudaSetDevice(devices_[s]);
    if (l->st[s]) cudaStreamSynchronize(l->st[s]), cudaStreamDestroy(l->st[s]);
    if (l->done[s]) cudaEventDestroy(l->done[s]);
  }
  cudaSetDevice(device_);
  if (l->start) cudaEventDestroy(l->start);
  delete l;
}

// ---- training and the lists ------------------------------------------------------------------
int ShardedIndex::sync_trained_state() {
  IvfIndex* s0 = shards_[0].get();
  std::vector<float> cent((size_t)s0->nlist() * d_), pq, opq;
  if (s0->get_centroids(cent.data())) return -1;
  IvfPqBase* pq0 = dynamic_cast<IvfPqBase*>(s0);
  IVFPQIndex* opq0 = dynamic_cast<IVFPQIndex*>(s0);
  if (pq0) {
    pq.resize((size_t)pq0->M() * pq0->ksub() * pq0->dsub());
    if (pq0->get_pq_centroids(pq.data())) return -1;
  }
  if (opq0 && opq0->has_opq()) {
    opq.resize((size_t)d_ * d_);
    if (opq0->get_opq(opq.data())) return -1;
  }
  for (size_t s = 1; s < shards_.size(); s++) {
    IvfIndex* sh = shards_[s].get();
    if (!opq.empty() && static_cast<IVFPQIndex*>(sh)->set_opq(opq.data())) return -1;
    if (sh->set_centroids(cent.data(), sh->nlist())) return -1;
    if (pq0 && static_cast<IvfPqBase*>(sh)->set_pq_centroids(pq.data())) return -1;  // and the precomputed table
  }
  cudaSetDevice(device_);
  return 0;
}

int ShardedIndex::train() {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (trained_) return 0;
  cudaSetDevice(device_);
  GB_CUDA(cudaStreamSynchronize(build_stream_));  // the appended rows, which shard 0 reads on its own stream
  // trained state set on shard 0 (the engine's Load) is taken as it is
  if (!shards_[0]->trained() && shards_[0]->train_on(*store_)) return -1;
  if (sync_trained_state()) return -1;
  std::unique_lock<std::shared_mutex> lk(mu_);
  trained_ = true;
  return 0;
}

int ShardedIndex::add_pending(const uint8_t* del_bitmap, int64_t rows) {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (!trained_) return 0;
  const int S = nshards();
  const int64_t BATCH = 1 << 20, ld = store_->stride();
  for (;;) {
    cudaSetDevice(device_);
    int64_t vid0 = indexed_count_, n = 0;
    const unsigned char* x = nullptr;
    Scratch s(build_stream_);
    {  // the batches of IvfIndex::add_pending
      std::shared_lock<std::shared_mutex> lk(mu_);
      const int64_t end = rows < 0 ? store_->size() : std::min(rows, store_->size());
      if (vid0 >= end) break;
      const int64_t span = store_->on_host() ? BATCH : store_->seg_rows();
      int64_t off = vid0 & (span - 1);
      n = std::min<int64_t>(std::min(end - vid0, span - off), BATCH);
      x = static_cast<const unsigned char*>(store_rows_dev(vid0, n, s));
      if (!x) return -1;
    }
    for (int i = 0; i < S; i++) {
      // shard i's rows of the batch, global vids first, first + S, ...: gathered on the primary device, then copied
      const int64_t first = vid0 + ((i - vid0 % S) % S + S) % S;
      if (first >= vid0 + n) continue;
      const int64_t cnt = (vid0 + n - first + S - 1) / S;
      cudaSetDevice(device_);
      void* g = s.alloc((size_t)cnt * ld);
      if (!g) return -1;
      GB_CUDA(cudaMemcpy2DAsync(g, ld, x + (first - vid0) * ld, (size_t)S * ld, ld, cnt, cudaMemcpyDeviceToDevice,
                                build_stream_));
      GB_CUDA(cudaEventRecord(build_ev_, build_stream_));
      IvfIndex* sh = shards_[i].get();
      cudaSetDevice(sh->device());
      Scratch ss(sh->build_stream_);
      GB_CUDA(cudaStreamWaitEvent(sh->build_stream_, build_ev_, 0));
      void* xs = ss.alloc((size_t)cnt * ld);
      if (!xs) return -1;
      GB_CUDA(cudaMemcpyPeerAsync(xs, sh->device(), g, device_, (size_t)cnt * ld, sh->build_stream_));
      std::lock_guard<std::mutex> sbg(sh->build_mu_);
      if (sh->index_batch(xs, cnt, first / S, del_bitmap)) return -1;  // waits for its stream: g and xs are free after
      sh->indexed_count_ = first / S + cnt;
    }
    indexed_count_ += n;
  }
  for (auto& sh : shards_)
    if (sh->lists_ && sh->lists_->compact_due()) {
      cudaSetDevice(sh->device());
      std::unique_lock<std::shared_mutex> lk(sh->mu_);
      if (sh->compact_locked()) return -1;
    }
  cudaSetDevice(device_);
  return 0;
}

int ShardedIndex::update_vector(int64_t vid, const void* x) {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (Index::update_vector(vid, x)) return -1;  // the raw row, on the primary device
  if (!trained_ || vid >= indexed_count_) return 0;
  const int S = nshards();
  IvfIndex* sh = shards_[vid % S].get();
  Scratch s(build_stream_);
  const void* xr = store_rows_dev(vid, 1, s);
  if (!xr) return -1;
  GB_CUDA(cudaEventRecord(build_ev_, build_stream_));
  cudaSetDevice(sh->device());
  Scratch ss(sh->build_stream_);
  GB_CUDA(cudaStreamWaitEvent(sh->build_stream_, build_ev_, 0));
  void* xs = ss.alloc((size_t)store_->stride());
  if (!xs) return -1;
  GB_CUDA(cudaMemcpyPeerAsync(xs, sh->device(), xr, device_, (size_t)store_->stride(), sh->build_stream_));
  std::lock_guard<std::mutex> sbg(sh->build_mu_);
  const int rc = sh->reindex_vector(vid / S, xs);  // waits for its stream
  cudaSetDevice(device_);
  return rc;
}

int ShardedIndex::delete_vectors(const int64_t* vids, int64_t n) {
  std::lock_guard<std::mutex> bg(build_mu_);
  const int S = nshards();
  std::vector<std::vector<int64_t>> local(S);
  for (int64_t i = 0; i < n; i++)
    if (vids[i] >= 0) local[vids[i] % S].push_back(vids[i] / S);
  for (int s = 0; s < S; s++)
    if (!local[s].empty() && shards_[s]->delete_vectors(local[s].data(), (int64_t)local[s].size())) return -1;
  return 0;
}

int64_t ShardedIndex::shard_words(int64_t bits) const {
  const int64_t S = nshards();
  return ((bits + S - 1) / S + 31) / 32 + 1;
}
int ShardedIndex::split_bitmap(const uint32_t* src, int64_t bits, uint32_t** out, Scratch& s) {
  const int64_t words = shard_words(bits);
  GB_ALLOC(dst, uint32_t, (size_t)nshards() * words, s);
  GB_CUDA(launch_split_bitmap(src, bits, nshards(), words, dst, s.stream()));
  *out = dst;
  return 0;
}

int ShardedIndex::purge_lists(float threshold, const uint8_t* del_bitmap, int64_t bitmap_bytes, int64_t* dropped) {
  if (dropped) *dropped = 0;
  std::lock_guard<std::mutex> bg(build_mu_);
  const int S = nshards();
  std::vector<std::vector<int>> sel(S);
  bool any = false;
  for (int i = 0; i < S; i++) {
    std::lock_guard<std::mutex> sbg(shards_[i]->build_mu_);
    sel[i] = shards_[i]->purge_candidates(threshold);
    any = any || !sel[i].empty();
  }
  if (!any) return 0;
  cudaSetDevice(device_);
  Scratch s(build_stream_);
  SearchContext ctx;
  ctx.del_bitmap = del_bitmap;
  ctx.bitmap_bits = del_bitmap ? bitmap_bytes * 8 : 0;
  FilterArgs f;
  uint32_t* split = nullptr;
  int64_t bits = 0;
  {
    std::shared_lock<std::shared_mutex> lk(mu_);
    bits = std::max<int64_t>(ctx.bitmap_bits, store_->size());  // what upload_bitmaps covers
    if (upload_bitmaps(ctx, &f, s)) return -1;
  }
  if (f.del_bits && split_bitmap(f.del_bits, bits, &split, s)) return -1;
  GB_CUDA(cudaEventRecord(build_ev_, build_stream_));
  const int64_t words = shard_words(bits);
  int64_t total = 0;
  for (int i = 0; i < S; i++) {
    if (sel[i].empty()) continue;
    IvfIndex* sh = shards_[i].get();
    std::lock_guard<std::mutex> sbg(sh->build_mu_);
    cudaSetDevice(sh->device());
    Scratch ss(sh->build_stream_);
    GB_CUDA(cudaStreamWaitEvent(sh->build_stream_, build_ev_, 0));
    uint32_t* bits_i = nullptr;
    if (split) {
      bits_i = ss.alloc_n<uint32_t>((size_t)words);
      if (!bits_i) return -1;
      GB_CUDA(cudaMemcpyPeerAsync(bits_i, sh->device(), split + (size_t)i * words, device_, (size_t)words * 4,
                                  sh->build_stream_));
    }
    std::unique_lock<std::shared_mutex> lk(sh->mu_);
    int64_t d = 0;
    if (sh->purge_locked(sel[i], bits_i, &d)) return -1;  // waits for its stream
    total += d;
  }
  cudaSetDevice(device_);
  if (dropped) *dropped = total;
  return 0;
}

int ShardedIndex::reset_index() {
  std::lock_guard<std::mutex> bg(build_mu_);
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  for (auto& sh : shards_)
    if (sh->reset_index()) return -1;
  cudaSetDevice(device_);
  indexed_count_ = 0;
  trained_ = false;
  return 0;
}

int64_t ShardedIndex::index_mem_bytes() const {
  int64_t b = 0;
  for (auto& sh : shards_) b += sh->index_mem_bytes();
  return b;
}
void ShardedIndex::charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) {
  const int S = nshards();  // vid v goes to shard v % S
  for (int s = 0; s < S; s++) shards_[s]->charge_index_rows(rows / S + (s < rows % S ? 1 : 0), out);
}

// ---- gamma's index file ----------------------------------------------------------------------
int ShardedIndex::capture_gamma(GammaImage* img) {
  if (!trained_) return 0;
  std::lock_guard<std::mutex> bg(build_mu_);
  IvfIndex* s0 = shards_[0].get();
  std::vector<IvfIndex*> shards;
  for (auto& sh : shards_) shards.push_back(sh.get());
  int rc;
  {
    std::lock_guard<std::mutex> sbg(s0->build_mu_);  // the other shards' lists change only under build_mu_, held here
    rc = s0->capture_head(indexed_count_, img);
    if (!rc) rc = IvfIndex::capture_lists(shards, img);
  }
  cudaSetDevice(device_);
  return rc;
}

int ShardedIndex::load_gamma(const std::string& dir, const std::string& abs_name, int64_t* load_num) {
  *load_num = 0;
  std::lock_guard<std::mutex> bg(build_mu_);
  int64_t rows;
  {
    std::shared_lock<std::shared_mutex> lk(mu_);
    rows = store_->size();
  }
  const GammaFileFormat gf = shards_[0]->gamma_format();
  if (FILE* f = fopen((dir + "/" + abs_name + "/" + gf.file).c_str(), "rb")) {
    fclose(f);
  } else {
    return 0;  // "isn't existed, skip loading": trained again after load (ivfflat.cc:846-850)
  }
  int64_t file_indexed = 0, live = 0;
  for (auto& sh : shards_) {
    int64_t n = 0, fi = 0;
    if (sh->load_gamma_part(dir, abs_name, rows, &n, &fi)) {
      // as an unsharded index whose file is refused: no list content from the file, the trained state kept (the file's
      // when its header was read, else what the shards held), the same on every shard
      const std::string err = last_error();
      for (auto& r : shards_) r->clear_lists();
      if (shards_[0]->trained()) sync_trained_state();
      set_last_error(err);
      cudaSetDevice(device_);
      return -1;
    }
    file_indexed = fi, live += n;
  }
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  trained_ = shards_[0]->trained();
  // IvFl: the file's indexed count; IwPQ: its live entries, which the shards counted between them
  indexed_count_ = gf.indexed_count ? file_indexed : live;
  *load_num = indexed_count_;
  return 0;
}

// ---- search ------------------------------------------------------------------------------------
int ShardedIndex::search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                                  unsigned long long* out_keys, Scratch& s) {
  const int S = nshards();
  cudaStream_t pst = s.stream();
  const int64_t bits = std::max<int64_t>(ctx.bitmap_bits, store_->size());  // what upload_bitmaps covered
  const int64_t words = shard_words(bits);
  uint32_t* split[2] = {nullptr, nullptr};
  if (f.del_bits && split_bitmap(f.del_bits, bits, &split[0], s)) return -1;
  if (f.filter_bits && split_bitmap(f.filter_bits, bits, &split[1], s)) return -1;
  const size_t qbytes = (size_t)nq * store_->stride(), kn = (size_t)nq * k;
  GB_ALLOC(all, unsigned long long, (size_t)S * kn, s);
  ShardLane* ln = shard_lane_acquire();
  if (!ln) return -1;
  int rc = 0;
  if (cudaEventRecord(ln->start, pst) != cudaSuccess) rc = -1;
  int touched = 0;  // shards whose stream waited on `start`: each records done[i] after whatever it enqueued
  // a cancelled search enqueues no further shard; the shards already enqueued poll the word in their kernels
  for (int i = 0; i < S && rc == 0 && !(i > 0 && cancel_is_set(f.cancel.word)); i++) {
    IvfIndex* sh = shards_[i].get();
    const int dev = devices_[i];
    cudaStream_t sst = ln->st[i];
    cudaSetDevice(dev);
    std::shared_lock<std::shared_mutex> lk(sh->mu_);  // a mutation of the shard drains what this enqueues
    Scratch ss(sst);
    cudaError_t e = cudaStreamWaitEvent(sst, ln->start, 0);
    if (e == cudaSuccess) touched++;
    const void* xq_i = xq;
    FilterArgs fi = f;
    // the shard's own `seen` flag, on its device
    if (e == cudaSuccess && cancel_poll_init(f.cancel.word, &fi, ss)) e = cudaErrorMemoryAllocation;
    fi.del_bits = split[0] ? split[0] + (size_t)i * words : nullptr;
    fi.filter_bits = split[1] ? split[1] + (size_t)i * words : nullptr;
    if (dev != device_ && e == cudaSuccess) {  // the queries and this shard's bitmaps on its device
      void* xc = ss.alloc(qbytes);
      e = xc ? cudaMemcpyPeerAsync(xc, dev, xq, device_, qbytes, sst) : cudaErrorMemoryAllocation;
      xq_i = xc;
      for (int w = 0; w < 2 && e == cudaSuccess; w++) {
        const uint32_t*& dst = w == 0 ? fi.del_bits : fi.filter_bits;
        if (!dst) continue;
        uint32_t* bc = ss.alloc_n<uint32_t>((size_t)words);
        e = bc ? cudaMemcpyPeerAsync(bc, dev, dst, device_, (size_t)words * 4, sst) : cudaErrorMemoryAllocation;
        dst = bc;
      }
    }
    unsigned long long* keys = nullptr;
    if (e != cudaSuccess) {
      set_last_error(std::string("shard ") + std::to_string(i) + ": staging: " + cudaGetErrorString(e));
      rc = -1;
    } else if (!(keys = ss.alloc_n<unsigned long long>(kn))) {
      rc = -1;
    } else {
      rc = sh->search_keys_dev(ctx, fi, metric, nq, xq_i, k, keys, ss);
    }
    if (rc == 0 && (e = cudaMemcpyPeerAsync(all + (size_t)i * kn, device_, keys, dev, kn * 8, sst)) != cudaSuccess) {
      set_last_error(std::string("shard ") + std::to_string(i) + ": result copy: " + cudaGetErrorString(e));
      rc = -1;
    }
    if (i < touched) cudaEventRecord(ln->done[i], sst);
    sh->note_search_enqueued(sst);
  }
  cudaSetDevice(device_);
  for (int i = 0; i < touched; i++) cudaStreamWaitEvent(pst, ln->done[i], 0);  // `all` and the lane are free after
  shard_lane_release(ln);
  last_scan_kernel_ = shards_[0]->last_scan_kernel();
  if (rc) return rc;
  StageScope st(this, "shard_merge", pst);
  GB_CUDA(launch_merge_shard_keys(all, S, nq, k, out_keys, pst));
  return 0;
}

}  // namespace gb
