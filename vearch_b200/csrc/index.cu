// Host orchestration of the hot path (see index.h).  Reference call sites are cited inline.
#include <cuda.h>

#include "index.h"

#include <float.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <random>

#include "common.cuh"
#include "mem_ledger.h"

namespace gb {

// ------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
const char* last_error() { return g_last_error.c_str(); }

static inline int64_t round_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

// SM count of a device, queried once (grids of the persistent kernels, work-splitting heuristics)
static int sm_count(int device) {
  static std::mutex mu;
  static std::vector<int> cache;
  std::lock_guard<std::mutex> lk(mu);
  if ((int)cache.size() <= device) cache.resize(device + 1, 0);
  if (!cache[device]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
    cache[device] = n;
  }
  return cache[device];
}

static cudaStream_t thread_stream(int device) {
  static thread_local cudaStream_t st[64] = {nullptr};
  if (device < 0 || device >= 64) return nullptr;
  if (!st[device]) {
    cudaSetDevice(device);
    cudaStreamCreateWithFlags(&st[device], cudaStreamNonBlocking);
  }
  return st[device];
}

// A second stream beside thread_stream(device), for work a search forks off its own stream and joins back (ForkJoin),
// with the two events that order it.  Same (default) priority as the search stream: the side chain's blocks then take
// what the search stream's grid leaves free instead of displacing its CTAs (at high priority the IVF-PQ phase A slowed
// by as much as the side chain saved, BASELINE.md section 4).  Per thread, like the search stream, so concurrent
// searches never share one.
struct SideStream {
  cudaStream_t st = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
};
static const SideStream* thread_side_stream(int device) {
  static thread_local SideStream ss[64];
  if (device < 0 || device >= 64) return nullptr;
  SideStream& s = ss[device];
  if (!s.st) {
    cudaSetDevice(device);
    if (cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming) != cudaSuccess ||
        cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking) != cudaSuccess) {
      s.st = nullptr;
      return nullptr;
    }
  }
  return &s;
}

// Work on a side stream between a fork from the parent stream and the join back into it.  Scratch is allocated and
// freed stream-ordered on the parent, so what the side stream uses must be allocated before fork(), and every exit path
// joins (the destructor) before that scratch is freed.
class ForkJoin {
 public:
  ForkJoin(cudaStream_t parent, const SideStream& side) : parent_(parent), side_(side) {}
  ForkJoin(const ForkJoin&) = delete;
  ForkJoin& operator=(const ForkJoin&) = delete;
  ~ForkJoin() { join(); }
  cudaError_t fork() {
    cudaError_t e = cudaEventRecord(side_.fork, parent_);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(side_.st, side_.fork, 0);
    if (e == cudaSuccess) forked_ = true;
    return e;
  }
  cudaError_t join() {
    if (!forked_) return cudaSuccess;
    forked_ = false;
    cudaError_t e = cudaEventRecord(side_.join, side_.st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(parent_, side_.join, 0);
    if (e != cudaSuccess) cudaStreamSynchronize(side_.st);  // the parent cannot wait for it: nothing may still run there
    return e;
  }
  cudaStream_t side() const { return side_.st; }

 private:
  cudaStream_t parent_;
  const SideStream& side_;
  bool forked_ = false;
};

// ------------------------------------------------------------------------------------------
Scratch::~Scratch() {
  for (void* p : ptrs_) cudaFreeAsync(p, st_);
}
void* Scratch::alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0) bytes = 16;
  cudaError_t e = cudaMallocAsync(&p, bytes, st_);
  if (e != cudaSuccess) {
    set_last_error(std::string("cudaMallocAsync(") + std::to_string(bytes) + "): " + cudaGetErrorString(e));
    return nullptr;
  }
  ptrs_.push_back(p);
  return p;
}
#define GB_ALLOC(var, T, n, s)                \
  T* var = (s).alloc_n<T>((size_t)(n));       \
  if (!var) return -1

cudaError_t upload_rows_padded(float* dst, const float* src, int64_t n, int d, int dpad, cudaStream_t st) {
  if (dpad != d) {
    const cudaError_t e = cudaMemsetAsync(dst, 0, (size_t)n * dpad * 4, st);
    if (e != cudaSuccess) return e;
  }
  return cudaMemcpy2DAsync(dst, (size_t)dpad * 4, src, (size_t)d * 4, (size_t)d * 4, n, cudaMemcpyHostToDevice, st);
}

// ------------------------------------------------------------------------------------------
// Segments are VIRTUAL address ranges of seg_rows rows; physical HBM is mapped into them in chunks as rows
// arrive (CUDA virtual memory management: cuMemAddressReserve / cuMemCreate / cuMemMap, reached through
// cudaGetDriverEntryPoint so the library still links only the static runtime).  A 100-document partition
// therefore costs one 2 MiB granule, not a 1M-row segment (3 GiB at d = 768), while row addresses stay
// stable and segment-contiguous for the kernels (MemoryRawVector grows incrementally as well,
// vector/memory_raw_vector.cc:152-240).  Without VMM support a segment is one cudaMalloc as before.
namespace {
struct VmmApi {
  CUresult (*reserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*addr_free)(CUdeviceptr, size_t) = nullptr;
  CUresult (*create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*release)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*unmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*set_access)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*granularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  bool ok = false;
};
const VmmApi& vmm_api() {
  static const VmmApi api = [] {
    VmmApi a;
    const char* off = getenv("GB_VMM");
    if (off && atoi(off) == 0) return a;
    auto get = [](const char* name, void** fn) {
      cudaDriverEntryPointQueryResult q;
      return cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess && *fn;
    };
    a.ok = get("cuMemAddressReserve", (void**)&a.reserve) && get("cuMemAddressFree", (void**)&a.addr_free) &&
           get("cuMemCreate", (void**)&a.create) && get("cuMemRelease", (void**)&a.release) && get("cuMemMap", (void**)&a.map) &&
           get("cuMemUnmap", (void**)&a.unmap) && get("cuMemSetAccess", (void**)&a.set_access) &&
           get("cuMemGetAllocationGranularity", (void**)&a.granularity);
    cudaGetLastError();
    return a;
  }();
  return api;
}
// the VMM allocation granularity on a device; 0 without VMM
size_t vmm_granularity(int device) {
  static std::atomic<size_t> cache[64];
  if (device >= 0 && device < 64 && cache[device].load()) return cache[device].load();
  const VmmApi& api = vmm_api();
  if (!api.ok) return 0;
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  size_t gran = 0;
  if (api.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS) return 0;
  if (device >= 0 && device < 64) cache[device] = gran;
  return gran;
}
// the next chunk mapped into a segment with `mapped` of va_bytes mapped and `need` wanted: geometric steps (a quarter of
// what is mapped, at least one granule, at most 256 MiB), never past the segment
size_t map_step(size_t mapped, size_t need, size_t gran, size_t va_bytes) {
  size_t step = std::max(gran, std::min<size_t>(mapped / 4, (size_t)256 << 20));
  step = (size_t)round_up((int64_t)std::max(step, std::min(need - mapped, (size_t)256 << 20)), (int64_t)gran);
  return std::min(step, va_bytes - mapped);
}
}  // namespace

RawStore::RawStore(int row_bytes, int seg_shift, bool host)
    : row_bytes_(row_bytes), stride_((int)round_up(row_bytes, 16)), seg_shift_(host ? std::min(seg_shift, kHostSegShift) : seg_shift), host_(host) {
  mem::dev_malloc(&d_segs_, sizeof(float*) * kMaxSegs);
  cudaGetDevice(&device_);
}
RawStore::~RawStore() {
  const VmmApi& api = vmm_api();
  for (Seg& sg : segs_) {
    if (host_) {
      mem::host_free(sg.base);
      continue;
    }
    if (!sg.vmm) {
      mem::dev_free(sg.base);
      continue;
    }
    size_t off = 0;
    for (auto& c : sg.chunks) {
      api.unmap((CUdeviceptr)sg.base + off, c.second);
      api.release(c.first);
      mem::charge(device_, -(int64_t)c.second);
      off += c.second;
    }
    api.addr_free((CUdeviceptr)sg.base, sg.va_bytes);
  }
  mem::dev_free(d_segs_);
}
int RawStore::new_segment() {
  if ((int)segs_.size() >= kMaxSegs) {
    set_last_error("raw store: too many segments");
    return -1;
  }
  Seg sg;
  const size_t bytes = (size_t)seg_rows() * stride_;
  if (host_) {  // pinned, mapped into every device's address space; kernels read it through the device pointer
    GB_CUDA(mem::host_alloc(reinterpret_cast<void**>(&sg.base), bytes, cudaHostAllocMapped | cudaHostAllocPortable));
    memset(sg.base, 0, bytes);  // pad columns must read as zero
    unsigned char* dev = nullptr;
    const cudaError_t e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&dev), sg.base, 0);
    if (e != cudaSuccess) {
      mem::host_free(sg.base);
      set_last_error(std::string("raw store: cudaHostGetDevicePointer: ") + cudaGetErrorString(e));
      return -1;
    }
    sg.mapped = bytes;
    host_bytes_ += (int64_t)bytes;
    segs_.push_back(sg);
    GB_CUDA(cudaMemcpy(d_segs_ + segs_.size() - 1, &dev, sizeof(dev), cudaMemcpyHostToDevice));
    return 0;
  }
  const VmmApi& api = vmm_api();
  if (api.ok) {
    const size_t gran = vmm_granularity(device_);
    if (gran > 0) {
      sg.gran = gran;
      sg.va_bytes = (size_t)round_up((int64_t)bytes, (int64_t)gran);
      CUdeviceptr p = 0;
      if (api.reserve(&p, sg.va_bytes, 0, 0, 0) == CUDA_SUCCESS) {
        sg.base = reinterpret_cast<unsigned char*>(p);
        sg.vmm = true;
      }
    }
  }
  if (!sg.vmm) {  // no VMM: the whole segment at once
    GB_CUDA(mem::dev_malloc(&sg.base, bytes));
    GB_CUDA(cudaMemset(sg.base, 0, bytes));
    sg.mapped = bytes;
    phys_bytes_ += (int64_t)bytes;
  }
  segs_.push_back(sg);
  GB_CUDA(cudaMemcpy(d_segs_ + segs_.size() - 1, &sg.base, sizeof(sg.base), cudaMemcpyHostToDevice));
  return 0;
}
// physical memory behind the first `rows` rows of segment si
int RawStore::map_rows(int si, int64_t rows) {
  Seg& sg = segs_[si];
  const size_t need = (size_t)rows * stride_;
  if (need <= sg.mapped) return 0;
  const VmmApi& api = vmm_api();
  while (sg.mapped < need) {
    const size_t step = map_step(sg.mapped, need, sg.gran, sg.va_bytes);
    CUmemAllocationProp prop = {};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device_;
    CUmemGenericAllocationHandle hnd;
    if (api.create(&hnd, step, &prop, 0) != CUDA_SUCCESS) {
      set_last_error("raw store: out of device memory (cuMemCreate)");
      return -1;
    }
    const CUdeviceptr at = (CUdeviceptr)sg.base + sg.mapped;
    CUmemAccessDesc acc = {};
    acc.location = prop.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (api.map(at, step, 0, hnd, 0) != CUDA_SUCCESS || api.set_access(at, step, &acc, 1) != CUDA_SUCCESS) {
      api.release(hnd);
      set_last_error("raw store: cuMemMap failed");
      return -1;
    }
    GB_CUDA(cudaMemset(reinterpret_cast<void*>(at), 0, step));  // pad columns must read as zero
    sg.chunks.emplace_back(hnd, step);
    mem::charge(device_, (int64_t)step);
    sg.mapped += step;
    phys_bytes_ += (int64_t)step;
  }
  return 0;
}
int RawStore::ensure(int64_t n_total) {
  while ((int64_t)segs_.size() * seg_rows() < n_total)
    if (new_segment()) return -1;
  for (int si = (int)(n_ >> seg_shift_); si < (int)segs_.size(); si++) {
    const int64_t rows = std::min<int64_t>(seg_rows(), n_total - (int64_t)si * seg_rows());
    if (rows > 0 && map_rows(si, rows)) return -1;
  }
  return 0;
}
int64_t RawStore::growth_bytes(int64_t n_total, int64_t* rows) const {
  const size_t seg_bytes = (size_t)seg_rows() * stride_;
  const size_t gran = host_ ? 0 : vmm_granularity(device_);
  int64_t b = 0;
  for (int64_t si = n_ >> seg_shift_; si * seg_rows() < n_total; si++) {
    const size_t need = (size_t)std::min<int64_t>(seg_rows(), n_total - si * seg_rows()) * stride_;
    const bool exists = si < (int64_t)segs_.size();
    if (exists ? !segs_[si].vmm : (host_ || !gran)) {  // a whole segment at once, or already there
      if (!exists) b += (int64_t)seg_bytes;
      continue;
    }
    size_t mapped = exists ? segs_[si].mapped : 0;
    const size_t sg_gran = exists ? segs_[si].gran : gran;
    const size_t va = exists ? segs_[si].va_bytes : (size_t)round_up((int64_t)seg_bytes, (int64_t)gran);
    while (mapped < need) {
      const size_t step = map_step(mapped, need, sg_gran, va);
      mapped += step;
      b += (int64_t)step;
    }
  }
  if (rows) *rows = b / stride_;
  if (shadow_) b += shadow_->growth_bytes(n_total, nullptr);
  return b;
}
// Host placement: the segments are ordinary (pinned) host memory, so host rows move with memcpy and device rows with
// device-to-host copies.  A search may still be reading a row when update_host overwrites it: the caller holds the
// index lock exclusively and has drained in-flight searches first (Index::update_vector).
int RawStore::append_host(const void* xv, int64_t n, cudaStream_t st) {
  const unsigned char* x = static_cast<const unsigned char*>(xv);
  if (ensure(n_ + n)) return -1;
  int64_t done = 0;
  while (done < n) {
    int64_t vid = n_ + done;
    int64_t si = vid >> seg_shift_, off = vid & (seg_rows() - 1);
    int64_t cnt = std::min(n - done, seg_rows() - off);
    if (host_) {
      for (int64_t i = 0; i < cnt; i++) memcpy(segs_[si].base + (off + i) * stride_, x + (done + i) * row_bytes_, row_bytes_);
    } else {
      GB_CUDA(cudaMemcpy2DAsync(segs_[si].base + off * stride_, stride_, x + done * row_bytes_, row_bytes_, row_bytes_,
                                (size_t)cnt, cudaMemcpyHostToDevice, st));
      if (encode_shadow(si, off, cnt, st)) return -1;
    }
    done += cnt;
  }
  GB_CUDA(cudaStreamSynchronize(st));
  n_ += n;
  if (shadow_) shadow_->n_ = n_;
  return 0;
}
int RawStore::append_device(const void* xv, int64_t ld_bytes, int64_t n, cudaStream_t st) {
  const unsigned char* x = static_cast<const unsigned char*>(xv);
  if (ensure(n_ + n)) return -1;
  int64_t done = 0;
  while (done < n) {
    int64_t vid = n_ + done;
    int64_t si = vid >> seg_shift_, off = vid & (seg_rows() - 1);
    int64_t cnt = std::min(n - done, seg_rows() - off);
    GB_CUDA(cudaMemcpy2DAsync(segs_[si].base + off * stride_, stride_, x + done * ld_bytes, (size_t)ld_bytes, row_bytes_,
                              (size_t)cnt, host_ ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, st));
    if (encode_shadow(si, off, cnt, st)) return -1;
    done += cnt;
  }
  GB_CUDA(cudaStreamSynchronize(st));
  n_ += n;
  if (shadow_) shadow_->n_ = n_;
  return 0;
}
int RawStore::update_host(int64_t vid, const void* x, cudaStream_t st) {
  if (vid < 0 || vid >= n_) return -1;
  int64_t si = vid >> seg_shift_, off = vid & (seg_rows() - 1);
  if (host_) {
    memcpy(segs_[si].base + off * stride_, x, row_bytes_);
    return 0;
  }
  GB_CUDA(cudaMemcpyAsync(segs_[si].base + off * stride_, x, row_bytes_, cudaMemcpyHostToDevice, st));
  if (encode_shadow(si, off, 1, st)) return -1;
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}
void RawStore::enable_shadow() {
  if (host_ || shadow_ || n_ > 0 || row_bytes_ % 4) return;
  const int cols16 = (int)round_up(stride_ / 4, 16);
  shadow_.reset(new RawStore(cols16 + 16, seg_shift_, false));
}
// the shadow rows of fp32 rows [off, off + cnt) of segment si, ordered on st after their copy
int RawStore::encode_shadow(int64_t si, int64_t off, int64_t cnt, cudaStream_t st) {
  if (!shadow_) return 0;
  if (shadow_->ensure((si << seg_shift_) + off + cnt)) return -1;
  GB_CUDA(launch_shadow_encode(seg((int)si) + off * stride_ / 4, stride_ / 4, cnt, (int)(stride_ / 4),
                               shadow_->segs_[si].base + off * shadow_->stride_, shadow_->stride_, st));
  return 0;
}
int RawStore::get_host(int64_t vid, void* out) const {
  if (vid < 0 || vid >= n_) return -1;
  int64_t si = vid >> seg_shift_, off = vid & (seg_rows() - 1);
  if (host_) {
    memcpy(out, segs_[si].base + off * stride_, row_bytes_);
    return 0;
  }
  GB_CUDA(cudaMemcpy(out, segs_[si].base + off * stride_, row_bytes_, cudaMemcpyDeviceToHost));
  return 0;
}
int RawStore::get_rows_host(int64_t start, int64_t n, void* outv) const {
  unsigned char* out = static_cast<unsigned char*>(outv);
  if (start < 0 || n < 0 || start + n > n_) return -1;
  int64_t done = 0;
  while (done < n) {
    int64_t vid = start + done;
    int64_t si = vid >> seg_shift_, off = vid & (seg_rows() - 1);
    int64_t cnt = std::min(n - done, seg_rows() - off);
    if (host_) {
      for (int64_t i = 0; i < cnt; i++) memcpy(out + (done + i) * row_bytes_, segs_[si].base + (off + i) * stride_, row_bytes_);
    } else {
      GB_CUDA(cudaMemcpy2D(out + done * row_bytes_, row_bytes_, segs_[si].base + off * stride_, stride_, row_bytes_,
                           (size_t)cnt, cudaMemcpyDeviceToHost));
    }
    done += cnt;
  }
  return 0;
}
cudaError_t RawStore::copy_rows_to_device(int64_t start, int64_t n, void* dstv, cudaStream_t st) const {
  unsigned char* dst = static_cast<unsigned char*>(dstv);
  int64_t done = 0;
  while (done < n) {
    int64_t vid = start + done;
    int64_t si = vid >> seg_shift_, off = vid & (seg_rows() - 1);
    int64_t cnt = std::min(n - done, seg_rows() - off);
    const cudaError_t e = cudaMemcpyAsync(dst + done * stride_, segs_[si].base + off * stride_, (size_t)cnt * stride_,
                                          host_ ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return e;
    done += cnt;
  }
  return cudaSuccess;
}
const float* RawStore::contiguous(int64_t n, Scratch& s) {
  if (!host_ && n <= seg_rows()) return segs_.empty() ? nullptr : seg(0);
  float* buf = s.alloc_n<float>((size_t)n * stride_ / 4);
  if (!buf) return nullptr;
  const cudaError_t e = copy_rows_to_device(0, n, buf, s.stream());
  if (e != cudaSuccess) {
    set_last_error(std::string("raw store: copy of the training rows: ") + cudaGetErrorString(e));
    return nullptr;
  }
  return buf;
}

// ------------------------------------------------------------------------------------------
static std::atomic<uint64_t> g_lists_uid{1};
IvfLists::IvfLists(int nlist, int code_bytes) : nlist_(nlist), code_bytes_(code_bytes), uid_(g_lists_uid.fetch_add(1)) {
  h_data_.assign(nlist, nullptr);
  h_ids_.assign(nlist, nullptr);
  h_len_.assign(nlist, 0);
  h_cap_.assign(nlist, 0);
  h_dead_.assign(nlist, 0);
  mem::dev_malloc(&d_data_, sizeof(void*) * nlist);
  mem::dev_malloc(&d_ids_, sizeof(int64_t*) * nlist);
  mem::dev_malloc(&d_len_, sizeof(int) * nlist);
  cudaMemset(d_data_, 0, sizeof(void*) * nlist);
  cudaMemset(d_ids_, 0, sizeof(int64_t*) * nlist);
  cudaMemset(d_len_, 0, sizeof(int) * nlist);
}
IvfLists::~IvfLists() {
  for (void* p : slabs_) mem::dev_free(p);
  mem::dev_free(d_data_);
  mem::dev_free(d_ids_);
  mem::dev_free(d_len_);
}
ListDirectory IvfLists::directory() const {
  ListDirectory dir;
  dir.vecs = reinterpret_cast<const float* const*>(d_data_);
  dir.codes = reinterpret_cast<const uint8_t* const*>(d_data_);
  dir.ids = reinterpret_cast<const int64_t* const*>(d_ids_);
  dir.len = d_len_;
  dir.nlist = nlist_;
  return dir;
}
void* IvfLists::slab_alloc(size_t bytes) {
  bytes = (size_t)round_up((int64_t)bytes, 256);
  if (bytes > slab_left_) return nullptr;
  void* p = slab_cur_;
  slab_cur_ += bytes;
  slab_left_ -= bytes;
  return p;
}
int IvfLists::slab_reserve(size_t need_bytes) {
  if (need_bytes <= slab_left_) return 0;
  size_t slab = std::max<size_t>(need_bytes, (size_t)64 << 20);
  void* p = nullptr;
  GB_CUDA(mem::dev_malloc(&p, slab));
  slabs_.push_back(p);
  slab_cur_ = static_cast<char*>(p);
  slab_left_ = slab;
  bytes_ += (int64_t)slab;
  return 0;
}
int IvfLists::reserve(const std::vector<int>& add, cudaStream_t st) {
  // pass 1: how many bytes do the growing lists need
  std::vector<int> newcap(nlist_, 0);
  size_t need_bytes = 0;
  for (int l = 0; l < nlist_; l++) {
    if (add[l] <= 0) continue;
    int64_t need = (int64_t)h_len_[l] + add[l];
    if (need <= h_cap_[l]) continue;
    // growth policy: at least x1.5 (reference grows by 1.1 + pi/2 - atan(n), realtime_mem_data.cc:110-113)
    int64_t nc = std::max<int64_t>(need, (int64_t)h_cap_[l] * 3 / 2);
    nc = round_up(nc, 32);
    if (nc > INT32_MAX) {
      set_last_error("inverted list too long");
      return -1;
    }
    newcap[l] = (int)nc;
    need_bytes += (size_t)round_up(nc * code_bytes_ + 16, 256) + (size_t)round_up(nc * 8, 256);
  }
  if (need_bytes == 0) return 0;
  if (slab_reserve(need_bytes)) return -1;
  for (int l = 0; l < nlist_; l++) {
    if (!newcap[l]) continue;
    void* nd = slab_alloc((size_t)newcap[l] * code_bytes_ + 16);
    int64_t* ni = static_cast<int64_t*>(slab_alloc((size_t)newcap[l] * 8));
    if (!nd || !ni) {
      set_last_error("slab exhausted");
      return -1;
    }
    if (h_len_[l] > 0) {  // copy-on-grow; the old region stays valid for in-flight searches
      GB_CUDA(cudaMemcpyAsync(nd, h_data_[l], (size_t)h_len_[l] * code_bytes_, cudaMemcpyDeviceToDevice, st));
      GB_CUDA(cudaMemcpyAsync(ni, h_ids_[l], (size_t)h_len_[l] * 8, cudaMemcpyDeviceToDevice, st));
    }
    h_data_[l] = nd;
    h_ids_[l] = ni;
    h_cap_[l] = newcap[l];
  }
  GB_CUDA(cudaMemcpyAsync(d_data_, h_data_.data(), sizeof(void*) * nlist_, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_ids_, h_ids_.data(), sizeof(int64_t*) * nlist_, cudaMemcpyHostToDevice, st));
  return 0;
}
int IvfLists::commit(const std::vector<int>& add, cudaStream_t st) {
  for (int l = 0; l < nlist_; l++) {
    h_len_[l] += add[l];
    total_ += add[l];
    if (h_len_[l] > max_len_) max_len_ = h_len_[l];
  }
  // length is published after the data (realtime_mem_data.cc:292-293): same stream, later op
  GB_CUDA(cudaMemcpyAsync(d_len_, h_len_.data(), sizeof(int) * nlist_, cudaMemcpyHostToDevice, st));
  return 0;
}
int64_t IvfLists::packed_bytes() const {
  int64_t b = 0;
  for (int l = 0; l < nlist_; l++) {
    if (h_len_[l] == 0) continue;
    const int64_t cap = round_up(h_len_[l], 32);
    b += round_up(cap * code_bytes_ + 16, 256) + round_up(cap * 8, 256);
  }
  return b;
}
int IvfLists::compact(cudaStream_t st) {
  const int64_t need = packed_bytes();
  if (need == 0 || slabs_.empty()) return 0;
  void* slab = nullptr;
  if (mem::dev_malloc(&slab, (size_t)need) != cudaSuccess) {
    cudaGetLastError();
    return 0;  // not enough room to re-pack: keep the current layout
  }
  char* cur = static_cast<char*>(slab);
  for (int l = 0; l < nlist_; l++) {
    if (h_len_[l] == 0) {
      h_data_[l] = nullptr, h_ids_[l] = nullptr, h_cap_[l] = 0;
      continue;
    }
    const int64_t cap = round_up(h_len_[l], 32);
    void* nd = cur;
    cur += round_up(cap * code_bytes_ + 16, 256);
    int64_t* ni = reinterpret_cast<int64_t*>(cur);
    cur += round_up(cap * 8, 256);
    GB_CUDA(cudaMemcpyAsync(nd, h_data_[l], (size_t)h_len_[l] * code_bytes_, cudaMemcpyDeviceToDevice, st));
    GB_CUDA(cudaMemcpyAsync(ni, h_ids_[l], (size_t)h_len_[l] * 8, cudaMemcpyDeviceToDevice, st));
    h_data_[l] = nd, h_ids_[l] = ni, h_cap_[l] = (int)cap;
  }
  GB_CUDA(cudaMemcpyAsync(d_data_, h_data_.data(), sizeof(void*) * nlist_, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_ids_, h_ids_.data(), sizeof(int64_t*) * nlist_, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaDeviceSynchronize());  // copies done, and no kernel of an earlier search still reads the old slabs
  for (void* p : slabs_) mem::dev_free(p);
  slabs_.assign(1, slab);
  slab_cur_ = nullptr;
  slab_left_ = 0;
  bytes_ = need;
  return 0;
}
int IvfLists::tombstone(int list, int pos, cudaStream_t st) {
  if (list < 0 || list >= nlist_ || pos < 0 || pos >= h_len_[list]) return -1;
  int64_t v;
  GB_CUDA(cudaMemcpyAsync(&v, h_ids_[list] + pos, 8, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  if (v & kDelIdxMask) return 0;  // already tombstoned, already counted
  v |= kDelIdxMask;
  GB_CUDA(cudaMemcpyAsync(h_ids_[list] + pos, &v, 8, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaStreamSynchronize(st));
  h_dead_[list]++;  // realtime_mem_data.cc:315
  return 0;
}

int IvfLists::purge(const std::vector<int>& lists, const uint32_t* d_del_bits, cudaStream_t st, Purged* out) {
  *out = Purged();
  std::vector<int> sel, chunk0(1, 0);
  std::vector<PurgeChunk> chunks;
  for (int l : lists) {
    if (l < 0 || l >= nlist_ || h_len_[l] == 0) continue;
    for (int first = 0; first < h_len_[l]; first += kPurgeChunk) chunks.push_back(PurgeChunk{(int)sel.size(), first});
    sel.push_back(l);
    chunk0.push_back((int)chunks.size());
  }
  const int nsel = (int)sel.size(), nchunks = (int)chunks.size();
  if (nsel == 0) return 0;
  Scratch s(st);
  GB_ALLOC(d_sel, int, nsel, s);
  GB_ALLOC(d_chunk0, int, nsel + 1, s);
  GB_ALLOC(d_chunks, PurgeChunk, nchunks, s);
  GB_ALLOC(d_chunk_off, int, nchunks, s);
  GB_ALLOC(d_counts, unsigned long long, nsel + 2, s);  // vid range, then the lists' live counts (as ints)
  int* d_live = reinterpret_cast<int*>(d_counts + 2);
  GB_CUDA(cudaMemcpyAsync(d_sel, sel.data(), sizeof(int) * nsel, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_chunk0, chunk0.data(), sizeof(int) * (nsel + 1), cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_chunks, chunks.data(), sizeof(PurgeChunk) * nchunks, cudaMemcpyHostToDevice, st));
  const ListDirectory dir = directory();
  GB_CUDA(launch_purge_count(dir, d_sel, d_chunk0, nsel, d_chunks, nchunks, d_del_bits, d_chunk_off, d_live, d_counts, st));
  // the one download that sizes the destinations and the new-position table
  std::vector<unsigned long long> h_counts((size_t)2 + (nsel + 1) / 2);
  GB_CUDA(cudaMemcpyAsync(h_counts.data(), d_counts, 16 + sizeof(int) * nsel, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  const int* live = reinterpret_cast<const int*>(h_counts.data() + 2);
  const int64_t vid_min = (int64_t)h_counts[0], vid_span = (int64_t)h_counts[1] - vid_min + 1;
  // fresh regions, as reserve() takes them: the old ones stay valid for whatever still reads them
  std::vector<int> newcap(nsel, 0);
  size_t need_bytes = 0;
  for (int i = 0; i < nsel; i++) {
    out->dropped += h_len_[sel[i]] - live[i];
    if (live[i] == 0) continue;
    newcap[i] = (int)round_up(live[i], 32);
    need_bytes += (size_t)round_up((int64_t)newcap[i] * code_bytes_ + 16, 256) + (size_t)round_up((int64_t)newcap[i] * 8, 256);
  }
  if (out->dropped == 0) return 0;  // nothing to drop: the lists stay where they are
  if (slab_reserve(need_bytes)) return -1;
  std::vector<void*> nd(nsel, nullptr);
  std::vector<int64_t*> ni(nsel, nullptr);
  uintptr_t bits = (uintptr_t)code_bytes_ | 16;
  for (int i = 0; i < nsel; i++) {
    if (!newcap[i]) continue;
    nd[i] = slab_alloc((size_t)newcap[i] * code_bytes_ + 16);
    ni[i] = static_cast<int64_t*>(slab_alloc((size_t)newcap[i] * 8));
    if (!nd[i] || !ni[i]) {
      set_last_error("slab exhausted");
      return -1;
    }
    bits |= (uintptr_t)nd[i] | (uintptr_t)h_data_[sel[i]];
  }
  const int align = (int)(bits & (~bits + 1));  // lowest set bit: at most 16
  GB_ALLOC(d_nd, void*, nsel, s);
  GB_ALLOC(d_ni, int64_t*, nsel, s);
  GB_ALLOC(d_newpos, unsigned long long, vid_span, s);
  GB_CUDA(cudaMemcpyAsync(d_nd, nd.data(), sizeof(void*) * nsel, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_ni, ni.data(), sizeof(int64_t*) * nsel, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemsetAsync(d_newpos, 0xFF, (size_t)vid_span * 8, st));
  GB_CUDA(launch_purge_scatter(dir, d_sel, d_chunks, nchunks, d_del_bits, d_chunk_off, code_bytes_, align, d_nd, d_ni, d_newpos,
                               vid_min, st));
  out->vid_min = vid_min;
  out->newpos.resize((size_t)vid_span);
  GB_CUDA(cudaMemcpyAsync(out->newpos.data(), d_newpos, (size_t)vid_span * 8, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));  // the scatter is done (and has not failed) before anything is published
  for (int i = 0; i < nsel; i++) {
    const int l = sel[i];
    h_data_[l] = nd[i], h_ids_[l] = ni[i], h_cap_[l] = newcap[i];
  }
  GB_CUDA(cudaMemcpyAsync(d_data_, h_data_.data(), sizeof(void*) * nlist_, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_ids_, h_ids_.data(), sizeof(int64_t*) * nlist_, cudaMemcpyHostToDevice, st));
  for (int i = 0; i < nsel; i++) {
    h_len_[sel[i]] = live[i];
    h_dead_[sel[i]] = 0;
  }
  total_ -= out->dropped;
  max_len_ = *std::max_element(h_len_.begin(), h_len_.end());
  GB_CUDA(cudaMemcpyAsync(d_len_, h_len_.data(), sizeof(int) * nlist_, cudaMemcpyHostToDevice, st));
  content_gen_++;
  return 0;
}
int IvfLists::download_list(int l, std::vector<uint8_t>* codes, std::vector<int64_t>* ids) const {
  if (l < 0 || l >= nlist_) return -1;
  int len = h_len_[l];
  if (codes) {
    codes->resize((size_t)len * code_bytes_);
    if (len) GB_CUDA(cudaMemcpy(codes->data(), h_data_[l], codes->size(), cudaMemcpyDeviceToHost));
  }
  if (ids) {
    ids->resize(len);
    if (len) GB_CUDA(cudaMemcpy(ids->data(), h_ids_[l], (size_t)len * 8, cudaMemcpyDeviceToHost));
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
namespace {
struct LiveIndexes {
  std::mutex mu;
  std::vector<Index*> all;
};
LiveIndexes& live_indexes() {
  static LiveIndexes* s = new LiveIndexes;  // leaked on purpose: must outlive every static destructor
  return *s;
}
// the memory limit's trim: the idle scan scratch of every index on the device
void release_idle_scratch_on(int device) {
  std::lock_guard<std::mutex> g(live_indexes().mu);
  for (Index* i : live_indexes().all)
    if (i->device() == device) i->release_idle_scratch();
}
void quiesce_all_indexes() {
  std::vector<Index*> v;
  {
    std::lock_guard<std::mutex> g(live_indexes().mu);
    v = live_indexes().all;
  }
  for (Index* i : v) i->quiesce();
}
}  // namespace

Index::Index(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift, int row_bytes)
    : type_(type), gpu_contract_(is_gpu_index_type(type)), d_(d), dpad_((int)round_up(d, 4)), device_(device), mp_(mp) {
  cudaSetDevice(device_);
  mem::configure_pool(device_);
  {  // the CUDA runtime is initialised by now, so this hook runs before its teardown
    std::lock_guard<std::mutex> g(live_indexes().mu);
    static bool hooked = (atexit(quiesce_all_indexes), mem::set_scratch_release(release_idle_scratch_on), true);
    (void)hooked;
    live_indexes().all.push_back(this);
  }
  store_.reset(new RawStore(row_bytes > 0 ? row_bytes : 4 * d, seg_shift, mp.host_store));
  cudaStreamCreateWithFlags(&build_stream_, cudaStreamNonBlocking);
}
void Index::quiesce() {
  {
    std::lock_guard<std::mutex> lk(co_mu_);
    co_stop_ = true;
  }
  co_cv_.notify_all();
  if (co_thread_.joinable()) co_thread_.join();
}

Index::~Index() {
  drain_searches();
  {
    std::lock_guard<std::mutex> g(live_indexes().mu);
    auto& a = live_indexes().all;
    a.erase(std::remove(a.begin(), a.end(), this), a.end());
  }
  quiesce();
  for (auto& b : big_) {
    mem::dev_free(b.p);
    cudaEventDestroy(b.done);
  }
  if (build_stream_) cudaStreamDestroy(build_stream_);
}
void* Index::big_acquire(size_t bytes, cudaStream_t st) {
  std::lock_guard<std::mutex> g(big_mu_);
  int best = -1;
  for (size_t i = 0; i < big_.size(); i++)
    if (!big_[i].busy && big_[i].cap >= bytes && (best < 0 || big_[i].cap < big_[best].cap)) best = (int)i;
  if (best < 0) {
    free_idle_big_locked();  // drop idle buffers that are too small before growing
    BigBuf b;
    b.cap = bytes + bytes / 4;
    b.busy = false;
    if (mem::dev_malloc(&b.p, b.cap) != cudaSuccess) {
      b.cap = bytes;
      if (mem::dev_malloc(&b.p, b.cap) != cudaSuccess) {
        set_last_error("cudaMalloc(" + std::to_string(bytes) + ") failed for scan scratch");
        return nullptr;
      }
    }
    cudaEventCreateWithFlags(&b.done, cudaEventDisableTiming);
    cudaEventRecord(b.done, st);
    big_.push_back(b);
    best = (int)big_.size() - 1;
  }
  big_[best].busy = true;
  cudaStreamWaitEvent(st, big_[best].done, 0);  // previous user's kernels (possibly on another stream)
  return big_[best].p;
}
void Index::free_idle_big_locked() {
  for (size_t i = 0; i < big_.size();) {
    if (!big_[i].busy) {
      cudaEventSynchronize(big_[i].done);
      mem::dev_free(big_[i].p);
      cudaEventDestroy(big_[i].done);
      big_.erase(big_.begin() + i);
    } else {
      i++;
    }
  }
}
void Index::release_idle_scratch() {
  std::lock_guard<std::mutex> g(big_mu_);
  free_idle_big_locked();
}
void Index::memory_charges(int64_t n_total, std::vector<mem::Charge>* out) {
  int64_t rows = 0;
  const int64_t grow = store_->growth_bytes(n_total, &rows);
  if (grow == 0) return;
  out->push_back({store_->on_host() ? mem::kHost : device_, grow});
  charge_index_rows(rows, out);
}
void IvfIndex::charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) {
  out->push_back({device_, rows * (code_bytes() + 8)});
}
void IVFFlatIndex::charge_index_rows(int64_t rows, std::vector<mem::Charge>* out) {
  IvfIndex::charge_index_rows(rows, out);
  std::shared_lock<std::shared_mutex> lk(mirror_rw_);
  if (mirror_.base)  // a tile of 128 rows and their norms
    out->push_back({device_, rows * (int64_t)((size_t)tc_mirror_tile_floats((int)round_up(dpad_, 16)) * 4 + 512) / 128});
}
void Index::big_release(void* p, cudaStream_t st) {
  std::lock_guard<std::mutex> g(big_mu_);
  for (auto& b : big_)
    if (b.p == p) {
      cudaEventRecord(b.done, st);
      b.busy = false;
    }
}
void Index::note_search_enqueued(cudaStream_t st) {
  cudaEvent_t e;
  if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return;
  cudaEventRecord(e, st);
  std::lock_guard<std::mutex> g(inflight_mu_);
  if (inflight_.size() >= 64) {  // forget the ones that have completed
    size_t w = 0;
    for (size_t i = 0; i < inflight_.size(); i++) {
      if (cudaEventQuery(inflight_[i]) == cudaSuccess)
        cudaEventDestroy(inflight_[i]);
      else
        inflight_[w++] = inflight_[i];
    }
    inflight_.resize(w);
    cudaGetLastError();  // cudaErrorNotReady from the queries is not an error
  }
  inflight_.push_back(e);
}
void Index::drain_searches() {
  std::lock_guard<std::mutex> g(inflight_mu_);
  for (cudaEvent_t e : inflight_) {
    cudaEventSynchronize(e);
    cudaEventDestroy(e);
  }
  inflight_.clear();
}
void Index::scan_timer_begin(cudaStream_t st) {
  if (!time_scan_) return;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, st);
  std::lock_guard<std::mutex> g(ev_mu_);
  scan_events_.emplace_back(e0, e1);
}
void Index::scan_timer_end(cudaStream_t st) {
  if (!time_scan_) return;
  std::lock_guard<std::mutex> g(ev_mu_);
  if (!scan_events_.empty()) cudaEventRecord(scan_events_.back().second, st);
}
void Index::stage_begin(const char* name, cudaStream_t st) {
  if (!time_scan_) return;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, st);
  std::lock_guard<std::mutex> g(ev_mu_);
  stage_events_.push_back({name, e0, e1});
}
void Index::stage_end(cudaStream_t st) {
  if (!time_scan_) return;
  std::lock_guard<std::mutex> g(ev_mu_);
  if (!stage_events_.empty()) cudaEventRecord(stage_events_.back().e1, st);
}
std::vector<std::pair<std::string, float>> Index::stage_times() {
  std::lock_guard<std::mutex> g(ev_mu_);
  std::vector<std::pair<std::string, float>> out;
  for (auto& ev : stage_events_) {
    float ms = 0.f;
    if (cudaEventSynchronize(ev.e1) != cudaSuccess || cudaEventElapsedTime(&ms, ev.e0, ev.e1) != cudaSuccess) ms = 0.f;
    cudaEventDestroy(ev.e0);
    cudaEventDestroy(ev.e1);
    bool found = false;
    for (auto& o : out)
      if (o.first == ev.name) o.second += ms, found = true;
    if (!found) out.emplace_back(ev.name, ms);
  }
  stage_events_.clear();
  return out;
}
float Index::last_scan_ms() {
  std::lock_guard<std::mutex> g(ev_mu_);
  float total = 0.f;
  for (auto& ev : scan_events_) {
    float ms = 0.f;
    if (cudaEventSynchronize(ev.second) == cudaSuccess && cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess)
      total += ms;
    cudaEventDestroy(ev.first);
    cudaEventDestroy(ev.second);
  }
  scan_events_.clear();
  return total;
}
int Index::add_vectors(const void* x, int64_t n) {
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  return store_->append_host(x, n, build_stream_);
}
int Index::add_vectors_device(const float* x, int64_t ld, int64_t n) {
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  return store_->append_device(x, ld * 4, n, build_stream_);
}

const void* Index::store_rows_dev(int64_t vid0, int64_t n, Scratch& s) {
  const int64_t si = vid0 >> store_->seg_shift(), off = vid0 & (store_->seg_rows() - 1);
  if (!store_->on_host()) return store_->seg_bytes((int)si) + off * store_->stride();
  void* buf = s.alloc((size_t)n * store_->stride());
  if (!buf) return nullptr;
  const cudaError_t e = store_->copy_rows_to_device(vid0, n, buf, s.stream());
  if (e != cudaSuccess) {
    set_last_error(std::string("raw store: copy of rows to the device: ") + cudaGetErrorString(e));
    return nullptr;
  }
  return buf;
}

Index::CopyLane::~CopyLane() {
  for (int b = 0; b < 2; b++) {
    if (copied[b]) cudaEventDestroy(copied[b]);
    if (reusable[b]) cudaEventDestroy(reusable[b]);
  }
  if (cs) cudaStreamDestroy(cs);
}
Index::CopyLane* Index::lane_acquire() {
  std::lock_guard<std::mutex> g(lane_mu_);
  if (!free_lanes_.empty()) {
    CopyLane* l = free_lanes_.back();
    free_lanes_.pop_back();
    return l;
  }
  std::unique_ptr<CopyLane> l(new CopyLane);
  cudaError_t e = cudaStreamCreateWithFlags(&l->cs, cudaStreamNonBlocking);
  for (int b = 0; b < 2 && e == cudaSuccess; b++) {
    e = cudaEventCreateWithFlags(&l->copied[b], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&l->reusable[b], cudaEventDisableTiming);
  }
  if (e != cudaSuccess) {
    set_last_error(std::string("copy stream for the host store: ") + cudaGetErrorString(e));
    return nullptr;
  }
  lanes_.push_back(std::move(l));
  return lanes_.back().get();
}
void Index::lane_release(CopyLane* l) {
  std::lock_guard<std::mutex> g(lane_mu_);
  free_lanes_.push_back(l);
}

int Index::upload_bitmaps(const SearchContext& ctx, FilterArgs* f, Scratch& s) {
  f->del_bits = nullptr;
  f->filter_bits = nullptr;
  f->min_score = ctx.min_score;
  f->max_score = ctx.max_score;
  // the kernels index bitmaps by vid; pad to cover every stored vector
  int64_t bits = std::max<int64_t>(ctx.bitmap_bits, store_->size());
  size_t words = (size_t)((bits + 31) / 32) + 1;
  size_t have = (size_t)((ctx.bitmap_bits + 7) / 8);
  for (int which = 0; which < 2; which++) {
    const uint32_t* src_dev = which == 0 ? ctx.del_bits_dev : ctx.filter_bits_dev;
    const uint8_t* src = which == 0 ? ctx.del_bitmap : ctx.filter_bitmap;
    if (!src && !src_dev) continue;
    if (src_dev && ctx.bits_dev_words >= (int64_t)words) {  // already padded: the scan reads it in place
      if (which == 0)
        f->del_bits = src_dev;
      else
        f->filter_bits = src_dev;
      continue;
    }
    uint32_t* dev = s.alloc_n<uint32_t>(words);
    if (!dev) return -1;
    // ids beyond the caller's bitmap: not deleted / not allowed
    GB_CUDA(cudaMemsetAsync(dev, 0, words * 4, s.stream()));
    if (src_dev)
      GB_CUDA(cudaMemcpyAsync(dev, src_dev, have, cudaMemcpyDeviceToDevice, s.stream()));
    else
      GB_CUDA(cudaMemcpyAsync(dev, src, have, cudaMemcpyHostToDevice, s.stream()));
    if (which == 0)
      f->del_bits = dev;
    else
      f->filter_bits = dev;
  }
  return 0;
}

const void* Index::upload_queries(int nq, const void* x, Scratch& s) {
  const size_t rb = store_->row_bytes(), ld = store_->stride();
  void* dq = s.alloc((size_t)nq * ld);
  if (!dq) return nullptr;
  cudaError_t e = rb == ld ? cudaSuccess : cudaMemsetAsync(dq, 0, (size_t)nq * ld, s.stream());
  if (e == cudaSuccess) e = cudaMemcpy2DAsync(dq, ld, x, rb, rb, nq, cudaMemcpyHostToDevice, s.stream());
  if (e != cudaSuccess) {
    set_last_error(std::string("query upload: ") + cudaGetErrorString(e));
    return nullptr;
  }
  return dq;
}

int Index::download_results(const unsigned long long* keys, int nq, int k, int metric, float* out_dis, int64_t* out_ids,
                            Scratch& s) {
  cudaStream_t st = s.stream();
  GB_ALLOC(dd, float, (size_t)nq * k, s);
  GB_ALLOC(di, int64_t, (size_t)nq * k, s);
  GB_CUDA(launch_decode_keys(keys, k, nq, k, metric, dd, di, 0, st));
  GB_CUDA(cudaMemcpyAsync(out_dis, dd, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaMemcpyAsync(out_ids, di, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int Index::search_keys(const SearchContext& ctx, int nq, const void* xq, int k, unsigned long long** out_keys, Scratch& s) {
  if (k <= 0 || k > 4096) {
    set_last_error("topK must be in [1, 4096]");
    return -1;
  }
  cudaStream_t st = s.stream();
  FilterArgs f;
  if (upload_bitmaps(ctx, &f, s)) return -1;
  const int metric = search_metric(ctx);
  GB_ALLOC(keys, unsigned long long, (size_t)nq * k, s);
  *out_keys = keys;
  int rc;
  if (ctx.params.brute_force || !trained_) {
    // brute-force fallback of the IVF models (gamma_index_ivfflat.cc:541-550, ivfpq.cc:561-570)
    rc = flat_search_dev(ctx, f, metric, nq, xq, k, store_->size(), keys, s);
  } else {
    rc = search_keys_dev(ctx, f, metric, nq, xq, k, keys, s);
    // enable_realtime (vector_manager.cc:854-889, 971-1053): vectors stored but not yet indexed are
    // searched brute-force (the reference's MemoryBuffer FLAT index) and merged by score
    const int64_t tail0 = indexed_count_, tail1 = store_->size();
    if (rc == 0 && ctx.search_unindexed_tail && tail1 > tail0) {
      GB_ALLOC(both, unsigned long long, (size_t)nq * 2 * k, s);
      GB_CUDA(cudaMemcpy2DAsync(both, (size_t)2 * k * 8, keys, (size_t)k * 8, (size_t)k * 8, nq,
                                cudaMemcpyDeviceToDevice, st));
      GB_ALLOC(tailk, unsigned long long, (size_t)nq * k, s);
      rc = flat_search_dev(ctx, f, metric, nq, xq, k, tail1, tailk, s, tail0);
      if (rc == 0) {
        GB_CUDA(cudaMemcpy2DAsync(both + k, (size_t)2 * k * 8, tailk, (size_t)k * 8, (size_t)k * 8, nq,
                                  cudaMemcpyDeviceToDevice, st));
        GB_CUDA(launch_select_keys(both, (int64_t)2 * k, nq, 2 * k, k, keys, k, st));
      }
    }
  }
  note_search_enqueued(st);
  return rc;
}

int Index::search_device(const SearchContext& ctx, int nq, const float* x_dev, int64_t ldx, int k, float* out_dis_dev,
                         int64_t* out_ids_dev, cudaStream_t st, unsigned long long* out_keys_dev) {
  if (nq <= 0) return 0;
  if (check_gpu_request(ctx, nq, k)) return -1;
  cudaSetDevice(device_);
  std::shared_lock<std::shared_mutex> lk(mu_);
  Scratch s(st);
  const float* xq = x_dev;
  int64_t ldq = ldx;
  if ((ldx & 3) || (reinterpret_cast<uintptr_t>(x_dev) & 15)) {  // re-pack into 16-byte aligned rows
    float* buf = s.alloc_n<float>((size_t)nq * dpad_);
    if (!buf) return -1;
    GB_CUDA(cudaMemsetAsync(buf, 0, (size_t)nq * dpad_ * 4, st));
    GB_CUDA(cudaMemcpy2DAsync(buf, (size_t)dpad_ * 4, x_dev, (size_t)ldx * 4, (size_t)d_ * 4, nq,
                              cudaMemcpyDeviceToDevice, st));
    xq = buf;
    ldq = dpad_;
  } else if (ldx < dpad_) {
    set_last_error("query row stride smaller than padded dimension");
    return -1;
  }
  // the device kernels take a dense nq x dpad block
  if (ldq != dpad_) {
    float* buf = s.alloc_n<float>((size_t)nq * dpad_);
    if (!buf) return -1;
    GB_CUDA(cudaMemcpy2DAsync(buf, (size_t)dpad_ * 4, xq, (size_t)ldq * 4, (size_t)dpad_ * 4, nq,
                              cudaMemcpyDeviceToDevice, st));
    xq = buf;
  }
  unsigned long long* keys;
  if (int rc = search_keys(ctx, nq, xq, k, &keys, s)) return rc;
  if (out_keys_dev) GB_CUDA(cudaMemcpyAsync(out_keys_dev, keys, (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, st));
  if (out_dis_dev && out_ids_dev)
    GB_CUDA(launch_decode_keys(keys, k, nq, k, search_metric(ctx), out_dis_dev, out_ids_dev, 0, st));
  return 0;
}

static bool coalesce_enabled() {
  static int v = [] {
    const char* e = getenv("GB_COALESCE");
    return e ? atoi(e) : 1;
  }();
  return v != 0;
}
static constexpr int kCoalesceMaxNq = 16;     // requests at most this large are merged
static constexpr int kCoalesceMaxBatch = 512;  // queries per merged device batch (reference kMaxBatch)

bool Index::coalescable(const SearchContext& ctx, int nq) const {
  return coalesce_enabled() && nq <= kCoalesceMaxNq && !ctx.del_bitmap && !ctx.filter_bitmap && !ctx.del_bits_dev &&
         !ctx.filter_bits_dev;
}

static bool same_signature(const SearchContext& a, int ka, const SearchContext& b, int kb) {
  return ka == kb && a.min_score == b.min_score && a.max_score == b.max_score && a.params.nprobe == b.params.nprobe &&
         a.params.metric == b.params.metric && a.params.recall_num == b.params.recall_num &&
         a.params.brute_force == b.params.brute_force && a.search_unindexed_tail == b.search_unindexed_tail &&
         a.params.qb == b.params.qb && a.params.given == b.params.given;
}

void Index::coalesce_loop() {
  cudaSetDevice(device_);
  std::vector<CoReq*> batch;
  std::vector<unsigned char> xs;
  std::vector<float> dd;
  std::vector<int64_t> ii;
  for (;;) {
    batch.clear();
    {
      std::unique_lock<std::mutex> lk(co_mu_);
      co_cv_.wait(lk, [this] { return co_stop_ || !co_queue_.empty(); });
      if (co_stop_ && co_queue_.empty()) return;
      CoReq* first = co_queue_.front();
      int total = 0;
      for (size_t i = 0; i < co_queue_.size();) {  // whatever piled up while the previous batch ran
        CoReq* r = co_queue_[i];
        if (total + r->nq <= kCoalesceMaxBatch && same_signature(*first->ctx, first->k, *r->ctx, r->k)) {
          batch.push_back(r);
          total += r->nq;
          co_queue_.erase(co_queue_.begin() + i);
        } else {
          i++;
        }
      }
    }
    int total = 0;
    for (CoReq* r : batch) total += r->nq;
    const int k = batch[0]->k;
    int rc;
    if (batch.size() == 1) {
      rc = search_direct(*batch[0]->ctx, batch[0]->nq, batch[0]->x, k, batch[0]->out_dis, batch[0]->out_ids);
    } else {
      const size_t rb = store_->row_bytes();
      xs.resize((size_t)total * rb);
      dd.resize((size_t)total * k);
      ii.resize((size_t)total * k);
      size_t o = 0;
      for (CoReq* r : batch) {
        memcpy(xs.data() + o * rb, r->x, (size_t)r->nq * rb);
        o += r->nq;
      }
      rc = search_direct(*batch[0]->ctx, total, xs.data(), k, dd.data(), ii.data());
      o = 0;
      for (CoReq* r : batch) {
        if (rc == 0) {
          memcpy(r->out_dis, dd.data() + o * k, (size_t)r->nq * k * 4);
          memcpy(r->out_ids, ii.data() + o * k, (size_t)r->nq * k * 8);
        }
        o += r->nq;
      }
    }
    std::string err = rc ? last_error() : "";
    {
      std::lock_guard<std::mutex> lk(co_mu_);
      for (CoReq* r : batch) {
        r->rc = rc;
        r->err = err;
        r->done = true;
      }
    }
    co_done_cv_.notify_all();
  }
}

int Index::check_gpu_request(const SearchContext& ctx, int nq, int k) const {
  if (!gpu_contract_) return 0;
  if (nq > kGpuMaxReq) {  // CommonSearch (gamma_gpu_search_base.h:48-52)
    set_last_error("req num [" + std::to_string(nq) + "] should not larger than [" + std::to_string(kGpuMaxReq) + "]");
    return -1;
  }
  // GetRecallNum: max(k, recall_num) for GPU_IVFPQ; GPU_IVFFLAT's is always k (gamma_gpu_search_base.h:74-81)
  const int recall = type_ == "GPU_IVFPQ" ? std::max(k, ctx.params.recall_num) : k;
  if (recall > kGpuMaxK) {
    set_last_error("topK num [" + std::to_string(recall) + "] should not larger than [" + std::to_string(kGpuMaxK) + "]");
    return -1;
  }
  return 0;
}

int Index::search(const SearchContext& ctx, int nq, const void* x, int k, float* out_dis, int64_t* out_ids) {
  if (nq <= 0) return 0;
  if (check_gpu_request(ctx, nq, k)) return -1;  // per call, before coalescing merges calls into one device batch
  if (!coalescable(ctx, nq)) return search_direct(ctx, nq, x, k, out_dis, out_ids);
  CoReq req;
  req.ctx = &ctx, req.nq = nq, req.k = k, req.x = x, req.out_dis = out_dis, req.out_ids = out_ids;
  {
    std::unique_lock<std::mutex> lk(co_mu_);
    if (!co_started_) {
      co_started_ = true;
      co_thread_ = std::thread(&Index::coalesce_loop, this);
    }
    co_queue_.push_back(&req);
    co_cv_.notify_one();
    co_done_cv_.wait(lk, [&req] { return req.done; });
  }
  if (req.rc) set_last_error(req.err);
  return req.rc;
}

int Index::search_direct(const SearchContext& ctx, int nq, const void* x, int k, float* out_dis, int64_t* out_ids) {
  if (nq <= 0) return 0;
  cudaSetDevice(device_);
  Scratch s(thread_stream(device_));
  const void* xq = upload_queries(nq, x, s);
  if (!xq) return -1;
  unsigned long long* keys;
  {
    std::shared_lock<std::shared_mutex> lk(mu_);
    if (int rc = search_keys(ctx, nq, xq, k, &keys, s)) return rc;
  }
  return download_results(keys, nq, k, search_metric(ctx), out_dis, out_ids, s);
}

cudaError_t Index::flat_tile(const void* xq, int nq, const void* rows, int m, int metric, float* scores, int64_t ldo,
                             cudaStream_t st) {
  last_scan_kernel_ = "dist_tile_kernel+select_rows_kernel";
  return launch_dist_matrix(static_cast<const float*>(xq), dpad_, nq, static_cast<const float*>(rows), dpad_, m, dpad_, metric,
                            scores, ldo, st);
}

// GammaFLATIndex::Search (gamma_index_flat.cc:130-370): every stored row, filters before top-k.
int Index::flat_search_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xqv, int k,
                           int64_t nrows, unsigned long long* out_keys, Scratch& s, int64_t row_begin) {
  (void)ctx;
  cudaStream_t st = s.stream();
  if (nrows <= row_begin) return launch_fill_u64(out_keys, (int64_t)nq * k, kKeySentinel, st) == cudaSuccess ? 0 : -1;
  const unsigned char* xq = static_cast<const unsigned char*>(xqv);
  const int64_t ld = store_->stride();
  const int64_t CC = std::min<int64_t>(131072, store_->seg_rows());  // DB rows per distance block
  struct Chunk {
    const unsigned char* base;
    int64_t id0;
    int cnt;
  };
  std::vector<Chunk> chunks;
  for (int64_t r = row_begin; r < nrows;) {
    int64_t si = r >> store_->seg_shift(), off = r & (store_->seg_rows() - 1);
    int64_t cnt = std::min<int64_t>(std::min(nrows - r, store_->seg_rows() - off), CC);
    chunks.push_back({store_->seg_bytes((int)si) + off * ld, r, (int)cnt});
    r += cnt;
  }
  const int nch = (int)chunks.size();
  int64_t ldo = round_up(std::min<int64_t>(CC, nrows - row_begin), 4);
  int QB = (int)std::max<int64_t>(1, std::min<int64_t>(nq, ((int64_t)1 << 28) / ldo));  // <= 1 GiB of scores
  GB_ALLOC(scores, float, (size_t)QB * ldo, s);
  // the chunks' partial keys of a block of PB queries stay within kScanPartialBudget (one query at least); each block is
  // merged into out_keys before the next one reuses them
  const int PB = nch > 1 ? (int)std::max<int64_t>(1, std::min<int64_t>(nq, kScanPartialBudget / ((int64_t)nch * k * 8)))
                         : nq;
  unsigned long long* partial = out_keys;
  if (nch > 1) {
    partial = s.alloc_n<unsigned long long>((size_t)PB * nch * k);
    if (!partial) return -1;
  }
  if (store_->on_host()) {
    // Host placement: each chunk is copied once, on a copy stream, into one of two HBM staging buffers, so the copy of
    // chunk c + 1 overlaps the distance and select kernels of chunk c.  The chunks, kernels and partial merge are those
    // of the HBM store, so the keys are the same; the scan runs at PCIe speed, not at HBM speed.
    struct LaneScope {  // the lane goes back to the pool on every exit path, once this search's copies are enqueued
      Index* ix;
      CopyLane* l;
      ~LaneScope() {
        if (l) ix->lane_release(l);
      }
    } lane{this, lane_acquire()};
    if (!lane.l) return -1;
    CopyLane& cl = *lane.l;
    void* stage[2];
    for (int b = 0; b < 2; b++) {
      stage[b] = s.alloc((size_t)CC * ld);
      if (!stage[b]) return -1;
      GB_CUDA(cudaEventRecord(cl.reusable[b], st));  // the buffers are allocated in stream order on st
    }
    scan_timer_begin(st);
    int copies = 0;
    for (int p0 = 0; p0 < nq; p0 += PB) {  // one block unless the partials need more: the rows stream once per block
      const int pb = std::min(PB, nq - p0);
      for (int c = 0; c < nch; c++, copies++) {
        const int b = copies & 1;
        GB_CUDA(cudaStreamWaitEvent(cl.cs, cl.reusable[b], 0));
        GB_CUDA(cudaMemcpyAsync(stage[b], chunks[c].base, (size_t)chunks[c].cnt * ld, cudaMemcpyHostToDevice, cl.cs));
        GB_CUDA(cudaEventRecord(cl.copied[b], cl.cs));
        GB_CUDA(cudaStreamWaitEvent(st, cl.copied[b], 0));
        for (int q0 = 0; q0 < pb; q0 += QB) {
          int qb = std::min(QB, pb - q0);
          GB_CUDA(flat_tile(xq + (p0 + q0) * ld, qb, stage[b], chunks[c].cnt, metric, scores, ldo, st));
          GB_CUDA(launch_select_scores(scores, ldo, qb, chunks[c].cnt, chunks[c].id0, k, metric, f,
                                       (nch > 1 ? partial + (int64_t)q0 * nch * k : out_keys + (int64_t)(p0 + q0) * k) +
                                           (int64_t)c * k,
                                       (int64_t)nch * k, st));
        }
        GB_CUDA(cudaEventRecord(cl.reusable[b], st));
      }
      if (nch > 1) GB_CUDA(launch_select_keys(partial, (int64_t)nch * k, pb, nch * k, k, out_keys + (int64_t)p0 * k, k, st));
    }
    scan_timer_end(st);
    return 0;
  }
  scan_timer_begin(st);
  for (int p0 = 0; p0 < nq; p0 += PB) {
    const int pb = std::min(PB, nq - p0);
    for (int q0 = 0; q0 < pb; q0 += QB) {
      int qb = std::min(QB, pb - q0);
      for (int c = 0; c < nch; c++) {
        GB_CUDA(flat_tile(xq + (p0 + q0) * ld, qb, chunks[c].base, chunks[c].cnt, metric, scores, ldo, st));
        GB_CUDA(launch_select_scores(scores, ldo, qb, chunks[c].cnt, chunks[c].id0, k, metric, f,
                                     (nch > 1 ? partial + (int64_t)q0 * nch * k : out_keys + (int64_t)(p0 + q0) * k) +
                                         (int64_t)c * k,
                                     (int64_t)nch * k, st));
      }
    }
    if (nch > 1) GB_CUDA(launch_select_keys(partial, (int64_t)nch * k, pb, nch * k, k, out_keys + (int64_t)p0 * k, k, st));
  }
  scan_timer_end(st);
  return 0;
}

int FlatIndex::search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq, int k,
                               unsigned long long* out_keys, Scratch& s) {
  return flat_search_dev(ctx, f, metric, nq, xq, k, store_->size(), out_keys, s);
}

// ------------------------------------------------------------------------------------------
// k-means (faiss::Clustering restated, SURVEY Appendix A).  Assign runs on device (K2 kernel with
// fused argmin), the centroid update is a deterministic segmented mean on device, the control
// logic (seeded permutations, empty-cluster split) runs on host.
static void rand_perm_mt(std::vector<int32_t>& perm, int64_t n, int64_t seed) {
  perm.resize(n);
  for (int64_t i = 0; i < n; i++) perm[i] = (int32_t)i;
  std::mt19937 mt((unsigned)seed);
  for (int64_t i = 0; i + 1 < n; i++) {
    int64_t i2 = i + (int64_t)(mt() % (uint32_t)(n - i));
    std::swap(perm[i], perm[i2]);
  }
}

// faiss's max_train_points rule: the first n_out rows of a seeded permutation (seed 1234) of the n rows of x (stride
// dpad), or x itself when n_out == n
static int subsample_rows(const float* x, int64_t n, int64_t n_out, int dpad, const float** out, Scratch& s) {
  *out = x;
  if (n_out >= n) return 0;
  cudaStream_t st = s.stream();
  std::vector<int32_t> perm;
  rand_perm_mt(perm, n, 1234);
  GB_ALLOC(d_idx, int32_t, n_out, s);
  GB_CUDA(cudaMemcpyAsync(d_idx, perm.data(), (size_t)n_out * 4, cudaMemcpyHostToDevice, st));
  GB_ALLOC(sub, float, (size_t)n_out * dpad, s);
  GB_CUDA(launch_gather_rows(x, dpad, d_idx, n_out, dpad, sub, dpad, st));
  GB_CUDA(cudaStreamSynchronize(st));
  *out = sub;
  return 0;
}

// the k x d centroids appended to a trace's snapshot (stream-ordered, synchronous)
static cudaError_t trace_centroids(const float* centroids, int64_t ldc, int k, int d, std::vector<float>& out,
                                   cudaStream_t st) {
  const size_t at = out.size();
  out.resize(at + (size_t)k * d);
  cudaError_t e = cudaMemcpy2DAsync(out.data() + at, (size_t)d * 4, centroids, (size_t)ldc * 4, (size_t)d * 4, k,
                                    cudaMemcpyDeviceToHost, st);
  return e != cudaSuccess ? e : cudaStreamSynchronize(st);
}

// The rows whose every tensor-core score is NaN (ord 0xFFFFFFFF as argmin_ord ranks it): a row holding a NaN, or an
// infinity, whose TF32 split hi + (inf - hi) carries a NaN into every dot.  Scored again on the exact kernel, an
// infinite row keeps its +-inf scores, so under IP it goes to the first centroid whose dot is +inf, as faiss's and the
// CUDA-core assignment do.  h_best: the rows' keys on the host, updated in place.
static int rescore_unscored(const float* x, int64_t ldx, int64_t n, int d, int dpad, const float* centroids, int64_t ldc,
                            int k, int metric, std::vector<unsigned long long>& h_best, cudaStream_t st) {
  std::vector<int32_t> rows;
  for (int64_t i = 0; i < n; i++)
    if ((uint32_t)(h_best[i] >> 32) == 0xFFFFFFFFu) rows.push_back((int32_t)i);
  if (rows.empty()) return 0;
  const int64_t m = (int64_t)rows.size();
  Scratch s(st);
  GB_ALLOC(d_rows, int32_t, m, s);
  GB_ALLOC(xr, float, (size_t)m * dpad, s);
  GB_ALLOC(kr, unsigned long long, m, s);
  GB_CUDA(cudaMemcpyAsync(d_rows, rows.data(), (size_t)m * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(launch_gather_rows(x, ldx, d_rows, m, d, xr, dpad, st));
  GB_CUDA(launch_fill_u64(kr, m, kKeySentinel, st));
  GB_CUDA(launch_dist_argmin(xr, dpad, (int)m, centroids, ldc, k, dpad, metric, kr, 0, st));
  std::vector<unsigned long long> hk(m);
  GB_CUDA(cudaMemcpyAsync(hk.data(), kr, (size_t)m * 8, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  for (int64_t j = 0; j < m; j++) h_best[rows[j]] = hk[j];
  return 0;
}

int kmeans_device(const float* x_in, int64_t ldx_in, int64_t n_in, int d, int k, const KMeansParams& kp,
                  float* centroids, int64_t ldc, cudaStream_t st, std::vector<float>* obj, KMeansTrace* trace) {
  if (n_in < k) {
    set_last_error("kmeans: fewer training points than centroids");
    return -1;
  }
  if (n_in > INT32_MAX) {
    set_last_error("kmeans: too many points");
    return -1;
  }
  Scratch s(st);
  const int dpad = (int)round_up(d, 4);
  const float* x = x_in;
  int64_t ldx = ldx_in, n = n_in;
  std::vector<int32_t> perm;
  if (kp.max_points_per_centroid > 0 && n_in > (int64_t)k * kp.max_points_per_centroid) {
    n = (int64_t)k * kp.max_points_per_centroid;
    rand_perm_mt(perm, n_in, kp.seed);
    if (trace) trace->sample.assign(perm.begin(), perm.begin() + n);
    GB_ALLOC(d_idx, int32_t, n, s);
    GB_CUDA(cudaMemcpyAsync(d_idx, perm.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    GB_ALLOC(xs, float, (size_t)n * dpad, s);
    GB_CUDA(launch_gather_rows(x_in, ldx_in, d_idx, n, d, xs, dpad, st));
    GB_CUDA(cudaStreamSynchronize(st));
    x = xs;
    ldx = dpad;
  }
  // initial centroids = first k entries of a seeded permutation (or the caller's, for a hot start)
  GB_ALLOC(d_perm, int32_t, n, s);
  GB_ALLOC(d_off, int32_t, k + 1, s);
  if (!kp.hot_start) {
    rand_perm_mt(perm, n, kp.seed + 1);
    GB_CUDA(cudaMemcpyAsync(d_perm, perm.data(), (size_t)k * 4, cudaMemcpyHostToDevice, st));
    GB_CUDA(launch_gather_rows(x, ldx, d_perm, k, d, centroids, ldc, st));
    if (kp.spherical) GB_CUDA(launch_normalize_rows(centroids, ldc, k, d, st));
  }
  GB_CUDA(cudaStreamSynchronize(st));
  if (trace) GB_CUDA(trace_centroids(centroids, ldc, k, d, trace->init, st));

  GB_ALLOC(best, unsigned long long, n, s);
  std::vector<unsigned long long> h_best(n);
  std::vector<int32_t> h_off(k + 1), h_perm(n), cursor(k);
  std::vector<float> hassign(k), h_cent;
  const int metric = kp.spherical && !kp.l2_assign ? kMetricIP : kMetricL2;  // gamma's quantizer is IndexFlat(d, metric)
  const bool use_tc = k >= 64;  // tensor-core (wgmma 3xTF32) distance tiles
  for (int it = 0; it < kp.niter; it++) {
    GB_CUDA(launch_fill_u64(best, n, kKeySentinel, st));
    if (use_tc) {
      GB_CUDA(launch_dist_argmin_tc(x, ldx, (int)n, centroids, ldc, k, dpad, metric, best, st));
    } else {
      GB_CUDA(launch_dist_argmin(x, ldx, (int)n, centroids, ldc, k, dpad, metric, best, 0, st));
    }
    GB_CUDA(cudaMemcpyAsync(h_best.data(), best, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    if (use_tc && rescore_unscored(x, ldx, n, d, dpad, centroids, ldc, k, metric, h_best, st)) return -1;
    // stable counting sort of the points by label (point order inside a cluster = faiss's sum order)
    std::fill(h_off.begin(), h_off.end(), 0);
    double o = 0;
    for (int64_t i = 0; i < n; i++) {
      // faiss's assignment takes a centroid only when its score beats the start value FLT_MAX (-FLT_MAX under IP):
      // a row without one (NaN, infinite) goes to cluster 0
      const float sc = ord2score((uint32_t)(h_best[i] >> 32), metric);
      if ((uint32_t)h_best[i] >= (uint32_t)k || !(metric == kMetricL2 ? sc < FLT_MAX : sc > -FLT_MAX))
        h_best[i] &= 0xFFFFFFFF00000000ull;
      h_off[(uint32_t)h_best[i] + 1]++;
      if (obj) o += sc;
      if (trace) {
        trace->labels.push_back((int32_t)(uint32_t)h_best[i]);
        trace->scores.push_back(sc);
      }
    }
    if (obj) obj->push_back((float)o);
    for (int c = 0; c < k; c++) {
      hassign[c] = (float)h_off[c + 1];
      h_off[c + 1] += h_off[c];
      cursor[c] = h_off[c];
    }
    for (int64_t i = 0; i < n; i++) h_perm[cursor[(uint32_t)h_best[i]]++] = (int32_t)i;
    GB_CUDA(cudaMemcpyAsync(d_perm, h_perm.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaMemcpyAsync(d_off, h_off.data(), (size_t)(k + 1) * 4, cudaMemcpyHostToDevice, st));
    GB_CUDA(launch_segment_mean(x, ldx, d, d_perm, d_off, k, centroids, ldc, st));
    if (trace) GB_CUDA(trace_centroids(centroids, ldc, k, d, trace->mean, st));
    // split_clusters: re-seed empty clusters from big ones (EPS = 1/1024, rng(1234))
    bool any_empty = false;
    for (int c = 0; c < k; c++) any_empty |= (hassign[c] == 0);
    if (any_empty) {
      h_cent.resize((size_t)k * ldc);
      GB_CUDA(cudaMemcpyAsync(h_cent.data(), centroids, (size_t)k * ldc * 4, cudaMemcpyDeviceToHost, st));
      GB_CUDA(cudaStreamSynchronize(st));
      const float EPS = 1.0f / 1024.0f;
      std::mt19937 rng(1234u);
      for (int ci = 0; ci < k; ci++) {
        if (hassign[ci] != 0) continue;
        int cj;
        for (cj = 0;; cj = (cj + 1) % k) {
          float p = (hassign[cj] - 1.0f) / (float)(n - k);
          float r = (float)rng() / (float)4294967295u;
          if (r < p) break;
        }
        float* a = h_cent.data() + (size_t)ci * ldc;
        float* b = h_cent.data() + (size_t)cj * ldc;
        memcpy(a, b, sizeof(float) * d);
        for (int j = 0; j < d; j++) {
          if (j % 2 == 0) {
            a[j] *= 1 + EPS;
            b[j] *= 1 - EPS;
          } else {
            a[j] *= 1 - EPS;
            b[j] *= 1 + EPS;
          }
        }
        hassign[ci] = hassign[cj] / 2;
        hassign[cj] -= hassign[ci];
      }
      GB_CUDA(cudaMemcpyAsync(centroids, h_cent.data(), (size_t)k * ldc * 4, cudaMemcpyHostToDevice, st));
    }
    if (trace) GB_CUDA(trace_centroids(centroids, ldc, k, d, trace->split, st));
    if (kp.spherical) GB_CUDA(launch_normalize_rows(centroids, ldc, k, d, st));
    GB_CUDA(cudaStreamSynchronize(st));
    if (trace) GB_CUDA(trace_centroids(centroids, ldc, k, d, trace->norm, st));
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
IvfIndex::IvfIndex(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift, int row_bytes)
    : Index(type, d, mp, device, seg_shift, row_bytes), nlist_(mp.ncentroids) {
  mem::dev_malloc(&d_centroids_, (size_t)nlist_ * dpad_ * 4);
  cudaMemset(d_centroids_, 0, (size_t)nlist_ * dpad_ * 4);
  const int64_t ctiles = (nlist_ + 127) / 128;
  mem::dev_malloc(&d_cent_tiles_, (size_t)ctiles * tc_mirror_tile_floats((int)round_up(dpad_, 16)) * 4);
  mem::dev_malloc(&d_cent_norms_, (size_t)ctiles * 128 * 4);
  rebuild_centroid_tiles(0);
  cudaStreamSynchronize(0);
}
IvfIndex::~IvfIndex() {
  mem::dev_free(d_centroids_);
  mem::dev_free(d_cent_tiles_);
  mem::dev_free(d_cent_norms_);
}
IVFFlatIndex::IVFFlatIndex(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift)
    : IvfIndex(type, d, mp, device, seg_shift) {
  if (metric() == kMetricL2) {  // inner products are scanned unshifted: no table
    mem::dev_malloc(&d_shifts_, (size_t)nlist_ * dpad_ * 4);
    cudaMemset(d_shifts_, 0, (size_t)nlist_ * dpad_ * 4);  // = the zero centroids of an untrained index
  }
}
IVFFlatIndex::~IVFFlatIndex() {
  if (d_shifts_) mem::dev_free(d_shifts_);
  if (mirror_.base) mem::dev_free(mirror_.base);
  if (mirror_.norms) mem::dev_free(mirror_.norms);
  if (mirror_.d_tile0) mem::dev_free(mirror_.d_tile0);
  if (d_rowptr_) mem::dev_free(d_rowptr_);
}
int IvfIndex::rebuild_centroid_tiles(cudaStream_t st) {
  GB_CUDA(launch_tc_stage_rows(d_centroids_, dpad_, nlist_, dpad_, (int)round_up(dpad_, 16), d_cent_tiles_, d_cent_norms_, st));
  return centroids_changed(st);
}
int IVFFlatIndex::centroids_changed(cudaStream_t st) {
  if (!d_shifts_) return 0;  // inner product: the mirror holds the raw rows, whatever the centroids
  GB_CUDA(launch_list_shifts(d_centroids_, dpad_, nlist_, d_, d_shifts_, st));
  std::unique_lock<std::shared_mutex> ml(mirror_rw_);
  mirror_.lens.clear();  // staged with the old shifts: rebuilt by the next list-major search
  return 0;
}
int IVFFlatIndex::get_list_shifts(float* host) const {
  if (!d_shifts_) {
    set_last_error("IVFFLAT: list shifts exist only under L2");
    return -1;
  }
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy2D(host, (size_t)d_ * 4, d_shifts_, (size_t)dpad_ * 4, (size_t)d_ * 4, nlist_, cudaMemcpyDeviceToHost));
  return 0;
}

int64_t IvfIndex::training_threshold() const {
  // Indexing() clamps to [39, 256] * nlist in size_t (gamma_index_ivfflat.cc:350-375, gamma_index_ivfpq.cc:304-329):
  // from nlist = 2^23 on, 256 * nlist no longer fits an int
  int64_t t = mp_.training_threshold ? mp_.training_threshold : default_training_threshold();
  if (t < nlist_)
    t = (int64_t)nlist_ * 39;
  else if (t > (int64_t)nlist_ * 256)
    t = (int64_t)nlist_ * 256;
  return t;
}
static int64_t tc_tile_bytes(int dpad) { return tc_mirror_tile_floats((int)round_up(dpad, 16)) * 4 + 512; }
int64_t IvfIndex::index_mem_bytes() const {
  const int64_t cent_tiles = (nlist_ + 127) / 128 * tc_tile_bytes(dpad_);
  return (int64_t)nlist_ * dpad_ * 4 + cent_tiles + (lists_ ? lists_->mem_bytes() : 0);
}
int64_t IVFFlatIndex::index_mem_bytes() const {
  return IvfIndex::index_mem_bytes() + (d_shifts_ ? (int64_t)nlist_ * dpad_ * 4 : 0) + mirror_.cap_tiles * tc_tile_bytes(dpad_) +
         rowptr_cap_ * (int64_t)sizeof(float*);
}
int IvfIndex::set_centroids(const float* host, int nlist) {
  if (nlist != nlist_) {
    set_last_error("set_centroids: nlist mismatch");
    return -1;
  }
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  GB_CUDA(cudaMemset(d_centroids_, 0, (size_t)nlist_ * dpad_ * 4));
  GB_CUDA(cudaMemcpy2D(d_centroids_, (size_t)dpad_ * 4, host, (size_t)d_ * 4, (size_t)d_ * 4, nlist_,
                       cudaMemcpyHostToDevice));
  if (rebuild_centroid_tiles(0)) return -1;
  GB_CUDA(cudaStreamSynchronize(0));  // searches run on other (non-blocking) streams
  if (!lists_) lists_.reset(new IvfLists(nlist_, code_bytes()));
  trained_ = true;
  return 0;
}
int IvfIndex::get_centroids(float* host) const {
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy2D(host, (size_t)d_ * 4, d_centroids_, (size_t)dpad_ * 4, (size_t)d_ * 4, nlist_,
                       cudaMemcpyDeviceToHost));
  return 0;
}

// GammaIVFFlatIndex::Indexing (gamma_index_ivfflat.cc:342-411): train on the FIRST num vectors.
int IvfIndex::train() { return train_on(*store_); }
int IvfIndex::train_on(RawStore& src) {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (trained_) return 0;
  cudaSetDevice(device_);
  int64_t num = training_threshold();
  if (num > src.size()) {
    set_last_error("vector total count less than training_threshold");
    return -1;
  }
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  cudaStream_t st = build_stream_;
  Scratch s(st);
  const float* xt = src.contiguous(num, s);
  if (!xt) return -1;
  xt = train_transform(xt, num, s);  // OPQ: learn the rotation, continue on the rotated slab
  if (!xt) return -1;
  if (kmeans_device(xt, dpad_, num, d_, nlist_, coarse_kmeans_params(), d_centroids_, dpad_, st, nullptr)) return -1;
  if (rebuild_centroid_tiles(st)) return -1;
  if (train_extra(xt, num, s)) return -1;
  GB_CUDA(cudaStreamSynchronize(st));
  if (!lists_) lists_.reset(new IvfLists(nlist_, code_bytes()));
  trained_ = true;
  return 0;
}

int IvfIndex::assign_dev(const float* x, int64_t ldx, int64_t n, int32_t* out, Scratch& s) {
  cudaStream_t st = s.stream();
  GB_ALLOC(best, unsigned long long, n, s);
  GB_CUDA(launch_fill_u64(best, n, kKeySentinel, st));
  // always the exact CUDA-core kernel, never the tensor-core tiles: list membership stays deterministic against the oracle
  const int metric = coarse_metric(mp_.metric);
  GB_CUDA(launch_dist_argmin(x, ldx, (int)n, d_centroids_, dpad_, nlist_, dpad_, metric, best, 0, st));
  GB_CUDA(launch_split_keys(best, n, metric, nullptr, out, st));
  return 0;
}

int IVFFlatIndex::append_batch(const void* xv, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                               const std::vector<int>& add, Scratch& s) {
  const float* x = static_cast<const float*>(xv);
  GB_CUDA(launch_ivf_append_vecs(x, dpad_, n, dpad_, d_list, d_pos, reinterpret_cast<float* const*>(lists_->d_data()),
                                 lists_->d_ids(), vid0, s.stream()));
  // the tensor-core mirror's rows after the list data, before the new lengths are committed
  return mirror_append(x, n, d_list, d_pos, add, s.stream());
}

// GammaIVFFlatIndex::Add (gamma_index_ivfflat.cc:413-474) driven like
// VectorManager::AddRTVecsToIndex (vector_manager.cc:572-702), in large device batches.
int IvfIndex::assign_batch(const void* x, int64_t n, const void** xc, int32_t* out, Scratch& s) {
  const float* xt = transform_dev(static_cast<const float*>(x), n, s);  // OPQ rotation; the raw store keeps the original rows
  if (!xt) return -1;
  *xc = xt;
  return assign_dev(xt, dpad_, n, out, s);
}

int IvfIndex::index_batch(const void* x, int64_t n, int64_t vid0, const uint8_t* del_bitmap) {
  cudaStream_t st = build_stream_;
  Scratch s(st);
  GB_ALLOC(d_assign, int32_t, n, s);
  if (assign_batch(x, n, &x, d_assign, s)) return -1;
  std::vector<int32_t> h_list(n), h_pos(n);
  GB_CUDA(cudaMemcpyAsync(h_list.data(), d_assign, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  std::vector<int> add(nlist_, 0);
  const std::vector<int>& lens = lists_->lens();
  if ((int64_t)vid2pos_.size() < vid0 + n) vid2pos_.resize(vid0 + n, ~(uint64_t)0);
  for (int64_t i = 0; i < n; i++) {
    int64_t vid = vid0 + i, gvid = global_vid(vid);
    int l = h_list[i];
    if (del_bitmap && ((del_bitmap[gvid >> 3] >> (gvid & 7)) & 1)) {  // ivfflat.cc:436: deleted before indexing
      h_list[i] = -1;
      h_pos[i] = 0;
      continue;
    }
    if (l < 0 || l >= nlist_) l = (int)(gvid % nlist_);  // ivfflat.cc:443-446
    h_list[i] = l;
    h_pos[i] = lens[l] + add[l]++;  // insertion (vid) order inside the list
    vid2pos_[vid] = ((uint64_t)l << 32) | (uint32_t)h_pos[i];
  }
  GB_ALLOC(d_list, int32_t, n, s);
  GB_ALLOC(d_pos, int32_t, n, s);
  GB_CUDA(cudaMemcpyAsync(d_list, h_list.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_pos, h_pos.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();  // kernels of earlier searches read lengths and base pointers at run time
  if (lists_->reserve(add, st)) return -1;
  // data first, the new lengths last (realtime_mem_data.cc:292-293)
  if (append_batch(x, n, vid0, d_list, d_pos, add, s)) return -1;
  if (lists_->commit(add, st)) return -1;
  if (lists_changed(st)) return -1;
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int IvfIndex::add_pending(const uint8_t* del_bitmap) {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (!trained_) return 0;
  cudaSetDevice(device_);
  const int64_t BATCH = 1 << 20;
  for (;;) {
    int64_t vid0 = indexed_count_, n = 0;
    const void* x = nullptr;
    Scratch s(build_stream_);
    {  // add_vectors (exclusive mu_) may append segments while we look: the segment table is read under the shared lock
      std::shared_lock<std::shared_mutex> lk(mu_);
      if (vid0 >= store_->size()) break;
      // HBM rows are indexed in place, so a batch ends at its segment's end.  Host rows are copied to HBM first, across
      // segments: their batches end at the same BATCH-aligned rows, so both placements build the same list layout.
      const int64_t span = store_->on_host() ? BATCH : store_->seg_rows();
      int64_t off = vid0 & (span - 1);
      n = std::min<int64_t>(std::min(store_->size() - vid0, span - off), BATCH);
      x = store_rows_dev(vid0, n, s);
      if (!x) return -1;
    }
    if (index_batch(x, n, vid0, del_bitmap)) return -1;
    indexed_count_ += n;
  }
  // a bulk build leaves most of the slab space in regions the lists have outgrown: re-pack once the
  // waste is worth a copy (more than half of the live bytes and more than 1 GiB)
  if (lists_ && lists_->compact_due()) {
    std::unique_lock<std::shared_mutex> lk(mu_);
    if (compact_locked()) return -1;
  }
  return 0;
}

int IvfIndex::reset_index() {
  std::lock_guard<std::mutex> bg(build_mu_);
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  cudaDeviceSynchronize();  // kernels of earlier device-resident searches may still read the lists
  lists_.reset();
  vid2pos_.clear();
  del_counted_.clear();
  reset_codec();
  indexed_count_ = 0;
  trained_ = false;
  return 0;
}

void IvfIndex::clear_lists() {
  std::lock_guard<std::mutex> bg(build_mu_);
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  if (lists_) lists_.reset(new IvfLists(nlist_, code_bytes()));
  vid2pos_.clear();
  del_counted_.clear();
  indexed_count_ = 0;
  if (lists_) lists_changed(build_stream_);
  cudaStreamSynchronize(build_stream_);
}

void IVFFlatIndex::reset_codec() {
  std::unique_lock<std::shared_mutex> ml(mirror_rw_);
  mirror_.lens.clear();
}

int IvfIndex::compact_lists() {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (!lists_) return 0;
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  return compact_locked();
}
int IvfIndex::compact_locked() {
  if (lists_->compact(build_stream_) || lists_changed(build_stream_)) return -1;
  GB_CUDA(cudaStreamSynchronize(build_stream_));
  return 0;
}

// Host placement: the winner re-score of the list-major scan reads the list rows, byte copies of the raw rows, through
// a per-vid row-pointer table, so an IVF-Flat search never reads host memory.  Rebuilt whole after every change of the
// lists (growth and compaction move them), with mu_ held exclusively and earlier searches drained.
int IVFFlatIndex::lists_changed(cudaStream_t st) {
  if (!rescore_from_lists() || !lists_) return 0;
  drain_searches();  // no kernel of an earlier search reads the table while it is rewritten or freed
  const int64_t need = (int64_t)vid2pos_.size();
  if (need > rowptr_cap_) {
    const int64_t cap = std::max<int64_t>(need, rowptr_cap_ + rowptr_cap_ / 2);
    const float** p = nullptr;
    GB_CUDA(mem::dev_malloc(&p, (size_t)cap * sizeof(float*)));
    GB_CUDA(cudaMemsetAsync(p, 0, (size_t)cap * sizeof(float*), st));
    mem::dev_free(d_rowptr_);
    d_rowptr_ = p;
    rowptr_cap_ = cap;
  }
  GB_CUDA(launch_ivf_rowptrs(lists_->directory(), dpad_, d_rowptr_, st));
  return 0;
}

int Index::update_vector(int64_t vid, const void* x) {
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  // host rows are overwritten by the CPU at once, not in stream order: no kernel or copy of an earlier search may still
  // read them
  if (store_->on_host()) drain_searches();
  return store_->update_host(vid, x, build_stream_);
}

// GammaIVFFlatIndex::Update / GammaIVFPQIndex::Update (gamma_index_ivfflat.cc:476-522,
// gamma_index_ivfpq.cc:402-453): tombstone the old entry, append the new vector to its list.
int IvfIndex::update_vector(int64_t vid, const void* x) {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (Index::update_vector(vid, x)) return -1;
  if (!trained_ || vid >= indexed_count_) return 0;  // not indexed yet: the add path will pick it up
  Scratch s(build_stream_);
  const void* x_dev = store_rows_dev(vid, 1, s);
  if (!x_dev) return -1;
  return reindex_vector(vid, x_dev);
}
int IvfIndex::reindex_vector(int64_t vid, const void* x_dev) {
  if (vid < (int64_t)vid2pos_.size() && vid2pos_[vid] != ~(uint64_t)0) {
    std::unique_lock<std::shared_mutex> lk(mu_);
    const int l = (int)(vid2pos_[vid] >> 32);
    if (vid < (int64_t)del_counted_.size() && del_counted_[vid]) {  // counted as deleted: the tombstone counts it instead
      del_counted_[vid] = false;
      lists_->add_dead(l, -1);
    }
    if (lists_->tombstone(l, (int)(uint32_t)vid2pos_[vid], build_stream_)) return -1;
  }
  return index_batch(x_dev, 1, vid, nullptr);
}

int IvfIndex::delete_vectors(const int64_t* vids, int64_t n) {
  std::lock_guard<std::mutex> bg(build_mu_);
  if (!lists_) return 0;
  for (int64_t i = 0; i < n; i++) {
    const int64_t vid = vids[i];
    if (vid < 0 || vid >= (int64_t)vid2pos_.size() || vid2pos_[vid] == ~(uint64_t)0) continue;
    if (del_counted_.size() < vid2pos_.size()) del_counted_.resize(vid2pos_.size(), false);
    if (del_counted_[vid]) continue;
    del_counted_[vid] = true;
    lists_->add_dead((int)(vid2pos_[vid] >> 32), 1);  // realtime_mem_data.cc:194
  }
  return 0;
}

int IvfIndex::dead_counts(int* out) {
  std::lock_guard<std::mutex> bg(build_mu_);
  for (int l = 0; l < nlist_; l++) out[l] = lists_ ? lists_->dead_counts()[l] : 0;
  return 0;
}

std::vector<int> IvfIndex::purge_candidates(float threshold) const {
  std::vector<int> sel;
  if (!lists_) return sel;
  for (int l = 0; l < nlist_; l++) {
    const int dead = lists_->dead_counts()[l], len = lists_->lens()[l];
    if (dead > 0 && len > 0 && (float)dead / (float)len >= threshold) sel.push_back(l);  // Compactable (realtime_mem_data.cc:366-370)
  }
  return sel;
}

int IvfIndex::purge_lists(float threshold, const uint8_t* del_bitmap, int64_t bitmap_bytes, int64_t* dropped) {
  if (dropped) *dropped = 0;
  std::lock_guard<std::mutex> bg(build_mu_);
  const std::vector<int> sel = purge_candidates(threshold);
  if (sel.empty()) return 0;
  cudaSetDevice(device_);
  Scratch s(build_stream_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  SearchContext ctx;
  ctx.del_bitmap = del_bitmap;
  ctx.bitmap_bits = del_bitmap ? bitmap_bytes * 8 : 0;
  FilterArgs f;
  if (upload_bitmaps(ctx, &f, s)) return -1;
  return purge_locked(sel, f.del_bits, dropped);
}

int IvfIndex::purge_locked(const std::vector<int>& sel, const uint32_t* d_del_bits, int64_t* dropped) {
  cudaStream_t st = build_stream_;
  std::vector<char> purged(nlist_, 0);
  for (int l : sel) purged[l] = 1;
  drain_searches();  // kernels of earlier searches read lengths and base pointers at run time
  IvfLists::Purged pg;
  if (lists_->purge(sel, d_del_bits, st, &pg)) return -1;
  if (pg.dropped == 0) return 0;
  // vid_bucket_no_pos_ of every vid that was in a purged list, from the table the scatter wrote
  const int64_t hi = std::min<int64_t>((int64_t)vid2pos_.size(), pg.vid_min + (int64_t)pg.newpos.size());
  for (int64_t vid = pg.vid_min; vid < hi; vid++) {
    const uint64_t old = vid2pos_[vid];
    if (old == ~(uint64_t)0 || !purged[old >> 32]) continue;
    const uint64_t now = pg.newpos[vid - pg.vid_min];
    vid2pos_[vid] = now;
    if (vid < (int64_t)del_counted_.size() && del_counted_[vid]) {
      if (now == ~(uint64_t)0)
        del_counted_[vid] = false;
      else
        lists_->add_dead((int)(now >> 32), 1);  // deleted, but not in this bitmap: still there, still counted
    }
  }
  if (lists_changed(st)) return -1;
  GB_CUDA(cudaStreamSynchronize(st));
  if (dropped) *dropped = pg.dropped;
  // the regions the purged lists left behind are reclaimed by the re-pack, under its own policy
  if (lists_->compact_due() && compact_locked()) return -1;
  return 0;
}

int IvfIndex::resolve_nprobe(const SearchContext& ctx) const {
  int nprobe = mp_.nprobe;
  // ivfflat.cc:551-559; the GPU types' GetNprobe (gamma_index_ivfpq_gpu.cc:584-594) also refuses a request above kGpuMaxK
  const int max_req = gpu_contract_ ? std::min(nlist_, kGpuMaxK) : nlist_;
  if (ctx.params.nprobe > 0 && ctx.params.nprobe <= max_req) nprobe = ctx.params.nprobe;
  if (nprobe > nlist_) nprobe = nlist_;
  if (nprobe > 4096) nprobe = 4096;
  return nprobe;
}

// GB_COARSE_FUSED=0: always write the query x centroid score matrix and select from it (A/B runs; the reference of the
// fused path's tests).  Read per call: tests flip it between searches of one process.
static bool coarse_fused_enabled() {
  const char* e = getenv("GB_COARSE_FUSED");
  return e ? atoi(e) != 0 : true;
}

// quantizer->search (gamma_index_ivfflat.cc:568 / gamma_index_ivfpq.cc:595)
int IvfIndex::coarse_dev(int nq, const void* xqv, int nprobe, int metric, int32_t* probe_ids, float* coarse_dis,
                         Scratch& s) {
  cudaStream_t st = s.stream();
  const float* xq = static_cast<const float*>(xqv);
  GB_ALLOC(keys, unsigned long long, (size_t)nq * nprobe, s);
  const bool tc = nlist_ >= 64 && nq >= 32;
  const int k16 = (int)round_up(dpad_, 16);
  if (tc && coarse_fused_enabled() && nprobe <= kCoarseMaxK && k16 > 16) {
    // fused: each query's best nprobe keys straight from the tensor-core tiles; no score matrix
    const int nqt = (nq + 127) / 128, nsm = sm_count(device_);
    GB_ALLOC(a_tiles, float, (size_t)nqt * tc_mirror_tile_floats(k16), s);
    GB_ALLOC(a_norms, float, (size_t)nqt * 128, s);
    GB_ALLOC(ws, unsigned char, coarse_topk_workspace_bytes(nq, nlist_, nprobe, nsm), s);
    StageScope stage(this, "coarse_quantizer", st);
    last_coarse_kernel_ = "coarse_topk_kernel";
    GB_CUDA(launch_tc_stage_rows(xq, dpad_, nq, dpad_, k16, a_tiles, a_norms, st));
    GB_CUDA(launch_coarse_topk(a_tiles, a_norms, nq, d_cent_tiles_, d_cent_norms_, nlist_, k16, metric, nprobe, nsm, ws, keys,
                               st));
    GB_CUDA(launch_split_keys(keys, (int64_t)nq * nprobe, metric, coarse_dis, probe_ids, st));
    return 0;
  }
  int64_t ldo = round_up(nlist_, 4);
  GB_ALLOC(scores, float, (size_t)nq * ldo, s);
  StageScope stage(this, "coarse_quantizer", st);
  last_coarse_kernel_ = tc ? "dist_tc_kernel+select_rows_kernel" : "dist_tile_kernel+select_rows_kernel";
  if (tc) {
    GB_CUDA(launch_dist_matrix_tc(xq, dpad_, nq, d_centroids_, dpad_, nlist_, dpad_, metric, scores, ldo, st));
  } else {
    GB_CUDA(launch_dist_matrix(xq, dpad_, nq, d_centroids_, dpad_, nlist_, dpad_, metric, scores, ldo, st));
  }
  FilterArgs nf{nullptr, nullptr, -FLT_MAX, FLT_MAX};
  GB_CUDA(launch_select_scores(scores, ldo, nq, nlist_, 0, nprobe, metric, nf, keys, nprobe, st));
  GB_CUDA(launch_split_keys(keys, (int64_t)nq * nprobe, metric, coarse_dis, probe_ids, st));
  return 0;
}

// List-major scan (DESIGN.md K3-LM): worthwhile when many queries of the batch probe each list.
// Host side: group the (query, probe) pairs by list (stable counting sort), give every pair a
// score segment of len(list) floats, cut (list, 128 pairs, 128 rows) tiles; device side: grouped
// GEMM on wgmma + segment select.

int IvfIndex::alloc_pair_grouping(int64_t npairs, int64_t max_items, LmGrouping* g, Scratch& s) {
  GB_ALLOC(d_cnt, int32_t, nlist_, s);
  GB_ALLOC(d_start, int32_t, nlist_, s);
  GB_ALLOC(d_cursor, int32_t, nlist_, s);
  GB_ALLOC(d_item_start, int32_t, nlist_, s);
  GB_ALLOC(d_grp_start, int32_t, nlist_, s);
  GB_ALLOC(totals, int64_t, 3, s);
  GB_ALLOC(pair_j, int64_t, npairs, s);
  GB_ALLOC(items, LmTile, max_items, s);
  *g = {d_cnt, d_start, d_cursor, d_item_start, d_grp_start, totals, pair_j, items};
  return 0;
}
cudaError_t IvfIndex::group_pairs_by_list(const int32_t* probe_ids, int64_t npairs, int nseg, int group,
                                          const LmGrouping& g, cudaStream_t st) {
  return launch_lmk_group(probe_ids, npairs, lists_->directory(), nseg, group, g.cnt, g.start, g.cursor, g.item_start,
                          g.grp_start, g.totals, g.pair_j, g.items, st);
}

// called from index_batch with mu_ held exclusively: no search is inside ensure_mirror.  Kernels of an
// earlier search_device may still be running, but they only look at rows below the lengths they were
// launched with, and the rows written here lie above those.
int IVFFlatIndex::mirror_append(const float* x, int64_t n, const int32_t* d_list, const int32_t* d_pos,
                                const std::vector<int>& add, cudaStream_t st) {
  if (!mirror_.base || mirror_.disabled || mirror_.lens.size() != (size_t)nlist_) return 0;
  std::vector<int> lens = lists_->lens();  // lengths BEFORE this batch is committed
  for (int l = 0; l < nlist_; l++) {
    if (mirror_.lens[l] != lens[l] || mirror_.content_gen != lists_->content_gen() ||
        (int64_t)lens[l] + add[l] > (int64_t)mirror_.list_tiles[l] * 128) {
      mirror_.lens.clear();  // stale: outgrown, purged or out of step; rebuilt by the next list-major search
      return 0;
    }
    lens[l] += add[l];
  }
  GB_CUDA(launch_tc_mirror_append(x, dpad_, n, dpad_, (int)round_up(dpad_, 16), d_list, d_pos, mirror_.d_tile0,
                                  d_shifts_, mirror_.base, mirror_.norms, st));
  mirror_.lens = lens;
  return 0;
}

int IVFFlatIndex::ensure_mirror(std::shared_lock<std::shared_mutex>& lk, cudaStream_t st) {
  if (!lists_) return 1;
  lk.lock();
  if (mirror_.disabled) return 1;
  if (mirror_current()) return 0;
  lk.unlock();
  {
    std::unique_lock<std::shared_mutex> x(mirror_rw_);
    if (!mirror_.disabled && !mirror_current()) {
      const std::vector<int>& lens = lists_->lens();
      const int k16 = (int)round_up(dpad_, 16);
      const size_t tile_bytes = (size_t)tc_mirror_tile_floats(k16) * 4;
      cudaDeviceSynchronize();  // kernels of other searches may still be reading the mirror
      if (mirror_.base) mem::dev_free(mirror_.base);
      if (mirror_.norms) mem::dev_free(mirror_.norms);
      mirror_.base = mirror_.norms = nullptr;
      mirror_.cap_tiles = 0;
      size_t free_b = 0, total_b = 0;
      cudaMemGetInfo(&free_b, &total_b);
      std::vector<int64_t> tile0(nlist_ + 1, 0);
      std::vector<int> list_tiles(nlist_, 0);
      int64_t tiles = 0;
      for (int slack = 8; slack >= 0 && !mirror_.base; slack -= 8) {  // 1/8 more rows per list, else none
        for (int l = 0; l < nlist_; l++) {
          const int64_t rows = slack ? (int64_t)lens[l] + lens[l] / slack : lens[l];
          list_tiles[l] = (int)((rows + 127) / 128);
          tile0[l + 1] = tile0[l] + list_tiles[l];
        }
        tiles = tile0[nlist_];
        const size_t need = (size_t)std::max<int64_t>(tiles, 1) * (tile_bytes + 512);
        if (need + ((size_t)4 << 30) > free_b) continue;
        if (mem::dev_malloc(&mirror_.base, (size_t)std::max<int64_t>(tiles, 1) * tile_bytes) != cudaSuccess ||
            mem::dev_malloc(&mirror_.norms, (size_t)std::max<int64_t>(tiles, 1) * 512) != cudaSuccess) {
          if (mirror_.base) mem::dev_free(mirror_.base);
          mirror_.base = nullptr;
          cudaGetLastError();
        }
      }
      if (!mirror_.base) {
        mirror_.disabled = true;  // HBM too full for a second, doubled copy of the lists
      } else {
        mirror_.cap_tiles = tiles;
        mirror_.list_tiles = list_tiles;
      }
      if (!mirror_.disabled) {
        if (!mirror_.d_tile0 && mem::dev_malloc(&mirror_.d_tile0, sizeof(int64_t) * (nlist_ + 1)) != cudaSuccess) return -1;
        GB_CUDA(cudaMemcpyAsync(mirror_.d_tile0, tile0.data(), sizeof(int64_t) * (nlist_ + 1), cudaMemcpyHostToDevice, st));
        GB_CUDA(launch_tc_mirror_build(lists_->directory(), dpad_, k16, mirror_.d_tile0, tiles,
                                       d_shifts_, mirror_.base, mirror_.norms, st));
        GB_CUDA(cudaStreamSynchronize(st));  // tile0 is a stack vector; other streams may use the mirror next
        mirror_.tiles = tiles;
        mirror_.lens = lens;
        mirror_.content_gen = lists_->content_gen();
        mirror_.builds++;
      }
    }
  }
  lk.lock();
  if (mirror_.disabled) return 1;
  return mirror_current() ? 0 : 1;
}

int IVFFlatIndex::scan_listmajor_dev(const FilterArgs& f, int metric, int nq, const float* xq, int k,
                                     const int32_t* probe_ids, int nprobe, unsigned long long* out_keys, Scratch& s) {
  const int64_t npairs = (int64_t)nq * nprobe;
  if (npairs < (int64_t)nlist_ * 32) return 1;  // < 32 queries per list on average
  // the mirror is staged for the index's metric (shifted under L2), so a search under the other metric scans
  // query-major
  if (metric != this->metric()) return 1;
  const float* shifts = d_shifts_;  // L2 index (the metrics agree): shifted; IP: nullptr
  cudaStream_t st = s.stream();
  ListDirectory dir = lists_->directory();
  if (k <= kLmkMaxK) {
    // fused top-k epilogue: no score round trip through HBM, no host synchronisation
    const int nseg = (int)std::min<int64_t>(8, std::max<int64_t>(1, (lists_->max_len() + kLmkSegRows - 1) / kLmkSegRows));
    const int64_t max_items = (npairs / 128 + nlist_) * nseg;
    if (max_items > INT32_MAX) return 1;
    GB_ALLOC(d_tau, unsigned long long, nq, s);
    const size_t nout = (size_t)npairs * nseg * k;
    GB_ALLOC(d_out, unsigned long long, nout, s);
    GB_CUDA(cudaMemsetAsync(d_tau, 0xFF, sizeof(unsigned long long) * nq, st));
    GB_CUDA(cudaMemsetAsync(d_out, 0xFF, sizeof(unsigned long long) * nout, st));
    LmGrouping g;
    if (alloc_pair_grouping(npairs, max_items, &g, s)) return -1;
    GB_CUDA(group_pairs_by_list(probe_ids, npairs, nseg, 128, g, st));
    const int k16 = (int)round_up(dpad_, 16);
    const int64_t max_groups = npairs / 128 + nlist_;
    const size_t slot_bytes = (size_t)128 * k16 * 8, a_bytes = (size_t)max_groups * (slot_bytes + 128 * 4);
    std::shared_lock<std::shared_mutex> mlk(mirror_rw_, std::defer_lock);
    // TMA-fed from the mirror when it applies and fits, else the register-staged pipeline over the lists themselves
    bool tma = k <= 32 && k16 > 16 && a_bytes <= ((size_t)8 << 30) && ensure_mirror(mlk, st) == 0;
    if (tma) {
      BigScope big(this, a_bytes, st);
      if (!big.p) return -1;
      float* a_scratch = static_cast<float*>(big.p);
      float* a_norms = reinterpret_cast<float*>(reinterpret_cast<char*>(a_scratch) + (size_t)max_groups * slot_bytes);
      TcMirrorView mv{mirror_.base, mirror_.d_tile0, mirror_.norms, k16};
      last_scan_kernel_ = "ivf_listmajor_tma_kernel";
      scan_timer_begin(st);
      GB_CUDA(launch_lm_stage_queries(xq, dpad_, dpad_, k16, g.items, (int)max_items, g.totals, g.pair_j, nprobe, shifts,
                                      a_scratch, a_norms, st));
      GB_CUDA(launch_ivf_listmajor_tma(a_scratch, a_norms, mv, g.items, (int)max_items, g.totals, g.pair_j, nprobe, dir, k,
                                       nseg, metric, f, d_tau, d_out, st));
      scan_timer_end(st);
    } else {
      last_scan_kernel_ = "ivf_listmajor_pipe_kernel";
      scan_timer_begin(st);
      GB_CUDA(launch_ivf_listmajor_pipe(xq, dpad_, dpad_, g.items, (int)max_items, g.totals, g.pair_j, nprobe, dir, shifts, k,
                                        nseg, metric, f, d_tau, d_out, st));
      scan_timer_end(st);
    }
    if (mlk.owns_lock()) mlk.unlock();
    GB_CUDA(launch_select_keys(d_out, (int64_t)nprobe * nseg * k, nq, nprobe * nseg * k, k, out_keys, k, st));
    return 0;
  }
  GB_ALLOC(d_cnt, int32_t, nlist_, s);
  GB_ALLOC(d_start, int32_t, nlist_, s);
  GB_ALLOC(d_cursor, int32_t, nlist_, s);
  GB_ALLOC(d_tile_start, int32_t, nlist_, s);
  GB_ALLOC(d_base_off, int64_t, nlist_, s);
  GB_ALLOC(d_totals, int64_t, 3, s);
  GB_CUDA(launch_lm_count_scan(probe_ids, npairs, dir, d_cnt, d_start, d_base_off, d_tile_start, d_totals, st));
  int64_t h_totals[3] = {0, 0, 0};
  GB_CUDA(cudaMemcpyAsync(h_totals, d_totals, sizeof(h_totals), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  const int64_t total = h_totals[0], ntiles = h_totals[1];
  if (total > ((int64_t)3 << 30) || ntiles > INT32_MAX) return 1;  // > 12 GiB of scores: query-major scan instead
  GB_ALLOC(d_pair_q, int32_t, npairs, s);
  GB_ALLOC(d_pair_off, int64_t, npairs, s);
  GB_ALLOC(d_seg_off, int64_t, npairs, s);
  GB_ALLOC(d_tiles, LmTile, std::max<int64_t>(ntiles, 1), s);
  BigScope big(this, (size_t)std::max<int64_t>(total, 1) * 4, st);
  if (!big.p) return -1;
  float* scores = static_cast<float*>(big.p);
  GB_CUDA(launch_lm_assign_tiles(probe_ids, npairs, nprobe, dir, d_cnt, d_start, d_cursor, d_base_off, d_tile_start,
                                 d_pair_q, d_pair_off, d_seg_off, d_tiles, st));
  last_scan_kernel_ = "ivf_listmajor_tc_kernel+seg_select_kernel";
  scan_timer_begin(st);
  GB_CUDA(launch_ivf_listmajor_tc(xq, dpad_, dpad_, d_tiles, (int)ntiles, d_pair_q, d_pair_off, dir, shifts, metric, scores,
                                  st));
  GB_CUDA(launch_seg_select(scores, d_seg_off, probe_ids, nq, nprobe, dir, k, metric, f, out_keys, st));
  scan_timer_end(st);
  return 0;
}

int IVFFlatIndex::scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xqv,
                           const void* xq_raw, int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                           unsigned long long* out_keys, Scratch& s) {
  (void)ctx;
  (void)xq_raw;  // no transform: xq is the raw queries
  (void)coarse_dis;
  cudaStream_t st = s.stream();
  const float* xq = static_cast<const float*>(xqv);
  // The list-major scan selects on 3xTF32 tensor-core scores.  Under L2 it evaluates |x - s|^2 + |y - s|^2 -
  // 2 (x - s).(y - s) with s = s_l, the shift of the probed list (d_shifts_, near its centroid), so the cancellation
  // error scales with the residual norms: on raw vectors with a common offset (|x|^2 ~ 1e8 at offset 1000, d = 128) the
  // rounding of |x|^2 + |y|^2 alone would exceed the gaps between neighbours.  The k winners are re-scored with the
  // direct fp32 form from the raw vectors and re-sorted (rerank_kernel, k rows per query), so every distance that
  // leaves the index is the exact-kernel value; on integer-valued data with integer shifts both forms are exact and
  // nothing changes.
  GB_ALLOC(lm_keys, unsigned long long, (size_t)nq * k, s);
  int lm = scan_listmajor_dev(f, metric, nq, xq, k, probe_ids, nprobe, lm_keys, s);
  if (lm < 0) return lm;
  if (lm == 0) {
    if ((dpad_ & 3) == 0 && k <= 8192) {
      if (rescore_from_lists()) {  // the list rows, through the row-pointer table (lists_changed)
        if (!d_rowptr_) {
          set_last_error("IVFFLAT: the row-pointer table of the host store was not built");
          return -1;
        }
        GB_CUDA(launch_rerank(lm_keys, k, nq, xq, dpad_, dpad_, d_rowptr_, 0, dpad_, false, k, metric, f, out_keys, st));
      } else {
        GB_CUDA(launch_rerank(lm_keys, k, nq, xq, dpad_, dpad_, store_->d_segs(), store_->seg_shift(), dpad_, false, k,
                              metric, f, out_keys, st));
      }
    } else {
      GB_CUDA(cudaMemcpyAsync(out_keys, lm_keys, (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, st));
    }
    return 0;
  }
  // Every query keeps k keys per (probe, split) until the merge, and the split count follows the longest list of the
  // index: one list of 2^20 rows gives every query 128 splits per probe.  The batch is scanned in query blocks whose
  // partials stay within kScanPartialBudget, as flat_search_dev blocks its score tiles.  A block holds one query at
  // least, so a single query's nprobe x nsplit x k keys are the residual (nprobe 2048 over a 2^20-row list at
  // k = 4096: 8.6 GB); cutting the probes as well would bound that too.
  int nparts = ivfflat_scan_nparts(nprobe, lists_->max_len());
  const int64_t per_query = (int64_t)nparts * k * 8;
  const int QB = (int)std::max<int64_t>(1, std::min<int64_t>(nq, kScanPartialBudget / per_query));
  GB_ALLOC(partial, unsigned long long, (size_t)QB * nparts * k, s);
  int avg_len = (int)(lists_->total() / std::max(1, nlist_));
  for (int q0 = 0; q0 < nq; q0 += QB) {  // the scan timer covers the scans, never the merges (last_scan_ms sums them)
    const int qb = std::min(QB, nq - q0);
    nparts = ivfflat_scan_nparts(nprobe, lists_->max_len());
    scan_timer_begin(st);
    GB_CUDA(launch_ivfflat_scan(xq + (int64_t)q0 * dpad_, dpad_, qb, dpad_, probe_ids + (int64_t)q0 * nprobe, nprobe,
                                lists_->directory(), lists_->max_len(), avg_len, k, metric, f, partial, &nparts,
                                &last_scan_kernel_, st));
    scan_timer_end(st);
    GB_CUDA(launch_select_keys(partial, (int64_t)nparts * k, qb, nparts * k, k, out_keys + (int64_t)q0 * k, k, st));
  }
  return 0;
}

// GammaIVFFlatIndex::Search (gamma_index_ivfflat.cc:524-577)
int IvfIndex::search_keys_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq_in, int k,
                              unsigned long long* out_keys, Scratch& s) {
  const void* xq = transform_dev(static_cast<const float*>(xq_in), nq, s);  // the identity unless an OPQ rotation is set
  if (!xq) return -1;
  const int nprobe = resolve_nprobe(ctx);
  const int64_t ld = store_->stride();
  const int QB = 16384;
  for (int q0 = 0; q0 < nq; q0 += QB) {
    int qb = std::min(QB, nq - q0);
    Scratch sb(s.stream());
    GB_ALLOC(probe_ids, int32_t, (size_t)qb * nprobe, sb);
    GB_ALLOC(coarse_dis, float, (size_t)qb * nprobe, sb);
    const void* xb = static_cast<const unsigned char*>(xq) + q0 * ld;
    if (coarse_dev(qb, xb, nprobe, coarse_metric(metric), probe_ids, coarse_dis, sb)) return -1;
    if (scan_dev(ctx, f, metric, qb, xb, static_cast<const unsigned char*>(xq_in) + q0 * ld, k, probe_ids, coarse_dis, nprobe,
                 out_keys + (int64_t)q0 * k, sb))
      return -1;
  }
  return 0;
}

int IvfIndex::coarse_search_host(int nq, const void* x, int nprobe, float* out_dis, int64_t* out_ids) {
  if (nq <= 0) return 0;
  if (!trained_ || nprobe <= 0 || nprobe > std::min(nlist_, 4096)) {
    set_last_error("coarse_search: untrained index or nprobe out of range");
    return -1;
  }
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  std::shared_lock<std::shared_mutex> lk(mu_);
  Scratch s(st);
  const void* dq = upload_queries(nq, x, s);
  if (!dq) return -1;
  GB_ALLOC(ids, int32_t, (size_t)nq * nprobe, s);
  GB_ALLOC(dis, float, (size_t)nq * nprobe, s);
  const float* dqt = transform_dev(static_cast<const float*>(dq), nq, s);
  if (!dqt || coarse_dev(nq, dqt, nprobe, coarse_metric(mp_.metric), ids, dis, s)) return -1;
  std::vector<int32_t> h((size_t)nq * nprobe);
  GB_CUDA(cudaMemcpyAsync(h.data(), ids, h.size() * 4, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaMemcpyAsync(out_dis, dis, h.size() * 4, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  for (size_t i = 0; i < h.size(); i++) out_ids[i] = h[i];
  return 0;
}

int IvfIndex::search_preassigned_host(const SearchContext& ctx, int nq, const void* x, int k, const int64_t* keys,
                                      const float* coarse_dis, int nprobe, float* out_dis, int64_t* out_ids) {
  if (nq <= 0) return 0;
  if (check_gpu_request(ctx, nq, k)) return -1;
  if (!trained_ || !lists_ || k <= 0 || k > 4096 || nprobe <= 0 || nprobe > 4096) {
    set_last_error("search_preassigned: untrained index, topK or nprobe out of range");
    return -1;
  }
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  std::shared_lock<std::shared_mutex> lk(mu_);
  Scratch s(st);
  const void* dq = upload_queries(nq, x, s);
  if (!dq) return -1;
  std::vector<int32_t> h((size_t)nq * nprobe);
  for (size_t i = 0; i < h.size(); i++) h[i] = (int32_t)keys[i];
  GB_ALLOC(ids, int32_t, h.size(), s);
  GB_ALLOC(dis, float, h.size(), s);
  GB_CUDA(cudaMemcpyAsync(ids, h.data(), h.size() * 4, cudaMemcpyHostToDevice, st));
  if (coarse_dis) {
    GB_CUDA(cudaMemcpyAsync(dis, coarse_dis, h.size() * 4, cudaMemcpyHostToDevice, st));
  } else {
    GB_CUDA(cudaMemsetAsync(dis, 0, h.size() * 4, st));
  }
  FilterArgs f;
  if (upload_bitmaps(ctx, &f, s)) return -1;
  const int metric = search_metric(ctx);
  GB_ALLOC(okeys, unsigned long long, (size_t)nq * k, s);
  const float* dqt = transform_dev(static_cast<const float*>(dq), nq, s);
  if (!dqt) return -1;
  if (scan_dev(ctx, f, metric, nq, dqt, dq, k, ids, dis, nprobe, okeys, s)) return -1;
  return download_results(okeys, nq, k, metric, out_dis, out_ids, s);  // synchronises before h goes
}

// ------------------------------------------------------------------------------------------
IvfPqBase::IvfPqBase(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift, int M, int ksub)
    : IvfIndex(type, d, mp, device, seg_shift), M_(M), dsub_(d / M), ksub_(ksub) {
  mem::dev_malloc(&d_pq_, (size_t)M_ * ksub_ * dsub_ * 4);
  cudaMemset(d_pq_, 0, (size_t)M_ * ksub_ * dsub_ * 4);
}
IvfPqBase::~IvfPqBase() { mem::dev_free(d_pq_); }
int64_t IvfPqBase::index_mem_bytes() const { return IvfIndex::index_mem_bytes() + (int64_t)M_ * ksub_ * dsub_ * 4; }
int IvfPqBase::set_pq_centroids(const float* host) {
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  GB_CUDA(cudaMemcpy(d_pq_, host, (size_t)M_ * ksub_ * dsub_ * 4, cudaMemcpyHostToDevice));
  if (codebook_changed(build_stream_)) return -1;
  GB_CUDA(cudaStreamSynchronize(build_stream_));
  return 0;
}
int IvfPqBase::get_pq_centroids(float* host) const {
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy(host, d_pq_, (size_t)M_ * ksub_ * dsub_ * 4, cudaMemcpyDeviceToHost));
  return 0;
}

int IvfPqBase::train_codebook(const float* x, int64_t n, Scratch& s) {
  cudaStream_t st = s.stream();
  const int dsp = (int)round_up(dsub_, 4);
  GB_ALLOC(slice, float, (size_t)n * dsp, s);
  GB_ALLOC(cent, float, (size_t)ksub_ * dsp, s);
  KMeansParams kp;  // ClusteringParameters defaults: niter 25, seed 1234, max 256 points per centroid
  for (int m = 0; m < M_; m++) {
    GB_CUDA(launch_slice_cols(x, dpad_, n, m * dsub_, dsub_, slice, dsp, st));
    if (kmeans_device(slice, dsp, n, dsub_, ksub_, kp, cent, dsp, st, nullptr)) return -1;
    GB_CUDA(cudaMemcpy2DAsync(d_pq_ + (size_t)m * ksub_ * dsub_, (size_t)dsub_ * 4, cent, (size_t)dsp * 4, (size_t)dsub_ * 4,
                              ksub_, cudaMemcpyDeviceToDevice, st));
  }
  return codebook_changed(st);
}

int IvfPqBase::append_batch(const void* xv, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                            const std::vector<int>& add, Scratch& s) {
  (void)add;
  const float* x = static_cast<const float*>(xv);
  cudaStream_t st = s.stream();
  const int cb = code_bytes();
  GB_ALLOC(codes, uint8_t, (size_t)n * cb, s);
  GB_CUDA(encode_dev(x, n, d_list, codes, st));  // residual codecs: w.r.t. the assigned list
  GB_CUDA(launch_ivf_append_codes(codes, n, cb, d_list, d_pos, reinterpret_cast<uint8_t* const*>(lists_->d_data()),
                                  lists_->d_ids(), vid0, st));
  return 0;
}

int IvfPqBase::encode_host(const float* x, int64_t n, const int64_t* assign, uint8_t* codes_out) {
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  Scratch s(st);
  const int cb = code_bytes();
  GB_ALLOC(dx, float, (size_t)n * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, n, d_, dpad_, st));
  int32_t* da = nullptr;
  std::vector<int32_t> h;
  if (assign) {
    h.assign(assign, assign + n);
    da = s.alloc_n<int32_t>(n);
    if (!da) return -1;
    GB_CUDA(cudaMemcpyAsync(da, h.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  }
  GB_ALLOC(codes, uint8_t, (size_t)n * cb, s);
  GB_CUDA(encode_dev(dx, n, da, codes, st));
  GB_CUDA(cudaMemcpyAsync(codes_out, codes, (size_t)n * cb, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// ------------------------------------------------------------------------------------------
// gamma_index_ivfpq.cc:122-124: nsubvector defaults to d / 2
IVFPQIndex::IVFPQIndex(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift)
    : IvfPqBase(type, d, mp, device, seg_shift, std::max(1, mp.nsubvector > 0 ? mp.nsubvector : d / 2), 1 << mp.nbits),
      nbits_(mp.nbits) {
  if (!gpu_contract_) store_->enable_shadow();  // GPU_IVFPQ never re-ranks
  if (mp.opq_nsubvector > 0) {  // faiss::OPQMatrix(d, opq_nsubvector, d) (gamma_index_ivfpq.cc:168-178)
    mem::dev_malloc(&d_opq_, (size_t)d * dpad_ * 4);
    cudaMemset(d_opq_, 0, (size_t)d * dpad_ * 4);
  }
}

// ---- OPQ (faiss::OPQMatrix restated; VectorTransform.cpp of faiss v1.14.1 is not vendored) -------------
// train: centre the (sub-sampled, <= 65536) training set, start from a random orthonormal matrix, then 50
// rounds of { project; train a PQ on the projection (40 k-means iterations in the first round, 4 hot-started
// ones afterwards, <= 1000 points per centroid); reconstruct; solve the orthogonal Procrustes problem
// min ||X R^T - Y|| by an SVD of X^T Y }.  The projection and X^T Y run on the device, the d x d SVD (one-sided
// Jacobi, double precision) on the host.  The random start cannot reproduce faiss's generator, so parity with
// the reference is statistical (recall), as for k-means.
namespace {
// A (d x d2, row-major) = U diag(s) V^T by one-sided Jacobi on the columns; returns U (d x d2) and V (d2 x d2)
void jacobi_svd(std::vector<double>& a, int d, int d2, std::vector<double>* u, std::vector<double>* v) {
  v->assign((size_t)d2 * d2, 0.0);
  for (int i = 0; i < d2; i++) (*v)[(size_t)i * d2 + i] = 1.0;
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = 0;
    for (int p = 0; p < d2 - 1; p++)
      for (int q = p + 1; q < d2; q++) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < d; i++) {
          const double x = a[(size_t)i * d2 + p], y = a[(size_t)i * d2 + q];
          alpha += x * x, beta += y * y, gamma += x * y;
        }
        if (fabs(gamma) <= 1e-15 * sqrt(alpha * beta) || gamma == 0) continue;
        off = std::max(off, fabs(gamma) / sqrt(alpha * beta + 1e-300));
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        for (int i = 0; i < d; i++) {
          const double x = a[(size_t)i * d2 + p], y = a[(size_t)i * d2 + q];
          a[(size_t)i * d2 + p] = c * x - sn * y, a[(size_t)i * d2 + q] = sn * x + c * y;
        }
        for (int i = 0; i < d2; i++) {
          const double x = (*v)[(size_t)i * d2 + p], y = (*v)[(size_t)i * d2 + q];
          (*v)[(size_t)i * d2 + p] = c * x - sn * y, (*v)[(size_t)i * d2 + q] = sn * x + c * y;
        }
      }
    if (off < 1e-12) break;
  }
  u->assign((size_t)d * d2, 0.0);
  for (int j = 0; j < d2; j++) {
    double nrm = 0;
    for (int i = 0; i < d; i++) nrm += a[(size_t)i * d2 + j] * a[(size_t)i * d2 + j];
    nrm = sqrt(nrm);
    for (int i = 0; i < d; i++) (*u)[(size_t)i * d2 + j] = nrm > 1e-300 ? a[(size_t)i * d2 + j] / nrm : (i == j ? 1.0 : 0.0);
  }
}
}  // namespace

int IVFPQIndex::set_opq(const float* host_A) {
  if (!d_opq_) {
    set_last_error("index was created without opq");
    return -1;
  }
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  GB_CUDA(cudaMemset(d_opq_, 0, (size_t)d_ * dpad_ * 4));
  GB_CUDA(cudaMemcpy2D(d_opq_, (size_t)dpad_ * 4, host_A, (size_t)d_ * 4, (size_t)d_ * 4, d_, cudaMemcpyHostToDevice));
  opq_trained_ = true;
  return 0;
}
int IVFPQIndex::get_opq(float* host_A) const {
  if (!d_opq_) {
    set_last_error("index was created without opq");
    return -1;
  }
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy2D(host_A, (size_t)d_ * 4, d_opq_, (size_t)dpad_ * 4, (size_t)d_ * 4, d_, cudaMemcpyDeviceToHost));
  return 0;
}

// y = A x for n rows (stride dpad, padding columns zero): one exact fp32 contraction against the rows of A
const float* IVFPQIndex::transform_dev(const float* x, int64_t n, Scratch& s) {
  if (!d_opq_ || !opq_trained_ || n <= 0) return x;
  cudaStream_t st = s.stream();
  float* y = s.alloc_n<float>((size_t)n * dpad_);
  if (!y) return nullptr;
  if (dpad_ != d_ && cudaMemsetAsync(y, 0, (size_t)n * dpad_ * 4, st) != cudaSuccess) return nullptr;
  for (int64_t r0 = 0; r0 < n; r0 += (1 << 20)) {
    const int nr = (int)std::min<int64_t>(n - r0, 1 << 20);
    if (launch_dist_matrix(x + r0 * dpad_, dpad_, nr, d_opq_, dpad_, d_, dpad_, kMetricIP, y + r0 * dpad_, dpad_, st) !=
        cudaSuccess) {
      set_last_error("opq apply failed");
      return nullptr;
    }
  }
  return y;
}

int IVFPQIndex::apply_opq_host(const float* x, int64_t n, float* out) {
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  std::shared_lock<std::shared_mutex> lk(mu_);
  Scratch s(st);
  GB_ALLOC(dx, float, (size_t)n * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, n, d_, dpad_, st));
  const float* y = transform_dev(dx, n, s);
  if (!y) return -1;
  GB_CUDA(cudaMemcpy2DAsync(out, (size_t)d_ * 4, y, (size_t)dpad_ * 4, (size_t)d_ * 4, n, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

const float* IVFPQIndex::train_transform(const float* xt, int64_t n_in, Scratch& s) {
  if (!d_opq_) return xt;
  if (opq_trained_) return transform_dev(xt, n_in, s);
  cudaStream_t st = s.stream();
  const int d = d_, Mo = mp_.opq_nsubvector, dso = d / Mo, dsp = (int)round_up(dso, 4);
  const int64_t n = std::min<int64_t>(n_in, 256 * 256);  // max_train_points
  const float* xs;
  if (subsample_rows(xt, n_in, n, dpad_, &xs, s)) return nullptr;
  const int64_t ldn = round_up(n, 4);
  float* xc = s.alloc_n<float>((size_t)n * dpad_);      // centred training set
  float* xproj = s.alloc_n<float>((size_t)n * dpad_);
  float* recon = s.alloc_n<float>((size_t)n * dpad_);
  float* xT = s.alloc_n<float>((size_t)d * ldn);
  float* rT = s.alloc_n<float>((size_t)d * ldn);
  float* xxr = s.alloc_n<float>((size_t)d * dpad_);
  float* slice = s.alloc_n<float>((size_t)n * dsp);
  float* cent = s.alloc_n<float>((size_t)Mo * 256 * dsp);  // per-subspace centroids, kept across rounds
  float* pqc = s.alloc_n<float>((size_t)Mo * 256 * dso);
  uint8_t* codes = s.alloc_n<uint8_t>((size_t)n * Mo);
  if (!xc || !xproj || !recon || !xT || !rT || !xxr || !slice || !cent || !pqc || !codes) return nullptr;
  auto ck = [](cudaError_t e) { return e == cudaSuccess; };
  if (!ck(launch_center_rows(xs, dpad_, n, d, xc, dpad_, st)) || !ck(cudaMemsetAsync(xT, 0, (size_t)d * ldn * 4, st)) ||
      !ck(cudaMemsetAsync(rT, 0, (size_t)d * ldn * 4, st)) || !ck(cudaMemsetAsync(recon, 0, (size_t)n * dpad_ * 4, st)) ||
      !ck(launch_transpose(xc, dpad_, n, d, xT, ldn, st)))
    return nullptr;
  // random orthonormal start: Gaussian matrix (mt19937, seed 1234), Gram-Schmidt on the rows
  std::vector<double> R((size_t)d * d);
  {
    std::mt19937 rng(1234);
    std::normal_distribution<double> nd(0.0, 1.0);
    for (auto& v : R) v = nd(rng);
    for (int i = 0; i < d; i++) {
      for (int p = 0; p < i; p++) {
        double dot = 0;
        for (int j = 0; j < d; j++) dot += R[(size_t)i * d + j] * R[(size_t)p * d + j];
        for (int j = 0; j < d; j++) R[(size_t)i * d + j] -= dot * R[(size_t)p * d + j];
      }
      double nrm = 0;
      for (int j = 0; j < d; j++) nrm += R[(size_t)i * d + j] * R[(size_t)i * d + j];
      nrm = sqrt(nrm);
      for (int j = 0; j < d; j++) R[(size_t)i * d + j] /= nrm;
    }
  }
  std::vector<float> Rf((size_t)d * d), hx((size_t)d * dpad_);
  std::vector<double> a, U, V;
  const int niter = 50, niter_pq_0 = 40, niter_pq = 4;
  for (int it = 0; it < niter; it++) {
    for (size_t i = 0; i < R.size(); i++) Rf[i] = (float)R[i];
    if (!ck(upload_rows_padded(d_opq_, Rf.data(), d, d, dpad_, st)) || !ck(cudaMemsetAsync(xproj, 0, (size_t)n * dpad_ * 4, st)) ||
        !ck(launch_dist_matrix(xc, dpad_, (int)n, d_opq_, dpad_, d, dpad_, kMetricIP, xproj, dpad_, st)))
      return nullptr;
    KMeansParams kp;
    kp.niter = it == 0 ? niter_pq_0 : niter_pq;
    kp.max_points_per_centroid = 1000;
    kp.hot_start = it > 0;
    for (int m = 0; m < Mo; m++) {
      if (!ck(launch_slice_cols(xproj, dpad_, n, m * dso, dso, slice, dsp, st))) return nullptr;
      if (kmeans_device(slice, dsp, n, dso, 256, kp, cent + (size_t)m * 256 * dsp, dsp, st, nullptr)) return nullptr;
      if (!ck(cudaMemcpy2DAsync(pqc + (size_t)m * 256 * dso, (size_t)dso * 4, cent + (size_t)m * 256 * dsp, (size_t)dsp * 4,
                                (size_t)dso * 4, 256, cudaMemcpyDeviceToDevice, st)))
        return nullptr;
    }
    if (!ck(launch_pq_encode(xproj, dpad_, n, nullptr, 0, nullptr, pqc, Mo, dso, codes, st)) ||
        !ck(launch_pq_decode(codes, n, pqc, Mo, dso, recon, dpad_, st)) || !ck(launch_transpose(recon, dpad_, n, d, rT, ldn, st)) ||
        !ck(launch_dist_matrix(xT, ldn, d, rT, ldn, d, (int)ldn, kMetricIP, xxr, dpad_, st)) ||
        !ck(cudaMemcpyAsync(hx.data(), xxr, (size_t)d * dpad_ * 4, cudaMemcpyDeviceToHost, st)) || !ck(cudaStreamSynchronize(st)))
      return nullptr;
    a.assign((size_t)d * d, 0.0);  // X^T Y, d x d
    for (int i = 0; i < d; i++)
      for (int j = 0; j < d; j++) a[(size_t)i * d + j] = hx[(size_t)i * dpad_ + j];
    jacobi_svd(a, d, d, &U, &V);
    // R^T = U V^T  =>  R[i][j] = sum_k V[i][k] U[j][k]
    for (int i = 0; i < d; i++)
      for (int j = 0; j < d; j++) {
        double acc = 0;
        for (int kk = 0; kk < d; kk++) acc += V[(size_t)i * d + kk] * U[(size_t)j * d + kk];
        R[(size_t)i * d + j] = acc;
      }
  }
  for (size_t i = 0; i < R.size(); i++) Rf[i] = (float)R[i];
  if (!ck(upload_rows_padded(d_opq_, Rf.data(), d, d, dpad_, st)) || !ck(cudaStreamSynchronize(st)))
    return nullptr;
  opq_trained_ = true;
  return transform_dev(xt, n_in, s);
}

IVFPQIndex::~IVFPQIndex() {
  if (d_opq_) mem::dev_free(d_opq_);
  mem::dev_free(d_table_);
  mem::dev_free(d_cb8_);
  mem::dev_free(d_cbnrm_);
  if (pqn_.base) mem::dev_free(pqn_.base);
  if (pqn_.d_off) mem::dev_free(pqn_.d_off);
}
// gamma_index_ivfpq.cc:139-144; GPU_IVFPQ: ncentroids * max_points_per_centroid (gamma_index_ivfpq_gpu.cc:208-212)
int64_t IVFPQIndex::default_training_threshold() const {
  if (gpu_contract_) return (int64_t)nlist_ * 256;
  return std::max<int64_t>((int64_t)nlist_ * 200, 256);
}
KMeansParams IVFPQIndex::coarse_kmeans_params() const {
  KMeansParams kp;
  kp.niter = 10;                            // gamma_index_ivfpq.cc:188
  kp.spherical = mp_.metric == kMetricIP;  // gamma_index_ivfpq.cc:189-191
  return kp;
}
int64_t IVFPQIndex::index_mem_bytes() const {
  return IvfPqBase::index_mem_bytes() + (d_table_ ? (int64_t)nlist_ * M_ * ksub_ * 4 : 0);
}
int IVFPQIndex::codebook_changed(cudaStream_t st) {
  pq_gen_++;  // the per-entry norm cache belongs to the previous codebook
  // tables of the tensor-core filter (kernels_pqtc.cu): int8 codebook (one scale sb), centroid norms, and the bounds on
  // |r| and on its quantisation error that its error margin uses
  if (ksub_ == 256 && pqtc_supported(M_, dsub_)) {
    if (!d_cb8_) GB_CUDA(mem::dev_malloc(&d_cb8_, (size_t)M_ * 256 * dsub_));
    if (!d_cbnrm_) GB_CUDA(mem::dev_malloc(&d_cbnrm_, ((size_t)M_ * 256 + 4) * 4));
    GB_CUDA(launch_pqtc_tables(d_pq_, M_, dsub_, d_cb8_, d_cbnrm_, d_cbnrm_ + (size_t)M_ * 256, st));
  }
  if (mp_.metric != kMetricL2) return 0;  // IP: tab = ip table, dis0 = <x, centroid>
  if (!d_table_) GB_CUDA(mem::dev_malloc(&d_table_, (size_t)nlist_ * M_ * ksub_ * 4));
  GB_CUDA(launch_pq_precompute_table(d_centroids_, dpad_, nlist_, d_pq_, M_, dsub_, d_table_, st, ksub_));
  return 0;
}
int IVFPQIndex::get_precomputed_table(float* host) const {
  if (!d_table_) {
    set_last_error("no precomputed table (IP metric or untrained)");
    return -1;
  }
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy(host, d_table_, (size_t)nlist_ * M_ * ksub_ * 4, cudaMemcpyDeviceToHost));
  return 0;
}

// faiss IndexIVFPQ::train_residual restated: residuals of (a subsample of <= 256*ksub, max_points_per_centroid * ksub)
// training vectors -> ProductQuantizer::train = M independent ksub-means on the dsub-wide slices.
int IVFPQIndex::train_extra(const float* xtrain, int64_t n, Scratch& s) {
  if (d_ % M_ != 0) {
    set_last_error("dimension not divisible by nsubvector");
    return -1;
  }
  const int64_t npq = std::min<int64_t>(n, (int64_t)256 * ksub_);
  const float* xs;
  if (subsample_rows(xtrain, n, npq, dpad_, &xs, s)) return -1;
  GB_ALLOC(assign, int32_t, npq, s);
  if (assign_dev(xs, dpad_, npq, assign, s)) return -1;
  GB_ALLOC(resid, float, (size_t)npq * dpad_, s);
  GB_CUDA(launch_residual(xs, dpad_, npq, d_, d_centroids_, dpad_, assign, resid, dpad_, s.stream()));
  return train_codebook(resid, npq, s);
}

// GammaIVFPQIndex::Add (gamma_index_ivfpq.cc:455-540): residual -> pq.compute_codes -> AddKeys.  Below 8 bits the
// per-(row, sub-quantiser) encoder writes one byte per code to scratch and one thread per row packs them (threads of
// the encoder would share output bytes).
cudaError_t IVFPQIndex::encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st) {
  if (!lists) return cudaErrorInvalidValue;  // residual codes need each row's list
  if (nbits_ == 8) return launch_pq_encode(x, dpad_, n, d_centroids_, dpad_, lists, d_pq_, M_, dsub_, codes, st);
  Scratch s(st);
  uint8_t* raw = s.alloc_n<uint8_t>((size_t)n * M_);
  if (!raw) return cudaErrorMemoryAllocation;
  const cudaError_t e = launch_pq_encode(x, dpad_, n, d_centroids_, dpad_, lists, d_pq_, M_, dsub_, raw, st, ksub_);
  if (e != cudaSuccess) return e;
  return launch_pq_pack_codes(raw, n, M_, nbits_, codes, st);
}

// Cache of |r_e|^2 per list entry for the tensor-core filter.  Searches hold mu_ shared, appends hold it exclusively and
// drain in-flight searches before the lists change, so whenever the key (list set, content generation, lengths, codebook
// generation) differs
// from the cached one no kernel is reading the cache; the rebuild (one pass over the codes) is serialised by pqn_mu_ and
// synchronised before other streams may use it.
int IVFPQIndex::ensure_pq_norms(cudaStream_t st) {
  std::lock_guard<std::mutex> g(pqn_mu_);
  const std::vector<int>& lens = lists_->lens();
  if (pqn_.base && pqn_.lists_uid == lists_->uid() && pqn_.content_gen == lists_->content_gen() && pqn_.pq_gen == pq_gen_ &&
      pqn_.lens == lens)
    return 0;
  std::vector<int64_t> off((size_t)nlist_ + 1, 0);
  for (int l = 0; l < nlist_; l++) off[l + 1] = off[l] + round_up(lens[l], 32);
  const size_t total = (size_t)off[nlist_] + 128;  // a tile's 16-byte rounded tail may run past the last entry
  if (total > pqn_.cap) {
    if (pqn_.base) {
      cudaDeviceSynchronize();
      mem::dev_free(pqn_.base);
      pqn_.base = nullptr;
    }
    const size_t cap = total + total / 4;
    if (mem::dev_malloc(&pqn_.base, cap * 4) != cudaSuccess) {
      cudaGetLastError();
      pqn_.cap = 0;
      return 1;  // no room: the caller scans with the exact kernel
    }
    pqn_.cap = cap;
  }
  if (!pqn_.d_off) GB_CUDA(mem::dev_malloc(&pqn_.d_off, sizeof(int64_t) * ((size_t)nlist_ + 1)));
  GB_CUDA(cudaMemcpyAsync(pqn_.d_off, off.data(), sizeof(int64_t) * ((size_t)nlist_ + 1), cudaMemcpyHostToDevice, st));
  GB_CUDA(launch_pq_entry_norms(lists_->directory(), nlist_, lists_->max_len(), M_, d_cbnrm_, pqn_.d_off, pqn_.base, st));
  GB_CUDA(cudaStreamSynchronize(st));
  pqn_.lens = lens;
  pqn_.lists_uid = lists_->uid();
  pqn_.content_gen = lists_->content_gen();
  pqn_.pq_gen = pq_gen_;
  return 0;
}

// List-major IVF-PQ scan (kernels_pqtc.cu): exact scan of the first pa probes -> per-query bound ->
// tensor-core filter over the remaining probes -> exact re-score of the candidates.  Returns 1 when
// the batch / shape does not qualify (caller builds ip and runs the exact kernel over all probes), before any work.
// Otherwise it builds the query's inner-product table ip itself.
//
// Only the filter's thresholds need phase A's bounds: the pair grouping and the operand staging read the plan alone, so
// they run on a side stream while this stream builds ip and runs phase A, and pq_bind_bounds sets the thresholds after
// the join.
int IVFPQIndex::scan_listmajor_pq(const FilterArgs& f, int metric, int nq, const float* xq, int kk, float* ip,
                                  const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                                  unsigned long long* adc_out, bool need_sorted, Scratch& s) {
  if (ksub_ != 256 || !d_cb8_ || !pqtc_supported(M_, dsub_) || dpad_ != d_) return 1;  // the filter reads 8-bit codes
  if (kk > 2048 || nprobe < 2 || nprobe > 65535 || nq > 65535) return 1;  // (query, probe) travel as 16-bit fields of a candidate record
  const int64_t npairs = (int64_t)nq * nprobe;
  if (npairs < (int64_t)nlist_ * 32) return 1;  // < 32 queries per list on average
  const int nseg = (int)std::min<int64_t>(64, std::max<int64_t>(1, (lists_->max_len() + kLmkSegRows - 1) / kLmkSegRows));
  const int pq_group = 256;  // pairs per group: two 128-row operand tiles that share every decoded entry tile
  const int64_t max_groups = npairs / pq_group + nlist_;
  const int64_t max_items = max_groups * nseg;
  if (max_items > INT32_MAX) return 1;
  if (metric == kMetricL2) {
    const int nr = ensure_pq_norms(s.stream());
    if (nr) return nr;
  }
  cudaStream_t st = s.stream();
  const SideStream* side = thread_side_stream(device_);
  if (!side) {
    set_last_error("cannot create the list-major scan's side stream");
    return -1;
  }
  ListDirectory dir = lists_->directory();
  // phase A, per query: its first probes in full -- the fewest whose lists hold >= 4 k' entries together (so that its
  // k'-th exact score is a tight bound B_q), at most pa_max; phase B filters the other probes.
  const int pa_max = std::min(nprobe - 1, 8);
  const long long pa_target = 4 * (long long)kk;
  const int cap = std::max(2048, std::min(8192, next_pow2(8 * kk)));
  const int nsm = sm_count(device_);
  snprintf(last_scan_info_, sizeof(last_scan_info_),
           "{\"phase_a_max_probes\": %d, \"phase_a_target_entries\": %lld, \"candidate_cap\": %d, \"kprime\": %d}", pa_max,
           pa_target, cap, kk);
  GB_ALLOC(d_probes_a, int32_t, npairs, s);
  GB_ALLOC(d_probes_b, int32_t, npairs, s);
  GB_ALLOC(d_row_limit, int, npairs, s);
  GB_CUDA(launch_pqtc_plan_phase_a(probe_ids, npairs, nprobe, pa_max, pa_target, dir.len, d_probes_a, d_probes_b, d_row_limit,
                                   st));

  const int pgA = nq >= nsm * 4 ? std::min(pa_max, 32) : 1;  // one CTA per query when there are queries enough
  const int ngA = (pa_max + pgA - 1) / pgA;
  GB_ALLOC(partA, unsigned long long, (size_t)nq * ngA * kk, s);
  unsigned long long* keysA = partA;
  if (ngA > 1) {
    keysA = s.alloc_n<unsigned long long>((size_t)nq * kk);
    if (!keysA) return -1;
  }
  // phase B's scratch: everything the side stream touches is allocated before the fork
  GB_ALLOC(d_cand_cnt, int, nq, s);
  const size_t tile_bytes = (size_t)(d_ / 16) * 2048;
  const size_t a_bytes = (size_t)max_groups * 2 * tile_bytes;
  const size_t meta_bytes = (size_t)max_groups * pq_group * pqtc_pair_meta_bytes();
  const size_t cand_bytes = (size_t)nq * cap * 8;
  BigScope big(this, a_bytes + meta_bytes + cand_bytes, st);
  if (!big.p) return -1;
  unsigned char* a_scratch = static_cast<unsigned char*>(big.p);
  void* meta = a_scratch + a_bytes;
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(a_scratch + a_bytes + meta_bytes);
  LmGrouping g;
  if (alloc_pair_grouping(npairs, max_items, &g, s)) return -1;

  // ---- phase B's set-up on the side stream: group the remaining pairs by list, stage the operand tiles ----
  ForkJoin fj(st, *side);  // declared after the scratch: joined on every exit before any of it is freed
  GB_CUDA(fj.fork());
  stage_begin("pq_group_and_stage_pairs", fj.side());
  GB_CUDA(cudaMemsetAsync(d_cand_cnt, 0, sizeof(int) * nq, fj.side()));
  GB_CUDA(group_pairs_by_list(d_probes_b, npairs, nseg, pq_group, g, fj.side()));
  GB_CUDA(launch_pq_stage_pairs(xq, dpad_, d_, d_centroids_, dpad_, g.items, (int)max_items, g.totals, g.pair_j, nprobe,
                                coarse_dis, d_cbnrm_ + (size_t)M_ * 256, f, metric, a_scratch, meta, max_groups,
                                d_cand_cnt, cap, d_row_limit, fj.side()));
  stage_end(fj.side());

  // ---- meanwhile, phase A: exact keys of each query's leading probes ----
  {
    StageScope stage(this, "pq_ip_table", st);
    GB_CUDA(launch_pq_ip_table(xq, dpad_, nq, d_pq_, M_, dsub_, ip, st, ksub_));
  }
  stage_begin("pq_phaseA_exact_scan", st);
  // one group per query: its k' best come back unordered with the largest (the bound) in slot k' - 1 -- nobody needs
  // them sorted (launch_select_keys below, used when the probes were split over groups, sorts anyway)
  GB_CUDA(launch_ivfpq_scan(ip, nq, d_probes_a, coarse_dis, pa_max, pgA, dir, M_, d_table_, kk, metric, f, partA, st, nprobe,
                            nullptr, 0, d_row_limit, /*sorted_out=*/ngA > 1));
  if (ngA > 1) GB_CUDA(launch_select_keys(partA, (int64_t)ngA * kk, nq, ngA * kk, kk, keysA, kk, st));
  stage_end(st);

  // ---- phase B: the pairs' thresholds from the bounds, filter ----
  GB_CUDA(fj.join());
  {
    StageScope stage(this, "pq_bind_bounds", st);
    GB_CUDA(launch_pq_bind_bounds(g.totals, max_groups, nprobe, coarse_dis, keysA, kk, kk, f, metric, meta, d_cand_cnt,
                                  cap, st));
  }
  scan_timer_begin(st);  // the dominant kernel: the roofline in bench.py is this launch alone
  stage_begin("pqtc_scan_kernel", st);
  GB_CUDA(launch_pqtc_scan(a_scratch, meta, d_cb8_, pqn_.base, pqn_.d_off, g.items, (int)max_items, g.totals, dir, M_, dsub_, f,
                           metric, d_cand_cnt, cand, cap, nsm, st));
  stage_end(st);
  scan_timer_end(st);
  stage_begin("pq_rescore_and_fallback", st);

  // ---- phase C: candidates -> reference arithmetic, merged with phase A's keys ----
  GB_CUDA(launch_pq_rescore(ip, nq, probe_ids, coarse_dis, nprobe, dir, M_, d_table_, d_cand_cnt, cand, cap, keysA, kk, kk,
                            metric, d_row_limit, f, need_sorted, adc_out, st));
  // queries whose candidate list overflowed (or that had no bound): exact kernel over all probes, flag-gated
  const int ngF = (nprobe + 31) / 32;
  GB_ALLOC(partF, unsigned long long, (size_t)nq * ngF * kk, s);
  GB_CUDA(launch_ivfpq_scan(ip, nq, probe_ids, coarse_dis, nprobe, 32, dir, M_, d_table_, kk, metric, f, partF, st, nprobe,
                            d_cand_cnt, cap));
  GB_CUDA(launch_pq_fallback_merge(d_cand_cnt, cap, nq, partF, ngF, kk, adc_out, st));
  stage_end(st);
  return 0;
}

// Metric check, ADC depth, query-major list scan + merge of its CTA groups, exact re-rank
int IvfIndex::scan_query_major_dev(const char* kernel, const SearchContext& ctx, const FilterArgs& f, int metric, int nq,
                                   const float* rerank_xq, int k, int nprobe, int max_kk, const std::string& limit_at,
                                   unsigned long long* out_keys, Scratch& s,
                                   const std::function<int(int, unsigned long long*, bool)>& prepare,
                                   const std::function<cudaError_t(int, int, unsigned long long*)>& launch) {
  cudaStream_t st = s.stream();
  if (metric != mp_.metric) {
    set_last_error(type_ + ": per-request metric must equal the trained metric");
    return -1;
  }
  // recall_num / re-rank semantics: gamma_index_ivfpq.cc:764-770.  The GPU types never re-rank ("IVFPQ doesn't support
  // rerank", gamma_index_ivfpq_gpu.cc:565): recall_num is checked at the search entry and changes nothing else.
  const bool rerank = ctx.params.recall_num > 0 && !gpu_contract_;
  const int kk = rerank ? std::max(k, ctx.params.recall_num) : k;
  if (kk > max_kk) {
    set_last_error(type_ + ": recall_num / topn [" + std::to_string(kk) + "] above " + std::to_string(max_kk) +
                   " is not supported by this engine at " + limit_at);
    return -1;
  }
  unsigned long long* keys = out_keys;
  if (rerank) {
    keys = s.alloc_n<unsigned long long>((size_t)nq * kk);
    if (!keys) return -1;
  }
  // the exact re-rank takes its candidates in any order; without it the keys are the result and must be sorted
  const int rc = prepare(kk, keys, !rerank);
  if (rc < 0) return -1;
  if (rc == 1) {
    const int nsm = sm_count(device_);
    const int pg = (int)std::min<int64_t>(32, std::max<int64_t>(1, (int64_t)nprobe * nq / ((int64_t)nsm * 32)));
    const int ngroups = (nprobe + pg - 1) / pg;
    GB_ALLOC(partial, unsigned long long, (size_t)nq * ngroups * kk, s);
    last_scan_kernel_ = kernel;
    snprintf(last_scan_info_, sizeof(last_scan_info_), "{\"probes_per_cta\": %d}", pg);
    scan_timer_begin(st);
    stage_begin(kernel, st);
    GB_CUDA(launch(kk, pg, partial));
    stage_end(st);
    scan_timer_end(st);
    if (ngroups > 1) {
      GB_CUDA(launch_select_keys(partial, (int64_t)ngroups * kk, nq, ngroups * kk, kk, keys, kk, st));
    } else {
      GB_CUDA(cudaMemcpyAsync(keys, partial, (size_t)nq * kk * 8, cudaMemcpyDeviceToDevice, st));
    }
  }
  if (rerank && store_->has_shadow()) {
    int* surv = rr_stats_ ? s.alloc_n<int>((size_t)nq) : nullptr;
    {
      StageScope stage(this, "rerank_kernel", st);
      GB_CUDA(launch_rerank_prefilter(keys, kk, nq, rerank_xq, dpad_, dpad_, store_->d_segs(), store_->seg_shift(), dpad_,
                                      store_->shadow_segs(), store_->shadow_stride(), k, metric, f, out_keys, surv, st));
    }
    if (surv) {
      std::vector<int> h(nq);
      GB_CUDA(cudaMemcpyAsync(h.data(), surv, (size_t)nq * sizeof(int), cudaMemcpyDeviceToHost, st));
      GB_CUDA(cudaStreamSynchronize(st));
      std::lock_guard<std::mutex> g(ev_mu_);
      rr_survivors_.insert(rr_survivors_.end(), h.begin(), h.end());
    }
  } else if (rerank) {
    StageScope stage(this, "rerank_kernel", st);
    // host placement: the candidate rows come over PCIe straight from the mapped segments
    GB_CUDA(launch_rerank(keys, kk, nq, rerank_xq, dpad_, dpad_, store_->d_segs(), store_->seg_shift(), dpad_,
                          store_->on_host(), k, metric, f, out_keys, st));
  }
  return 0;
}

// GammaIVFPQIndex::search_preassigned (gamma_index_ivfpq.cc:730-947)
int IVFPQIndex::scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xqv,
                         const void* xq_raw, int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                         unsigned long long* out_keys, Scratch& s) {
  cudaStream_t st = s.stream();
  const float* xq = static_cast<const float*>(xqv);
  float* ip = nullptr;
  auto prepare = [&](int kk, unsigned long long* keys, bool need_sorted) {
    ip = s.alloc_n<float>((size_t)nq * M_ * ksub_);
    if (!ip) return -1;
    // the list-major scan builds ip itself, beside its pair grouping; it declines (1) before that
    const int lm = scan_listmajor_pq(f, metric, nq, xq, kk, ip, probe_ids, coarse_dis, nprobe, keys, need_sorted, s);
    if (lm == 0) last_scan_kernel_ = "pqtc_scan_kernel";
    if (lm == 1) {
      StageScope stage(this, "pq_ip_table", st);
      GB_CUDA(launch_pq_ip_table(xq, dpad_, nq, d_pq_, M_, dsub_, ip, st, ksub_));
    }
    return lm;
  };
  auto launch = [&](int kk, int pg, unsigned long long* partial) {
    if (nbits_ < 8)
      return launch_ivfpq_packed_scan(ip, nq, probe_ids, coarse_dis, nprobe, pg, lists_->directory(), M_, nbits_, d_table_,
                                      kk, metric, f, partial, st);
    return launch_ivfpq_scan(ip, nq, probe_ids, coarse_dis, nprobe, pg, lists_->directory(), M_, d_table_, kk, metric, f,
                             partial, st);
  };
  // "for opq, rerank need raw vector" (gamma_index_ivfpq.cc:735): original queries against the raw store
  return scan_query_major_dev(nbits_ < 8 ? "ivfpq_packed_scan_kernel" : "ivfpq_scan_kernel", ctx, f, metric, nq,
                              static_cast<const float*>(xq_raw), k, nprobe, ivfpq_scan_max_k(M_, nbits_),
                              "nsubvector " + std::to_string(M_), out_keys, s, prepare, launch);
}

// ------------------------------------------------------------------------------------------
// gamma_index_ivfpqfs.cc:95-104: IndexFlatL2 quantiser, spherical for IP, niter kept
KMeansParams IVFPQFastScanIndex::coarse_kmeans_params() const {
  KMeansParams kp;
  kp.spherical = mp_.metric == kMetricIP;
  kp.l2_assign = true;
  return kp;
}

// faiss ProductQuantizer::train with ksub = 16 on the raw training vectors (by_residual = false): the same
// sub-sampling rule as the 256-centroid IVFPQ codebook (at most 256 * ksub points), then M independent 16-means.
int IVFPQFastScanIndex::train_extra(const float* xtrain, int64_t n, Scratch& s) {
  const int64_t npq = std::min<int64_t>(n, 256 * kKsub);
  const float* xs;
  if (subsample_rows(xtrain, n, npq, dpad_, &xs, s)) return -1;
  return train_codebook(xs, npq, s);
}

cudaError_t IVFPQFastScanIndex::encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st) {
  (void)lists;  // codes of the raw vectors
  return launch_pqfs_encode(x, dpad_, n, d_pq_, M_, dsub_, codes, st);
}

int IVFPQFastScanIndex::lut_host(int nq, const float* x, int metric, uint8_t* lut8_out, float* ab_out) {
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  Scratch s(st);
  GB_ALLOC(dx, float, (size_t)nq * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, nq, d_, dpad_, st));
  GB_ALLOC(lut, uint8_t, (size_t)nq * M_ * kKsub, s);
  GB_ALLOC(ab, float, (size_t)nq * 2, s);
  GB_CUDA(launch_pqfs_lut(dx, dpad_, nq, d_pq_, M_, dsub_, metric >= 0 ? metric : mp_.metric, lut, ab, st));
  GB_CUDA(cudaMemcpyAsync(lut8_out, lut, (size_t)nq * M_ * kKsub, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaMemcpyAsync(ab_out, ab, (size_t)nq * 8, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// IndexIVFFastScan::search_preassigned restated over this engine's lists, filters applied before selection;
// recall_num > 0 re-ranks the recall_num best exactly from the raw vectors, as IVFPQ does
int IVFPQFastScanIndex::scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xqv,
                                 const void* xq_raw, int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                                 unsigned long long* out_keys, Scratch& s) {
  (void)coarse_dis;  // no residual: the list's coarse distance takes no part in the score
  cudaStream_t st = s.stream();
  const float* xq = static_cast<const float*>(xqv);
  uint8_t* lut = nullptr;
  float* ab = nullptr;
  auto prepare = [&](int, unsigned long long*, bool) {
    lut = s.alloc_n<uint8_t>((size_t)nq * M_ * kKsub);
    ab = s.alloc_n<float>((size_t)nq * 2);
    if (!lut || !ab) return -1;
    StageScope stage(this, "pqfs_lut_kernel", st);
    GB_CUDA(launch_pqfs_lut(xq, dpad_, nq, d_pq_, M_, dsub_, metric, lut, ab, st));
    return 1;
  };
  auto launch = [&](int kk, int pg, unsigned long long* partial) {
    return launch_ivfpqfs_scan(lut, ab, nq, probe_ids, nprobe, pg, lists_->directory(), M_, kk, metric, f, partial, st);
  };
  return scan_query_major_dev("ivfpqfs_scan_kernel", ctx, f, metric, nq, static_cast<const float*>(xq_raw), k, nprobe, 4096,
                              "nsubvector " + std::to_string(M_), out_keys, s, prepare, launch);
}

// ------------------------------------------------------------------------------------------
// GammaIndexBinaryIVF (gamma_index_binary_ivf.cc) over faiss::IndexBinaryIVF
BinaryIvfIndex::BinaryIvfIndex(int d_bits, const ModelParams& mp, int device, int seg_shift)
    : IvfIndex("BINARYIVF", d_bits, mp, device, seg_shift, d_bits / 8), cb_(d_bits / 8) {
  ldw_ = store_->stride() / 4;
  mp_.metric = kMetricL2;  // Hamming distances rank like L2: smaller first
  mem::dev_malloc(&d_bcent_, (size_t)nlist_ * ldw_ * 4);
  cudaMemset(d_bcent_, 0, (size_t)nlist_ * ldw_ * 4);
}
BinaryIvfIndex::~BinaryIvfIndex() { mem::dev_free(d_bcent_); }
int64_t BinaryIvfIndex::index_mem_bytes() const { return IvfIndex::index_mem_bytes() + (int64_t)nlist_ * ldw_ * 4; }

// GammaIndexBinaryIVF::Indexing (gamma_index_binary_ivf.cc:212-270) -> faiss IndexBinaryIVF::train, through
// IvfIndex::train: the first num rows expanded to +-1 floats, faiss Clustering (niter 10, Init) with an IndexFlatL2,
// centroids packed by sign
KMeansParams BinaryIvfIndex::coarse_kmeans_params() const {
  KMeansParams kp;
  kp.niter = 10;  // gamma_index_binary_ivf.cc:97
  return kp;
}
// xt: the packed training rows as RawStore::contiguous leaves them; the result is one fp32 slab of n x dpad floats
const float* BinaryIvfIndex::train_transform(const float* xt, int64_t n, Scratch& s) {
  float* xf = s.alloc_n<float>((size_t)n * dpad_);
  if (!xf) return nullptr;
  const cudaError_t e = launch_binary_to_real(reinterpret_cast<const uint8_t*>(xt), ldw_ * 4, n, d_, xf, dpad_, s.stream());
  if (e != cudaSuccess) {
    set_last_error(std::string("BINARYIVF: binary_to_real: ") + cudaGetErrorString(e));
    return nullptr;
  }
  return xf;
}
int BinaryIvfIndex::centroids_changed(cudaStream_t st) {
  GB_CUDA(launch_real_to_binary(d_centroids_, dpad_, nlist_, d_, d_bcent_, ldw_ * 4, st));
  return 0;
}

int BinaryIvfIndex::set_binary_centroids(const uint8_t* host, int nlist) {
  if (nlist != nlist_) {
    set_last_error("set_centroids: nlist mismatch");
    return -1;
  }
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  GB_CUDA(cudaMemset(d_bcent_, 0, (size_t)nlist_ * ldw_ * 4));
  GB_CUDA(cudaMemcpy2D(d_bcent_, (size_t)ldw_ * 4, host, cb_, cb_, nlist_, cudaMemcpyHostToDevice));
  if (!lists_) lists_.reset(new IvfLists(nlist_, code_bytes()));
  trained_ = true;
  return 0;
}
int BinaryIvfIndex::get_binary_centroids(uint8_t* host) const {
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy2D(host, cb_, d_bcent_, (size_t)ldw_ * 4, cb_, nlist_, cudaMemcpyDeviceToHost));
  return 0;
}

int BinaryIvfIndex::hamming_topk(const uint32_t* xq, int nq, int k, unsigned long long* keys, Scratch& s) {
  cudaStream_t st = s.stream();
  const int64_t ldo = round_up(nlist_, 4);
  const int QB = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)nq, ((int64_t)1 << 28) / ldo, 65536}));
  GB_ALLOC(scores, float, (size_t)QB * ldo, s);
  const FilterArgs none{nullptr, nullptr, -FLT_MAX, FLT_MAX};
  for (int q0 = 0; q0 < nq; q0 += QB) {
    const int qb = std::min(QB, nq - q0);
    GB_CUDA(launch_hamming_tile(xq + (int64_t)q0 * ldw_, ldw_, qb, reinterpret_cast<const uint32_t*>(d_bcent_), ldw_, nlist_,
                                (cb_ + 3) / 4, scores, ldo, st));
    GB_CUDA(launch_select_scores(scores, ldo, qb, nlist_, 0, k, kMetricL2, none, keys + (int64_t)q0 * k, k, st));
  }
  return 0;
}

// IndexBinaryFlat::assign: the Hamming-nearest centroid, the smaller list id among equals
int BinaryIvfIndex::assign_batch(const void* x, int64_t n, const void** xc, int32_t* out, Scratch& s) {
  *xc = x;
  GB_ALLOC(best, unsigned long long, n, s);
  if (hamming_topk(static_cast<const uint32_t*>(x), (int)n, 1, best, s)) return -1;
  GB_CUDA(launch_split_keys(best, n, kMetricL2, nullptr, out, s.stream()));
  return 0;
}

// the list entry is the row's d / 8 bytes as they are (IndexBinaryIVF::add_core)
int BinaryIvfIndex::append_batch(const void* x, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                                 const std::vector<int>& add, Scratch& s) {
  (void)add;
  cudaStream_t st = s.stream();
  GB_ALLOC(codes, uint8_t, (size_t)n * cb_, s);
  GB_CUDA(cudaMemcpy2DAsync(codes, cb_, x, (size_t)ldw_ * 4, cb_, n, cudaMemcpyDeviceToDevice, st));
  GB_CUDA(launch_ivf_append_codes(codes, n, cb_, d_list, d_pos, reinterpret_cast<uint8_t* const*>(lists_->d_data()),
                                  lists_->d_ids(), vid0, st));
  return 0;
}

// launch_hamming_tile, in launches of at most kHammingTileMaxQueries queries
cudaError_t BinaryIvfIndex::flat_tile(const void* xq, int nq, const void* rows, int m, int metric, float* scores, int64_t ldo,
                                      cudaStream_t st) {
  (void)metric;
  last_scan_kernel_ = "hamming_tile_kernel+select_rows_kernel";
  for (int q0 = 0; q0 < nq; q0 += kHammingTileMaxQueries) {
    const cudaError_t e = launch_hamming_tile(static_cast<const uint32_t*>(xq) + q0 * ldw_, ldw_,
                                              std::min(kHammingTileMaxQueries, nq - q0), static_cast<const uint32_t*>(rows),
                                              ldw_, m, (cb_ + 3) / 4, scores + q0 * ldo, ldo, st);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// quantizer->search: the nprobe Hamming-nearest centroids, the smaller list id among equals
int BinaryIvfIndex::coarse_dev(int nq, const void* xq, int nprobe, int metric, int32_t* probe_ids, float* coarse_dis,
                               Scratch& s) {
  (void)metric;
  GB_ALLOC(keys, unsigned long long, (size_t)nq * nprobe, s);
  if (hamming_topk(static_cast<const uint32_t*>(xq), nq, nprobe, keys, s)) return -1;
  GB_CUDA(launch_split_keys(keys, (int64_t)nq * nprobe, kMetricL2, coarse_dis, probe_ids, s.stream()));
  return 0;
}

// search_knn_hamming_heap over the probed lists: the shared query-major list scan with the Hamming codec, then the merge
// of its CTA groups
int BinaryIvfIndex::scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xq,
                             const void* xq_raw, int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe,
                             unsigned long long* out_keys, Scratch& s) {
  (void)ctx;
  (void)metric;
  (void)xq_raw;  // no transform
  (void)coarse_dis;  // the list's coarse distance takes no part in the score
  cudaStream_t st = s.stream();
  const int max_k = binary_scan_max_k(cb_);
  if (k > max_k) {
    set_last_error(type_ + ": topK [" + std::to_string(k) + "] above " + std::to_string(max_k) +
                   " is not supported by this engine at " + std::to_string(d_) + " bits");
    return -1;
  }
  const int nsm = sm_count(device_);
  const int pg = (int)std::min<int64_t>(32, std::max<int64_t>(1, (int64_t)nprobe * nq / ((int64_t)nsm * 32)));
  const int ngroups = (nprobe + pg - 1) / pg;
  GB_ALLOC(partial, unsigned long long, (size_t)nq * ngroups * k, s);
  last_scan_kernel_ = "binary_ivf_scan_kernel";
  snprintf(last_scan_info_, sizeof(last_scan_info_), "{\"probes_per_cta\": %d}", pg);
  scan_timer_begin(st);
  GB_CUDA(launch_binary_ivf_scan(static_cast<const uint32_t*>(xq), ldw_, nq, probe_ids, nprobe, pg, lists_->directory(), cb_, k,
                                 f, partial, st));
  scan_timer_end(st);
  if (ngroups > 1) {
    GB_CUDA(launch_select_keys(partial, (int64_t)ngroups * k, nq, ngroups * k, k, out_keys, k, st));
  } else {
    GB_CUDA(cudaMemcpyAsync(out_keys, partial, (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// GammaIVFRABITQIndex (gamma_index_ivfrabitq.cc)
int64_t RaBitQIndex::default_training_threshold() const {  // gamma_index_ivfrabitq.cc:69-76, as IVFPQ
  return std::max<int64_t>((int64_t)nlist_ * 200, 256);
}
// gamma_index_ivfrabitq.cc:80-120: IndexFlat quantiser under the index metric, niter 10, spherical for IP.  faiss's
// RaBitQuantizer::train [faiss-restated, not verifiable here] learns nothing, so the coarse centroids are the whole model.
KMeansParams RaBitQIndex::coarse_kmeans_params() const {
  KMeansParams kp;
  kp.niter = 10;
  kp.spherical = mp_.metric == kMetricIP;
  return kp;
}

// by_residual: each row's code is of its residual to the list it was assigned to
int RaBitQIndex::append_batch(const void* xv, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                              const std::vector<int>& add, Scratch& s) {
  (void)add;
  cudaStream_t st = s.stream();
  const int cb = code_bytes();
  GB_ALLOC(codes, uint8_t, (size_t)n * cb, s);
  GB_CUDA(launch_rabitq_encode(static_cast<const float*>(xv), dpad_, n, d_list, d_centroids_, dpad_, d_, nb_bits_, codes, st));
  GB_CUDA(launch_ivf_append_codes(codes, n, cb, d_list, d_pos, reinterpret_cast<uint8_t* const*>(lists_->d_data()),
                                  lists_->d_ids(), vid0, st));
  return 0;
}

int RaBitQIndex::encode_host(const float* x, int64_t n, const int64_t* assign, uint8_t* codes_out) {
  std::shared_lock<std::shared_mutex> lk(mu_);  // the centroids stay put while the rows are encoded against them
  if (!trained_) {
    set_last_error("IVFRABITQ: encode needs trained centroids");
    return -1;
  }
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  Scratch s(st);
  const int cb = code_bytes();
  GB_ALLOC(dx, float, (size_t)n * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, n, d_, dpad_, st));
  std::vector<int32_t> h(assign, assign + n);
  for (int32_t l : h)
    if (l < 0 || l >= nlist_) {
      set_last_error("IVFRABITQ: list id out of range");
      return -1;
    }
  GB_ALLOC(da, int32_t, n, s);
  GB_CUDA(cudaMemcpyAsync(da, h.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
  GB_ALLOC(codes, uint8_t, (size_t)n * cb, s);
  GB_CUDA(launch_rabitq_encode(dx, dpad_, n, da, d_centroids_, dpad_, d_, nb_bits_, codes, st));
  GB_CUDA(cudaMemcpyAsync(codes_out, codes, (size_t)n * cb, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int RaBitQIndex::estimate_host(int nq, const float* x, const int64_t* lists, int qb, int metric, float* out) {
  std::shared_lock<std::shared_mutex> lk(mu_);
  if (!trained_ || !lists_) {
    set_last_error("IVFRABITQ: estimate needs a trained index");
    return -1;
  }
  if (qb < 0 || qb > 8) {
    set_last_error("IVFRABITQ: qb must be in [0, 8]");
    return -1;
  }
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  Scratch s(st);
  std::vector<int32_t> qo(nq), lo(nq);
  std::vector<int64_t> off(nq);
  int64_t total = 0;
  for (int j = 0; j < nq; j++) {
    if (lists[j] < 0 || lists[j] >= nlist_) {
      set_last_error("IVFRABITQ: list id out of range");
      return -1;
    }
    qo[j] = j;
    lo[j] = (int32_t)lists[j];
    off[j] = total;
    total += lists_->lens()[lists[j]];
  }
  GB_ALLOC(dx, float, (size_t)nq * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, nq, d_, dpad_, st));
  GB_ALLOC(dq, int32_t, nq, s);
  GB_ALLOC(dl, int32_t, nq, s);
  GB_ALLOC(doff, int64_t, nq, s);
  GB_ALLOC(dout, float, total + 1, s);
  GB_CUDA(cudaMemcpyAsync(dq, qo.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(dl, lo.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(doff, off.data(), (size_t)nq * 8, cudaMemcpyHostToDevice, st));
  GB_CUDA(launch_rabitq_estimate(dx, dpad_, d_centroids_, dpad_, d_, nb_bits_, qb, metric, lists_->directory(), dq, dl, doff, nq,
                                 dout, st));
  GB_CUDA(cudaMemcpyAsync(out, dout, (size_t)total * 4, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// IVFRaBitQ search_preassigned over this engine's lists (gamma_index_ivfrabitq.cc:553-633): the estimator scan selects the
// k' = max(k, recall_num) best estimates, filters applied before selection; recall_num > 0 re-ranks them exactly from the
// raw vectors, otherwise the estimates are the scores
int RaBitQIndex::scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xqv, const void* xq_raw,
                          int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
                          Scratch& s) {
  (void)xq_raw;      // no transform
  (void)coarse_dis;  // dis0 is recomputed by the scan in its own fixed order
  const float* xq = static_cast<const float*>(xqv);
  const int qb = (ctx.params.qb >= 0 && ctx.params.qb <= 8) ? ctx.params.qb : qb_;  // gamma_index_ivfrabitq.cc:215-223
  auto prepare = [&](int, unsigned long long*, bool) { return 1; };  // the scan forms its tables per (query, list)
  auto launch = [&](int kk, int pg, unsigned long long* partial) {
    snprintf(last_scan_info_, sizeof(last_scan_info_), "{\"probes_per_cta\": %d, \"qb\": %d}", pg, qb);
    return launch_rabitq_scan(xq, dpad_, nq, d_centroids_, dpad_, d_, nb_bits_, qb, probe_ids, nprobe, pg, lists_->directory(),
                              kk, metric, f, partial, s.stream());
  };
  return scan_query_major_dev("rabitq_scan_kernel", ctx, f, metric, nq, xq, k, nprobe, rabitq_scan_max_k(d_, nb_bits_, qb),
                              "dimension " + std::to_string(d_), out_keys, s, prepare, launch);
}

// ------------------------------------------------------------------------------------------
// GammaVearchIndex (gamma_index_vearch.cc) over ScaNN's asymmetric hashing (GetConfig, :128-259)
VearchIndex::VearchIndex(int d, const ModelParams& mp, int device, int seg_shift)
    : IvfIndex("VEARCH", d, mp, device, seg_shift), nb_(scann_blocks(d, mp.nsubvector)) {
  // GetConfig: a negative threshold is written as nan, and L2 forces nan (no noise shaping)
  if (mp_.ns_threshold < 0 || mp_.metric == kMetricL2) mp_.ns_threshold = std::nan("");
  mem::dev_malloc(&d_cb_, (size_t)16 * d * 4);
  cudaMemset(d_cb_, 0, (size_t)16 * d * 4);
  if (mp_.reordering) store_->enable_shadow();  // only reordering re-ranks
}
VearchIndex::~VearchIndex() { mem::dev_free(d_cb_); }
int64_t VearchIndex::index_mem_bytes() const { return IvfIndex::index_mem_bytes() + (int64_t)16 * d_ * 4; }

// partitioning: 12 iterations, SPHERICAL under IP, the database assigned by SquaredL2Distance
KMeansParams VearchIndex::coarse_kmeans_params() const {
  KMeansParams kp;
  kp.niter = 12;
  kp.spherical = mp_.metric == kMetricIP;
  kp.l2_assign = true;
  return kp;
}

// GammaVearchIndex::Search (:483-487): the request's nprobe when it is in (0, ncentroids), else the index's 512 leaves.
// The request's nprobe defaults to 50 for an empty parameter string (VearchRetrievalParameters(type), the constructor
// Parse takes then) and to 80 otherwise (VearchRetrievalParameters()).  The leaves are clamped to nlist here.
int VearchIndex::resolve_nprobe(const SearchContext& ctx) const {
  const int req = ctx.params.nprobe > 0 ? ctx.params.nprobe : (ctx.params.given ? 80 : 50);
  const int leaves = req < nlist_ ? req : std::min(kDefaultLeaves, nlist_);
  return std::min(leaves, 4096);
}

cudaError_t VearchIndex::encode_dev(const float* x, int64_t n, const int32_t* lists, uint8_t* codes, cudaStream_t st) {
  // residuals under IP (use_residual_quantization), raw rows under L2
  return launch_scann_encode(x, dpad_, n, mp_.metric == kMetricIP ? lists : nullptr, d_centroids_, dpad_, d_, mp_.nsubvector,
                             d_cb_, mp_.ns_threshold, codes, st);
}

// AhImpl::TrainAsymmetricHashing (asymmetric_hashing_impl.cc:150-248): per block a 16-centre k-means (10 iterations) of
// the training sample's residuals (IP) or rows (L2), its centres then ordered by cluster size, largest first (a stable
// order among equal sizes; ScaNN's std::sort leaves it open), rotated by ((b / 2) % max(1, 16 / 16)) * 16 = 0 places,
// and reversed in every odd block b
int VearchIndex::train_extra(const float* xtrain, int64_t n, Scratch& s) {
  cudaStream_t st = s.stream();
  const float* xs = xtrain;
  if (mp_.metric == kMetricIP) {
    GB_ALLOC(assign, int32_t, n, s);
    if (assign_dev(xtrain, dpad_, n, assign, s)) return -1;
    GB_ALLOC(res, float, (size_t)n * dpad_, s);
    GB_CUDA(launch_residual(xtrain, dpad_, n, d_, d_centroids_, dpad_, assign, res, dpad_, st));
    xs = res;
  }
  const int w = d_ / mp_.nsubvector;
  const int wmax = std::max(w, d_ - mp_.nsubvector * w);
  const int dsp = (int)round_up(wmax, 4);
  GB_ALLOC(slice, float, (size_t)n * dsp, s);
  GB_ALLOC(cent, float, (size_t)16 * dsp, s);
  GB_ALLOC(best, unsigned long long, n, s);
  KMeansParams kp;
  kp.niter = 10;
  kp.max_points_per_centroid = 0;  // the whole sample (expected_sample_size = the training threshold)
  std::vector<float> cb((size_t)16 * d_), hc((size_t)16 * dsp);
  std::vector<unsigned long long> hb(n);
  for (int b = 0; b < nb_; b++) {
    const int s0 = b * w, wb = b < mp_.nsubvector ? w : d_ - mp_.nsubvector * w;
    GB_CUDA(launch_slice_cols(xs, dpad_, n, s0, wb, slice, dsp, st));
    GB_CUDA(cudaMemsetAsync(cent, 0, (size_t)16 * dsp * 4, st));
    if (kmeans_device(slice, dsp, n, wb, 16, kp, cent, dsp, st, nullptr)) return -1;
    // cluster sizes: the sample assigned to the final centres (L2, the first minimum)
    GB_CUDA(launch_fill_u64(best, n, kKeySentinel, st));
    GB_CUDA(launch_dist_argmin(slice, dsp, (int)n, cent, dsp, 16, dsp, kMetricL2, best, 0, st));
    GB_CUDA(cudaMemcpyAsync(hb.data(), best, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaMemcpyAsync(hc.data(), cent, hc.size() * 4, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    std::vector<int64_t> size(16, 0);
    for (int64_t i = 0; i < n; i++) size[(uint32_t)hb[i] & 15]++;
    std::vector<int> perm(16);
    for (int c = 0; c < 16; c++) perm[c] = c;
    std::stable_sort(perm.begin(), perm.end(), [&](int a, int c) { return size[a] > size[c]; });
    if (b & 1) std::reverse(perm.begin(), perm.end());
    for (int c = 0; c < 16; c++)
      memcpy(&cb[(size_t)16 * s0 + (size_t)c * wb], &hc[(size_t)perm[c] * dsp], (size_t)wb * 4);
  }
  GB_CUDA(cudaMemcpyAsync(d_cb_, cb.data(), cb.size() * 4, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaStreamSynchronize(st));  // cb leaves scope
  return 0;
}

int VearchIndex::append_batch(const void* xv, int64_t n, int64_t vid0, const int32_t* d_list, const int32_t* d_pos,
                              const std::vector<int>& add, Scratch& s) {
  (void)add;
  cudaStream_t st = s.stream();
  const int cb = code_bytes();
  GB_ALLOC(codes, uint8_t, (size_t)n * cb, s);
  GB_CUDA(encode_dev(static_cast<const float*>(xv), n, d_list, codes, st));
  GB_CUDA(launch_ivf_append_codes(codes, n, cb, d_list, d_pos, reinterpret_cast<uint8_t* const*>(lists_->d_data()),
                                  lists_->d_ids(), vid0, st));
  return 0;
}

int VearchIndex::set_codebook(const float* host) {
  cudaSetDevice(device_);
  std::unique_lock<std::shared_mutex> lk(mu_);
  drain_searches();
  GB_CUDA(cudaMemcpy(d_cb_, host, (size_t)16 * d_ * 4, cudaMemcpyHostToDevice));
  return 0;
}
int VearchIndex::get_codebook(float* host) const {
  std::shared_lock<std::shared_mutex> lk(mu_);  // set_codebook and training write it under the exclusive lock
  cudaSetDevice(device_);
  GB_CUDA(cudaMemcpy(host, d_cb_, (size_t)16 * d_ * 4, cudaMemcpyDeviceToHost));
  return 0;
}

int VearchIndex::encode_host(const float* x, int64_t n, const int64_t* assign, uint8_t* codes_out) {
  std::shared_lock<std::shared_mutex> lk(mu_);  // the centroids stay put while the rows are encoded against them
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  Scratch s(st);
  GB_ALLOC(dx, float, (size_t)n * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, n, d_, dpad_, st));
  GB_ALLOC(da, int32_t, std::max<int64_t>(n, 1), s);
  if (mp_.metric == kMetricIP) {
    std::vector<int32_t> h(n);
    for (int64_t i = 0; i < n; i++) {
      if (!assign || assign[i] < 0 || assign[i] >= nlist_) {
        set_last_error("VEARCH: encode needs each row's list id in [0, nlist) under InnerProduct");
        return -1;
      }
      h[i] = (int32_t)assign[i];
    }
    GB_CUDA(cudaMemcpyAsync(da, h.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    GB_CUDA(cudaStreamSynchronize(st));  // h leaves scope
  }
  GB_ALLOC(codes, uint8_t, (size_t)n * code_bytes(), s);
  GB_CUDA(encode_dev(dx, n, da, codes, st));
  GB_CUDA(cudaMemcpyAsync(codes_out, codes, (size_t)n * code_bytes(), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int VearchIndex::lut_host(int nq, const float* x, uint8_t* lut_out, float* mult_out) {
  std::shared_lock<std::shared_mutex> lk(mu_);  // the codebook stays put while the tables are built from it
  cudaSetDevice(device_);
  cudaStream_t st = thread_stream(device_);
  Scratch s(st);
  GB_ALLOC(dx, float, (size_t)nq * dpad_, s);
  GB_CUDA(upload_rows_padded(dx, x, nq, d_, dpad_, st));
  GB_ALLOC(lut, uint8_t, (size_t)nq * nb_ * 16, s);
  GB_ALLOC(mult, float, nq, s);
  GB_CUDA(launch_scann_lut(dx, dpad_, nq, d_, mp_.nsubvector, d_cb_, mp_.metric, lut, mult, st));
  GB_CUDA(cudaMemcpyAsync(lut_out, lut, (size_t)nq * nb_ * 16, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaMemcpyAsync(mult_out, mult, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// ScannSearch over this engine's lists: the table sum (plus <q, c_l> under IP) ranks the entries, filters, tombstones
// and the score window apply before selection, and with reordering the k' = max(k, recall_num) best are re-ranked
// exactly from the raw vectors.  recall_num defaults to 100 (both VearchRetrievalParameters constructors).
int VearchIndex::scan_dev(const SearchContext& ctx, const FilterArgs& f, int metric, int nq, const void* xqv, const void* xq_raw,
                          int k, const int32_t* probe_ids, const float* coarse_dis, int nprobe, unsigned long long* out_keys,
                          Scratch& s) {
  (void)xq_raw;  // no transform
  cudaStream_t st = s.stream();
  const float* xq = static_cast<const float*>(xqv);
  SearchContext c = ctx;
  c.params.recall_num = mp_.reordering ? (ctx.params.recall_num > 0 ? ctx.params.recall_num : 100) : 0;
  uint8_t* lut = nullptr;
  float* mult = nullptr;
  const float* leaf = coarse_dis;  // read only under IP, where it is replaced by the fixed-order <q, c_l>
  auto prepare = [&](int, unsigned long long*, bool) {
    lut = s.alloc_n<uint8_t>((size_t)nq * nb_ * 16);
    mult = s.alloc_n<float>(nq);
    if (!lut || !mult) return -1;
    StageScope stage(this, "scann_lut_kernel", st);
    GB_CUDA(launch_scann_lut(xq, dpad_, nq, d_, mp_.nsubvector, d_cb_, metric, lut, mult, st));
    if (metric == kMetricIP) {
      float* lf = s.alloc_n<float>((size_t)nq * nprobe);
      if (!lf) return -1;
      GB_CUDA(launch_scann_leaf(xq, dpad_, nq, probe_ids, nprobe, d_centroids_, dpad_, nlist_, d_, lf, st));
      leaf = lf;
    }
    return 1;
  };
  auto launch = [&](int kk, int pg, unsigned long long* partial) {
    return launch_vearch_scan(lut, mult, leaf, nq, probe_ids, nprobe, pg, lists_->directory(), nb_, kk, metric, f, partial, st);
  };
  return scan_query_major_dev("vearch_scan_kernel", c, f, metric, nq, xq, k, nprobe, vearch_scan_max_k(nb_),
                              "nsubvector " + std::to_string(mp_.nsubvector), out_keys, s, prepare, launch);
}

// ------------------------------------------------------------------------------------------
Index* create_index(const std::string& type, int d, const ModelParams& mp, int device, int seg_shift) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
    set_last_error("no CUDA device " + std::to_string(device) + " (this engine has no CPU path)");
    return nullptr;
  }
  if (d <= 0) {
    set_last_error("invalid dimension");
    return nullptr;
  }
  if (type == "FLAT") return new FlatIndex(d, mp, device, seg_shift);
  if (type == "IVFFLAT" || type == "GPU_IVFFLAT") {
    // small batches scan query-major (ivfflat_scan_kernel), whose ring, query and k = 4096 queue must fit one CTA's
    // shared memory; refused here rather than as a CUDA error at every such search
    int max_d = 0;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = ivfflat_scan_max_dim(&max_d);
    if (e != cudaSuccess) {
      set_last_error(type + ": cannot query the list scan kernel: " + cudaGetErrorString(e));
      return nullptr;
    }
    if (round_up(d, 4) > max_d) {
      set_last_error(type + ": dimension [" + std::to_string(d) + "] above " + std::to_string(max_d) +
                     " is not supported by this engine");
      return nullptr;
    }
  }
  if (type == "IVFFLAT") {
    if (mp.ncentroids <= 0 || mp.nprobe > mp.ncentroids) {  // gamma_index_ivfflat.cc:277-286
      set_last_error("nprobe should be less than ncentroids");
      return nullptr;
    }
    return new IVFFlatIndex(type, d, mp, device, seg_shift);
  }
  if (type == "IVFPQ") {
    int M = mp.nsubvector > 0 ? mp.nsubvector : d / 2;
    if (M <= 0 || d % M != 0) {  // gamma_index_ivfpq.cc:125-133
      set_last_error("Dimension [" + std::to_string(d) + "] cannot divide by nsubvector [" + std::to_string(M) + "].");
      return nullptr;
    }
    // gamma_index_ivfpq.cc:182 takes any nbits; 1..8 here (IVFPQIndex::kMaxNbits)
    if (mp.nbits < 1) {
      set_last_error("invalid nbits_per_idx =" + std::to_string(mp.nbits));
      return nullptr;
    }
    if (mp.nbits > IVFPQIndex::kMaxNbits) {
      set_last_error("IVFPQ: nbits_per_idx [" + std::to_string(mp.nbits) + "] above " +
                     std::to_string(IVFPQIndex::kMaxNbits) + " is not supported by this engine");
      return nullptr;
    }
    // the query-major scan holds the [M][2^nbits] fp32 table in one CTA's shared memory: an M it cannot search at all
    // is refused here rather than at the first search (the reference has no such limit)
    if (ivfpq_scan_max_k(M, mp.nbits) < 1) {
      int max_m = M;
      while (max_m > 1 && ivfpq_scan_max_k(max_m, mp.nbits) < 1) max_m--;
      set_last_error("IVFPQ: nsubvector [" + std::to_string(M) + "] above " + std::to_string(max_m) + " at nbits_per_idx " +
                     std::to_string(mp.nbits) + " is not supported by this engine");
      return nullptr;
    }
    if (mp.opq_nsubvector > 0 && d % mp.opq_nsubvector != 0) {  // gamma_index_ivfpq.cc:169-176
      set_last_error(std::to_string(d) + " % " + std::to_string(mp.opq_nsubvector) +
                     " != 0, opq nsubvector should be divisible by dimension.");
      return nullptr;
    }
    if (mp.ncentroids <= 0 || mp.nprobe > mp.ncentroids) {
      set_last_error("nprobe should be less than ncentroids");
      return nullptr;
    }
    return new IVFPQIndex(type, d, mp, device, seg_shift);
  }
  if (type == "GPU_IVFPQ") {  // IVFPQGPUModelParams::Parse / Validate, GammaIVFPQGPUIndex::Init (gamma_index_ivfpq_gpu.cc:62-200)
    std::string err;
    const int M = mp.has_nsubvector ? mp.nsubvector_arg : IVFPQIndex::kGpuDefaultM;
    if (mp.has_ncentroids && mp.ncentroids_arg <= 0)
      err = "invalid ncentroids =" + std::to_string(mp.ncentroids_arg);
    else if (mp.has_nsubvector && mp.nsubvector_arg <= 0)
      err = "invalid nsubvector =" + std::to_string(mp.nsubvector_arg);
    else if (mp.has_nbits && mp.nbits_arg <= 0)
      err = "invalid nbits_per_idx =" + std::to_string(mp.nbits_arg);
    else if (mp.has_nprobe && mp.nprobe_arg <= 0)
      err = "invalid nprobe =" + std::to_string(mp.nprobe_arg);
    else if (mp.has_nprobe && mp.nprobe > mp.ncentroids)
      err = "nprobe should less than ncentroids";
    else if (!mp.metric_unknown.empty())
      err = "invalid metric_type = " + mp.metric_unknown;
    else if (M % 4 != 0)  // Validate() logs these and returns ParamError() without text
      err = "only support multiple of 4 now, nsubvector=" + std::to_string(M);
    else if (mp.nbits != 8)
      err = "only support 8 now, nbits_per_idx=" + std::to_string(mp.nbits);
    else if (d % M != 0)
      err = "Dimension [" + std::to_string(d) + "] cannot divide by nsubvector [" + std::to_string(M) + "].";
    else if (ivfpq_scan_max_k(M, 8) < Index::kGpuMaxK) {
      // the query-major scan must select the type's own ceiling k' = 2048 beside the [M][256] fp32 table
      int max_m = M;
      while (max_m > 4 && ivfpq_scan_max_k(max_m, 8) < Index::kGpuMaxK) max_m -= 4;
      err = "GPU_IVFPQ: nsubvector [" + std::to_string(M) + "] above " + std::to_string(max_m) +
            " is not supported by this engine";
    }
    if (!err.empty()) {
      set_last_error(err);
      return nullptr;
    }
    ModelParams g = mp;
    g.nsubvector = M;
    g.opq_nsubvector = 0;  // the GPU type reads no "opq" object
    g.has_opq = false;
    return new IVFPQIndex(type, d, g, device, seg_shift);
  }
  if (type == "GPU_IVFFLAT") {  // IVFFlatGPUModelParams::Parse / Validate (gamma_index_ivfflat_gpu.h:64-110)
    // ncentroids and nprobe as given (even <= 0); an unknown metric_type was ignored; nprobe > ncentroids is accepted
    ModelParams g = mp;
    if (mp.has_ncentroids) g.ncentroids = mp.ncentroids_arg;
    if (mp.has_nprobe) g.nprobe = mp.nprobe_arg;
    if (g.ncentroids <= 0 || g.nprobe <= 0 || mp.bucket_init_arg <= 0 || mp.bucket_max_arg <= 0 ||
        mp.bucket_init_arg > mp.bucket_max_arg) {
      set_last_error("Invalid parameters");
      return nullptr;
    }
    return new IVFFlatIndex(type, d, g, device, seg_shift);
  }
  if (type == "IVFPQFastScan") {  // IVFPQFastScanModelParams::Validate (gamma_index_ivfpqfs.h:231-245)
    if (mp.nsubvector <= 0 || d % mp.nsubvector != 0) {
      set_last_error("Dimension [" + std::to_string(d) + "] cannot divide by nsubvector [" + std::to_string(mp.nsubvector) +
                     "].");
      return nullptr;
    }
    if (mp.nsubvector > IVFPQFastScanIndex::kMaxM) {
      set_last_error("IVFPQFastScan: nsubvector [" + std::to_string(mp.nsubvector) + "] above " +
                     std::to_string(IVFPQFastScanIndex::kMaxM) + " is not supported by this engine");
      return nullptr;
    }
    if (mp.bbs < -1) {
      set_last_error("invalid bbs =" + std::to_string(mp.bbs));
      return nullptr;
    }
    if (mp.bbs > 0 && mp.bbs % 32 != 0) {
      set_last_error("bbs only supports the case where 32 can be divided evenly, bbs=" + std::to_string(mp.bbs));
      return nullptr;
    }
    if (mp.has_opq) {
      set_last_error("IVFPQFastScan: opq is not supported by this engine");
      return nullptr;
    }
    if (mp.ncentroids <= 0 || mp.nprobe > mp.ncentroids) {
      set_last_error("nprobe should be less than ncentroids");
      return nullptr;
    }
    return new IVFPQFastScanIndex(d, mp, device, seg_shift);
  }
  if (type == "BINARYIVF") {  // BinaryModelParams::Parse (gamma_index_binary_ivf.cc:33-50): only ncentroids is read
    if (d % 8 != 0) {
      set_last_error("BINARYIVF: dimension [" + std::to_string(d) + "] must be a multiple of 8 bits");
      return nullptr;
    }
    if (mp.ncentroids_arg < -1) {
      set_last_error("invalid ncentroids = " + std::to_string(mp.ncentroids_arg));
      return nullptr;
    }
    ModelParams bmp = mp;
    bmp.ncentroids = mp.ncentroids_arg > 0 ? mp.ncentroids_arg : BinaryIvfIndex::kDefaultNlist;
    bmp.nprobe = BinaryIvfIndex::kDefaultNprobe;  // the reference ignores nprobe, metric_type and nsubvector
    if (binary_scan_max_k(d / 8) < 1) {
      set_last_error("BINARYIVF: dimension [" + std::to_string(d) + "] is too large for the list scan of this engine");
      return nullptr;
    }
    return new BinaryIvfIndex(d, bmp, device, seg_shift);
  }
  if (type == "IVFRABITQ") {  // IVFRABITQModelParams::Parse / Validate (gamma_index_ivfrabitq.h:370-510)
    if (mp.nb_bits < 1 || mp.nb_bits > 9) {
      set_last_error("invalid nb_bits =" + std::to_string(mp.nb_bits) + " should be integer in [1, 9]");
      return nullptr;
    }
    if (mp.qb < 0 || mp.qb > 8) {
      set_last_error("invalid qb =" + std::to_string(mp.qb) + " should be integer in [0, 8]");
      return nullptr;
    }
    if (mp.ncentroids <= 0 || mp.nprobe > mp.ncentroids) {
      set_last_error("nprobe should be less than ncentroids");
      return nullptr;
    }
    if (d > kRabitqMaxDim) {
      set_last_error("IVFRABITQ: dimension [" + std::to_string(d) + "] above " + std::to_string(kRabitqMaxDim) +
                     " is not supported by this engine");
      return nullptr;
    }
    // the scan's shared memory (stages, the k' queue, the qb = 8 table) must admit k' = 4096 (the lane rule of
    // kernels_rabitq.cu makes it so for every accepted (d, nb_bits)); refused here rather than at every search
    if (rabitq_scan_max_k(d, mp.nb_bits, 8) < 4096) {
      set_last_error("IVFRABITQ: dimension [" + std::to_string(d) + "] at nb_bits " + std::to_string(mp.nb_bits) +
                     " is too large for the list scan of this engine");
      return nullptr;
    }
    return new RaBitQIndex(d, mp, device, seg_shift);
  }
  if (type == "VEARCH") {  // VearchModelParams::Parse / Validate (gamma_index_vearch.cc:40-115); the limits are this engine's
    if (mp.nsubvector > d) {
      set_last_error("VEARCH: nsubvector [" + std::to_string(mp.nsubvector) + "] above the dimension [" + std::to_string(d) +
                     "] is not supported by this engine");
      return nullptr;
    }
    const int nb = scann_blocks(d, mp.nsubvector);
    if (nb > VearchIndex::kMaxBlocks) {
      set_last_error("VEARCH: " + std::to_string(nb) + " blocks (nsubvector " + std::to_string(mp.nsubvector) + ") above " +
                     std::to_string(VearchIndex::kMaxBlocks) + " is not supported by this engine");
      return nullptr;
    }
    // every accepted block count must let the scan select k' = 4096 beside its byte-pair table
    if (vearch_scan_max_k(nb) < 4096) {
      set_last_error("VEARCH: " + std::to_string(nb) + " blocks are too many for the list scan of this engine");
      return nullptr;
    }
    return new VearchIndex(d, mp, device, seg_shift);
  }
  set_last_error("unsupported index type " + type);
  return nullptr;
}

// ------------------------------------------------------------------------------------------
namespace {
// Router merge (mergeSortedArrays, client.go:1530-1589) on device: per query, k-way merge keyed by
// (score, later partition first).  Input scores are already sorted per partition.
template <bool FROM_KEYS>  // FROM_KEYS: `ids` holds the partitions' result keys (score bits << 32 | local id)
__global__ void merge_partitions_kernel(const float* __restrict__ dis, const int64_t* __restrict__ ids, int nparts,
                                        int nq, int k, int metric, float* __restrict__ out_dis,
                                        int64_t* __restrict__ out_ids) {
  extern __shared__ unsigned long long mk[];  // [NP] keys, then [NP] payload
  const int q = blockIdx.x;
  const int total = nparts * k;
  int NP = 1;
  while (NP < total) NP <<= 1;
  unsigned long long* pay = mk + NP;
  for (int i = threadIdx.x; i < NP; i += blockDim.x) {
    unsigned long long key = kKeySentinel, pl = 0;
    if (i < total) {
      int p = i / k, j = i - p * k;
      // low word: later partition first, then rank inside the partition
      const uint32_t lo = ((uint32_t)(nparts - 1 - p) << 16) | (uint32_t)j;
      if (FROM_KEYS) {
        const unsigned long long pk = (unsigned long long)ids[((int64_t)p * nq + q) * k + j];
        if (pk != kKeySentinel) {
          key = make_key((uint32_t)(pk >> 32), lo);
          pl = ((unsigned long long)p << 32) | (uint32_t)pk;
        }
      } else {
        int64_t id = ids[((int64_t)p * nq + q) * k + j];
        if (id >= 0) {
          float s = dis[((int64_t)p * nq + q) * k + j];
          key = make_key(score2ord(s, metric), lo);
          pl = ((unsigned long long)p << 32) | (uint32_t)id;
        }
      }
    }
    mk[i] = key;
    pay[i] = pl;
  }
  __syncthreads();
  // bitonic sort on keys carrying the payload
  for (int kk = 2; kk <= NP; kk <<= 1)
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < NP; i += blockDim.x) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned long long a = mk[i], b = mk[ixj];
          bool up = ((i & kk) == 0);
          if ((a > b) == up) {
            mk[i] = b;
            mk[ixj] = a;
            unsigned long long t = pay[i];
            pay[i] = pay[ixj];
            pay[ixj] = t;
          }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    if (i < NP && mk[i] != kKeySentinel) {
      out_dis[(int64_t)q * k + i] = ord2score((uint32_t)(mk[i] >> 32), metric);
      out_ids[(int64_t)q * k + i] = (int64_t)pay[i];
    } else {
      out_dis[(int64_t)q * k + i] = metric == kMetricL2 ? FLT_MAX : -FLT_MAX;
      out_ids[(int64_t)q * k + i] = -1;
    }
  }
}
}  // namespace

int merge_partition_keys_device(const unsigned long long* keys, int nparts, int nq, int k, int metric, float* out_dis,
                                int64_t* out_ids, cudaStream_t st) {
  if (nq <= 0) return 0;
  int NP = next_pow2(nparts * k);
  if (nparts > 65535 || k > 65535 || NP > 8192) {
    set_last_error("merge_partitions: nparts*k too large");
    return -1;
  }
  size_t smem = (size_t)NP * 16;
  if (smem > 48 * 1024)
    GB_CUDA(cudaFuncSetAttribute(merge_partitions_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  merge_partitions_kernel<true><<<nq, 256, smem, st>>>(nullptr, reinterpret_cast<const int64_t*>(keys), nparts, nq, k, metric,
                                                       out_dis, out_ids);
  note_launch();
  GB_CUDA(cudaGetLastError());
  return 0;
}

int merge_partitions_device(const float* dis, const int64_t* ids, int nparts, int nq, int k, int metric, float* out_dis,
                            int64_t* out_ids, cudaStream_t st) {
  if (nq <= 0) return 0;
  int NP = next_pow2(nparts * k);
  if (nparts > 65535 || k > 65535 || NP > 8192) {
    set_last_error("merge_partitions: nparts*k too large");
    return -1;
  }
  size_t smem = (size_t)NP * 16;
  if (smem > 48 * 1024)
    GB_CUDA(cudaFuncSetAttribute(merge_partitions_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  merge_partitions_kernel<false><<<nq, 256, smem, st>>>(dis, ids, nparts, nq, k, metric, out_dis, out_ids);
  note_launch();
  GB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace gb
