// The memory ledger (see mem_ledger.h).
#include "mem_ledger.h"

#include <algorithm>
#include <atomic>
#include <fstream>
#include <mutex>
#include <string>
#include <unordered_map>

namespace gb {
namespace mem {

namespace {
constexpr int kMaxDevices = 64;
constexpr int kSlots = kMaxDevices + 1;  // the devices, then the host

int slot(int where) { return where >= 0 && where < kMaxDevices ? where : kMaxDevices; }

struct Ledger {
  std::atomic<int64_t> tracked[kSlots] = {};
  std::atomic<int64_t> total[kSlots] = {};     // 0: not read yet
  std::atomic<int64_t> override_[kSlots] = {};  // set_total
  std::atomic<bool> pool[kMaxDevices] = {};     // configure_pool ran
  std::atomic<int> percent{0};
  std::atomic<void (*)(int)> scratch_release{nullptr};
  std::mutex mu;                                        // sizes of the live allocations
  std::unordered_map<void*, std::pair<int, size_t>> sizes;  // pointer -> (slot, bytes)
};
Ledger& L() {
  static Ledger* l = new Ledger;  // leaked on purpose: frees in static destructors still find it
  return *l;
}

void remember(void* p, int where, size_t bytes) {
  Ledger& l = L();
  l.tracked[slot(where)] += (int64_t)bytes;
  std::lock_guard<std::mutex> g(l.mu);
  l.sizes[p] = {slot(where), bytes};
}
void forget(void* p) {
  Ledger& l = L();
  std::lock_guard<std::mutex> g(l.mu);
  auto it = l.sizes.find(p);
  if (it == l.sizes.end()) return;
  l.tracked[it->second.first] -= (int64_t)it->second.second;
  l.sizes.erase(it);
}

// memoryManager.cc:50-80: MemTotal, or a readable cgroup v1 limit when it is smaller
int64_t host_total() {
  int64_t meminfo = -1, cgroup = -1;
  std::ifstream f("/proc/meminfo");
  std::string key;
  int64_t kb;
  while (f >> key >> kb) {
    if (key == "MemTotal:") {
      meminfo = kb * 1024;
      break;
    }
    f.ignore(1 << 20, '\n');
  }
  std::ifstream c("/sys/fs/cgroup/memory/memory.limit_in_bytes");
  unsigned long long v;
  if (c >> v) cgroup = (int64_t)std::min<unsigned long long>(v, INT64_MAX);
  if (meminfo < 0) return cgroup;
  if (cgroup < 0) return meminfo;
  return std::min(meminfo, cgroup);
}

int64_t total_of(int s) {
  Ledger& l = L();
  const int64_t o = l.override_[s].load();
  if (o > 0) return o;
  int64_t t = l.total[s].load();
  if (t == 0) {
    if (s == kMaxDevices) {
      t = host_total();
    } else {
      cudaDeviceProp prop;
      t = cudaGetDeviceProperties(&prop, s) == cudaSuccess ? (int64_t)prop.totalGlobalMem : -1;
      cudaGetLastError();
    }
    l.total[s] = t;
  }
  return t;
}

bool over(const std::vector<Charge>& c) {
  for (size_t i = 0; i < c.size(); i++) {
    bool first = true;  // each place once, with all that is charged to it
    for (size_t j = 0; j < i; j++) first = first && slot(c[j].where) != slot(c[i].where);
    if (!first) continue;
    int64_t bytes = 0;
    for (size_t j = i; j < c.size(); j++)
      if (slot(c[j].where) == slot(c[i].where)) bytes += c[j].bytes;
    const int64_t lim = limit(c[i].where);
    if (lim > 0 && usage(c[i].where) + bytes > lim) return true;
  }
  return false;
}
}  // namespace

cudaError_t dev_malloc(void** p, size_t bytes) {
  *p = nullptr;
  const cudaError_t e = cudaMalloc(p, bytes);
  if (e != cudaSuccess) return e;
  int dev = 0;
  cudaGetDevice(&dev);
  remember(*p, dev, bytes);
  return cudaSuccess;
}
void dev_free(void* p) {
  if (!p) return;
  forget(p);
  cudaFree(p);
}
cudaError_t host_alloc(void** p, size_t bytes, unsigned flags) {
  *p = nullptr;
  const cudaError_t e = cudaHostAlloc(p, bytes, flags);
  if (e == cudaSuccess) remember(*p, kHost, bytes);
  return e;
}
void host_free(void* p) {
  if (!p) return;
  forget(p);
  cudaFreeHost(p);
}
void charge(int where, int64_t bytes) { L().tracked[slot(where)] += bytes; }

void configure_pool(int device) {
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) != cudaSuccess) return;
  uint64_t thr = UINT64_MAX;  // keep scratch memory cached between searches
  cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  if (device >= 0 && device < kMaxDevices) L().pool[device] = true;
}

int64_t pool_reserved(int device) {
  if (device < 0 || device >= kMaxDevices || !L().pool[device].load()) return 0;
  cudaMemPool_t pool;
  uint64_t v = 0;
  if (cudaDeviceGetDefaultMemPool(&pool, device) != cudaSuccess ||
      cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &v) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return (int64_t)v;
}
int64_t usage(int where) { return L().tracked[slot(where)].load() + (where >= 0 ? pool_reserved(where) : 0); }

void set_limit_percent(int percent) { L().percent = std::max(percent, 0); }
int64_t limit(int where) {
  const int p = L().percent.load();
  if (p <= 0) return 0;
  const int64_t t = total_of(slot(where));
  return t > 0 ? t / 100 * p + t % 100 * p / 100 : 0;
}
bool limited() { return L().percent.load() > 0; }
void set_total(int where, int64_t bytes) { L().override_[slot(where)] = std::max<int64_t>(bytes, 0); }

void set_scratch_release(void (*fn)(int device)) { L().scratch_release = fn; }

bool admit(const std::vector<Charge>& charges) {
  if (!limited() || !over(charges)) return true;
  // memoryManager.cc's malloc_trim: give back what is held but unused, then look again
  void (*release)(int) = L().scratch_release.load();
  int cur = 0;
  cudaGetDevice(&cur);
  for (const Charge& c : charges) {
    if (c.where < 0 || c.where >= kMaxDevices) continue;
    if (release) release(c.where);
    cudaMemPool_t pool;
    if (L().pool[c.where].load() && cudaDeviceGetDefaultMemPool(&pool, c.where) == cudaSuccess) {
      // scratch freed in stream order is released only once the host has seen the frees complete
      cudaSetDevice(c.where);
      cudaDeviceSynchronize();
      cudaMemPoolTrimTo(pool, 0);
    }
    cudaGetLastError();
  }
  cudaSetDevice(cur);
  return !over(charges);
}

}  // namespace mem
}  // namespace gb
