// The memory ledger: every byte this library obtains from the driver, per device and for the host, and the limit
// SetMemoryLimitConfig puts on it (memory/memoryManager.cc, DESIGN.md section 8).  Device memory comes from
// dev_malloc / dev_free, pinned host memory from host_alloc / host_free; memory obtained any other way (the raw
// store's VMM granules) is reported through charge().  The stream-ordered pool every search's scratch comes from is
// not tracked: its reserved bytes are read from the driver when usage is asked for.  Only this module knows the
// counters.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace gb {
namespace mem {

constexpr int kHost = -1;  // `where` of host memory; any other value is a device ordinal

cudaError_t dev_malloc(void** p, size_t bytes);  // cudaMalloc on the current device, charged to it
template <typename T>
cudaError_t dev_malloc(T** p, size_t bytes) {
  return dev_malloc(static_cast<void**>(static_cast<void*>(p)), bytes);
}
void dev_free(void* p);  // cudaFree of a dev_malloc'd pointer (nullptr: nothing)
cudaError_t host_alloc(void** p, size_t bytes, unsigned flags);  // cudaHostAlloc, charged to the host
void host_free(void* p);
void charge(int where, int64_t bytes);  // memory obtained (> 0) or returned (< 0) outside the calls above

// the device's default memory pool, as the library keeps it: nothing released between searches.  Its reserved bytes
// count from then on.
void configure_pool(int device);

// tracked bytes, plus on a device the reserved bytes of its configured pool
int64_t usage(int where);
int64_t pool_reserved(int device);
// percent of total memory (SetMemoryLimitConfig); 0: no limit
void set_limit_percent(int percent);
int64_t limit(int where);  // bytes; 0: no limit
bool limited();            // a limit is set
// the total memory the percentage applies to (a test hook): bytes > 0 replaces the device's HBM or the host's memory,
// 0 restores it
void set_total(int where, int64_t bytes);

// Admission: true when, for every place, usage + the bytes charged to it there stay within its limit.  Before it
// refuses, the memory the library holds but does not use is released (the pools trimmed, the idle scratch buffers of
// the indexes on those devices freed) and the check repeated.
struct Charge {
  int where;
  int64_t bytes;
};
bool admit(const std::vector<Charge>& charges);
// what admit calls to free the idle scratch buffers of a device's indexes (set once by the index module)
void set_scratch_release(void (*fn)(int device));

}  // namespace mem
}  // namespace gb
