// The stage of a backup or dump (DESIGN.md §8, backup and snapshots): one byte range a capture copies the partition's
// state into while the table lock is held, and the writer reads after the lock is released.  It lives in HBM, charged
// to the memory ledger like every device allocation, or in pinned host memory when the device cannot hold it: the
// memory limit would be passed, or cudaMalloc fails.  A capture is never refused for the limit.  Pinned host memory is
// mapped, so the kernels that fill a device stage fill a host one through the same pointer.
#pragma once
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "mem_ledger.h"

namespace gb {

class Stage {
 public:
  Stage() = default;
  ~Stage() { release(); }
  Stage(const Stage&) = delete;
  Stage& operator=(const Stage&) = delete;
  Stage(Stage&& o) noexcept { *this = static_cast<Stage&&>(o); }
  Stage& operator=(Stage&& o) noexcept;
  // `bytes` on device `device` (mem::kHost: in pinned host memory); -1 only when neither place can hold them
  int alloc(size_t bytes, int device);
  void release();
  uint8_t* data() const { return p_; }
  size_t size() const { return bytes_; }
  bool on_host() const { return where_ == mem::kHost; }
  // bytes [off, off + n) to `out` (host memory)
  int read(size_t off, size_t n, void* out) const;
  // bytes [off, off + n) appended to f; false on a copy or write error
  bool write(FILE* f, size_t off, size_t n) const;

 private:
  uint8_t* p_ = nullptr;
  size_t bytes_ = 0;
  int where_ = mem::kHost;
};

// bytes staged in HBM and in pinned host memory by the last capture that finished (gb_debug_backup_stage)
void note_capture_stage(int64_t device_bytes, int64_t host_bytes);
void last_capture_stage(int64_t* device_bytes, int64_t* host_bytes);

}  // namespace gb
