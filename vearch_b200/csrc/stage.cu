// The stage of a backup or dump (see stage.h).
#include "stage.h"

#include <string.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "index.h"

namespace gb {

Stage& Stage::operator=(Stage&& o) noexcept {
  if (this != &o) {
    release();
    p_ = o.p_, bytes_ = o.bytes_, where_ = o.where_;
    o.p_ = nullptr, o.bytes_ = 0, o.where_ = mem::kHost;
  }
  return *this;
}

int Stage::alloc(size_t bytes, int device) {
  release();
  if (bytes == 0) return 0;
  void* p = nullptr;
  if (device != mem::kHost && mem::admit({{device, (int64_t)bytes}})) {
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    const cudaError_t e = mem::dev_malloc(&p, bytes);
    cudaSetDevice(cur);
    if (e == cudaSuccess) {
      p_ = static_cast<uint8_t*>(p), bytes_ = bytes, where_ = device;
      return 0;
    }
    cudaGetLastError();  // the device cannot hold it: pinned host memory instead
  }
  const cudaError_t e = mem::host_alloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_last_error("cannot stage " + std::to_string(bytes) + " bytes in HBM or pinned host memory: " +
                   cudaGetErrorString(e));
    return -1;
  }
  p_ = static_cast<uint8_t*>(p), bytes_ = bytes, where_ = mem::kHost;
  return 0;
}

void Stage::release() {
  if (!p_) return;
  if (on_host()) {
    mem::host_free(p_);
  } else {
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(where_);
    mem::dev_free(p_);
    cudaSetDevice(cur);
  }
  p_ = nullptr, bytes_ = 0, where_ = mem::kHost;
}

int Stage::read(size_t off, size_t n, void* out) const {
  if (off + n > bytes_) return -1;
  if (n == 0) return 0;
  if (on_host()) {
    memcpy(out, p_ + off, n);
    return 0;
  }
  GB_CUDA(cudaMemcpy(out, p_ + off, n, cudaMemcpyDeviceToHost));
  return 0;
}

bool Stage::write(FILE* f, size_t off, size_t n) const {
  if (off + n > bytes_) return false;
  if (on_host()) return n == 0 || fwrite(p_ + off, 1, n, f) == n;
  std::vector<uint8_t> buf(std::min<size_t>(n, (size_t)32 << 20));
  for (size_t done = 0; done < n; done += buf.size()) {
    const size_t c = std::min(buf.size(), n - done);
    if (read(off + done, c, buf.data()) || fwrite(buf.data(), 1, c, f) != c) return false;
  }
  return true;
}

namespace {
std::atomic<int64_t> g_stage_dev{0}, g_stage_host{0};
}
void note_capture_stage(int64_t device_bytes, int64_t host_bytes) {
  g_stage_dev = device_bytes;
  g_stage_host = host_bytes;
}
void last_capture_stage(int64_t* device_bytes, int64_t* host_bytes) {
  *device_bytes = g_stage_dev.load();
  *host_bytes = g_stage_host.load();
}

}  // namespace gb
