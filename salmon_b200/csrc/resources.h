// resources.h -- one owner for the CUDA resources of a library object: device and page-locked buffers, streams, events.
// The object's kernel argument structs keep plain pointers; the owner records what it allocated into them and releases
// all of it, on the object's device, when it is destroyed.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <unordered_map>
#include <vector>

#include "../../include/salmon_b200.h"

namespace sb {

void set_error(const char* fmt, ...);

// process-wide (sb_debug_device_memory): [0] live buffers, streams and events, [1] live buffer bytes, [2] buffers,
// streams and events made since the library was loaded
inline std::atomic<uint64_t> g_resource_stats[3];

class Resources {
 public:
  explicit Resources(int device = -1) : device_(device) {}
  Resources(const Resources&) = delete;
  Resources& operator=(const Resources&) = delete;
  ~Resources() {
    if (device_ >= 0 && !(bufs_.empty() && streams_.empty() && events_.empty())) cudaSetDevice(device_);
    for (auto& kv : bufs_) free_buf(kv.first, kv.second);
    for (cudaEvent_t e : events_) { cudaEventDestroy(e); counted(-1, 0); }
    for (cudaStream_t s : streams_) { cudaStreamDestroy(s); counted(-1, 0); }
  }

  // exactly max(n, 1) elements; *p is overwritten (buffers sized once)
  template <class T> int alloc(T** p, size_t n) { return malloc_buf((void**)p, std::max<size_t>(n, 1) * sizeof(T), false); }

  // keeps *p when it holds max(n, 1) elements; else frees it and allocates with a little slack against small size
  // changes, so that repeated calls at the same size never allocate again
  template <class T> int grow(T** p, size_t n) {
    const size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
    if (*p && capacity(*p) >= bytes) return SB_OK;
    release(*p);
    *p = nullptr;
    return malloc_buf((void**)p, bytes + bytes / 16 + 256, false);
  }

  // keeps *p when it holds n elements; else at least doubles it, copying the first `used` elements on stream `st`
  template <class T> int grow_keep(T** p, size_t used, size_t n, cudaStream_t st) {
    const size_t cap = *p ? capacity(*p) / sizeof(T) : 0;
    if (n <= cap) return SB_OK;
    T* q = nullptr;
    const int rc = alloc(&q, std::max(n, 2 * cap));
    if (rc != SB_OK) return rc;
    cudaError_t e = used ? cudaMemcpyAsync(q, *p, used * sizeof(T), cudaMemcpyDeviceToDevice, st) : cudaSuccess;
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
      release(q);
      set_error("growing a device buffer to %zu bytes: %s", std::max(n, 2 * cap) * sizeof(T), cudaGetErrorString(e));
      return SB_ERR_CUDA;
    }
    release(*p);
    *p = q;
    return SB_OK;
  }

  // page-locked host memory, exactly max(n, 1) elements
  template <class T> int alloc_host(T** p, size_t n) { return malloc_buf((void**)p, std::max<size_t>(n, 1) * sizeof(T), true); }

  int stream(cudaStream_t* s, unsigned flags) {
    const cudaError_t e = cudaStreamCreateWithFlags(s, flags);
    if (e != cudaSuccess) { *s = nullptr; set_error("cudaStreamCreateWithFlags failed: %s", cudaGetErrorString(e)); return SB_ERR_CUDA; }
    streams_.push_back(*s);
    counted(1, 0);
    return SB_OK;
  }
  int event(cudaEvent_t* ev, unsigned flags) {
    const cudaError_t e = cudaEventCreateWithFlags(ev, flags);
    if (e != cudaSuccess) { *ev = nullptr; set_error("cudaEventCreateWithFlags failed: %s", cudaGetErrorString(e)); return SB_ERR_CUDA; }
    events_.push_back(*ev);
    counted(1, 0);
    return SB_OK;
  }

  // gives one buffer of this owner back early; anything else (nullptr included) is ignored
  void release(void* p) {
    auto it = p ? bufs_.find(p) : bufs_.end();
    if (it == bufs_.end()) return;
    free_buf(it->first, it->second);
    bufs_.erase(it);
  }

 private:
  struct Buf { size_t bytes; bool host; };

  size_t capacity(const void* p) const {
    auto it = bufs_.find(const_cast<void*>(p));
    return it == bufs_.end() ? 0 : it->second.bytes;
  }
  int malloc_buf(void** p, size_t bytes, bool host) {
    const cudaError_t e = host ? cudaMallocHost(p, bytes) : cudaMalloc(p, bytes);
    if (e != cudaSuccess) {
      *p = nullptr;
      set_error("%s(%zu bytes) failed: %s", host ? "cudaMallocHost" : "cudaMalloc", bytes, cudaGetErrorString(e));
      return SB_ERR_NOMEM;
    }
    bufs_[*p] = Buf{bytes, host};
    counted(1, (int64_t)bytes);
    return SB_OK;
  }
  static void free_buf(void* p, const Buf& b) {
    if (b.host) cudaFreeHost(p); else cudaFree(p);
    counted(-1, -(int64_t)b.bytes);
  }
  static void counted(int n, int64_t bytes) {
    g_resource_stats[0] += (uint64_t)(int64_t)n;
    g_resource_stats[1] += (uint64_t)bytes;
    if (n > 0) g_resource_stats[2] += 1;
  }

  int device_;
  std::unordered_map<void*, Buf> bufs_;
  std::vector<cudaStream_t> streams_;
  std::vector<cudaEvent_t> events_;
};

}  // namespace sb
