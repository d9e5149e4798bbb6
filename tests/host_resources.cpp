// Host build of sb::Resources (salmon_b200/csrc/resources.h) over a stub CUDA runtime that serves buffers, streams
// and events from host memory, counts them, and can fail its k-th call.  Usage: host_resources <check>; exit code 0
// when the check passes.  tests/test_resources_cpu.py runs every check, also under AddressSanitizer / LeakSanitizer.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>

#include "../salmon_b200/csrc/resources.h"

// ---- stub runtime ---------------------------------------------------------------------------------------------------
namespace stub {
struct Block { size_t bytes; bool host; };
std::map<void*, Block> bufs;                  // live buffers
int live_handles = 0;                         // live streams and events
long calls = 0, fail_at = 0;                  // calls that can fail; fail_at = k fails the k-th (0: none)
long mallocs = 0, set_device = 0;
bool fail() { return ++calls == fail_at; }
cudaError_t take(void** p, size_t n, bool host) {
  if (fail()) { *p = (void*)0x1; return cudaErrorMemoryAllocation; }   // garbage on failure, as a runtime may leave
  *p = malloc(n ? n : 1);
  bufs[*p] = Block{n, host};
  ++mallocs;
  return cudaSuccess;
}
cudaError_t give(void* p, bool host) {
  if (!p) return cudaSuccess;
  auto it = bufs.find(p);
  if (it == bufs.end() || it->second.host != host) { fprintf(stderr, "stub: bad free of %p\n", p); abort(); }
  bufs.erase(it);
  free(p);
  return cudaSuccess;
}
bool live(const void* p) { return bufs.count(const_cast<void*>(p)) != 0; }
size_t bytes_of(const void* p) { return bufs.at(const_cast<void*>(p)).bytes; }
}  // namespace stub

extern "C" {
cudaError_t cudaMalloc(void** p, size_t n) { return stub::take(p, n, false); }
cudaError_t cudaMallocHost(void** p, size_t n) { return stub::take(p, n, true); }
cudaError_t cudaFree(void* p) { return stub::give(p, false); }
cudaError_t cudaFreeHost(void* p) { return stub::give(p, true); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned int) {
  if (stub::fail()) return cudaErrorInvalidValue;
  *s = (cudaStream_t) new int(1);
  ++stub::live_handles;
  return cudaSuccess;
}
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned int) {
  if (stub::fail()) return cudaErrorInvalidValue;
  *e = (cudaEvent_t) new int(2);
  ++stub::live_handles;
  return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s) { delete (int*)s; --stub::live_handles; return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete (int*)e; --stub::live_handles; return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t n, enum cudaMemcpyKind, cudaStream_t) {
  if (stub::fail()) return cudaErrorInvalidValue;
  memcpy(dst, src, n);
  return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaSetDevice(int) { ++stub::set_device; return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t) { return "stub error"; }
}

namespace sb {
static char g_err[512];
void set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap); }
}  // namespace sb

#define SB_TRY(x) do { int _r = (x); if (_r != SB_OK) return _r; } while (0)
#define CHECK(x) do { if (!(x)) { fprintf(stderr, "%s:%d: CHECK(%s) failed\n", __FILE__, __LINE__, #x); return 1; } } while (0)

static uint64_t stat(int i) { return sb::g_resource_stats[i].load(); }

// ---- checks ---------------------------------------------------------------------------------------------------------
// grow keeps a buffer that holds the request and reallocates, with slack bytes/16 + 256, one that does not
static int check_grow() {
  {
    sb::Resources r(0);
    double* p = nullptr;
    CHECK(r.grow(&p, 1000) == SB_OK && p && stub::bytes_of(p) == 8000 + 500 + 256);
    double* const first = p;
    const long m = stub::mallocs;
    CHECK(r.grow(&p, 1000) == SB_OK && p == first);
    CHECK(r.grow(&p, 1094) == SB_OK && p == first);     // 8752 bytes fit the 8756
    CHECK(r.grow(&p, 1) == SB_OK && r.grow(&p, 0) == SB_OK && p == first);
    CHECK(stub::mallocs == m);
    CHECK(r.grow(&p, 1095) == SB_OK && stub::mallocs == m + 1);   // 8760 bytes do not
    CHECK(stub::bytes_of(p) == 8760 + 547 + 256 && !stub::live(first) && stub::bufs.size() == 1);
    uint8_t* z = nullptr;
    CHECK(r.grow(&z, 0) == SB_OK && stub::bytes_of(z) == 1 + 0 + 256);
    CHECK(stat(0) == 2 && stat(1) == 8760 + 547 + 256 + 257);
  }
  CHECK(stub::bufs.empty() && stat(0) == 0 && stat(1) == 0);
  return 0;
}

// alloc is exact (at least one element); page-locked buffers go back through cudaFreeHost; release frees one buffer
// early and ignores pointers the owner did not make
static int check_alloc_release() {
  const long sd = stub::set_device;
  { sb::Resources r(3); }
  CHECK(stub::set_device == sd);                          // an empty owner does not touch the device
  {
    sb::Resources r(3);
    int32_t *a = nullptr, *b = nullptr;
    uint64_t* h = nullptr;
    CHECK(r.alloc(&a, 10) == SB_OK && stub::bytes_of(a) == 40);
    CHECK(r.alloc(&b, 0) == SB_OK && stub::bytes_of(b) == 4);
    CHECK(r.alloc_host(&h, 3) == SB_OK && stub::bytes_of(h) == 24 && stub::bufs.at(h).host);
    int foreign = 0;
    r.release(&foreign);
    r.release(nullptr);
    CHECK(stub::bufs.size() == 3);
    r.release(a);
    CHECK(!stub::live(a) && stub::bufs.size() == 2 && stat(0) == 2 && stat(1) == 28);
    cudaStream_t s = nullptr;
    cudaEvent_t e = nullptr;
    CHECK(r.stream(&s, 0) == SB_OK && r.event(&e, 0) == SB_OK && s && e && stub::live_handles == 2 && stat(0) == 4);
  }
  CHECK(stub::set_device == sd + 1 && stub::bufs.empty() && stub::live_handles == 0 && stat(0) == 0 && stat(1) == 0);
  return 0;
}

// grow_keep: at least doubles, keeps the first `used` elements, frees the old buffer
static int check_grow_keep() {
  sb::Resources r;
  uint32_t* p = nullptr;
  CHECK(r.grow_keep(&p, 0, 10, nullptr) == SB_OK && stub::bytes_of(p) == 40);
  for (uint32_t i = 0; i < 10; ++i) p[i] = 100 + i;
  uint32_t* const first = p;
  CHECK(r.grow_keep(&p, 10, 10, nullptr) == SB_OK && p == first);
  CHECK(r.grow_keep(&p, 7, 11, nullptr) == SB_OK && p != first && !stub::live(first) && stub::bytes_of(p) == 80);
  for (uint32_t i = 0; i < 7; ++i) CHECK(p[i] == 100 + i);
  CHECK(r.grow_keep(&p, 20, 50, nullptr) == SB_OK && stub::bytes_of(p) == 200 && stub::bufs.size() == 1);
  for (uint32_t i = 0; i < 7; ++i) CHECK(p[i] == 100 + i);
  return 0;
}

// a create-like sequence, stopping at the first failure as the library's callers do
struct Obj {
  double *a = nullptr, *g = nullptr;
  uint64_t* h = nullptr;
  uint32_t* k = nullptr;
  cudaStream_t s = nullptr;
  cudaEvent_t e[2] = {nullptr, nullptr};
};
static int create_like(sb::Resources& r, Obj& o) {
  SB_TRY(r.stream(&o.s, cudaStreamNonBlocking));
  for (auto& e : o.e) SB_TRY(r.event(&e, cudaEventDisableTiming));
  SB_TRY(r.alloc(&o.a, 100));
  SB_TRY(r.alloc_host(&o.h, 9));
  SB_TRY(r.grow(&o.g, 10));
  SB_TRY(r.grow(&o.g, 5000));                             // reallocates
  SB_TRY(r.grow_keep(&o.k, 0, 16, o.s));
  SB_TRY(r.grow_keep(&o.k, 16, 17, o.s));                 // reallocates and copies
  r.release(o.a);
  o.a = nullptr;
  SB_TRY(r.alloc(&o.a, 3));
  return SB_OK;
}

// for every k, failing the k-th runtime call leaves every pointer either null or live, and nothing live afterwards
static int check_fail_kth() {
  stub::calls = 0; stub::fail_at = 0;
  {
    sb::Resources r(0);
    Obj o;
    CHECK(create_like(r, o) == SB_OK);
  }
  const long n = stub::calls;
  CHECK(n == 11);
  for (long k = 1; k <= n; ++k) {
    stub::calls = 0; stub::fail_at = k;
    {
      sb::Resources r(0);
      Obj o;
      const int rc = create_like(r, o);
      CHECK(rc == SB_ERR_NOMEM || rc == SB_ERR_CUDA);
      const void* ptrs[] = {o.a, o.g, o.h, o.k};
      for (const void* q : ptrs) CHECK(!q || stub::live(q));
      CHECK(stat(0) == stub::bufs.size() + (size_t)stub::live_handles);
      CHECK(strlen(sb::g_err) > 0);
    }
    CHECK(stub::bufs.empty() && stub::live_handles == 0 && stat(0) == 0 && stat(1) == 0);
    sb::g_err[0] = 0;
  }
  stub::fail_at = 0;
  return 0;
}

int main(int argc, char** argv) {
  const std::string what = argc > 1 ? argv[1] : "";
  if (what == "grow") return check_grow();
  if (what == "alloc_release") return check_alloc_release();
  if (what == "grow_keep") return check_grow_keep();
  if (what == "fail_kth") return check_fail_kth();
  fprintf(stderr, "unknown check %s\n", what.c_str());
  return 2;
}
