// Process-wide plumbing of libpds_b200: error channel, launch counter, device checks, stream-ordered scratch,
// pinned host buffer pool.  There is deliberately NO CPU compute path in this library: if no CUDA device is
// usable every entry point fails with an explicit error.
#include "../common.h"
#include "host.h"
#include <mutex>
#include <vector>
#include <map>
#include <cstring>
#include <cstdlib>

namespace pdsb {

static thread_local std::string t_error;
std::atomic<int64_t> g_kernel_launches{0};

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  t_error = buf;
}
const char* get_error() { return t_error.c_str(); }

static std::once_flag g_dev_once;
static int g_dev_ok = 0;
static int g_sm_count[64];
static std::string g_dev_err;

int require_device() {
  std::call_once(g_dev_once, [] {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
      g_dev_err = std::string("no usable CUDA device (") + cudaGetErrorString(e) +
                  "); libpds_b200 has no CPU fallback";
      return;
    }
    for (int d = 0; d < n && d < 64; ++d) {
      cudaDeviceProp prop;
      if (cudaGetDeviceProperties(&prop, d) == cudaSuccess) {
        g_sm_count[d] = prop.multiProcessorCount;
        // keep freed scratch cached in the default pool instead of returning it to the OS every sync
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, d) == cudaSuccess) {
          uint64_t thr = UINT64_MAX;
          cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
      }
    }
    g_dev_ok = 1;
  });
  if (!g_dev_ok) { set_error("%s", g_dev_err.c_str()); return 1; }
  return 0;
}

int sm_count() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64 || g_sm_count[d] <= 0) return 132;   // H100 SXM
  return g_sm_count[d];
}

int dev_alloc(void** p, size_t bytes, cudaStream_t s) {
  if (bytes == 0) bytes = 16;
  cudaError_t e = cudaMallocAsync(p, bytes, s);
  if (e != cudaSuccess) {
    set_error("device allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
    *p = nullptr;
    return 1;
  }
  return 0;
}
void dev_free(void* p, cudaStream_t s) { if (p) cudaFreeAsync(p, s); }

// ---------------- pinned host pool (size-bucketed free lists) ----------------
namespace {
std::mutex g_pin_mu;
std::multimap<size_t, void*> g_pin_free;
std::map<void*, size_t> g_pin_size;
size_t g_pin_cached = 0;
constexpr size_t kPinCacheCap = size_t(24) << 30;   // keep at most 24 GiB of pinned buffers cached

size_t round_bucket(size_t b) {
  size_t g = 1 << 16;
  while (g < b) g <<= 1;
  // finer granularity for big buffers: round up to 1/8 of the power of two
  if (g >= (size_t(1) << 24)) { size_t step = g >> 3; return ((b + step - 1) / step) * step; }
  return g;
}
}  // namespace

void* pinned_alloc(size_t bytes) {
  size_t b = round_bucket(bytes ? bytes : 1);
  {
    std::lock_guard<std::mutex> lk(g_pin_mu);
    auto it = g_pin_free.lower_bound(b);
    if (it != g_pin_free.end() && it->first <= b + (b >> 2)) {
      void* p = it->second;
      g_pin_cached -= it->first;
      g_pin_free.erase(it);
      return p;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaHostAlloc(&p, b, cudaHostAllocPortable)   /* results may be filled by several devices */;
  if (e != cudaSuccess) { set_error("pinned host allocation of %zu bytes failed: %s", b, cudaGetErrorString(e)); return nullptr; }
  std::lock_guard<std::mutex> lk(g_pin_mu);
  g_pin_size[p] = b;
  return p;
}

void pinned_free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_pin_mu);
  auto it = g_pin_size.find(p);
  if (it == g_pin_size.end()) return;
  size_t b = it->second;
  if (g_pin_cached + b > kPinCacheCap) {
    g_pin_size.erase(it);
    cudaFreeHost(p);
    return;
  }
  g_pin_cached += b;
  g_pin_free.emplace(b, p);
}

// ---------------- per-thread stream ----------------
int thread_stream(cudaStream_t* s) {
  static thread_local cudaStream_t s_stream = nullptr;
  static thread_local int s_dev = -1;
  int d = 0;
  PDSB_CUDA_OK(cudaGetDevice(&d));
  if (s_dev != d) {
    PDSB_CUDA_OK(cudaStreamCreateWithFlags(&s_stream, cudaStreamNonBlocking));
    s_dev = d;
  }
  *s = s_stream;
  return 0;
}

}  // namespace pdsb
