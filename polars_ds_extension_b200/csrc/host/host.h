// Host-side internals shared by api_dev.cc / lr_host.cc / grouped_host.cc / models_host.cc / multi_gpu.cc / h2d.cc / the
// plugin ABI layer.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <string>
#include <vector>
#include <deque>
#include <memory>
#include <thread>
#include <mutex>
#include <condition_variable>
#include <future>
#include <functional>
#include "../../../include/pdsb.h"
#include "../common.h"

namespace pdsb {

void* pinned_alloc(size_t bytes);
void pinned_free(void* p);
int thread_stream(cudaStream_t* s);     // this thread's stream on the current device

// RAII bag of stream-ordered device allocations
struct DevBag {
  cudaStream_t s;
  std::vector<void*> ptrs;
  explicit DevBag(cudaStream_t st) : s(st) {}
  ~DevBag() { for (void* p : ptrs) dev_free(p, s); }
  template <typename U> U* alloc(size_t count) {
    void* p = nullptr;
    if (dev_alloc(&p, count * sizeof(U), s)) return nullptr;
    ptrs.push_back(p);
    return reinterpret_cast<U*>(p);
  }
};

inline int64_t pad_ld(int64_t n) { return (n + 31) & ~int64_t(31); }   // 128-byte aligned columns

// NVTX range per host phase (SURVEY.md §5: the reference has no tracing; nsys / ncu --nvtx group by these names)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// null policy of the reference (src/linear/mod.rs:34-66).  The reference parses the fill as NullPolicy<f64> for the f64
// symbols and NullPolicy<f32> for the _f32 twins, so the literal is kept rounded once to each: (float)strtod would round
// a decimal string twice.
enum class NullKind { RAISE, SKIP, SKIP_WINDOW, IGNORE, FILL, FILL_WINDOW };
struct NullPolicy {
  NullKind kind;
  double fill;
  float fill_f32;
  template <typename T> T fill_as() const;
};
template <> inline double NullPolicy::fill_as<double>() const { return fill; }
template <> inline float NullPolicy::fill_as<float>() const { return fill_f32; }
// returns 0 / 1 ("Invalid NullPolicy.")
int parse_null_policy(const char* s, NullPolicy* out);

// group g is rows [offsets[g], offsets[g+1]) of n (host offsets, n_groups >= 1); 0 / 1 with "<what>: bad group offsets"
// or "<what>: group offsets must be non-decreasing and within [0, n] (group g)" (grouped_host.cc)
int check_group_offsets(const int64_t* offsets, int64_t n_groups, int64_t n, const char* what = "grouped lin_reg");

int solver_from_string(const char* s);   // lr/mod.rs:18-27
int se_type_from_string(const char* s);  // linear_regression.rs:122-132

// ---- host -> device copies (h2d.cc) ----
// One contiguous host range -> one device range.  Pinned sources go straight to the copy engine; pageable sources
// (what Polars hands a plugin) are staged through a per-device ring of pinned slots by a few host threads, so the
// page-by-page driver path (a single staging thread) is never taken for large buffers.
struct H2DSeg { void* dst; const void* src; size_t bytes; };
// Enqueue all copies; on return `s` is ordered after every one of them (the host may still be copying nothing: all
// staging memcpy()s are complete on return, only DMA may be in flight).  Destinations must have been allocated on `s`.
int h2d_execute(const std::vector<H2DSeg>& segs, cudaStream_t s);
// statistics of the last h2d_execute on this thread: bytes that took the staged (pageable) route
size_t h2d_last_staged_bytes();

// ---- multi-GPU (multi_gpu.cc) ----
struct DeviceWorker {
  int device;
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<std::packaged_task<int()>> q;
  bool stop = false;
  explicit DeviceWorker(int dev);
  ~DeviceWorker();
  std::future<int> submit(std::function<int()> fn);
};
struct DeviceGroup {
  std::vector<int> devices;
  std::vector<void*> comms;                            // ncclComm_t per device (in-process communicator)
  std::vector<std::unique_ptr<DeviceWorker>> workers;  // one persistent thread per device
  ~DeviceGroup();
};
DeviceGroup* active_group();                 // nullptr: single-device operation
int group_allreduce_f64(DeviceGroup* g, int idx, double* buf, size_t count, cudaStream_t s);
bool world_enabled();                        // one-process-per-GPU communicator joined (pdsb_comm_init_rank)
int world_size();
int world_rank();
int world_allreduce_f64(double* buf, size_t count, cudaStream_t s);
int world_allgather_f64(const double* send, double* recv, size_t count, cudaStream_t s);

// ---- Arrow ingest and results of the host entries, single (lr_host.cc) and grouped (grouped_host.cc) ----
// Library-internal: hidden, so none of them joins the shared library's exported symbols.
#pragma GCC visibility push(hidden)

int64_t col_len(const pdsb_column& c);
int64_t col_nulls(const pdsb_column& c);

// Rows of a chunked column, read in non-decreasing row order: at(r) is row r's validity and, when valid, its value in *v
// (F64 or F32; NaN for any other dtype).  r < col_len(c).
struct RowReader {
  const pdsb_column& c;
  int ci = 0;          // the chunk that holds row c0 onwards
  int64_t c0 = 0;
  bool at(int64_t r, double* v);
};

// All host->device copies of one frame are collected first and executed together (h2d.cc: pinned sources DMA directly,
// pageable sources are staged by several host threads); kernels that consume uploaded raw bytes run afterwards.
struct UploadPlan {
  std::vector<H2DSeg> segs;
  std::vector<std::function<int()>> after;      // K1 launches that read the uploaded raw / validity bytes
  int run(cudaStream_t s) {
    if (h2d_execute(segs, s)) return 1;
    for (auto& f : after) if (f()) return 1;
    segs.clear(); after.clear();
    return 0;
  }
};

// Upload one column into dst[0..n) as T.  mode: 0 null->NaN, 1 null->fill, 2 null->0
template <typename T>
int upload_column(const pdsb_column& c, T* dst, int mode, T fill, DevBag& bag, UploadPlan& plan, cudaStream_t s);
// The per-row null mask of cols[0 .. n_cols): a new [ld] array, 1 where every one of the columns is valid and 0 where one
// is null.  The fill to 1 is launched now; the validity uploads and the launches that clear the null rows go into plan.
template <typename T>
T* row_mask(const pdsb_column* cols, int n_cols, int64_t n, int64_t ld, DevBag& bag, UploadPlan& plan, cudaStream_t s);
// cols[0 .. k) into new f64 arrays dst[0 .. k) of n each (nulls -> NaN), in one plan run
int upload_f64(const pdsb_column* cols, int k, int64_t n, double** dst, DevBag& bag, cudaStream_t s);

template <typename T>
struct Frame {
  T* Z = nullptr;       // [ld x (t + p)] column-major: targets first, then features
  int64_t ld = 0, n = 0;
  int p = 0, t = 0;
  T* mask = nullptr;    // per-row validity (nullptr: every row valid)
  T* w = nullptr;
  bool any_null = false;
  const T* Y() const { return Z; }
  const T* X() const { return Z + (size_t)t * ld; }
};
// The reference's shape checks on [targets | features], in its order; returns the row count, or -1 with the error set.
int64_t checked_rows(const pdsb_column* cols, int n_cols, int n_targets);
// "Shape of weights is not the same as the data." unless w has n rows.  Apart from checked_rows: lin_reg checks the
// weights' length before the null policy, the reports after it.
int check_weights(const pdsb_column& w, int64_t n);
// Null policy + upload of [targets | features] (+ weights) into a new device frame.  online = rolling/recursive: rows
// are never dropped, nulls become NaN (or the fill value) and the kernel masks them.
template <typename T>
int build_frame(const pdsb_column* cols, int n_cols, int n_targets, const pdsb_column* wcol, const NullPolicy& pol,
                bool multi, bool online, Frame<T>& F, DevBag& bag, cudaStream_t s);

// pl_lr's dispatch (linear_regression.rs:436-498) for p features and t targets
pdsb_solve_opts lr_solve_opts(const pdsb_lr_kwargs* kw, int p, int t, bool is_f32, int want_pred);

// A new pinned buffer of `bytes`, owned by r (freed by pdsb_host_result_free)
void* result_buf(pdsb_host_result* r, size_t bytes);
// *dst = a result buffer of `bytes`, filled from the device array `src` on `s` (complete at the next synchronize)
template <typename U>
int result_copy(pdsb_host_result* r, U*& dst, const void* src, size_t bytes, cudaStream_t s) {
  void* p = result_buf(r, bytes);
  if (!p) return 1;
  dst = static_cast<U*>(p);
  PDSB_CUDA_OK(cudaMemcpyAsync(p, src, bytes, cudaMemcpyDeviceToHost, s));
  return 0;
}

// the checked group offsets on the device, n_groups + 1 entries (grouped_host.cc)
int upload_offsets(const int64_t* offsets, int64_t n_groups, int64_t*& doff, DevBag& bag, cudaStream_t s);
// the per-group statuses [count] back in h, then a synchronise: every copy queued before them has landed as well
int download_status(const int* dst, size_t count, std::vector<int>& h, cudaStream_t s);

// Every extern "C" host entry runs this way: require_device, then the entry's own argument checks (`args` sets the
// error and returns 1 for a bad call), then a zeroed result, the call, and the result freed again when the call fails.
// ARGS_FIRST: the argument checks read host data only and run before require_device, so a bad call gives its own
// message on every machine.
template <bool ARGS_FIRST = false, typename Args, typename Call>
int guarded(pdsb_host_result* out, Args args, Call call) {
  if (ARGS_FIRST ? (args() || require_device()) : (require_device() || args())) return 1;
  memset(out, 0, sizeof(*out));
  const int rc = call();
  if (rc) pdsb_host_result_free(out);
  return rc;
}
// the argument checks of the lin_reg-family entries; the grouped ones look at their offsets first (null_group_args)
int null_args(const void* kw, const void* cols, const void* out);
// pca / pca_by: f32 columns stay f32 on the device when every column is f32
bool all_f32(const pdsb_column* cols, int n_cols);

#pragma GCC visibility pop

}  // namespace pdsb
