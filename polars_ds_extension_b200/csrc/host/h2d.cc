// Host -> device transport of the packer (replaces the memcpy into the Vec of series_to_slice_inner,
// /root/reference/src/utils/mod.rs:101-206, by DMA into the device frame).
//
// Polars hands a plugin PAGEABLE Arrow buffers.  cudaMemcpyAsync on pageable memory goes through the driver's own
// staging path (one thread, page by page) and reaches a fraction of the PCIe rate, so large pageable ranges are staged
// here instead: W host threads copy 8 MiB pieces into a per-device ring of pinned slots (two per thread) and each
// piece is DMA'd from its slot on the thread's own stream — memcpy of piece k+1 overlaps the DMA of piece k, and W
// memcpy streams together exceed what one PCIe Gen5 x16 link carries.  Pinned sources (cudaHostAlloc /
// cudaHostRegister) skip all of this.
#include "../common.h"
#include "host.h"
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>
#include <atomic>
#include <map>

namespace pdsb {

namespace {

constexpr size_t PIECE = size_t(8) << 20;
constexpr size_t STAGE_MIN = size_t(1) << 20;      // smaller pageable ranges: the driver's path is fine
constexpr int MAX_W = 32;

struct StageRes {
  void* slot[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  cudaEvent_t done = nullptr;
  cudaStream_t st = nullptr;
  bool used[2] = {false, false};
};
struct StagePool {
  std::mutex mu;                  // one staged upload per device at a time (callers on other threads queue here)
  std::vector<StageRes> res;
  cudaEvent_t start = nullptr;
};
std::mutex g_pools_mu;
std::map<int, std::unique_ptr<StagePool>> g_pools;

StagePool* pool_for(int dev) {
  std::lock_guard<std::mutex> lk(g_pools_mu);
  auto& p = g_pools[dev];
  if (!p) p.reset(new StagePool());
  return p.get();
}

int ensure_res(StagePool* P, int w) {
  if (!P->start) PDSB_CUDA_OK(cudaEventCreateWithFlags(&P->start, cudaEventDisableTiming));
  while ((int)P->res.size() < w) {
    StageRes r;
    for (int i = 0; i < 2; ++i) {
      PDSB_CUDA_OK(cudaHostAlloc(&r.slot[i], PIECE, cudaHostAllocPortable));
      PDSB_CUDA_OK(cudaEventCreateWithFlags(&r.ev[i], cudaEventDisableTiming));
    }
    PDSB_CUDA_OK(cudaEventCreateWithFlags(&r.done, cudaEventDisableTiming));
    PDSB_CUDA_OK(cudaStreamCreateWithFlags(&r.st, cudaStreamNonBlocking));
    P->res.push_back(r);
  }
  return 0;
}

// CPUs this process may actually burn: the cgroup CPU quota (containers: cpu.max "quota period"), else 0 = no limit.
// hardware_concurrency() reports all of the host's cores also when the quota is much smaller, and staging threads
// beyond the quota are throttled as a group (on a 16-CPU quota, 32 staging threads were measured at twice the time of 6).
double cgroup_cpu_quota() {
  double q = 0.0;
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {            // cgroup v2
    char a[64] = {0};
    double period = 0.0;
    if (fscanf(f, "%63s %lf", a, &period) == 2 && strcmp(a, "max") != 0 && period > 0.0) q = atof(a) / period;
    fclose(f);
    return q;
  }
  FILE* fq = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r");    // cgroup v1
  FILE* fp = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
  if (fq && fp) {
    double quota = -1.0, period = 0.0;
    if (fscanf(fq, "%lf", &quota) == 1 && fscanf(fp, "%lf", &period) == 1 && quota > 0.0 && period > 0.0) q = quota / period;
  }
  if (fq) fclose(fq);
  if (fp) fclose(fp);
  return q;
}

int staging_threads() {
  static int w = [] {
    const char* e = getenv("PDS_B200_H2D_THREADS");
    if (e && atoi(e) > 0) return std::min(MAX_W, atoi(e));
    DeviceGroup* g = active_group();
    unsigned ndev = g ? (unsigned)g->devices.size() : 1u;
    // one process per GPU (torchrun): the node's CPUs are shared by LOCAL_WORLD_SIZE such processes
    if (const char* lws = getenv("LOCAL_WORLD_SIZE")) ndev = std::max<unsigned>(ndev, (unsigned)std::max(1, atoi(lws)));
    const double quota = cgroup_cpu_quota();
    if (quota >= 1.0)      // ~0.4 of the quota: the copies need headroom for the DMA completion work and the caller
      return (int)std::min<unsigned>(MAX_W, std::max<unsigned>(2, (unsigned)(quota * 0.4 / ndev + 0.5)));
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    return (int)std::min<unsigned>(16, std::max<unsigned>(2, hw / (2 * ndev)));
  }();
  return w;
}

bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

struct Piece { char* dst; const char* src; size_t bytes; };
thread_local size_t t_staged = 0;

}  // namespace

size_t h2d_last_staged_bytes() { return t_staged; }

int h2d_execute(const std::vector<H2DSeg>& segs, cudaStream_t s) {
  NvtxRange nv("pdsb:h2d");
  t_staged = 0;
  std::vector<Piece> pieces;
  for (const H2DSeg& g : segs) {
    if (!g.bytes) continue;
    if (g.bytes < STAGE_MIN || is_pinned(g.src)) {
      PDSB_CUDA_OK(cudaMemcpyAsync(g.dst, g.src, g.bytes, cudaMemcpyHostToDevice, s));
      continue;
    }
    for (size_t off = 0; off < g.bytes; off += PIECE)
      pieces.push_back({(char*)g.dst + off, (const char*)g.src + off, std::min(PIECE, g.bytes - off)});
    t_staged += g.bytes;
  }
  if (pieces.empty()) return 0;
  int dev = 0;
  PDSB_CUDA_OK(cudaGetDevice(&dev));
  StagePool* P = pool_for(dev);
  std::lock_guard<std::mutex> lk(P->mu);
  const int W = (int)std::min<size_t>(staging_threads(), pieces.size());
  if (ensure_res(P, W)) return 1;
  // destinations were allocated (stream-ordered) on `s`: the staging streams start after that point
  PDSB_CUDA_OK(cudaEventRecord(P->start, s));
  std::atomic<size_t> next{0};
  std::atomic<int> failed{0};
  std::vector<std::string> errs(W);
  auto work = [&](int w) {
    StageRes& R = P->res[w];
    if (cudaSetDevice(dev) != cudaSuccess || cudaStreamWaitEvent(R.st, P->start, 0) != cudaSuccess) { failed = 1; errs[w] = "staging stream setup failed"; return; }
    int k = 0;
    for (;;) {
      const size_t i = next.fetch_add(1);
      if (i >= pieces.size() || failed.load()) break;
      const Piece& pc = pieces[i];
      if (R.used[k] && cudaEventSynchronize(R.ev[k]) != cudaSuccess) { failed = 1; errs[w] = "staging event wait failed"; break; }
      memcpy(R.slot[k], pc.src, pc.bytes);
      cudaError_t e = cudaMemcpyAsync(pc.dst, R.slot[k], pc.bytes, cudaMemcpyHostToDevice, R.st);
      if (e == cudaSuccess) e = cudaEventRecord(R.ev[k], R.st);
      if (e != cudaSuccess) { failed = 1; errs[w] = std::string("staged H2D failed: ") + cudaGetErrorString(e); break; }
      R.used[k] = true;
      k ^= 1;
    }
    cudaEventRecord(R.done, R.st);
  };
  std::vector<std::thread> th;
  for (int w = 1; w < W; ++w) th.emplace_back(work, w);
  work(0);
  for (auto& t : th) t.join();
  for (int w = 0; w < W; ++w) PDSB_CUDA_OK(cudaStreamWaitEvent(s, P->res[w].done, 0));
  if (failed.load()) {
    for (auto& e : errs) if (!e.empty()) { set_error("%s", e.c_str()); break; }
    return 1;
  }
  return 0;
}

}  // namespace pdsb
