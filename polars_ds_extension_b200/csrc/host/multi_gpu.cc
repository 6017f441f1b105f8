// Row-sharding across GPUs INSIDE the library (SURVEY.md §8e, north_star: "partitions the frame across the 8 GPUs and
// NCCL-allreduces the p x p partial Grams over NVLink before a single solve").
//
// Two ways a fit spans several GPUs, both ending in the same ncclAllReduce(sum, f64) of the moments:
//   * device group (single process — what a Polars process is): PDS_B200_DEVICES / pdsb_set_devices choose k devices;
//     one persistent worker thread per device owns its streams and scratch; a plugin call splits its rows into k
//     contiguous shards, every worker uploads its shard over ITS OWN PCIe link, builds the partial moments, joins the
//     in-process NCCL communicator (ncclCommInitAll), solves redundantly and predicts its shard;
//   * world communicator (one process per GPU — torchrun, Dask, Ray): pdsb_comm_init_rank joins an NCCL communicator
//     whose unique id the launcher distributed; every rank's plugin call then contributes its rows to ONE fit.
// The reference has no counterpart (single process, shared memory; SURVEY.md §2a); the Gram being sharded is
// get_xtx_with_lambda / build_xty (/root/reference/src/linear/lr/lr_solvers.rs:183-211, 262-278).
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy torch already loaded, or the system one) so the library
// itself keeps linking against nothing but the CUDA runtime.
#include "../common.h"
#include "host.h"
#include <nccl.h>
#include <dlfcn.h>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <sstream>

namespace pdsb {

// ------------------------------------------------------------------ NCCL, bound at run time -------------
namespace {
struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string err;
};

NcclApi* nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {getenv("PDS_B200_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      if (!n || !*n) continue;
      api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.h) break;
      api.err = dlerror();
    }
    if (!api.h) return;
#define PDSB_SYM(field, name) api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.h, name)); if (!api.field) { api.err = std::string("missing symbol ") + name; api.h = nullptr; return; }
    PDSB_SYM(GetUniqueId, "ncclGetUniqueId")
    PDSB_SYM(CommInitRank, "ncclCommInitRank")
    PDSB_SYM(CommInitAll, "ncclCommInitAll")
    PDSB_SYM(CommDestroy, "ncclCommDestroy")
    PDSB_SYM(AllReduce, "ncclAllReduce")
    PDSB_SYM(AllGather, "ncclAllGather")
    PDSB_SYM(GetErrorString, "ncclGetErrorString")
    PDSB_SYM(GetVersion, "ncclGetVersion")
#undef PDSB_SYM
  });
  return api.h ? &api : nullptr;
}

int nccl_required(NcclApi** out) {
  NcclApi* a = nccl();
  if (!a) {
    set_error("multi-GPU fit needs NCCL (libnccl.so.2 could not be loaded: %s); set PDS_B200_NCCL_LIB or use one device",
              nccl() ? "" : "dlopen failed");
    return 1;
  }
  *out = a;
  return 0;
}

#define PDSB_NCCL_OK(expr)                                                                          \
  do {                                                                                              \
    ncclResult_t _r = (expr);                                                                       \
    if (_r != ncclSuccess) {                                                                        \
      ::pdsb::set_error("NCCL error at %s:%d: %s", __FILE__, __LINE__, api->GetErrorString(_r));    \
      return 1;                                                                                     \
    }                                                                                               \
  } while (0)

std::mutex g_group_mu;
std::unique_ptr<DeviceGroup> g_group;       // the active device group (nullptr: not resolved yet)
bool g_group_resolved = false;

// world communicator (one process per GPU)
std::mutex g_world_mu;
ncclComm_t g_world = nullptr;
int g_world_size = 1, g_world_rank = 0;
std::atomic<int> g_world_on{0};

std::vector<int> parse_devices(const char* e, int n_visible) {
  std::vector<int> d;
  if (!e || !*e) return d;
  std::string s(e);
  if (s == "all") { for (int i = 0; i < n_visible; ++i) d.push_back(i); return d; }
  if (s.find(',') == std::string::npos) {
    char* end = nullptr;
    long k = strtol(s.c_str(), &end, 10);
    if (end && *end == '\0' && k >= 1) { for (int i = 0; i < k && i < n_visible; ++i) d.push_back(i); return d; }
  }
  std::stringstream ss(s);
  std::string tok;
  while (std::getline(ss, tok, ',')) {
    char* end = nullptr;
    long k = strtol(tok.c_str(), &end, 10);
    if (end != tok.c_str() && k >= 0 && k < n_visible) d.push_back((int)k);
  }
  return d;
}
}  // namespace

// ------------------------------------------------------------------ device workers ----------------------
DeviceWorker::DeviceWorker(int dev) : device(dev) {
  th = std::thread([this] {
    cudaSetDevice(device);
    for (;;) {
      std::packaged_task<int()> job;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [this] { return stop || !q.empty(); });
        if (stop && q.empty()) return;
        job = std::move(q.front());
        q.pop_front();
      }
      job();
    }
  });
}
DeviceWorker::~DeviceWorker() {
  { std::lock_guard<std::mutex> lk(mu); stop = true; }
  cv.notify_all();
  if (th.joinable()) th.join();
}
std::future<int> DeviceWorker::submit(std::function<int()> fn) {
  std::packaged_task<int()> task(std::move(fn));
  std::future<int> f = task.get_future();
  { std::lock_guard<std::mutex> lk(mu); q.push_back(std::move(task)); }
  cv.notify_one();
  return f;
}

DeviceGroup::~DeviceGroup() {
  workers.clear();
  NcclApi* api = nccl();
  if (api) for (void* c : comms) if (c) api->CommDestroy((ncclComm_t)c);
}

static int make_group(const std::vector<int>& devs, std::unique_ptr<DeviceGroup>& out) {
  std::unique_ptr<DeviceGroup> g(new DeviceGroup());
  g->devices = devs;
  if (devs.size() > 1) {
    NcclApi* api;
    if (nccl_required(&api)) return 1;
    int cur = 0;
    cudaGetDevice(&cur);
    std::vector<ncclComm_t> comms(devs.size(), nullptr);
    ncclResult_t r = api->CommInitAll(comms.data(), (int)devs.size(), devs.data());
    cudaSetDevice(cur);
    if (r != ncclSuccess) { set_error("ncclCommInitAll over %zu devices failed: %s", devs.size(), api->GetErrorString(r)); return 1; }
    for (ncclComm_t c : comms) g->comms.push_back((void*)c);
    for (int d : devs) g->workers.emplace_back(new DeviceWorker(d));
  }
  out = std::move(g);
  return 0;
}

// the group named by PDS_B200_DEVICES (resolved once) or by the last pdsb_set_devices; nullptr = single device
DeviceGroup* active_group() {
  std::lock_guard<std::mutex> lk(g_group_mu);
  if (!g_group_resolved) {
    g_group_resolved = true;
    int nvis = 0;
    if (cudaGetDeviceCount(&nvis) != cudaSuccess) nvis = 0;
    std::vector<int> d = parse_devices(getenv("PDS_B200_DEVICES"), nvis);
    if (d.size() > 1) {
      std::unique_ptr<DeviceGroup> g;
      if (make_group(d, g) == 0) g_group = std::move(g);
      else fprintf(stderr, "libpds_b200: PDS_B200_DEVICES ignored: %s\n", get_error());
    }
  }
  return (g_group && g_group->devices.size() > 1) ? g_group.get() : nullptr;
}

int group_allreduce_f64(DeviceGroup* g, int idx, double* buf, size_t count, cudaStream_t s) {
  NcclApi* api;
  if (nccl_required(&api)) return 1;
  PDSB_NCCL_OK(api->AllReduce(buf, buf, count, ncclDouble, ncclSum, (ncclComm_t)g->comms[idx], s));
  return 0;
}

bool world_enabled() { return g_world_on.load() != 0; }
int world_size() { return world_enabled() ? g_world_size : 1; }
int world_rank() { return world_enabled() ? g_world_rank : 0; }

int world_allreduce_f64(double* buf, size_t count, cudaStream_t s) {
  NcclApi* api;
  if (nccl_required(&api)) return 1;
  std::lock_guard<std::mutex> lk(g_world_mu);       // collectives of one communicator are issued in one order
  if (!g_world) { set_error("world communicator is not initialised"); return 1; }
  PDSB_NCCL_OK(api->AllReduce(buf, buf, count, ncclDouble, ncclSum, g_world, s));
  return 0;
}

int world_allgather_f64(const double* send, double* recv, size_t count, cudaStream_t s) {
  NcclApi* api;
  if (nccl_required(&api)) return 1;
  std::lock_guard<std::mutex> lk(g_world_mu);
  if (!g_world) { set_error("world communicator is not initialised"); return 1; }
  PDSB_NCCL_OK(api->AllGather(send, recv, count, ncclDouble, g_world, s));
  return 0;
}

}  // namespace pdsb

using namespace pdsb;

extern "C" {

int pdsb_set_devices(const int* devices, int n) {
  if (require_device()) return 1;
  int nvis = 0;
  PDSB_CUDA_OK(cudaGetDeviceCount(&nvis));
  std::vector<int> d;
  for (int i = 0; i < n; ++i) {
    if (!devices || devices[i] < 0 || devices[i] >= nvis) { set_error("pdsb_set_devices: device %d is not visible (%d devices)", devices ? devices[i] : -1, nvis); return 1; }
    d.push_back(devices[i]);
  }
  std::unique_ptr<DeviceGroup> g;
  if (d.size() > 1 && make_group(d, g)) return 1;
  std::lock_guard<std::mutex> lk(g_group_mu);
  g_group = std::move(g);
  g_group_resolved = true;
  return 0;
}

int pdsb_device_group_size(void) {
  if (require_device()) return 0;
  DeviceGroup* g = active_group();
  return g ? (int)g->devices.size() : 1;
}

int pdsb_comm_unique_id(void* out128) {
  NcclApi* api;
  if (nccl_required(&api)) return 1;
  if (!out128) { set_error("pdsb_comm_unique_id: null buffer"); return 1; }
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  PDSB_NCCL_OK(api->GetUniqueId(&id));
  memcpy(out128, &id, sizeof(id));
  return 0;
}

int pdsb_comm_init_rank(int world, int rank, const void* id128) {
  if (require_device()) return 1;
  NcclApi* api;
  if (nccl_required(&api)) return 1;
  if (!id128 || world < 1 || rank < 0 || rank >= world) { set_error("pdsb_comm_init_rank: bad arguments"); return 1; }
  std::lock_guard<std::mutex> lk(g_world_mu);
  if (g_world) { api->CommDestroy(g_world); g_world = nullptr; g_world_on.store(0); }
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  PDSB_NCCL_OK(api->CommInitRank(&g_world, world, id, rank));
  g_world_size = world; g_world_rank = rank;
  g_world_on.store(world > 1 ? 1 : 0);
  return 0;
}

void pdsb_comm_destroy(void) {
  NcclApi* api = nccl();
  std::lock_guard<std::mutex> lk(g_world_mu);
  if (g_world && api) api->CommDestroy(g_world);
  g_world = nullptr; g_world_on.store(0); g_world_size = 1; g_world_rank = 0;
}

int pdsb_comm_size(void) { return world_size(); }

int pdsb_dev_allreduce_f64(double* buf, int64_t count, void* stream) {
  if (require_device()) return 1;
  if (!world_enabled()) return 0;                 // a world of one: the sum is the buffer itself
  return world_allreduce_f64(buf, (size_t)count, (cudaStream_t)stream);
}

int64_t pdsb_last_staged_bytes(void) { return (int64_t)h2d_last_staged_bytes(); }

int pdsb_nccl_version(void) {
  NcclApi* api = nccl();
  int v = 0;
  if (api) api->GetVersion(&v);
  return v;
}

}  // extern "C"
