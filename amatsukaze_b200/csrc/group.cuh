// group.cuh -- multi-GPU in the library (SURVEY.md 8(e)): ONE process, one context + stream + host thread per device,
// NCCL (ncclCommInitAll) for the only communication the path has -- the final gather of the per-frame result blocks, and
// the exact integer all-reduce of a frame-sharded LogoScan.  Included at the end of amtk_b200.cu (same translation unit).
//
// The path shards without any data-path collective: independent clips run one per GPU (BASELINE configs[4]; the
// reference schedules whole jobs per GPU, Server/ResourceManager.cs:81-85), so the kernels never talk to each other.
// NCCL is loaded with dlopen on first use: the library keeps loading on machines without it, and a process that already
// carries an NCCL (PyTorch) shares that copy.
#pragma once
#include <condition_variable>
#include <dlfcn.h>
#include <functional>
#include <sched.h>
#include <thread>

namespace amtk {

// ---- the handful of NCCL entry points used, bound at run time -------------------------------------------------------
typedef struct ncclComm* ncclComm_t;
enum { kNcclSuccess = 0 };
enum { kNcclInt32 = 2, kNcclUint64 = 5, kNcclFloat32 = 7 };     // ncclDataType_t values (nccl.h: ncclInt32 = 2, ncclUint64 = 5, ncclFloat32 = 7)
enum { kNcclSum = 0 };
struct NcclApi {
  void* handle = nullptr;
  int (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  int (*GetVersion)(int*) = nullptr;
  bool ok() const { return handle && CommInitAll && CommDestroy && AllGather && AllReduce && GroupStart && GroupEnd; }
};
static NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    for (const char* name : { "libnccl.so.2", "libnccl.so" }) {
      api.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) return;
    auto sym = [&](const char* n) { return dlsym(api.handle, n); };
    api.CommInitAll = reinterpret_cast<decltype(api.CommInitAll)>(sym("ncclCommInitAll"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(sym("ncclAllReduce"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(sym("ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(sym("ncclGroupEnd"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(sym("ncclGetVersion"));
  });
  return api;
}

// One persistent host thread per device: runs the (blocking, host-driven) library calls of its device so that eight
// host-clip passes stage their frames concurrently, pinned to the CPUs next to the GPU.
struct DeviceWorker {
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::function<int()> task;
  bool has_task = false, done = false, quit = false;
  int result = 1;
  std::string error;
  void run() {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv.wait(lk, [&] { return has_task || quit; });
      if (quit) return;
      std::function<int()> t = std::move(task);
      has_task = false;
      lk.unlock();
      const int r = t();
      const std::string e = r ? std::string() : std::string(amtk_last_error());
      lk.lock();
      result = r; error = e; done = true;
      cv.notify_all();
    }
  }
  void post(std::function<int()> t) {
    std::lock_guard<std::mutex> lk(mu);
    task = std::move(t); has_task = true; done = false;
    cv.notify_all();
  }
  int wait(std::string* err) {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return done; });
    if (!result && err && err->empty()) *err = error;
    return result;
  }
  void stop() {
    { std::lock_guard<std::mutex> lk(mu); quit = true; cv.notify_all(); }
    if (th.joinable()) th.join();
  }
};

// CPUs on the same PCIe root / NUMA node as a GPU, from sysfs (what `nvidia-smi topo -m` prints as CPU Affinity)
static bool gpu_local_cpus(int device, cpu_set_t* set) {
  char bdf[32] = { 0 };
  if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), device) != cudaSuccess) { cudaGetLastError(); return false; }
  for (char* p = bdf; *p; ++p) *p = (char)tolower(*p);
  const std::string path = std::string("/sys/bus/pci/devices/") + bdf + "/local_cpulist";
  FILE* fp = fopen(path.c_str(), "r");
  if (!fp) return false;
  char line[4096] = { 0 };
  const bool got = fgets(line, sizeof(line), fp) != nullptr;
  fclose(fp);
  if (!got) return false;
  CPU_ZERO(set);
  int n = 0;
  for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int a = 0, b = 0;
    if (sscanf(tok, "%d-%d", &a, &b) == 2) { for (int c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET(c, set); ++n; } }
    else if (sscanf(tok, "%d", &a) == 1 && a < CPU_SETSIZE) { CPU_SET(a, set); ++n; }
  }
  return n > 0;
}

}  // namespace amtk

struct amtk_group {
  int ndev = 0;
  std::vector<int> devices;
  std::vector<amtk_ctx*> ctx;
  std::vector<amtk::ncclComm_t> comm;
  std::vector<amtk::StreamHandle> gstream;           // side stream per device for the collectives
  std::vector<amtk::EventHandle> ev_compute, ev_gather;   // compute done -> gather may start; gather done -> buffers reusable
  std::vector<amtk::DevBuf<uint8_t>> send, recv;     // per device: result block / gathered blocks
  size_t send_bytes = 0;
  std::vector<std::vector<amtk::EventHandle>> marks;   // timing marks [slot][device]
  std::vector<std::unique_ptr<amtk::DeviceWorker>> workers;
  std::vector<int> numa_bound;
  int nccl_version = 0;
};

namespace amtk {

static int group_run(amtk_group* g, const std::function<int(int)>& fn) {     // fn(i) on every device's own thread, in parallel
  for (int i = 0; i < g->ndev; ++i) g->workers[i]->post([fn, i] { return fn(i); });
  std::string err; int ok = 1;
  for (int i = 0; i < g->ndev; ++i) ok &= g->workers[i]->wait(&err);
  if (!ok) set_error(err.empty() ? "group call failed" : err);
  return ok;
}
static bool nccl_ok(int r, const char* what) {
  if (r == kNcclSuccess) return true;
  const NcclApi& a = nccl_api();
  set_error(std::string("NCCL error: ") + (a.GetErrorString ? a.GetErrorString(r) : "?") + " in " + what);
  return false;
}
static int group_ensure_buffers(amtk_group* g, size_t send_bytes) {
  if (g->send_bytes >= send_bytes) return 1;
  return group_run(g, [g, send_bytes](int i) {
    DevSelect ds(g->ctx[i]); if (!ds.ok) return 0;
    g->send[i].reset(); g->recv[i].reset();
    AMTK_CUDA(cudaMalloc(g->send[i].put(), send_bytes));
    AMTK_CUDA(cudaMalloc(g->recv[i].put(), send_bytes * g->ndev));
    return 1;
  }) ? (g->send_bytes = send_bytes, 1) : 0;
}

}  // namespace amtk

extern "C" {

int amtk_group_create(int ndev, const int* devices, amtk_group** out) {
  if (!out || ndev < 1) AMTK_FAIL("amtk_group_create: bad argument");
  *out = nullptr;
  const int have = amtk_device_count();
  if (ndev > have) AMTK_FAIL("amtk_group_create: more devices requested than visible");
  amtk::NcclApi& api = amtk::nccl_api();
  if (ndev > 1 && !api.ok()) AMTK_FAIL("amtk_group_create: libnccl.so.2 not found (needed for more than one device)");
  std::unique_ptr<amtk_group> g(new amtk_group());
  g->ndev = ndev;
  for (int i = 0; i < ndev; ++i) g->devices.push_back(devices ? devices[i] : i);
  g->ctx.assign(ndev, nullptr); g->comm.assign(ndev, nullptr); g->gstream.resize(ndev);
  g->ev_compute.resize(ndev); g->ev_gather.resize(ndev);
  g->send.resize(ndev); g->recv.resize(ndev); g->numa_bound.assign(ndev, 0);
  for (int i = 0; i < ndev; ++i) {
    g->workers.emplace_back(new amtk::DeviceWorker());
    amtk::DeviceWorker* w = g->workers.back().get();
    w->th = std::thread([w] { w->run(); });
  }
  amtk_group* gp = g.get();
  // every device thread: bind to the GPU's CPUs (so its pinned staging memory is NUMA-local), create a stream + context
  int ok = amtk::group_run(gp, [gp](int i) {
    const int dev = gp->devices[i];
    cpu_set_t set;
    if (!getenv("AMTK_GROUP_NO_BIND") && amtk::gpu_local_cpus(dev, &set) && sched_setaffinity(0, sizeof(set), &set) == 0) gp->numa_bound[i] = CPU_COUNT(&set);
    AMTK_CUDA(cudaSetDevice(dev));
    amtk::StreamHandle st;
    AMTK_CUDA(cudaStreamCreateWithFlags(st.put(), cudaStreamNonBlocking));
    if (!amtk_ctx_create(dev, st, &gp->ctx[i])) return 0;
    gp->ctx[i]->owned_stream = std::move(st);
    AMTK_CUDA(cudaStreamCreateWithFlags(gp->gstream[i].put(), cudaStreamNonBlocking));
    AMTK_CUDA(cudaEventCreateWithFlags(gp->ev_compute[i].put(), cudaEventDisableTiming));
    AMTK_CUDA(cudaEventCreateWithFlags(gp->ev_gather[i].put(), cudaEventDisableTiming));
    AMTK_CUDA(cudaEventRecord(gp->ev_gather[i], gp->gstream[i]));
    return 1;
  });
  if (ok && ndev > 1) {
    ok = amtk::nccl_ok(api.CommInitAll(gp->comm.data(), ndev, gp->devices.data()), "ncclCommInitAll");
    if (ok && api.GetVersion) api.GetVersion(&gp->nccl_version);
  }
  if (!ok) { const std::string e = amtk_last_error(); amtk_group_destroy(g.release()); amtk::set_error(e); return 0; }
  *out = g.release();
  return 1;
}

void amtk_group_destroy(amtk_group* g) {
  if (!g) return;
  if (!g->workers.empty()) {
    amtk::group_run(g, [g](int i) {
      cudaSetDevice(g->devices[i]);
      if (g->ctx[i]) cudaStreamSynchronize(g->ctx[i]->stream);
      if (g->gstream[i]) cudaStreamSynchronize(g->gstream[i]);
      if (g->comm[i]) amtk::nccl_api().CommDestroy(g->comm[i]);
      if (g->ctx[i]) amtk_ctx_destroy(g->ctx[i]);
      return 1;
    });
    for (auto& w : g->workers) w->stop();
  }
  delete g;                      // the group's buffers, events and collective streams: every stream is idle by now
}

int amtk_group_size(const amtk_group* g) { return g ? g->ndev : 0; }
amtk_ctx* amtk_group_ctx(amtk_group* g, int i) { return (g && i >= 0 && i < g->ndev) ? g->ctx[i] : nullptr; }
int amtk_group_numa_cpus(const amtk_group* g, int i) { return (g && i >= 0 && i < g->ndev) ? g->numa_bound[i] : 0; }
int amtk_group_nccl_version(const amtk_group* g) { return g ? g->nccl_version : 0; }

int amtk_group_host_alloc(amtk_group* g, int i, size_t bytes, void** out) {
  if (!g || !out || i < 0 || i >= g->ndev) AMTK_FAIL("amtk_group_host_alloc: bad argument");
  // allocated (and first touched) by the device's own thread: the pages land on the GPU's NUMA node
  g->workers[i]->post([g, i, bytes, out] {
    DevSelect ds(g->ctx[i]); if (!ds.ok) return 0;
    AMTK_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
    memset(*out, 0, bytes);
    return 1;
  });
  std::string err;
  if (!g->workers[i]->wait(&err)) { amtk::set_error(err); return 0; }
  return 1;
}

// BASELINE configs[4]: ndev independent clips, one per device.  Enqueues on every device the fused pass (ScanFrame scores
// of logos[i] + combing counters) over clips[i] and then ONE ncclAllGather of the per-device result blocks
// ([nframes][2] float scores followed by [nframes][12] int32 counters) on a side stream.  Asynchronous for device clips:
// returns when the work is enqueued; amtk_group_fetch_results / amtk_group_synchronize wait for it.
int amtk_group_scan_comb_streams(amtk_group* g, const amtk_clip* clips, amtk_logo* const* logos, const amtk_comb_params* prm, int nframes) {
  if (!g || !clips || !logos || !prm || nframes < 1) AMTK_FAIL("amtk_group_scan_comb_streams: bad argument");
  const size_t block = (size_t)nframes * 14 * sizeof(int32_t);
  if (!amtk::group_ensure_buffers(g, block)) return 0;
  amtk::NcclApi& api = amtk::nccl_api();
  return amtk::group_run(g, [g, clips, logos, prm, nframes, block, &api](int i) {
    amtk_ctx* c = g->ctx[i];
    DevSelect ds(c); if (!ds.ok) return 0;
    float* scores = reinterpret_cast<float*>(g->send[i].get());
    int32_t* counts = reinterpret_cast<int32_t*>(g->send[i].get()) + (size_t)nframes * 2;
    AMTK_CUDA(cudaStreamWaitEvent(c->stream, g->ev_gather[i], 0));             // the previous gather has read the send block
    amtk_logo* lg = logos[i];
    if (!amtk_scan_comb_frames(c, &clips[i], &lg, 1, prm, 0, nframes, scores, counts, 1)) return 0;
    AMTK_CUDA(cudaEventRecord(g->ev_compute[i], c->stream));
    AMTK_CUDA(cudaStreamWaitEvent(g->gstream[i], g->ev_compute[i], 0));
    if (g->ndev > 1) {
      if (!amtk::nccl_ok(api.AllGather(g->send[i], g->recv[i], block / sizeof(int32_t), amtk::kNcclInt32, g->comm[i], g->gstream[i]), "ncclAllGather")) return 0;
    } else {
      AMTK_CUDA(cudaMemcpyAsync(g->recv[i], g->send[i], block, cudaMemcpyDeviceToDevice, g->gstream[i]));
    }
    AMTK_CUDA(cudaEventRecord(g->ev_gather[i], g->gstream[i]));
    return 1;
  });
}

// Copies the gathered results of the last pass (as held by device `from`) to the host:
// scores float[ndev][nframes][2], counts int32[ndev][nframes][12].
int amtk_group_fetch_results(amtk_group* g, int from, int nframes, float* scores, int32_t* counts) {
  if (!g || from < 0 || from >= g->ndev || !scores || !counts) AMTK_FAIL("amtk_group_fetch_results: bad argument");
  const size_t block = (size_t)nframes * 14 * sizeof(int32_t);
  if (g->send_bytes < block) AMTK_FAIL("amtk_group_fetch_results: no results of that size");
  g->workers[from]->post([g, from, nframes, scores, counts, block] {
    DevSelect ds(g->ctx[from]); if (!ds.ok) return 0;
    AMTK_CUDA(cudaStreamSynchronize(g->gstream[from]));
    std::vector<int32_t> tmp(block / 4 * g->ndev);
    AMTK_CUDA(cudaMemcpy(tmp.data(), g->recv[from], tmp.size() * 4, cudaMemcpyDeviceToHost));
    for (int d = 0; d < g->ndev; ++d) {
      const int32_t* b = tmp.data() + (size_t)d * nframes * 14;
      memcpy(scores + (size_t)d * nframes * 2, b, (size_t)nframes * 2 * sizeof(float));
      memcpy(counts + (size_t)d * nframes * 12, b + (size_t)nframes * 2, (size_t)nframes * 12 * sizeof(int32_t));
    }
    return 1;
  });
  std::string err;
  if (!g->workers[from]->wait(&err)) { amtk::set_error(err); return 0; }
  return 1;
}

int amtk_group_synchronize(amtk_group* g) {
  if (!g) AMTK_FAIL("null group");
  return amtk::group_run(g, [g](int i) {
    DevSelect ds(g->ctx[i]); if (!ds.ok) return 0;
    AMTK_CUDA(cudaStreamSynchronize(g->ctx[i]->stream));
    AMTK_CUDA(cudaStreamSynchronize(g->gstream[i]));
    return 1;
  });
}

// Device-side timing: a mark is one CUDA event per device, recorded after everything enqueued so far on the device's
// compute AND collective streams; elapsed = per-device milliseconds between two marks (the caller takes the maximum).
int amtk_group_mark(amtk_group* g, int slot) {
  if (!g || slot < 0 || slot > 63) AMTK_FAIL("amtk_group_mark: slot must be 0..63");
  if ((int)g->marks.size() <= slot) g->marks.resize(slot + 1);
  if (g->marks[slot].empty()) g->marks[slot].resize(g->ndev);
  return amtk::group_run(g, [g, slot](int i) {
    DevSelect ds(g->ctx[i]); if (!ds.ok) return 0;
    if (!g->marks[slot][i]) AMTK_CUDA(cudaEventCreate(g->marks[slot][i].put()));
    AMTK_CUDA(cudaStreamWaitEvent(g->ctx[i]->stream, g->ev_gather[i], 0));
    AMTK_CUDA(cudaEventRecord(g->marks[slot][i], g->ctx[i]->stream));
    return 1;
  });
}
int amtk_group_elapsed_ms(amtk_group* g, int slot_a, int slot_b, double* ms_per_device) {
  if (!g || !ms_per_device || slot_a < 0 || slot_b < 0 || slot_a >= (int)g->marks.size() || slot_b >= (int)g->marks.size() ||
      g->marks[slot_a].empty() || g->marks[slot_b].empty()) AMTK_FAIL("amtk_group_elapsed_ms: unknown mark");
  return amtk::group_run(g, [g, slot_a, slot_b, ms_per_device](int i) {
    DevSelect ds(g->ctx[i]); if (!ds.ok) return 0;
    AMTK_CUDA(cudaEventSynchronize(g->marks[slot_b][i]));
    float ms = 0;
    AMTK_CUDA(cudaEventElapsedTime(&ms, g->marks[slot_a][i], g->marks[slot_b][i]));
    ms_per_device[i] = ms;
    return 1;
  });
}

// Frame-sharded LogoScan (SURVEY 8(e)): device i accumulates frames [frame0[i], frame0[i] + nframes[i]) of ITS copy of the
// clip into scans[i]; then ONE ncclAllReduce(ncclSum, ncclUint64) over the accumulators (5 x pixels sums folded into the
// 3 per-pixel u64 + 8 scalars the kernels keep) makes every device hold the whole-clip sums.  Exact: integer addition.
int amtk_group_scan_add_frames(amtk_group* g, amtk_scan* const* scans, const amtk_clip* clips, int scanx, int scany,
                               const int* frame0, const int* nframes) {
  if (!g || !scans || !clips || !frame0 || !nframes) AMTK_FAIL("amtk_group_scan_add_frames: bad argument");
  amtk::NcclApi& api = amtk::nccl_api();
  return amtk::group_run(g, [g, scans, clips, scanx, scany, frame0, nframes, &api](int i) {
    amtk_scan* s = scans[i];
    if (!s || s->ctx != g->ctx[i]) AMTK_FAIL("amtk_group_scan_add_frames: scans[i] must belong to the group's context i");
    if (clips[i].bytes_per_sample != 1) AMTK_FAIL("amtk_group_scan_add_frames: 8-bit clips only");
    if (nframes[i] > 0 && !amtk_scan_add_frames(s, &clips[i], scanx, scany, frame0[i], nframes[i], nullptr, nullptr)) return 0;
    DevSelect ds(g->ctx[i]); if (!ds.ok) return 0;
    if (g->ndev > 1) {
      cudaStream_t st = g->ctx[i]->stream;
      if (!amtk::nccl_ok(api.GroupStart(), "ncclGroupStart")) return 0;
      const bool a = amtk::nccl_ok(api.AllReduce(s->dSums, s->dSums, s->npix * 3, amtk::kNcclUint64, amtk::kNcclSum, g->comm[i], st), "ncclAllReduce(sums)");
      const bool b = amtk::nccl_ok(api.AllReduce(s->dBg, s->dBg, 8, amtk::kNcclUint64, amtk::kNcclSum, g->comm[i], st), "ncclAllReduce(bg)");
      if (!amtk::nccl_ok(api.GroupEnd(), "ncclGroupEnd") || !a || !b) return 0;
      unsigned long long nv = 0;
      AMTK_CUDA(cudaMemcpyAsync(&nv, s->dBg + 6, sizeof(nv), cudaMemcpyDeviceToHost, st));
      AMTK_CUDA(cudaStreamSynchronize(st));
      s->nvalid = (int)nv;
    }
    return 1;
  });
}

}  // extern "C"
