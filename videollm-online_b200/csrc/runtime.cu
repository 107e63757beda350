// Process-wide runtime bits of libvlo_b200.so: thread-local error text, launch counter and the
// optional per-kernel-class CUDA-event profiler bench.py uses for its roofline numbers.
#include <atomic>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.h"

namespace vlo {

static thread_local std::string g_err;
void set_error(const std::string& m) { g_err = m; }
const char* last_error() { return g_err.c_str(); }
int fail(const std::string& m) {
  set_error(m);
  return -1;
}

bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("VLO_NO_PDL");
    on = (e != nullptr && e[0] == '1') ? 0 : 1;
  }
  // event-bracketed profiling wants serialised kernels: the per-class times then add up to the step
  return on == 1 && !prof_on();
}

// SMs of the current device (132 on an H100 SXM): persistent grids and split planning size themselves by it
int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

int ensure_max_smem(const void* func, int bytes) {
  static std::mutex mu;
  static std::vector<std::pair<int, const void*>> done;
  int dev = 0;
  VLO_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> g(mu);
  for (const auto& d : done)
    if (d.first == dev && d.second == func) return 0;
  VLO_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.emplace_back(dev, func);
  return 0;
}

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches += n; }
long long launch_count() { return g_launches.load(); }

// ---- profiler: one (start, stop) event pair per bracketed launch, recorded on the launching stream
namespace {
struct Rec {
  cudaEvent_t a, b;
  int cls;
  double bytes;
};
std::mutex g_pmu;
bool g_prof = false;
std::vector<Rec> g_recs;
std::vector<cudaEvent_t> g_pool;
int g_open = -1;

cudaEvent_t take_event() {
  if (!g_pool.empty()) {
    cudaEvent_t e = g_pool.back();
    g_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
}  // namespace

void prof_enable(bool on) {
  std::lock_guard<std::mutex> g(g_pmu);
  g_prof = on;
}
bool prof_on() { return g_prof; }

void prof_begin(int cls, cudaStream_t st, double algo_bytes) {
  if (!g_prof) return;
  std::lock_guard<std::mutex> g(g_pmu);
  Rec r{take_event(), take_event(), cls, algo_bytes};
  cudaEventRecord(r.a, st);
  g_recs.push_back(r);
  g_open = static_cast<int>(g_recs.size()) - 1;
}
void prof_end(cudaStream_t st) {
  if (!g_prof) return;
  std::lock_guard<std::mutex> g(g_pmu);
  if (g_open >= 0) cudaEventRecord(g_recs[g_open].b, st);
  g_open = -1;
}
// Sums per class since the last read; synchronises on the recorded events.
int prof_read(double* ms, long long* n, double* bytes, int ncls) {
  std::lock_guard<std::mutex> g(g_pmu);
  for (int i = 0; i < ncls; ++i) {
    ms[i] = 0;
    n[i] = 0;
    bytes[i] = 0;
  }
  for (Rec& r : g_recs) {
    float t = 0.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess &&
        r.cls >= 0 && r.cls < ncls) {
      ms[r.cls] += t;
      n[r.cls] += 1;
      bytes[r.cls] += r.bytes;
    }
    g_pool.push_back(r.a);
    g_pool.push_back(r.b);
  }
  g_recs.clear();
  cudaGetLastError();
  return 0;
}

}  // namespace vlo
