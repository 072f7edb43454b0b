// profile.cu -- optional per-kernel CUDA-event timing and a launch counter, host side only.
// bench.py uses this to measure the dominant kernel's average launch duration live, on the stream the kernels are
// launched on (torch.cuda.Event only sees torch's own ops), and to report how many of OUR kernels ran in the timed
// region.  Disabled by default: when off, a ProfScope costs one relaxed atomic increment.
#include <atomic>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace b2r {

int launch_priority(bool high) {
  struct Range {
    int least = 0, greatest = 0;
    Range() {
      if (cudaDeviceGetStreamPriorityRange(&least, &greatest) != cudaSuccess) least = greatest = 0;
      if (getenv("B2R_NO_PRIORITY")) greatest = least;  // A/B switch for measurements
    }
  };
  static const Range r;  // initialised once, thread-safely (forward and autograd-backward threads both launch)
  return high ? r.greatest : r.least;
}

// SM count of the CURRENT device (cached per device ordinal: one process may drive several GPUs)
int device_sm_count() {
  static std::atomic<int> cache[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;  // H100 SXM
    cache[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

static std::atomic<int> g_prof_on{0};
static std::atomic<unsigned long long> g_launches{0};
static std::mutex g_mu;
struct Pending { int id; cudaEvent_t a, b; };
static std::vector<Pending> g_pending;
static std::vector<cudaEvent_t> g_pool;
static double g_ms[B2R_NUM_KERNELS];
static unsigned long long g_cnt[B2R_NUM_KERNELS];

static cudaEvent_t get_event() {
  if (!g_pool.empty()) {
    cudaEvent_t e = g_pool.back();
    g_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

ProfScope::ProfScope(int id_, cudaStream_t st_, int launches) : id(id_), st(st_), on(g_prof_on.load(std::memory_order_relaxed) != 0) {
  g_launches.fetch_add((unsigned long long)launches, std::memory_order_relaxed);
  if (on) {
    std::lock_guard<std::mutex> lk(g_mu);
    a = get_event();
    cudaEventRecord(a, st);
  }
}

ProfScope::~ProfScope() {
  if (on) {
    std::lock_guard<std::mutex> lk(g_mu);
    cudaEvent_t b = get_event();
    cudaEventRecord(b, st);
    g_pending.push_back({id, a, b});
  }
}

static void drain_locked() {
  for (auto& p : g_pending) {
    cudaEventSynchronize(p.b);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) {
      g_ms[p.id] += ms;
      g_cnt[p.id] += 1;
    }
    g_pool.push_back(p.a);
    g_pool.push_back(p.b);
  }
  g_pending.clear();
}

}  // namespace b2r

using namespace b2r;

extern "C" {

void b2r_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!on) drain_locked();
  g_prof_on.store(on ? 1 : 0);
}

int b2r_profile_read(double* ms_sum, uint64_t* counts, int reset) {
  std::lock_guard<std::mutex> lk(g_mu);
  drain_locked();
  for (int i = 0; i < B2R_NUM_KERNELS; i++) {
    if (ms_sum) ms_sum[i] = g_ms[i];
    if (counts) counts[i] = g_cnt[i];
    if (reset) { g_ms[i] = 0.0; g_cnt[i] = 0; }
  }
  return B2R_NUM_KERNELS;
}

uint64_t b2r_launch_count(void) { return g_launches.load(); }

const char* b2r_kernel_name(int id) {
  static const char* names[B2R_NUM_KERNELS] = {"project", "tile_scan", "scatter", "sort_small", "sort_merge",
                                               "composite_fwd", "composite_bwd", "project_bwd", "misc"};
  return (id >= 0 && id < B2R_NUM_KERNELS) ? names[id] : "?";
}

}  // extern "C"