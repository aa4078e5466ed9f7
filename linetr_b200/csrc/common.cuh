// Shared host/device utilities of the linetr_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace ltr {

// ---------------------------------------------------------------- error reporting
extern thread_local std::string g_last_error;
int set_error(int code, const std::string& msg);

#define LTR_CUDA_TRY(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess)                                                              \
      return ::ltr::set_error(-2, std::string(#expr) + ": " + cudaGetErrorString(_e));  \
  } while (0)

#define LTR_TRY(expr)        \
  do {                       \
    int _rc = (expr);        \
    if (_rc != 0) return _rc; \
  } while (0)

// ---------------------------------------------------------------- instrumentation
// Kernel classes for launch counting and per-class CUDA-event timing (ltr_profile_*).
enum KernelClass : int {
  KC_SMALL_MLP = 0,
  KC_LINEAR,
  KC_IMG_CONVERT,
  KC_SIG_ATTN,
  KC_FINAL_NORM,
  KC_DIST,
  KC_SEGMEAN,
  KC_ARGMIN,
  KC_MUTUAL,
  KC_TOKEN_FUSED,
  KC_TOKENIZE,
  KC_DESC_TILES,
  KC_MATCH_TC,
  KC_MATCH_EXACT,
  KC_MATCH_TAIL,
  KC_LINE_GT,
  KC_TRIPLET,
  KC_HOMOGRAPHY,
  KC_WARP,
  KC_ESSENTIAL,
  KC_PHOTOMETRIC,
  KC_FUNDAMENTAL,
  KC_ABSOLUTE_POSE,
  KC_TRIANGULATE,
  KC_TRACKS,
  KC_BUNDLE,
  KC_GLOBAL_POSES,
  KC_RETRIEVAL,
  KC_DEBUG,
  KC_COUNT
};
const char* kernel_class_name(int kc);

extern std::atomic<int64_t> g_launches;

// Threading contract of the C ABI: any number of host threads may call into the library
// concurrently (e.g. one thread per GPU); the process-wide state below is guarded by g_state_mutex.
// Per-class profiling (ltr_profile_*) is a process-wide switch: arm it, run, read it - from one thread.
extern std::mutex g_state_mutex;

struct Profiler {
  std::atomic<bool> on{false};
  struct Rec { int kc; cudaEvent_t a, b; };
  std::vector<Rec> recs;          // guarded by g_state_mutex
  std::vector<cudaEvent_t> pool;  // guarded by g_state_mutex
  cudaEvent_t get();
};
extern Profiler g_prof;

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device AND per kernel: the value set for each
// (kernel address, device) pair.  Guarded by g_state_mutex.
inline std::map<std::pair<const void*, int>, size_t>& smem_set() {
  static std::map<std::pair<const void*, int>, size_t> set;
  return set;
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// A kernel launched with pdl (programmaticStreamSerialization) may have its CTAs become resident as
// soon as SMs free up at the tail of the previous kernel and run their prologue (barrier init,
// constant staging) there; pdl_wait() then blocks until the
// previous grid has completed and flushed, BEFORE anything it produced is read or anything it
// still reads is overwritten.  pdl_launch_dependents() at kernel entry lets the next kernel do
// the same behind this one.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------- kernel launch
// Every kernel the library launches goes through this call, one call per launch, in kernel class kc:
//  - smem > 0: first raises the kernel's MaxDynamicSharedMemorySize on the current device to smem, unless smem_set()
//    already holds at least that.  Without it a kernel gets 48 KB of static and dynamic shared memory together, so a
//    kernel with static shared memory can need it below 48 KB of dynamic.  The encoder's sizes are constant, so no
//    attribute call happens after its first encode, graph captures included;
//  - pdl: launched with programmatic stream serialization (the kernel must call pdl_wait(), above);
//  - profiling armed (ltr_profile_begin): an event pair on s brackets exactly this launch;
//  - a successful launch is counted (ltr_launch_count).  A failed one is neither counted nor profiled, and returns
//    LTR_E_CUDA (-2) with "<class> launch: <CUDA error>"; the error is taken off the runtime's last-error state, so the
//    caller's next CUDA error check does not see it again.
template <typename... KArgs, typename... Args>
inline int launch(int kc, bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                  Args&&... args) {
  auto fail = [kc](cudaError_t e) {
    cudaGetLastError();
    return set_error(-2, std::string(kernel_class_name(kc)) + " launch: " + cudaGetErrorString(e));
  };
  if (smem > 0) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return fail(e);
    std::lock_guard<std::mutex> lk(g_state_mutex);
    size_t& set = smem_set()[{reinterpret_cast<const void*>(kernel), dev}];
    if (set < smem) {
      e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return fail(e);
      set = smem;
    }
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  Profiler::Rec r{kc, nullptr, nullptr};
  if (g_prof.on.load(std::memory_order_relaxed)) {
    std::lock_guard<std::mutex> lk(g_state_mutex);
    r.a = g_prof.get();
    r.b = g_prof.get();
  }
  if (r.a) cudaEventRecord(r.a, s);
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  if (r.a) {
    if (e == cudaSuccess) cudaEventRecord(r.b, s);
    std::lock_guard<std::mutex> lk(g_state_mutex);
    if (e == cudaSuccess) {
      g_prof.recs.push_back(r);
    } else {
      g_prof.pool.push_back(r.a);
      g_prof.pool.push_back(r.b);
    }
  }
  if (e != cudaSuccess) return fail(e);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

// ---------------------------------------------------------------- debug tracing (clock64 stamps of CTA 0)
__device__ unsigned long long g_dbg_trace[128];
__device__ int g_dbg_on = 0;
#define LTR_DBG_STAMP(slot)                                            \
  do {                                                                 \
    if (g_dbg_on && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) g_dbg_trace[slot] = clock64(); \
  } while (0)

// ---------------------------------------------------------------- device helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Lines of image i: [begin, end).  cu == nullptr means a uniform batch of lpi lines/image.
__device__ __forceinline__ void image_range(const int* __restrict__ cu, int lpi, int i, int& b, int& e) {
  if (cu) { b = cu[i]; e = cu[i + 1]; } else { b = i * lpi; e = b + lpi; }
}

// SMs of the current device (persistent grids size themselves by it)
inline int device_sm_count() {
  static std::atomic<int> sms[64];   // zero-initialised; benign duplicate queries, no torn state
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  int v = sms[dev].load(std::memory_order_relaxed);
  if (!v) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (v <= 0) v = 132;
    sms[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

}  // namespace ltr
