// zk_launch.cuh — task launcher and device-memory helpers.
//
// CUDA build (the product): every task runs as one thread of `zk_task_kernel<Task>` on the
// library's stream; there is NO CPU execution path in that build.
// ZKA_HOSTSIM build (tests only, compiled with g++ by __graft_entry__.build_hostsim): the same task
// bodies are executed by a plain loop so the arithmetic/layout logic can be unit-tested in
// the GPU-less CI container.  It is never part of libzkattest.so.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <stdexcept>
#include <string>
#include <typeinfo>
#include <vector>

#include <cxxabi.h>

#if !defined(ZKA_HOSTSIM)
#include <cuda_runtime.h>
#endif

namespace zk {

#if !defined(ZKA_HOSTSIM)

#define ZK_CUDA_CHECK(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " + \
                               __FILE__ + ":" + std::to_string(__LINE__));                    \
  } while (0)

// resident CTAs per SM a task asks the register allocator for (specialise per task; default: no bound)
template <class Task>
struct TaskMinBlocks { static constexpr int value = 1; };

template <class Task>
__global__ void __launch_bounds__(128, TaskMinBlocks<Task>::value) zk_task_kernel(int n, Task task) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) task(t);
}

struct ProfEntry {
  uint64_t launches = 0;
  double ms = 0.0;
  uint64_t items = 0;
};
struct Stream {
  cudaStream_t s = nullptr;
  uint64_t launches = 0;
  // optional live profiling: one CUDA-event pair per launch on this stream
  bool profiling = false;
  struct Pending { const char* name; cudaEvent_t e0, e1; long long n; };
  std::vector<Pending> pending;
  std::map<std::string, ProfEntry> prof;
};

inline std::string demangle(const char* n) {
  int status = 0;
  char* d = abi::__cxa_demangle(n, nullptr, nullptr, &status);
  std::string r = (status == 0 && d) ? d : n;
  free(d);
  return r;
}
// fold finished event pairs into the per-task table (stream must be idle)
inline void prof_collect(Stream& st) {
  for (auto& p : st.pending) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, p.e0, p.e1);
    ProfEntry& e = st.prof[demangle(p.name)];
    e.launches++;
    e.ms += ms;
    e.items += (uint64_t)p.n;
    cudaEventDestroy(p.e0);
    cudaEventDestroy(p.e1);
  }
  st.pending.clear();
}

template <class Task>
inline void launch(Stream& st, long long n, const Task& task) {
  if (n <= 0) return;
  if (n > 0x7fffffffLL) throw std::runtime_error("launch too large");
  const int threads = 128;
  const int blocks = (int)((n + threads - 1) / threads);
  Stream::Pending pd{typeid(Task).name(), nullptr, nullptr, n};
  if (st.profiling) {
    ZK_CUDA_CHECK(cudaEventCreate(&pd.e0));
    ZK_CUDA_CHECK(cudaEventCreate(&pd.e1));
    ZK_CUDA_CHECK(cudaEventRecord(pd.e0, st.s));
  }
  zk_task_kernel<Task><<<blocks, threads, 0, st.s>>>((int)n, task);
  ZK_CUDA_CHECK(cudaGetLastError());
  if (st.profiling) {
    ZK_CUDA_CHECK(cudaEventRecord(pd.e1, st.s));
    st.pending.push_back(pd);
  }
  st.launches++;
}

inline void* dev_alloc(size_t bytes) {
  void* p = nullptr;
  ZK_CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 1));
  return p;
}
inline void dev_free(void* p) {
  if (p) cudaFree(p);
}
inline void copy_h2d(Stream& st, void* d, const void* h, size_t n) {
  if (n) ZK_CUDA_CHECK(cudaMemcpyAsync(d, h, n, cudaMemcpyDefault, st.s));
}
inline void copy_d2h(Stream& st, void* h, const void* d, size_t n) {
  if (n) ZK_CUDA_CHECK(cudaMemcpyAsync(h, d, n, cudaMemcpyDefault, st.s));
}
inline void copy_d2d(Stream& st, void* d, const void* s, size_t n) {
  if (n) ZK_CUDA_CHECK(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToDevice, st.s));
}
// strided rows: only the first `width` bytes of each of `height` rows cross PCIe
inline void copy_d2h_2d(Stream& st, void* h, size_t hpitch, const void* d, size_t dpitch, size_t width, size_t height) {
  if (width && height) ZK_CUDA_CHECK(cudaMemcpy2DAsync(h, hpitch, d, dpitch, width, height, cudaMemcpyDefault, st.s));
}
inline void dev_memset(Stream& st, void* d, int v, size_t n) {
  if (n) ZK_CUDA_CHECK(cudaMemsetAsync(d, v, n, st.s));
}
inline void sync(Stream& st) {
  ZK_CUDA_CHECK(cudaStreamSynchronize(st.s));
  if (!st.pending.empty()) prof_collect(st);
}
// auxiliary (copy) streams and the events that order them against the compute stream
struct Event { cudaEvent_t e = nullptr; };
inline void stream_create(Stream& st) {
  if (!st.s) ZK_CUDA_CHECK(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
}
inline void stream_destroy(Stream& st) {
  if (st.s) cudaStreamDestroy(st.s);
  st.s = nullptr;
}
inline void ev_record(Event& ev, Stream& st) {
  if (!ev.e) ZK_CUDA_CHECK(cudaEventCreateWithFlags(&ev.e, cudaEventDisableTiming));
  ZK_CUDA_CHECK(cudaEventRecord(ev.e, st.s));
}
inline void ev_wait(Stream& st, Event& ev) {   // no-op for an event that was never recorded
  if (ev.e) ZK_CUDA_CHECK(cudaStreamWaitEvent(st.s, ev.e, 0));
}
inline void ev_destroy(Event& ev) {
  if (ev.e) cudaEventDestroy(ev.e);
  ev.e = nullptr;
}
// is `p` a device-accessible pointer that kernels may dereference directly?
inline bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

#else  // ------------------------------------------------------------------ host simulator

struct ProfEntry {
  uint64_t launches = 0;
  double ms = 0.0;
  uint64_t items = 0;
};
struct Stream {
  uint64_t launches = 0;
  bool profiling = false;
  std::map<std::string, ProfEntry> prof;
};
template <class Task>
inline void launch(Stream& st, long long n, const Task& task) {
  for (long long t = 0; t < n; t++) task((int)t);
  st.launches++;
}
inline void* dev_alloc(size_t bytes) { return calloc(bytes ? bytes : 1, 1); }
inline void dev_free(void* p) { free(p); }
inline void copy_h2d(Stream&, void* d, const void* h, size_t n) { if (n) memcpy(d, h, n); }
inline void copy_d2h(Stream&, void* h, const void* d, size_t n) { if (n) memcpy(h, d, n); }
inline void copy_d2d(Stream&, void* d, const void* s, size_t n) { if (n) memcpy(d, s, n); }
inline void copy_d2h_2d(Stream&, void* h, size_t hpitch, const void* d, size_t dpitch, size_t width, size_t height) {
  for (size_t r = 0; r < height; r++) memcpy((char*)h + r * hpitch, (const char*)d + r * dpitch, width);
}
inline void dev_memset(Stream&, void* d, int v, size_t n) { if (n) memset(d, v, n); }
inline void sync(Stream&) {}
struct Event {};
inline void stream_create(Stream&) {}
inline void stream_destroy(Stream&) {}
inline void ev_record(Event&, Stream&) {}
inline void ev_wait(Stream&, Event&) {}
inline void ev_destroy(Event&) {}
inline bool is_device_ptr(const void*) { return false; }

#endif

// grow-only device buffer, freed when it goes out of scope
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { dev_free(p); }
  void release() {
    dev_free(p);
    p = nullptr;
    cap = 0;
  }
  template <class T>
  T* get(size_t count) {
    size_t bytes = count * sizeof(T);
    if (bytes > cap) {
      release();   // stays empty if the allocation throws
      size_t want = bytes + bytes / 8 + 256;
      p = dev_alloc(want);
      cap = want;
    }
    return reinterpret_cast<T*>(p);
  }
  // a buffer that will not grow (a multi-gigabyte table): no headroom
  template <class T>
  T* get_exact(size_t count) {
    release();
    p = dev_alloc(count * sizeof(T));
    cap = count * sizeof(T);
    return reinterpret_cast<T*>(p);
  }
};

// Hands out the buffers of a pool in call order.  A pipeline takes its buffers in the same order on every call (a
// buffer it does not need is taken at size 0), so each buffer of the pool keeps serving the same array and stops
// growing after the first calls.
struct Cursor {
  DevBuf *next_, *end_;
  template <size_t N>
  explicit Cursor(DevBuf (&pool)[N]) : next_(pool), end_(pool + N) {}
  DevBuf& next() {
    if (next_ == end_) throw std::runtime_error("workspace pool exhausted");
    return *next_++;
  }
  template <class T>
  T* take(size_t count) { return next().get<T>(count); }
  template <class T>   // null when not needed
  T* take_if(bool need, size_t count) {
    T* p = take<T>(need ? count : 0);
    return need ? p : nullptr;
  }
};

}  // namespace zk
