// Host-side launch helpers shared by every kernel file and the bindings: the launch check and counter, the dynamic
// shared-memory opt-in, and the dispatch of runtime values onto template arguments.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <mutex>
#include <set>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>

namespace pb {

// Kernels this process has enqueued (read by the bindings' launch_count); defined in bindings.cpp.
extern std::atomic<long long> g_launches;

// Call right after launching `n` kernels: raises the launch error, if any, otherwise counts the launches.
inline void launched(const char* name, int n = 1) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string(name) + " launch: " + cudaGetErrorString(e));
  g_launches += n;
}

// Lets `kernel` use `bytes` (its fixed size, above the default 48 KiB) of dynamic shared memory. The limit is an attribute of
// the kernel on one device, so it is raised once per (kernel, device). Safe to call from several host threads.
template <class Kernel>
void opt_in_smem(Kernel* kernel, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;   // (kernel, device)
  const void* k = reinterpret_cast<const void*>(kernel);
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  if (e == cudaSuccess && done.count({k, dev})) return;
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) throw std::runtime_error(std::string("dynamic shared memory opt-in: ") + cudaGetErrorString(e));
  done.insert({k, dev});
}

// f(std::bool_constant<b0>{}, std::bool_constant<b1>{}, ...): runtime flags as template arguments. Every combination of
// the flags is instantiated.
template <class F>
void with_bools(F&& f) {
  f();
}
template <class F, class... Rest>
void with_bools(F&& f, bool b, Rest... rest) {
  with_bools([&](auto... t) { !b ? f(std::false_type{}, t...) : f(std::true_type{}, t...); }, rest...);
}

// The LayerNorm kernels hold a row as N chunks of 256 elements: f(std::integral_constant<int, N>{}) with the least N of
// {1, 2, 3, 4, 6, 8, 10, 12, 16} that is >= nch, among those <= MAX. The caller has checked 1 <= nch <= MAX.
template <int MAX, int N, int... Rest, class F>
void with_ln_chunks_in(int nch, F& f) {
  if constexpr (N <= MAX) {
    if (nch <= N) return f(std::integral_constant<int, N>{});
    if constexpr (sizeof...(Rest) > 0) with_ln_chunks_in<MAX, Rest...>(nch, f);
  }
}
template <int MAX = 16, class F>
void with_ln_chunks(int nch, F&& f) {
  with_ln_chunks_in<MAX, 1, 2, 3, 4, 6, 8, 10, 12, 16>(nch, f);
}

}  // namespace pb
