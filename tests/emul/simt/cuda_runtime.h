// tests/emul/simt/cuda_runtime.h — TEST HARNESS ONLY (never shipped, never a fallback of the product).
//
// A stand-in for <cuda_runtime.h> that lets g++ compile the UNMODIFIED kernels of youtokentome_b200/csrc
// (train.cu, encode.cu, merge_loop.cuh) and run them on the CPU under a SIMT emulator:
//   * every CUDA thread is a fiber (own stack, hand-written context switch, simt_emu.cpp);
//   * warp collectives (__shfl_*_sync, __ballot_sync, __syncwarp) and __syncthreads are rendezvous points of
//     the fibers of a warp / block; cooperative grid.sync() is a pthread barrier between blocks, each block of
//     a cooperative launch running on its own OS thread (so `__shared__` = static thread_local is per block);
//   * atomics are real atomics; mbarrier / cp.async.bulk are modelled in merge_loop.cuh under YT_SIMT_EMU.
// The build container has no GPU: this is how the control flow of the kernels (tile rings, barrier phases,
// claim bitmaps, vector scans) is exercised by `pytest -m "not gpu"`.  It says nothing about memory-ordering
// races or performance — the GPU tests do.
#pragma once
#define YT_SIMT_EMU 1
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <functional>
#include <type_traits>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static thread_local

struct uint2 { uint32_t x, y; };
struct __attribute__((aligned(16))) uint4 { uint32_t x, y, z, w; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

namespace emu {
struct Coords { dim3 tid, bid, bdim, gdim; unsigned lane; };
extern thread_local Coords *t_coords;  // of the running fiber
void yield();                            // let the other fibers of the block run (spin loops)
// rendezvous of the live lanes of the calling warp: returns the 32 contributed values (valid until the
// caller's next collective) and the mask of lanes that took part
const uint64_t *warp_gather(uint64_t v, uint32_t *live);
void block_sync();
void grid_sync();
void *dyn_smem();
void launch(unsigned grid, unsigned block, size_t smem, const std::function<void()> &body);
void launch_cooperative(unsigned grid, unsigned block, size_t smem, const std::function<void()> &body);
unsigned n_sm();
template <class T> inline uint64_t to_bits(T v) {
  static_assert(sizeof(T) <= 8 && std::is_trivially_copyable<T>::value, "shuffle of a wide type");
  uint64_t b = 0;
  memcpy(&b, &v, sizeof(T));
  return b;
}
template <class T> inline T from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
}  // namespace emu

#define threadIdx (emu::t_coords->tid)
#define blockIdx (emu::t_coords->bid)
#define blockDim (emu::t_coords->bdim)
#define gridDim (emu::t_coords->gdim)

// ---- warp / block primitives ---------------------------------------------------------------------
template <class T> inline T __shfl_sync(unsigned, T v, int src, int = 32) {
  uint32_t live;
  const uint64_t *g = emu::warp_gather(emu::to_bits(v), &live);
  return emu::from_bits<T>(g[src & 31]);
}
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned delta, int = 32) {
  uint32_t live;
  const uint64_t *g = emu::warp_gather(emu::to_bits(v), &live);
  const unsigned lane = emu::t_coords->lane;
  return lane >= delta ? emu::from_bits<T>(g[lane - delta]) : v;
}
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned delta, int = 32) {
  uint32_t live;
  const uint64_t *g = emu::warp_gather(emu::to_bits(v), &live);
  const unsigned lane = emu::t_coords->lane;
  return lane + delta < 32 ? emu::from_bits<T>(g[lane + delta]) : v;
}
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) {
  uint32_t live;
  const uint64_t *g = emu::warp_gather(emu::to_bits(v), &live);
  return emu::from_bits<T>(g[(emu::t_coords->lane ^ (unsigned)m) & 31]);
}
inline unsigned __ballot_sync(unsigned, int pred) {
  uint32_t live;
  const uint64_t *g = emu::warp_gather(pred ? 1u : 0u, &live);
  unsigned m = 0;
  for (int i = 0; i < 32; i++)
    if (((live >> i) & 1u) && g[i]) m |= 1u << i;
  return m;
}
inline unsigned __reduce_max_sync(unsigned, unsigned v) {
  uint32_t live;
  const uint64_t *g = emu::warp_gather((uint64_t)v, &live);
  unsigned m = 0;
  for (int i = 0; i < 32; i++)
    if (((live >> i) & 1u) && (unsigned)g[i] > m) m = (unsigned)g[i];
  return m;
}
inline void __syncwarp(unsigned = 0xffffffffu) { uint32_t live; emu::warp_gather(0, &live); }
inline void __syncthreads() { emu::block_sync(); }
inline int __syncthreads_or(int pred) {  // three rendezvous: previous readers are gone, the flag is cleared, all have voted
  static thread_local int acc;
  emu::block_sync();
  acc = 0;
  emu::block_sync();
  if (pred) acc = 1;
  emu::block_sync();
  return acc;
}
inline void __threadfence_block() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
inline unsigned __fns(unsigned mask, unsigned base, int offset) {  // offset-th set bit at or above `base` (offset >= 1)
  for (unsigned i = base; i < 32; i++)
    if ((mask >> i) & 1u)
      if (--offset == 0) return i;
  return 0xffffffffu;
}
template <class T> inline T __ldg(const T *p) { return *p; }
template <class T> inline T __ldcg(const T *p) { return *(const volatile T *)p; }
inline uint4 __ldcg(const uint4 *p) {
  const volatile uint32_t *q = reinterpret_cast<const volatile uint32_t *>(p);
  return uint4{q[0], q[1], q[2], q[3]};
}

template <class T, class U> inline T atomicAdd(T *p, U v) { return __atomic_fetch_add(p, (T)v, __ATOMIC_SEQ_CST); }
template <class T, class U> inline T atomicOr(T *p, U v) { return __atomic_fetch_or(p, (T)v, __ATOMIC_SEQ_CST); }
template <class T, class U> inline T atomicAnd(T *p, U v) { return __atomic_fetch_and(p, (T)v, __ATOMIC_SEQ_CST); }
template <class T, class U> inline T atomicExch(T *p, U v) { return __atomic_exchange_n(p, (T)v, __ATOMIC_SEQ_CST); }
template <class T, class U, class V> inline T atomicCAS(T *p, U cmp, V val) {
  T expected = (T)cmp;
  __atomic_compare_exchange_n(p, &expected, (T)val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}
template <class T, class U> inline T atomicMax(T *p, U v) {
  T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old < (T)v && !__atomic_compare_exchange_n(p, &old, (T)v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}

template <class T, class U> inline T atomicMin(T *p, U v) {
  T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old > (T)v && !__atomic_compare_exchange_n(p, &old, (T)v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}

// CUDA's overloaded ::min / ::max on mixed integer types
template <class A, class B> inline typename std::common_type<A, B>::type min(A a, B b) {
  typedef typename std::common_type<A, B>::type C;
  return (C)a < (C)b ? (C)a : (C)b;
}
template <class A, class B> inline typename std::common_type<A, B>::type max(A a, B b) {
  typedef typename std::common_type<A, B>::type C;
  return (C)a > (C)b ? (C)a : (C)b;
}

// ---- runtime API: one synchronous "device" whose memory is host memory ------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorPeerAccessAlreadyEnabled = 704 };
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, h.reserved, sizeof(*p)); return cudaSuccess; }
inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }
inline cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice,
                      cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount, cudaDevAttrMaxSharedMemoryPerBlockOptin };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize };
struct EmuStream { int unused; };
struct EmuEvent { double ms; };
typedef EmuStream *cudaStream_t;
typedef EmuEvent *cudaEvent_t;
inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr a, int) {
  *v = a == cudaDevAttrMultiProcessorCount ? (int)emu::n_sm() : 232448;  // 227 KB, as on sm_90a
  return cudaSuccess;
}
inline cudaError_t cudaMalloc(void **p, size_t n) {
  *p = aligned_alloc(256, (n + 255) / 256 * 256);
  if (!*p) return cudaErrorMemoryAllocation;
  memset(*p, 0xcd, n);  // poison: kernels must not rely on zeroed allocations
  return cudaSuccess;
}
template <class T> inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc((void **)p, n); }
inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
constexpr unsigned cudaHostAllocDefault = 0;   // "pinned" host memory is plain host memory here
inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { *p = malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) {
  memmove(d, s, n);
  return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = new EmuStream(); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new EmuEvent(); return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  e->ms = ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
  return cudaSuccess;
}
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->ms - a->ms); return cudaSuccess; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
template <class F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) {
  *n = 1;
  return cudaSuccess;
}

// kernel<<<g, b, s, st>>>(args...) is rewritten by build_emu.py into EMU_LAUNCH(kernel, g, b, s, st, args...)
#define EMU_LAUNCH(K, g, b, s, st, ...) emu::launch((unsigned)(g), (unsigned)(b), (size_t)(s), [=]() { K(__VA_ARGS__); })
