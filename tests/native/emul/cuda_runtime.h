// cuda_runtime.h (TEST INFRASTRUCTURE) -- a small SIMT emulator that lets the engine's own
// kernel sources (maelstrom_b200/csrc/ms_kernels.cu, ms_engine.cu) be compiled with g++ and run
// on the CPU, so that `pytest -m "not gpu"` exercises the real kernel logic against the oracle.
//
// It is found before the CUDA toolkit's header only because tests/emul_lib.py puts this
// directory first on the include path and defines MS_EMUL.  Nothing in maelstrom_b200/ loads
// the resulting library: the product has no CPU path.
//
// Model: CTAs of a launch run one after another by default (the kernels never wait on a CTA that has not
// started; MS_EMUL_CTAS below runs them concurrently); the threads of a CTA are fibers switched cooperatively at __syncthreads() and at
// warp collectives (__shfl*_sync, __match_any_sync, __any_sync), which are evaluated when the
// last live lane arrives.  Lanes that reach different collectives abort the run (divergence
// check).  "Device" memory is host memory filled with 0xCD at allocation; IPC handles carry the
// raw pointer, so shards of one process can map each other.
//
// Streams are synchronous by default: every launch, copy and memset runs when it is enqueued.
// MS_EMUL_STREAMS=<seed> (or simt_streams(seed) at run time) makes them asynchronous: each stream
// is a FIFO of launches, async copies, memsets and event records; cudaStreamWaitEvent is a
// dependency on the recorded position; host synchronisation runs the queues up to the point it
// waits for (synchronous copies drain everything).  A seeded choice may start another stream's
// ready work first, and at a __syncthreads() of a running kernel may run another stream's ready
// work to completion while the CTA is parked (one nesting level).  So the journal stream of
// ms_run_streamed can read the state while a round of the next batch is half done.
//
// MS_EMUL_CTAS=<seed> (or simt_ctas(seed) at run time; -1 = off, the default) runs the CTAs of a launch of two or
// more concurrently: a pool of host threads per launching thread, 2 x MS_EMUL_SMS CTAs resident at once (one per
// thread, with its own fibers and, __shared__ being thread_local, its own shared memory), a finished CTA's thread
// taking the next block index.  A baton lets one thread run at a time, so a run is a function of the seed.  At a
// CTA's start, its first arrival at a __syncthreads(), every atomic*, __threadfence* and every spin-wait
// (__nanosleep / relax) a seeded choice may park the whole CTA and resume another; a parked CTA may be held for
// many switches.  All of them live in this directory: the kernel sources are compiled as they are.  Combined with MS_EMUL_STREAMS, nested stream work runs
// on the parked CTA's thread.  Stores still land in program order at once: no reordering between SMs.  The TSan
// build keeps sequential CTAs.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <functional>

#ifndef MS_EMUL
#error "tests/native/emul/cuda_runtime.h is only for -DMS_EMUL builds"
#endif

// ---------------------------------------------------------------- qualifiers
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __shared__ static thread_local
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

// ---------------------------------------------------------------- vector types
struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }

namespace simt {
struct Tls {
  uint3 tid;
  uint3 bid;
  dim3 bdim;
  dim3 gdim;
};
extern thread_local Tls tls;
void launch(unsigned grid, unsigned block, size_t dyn_smem, const std::function<void()>& body);
unsigned char* dyn_smem();
void sync_threads();
int sync_threads_or(int pred);
enum Op { OP_SHFL_UP = 1, OP_SHFL_XOR, OP_SHFL_IDX, OP_MATCH_ANY, OP_ANY, OP_BALLOT };
uint64_t warp_op(int op, unsigned mask, uint64_t v, int arg);
void relax();   // spin-wait hint: lets other host threads (shards) run
// MS_EMUL_CTAS: the places where a CTA of a concurrent launch may be parked for another one (simt.cpp)
enum Switch { SW_START, SW_BARRIER, SW_ATOMIC, SW_FENCE, SW_SPIN };
extern thread_local bool in_cta_pool;   // this host thread runs a CTA of a launch with several resident
void cta_switch(int why);
static inline void cta_point(int why) {
  if (in_cta_pool) cta_switch(why);
}
}  // namespace simt

#define threadIdx (simt::tls.tid)
#define blockIdx (simt::tls.bid)
#define blockDim (simt::tls.bdim)
#define gridDim (simt::tls.gdim)

// ---------------------------------------------------------------- intrinsics
static inline void __syncthreads() { simt::sync_threads(); }
static inline int __syncthreads_or(int p) { return simt::sync_threads_or(p); }
template <class T> static inline T __shfl_up_sync(unsigned m, T v, int d) {
  return (T)simt::warp_op(simt::OP_SHFL_UP, m, (uint64_t)v, d);
}
template <class T> static inline T __shfl_xor_sync(unsigned m, T v, int d) {
  return (T)simt::warp_op(simt::OP_SHFL_XOR, m, (uint64_t)v, d);
}
template <class T> static inline T __shfl_sync(unsigned m, T v, int lane) {
  return (T)simt::warp_op(simt::OP_SHFL_IDX, m, (uint64_t)v, lane);
}
static inline unsigned __match_any_sync(unsigned m, unsigned v) {
  return (unsigned)simt::warp_op(simt::OP_MATCH_ANY, m, v, 0);
}
static inline int __any_sync(unsigned m, int p) { return (int)simt::warp_op(simt::OP_ANY, m, p ? 1 : 0, 0); }
static inline unsigned __ballot_sync(unsigned m, int p) {
  return (unsigned)simt::warp_op(simt::OP_BALLOT, m, p ? 1 : 0, 0);
}
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) {
  return (unsigned long long)(((unsigned __int128)a * b) >> 64);
}
template <class T> static inline T __ldcg(const T* p) {
  T v;
  __builtin_memcpy(&v, (const void*)p, sizeof(T));   // a plain load (volatile does not copy structs)
  return v;
}
template <class T, class U> static inline void __stcg(T* p, U v) { *(volatile T*)p = (T)v; }
static inline void __threadfence() {
  simt::cta_point(simt::SW_FENCE);
  __atomic_thread_fence(__ATOMIC_SEQ_CST);
}
static inline void __threadfence_system() {
  simt::cta_point(simt::SW_FENCE);
  __atomic_thread_fence(__ATOMIC_SEQ_CST);
}
static inline void __nanosleep(unsigned) { simt::relax(); }
long long clock64();

template <class T, class U> static inline T atomicAdd(T* p, U v) {
  simt::cta_point(simt::SW_ATOMIC);
  return __atomic_fetch_add(p, (T)v, __ATOMIC_SEQ_CST);
}
template <class T, class U> static inline T atomicOr(T* p, U v) {
  simt::cta_point(simt::SW_ATOMIC);
  return __atomic_fetch_or(p, (T)v, __ATOMIC_SEQ_CST);
}
template <class T, class U> static inline T atomicMax(T* p, U v) {
  simt::cta_point(simt::SW_ATOMIC);
  T cur = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (cur < (T)v && !__atomic_compare_exchange_n(p, &cur, (T)v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return cur;
}
template <class T, class U, class V> static inline T atomicCAS(T* p, U cmp, V val) {
  simt::cta_point(simt::SW_ATOMIC);
  T expected = (T)cmp;
  __atomic_compare_exchange_n(p, &expected, (T)val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}

static inline int min(int a, int b) { return a < b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
static inline long min(long a, long b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }
static inline long max(long a, long b) { return a > b ? a : b; }

typedef struct simt_stream* cudaStream_t;

namespace simt {
// the arguments are evaluated and copied when the launch is enqueued, as a CUDA launch does
template <class K, class... A> static inline std::function<void()> bind_kernel(K k, A... a) {
  return [=]() { k(a...); };
}
void enqueue_launch(cudaStream_t s, const void* kern, unsigned grid, unsigned block, size_t dyn_smem,
                    std::function<void()> body);
}  // namespace simt

// kernel launch: MS_LAUNCH(kernel, grid, block, dynamic smem bytes, stream, args...).  Runs at once, or
// under MS_EMUL_STREAMS queues on its stream (simt.cpp).
#define MS_LAUNCH(kern, grid, block, smem, stream, ...)                                                 \
  simt::enqueue_launch((stream), (const void*)(kern), (unsigned)(grid), (unsigned)(block), (size_t)(smem), \
                       simt::bind_kernel(kern, __VA_ARGS__))

// ---------------------------------------------------------------- runtime API subset
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
typedef struct simt_event* cudaEvent_t;
typedef struct simt_graph* cudaGraph_t;
typedef struct simt_graph_exec* cudaGraphExec_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaIpcMemLazyEnablePeerAccess = 1 };
enum cudaStreamCaptureStatus { cudaStreamCaptureStatusNone = 0, cudaStreamCaptureStatusActive = 1 };
enum cudaStreamCaptureMode { cudaStreamCaptureModeGlobal = 0, cudaStreamCaptureModeThreadLocal = 1 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaIpcMemHandle_t { char reserved[64]; };
struct cudaDeviceProp {
  char name[256];
  int multiProcessorCount;
  size_t sharedMemPerBlockOptin;
  size_t totalGlobalMem;
  int major, minor;
};

const char* cudaGetErrorString(cudaError_t e);
cudaError_t cudaGetLastError();
cudaError_t cudaSetDevice(int);
cudaError_t cudaGetDeviceCount(int* n);
cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int dev);
cudaError_t cudaMalloc(void** p, size_t bytes);
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t bytes) { return cudaMalloc((void**)p, bytes); }
cudaError_t cudaFree(void* p);
enum { cudaHostAllocDefault = 0, cudaHostAllocPortable = 1, cudaHostAllocMapped = 2 };
static inline cudaError_t cudaHostAlloc(void** p, size_t bytes, unsigned) { *p = malloc(bytes); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind);
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr);
cudaError_t cudaMemset(void* d, int v, size_t n);
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr);
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned);
cudaError_t cudaStreamDestroy(cudaStream_t);
cudaError_t cudaStreamSynchronize(cudaStream_t);
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0);
cudaError_t cudaStreamIsCapturing(cudaStream_t, cudaStreamCaptureStatus*);
cudaError_t cudaStreamBeginCapture(cudaStream_t, cudaStreamCaptureMode);
cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t*);
cudaError_t cudaGraphInstantiate(cudaGraphExec_t*, cudaGraph_t, unsigned long long = 0);
cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t);
cudaError_t cudaGraphDestroy(cudaGraph_t);
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t);
cudaError_t cudaEventCreate(cudaEvent_t*);
cudaError_t cudaEventCreateWithFlags(cudaEvent_t*, unsigned);
cudaError_t cudaEventDestroy(cudaEvent_t);
cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr);
cudaError_t cudaEventSynchronize(cudaEvent_t);
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b);
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*);
cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned);
cudaError_t cudaIpcCloseMemHandle(void*);
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* nb, F, int, size_t) {
  *nb = 1;
  return cudaSuccess;
}
