// TEST INFRASTRUCTURE: a small SIMT emulator, so that the engine's CUDA source (kernels AND host code,
// taichi_mpm_b200/csrc/mpmb_engine.cu + mpmb_math.cuh, transformed only at its launch and inline-PTX sites by
// tests/simt/build_simt.py) can run on a machine without a GPU.  One OS thread; every CUDA thread of a CTA is a
// coroutine (ucontext); CTAs run one after another.  __syncthreads / __syncwarp / shuffles / match / votes are real
// rendezvous points (a barrier nobody can complete is reported as a deadlock, not a hang); shared memory is the
// kernel's own `static` storage; atomics are plain operations; cp.async copies at once; device memory is host
// memory.  It checks kernel LOGIC — indexing, barriers, orderings, host orchestration — not timing, not memory-
// model races, not codegen.  Never part of the product.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <functional>
#include <vector>

#define MPMB_HOST_MATH 1
#define MPMB_SIMT_HOST 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __shared__ static
#define __launch_bounds__(...)
#define __restrict__ __restrict
#define __align__(n) __attribute__((aligned(n)))

// ---- vector types
struct alignas(8) float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct int2 { int x, y; };
struct int3 { int x, y, z; };
struct alignas(16) int4 { int x, y, z, w; };
struct uint3 { unsigned x, y, z; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
// PRMT: result byte k = byte sel[k] of the 8-byte value {y:x}
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
  unsigned long long v = ((unsigned long long)y << 32) | x;
  unsigned r = 0;
  for (int k = 0; k < 4; k++) r |= (unsigned)((v >> (8 * ((s >> (4 * k)) & 7))) & 0xff) << (8 * k);
  return r;
}
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float3 make_float3(float x, float y, float z) { return float3{x, y, z}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline int3 make_int3(int x, int y, int z) { return int3{x, y, z}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }

// packed fp32 intrinsics of sm_100 (crt/sm_100_rt.h): per component the scalar IEEE operation
static inline float2 __ffma2_rn(float2 x, float2 y, float2 z) { return float2{fmaf(x.x, y.x, z.x), fmaf(x.y, y.y, z.y)}; }
static inline float2 __fmul2_rn(float2 x, float2 y) { return float2{x.x * y.x, x.y * y.y}; }
static inline float2 __fadd2_rn(float2 x, float2 y) { return float2{x.x + y.x, x.y + y.y}; }

namespace simt {
struct Thread {
  ucontext_t ctx;
  char *stack = nullptr;
  int state = 0;  // 0 runnable, 1 at block barrier, 2 done
  unsigned tid = 0;
  int or_gen = 0;  // which of the block's two __syncthreads_or accumulators this thread uses next
};
struct Warp {
  // collective in flight: phase 0 = collecting, 1 = releasing
  int phase = 0;
  unsigned arrived = 0, released = 0, exited = 0;
  long long val[32];
};
struct Block {
  std::vector<Thread> th;
  std::vector<Warp> warps;
  unsigned n = 0, at_barrier = 0, done = 0;
  int or_acc[2] = {0, 0};
  std::function<void()> body;
  ucontext_t main;
  int cur = -1;
};
extern Block *g_blk;
extern uint3 g_threadIdx, g_blockIdx;
extern dim3 g_blockDim, g_gridDim;
extern void *g_shared_handles[1024];
extern unsigned g_shared_ctr;
extern long long g_clock;

void yield();                        // back to the scheduler
void run(unsigned grid, unsigned block, const std::function<void()> &body);
long long *warp_exchange(unsigned mask, long long v, unsigned *participants);  // returns the 32 deposited values
void warp_release(unsigned mask);
inline unsigned lane() { return g_threadIdx.x & 31u; }

inline void cp_async(unsigned handle, const void *src, int bytes) { memcpy(g_shared_handles[handle & 1023u], src, (size_t)bytes); }

template <class K>
struct Launch {
  K k;
  unsigned grid, block;
  template <class... A>
  void operator()(A... a) const {
    K kk = k;
    run(grid, block, [=]() { kk(a...); });
  }
};
template <class K, class G, class B, class S, class St>
inline Launch<K> make_launch(K k, G g, B b, S, St) { return Launch<K>{k, (unsigned)g, (unsigned)b}; }
}  // namespace simt
#define SIMT_LAUNCH(k, ...) simt::make_launch(k, __VA_ARGS__)

#define threadIdx simt::g_threadIdx
#define blockIdx simt::g_blockIdx
#define blockDim simt::g_blockDim
#define gridDim simt::g_gridDim

// ---- synchronisation and warp collectives
void __syncthreads();
int __syncthreads_or(int pred);
void __syncwarp(unsigned mask = 0xffffffffu);
static inline unsigned __activemask() { return 0u; }   // 0 = "whoever is here": collectives given it act per lane (see below)
static inline int __shfl_sync(unsigned mask, int v, int src) {
  unsigned part; long long *a = simt::warp_exchange(mask, v, &part); int r = (int)a[src & 31]; simt::warp_release(mask); return r;
}
static inline int __shfl_up_sync(unsigned mask, int v, unsigned d) {
  unsigned part; long long *a = simt::warp_exchange(mask, v, &part); unsigned l = simt::lane(); int r = l >= d ? (int)a[l - d] : v; simt::warp_release(mask); return r;
}
static inline int __shfl_down_sync(unsigned mask, int v, unsigned d) {
  unsigned part; long long *a = simt::warp_exchange(mask, v, &part); unsigned l = simt::lane(); int r = l + d < 32 ? (int)a[l + d] : v; simt::warp_release(mask); return r;
}
static inline int __shfl_xor_sync(unsigned mask, int v, int x) {
  unsigned part; long long *a = simt::warp_exchange(mask, v, &part); int r = (int)a[(simt::lane() ^ x) & 31]; simt::warp_release(mask); return r;
}
static inline unsigned __match_any_sync(unsigned mask, int v) {
  unsigned part; long long *a = simt::warp_exchange(mask, v, &part); unsigned m = 0;
  for (int i = 0; i < 32; i++) if ((part >> i & 1u) && (int)a[i] == v) m |= 1u << i;
  simt::warp_release(mask); return m;
}
static inline unsigned __ballot_sync(unsigned mask, int p) {
  unsigned part; long long *a = simt::warp_exchange(mask, p != 0, &part); unsigned m = 0;
  for (int i = 0; i < 32; i++) if ((part >> i & 1u) && a[i]) m |= 1u << i;
  simt::warp_release(mask); return m;
}
// with __activemask() (= 0 here) the caller only asks for a warp-uniform hint: the lane's own answer is a valid one
static inline int __any_sync(unsigned mask, int p) { return mask == 0u ? 1 : (__ballot_sync(mask, p) != 0u); }
static inline int __all_sync(unsigned mask, int p) { unsigned part; if (mask == 0u) return p != 0; unsigned b = __ballot_sync(mask, p); (void)part; return b == (mask & b) && b != 0u ? (b == mask) : 0; }
static inline int __reduce_max_sync(unsigned mask, int v) {
  if (mask == 0u) return v;
  unsigned part; long long *a = simt::warp_exchange(mask, v, &part); int r = v;
  for (int i = 0; i < 32; i++) if (part >> i & 1u) r = std::max(r, (int)a[i]);
  simt::warp_release(mask); return r;
}
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __clz(int x) { return x == 0 ? 32 : __builtin_clz((unsigned)x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }

// ---- atomics (one OS thread: plain operations)
template <class T> static inline T atomicAdd(T *p, T v) { T o = *p; *p = o + v; return o; }
static inline int atomicAdd(int *p, int v) { int o = *p; *p = o + v; return o; }
static inline unsigned atomicAdd(unsigned *p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline int atomicOr(int *p, int v) { int o = *p; *p = o | v; return o; }
static inline unsigned atomicOr(unsigned *p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
static inline int atomicMax(int *p, int v) { int o = *p; *p = std::max(o, v); return o; }
static inline int atomicMin(int *p, int v) { int o = *p; *p = std::min(o, v); return o; }
static inline unsigned long long atomicMin(unsigned long long *p, unsigned long long v) { unsigned long long o = *p; *p = std::min(o, v); return o; }
static inline int atomicExch(int *p, int v) { int o = *p; *p = v; return o; }
static inline int atomicCAS(int *p, int c, int v) { int o = *p; if (o == c) *p = v; return o; }

// ---- CUDA's global min / max
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline float min(float a, float b) { return fminf(a, b); }
static inline float max(float a, float b) { return fmaxf(a, b); }

// ---- scalar intrinsics
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
#define __expf(x) expf(x)
#define __logf(x) logf(x)
#define __fdividef(a, b) ((a) / (b))
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline unsigned __cvta_generic_to_shared(const void *p) { unsigned h = (simt::g_shared_ctr++) & 1023u; simt::g_shared_handles[h] = const_cast<void *>(p); return h; }
static inline void __threadfence() {}
static inline void __threadfence_system() {}
static inline void __threadfence_block() {}
static inline void __nanosleep(unsigned) {}
static inline long long clock64() { return simt::g_clock += 1000; }
static inline void __trap() { abort(); }
#ifndef isfinite
using std::isfinite;
#endif

// ---- runtime API (device memory = host memory, streams and events do nothing)
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
struct cudaDeviceProp { char name[256]; int multiProcessorCount; size_t totalGlobalMem; int major, minor; };
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
// live allocations are counted, and one allocation can be made to fail (simt_fail_allocation below), so that tests can check
// that every allocation is freed, on every error path too
namespace simt {
extern long long g_live_allocs;   // device allocations not freed yet
extern long long g_fail_in;       // > 0: the g_fail_in-th cudaMalloc from now fails
}
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) {
  if (simt::g_fail_in > 0 && --simt::g_fail_in == 0) return cudaErrorMemoryAllocation;
  void *q = nullptr;
  if (posix_memalign(&q, 256, n ? n : 256)) return cudaErrorMemoryAllocation;
  memset(q, 0xCD, n);
  *p = (T *)q;
  simt::g_live_allocs++;
  return cudaSuccess;
}
static inline cudaError_t cudaFree(void *p) {
  if (p) { free(p); simt::g_live_allocs--; }
  return cudaSuccess;
}
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t = nullptr) {
  for (size_t r = 0; r < h; r++) memcpy((char *)d + r * dp, (const char *)s + r * sp, w);
  return cudaSuccess;
}
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
// CUDA graphs do not exist on the emulator: stream creation for capture fails, which turns the engine's graph path off
typedef void *cudaGraph_t;
typedef void *cudaGraphExec_t;
enum { cudaStreamNonBlocking = 1, cudaStreamCaptureModeThreadLocal = 1 };
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *, unsigned) { return cudaErrorNotSupported; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamBeginCapture(cudaStream_t, int) { return cudaErrorNotSupported; }
static inline cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t *) { return cudaErrorNotSupported; }
static inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t *, cudaGraph_t, unsigned long long) { return cudaErrorNotSupported; }
static inline cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }
static inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
static inline cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) { return cudaErrorNotSupported; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { memset(p, 0, sizeof(*p)); strcpy(p->name, "simt-emulator"); p->multiProcessorCount = 2; p->totalGlobalMem = (size_t)8 << 30; p->major = 10; return cudaSuccess; }
template <class K> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, K, int, size_t) { *n = 2; return cudaSuccess; }
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = nullptr; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *, void *) { return cudaErrorNotSupported; }
static inline cudaError_t cudaIpcOpenMemHandle(void **, cudaIpcMemHandle_t, unsigned) { return cudaErrorNotSupported; }
static inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }
