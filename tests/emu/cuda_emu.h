// cuda_emu.h — TEST-ONLY single-threaded CUDA emulator (fibers) for kernel-logic debugging on a box
// without a GPU.  It is never linked into the product library (libtcr_b200.so); tests/emu/Makefile builds
// the SAME kernel sources against this header into libtcr_emu.so, which only tests/ load.
//
// Model: blocks run sequentially; the threads of a block are ucontext fibers scheduled round-robin;
// __syncthreads/__syncwarp/shuffles are cooperative barriers.  Dynamic shared memory is poisoned with
// NaNs per block so uninitialised reads show up.  Memory-model bugs (races) are NOT caught here —
// that is what compute-sanitizer on the GPU box is for.
#pragma once
#include <ucontext.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#define TCR_EMU 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __constant__ static
#define __grid_constant__

struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct __attribute__((aligned(8))) float2 { float x, y; };
struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(8))) int2 { int x, y; };
struct __attribute__((aligned(16))) int4 { int x, y, z, w; };
struct __attribute__((aligned(16))) uint4 { unsigned x, y, z, w; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }

namespace emu {
struct ThreadCtx { uint3 tid; uint3 bid; unsigned char* smem; };
struct State {
  ThreadCtx* cur = nullptr;
  dim3 bdim, gdim;
  int last_error = 0;   // what cudaGetLastError returns (and clears): a launch the device would refuse
};
State& st();
// A launch whose grid or block CUDA would refuse (grid.x outside [1, 2^31 - 1], grid.y or grid.z outside [1, 65535], more than
// 1,024 threads or block.z > 64) runs nothing and returns cudaErrorInvalidConfiguration, which cudaGetLastError then reports.
int launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body);
int launch_cooperative(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body);   // all blocks co-resident
int launch_cluster(dim3 grid, dim3 block, size_t smem_bytes, unsigned cluster, const std::function<void()>& body);   // one cluster at a time
void gridsync();
unsigned cluster_rank();
unsigned cluster_size();
void cluster_sync();                                  // barrier over the CTAs of the running cluster
const void* dsmem(const void* local, unsigned rank);  // same offset in the shared memory of CTA `rank`
void syncthreads();
void syncwarp();
uint64_t warp_exchange(uint64_t v, int src_lane);   // every lane posts v, returns lane src_lane's value
unsigned ballot(int pred);
int lane_id();
}  // namespace emu

#define threadIdx (emu::st().cur->tid)
#define blockIdx (emu::st().cur->bid)
#define blockDim (emu::st().bdim)
#define gridDim (emu::st().gdim)
#define warpSize 32

static inline void __syncthreads() { emu::syncthreads(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::syncwarp(); }
static inline void __threadfence() {}
static inline void __threadfence_system() {}
static inline void __nanosleep(unsigned) {}
static inline void __threadfence_block() {}

template <class T> static inline uint64_t emu_bits(T v) { uint64_t b = 0; std::memcpy(&b, &v, sizeof(T)); return b; }
template <class T> static inline T emu_unbits(uint64_t b) { T v; std::memcpy(&v, &b, sizeof(T)); return v; }
template <class T> static inline T __shfl_sync(unsigned, T v, int src, int width = 32) {
  int lane = emu::lane_id();
  int base = lane - (lane % width);
  return emu_unbits<T>(emu::warp_exchange(emu_bits(v), base + (src % width)));
}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int width = 32) {
  int lane = emu::lane_id();
  int src = lane ^ m;
  if (src / width != lane / width) src = lane;
  return emu_unbits<T>(emu::warp_exchange(emu_bits(v), src));
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, int d, int width = 32) {
  int lane = emu::lane_id();
  int src = lane + d;
  if (src / width != lane / width) src = lane;
  return emu_unbits<T>(emu::warp_exchange(emu_bits(v), src));
}
template <class T> static inline T __shfl_up_sync(unsigned, T v, int d, int width = 32) {
  int lane = emu::lane_id();
  int src = lane - d;
  if (src < 0 || src / width != lane / width) src = lane;
  return emu_unbits<T>(emu::warp_exchange(emu_bits(v), src));
}
static inline unsigned __ballot_sync(unsigned, int pred) { return emu::ballot(pred); }

template <class T> static inline T atomicAdd(T* p, T v) { T old = *p; *p = old + v; return old; }
static inline unsigned atomicInc(unsigned* p, unsigned lim) { unsigned old = *p; *p = (old >= lim) ? 0 : old + 1; return old; }
template <class T> static inline T atomicExch(T* p, T v) { T old = *p; *p = v; return old; }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
template <class T> static inline T __ldcv(const T* p) { return *p; }
static inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }   // no contraction into an fma
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline unsigned __float_as_uint(float f) { return emu_unbits<unsigned>(emu_bits(f)); }
static inline float __uint_as_float(unsigned u) { return emu_unbits<float>(u); }
static inline float __int_as_float(int u) { return emu_unbits<float>((unsigned)u); }
static inline double __longlong_as_double(long long v) { return emu_unbits<double>((uint64_t)v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
static inline float __saturatef(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }
using std::fmaf;
using std::fmaxf;
using std::fminf;
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline size_t min(size_t a, size_t b) { return a < b ? a : b; }
static inline size_t max(size_t a, size_t b) { return a > b ? a : b; }

// ---- minimal runtime API (host memory stands in for device memory) ----
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidConfiguration = 9 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaErrorInvalidConfiguration ? "invalid configuration argument" : "emu"; }
static inline cudaError_t cudaGetLastError() {
  const cudaError_t e = emu::st().last_error;
  emu::st().last_error = cudaSuccess;
  return e;
}
static inline cudaError_t cudaPeekAtLastError() { return emu::st().last_error; }
static inline cudaError_t cudaMalloc(void** p, size_t n) {
  if (posix_memalign(p, 256, n ? n : 256) != 0) return cudaErrorMemoryAllocation;
  std::memset(*p, 0xFF, n);  // poison
  return cudaSuccess;
}
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { std::memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { std::memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
// streams and events: everything runs synchronously in the emulator, so these are bookkeeping no-ops
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = nullptr; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = (cudaEvent_t)1; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }

namespace tcr { void pdl_chain_reset(); }
#define TCR_LAUNCH(name, kernel, grid, block, smem, stream, ...) \
  emu::launch((grid), (block), (smem), [&]() { kernel(__VA_ARGS__); })
#define TCR_DYNAMIC_SMEM(name) unsigned char* name = emu::st().cur->smem
#define TCR_LAUNCH_CLUSTER(name, kernel, grid, block, smem, stream, cluster, ...) \
  emu::launch_cluster((grid), (block), (smem), (cluster), [&]() { kernel(__VA_ARGS__); })
#define TCR_LAUNCH_COOP(name, kernel, grid, block, smem, stream, arg) \
  emu::launch_cooperative((grid), (block), (smem), [&]() { kernel(arg); })
