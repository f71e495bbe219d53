// tcr_device.cuh — device-side helpers shared by all kernels of libtcr_b200 (sm_90a).
// The TCR_EMU branch only exists so tests/emu can run the same kernel logic on a CPU box;
// the product library is always built by nvcc without TCR_EMU.
#pragma once

#ifdef TCR_EMU
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#include <stdint.h>
namespace tcr {
void prof_begin(const char* name, cudaStream_t s);   // tcr_prof.cu: launch counter + optional CUDA-event bracket
void prof_end(cudaStream_t s);
}
namespace tcr {
bool pdl_enabled();                                   // tcr_prof.cu: env TCR_PDL (default on), false for the first launch of a call
void pdl_chain_reset();                               // called at every API entry point
// Every kernel of the library is launched with programmatic stream serialization: its CTAs may become resident and
// run their producer-independent prologue (mbarrier init, filter-bank TMA, smem padding) while the previous kernel
// drains; pdl_wait() (griddepcontrol.wait) is the point after which the previous kernel's results may be read.
// Every kernel calls pdl_wait() exactly once on every path, so completion is transitive along the stream.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, unsigned cluster,
                             Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (cluster > 1) {                // thread-block cluster along x: grid.x must be a multiple of `cluster`
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
}  // namespace tcr
// Opt a kernel in to `smem` bytes of dynamic shared memory; the attribute is per device, so is the cache (one per call site).
struct SmemOptIn {
  size_t limit[32];
  SmemOptIn() { for (auto& l : limit) l = 32 * 1024; }   // static smem counts against the 48 KB default
  template <typename K>
  cudaError_t ensure(K kernel, size_t smem) {
    int dev = 0;
    cudaGetDevice(&dev);
    size_t& lim = limit[dev & 31];
    if (smem <= lim) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) lim = smem;
    return e;
  }
};
// cluster launch: CTAs of a cluster share partial BatchNorm sums through distributed shared memory
#define TCR_LAUNCH_CLUSTER(name, kernel, grid, block, smem, stream, cluster, ...)                                   \
  do {                                                                                                              \
    tcr::prof_begin((name), (cudaStream_t)(stream));                                                                \
    tcr::launch_ex(kernel, dim3(grid), dim3(block), (size_t)(smem), (cudaStream_t)(stream), (unsigned)(cluster), __VA_ARGS__); \
    tcr::prof_end((cudaStream_t)(stream));                                                                          \
  } while (0)
#define TCR_LAUNCH(name, kernel, grid, block, smem, stream, ...)                                          \
  do {                                                                                                    \
    tcr::prof_begin((name), (cudaStream_t)(stream));                                                      \
    tcr::launch_ex(kernel, dim3(grid), dim3(block), (size_t)(smem), (cudaStream_t)(stream), 1u, __VA_ARGS__); \
    tcr::prof_end((cudaStream_t)(stream));                                                                \
  } while (0)
#define TCR_DYNAMIC_SMEM(name) extern __shared__ __align__(1024) unsigned char name[]
// cooperative launch (all CTAs co-resident): kernel arguments are packed into an array of pointers
#define TCR_LAUNCH_COOP(name, kernel, grid, block, smem, stream, arg)                                                  \
  do {                                                                                                                 \
    tcr::prof_begin((name), (cudaStream_t)(stream));                                                                   \
    void* coop_args_[] = {(void*)&(arg)};                                                                              \
    cudaLaunchCooperativeKernel((const void*)(kernel), (grid), (block), coop_args_, (smem), (cudaStream_t)(stream));   \
    tcr::prof_end((cudaStream_t)(stream));                                                                             \
  } while (0)
#endif

namespace tcr {

// CUDA's bound on gridDim.y and gridDim.z.  Kernels with one utterance (or stream) per blockIdx.y are launched in slices of at
// most this many rows, with the row pointers offset on the host, so any batch a handle accepts runs.
constexpr int kMaxGridRows = 65535;

// programmatic dependent launch (see launch_pdl): no-ops in a kernel that was launched without the attribute
__device__ __forceinline__ void pdl_wait() {
#ifndef TCR_EMU
  asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_trigger() {
#ifndef TCR_EMU
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}

// ---- thread-block cluster primitives (a kernel launched without a cluster dimension is a cluster of one CTA) ----
#ifndef TCR_EMU
__device__ __forceinline__ unsigned cluster_ctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned cluster_nctarank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
// all threads of all CTAs of the cluster; release/acquire: shared-memory writes before it are visible cluster-wide after it
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// read a float at the same shared-memory offset in CTA `rank` of the cluster (distributed shared memory)
__device__ __forceinline__ float ld_dsmem(const float* local, unsigned rank) {
  const uint32_t la = (uint32_t)__cvta_generic_to_shared(local);
  uint32_t ra;
  float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(ra) : "memory");
  return v;
}
// the same offset in all 8 CTAs of a cluster, summed in rank order: one asm block so the 8 loads are in flight together
__device__ __forceinline__ float sum_dsmem8(const float* local) {
  const uint32_t la = (uint32_t)__cvta_generic_to_shared(local);
  float v0, v1, v2, v3, v4, v5, v6, v7;
  asm volatile(
      "{\n\t.reg .u32 a0, a1, a2, a3, a4, a5, a6, a7;\n\t"
      "mapa.shared::cluster.u32 a0, %8, 0;\n\tmapa.shared::cluster.u32 a1, %8, 1;\n\t"
      "mapa.shared::cluster.u32 a2, %8, 2;\n\tmapa.shared::cluster.u32 a3, %8, 3;\n\t"
      "mapa.shared::cluster.u32 a4, %8, 4;\n\tmapa.shared::cluster.u32 a5, %8, 5;\n\t"
      "mapa.shared::cluster.u32 a6, %8, 6;\n\tmapa.shared::cluster.u32 a7, %8, 7;\n\t"
      "ld.shared::cluster.f32 %0, [a0];\n\tld.shared::cluster.f32 %1, [a1];\n\t"
      "ld.shared::cluster.f32 %2, [a2];\n\tld.shared::cluster.f32 %3, [a3];\n\t"
      "ld.shared::cluster.f32 %4, [a4];\n\tld.shared::cluster.f32 %5, [a5];\n\t"
      "ld.shared::cluster.f32 %6, [a6];\n\tld.shared::cluster.f32 %7, [a7];\n\t}"
      : "=f"(v0), "=f"(v1), "=f"(v2), "=f"(v3), "=f"(v4), "=f"(v5), "=f"(v6), "=f"(v7)
      : "r"(la)
      : "memory");
  return ((((((v0 + v1) + v2) + v3) + v4) + v5) + v6) + v7;
}
#else
__device__ __forceinline__ unsigned cluster_ctarank() { return emu::cluster_rank(); }
__device__ __forceinline__ unsigned cluster_nctarank() { return emu::cluster_size(); }
__device__ __forceinline__ void cluster_sync_all() { emu::cluster_sync(); }
__device__ __forceinline__ float ld_dsmem(const float* local, unsigned rank) { return *reinterpret_cast<const float*>(emu::dsmem(local, rank)); }
__device__ __forceinline__ float sum_dsmem8(const float* local) {
  float s = 0.f;
  for (unsigned q = 0; q < 8; ++q) s += ld_dsmem(local, q);
  return s;
}
#endif

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float2 ld2(const float* p) { return *reinterpret_cast<const float2*>(p); }
// L2-coherent loads for per-channel tables written earlier in the SAME launch (persistent kernel): never the .nc path
__device__ __forceinline__ float4 ldc4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float ldc1(const float* p) { return __ldcg(p); }

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

// ------------------------------------------------------------------------------------------
// TMA (bulk async copy) + mbarrier.  SASS: UBLKCP / SYNCS.  1-D bulk copies need 16-byte aligned
// source, destination and size.
// ------------------------------------------------------------------------------------------
#ifndef TCR_EMU
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
#else
__device__ __forceinline__ void mbar_init(uint64_t*, int) {}
__device__ __forceinline__ void mbar_expect_tx(uint64_t*, uint32_t) {}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t*) { memcpy(dst, src, bytes); }
__device__ __forceinline__ void mbar_wait(uint64_t*, uint32_t) { __syncthreads(); }  // all threads call it
#endif

// mbarrier state carried across uses: a standalone kernel initialises it on first use; the persistent step kernel
// initialises once and flips `parity` after every completed transaction phase.
struct MbarCtx { uint64_t* bar; uint32_t parity; bool ready; };
#ifndef TCR_EMU
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#else
__device__ __forceinline__ void fence_proxy_async() {}
#endif

// Grid-wide barrier for the cooperative (co-resident) persistent kernel: monotonically increasing arrival counter,
// zeroed by the host before the launch.  Same fence/atomic/spin pattern as cooperative_groups::grid::sync().
#ifndef TCR_EMU
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned nblocks, unsigned& epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ++epoch;
    __threadfence();
    atomicAdd(counter, 1u);
    const unsigned target = epoch * nblocks;
    unsigned v;
    for (;;) {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (v >= target) break;
      __nanosleep(200);          // back off: hundreds of CTAs polling one L2 line starve the CTAs that still work
    }
    __threadfence();
  }
  __syncthreads();
}
#else
__device__ __forceinline__ void grid_barrier(unsigned*, unsigned, unsigned& epoch) { ++epoch; emu::gridsync(); }
#endif

// Debug timeline: thread 0 of a CTA stamps %globaltimer (ns) into tl[cta * 8 + slot] when tl != nullptr.
#ifndef TCR_EMU
__device__ __forceinline__ void tl_stamp(long long* tl, int cta, int slot) {
  if (tl && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    tl[(size_t)cta * 8 + slot] = (long long)t;
  }
}
#else
__device__ __forceinline__ void tl_stamp(long long*, int, int) {}
#endif

// Counter-based RNG for dropout and the resident dataset's augmentation draws (TF's RNG is not reproducible; parity runs
// inject a mask instead): SplitMix64's output for the state seed + golden * (idx + 1).
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t seed, uint64_t idx) {
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (idx + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ float uniform01(uint64_t z) { return (float)(z >> 40) * (1.0f / 16777216.0f); }   // [0,1), 24 bits
__device__ __forceinline__ float uniform01(uint64_t seed, uint64_t idx) { return uniform01(splitmix64(seed, idx)); }

}  // namespace tcr
