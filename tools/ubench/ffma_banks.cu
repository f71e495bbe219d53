// Micro-benchmark: throughput of the 4x4 outer-product FFMA block (shared-memory operands) with float4 vs scalar accumulators.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ffma_banks ffma_banks.cu ; run on the GPU box.
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
extern "C" __global__ void __launch_bounds__(512,1) varA(int rows, int XS, int DS, float* out) {
  extern __shared__ float smem[];
  const int tid = threadIdx.x;
  for (int i = tid; i < 8192; i += 512) smem[i] = 1e-3f * i;
  __syncthreads();
  float4 acc[3][4];
  for (int j=0;j<3;++j) for (int i=0;i<4;++i) acc[j][i]=make_float4(0,0,0,0);
  int xrow = (tid&63)*4, drow = 4096 + (tid&63)*4;
  for (int r=0;r<rows;++r) {
    float4 d = ld4(smem+drow + (r&7)*DS), x[3];
    #pragma unroll
    for (int j=0;j<3;++j) x[j]=ld4(smem+xrow+((r&7)+j)*XS);
    #pragma unroll
    for (int j=0;j<3;++j) {
      acc[j][0].x=fmaf(x[j].x,d.x,acc[j][0].x); acc[j][0].y=fmaf(x[j].x,d.y,acc[j][0].y); acc[j][0].z=fmaf(x[j].x,d.z,acc[j][0].z); acc[j][0].w=fmaf(x[j].x,d.w,acc[j][0].w);
      acc[j][1].x=fmaf(x[j].y,d.x,acc[j][1].x); acc[j][1].y=fmaf(x[j].y,d.y,acc[j][1].y); acc[j][1].z=fmaf(x[j].y,d.z,acc[j][1].z); acc[j][1].w=fmaf(x[j].y,d.w,acc[j][1].w);
      acc[j][2].x=fmaf(x[j].z,d.x,acc[j][2].x); acc[j][2].y=fmaf(x[j].z,d.y,acc[j][2].y); acc[j][2].z=fmaf(x[j].z,d.z,acc[j][2].z); acc[j][2].w=fmaf(x[j].z,d.w,acc[j][2].w);
      acc[j][3].x=fmaf(x[j].w,d.x,acc[j][3].x); acc[j][3].y=fmaf(x[j].w,d.y,acc[j][3].y); acc[j][3].z=fmaf(x[j].w,d.z,acc[j][3].z); acc[j][3].w=fmaf(x[j].w,d.w,acc[j][3].w);
    }
  }
  for (int j=0;j<3;++j) for (int i=0;i<4;++i) st4(out + (((size_t)blockIdx.x*512+tid)*12+(j*4+i))*4, acc[j][i]);
}
extern "C" __global__ void __launch_bounds__(512,1) varB(int rows, int XS, int DS, float* out) {
  extern __shared__ float smem[];
  const int tid = threadIdx.x;
  for (int i = tid; i < 8192; i += 512) smem[i] = 1e-3f * i;
  __syncthreads();
  float acc[3][4][4];
  for (int j=0;j<3;++j) for (int i=0;i<4;++i) for (int c=0;c<4;++c) acc[j][i][c]=0.f;
  int xrow = (tid&63)*4, drow = 4096 + (tid&63)*4;
  for (int r=0;r<rows;++r) {
    float4 d4 = ld4(smem+drow + (r&7)*DS); float d[4]={d4.x,d4.y,d4.z,d4.w};
    float xx[3][4];
    #pragma unroll
    for (int j=0;j<3;++j) { float4 t=ld4(smem+xrow+((r&7)+j)*XS); xx[j][0]=t.x; xx[j][1]=t.y; xx[j][2]=t.z; xx[j][3]=t.w; }
    #pragma unroll
    for (int j=0;j<3;++j)
    #pragma unroll
      for (int c=0;c<4;++c)
    #pragma unroll
        for (int i=0;i<4;++i) acc[j][i][c]=fmaf(xx[j][i],d[c],acc[j][i][c]);
  }
  for (int j=0;j<3;++j) for (int i=0;i<4;++i) for (int c=0;c<4;++c) out[((size_t)blockIdx.x*512+tid)*48 + (j*4+i)*4+c] = acc[j][i][c];
}
// pure register FFMA chains: all operands even / mixed parity is up to ptxas; reference for the pipe rate
extern "C" __global__ void __launch_bounds__(512,1) varP(int rows, float* out) {
  float a[16]; for (int i=0;i<16;++i) a[i]=threadIdx.x*1e-3f+i;
  const float b=1.0000001f, c=1e-7f;
  for (int r=0;r<rows;++r) {
    #pragma unroll
    for (int k=0;k<3;++k)
    #pragma unroll
      for (int i=0;i<16;++i) a[i]=fmaf(a[i],b,c);
  }
  float s=0; for (int i=0;i<16;++i) s+=a[i];
  out[(size_t)blockIdx.x*512+threadIdx.x]=s;
}
int main() {
  float* out; cudaMalloc(&out, 132ull*512*48*4);
  cudaFuncSetAttribute(varA, cudaFuncAttributeMaxDynamicSharedMemorySize, 40000);
  cudaFuncSetAttribute(varB, cudaFuncAttributeMaxDynamicSharedMemorySize, 40000);
  cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int rows=4096;
  for (int rep=0; rep<3; ++rep) {
    float ms;
    cudaEventRecord(e0); varA<<<132,512,40000>>>(rows,52,52,out); cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms,e0,e1);
    printf("varA float4 acc : %.3f ms  -> %.2f cycles/FFMA/SMSP (at 1.965 GHz)\n", ms, ms*1e-3*1.965e9/(rows*48.0*4));
    cudaEventRecord(e0); varB<<<132,512,40000>>>(rows,52,52,out); cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms,e0,e1);
    printf("varB scalar acc : %.3f ms  -> %.2f cycles/FFMA/SMSP\n", ms, ms*1e-3*1.965e9/(rows*48.0*4));
    cudaEventRecord(e0); varP<<<132,512>>>(rows,out); cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms,e0,e1);
    printf("varP reg chains : %.3f ms  -> %.2f cycles/FFMA/SMSP\n", ms, ms*1e-3*1.965e9/(rows*48.0*4));
  }
  printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
