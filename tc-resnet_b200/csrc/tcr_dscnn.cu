// tcr_dscnn.cu — DS-CNN (Hello-Edge) forward pass for sm_90a: the reference's 2-D-conv comparison model
// (audio_nets/ds_cnn.py:20-118, BASELINE.json config 5), inference mode.
//
//   dscnn_conv_kernel      first layer: kh x kw conv from the single-channel feature map (+bias, BN, ReLU)
//   dscnn_dsblock_kernel   depthwise 3x3 (+bias, BN, ReLU) -> pointwise 1x1 (+bias, BN, ReLU) fused per tile of output rows:
//                          the input rows (+halo) and both filter banks are staged in shared memory, the depthwise result
//                          never leaves the SM, the pointwise conv is a register-tiled 4 positions x 4 channels contraction
//   dscnn_head_kernel      global average pool + fully connected (+bias) + softmax
// BatchNorm here has no gamma (slim default scale=False) and uses the moving statistics; bias + BN fold into one
// per-channel (scale, shift) pair computed while staging.
#ifndef TCR_EMU
#include <cuda.h>   // CUtensorMap (types only: the encoder is looked up through the runtime)
#endif
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <initializer_list>

#include "tcr_bn.cuh"
#include "tcr_net.h"

namespace tcr {

struct DsLayerDev {
  int type;                 // 0 conv, 1 separable
  int cin, cout, kh, kw, sh, sw, hin, win, hout, wout, pt, pl;
  int64_t w, b, beta, mm, mv;                // conv / depthwise
  int64_t pw, pb, pbeta, pmm, pmv;           // pointwise (separable only)
};

constexpr int kDsMaxLayers = 8;
struct DsNet {
  int nlayers, n, classes;
  DsLayerDev layer[kDsMaxLayers];
  int64_t fcw, fcb;
};

__device__ __forceinline__ void fold_bn(const float* p, int64_t b, int64_t beta, int64_t mm, int64_t mv, int c, float eps,
                                        float* scale, float* shift) {
  const float rstd = 1.0f / sqrtf(p[mv + c] + eps);
  scale[c] = rstd;
  shift[c] = (p[b + c] - p[mm + c]) * rstd + p[beta + c];
}
__device__ __forceinline__ float4 bn_relu4(float4 a, float4 s, float4 t) {
  return make_float4(fmaxf(fmaf(a.x, s.x, t.x), 0.f), fmaxf(fmaf(a.y, s.y, t.y), 0.f), fmaxf(fmaf(a.z, s.z, t.z), 0.f),
                     fmaxf(fmaf(a.w, s.w, t.w), 0.f));
}

// Input rows (with halo) and padded width of a tile of RH output rows.
TCR_HD inline int ds_in_rows(const DsLayerDev& L, int RH) { return (RH - 1) * L.sh + L.kh; }
TCR_HD inline int ds_in_cols(const DsLayerDev& L) { return (L.wout - 1) * L.sw + L.kw; }
TCR_HD inline int ds_tiles_per_utt(const DsLayerDev& L, int RH) { return (L.hout + RH - 1) / RH; }

// Shared-memory layout of one DS-CNN kernel, in floats.  The kernel carves its pointers from it; the host sizes the launch and
// checks its limits with the same function.  Regions: x the input tile(s) (xs floats per channel chunk, channel half or buffer,
// as the kernel describes), a the A operand ([buffers][hi, lo][K / 4][lba]) or the FMA block's depthwise output, b the B
// operand ([hi, lo][K / 4][gmma_lbb]) or an FMA kernel's filter bank, tab the per-channel tables, floats the total.
struct DsSmem { size_t x, a, b, tab, floats; int xs, lba; };
// The separable blocks' table region: depthwise taps [kh * kw][C], folded BatchNorm of the depthwise stage (sc1, sf1 [C]) and
// of the pointwise stage (sc2, sf2 [CO]).
struct DsTables { float *taps, *sc1, *sf1, *sc2, *sf2; };
TCR_HD inline size_t ds_tab_floats(int taps, int C, int CO) { return (size_t)taps * C + 2 * C + 2 * CO; }
__device__ __forceinline__ DsTables ds_stage_tables(float* base, const DsLayerDev& L, int taps, int C, int CO, const float* params,
                                                    float eps, int tid, int nthreads) {
  const DsTables t = {base, base + taps * C, base + taps * C + C, base + taps * C + 2 * C, base + taps * C + 2 * C + CO};
#pragma unroll 1  // at most one iteration per thread in the wgmma kernels; unrolled, the FMA block kernel spills
  for (int i = tid; i < taps * C / 4; i += nthreads) st4(t.taps + 4 * i, ldg4(params + L.w + 4 * i));
#pragma unroll 1
  for (int c = tid; c < C; c += nthreads) fold_bn(params, L.b, L.beta, L.mm, L.mv, c, eps, t.sc1, t.sf1);
#pragma unroll 1
  for (int c = tid; c < CO; c += nthreads) fold_bn(params, L.pb, L.pbeta, L.pmm, L.pmv, c, eps, t.sc2, t.sf2);
  return t;
}

// dscnn_conv_kernel, one utterance: x [hp][wp] (rounded to 4), b [kh * kw][cout], tab sc, sf [cout]
TCR_HD inline DsSmem conv_smem(const DsLayerDev& L) {
  DsSmem s = {};
  s.b = (ds_in_rows(L, L.hout) * ds_in_cols(L) + 3) & ~3;
  s.tab = s.b + (size_t)L.kh * L.kw * L.cout;
  s.floats = s.tab + 2 * L.cout;
  return s;
}
// dscnn_dsblock_kernel, RH output rows: x [hin_t][wp][C], a [RH * wout][C], b [C][COT] (a tile of COT output channels), tab
TCR_HD inline DsSmem dsblock_smem(const DsLayerDev& L, int RH, int COT) {
  DsSmem s = {};
  s.a = (size_t)ds_in_rows(L, RH) * ds_in_cols(L) * L.cin;
  s.b = s.a + (size_t)RH * L.wout * L.cin;
  s.tab = s.b + (size_t)L.cin * COT;
  s.floats = s.tab + ds_tab_floats(L.kh * L.kw, L.cin, L.cout);
  return s;
}

// ---- first layer: cin == 1 ----
__global__ void __launch_bounds__(256) dscnn_conv_kernel(DsLayerDev L, const float* __restrict__ params, const float* __restrict__ in,
                                                         float* __restrict__ out, float eps) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  const DsSmem S = conv_smem(L);
  const int hp = ds_in_rows(L, L.hout), wp = ds_in_cols(L);      // padded input extent
  float *xs = smem, *ws = smem + S.b, *sc = smem + S.tab, *sf = sc + L.cout;
  const int n = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < hp * wp; i += blockDim.x) {
    const int h = i / wp - L.pt, w = i % wp - L.pl;
    xs[i] = (h >= 0 && h < L.hin && w >= 0 && w < L.win) ? in[((size_t)n * L.hin + h) * L.win + w] : 0.f;
  }
  for (int i = tid; i < L.kh * L.kw * L.cout; i += blockDim.x) ws[i] = params[L.w + i];
  for (int c = tid; c < L.cout; c += blockDim.x) fold_bn(params, L.b, L.beta, L.mm, L.mv, c, eps, sc, sf);
  __syncthreads();
  const int c4n = L.cout >> 2, npos = L.hout * L.wout;
  for (int task = tid; task < npos * c4n; task += blockDim.x) {
    const int c4 = task % c4n, pos = task / c4n;
    const int oh = pos / L.wout, ow = pos - oh * L.wout;
    const float* xb = xs + oh * L.sh * wp + ow * L.sw;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < L.kh; ++i)
      for (int j = 0; j < L.kw; ++j) {
        const float x = xb[i * wp + j];
        const float4 w = ld4(ws + (i * L.kw + j) * L.cout + 4 * c4);
        acc.x = fmaf(x, w.x, acc.x); acc.y = fmaf(x, w.y, acc.y); acc.z = fmaf(x, w.z, acc.z); acc.w = fmaf(x, w.w, acc.w);
      }
    st4(out + ((size_t)n * npos + pos) * L.cout + 4 * c4, bn_relu4(acc, ld4(sc + 4 * c4), ld4(sf + 4 * c4)));
  }
}

// ---- depthwise-separable block, one CTA per (utterance, chunk of RH output rows) ----
constexpr int kDsTM = 4;
__global__ void __launch_bounds__(256) dscnn_dsblock_kernel(DsLayerDev L, int RH, int COT, const float* __restrict__ params,
                                                            const float* __restrict__ in, float* __restrict__ out, float eps) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  const int C = L.cin, CO = L.cout;
  const int n = blockIdx.y, h0 = blockIdx.x * RH, rh = imin(RH, L.hout - h0), tid = threadIdx.x;
  const int hin_t = ds_in_rows(L, RH), wp = ds_in_cols(L);      // staged input rows (with halo), padded width
  const DsSmem S = dsblock_smem(L, RH, COT);                     // COT = CO unless the bank exceeds shared memory: DS-CNN-L
  float *xs = smem, *ds = smem + S.a, *pws = smem + S.b;
  const int c4n = C >> 2;
  {
    const RowWalk w = row_walk(tid, blockDim.x, c4n);
    const int rows = hin_t * wp;
    if (w.row < rows) {
      int r = w.row / wp, col = w.row - r * wp;
      for (int row = w.row; row < rows; row += w.rstep) {
        const int h = h0 * L.sh - L.pt + r, x = col - L.pl;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h >= 0 && h < L.hin && x >= 0 && x < L.win) v = ld4(in + (((size_t)n * L.hin + h) * L.win + x) * C + 4 * w.c4);
        st4(xs + (size_t)row * C + 4 * w.c4, v);
        col += w.rstep;
        while (col >= wp) { col -= wp; ++r; }
      }
    }
  }
  auto load_slice = [&](int co0, int cot) {                      // pw[ci][co0 .. co0 + cot) -> pws[ci][COT]
    const int q4 = cot >> 2;
    for (int i = tid; i < C * q4; i += blockDim.x) {
      const int ci = i / q4, q = i - ci * q4;
      st4(pws + (size_t)ci * COT + 4 * q, ldg4(params + L.pw + (size_t)ci * CO + co0 + 4 * q));
    }
  };
  load_slice(0, imin(COT, CO));
  const DsTables T = ds_stage_tables(smem + S.tab, L, L.kh * L.kw, C, CO, params, eps, tid, blockDim.x);
  __syncthreads();
  // depthwise: thread owns 4 channels, walks output positions
  const int npos = rh * L.wout;
  {
    const RowWalk w = row_walk(tid, blockDim.x, c4n);
    if (w.row < npos) {
      const float4 s = ld4(T.sc1 + 4 * w.c4), t = ld4(T.sf1 + 4 * w.c4);
      int oh = w.row / L.wout, ow = w.row - oh * L.wout;
      for (int pos = w.row; pos < npos; pos += w.rstep) {
        const float* xb = xs + ((size_t)(oh * L.sh) * wp + ow * L.sw) * C + 4 * w.c4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = 0; i < L.kh; ++i)
          for (int j = 0; j < L.kw; ++j) {
            const float4 x = ld4(xb + ((size_t)i * wp + j) * C);
            const float4 k = ld4(T.taps + (i * L.kw + j) * C + 4 * w.c4);
            acc.x = fmaf(x.x, k.x, acc.x); acc.y = fmaf(x.y, k.y, acc.y); acc.z = fmaf(x.z, k.z, acc.z); acc.w = fmaf(x.w, k.w, acc.w);
          }
        st4(ds + (size_t)pos * C + 4 * w.c4, bn_relu4(acc, s, t));
        ow += w.rstep;
        while (ow >= L.wout) { ow -= L.wout; ++oh; }
      }
    }
  }
  __syncthreads();
  // pointwise: tasks of kDsTM positions x 4 output channels, positions of a task are NRT apart; one pass per tile of COT channels
  const int NRT = (npos + kDsTM - 1) / kDsTM;
  const size_t gbase = ((size_t)n * L.hout + h0) * L.wout;
  for (int co0 = 0; co0 < CO; co0 += COT) {
    const int cot = imin(COT, CO - co0), ncg = cot >> 2;
    if (co0 > 0) {
      __syncthreads();                                           // everybody is done with the previous slice
      load_slice(co0, cot);
      __syncthreads();
    }
    for (int task = tid; task < NRT * ncg; task += blockDim.x) {
      const int cg = task % ncg, rt = task / ncg;
      const float* xr[kDsTM];
#pragma unroll
      for (int i = 0; i < kDsTM; ++i) xr[i] = ds + (size_t)imin(rt + i * NRT, npos - 1) * C;
      float4 acc[kDsTM];
#pragma unroll
      for (int i = 0; i < kDsTM; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      const float* wk = pws + 4 * cg;
#pragma unroll 2
      for (int ci = 0; ci < C; ci += 4) {
        const float4 w0 = ld4(wk + (ci + 0) * COT), w1 = ld4(wk + (ci + 1) * COT), w2 = ld4(wk + (ci + 2) * COT), w3 = ld4(wk + (ci + 3) * COT);
#pragma unroll
        for (int i = 0; i < kDsTM; ++i) {
          const float4 x = ld4(xr[i] + ci);
          acc[i].x = fmaf(x.x, w0.x, acc[i].x); acc[i].y = fmaf(x.x, w0.y, acc[i].y); acc[i].z = fmaf(x.x, w0.z, acc[i].z); acc[i].w = fmaf(x.x, w0.w, acc[i].w);
          acc[i].x = fmaf(x.y, w1.x, acc[i].x); acc[i].y = fmaf(x.y, w1.y, acc[i].y); acc[i].z = fmaf(x.y, w1.z, acc[i].z); acc[i].w = fmaf(x.y, w1.w, acc[i].w);
          acc[i].x = fmaf(x.z, w2.x, acc[i].x); acc[i].y = fmaf(x.z, w2.y, acc[i].y); acc[i].z = fmaf(x.z, w2.z, acc[i].z); acc[i].w = fmaf(x.z, w2.w, acc[i].w);
          acc[i].x = fmaf(x.w, w3.x, acc[i].x); acc[i].y = fmaf(x.w, w3.y, acc[i].y); acc[i].z = fmaf(x.w, w3.z, acc[i].z); acc[i].w = fmaf(x.w, w3.w, acc[i].w);
        }
      }
      const float4 s = ld4(T.sc2 + co0 + 4 * cg), t = ld4(T.sf2 + co0 + 4 * cg);
#pragma unroll
      for (int i = 0; i < kDsTM; ++i) {
        const int pos = rt + i * NRT;
        if (pos < npos) st4(out + (gbase + pos) * CO + co0 + 4 * cg, bn_relu4(acc[i], s, t));
      }
    }
  }
}

// ---- depthwise-separable block with the pointwise 1x1 conv on the Hopper tensor cores (wgmma) ----
// The pointwise conv IS a dense [positions, C] x [C, CO] contraction (audio_nets/ds_cnn.py:56-59), 77 % of DS-CNN-S's FLOPs.
// Per tile: 128 accumulator rows (RH output rows x wout positions, RH * wout <= 128) x CO columns, held in the registers of the
// warpgroup(s) that issue the MMAs.
//   * single TF32 products miss the 1e-4 logit bound (6.7e-4 relative on a K = 64 dot product), so every operand is split
//     x = hi + lo with hi = x truncated to TF32 (low 13 mantissa bits cleared, lo = x - hi exact) and three MMAs accumulate
//     lo*hi + hi*lo + hi*hi in fp32: 4e-7 relative, the same as the FMA kernel;
//   * operands sit in shared memory in wgmma's K-major no-swizzle layout, element (row, k) at float offset
//     (k / 4) * LBO + row * 4 + k % 4: an 8-row core matrix is 128 contiguous bytes, 8-row groups are 128 B apart (SBO) and the
//     K-chunk stride LBO is padded by 16 B so that neither the depthwise stage's float4 stores nor the filter staging conflict;
//   * wgmma.mma_async m64nNk8 (TF32 operands, fp32 accumulators): one instruction covers 64 rows, K = 8 (two 4-wide chunks).
//     Thread (warp w of the warpgroup, lane l) holds rows 16 w + l / 4 and 16 w + l / 4 + 8, columns 8 j + 2 (l % 4) and + 1:
//     d[4 j + 2 h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e].
// The input rows are staged channel-chunk-major ([C/4][rows*wp][4]) so that lanes walking positions read conflict-free float4s.
#ifndef TCR_EMU
// wgmma shared-memory matrix descriptor: start address >> 4 in bits [0,14), leading (K-chunk) byte offset >> 4 in [16,30),
// stride (8-row group) byte offset >> 4 in [32,46); base offset 0 and layout type 0 (no swizzle) in the high bits.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 64] += A[64 x 8] B[64 x 8]^T, both operands K-major TF32 in shared memory
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db)
      : "memory");
}
// D[64 x 32] += A[64 x 8] B[32 x 8]^T
__device__ __forceinline__ void wgmma_m64n32k8_tf32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db)
      : "memory");
}
// Folded BatchNorm + ReLU of a warpgroup's accumulator fragment (NA instructions' worth of 64-row blocks, NJ 8-column groups)
// and the NHWC store: accumulator row m -> out[(gbase + m) * CO + col0 + column], rows >= npos are not stored.
template <int NA, int NJ>
__device__ __forceinline__ void gmma_epilogue(const float (&acc)[NA][4 * NJ], int m0, int col0, int CO, int npos, const float* sc,
                                              const float* sf, float* __restrict__ out, size_t gbase, int wtid) {
  const int r0 = m0 + 16 * (wtid >> 5) + ((wtid & 31) >> 2), c = 2 * (wtid & 3);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int co = col0 + 8 * j + c;
    const float2 s = ld2(sc + co), t = ld2(sf + co);
#pragma unroll
    for (int q = 0; q < 2 * NA; ++q) {                            // rows r0, r0 + 8, r0 + 64, r0 + 72
      const int m = r0 + 8 * (q & 1) + 64 * (q >> 1);
      if (m < npos) {
        const float* a = &acc[q >> 1][4 * j + 2 * (q & 1)];
        *reinterpret_cast<float2*>(out + (gbase + m) * CO + co) = make_float2(fmaxf(fmaf(a[0], s.x, t.x), 0.f), fmaxf(fmaf(a[1], s.y, t.y), 0.f));
      }
    }
  }
}
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
__device__ __forceinline__ void tf32_split(float4 v, float4& hi, float4& lo) {
  hi = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
  lo = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
}

__device__ __forceinline__ void cp_async16_zfill(float* dst_smem, const float* src, bool valid) {
  const uint32_t bytes = valid ? 16u : 0u;                        // src-size 0: the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "r"(bytes) : "memory");
}

constexpr int kTcThreads = 512;
constexpr int kWsProducerWarps = 10, kWsProducers = 32 * kWsProducerWarps, kWsConsumers = 128;
constexpr int kWsConsumerWarp0 = kTcThreads / 32 - 4;
constexpr int kLbaFull = 128 * 4 + 4;                             // K-chunk stride (floats) of a 128-row A operand, +16 B
TCR_HD constexpr int gmma_lbb(int co) { return co * 4 + 4; }     // K-chunk stride of the B operand
// Per-thread walks worked out once per kernel: dsblock_tc copies kDwCells input cells of its channel chunk per tile; the first
// conv's im2col walk copies kConvCells 4-byte input cells and gathers kConvTasks (position, tap chunk) operands per thread.
constexpr int kDwCells = 8, kConvCells = 4, kConvTasks = 4;

// Filter bank w[k][co] (K x CO) -> B operand [n = co][k] in the K-major layout, hi / lo parts; NB loads in flight per thread.
template <int NT, int CO, int NB>
__device__ __forceinline__ void stage_b(const float* __restrict__ w, int K, float* b_hi, float* b_lo, int tid) {
  constexpr int LBB = gmma_lbb(CO);
  for (int i0 = tid; i0 < K * CO; i0 += NT * NB) {
    float v[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) v[j] = i0 + NT * j < K * CO ? __ldg(w + i0 + NT * j) : 0.f;
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const int i = i0 + NT * j;
      if (i < K * CO) {
        const int k = i / CO, co = i - k * CO;
        const float hi = tf32_hi(v[j]);
        const int o = (k >> 2) * LBB + co * 4 + (k & 3);
        b_hi[o] = hi;
        b_lo[o] = v[j] - hi;
      }
    }
  }
}

// 3x3 / stride-1 depthwise + folded BN + ReLU of one (4-channel chunk, output column), sliding down the rows so that every input
// float4 is read once (3 loads per output instead of 9) and the 9 taps stay in registers: outputs [rb, re) of the tile.
// load(r, x) fetches the three taps of input row r; store(m, hi, lo) writes output row m's A operand.
template <class Load, class Store>
__device__ __forceinline__ void dw3_slide(int rb, int re, const float4 (&k)[9], float4 s, float4 t, Load load, Store store) {
  auto tap_row = [&](float4& acc, const float4 (&x)[3], int kr) {
    acc.x = fmaf(x[0].x, k[3 * kr].x, fmaf(x[1].x, k[3 * kr + 1].x, fmaf(x[2].x, k[3 * kr + 2].x, acc.x)));
    acc.y = fmaf(x[0].y, k[3 * kr].y, fmaf(x[1].y, k[3 * kr + 1].y, fmaf(x[2].y, k[3 * kr + 2].y, acc.y)));
    acc.z = fmaf(x[0].z, k[3 * kr].z, fmaf(x[1].z, k[3 * kr + 1].z, fmaf(x[2].z, k[3 * kr + 2].z, acc.z)));
    acc.w = fmaf(x[0].w, k[3 * kr].w, fmaf(x[1].w, k[3 * kr + 1].w, fmaf(x[2].w, k[3 * kr + 2].w, acc.w)));
  };
  float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0, acc2 = acc0;        // outputs r-2, r-1, r while input row r arrives
  for (int r = rb; r < re + 2; ++r) {
    float4 x[3];
    load(r, x);
    tap_row(acc0, x, 2);                                          // input row r is the bottom tap row of output r-2, the middle
    tap_row(acc1, x, 1);                                          // of r-1, the top of r
    tap_row(acc2, x, 0);
    if (r >= rb + 2) {
      float4 hi, lo;
      tf32_split(bn_relu4(acc0, s, t), hi, lo);
      store(r - 2, hi, lo);
    }
    acc0 = acc1; acc1 = acc2; acc2 = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// The lock-step kernels' MMA: warpgroup tid / 128 owns one quarter of the 128 x CO accumulator (rows m0 .., columns col0 ..),
// issues the 3 * KS wgmma m64n(CO/2)k8 of a tile on the A operand (stride kLbaFull) and drains it from its registers.  The
// descriptors are formed once; a k-step only adds its byte offset to the start-address field.
template <int CO>
struct TcQuarter {
  int m0, col0;
  uint64_t da_hi, da_lo, db_hi, db_lo;
  __device__ __forceinline__ TcQuarter(int tid, const float* a_hi, const float* a_lo, const float* b_hi, const float* b_lo) {
    static_assert(CO == 64, "one m64n32k8 quarter per warpgroup");
    const int g = tid >> 7;
    m0 = 64 * (g & 1);
    col0 = (g >> 1) * (CO / 2);
    da_hi = gmma_desc(smem_u32(a_hi + 4 * m0), kLbaFull * 4u, 128u);
    da_lo = gmma_desc(smem_u32(a_lo + 4 * m0), kLbaFull * 4u, 128u);
    db_hi = gmma_desc(smem_u32(b_hi + 4 * col0), gmma_lbb(CO) * 4u, 128u);
    db_lo = gmma_desc(smem_u32(b_lo + 4 * col0), gmma_lbb(CO) * 4u, 128u);
  }
  __device__ __forceinline__ void run(int KS, int npos, const float* sc, const float* sf, float* __restrict__ out, size_t gbase,
                                      int wtid) const {
    float acc[1][CO / 8 * 2];
#pragma unroll
    for (int i = 0; i < CO / 4; ++i) acc[0][i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {                       // lo*hi, hi*lo, hi*hi: the small terms first
      const uint64_t da0 = pass == 0 ? da_lo : da_hi, db0 = pass == 1 ? db_lo : db_hi;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)                            // one MMA covers K = 8 = two 4-wide chunks
        wgmma_m64n32k8_tf32(acc[0], da0 + (uint64_t)((2 * ks * kLbaFull * 4) >> 4), db0 + (uint64_t)((2 * ks * gmma_lbb(CO) * 4) >> 4));
    }
    wgmma_commit();
    wgmma_wait_all();
    gmma_epilogue<1, CO / 16>(acc, m0, col0, CO, npos, sc, sf, out, gbase, wtid);
  }
};

// The first conv's im2col walk for a CTA of NT threads striding it: the input cells a thread copies (4-byte cp.async, zero-filled
// halo) and the (position, 4-wide tap chunk) operands A[m][k] = x[oh*sh + k / kw][ow*sw + k % kw] it gathers are the same for
// every tile, so the walk is worked out once (host side: im2col_walk_fits).
TCR_HD inline bool im2col_walk_fits(const DsLayerDev& L, int RH, int NT) {
  return ds_in_rows(L, RH) * ds_in_cols(L) <= kConvCells * NT && 128 * (L.kh * L.kw / 4) <= kConvTasks * NT && ds_in_rows(L, RH) < 512;
}
template <int NT>
struct Im2colWalk {
  int tid, cells, tasks;
  int f_pk[kConvCells];                                           // position offset + pl | tile row | column valid
  int g_x01[kConvTasks], g_x23[kConvTasks], g_a[kConvTasks];      // tile offsets of the four taps of a chunk (16 bits each), A offset | row
  __device__ __forceinline__ Im2colWalk(const DsLayerDev& L, int RH, int tid_) : tid(tid_) {
    const int wp = ds_in_cols(L);
    cells = ds_in_rows(L, RH) * wp;
    tasks = 128 * (L.kh * L.kw >> 2);
#pragma unroll
    for (int j = 0; j < kConvCells; ++j) {
      const int i = tid + j * NT, r = i / wp, col = i - r * wp, x = col - L.pl;
      f_pk[j] = ((r * L.win + x + L.pl) << 10) | (r << 1) | ((i < cells && x >= 0 && x < L.win) ? 1 : 0);
    }
#pragma unroll
    for (int j = 0; j < kConvTasks; ++j) {
      const int task = tid + j * NT, m = task & 127, kc = task >> 7;
      const int oh = m / L.wout, ow = m - oh * L.wout;
      int e[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = 4 * kc + q, ki = k / L.kw, kj = k - ki * L.kw;
        e[q] = (oh * L.sh + ki) * wp + ow * L.sw + kj;
      }
      g_x01[j] = e[0] | (e[1] << 16);
      g_x23[j] = e[2] | (e[3] << 16);
      g_a[j] = ((kc * kLbaFull + 4 * m) << 7) | m;
    }
  }
  // input rows of the tile starting at output row h0 of utterance n -> xs [hin_t][wp]
  __device__ __forceinline__ void fetch(const DsLayerDev& L, const float* in, int n, int h0, float* xs) const {
    const int hb = h0 * L.sh - L.pt;
    const float* base = in + ((int64_t)n * L.hin + hb) * L.win - L.pl;
#pragma unroll
    for (int j = 0; j < kConvCells; ++j) {
      if (tid + j * NT < cells) {
        const int pk = f_pk[j], h = hb + ((pk >> 1) & 0x1FF);
        const bool ok = (pk & 1) && h >= 0 && h < L.hin;
        const uint32_t bytes = ok ? 4u : 0u;
        const float* src = ok ? base + (pk >> 10) : in;
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(xs + tid + j * NT)), "l"(src), "r"(bytes) : "memory");
      }
    }
  }
  // A operand (hi / lo) of a tile of npos positions; rows past npos are zero
  __device__ __forceinline__ void gather(const float* xs, int npos, float* a_hi, float* a_lo) const {
#pragma unroll
    for (int j = 0; j < kConvTasks; ++j) {
      if (tid + j * NT < tasks) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if ((g_a[j] & 127) < npos) v = make_float4(xs[g_x01[j] & 0xFFFF], xs[g_x01[j] >> 16], xs[g_x23[j] & 0xFFFF], xs[g_x23[j] >> 16]);
        float4 hi, lo;
        tf32_split(v, hi, lo);
        st4(a_hi + (g_a[j] >> 7), hi);
        st4(a_lo + (g_a[j] >> 7), lo);
      }
    }
  }
};

// dscnn_dsblock_tc: x [2][C4][xs] (channel-chunk-major input tiles, +16 B per chunk against conflicts), a [hi, lo][C4][kLbaFull],
// b [hi, lo][C4][gmma_lbb], tab
template <int C, int CO>
TCR_HD inline DsSmem dsblock_tc_smem(const DsLayerDev& L, int RH) {
  constexpr int C4 = C / 4;
  DsSmem s = {};
  s.xs = (RH + 2) * (L.wout + 2) * 4 + 4;
  s.lba = kLbaFull;
  s.a = 2 * (size_t)C4 * s.xs;
  s.b = s.a + 2 * (size_t)C4 * s.lba;
  s.tab = s.b + 2 * (size_t)C4 * gmma_lbb(CO);
  s.floats = s.tab + ds_tab_floats(9, C, CO);
  return s;
}
// dscnn_dsblock_ws: x [2 buffers][2 channel halves][xs] (TMA destination, xs a multiple of the 1024-byte swizzle atom), a [2][hi,
// lo][C4][lba] (A rows packed to the tile's rows, rounded to 8, +16 B), b [hi, lo][C4][gmma_lbb] (b_hi also absorbs the last A
// chunk's over-read), tab
template <int C, int CO>
TCR_HD inline DsSmem dsblock_ws_smem(const DsLayerDev& L, int RH) {
  constexpr int C4 = C / 4;
  DsSmem s = {};
  s.xs = (((RH + 2) * (L.wout + 2) * (C / 2) * 4 + 1023) & ~1023) / 4;
  s.lba = ((RH * L.wout + 7) & ~7) * 4 + 4;
  s.a = 4 * (size_t)s.xs;
  s.b = s.a + 4 * (size_t)C4 * s.lba;
  s.tab = s.b + 2 * (size_t)C4 * gmma_lbb(CO);
  s.floats = s.tab + ds_tab_floats(9, C, CO);
  return s;
}
// dscnn_conv_tc (nbuf 1) and dscnn_conv_ws (nbuf 2): a [nbuf][hi, lo][K4][kLbaFull], b [hi, lo][K4][gmma_lbb], tab sc, sf [CO],
// x [2][xs] (input rows [hin_t][wp], rounded to 4)
template <int CO>
TCR_HD inline DsSmem conv_tc_smem(const DsLayerDev& L, int RH, int nbuf) {
  const int K4 = L.kh * L.kw / 4;
  DsSmem s = {};
  s.xs = (ds_in_rows(L, RH) * ds_in_cols(L) + 3) & ~3;
  s.lba = kLbaFull;
  s.b = 2 * (size_t)nbuf * K4 * s.lba;
  s.tab = s.b + 2 * (size_t)K4 * gmma_lbb(CO);
  s.x = s.tab + 2 * CO;
  s.floats = s.x + 2 * (size_t)s.xs;
  return s;
}

// Persistent: a CTA keeps the split filter bank and the per-channel tables for all its tiles (tile = RH output rows of one
// utterance), and the next tile's input rows travel (cp.async) while the current tile is computed.
// Specialised for the 3x3 / stride-1 depthwise stage (every separable block of DS-CNN-S, audio_nets/ds_cnn.py:20-26):
//   * depthwise (dw3_slide): a thread owns (4 channels, one output column) and slides down the rows of the tile;
//   * the four warpgroups then each issue the MMAs of one quarter of the accumulator and drain it (TcQuarter).
template <int C, int CO>
__global__ void __launch_bounds__(kTcThreads, 1) dscnn_dsblock_tc_kernel(DsLayerDev L, int RH, int n_utt, const float* __restrict__ params,
                                                                  const float* __restrict__ in, float* __restrict__ out, float eps) {
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  constexpr int C4 = C / 4;
  const int tid = threadIdx.x;
  const int hin_t = RH + 2, wp = L.wout + 2;                      // 3x3, stride 1
  const DsSmem S = dsblock_tc_smem<C, CO>(L, RH);
  const int XP = S.xs;                                            // floats per channel chunk of an input tile
  float *xs0 = smem, *a_hi = smem + S.a, *a_lo = a_hi + (size_t)C4 * kLbaFull;
  float *b_hi = smem + S.b, *b_lo = b_hi + (size_t)C4 * gmma_lbb(CO);
  const int tpu = ds_tiles_per_utt(L, RH);
  const int ntiles = tpu * n_utt;
  // pointwise filters pw[ci][co] -> B operand (params are caller-owned: independent of the producer)
  stage_b<kTcThreads, CO, 8>(params + L.pw, C, b_hi, b_lo, tid);
  const DsTables T = ds_stage_tables(smem + S.tab, L, 9, C, CO, params, eps, tid, kTcThreads);
  pdl_wait();
  // input rows (+halo) of a tile, channel-chunk-major, asynchronously.  A thread copies the same (row, column) cells of every
  // tile (cell = tid / C4 + j * (threads / C4)), so the walk is worked out once: cell -> (tile row, column validity, element offset).
  constexpr int kRowStep = kTcThreads / C4;
  const int f_c4 = tid % C4, f_row0 = tid / C4, f_rows = hin_t * wp;
  int f_pk[kDwCells];
#pragma unroll
  for (int j = 0; j < kDwCells; ++j) {
    const int row = f_row0 + j * kRowStep;
    const int r = row / wp, col = row - r * wp, x = col - 1;
    const int okx = (row < f_rows && x >= 0 && x < L.win) ? 1 : 0;
    f_pk[j] = ((r * L.win + x + 1) << 9) | (r << 1) | okx;         // position offset + 1 (>= 0), tile row, column-valid bit
  }
  auto fetch_tile = [&](int tile, float* xs) {
    const int n = tile / tpu, h0 = (tile - n * tpu) * RH;
    const float* base = in + (((int64_t)n * L.hin + (h0 - 1)) * L.win - 1) * C + 4 * f_c4;      // never dereferenced out of range
    float* dst = xs + (size_t)f_c4 * XP + 4 * f_row0;
#pragma unroll
    for (int j = 0; j < kDwCells; ++j) {
      if (f_row0 + j * kRowStep < f_rows) {
        const int pk = f_pk[j], h = h0 - 1 + ((pk >> 1) & 0xFF);
        const bool ok = (pk & 1) && h >= 0 && h < L.hin;
        cp_async16_zfill(dst + 4 * j * kRowStep, ok ? base + (int64_t)(pk >> 9) * C : in, ok);
      }
    }
  };
  const TcQuarter<CO> q(tid, a_hi, a_lo, b_hi, b_lo);
  int tile = blockIdx.x, cur = 0;
  if (tile < ntiles) fetch_tile(tile, xs0);
  for (; tile < ntiles; tile += gridDim.x, cur ^= 1) {
    const int n = tile / tpu, h0 = (tile - n * tpu) * RH, rh = imin(RH, L.hout - h0);
    float* xs = xs0 + (size_t)cur * C4 * XP;
    asm volatile("cp.async.wait_all;" ::: "memory");
    // this tile's rows have landed, and every warpgroup has finished the previous tile's MMAs (the A tiles are free)
    __syncthreads();
    if (tile + (int)gridDim.x < ntiles) fetch_tile(tile + gridDim.x, xs0 + (size_t)(cur ^ 1) * C4 * XP);
    // depthwise 3x3 + folded BN + ReLU -> A operand (hi / lo): thread = (channel chunk, output column), sliding down the rows
    // row segments keep every thread busy: (segment, channel chunk, column) tasks, a segment re-reads its two halo rows
    const int ntask0 = C4 * L.wout;
    const int nseg = imax(1, imin(rh, kTcThreads / ntask0)), srows = (rh + nseg - 1) / nseg;
    for (int task = tid; task < ntask0 * nseg; task += kTcThreads) {
      const int seg = task / ntask0, t0 = task - seg * ntask0;
      const int c4 = t0 / L.wout, ow = t0 - c4 * L.wout;
      const int rb = seg * srows, re = imin(rh, rb + srows);       // output rows [rb, re) of the tile
      if (rb >= re) continue;
      float4 k[9];
#pragma unroll
      for (int j = 0; j < 9; ++j) k[j] = ld4(T.taps + j * C + 4 * c4);
      const float* xb = xs + (size_t)c4 * XP + 4 * ow;
      dw3_slide(
          rb, re, k, ld4(T.sc1 + 4 * c4), ld4(T.sf1 + 4 * c4),
          [&](int r, float4(&x)[3]) {
            x[0] = ld4(xb + 4 * (r * wp)); x[1] = ld4(xb + 4 * (r * wp + 1)); x[2] = ld4(xb + 4 * (r * wp + 2));
          },
          [&](int m, float4 hi, float4 lo) {
            st4(a_hi + (size_t)c4 * kLbaFull + 4 * (m * L.wout + ow), hi);
            st4(a_lo + (size_t)c4 * kLbaFull + 4 * (m * L.wout + ow), lo);
          });
    }
    // accumulator rows past rh * wout are never stored, whatever the A rows there hold (each output row depends on its own A row only)
    fence_proxy_async();                                         // generic-proxy stores of the operands -> visible to the async proxy
    __syncthreads();
    q.run(C / 8, rh * L.wout, T.sc2, T.sf2, out, ((size_t)n * L.hout + h0) * L.wout, tid & 127);
  }
}

// Warp-specialised version of the block above (the default): the stages of a tile run on different warps and meet on mbarriers,
// so the input fetch and the depthwise stage of the next tile overlap the MMAs and the epilogue of this one.
//   warps 0-9   producers: TMA fetch of the tile two ahead (cp.async.bulk.tensor into the input buffer they have just left) and
//               the depthwise stage, input tile -> A operand (hi / lo); both double-buffered
//   warps 12-15 consumer warpgroup: the 3 * C/8 k-steps of a tile (two wgmma m64nCOk8 each: accumulator rows 0-63, 64-127),
//               then the epilogue from its registers
// Barriers (index = tile parity): in_full (TMA complete_tx), a_full (producers), mma_done (the consumer warpgroup, once its
// MMAs have completed: the A buffer may be refilled).  A rows are packed to the tile's own row count (rounded to 8): the
// 128-row MMA then reads a few rows of the next K chunk as rows >= npos, whose accumulator rows are never stored.
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {       // arrives when this thread's earlier cp.asyncs have landed
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// The consumer role of the warp-specialised kernels (shared by the separable block and the first conv), one warpgroup
// (wtid = thread index within it): per tile 3 * K4/2 k-steps on A buffer it % 2, then the folded BatchNorm + ReLU and the
// NHWC store of the tile's rows.
template <int CO>
__device__ __forceinline__ void ws_consumer_role(const DsLayerDev& L, int RH, int tpu, int ntiles, int K4, int LBA, const float* a0,
                                                 const float* b_hi, const float* b_lo, const float* sc, const float* sf,
                                                 float* __restrict__ out, uint64_t* a_full, uint64_t* mma_done, int wtid) {
  static_assert(CO == 64, "one m64n64k8 per 64 accumulator rows");
  constexpr int LBB = gmma_lbb(CO);
  const uint64_t db_hi = gmma_desc(smem_u32(b_hi), LBB * 4u, 128u), db_lo = gmma_desc(smem_u32(b_lo), LBB * 4u, 128u);
  const int KS = K4 >> 1;
  int it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int b = it & 1, k = it >> 1;
    const float* a_hi = a0 + (size_t)b * 2 * K4 * LBA;
    const uint64_t da_hi = gmma_desc(smem_u32(a_hi), (uint32_t)LBA * 4u, 128u);
    const uint64_t da_lo = gmma_desc(smem_u32(a_hi + (size_t)K4 * LBA), (uint32_t)LBA * 4u, 128u);
    mbar_wait(&a_full[b], (uint32_t)(k & 1));
    float acc[2][CO / 2];
#pragma unroll
    for (int i = 0; i < CO / 2; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {                       // lo*hi, hi*lo, hi*hi: the small terms first
      const uint64_t da0 = pass == 0 ? da_lo : da_hi, db0 = pass == 1 ? db_lo : db_hi;
#pragma unroll 4
      for (int ks = 0; ks < KS; ++ks) {                          // one k-step covers K = 8 = two 4-wide chunks
        const uint64_t da = da0 + (uint64_t)((2 * ks * LBA * 4) >> 4), db = db0 + (uint64_t)((2 * ks * LBB * 4) >> 4);
        wgmma_m64n64k8_tf32(acc[0], da, db);
        wgmma_m64n64k8_tf32(acc[1], da + (uint64_t)((64 * 16) >> 4), db);   // rows 64-127: eight 8-row groups further
      }
    }
    wgmma_commit();
    wgmma_wait_all();
    mbar_arrive(&mma_done[b]);                                   // the A buffer is free for the tile two ahead
    const int n = tile / tpu, h0 = (tile - n * tpu) * RH, npos = imin(RH, L.hout - h0) * L.wout;
    gmma_epilogue<2, CO / 8>(acc, 0, 0, CO, npos, sc, sf, out, ((size_t)n * L.hout + h0) * L.wout, wtid);
  }
}

template <int C, int CO>
__global__ void __launch_bounds__(kTcThreads, 1) dscnn_dsblock_ws_kernel(const __grid_constant__ CUtensorMap in_map, DsLayerDev L, int RH, int n_utt,
                                                                         const float* __restrict__ params, float* __restrict__ out, float eps) {
  TCR_DYNAMIC_SMEM(smem_raw);
  __shared__ uint64_t in_full[2], a_full[2], mma_done[2];
  float* smem = reinterpret_cast<float*>(smem_raw);
  constexpr int C4 = C / 4;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int hin_t = RH + 2, wp = L.wout + 2;
  constexpr int CH = C / 2, CH4 = CH / 4;                         // channels per TMA box: 32 fp32 = one 128-byte swizzle row
  static_assert(CH * 4 == 128, "the input halves are 128-byte rows (SWIZZLE_128B)");
  const DsSmem S = dsblock_ws_smem<C, CO>(L, RH);
  const int XH = S.xs, LBA = S.lba;                               // floats per half input tile; K-chunk stride of the A tiles
  float *xs0 = smem, *a0 = smem + S.a, *b_hi = smem + S.b, *b_lo = b_hi + (size_t)C4 * gmma_lbb(CO);
  const int tpu = ds_tiles_per_utt(L, RH);
  const int ntiles = tpu * n_utt;
  if (tid == 0) {
    for (int b = 0; b < 2; ++b) {
      mbar_init(&in_full[b], 1);
      mbar_init(&a_full[b], kWsProducers);
      mbar_init(&mma_done[b], kWsConsumers);
    }
  }
  stage_b<kTcThreads, CO, 8>(params + L.pw, C, b_hi, b_lo, tid);
  const DsTables T = ds_stage_tables(smem + S.tab, L, 9, C, CO, params, eps, tid, kTcThreads);
  pdl_wait();
  fence_proxy_async();                                           // the B operand was written through the generic proxy
  __syncthreads();

  if (warp < kWsProducerWarps) {
    // ---- input fetch (TMA) + depthwise 3x3 + folded BN + ReLU -> A operand ----
    // One thread issues two 4-D tensor loads per tile (channel halves; box = 32 channels x (wout + 2) columns x (RH + 2) rows,
    // start (., -1, h0 - 1, n): the halo outside the feature map arrives as zeros) and the bytes land on `in_full`.  The box rows
    // are 128 bytes, SWIZZLE_128B: the 16-byte chunk j of position p sits at chunk j ^ (p & 7), so the 8 lanes of a quarter warp,
    // which read the same channel chunk of 8 consecutive positions, hit 8 different bank groups.
    const uint32_t tile_bytes = (uint32_t)(2 * hin_t * wp * CH * 4);
    auto fetch_tile = [&](int tile, float* xs, uint64_t* bar) {
      const int n = tile / tpu, h0 = (tile - n * tpu) * RH;
      mbar_expect_tx(bar, tile_bytes);
#pragma unroll
      for (int half = 0; half < 2; ++half)
        asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                     ::"r"(smem_u32(xs + (size_t)half * XH)), "l"(&in_map), "r"(half * CH), "r"(-1), "r"(h0 - 1), "r"(n), "r"(smem_u32(bar))
                     : "memory");
    };
    if (tid == 0) {
      int t0 = blockIdx.x;
      if (t0 < ntiles) fetch_tile(t0, xs0, &in_full[0]);
      t0 += gridDim.x;
      if (t0 < ntiles) fetch_tile(t0, xs0 + (size_t)2 * XH, &in_full[1]);
    }
    // thread = (channel chunk, output column), the same for every tile (host side: C4 * wout <= producers): its nine taps and
    // the folded BatchNorm stay in registers
    const bool active = tid < C4 * L.wout;
    const int c4 = active ? tid / L.wout : 0, ow = active ? tid - c4 * L.wout : 0;
    const int half = c4 / CH4, cl = c4 - half * CH4;
    float4 kk[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) kk[j] = ld4(T.taps + j * C + 4 * c4);
    const float4 s = ld4(T.sc1 + 4 * c4), t = ld4(T.sf1 + 4 * c4);
    int it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int b = it & 1, k = it >> 1;
      const int h0 = (tile % tpu) * RH, rh = imin(RH, L.hout - h0);
      float* xs = xs0 + (size_t)b * 2 * XH;
      float* a_hi = a0 + (size_t)b * 2 * C4 * LBA;
      float* a_lo = a_hi + (size_t)C4 * LBA;
      mbar_wait(&in_full[b], (uint32_t)(k & 1));
      if (it >= 2) mbar_wait(&mma_done[b], (uint32_t)((k - 1) & 1));             // the MMAs of tile it-2 have read this A buffer
      if (active) {
        const float* xh = xs + (size_t)half * XH;
        float* ah = a_hi + (size_t)c4 * LBA + 4 * ow;
        float* al = a_lo + (size_t)c4 * LBA + 4 * ow;
        dw3_slide(
            0, rh, kk, s, t,
            [&](int r, float4(&x)[3]) {
              const int p = ow + r * wp;                          // position (tile row r, column ow) of the padded tile
#pragma unroll
              for (int j = 0; j < 3; ++j) x[j] = ld4(xh + (p + j) * CH + (((cl ^ (p + j)) & 7) << 2));
            },
            [&](int m, float4 hi, float4 lo) {
              st4(ah + 4 * m * L.wout, hi);
              st4(al + 4 * m * L.wout, lo);
            });
      }
      fence_proxy_async();                                       // operand stores -> visible to the async proxy (wgmma)
      mbar_arrive(&a_full[b]);
      const int nxt = tile + 2 * (int)gridDim.x;                  // refill this input buffer once every producer has left it
      if (nxt < ntiles) {
        asm volatile("bar.sync 1, %0;" ::"n"(kWsProducers) : "memory");
        if (tid == 0) fetch_tile(nxt, xs, &in_full[b]);
      }
    }
  } else if (warp >= kWsConsumerWarp0) {
    ws_consumer_role<CO>(L, RH, tpu, ntiles, C4, LBA, a0, b_hi, b_lo, T.sc2, T.sf2, out, a_full, mma_done, tid - 32 * kWsConsumerWarp0);
  }
}

// First conv, warp-specialised (same roles and barriers as the block kernel): the producers copy the tile's input rows and
// gather its im2col operand (Im2colWalk) into the A buffer of the tile, and refill the input buffer for the tile two ahead;
// K = kh * kw (40).
template <int CO>
__global__ void __launch_bounds__(kTcThreads, 1) dscnn_conv_ws_kernel(DsLayerDev L, int RH, int n_utt, const float* __restrict__ params,
                                                                      const float* __restrict__ in, float* __restrict__ out, float eps) {
  TCR_DYNAMIC_SMEM(smem_raw);
  __shared__ uint64_t in_full[2], a_full[2], mma_done[2];
  float* smem = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int K = L.kh * L.kw, K4 = K >> 2;
  const DsSmem S = conv_tc_smem<CO>(L, RH, 2);
  float *a0 = smem, *b_hi = smem + S.b, *b_lo = b_hi + (size_t)K4 * gmma_lbb(CO);
  float *sc = smem + S.tab, *sf = sc + CO, *xs0 = smem + S.x;
  const int tpu = ds_tiles_per_utt(L, RH);
  const int ntiles = tpu * n_utt;
  if (tid == 0) {
    for (int b = 0; b < 2; ++b) {
      mbar_init(&in_full[b], kWsProducers);
      mbar_init(&a_full[b], kWsProducers);
      mbar_init(&mma_done[b], kWsConsumers);
    }
  }
  stage_b<kTcThreads, CO, 1>(params + L.w, K, b_hi, b_lo, tid);
  for (int c = tid; c < CO; c += kTcThreads) fold_bn(params, L.b, L.beta, L.mm, L.mv, c, eps, sc, sf);
  pdl_wait();
  fence_proxy_async();
  __syncthreads();

  if (warp < kWsProducerWarps) {
    const Im2colWalk<kWsProducers> walk(L, RH, tid);
    auto fetch_tile = [&](int tile, float* xs, uint64_t* bar) {
      const int n = tile / tpu;
      walk.fetch(L, in, n, (tile - n * tpu) * RH, xs);
      cp_async_mbar_arrive(bar);
    };
    {
      int t0 = blockIdx.x;
      if (t0 < ntiles) fetch_tile(t0, xs0, &in_full[0]);
      t0 += gridDim.x;
      if (t0 < ntiles) fetch_tile(t0, xs0 + S.xs, &in_full[1]);
    }
    int it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int b = it & 1, k = it >> 1;
      const int h0 = (tile % tpu) * RH, npos = imin(RH, L.hout - h0) * L.wout;
      float* xs = xs0 + b * S.xs;
      float* a_hi = a0 + (size_t)b * 2 * K4 * kLbaFull;
      mbar_wait(&in_full[b], (uint32_t)(k & 1));
      if (it >= 2) mbar_wait(&mma_done[b], (uint32_t)((k - 1) & 1));             // the MMAs of tile it-2 have read this A buffer
      walk.gather(xs, npos, a_hi, a_hi + (size_t)K4 * kLbaFull);
      fence_proxy_async();
      mbar_arrive(&a_full[b]);
      const int nxt = tile + 2 * (int)gridDim.x;
      if (nxt < ntiles) {
        asm volatile("bar.sync 1, %0;" ::"n"(kWsProducers) : "memory");
        fetch_tile(nxt, xs, &in_full[b]);
      }
    }
  } else if (warp >= kWsConsumerWarp0) {
    ws_consumer_role<CO>(L, RH, tpu, ntiles, K4, kLbaFull, a0, b_hi, b_lo, sc, sf, out, a_full, mma_done, tid - 32 * kWsConsumerWarp0);
  }
}

// First layer (kh x kw conv from the single-channel feature map, audio_nets/ds_cnn.py:21 `conv_1`) as an implicit GEMM on
// wgmma: the im2col operand (Im2colWalk) is gathered from the staged input rows straight into the canonical operand layout
// (hi / lo), B = the filter bank [co][k], K = kh * kw (40), same persistent / quarter-per-warpgroup structure as the lock-step
// block kernel above.
template <int CO>
__global__ void __launch_bounds__(kTcThreads, 1) dscnn_conv_tc_kernel(DsLayerDev L, int RH, int n_utt, const float* __restrict__ params,
                                                                      const float* __restrict__ in, float* __restrict__ out, float eps) {
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x;
  const int K = L.kh * L.kw, K4 = K >> 2;
  const DsSmem S = conv_tc_smem<CO>(L, RH, 1);
  float *a_hi = smem, *a_lo = a_hi + (size_t)K4 * kLbaFull, *b_hi = smem + S.b, *b_lo = b_hi + (size_t)K4 * gmma_lbb(CO);
  float *sc = smem + S.tab, *sf = sc + CO, *xs0 = smem + S.x;
  const int tpu = ds_tiles_per_utt(L, RH);
  const int ntiles = tpu * n_utt;
  stage_b<kTcThreads, CO, 1>(params + L.w, K, b_hi, b_lo, tid);
  for (int c = tid; c < CO; c += kTcThreads) fold_bn(params, L.b, L.beta, L.mm, L.mv, c, eps, sc, sf);
  pdl_wait();
  const Im2colWalk<kTcThreads> walk(L, RH, tid);
  auto fetch_tile = [&](int tile, float* xs) {
    const int n = tile / tpu;
    walk.fetch(L, in, n, (tile - n * tpu) * RH, xs);
  };
  const TcQuarter<CO> q(tid, a_hi, a_lo, b_hi, b_lo);
  int tile = blockIdx.x, cur = 0;
  if (tile < ntiles) fetch_tile(tile, xs0);
  for (; tile < ntiles; tile += gridDim.x, cur ^= 1) {
    const int n = tile / tpu, h0 = (tile - n * tpu) * RH, npos = imin(RH, L.hout - h0) * L.wout;
    const float* xs = xs0 + cur * S.xs;
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();                                             // rows landed; the previous tile's MMAs are done with A
    if (tile + (int)gridDim.x < ntiles) fetch_tile(tile + gridDim.x, xs0 + (cur ^ 1) * S.xs);
    walk.gather(xs, npos, a_hi, a_lo);
    fence_proxy_async();
    __syncthreads();
    q.run(K >> 3, npos, sc, sf, out, ((size_t)n * L.hout + h0) * L.wout, tid & 127);
  }
}
#endif

// ---- head: one CTA per utterance ----
__global__ void __launch_bounds__(256) dscnn_head_kernel(int npos, int C, int classes, int64_t fcw, int64_t fcb,
                                                         const float* __restrict__ params, const float* __restrict__ in,
                                                         float* __restrict__ logits, float* __restrict__ probs) {
  pdl_wait();
  __shared__ __align__(16) float s_red[1024];
  __shared__ float s_pool[320];
  __shared__ float s_logit[kMaxClasses];
  const int n = blockIdx.x, tid = threadIdx.x;
  int nseg;
  if ((C & 3) == 0) {                                             // float4 loads: thread = (segment of positions, 4 channels)
    const int C4 = C >> 2;
    nseg = imax(1, imin((int)blockDim.x / C4, 1024 / C));
    const int seg = tid / C4, c4 = tid - seg * C4;
    if (seg < nseg) {
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
      const float* src = in + (size_t)n * npos * C + 4 * c4;
#pragma unroll 4
      for (int p = seg; p < npos; p += nseg) {
        const float4 v = ldg4(src + (size_t)p * C);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
      st4(s_red + seg * C + 4 * c4, s);
    }
  } else {
    nseg = imax(1, imin((int)blockDim.x / C, 1024 / C));
    const int seg = tid / C, c = tid - seg * C;
    if (seg < nseg) {
      float s = 0.f;
      for (int p = seg; p < npos; p += nseg) s += in[((size_t)n * npos + p) * C + c];
      s_red[seg * C + c] = s;
    }
  }
  __syncthreads();
  for (int c = tid; c < C; c += blockDim.x) {
    float tot = 0.f;
    for (int q = 0; q < nseg; ++q) tot += s_red[q * C + c];
    s_pool[c] = tot / (float)npos;
  }
  __syncthreads();
  if (tid < classes) {
    float acc = params[fcb + tid];
    for (int k = 0; k < C; ++k) acc = fmaf(s_pool[k], params[fcw + (int64_t)k * classes + tid], acc);
    s_logit[tid] = acc;
    if (logits) logits[(size_t)n * classes + tid] = acc;
  }
  __syncthreads();
  if (tid < classes && probs) {
    float mx = -3.0e38f;
    for (int k = 0; k < classes; ++k) mx = fmaxf(mx, s_logit[k]);
    float se = 0.f;
    for (int k = 0; k < classes; ++k) se += expf(s_logit[k] - mx);
    probs[(size_t)n * classes + tid] = expf(s_logit[tid] - mx) / se;
  }
}

}  // namespace tcr

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
using namespace tcr;

struct tcr_dscnn {
  tcr_dscnn_config cfg;
  DsNet net;
  std::vector<tcr_param_desc> table;
  int64_t n_params = 0, flops = 0;
  float* act[2] = {nullptr, nullptr};
  size_t act_floats = 0;
  int sms = 1;
  bool use_tc = true;        // pointwise convs on the tensor cores (wgmma) where they fit (env TCR_DSCNN_TC=0: register-tiled FMA everywhere)
  bool tc_ws = true;         // warp-specialised wgmma block kernel (env TCR_DSCNN_TC=1: the lock-step version)
#ifndef TCR_EMU
  struct InMap { CUtensorMap map; const void* ptr = nullptr; int rh = 0; };
  std::vector<InMap> in_maps;   // per layer: TMA descriptor of the block's input activations (re-encoded if the buffer changes)
#endif
};

#ifndef TCR_EMU
// 4-D tensor map over the NHWC activations [n][h][w][c] (innermost first: c, w, h, n), box = 32 channels x wp columns x hin_t rows,
// 128-byte swizzle; out-of-range coordinates (the SAME-padding halo) are filled with zeros.  The driver entry point is looked up at
// run time (no link against libcuda).
static int ds_encode_in_map(CUtensorMap* map, const float* base, int c, int w, int h, int n, int box_w, int box_h) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
      set_error("cuTensorMapEncodeTiled is not available");
      return TCR_ERR_CUDA;
    }
    encode = (EncodeFn)fn;
  }
  const cuuint64_t gdim[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const cuuint64_t gstride[3] = {(cuuint64_t)c * 4, (cuuint64_t)w * c * 4, (cuuint64_t)h * w * c * 4};
  const cuuint32_t box[4] = {32u, (cuuint32_t)box_w, (cuuint32_t)box_h, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed"); return TCR_ERR_CUDA; }
  return TCR_OK;
}
#endif

static void ds_same(int len, int k, int s, int* out, int* lead) {
  *out = (len + s - 1) / s;
  const int total = std::max((*out - 1) * s + k - len, 0);
  *lead = total / 2;
}

extern "C" int tcr_dscnn_create(const tcr_dscnn_config* cfg, tcr_dscnn** out) {
  if (!cfg || !out) { set_error("NULL argument"); return TCR_ERR_INVALID; }
  *out = nullptr;
  if (cfg->size != 'S' && cfg->size != 'M' && cfg->size != 'L') { set_error("DS-CNN size must be 'S', 'M' or 'L'"); return TCR_ERR_INVALID; }
  if (cfg->max_batch <= 0 || cfg->height <= 0 || cfg->width <= 0 || cfg->num_classes <= 0 || cfg->num_classes > kMaxClasses) {
    set_error("bad DS-CNN configuration");
    return TCR_ERR_INVALID;
  }
  tcr_dscnn* d = new tcr_dscnn();
  d->cfg = *cfg;
  if (const char* e = getenv("TCR_DSCNN_TC")) { d->use_tc = e[0] != '0'; d->tc_ws = e[0] != '1'; }
  struct Def { int type, depth, kh, kw, sh, sw; const char* scope; };
  std::vector<Def> defs;
  if (cfg->size == 'S') {
    defs = {{0, 64, 10, 4, 2, 2, "conv_1"}, {1, 64, 3, 3, 1, 1, "conv_ds_1"}, {1, 64, 3, 3, 1, 1, "conv_ds_2"},
            {1, 64, 3, 3, 1, 1, "conv_ds_3"}, {1, 64, 3, 3, 1, 1, "conv_ds_4"}};
  } else if (cfg->size == 'M') {
    defs = {{0, 172, 10, 4, 2, 1, "conv_1"}, {1, 172, 3, 3, 2, 2, "conv_ds_1"}, {1, 172, 3, 3, 1, 1, "conv_ds_2"},
            {1, 172, 3, 3, 1, 1, "conv_ds_3"}, {1, 172, 3, 3, 1, 1, "conv_ds_4"}};
  } else {
    defs = {{0, 276, 10, 4, 2, 1, "conv_1"}, {1, 276, 3, 3, 2, 2, "conv_ds_1"}, {1, 276, 3, 3, 1, 1, "conv_ds_2"},
            {1, 276, 3, 3, 1, 1, "conv_ds_3"}, {1, 276, 3, 3, 1, 1, "conv_ds_4"}, {1, 276, 3, 3, 1, 1, "conv_ds_5"}};
  }
  int64_t off = 0;
  auto add = [&](const std::string& name, int kind, std::initializer_list<int> shape) {
    tcr_param_desc t;
    memset(&t, 0, sizeof(t));
    snprintf(t.name, sizeof(t.name), "%s", name.c_str());
    t.kind = kind;
    t.rank = (int)shape.size();
    int64_t numel = 1;
    int i = 0;
    for (int s : shape) { t.shape[i++] = s; numel *= s; }
    t.offset = off;
    t.numel = numel;
    d->table.push_back(t);
    off += numel;
    return t.offset;
  };
  int h = cfg->height, w = cfg->width, cin = 1;
  d->net.nlayers = 0;
  for (const Def& df : defs) {
    DsLayerDev L;
    memset(&L, 0, sizeof(L));
    L.type = df.type; L.cin = cin; L.cout = df.depth; L.kh = df.kh; L.kw = df.kw; L.sh = df.sh; L.sw = df.sw; L.hin = h; L.win = w;
    ds_same(h, df.kh, df.sh, &L.hout, &L.pt);
    ds_same(w, df.kw, df.sw, &L.wout, &L.pl);
    const std::string s = std::string("DSCNN/") + df.scope;
    if (df.type == 0) {
      L.w = add(s + "/weights", TCR_KIND_WEIGHT, {df.kh, df.kw, cin, df.depth});
      L.b = add(s + "/biases", TCR_KIND_BETA, {df.depth});
      L.beta = add(s + "/batch_norm/beta", TCR_KIND_BETA, {df.depth});
      L.mm = add(s + "/batch_norm/moving_mean", TCR_KIND_MOVING_MEAN, {df.depth});
      L.mv = add(s + "/batch_norm/moving_variance", TCR_KIND_MOVING_VAR, {df.depth});
      d->flops += 2ll * L.hout * L.wout * df.kh * df.kw * cin * df.depth;
    } else {
      L.w = add(s + "/depthwise_conv/depthwise_weights", TCR_KIND_WEIGHT, {df.kh, df.kw, cin, 1});
      L.b = add(s + "/depthwise_conv/biases", TCR_KIND_BETA, {cin});
      L.beta = add(s + "/dw_batch_norm/beta", TCR_KIND_BETA, {cin});
      L.mm = add(s + "/dw_batch_norm/moving_mean", TCR_KIND_MOVING_MEAN, {cin});
      L.mv = add(s + "/dw_batch_norm/moving_variance", TCR_KIND_MOVING_VAR, {cin});
      L.pw = add(s + "/pointwise_conv/weights", TCR_KIND_WEIGHT, {1, 1, cin, df.depth});
      L.pb = add(s + "/pointwise_conv/biases", TCR_KIND_BETA, {df.depth});
      L.pbeta = add(s + "/pw_batch_norm/beta", TCR_KIND_BETA, {df.depth});
      L.pmm = add(s + "/pw_batch_norm/moving_mean", TCR_KIND_MOVING_MEAN, {df.depth});
      L.pmv = add(s + "/pw_batch_norm/moving_variance", TCR_KIND_MOVING_VAR, {df.depth});
      d->flops += 2ll * L.hout * L.wout * df.kh * df.kw * cin + 2ll * L.hout * L.wout * cin * df.depth;
    }
    if (df.depth % 4) { delete d; set_error("DS-CNN depth must be a multiple of 4"); return TCR_ERR_UNSUPPORTED; }
    d->net.layer[d->net.nlayers++] = L;
    d->act_floats = std::max(d->act_floats, (size_t)L.hout * L.wout * df.depth);
    h = L.hout; w = L.wout; cin = df.depth;
  }
  d->net.classes = cfg->num_classes;
  d->net.fcw = add("DSCNN/fc1/weights", TCR_KIND_WEIGHT, {cin, cfg->num_classes});
  d->net.fcb = add("DSCNN/fc1/biases", TCR_KIND_BETA, {cfg->num_classes});
  d->flops += 2ll * cin * cfg->num_classes;
  d->n_params = off;
  if (cudaSetDevice(cfg->device) != cudaSuccess) { delete d; set_error("cudaSetDevice failed"); return TCR_ERR_CUDA; }
#ifndef TCR_EMU
  cudaDeviceGetAttribute(&d->sms, cudaDevAttrMultiProcessorCount, cfg->device);
#endif
  for (int i = 0; i < 2; ++i)
    if (cudaMalloc((void**)&d->act[i], d->act_floats * cfg->max_batch * sizeof(float)) != cudaSuccess) {
      tcr_dscnn_destroy(d);
      set_error("cudaMalloc failed for the DS-CNN activation buffers");
      return TCR_ERR_CUDA;
    }
  *out = d;
  return TCR_OK;
}

extern "C" int tcr_dscnn_destroy(tcr_dscnn* d) {
  if (!d) return TCR_OK;
  for (int i = 0; i < 2; ++i)
    if (d->act[i]) cudaFree(d->act[i]);
  delete d;
  return TCR_OK;
}

extern "C" int tcr_dscnn_param_table(const tcr_dscnn* d, const tcr_param_desc** descs, int32_t* count, int64_t* num_params,
                                     int64_t* forward_flops_per_utt) {
  if (!d || !descs || !count) { set_error("NULL argument"); return TCR_ERR_INVALID; }
  *descs = d->table.data();
  *count = (int32_t)d->table.size();
  if (num_params) *num_params = d->n_params;
  if (forward_flops_per_utt) *forward_flops_per_utt = d->flops;
  return TCR_OK;
}

// Tile rows of the wgmma kernels: at most 128 accumulator rows (RH * wout) per tile, balanced (25 rows -> 5 tiles of 5).
static int ds_tile_rows(const DsLayerDev& L) {
  const int cap = std::max(1, std::min(L.hout, 128 / std::max(1, std::min(L.wout, 128))));
  const int tiles = (L.hout + cap - 1) / cap;
  return (L.hout + tiles - 1) / tiles;
}

// Launches layer l: in [n, hin, win, cin] -> out [n, hout, wout, cout] (NHWC).  The kernel is chosen here, once for both entry
// points: wgmma where the layer's shape fits the tensor-core kernels (TCR_DSCNN_TC), the register-tiled FMA kernels otherwise.
// The warp-specialised block kernel reads its input through a TMA map over max_batch utterances, so only from an activation
// buffer of the handle.
static int ds_launch_layer(tcr_dscnn* d, int l, const float* params, const float* in, float* out, int32_t n, cudaStream_t s) {
  const DsLayerDev& L = d->net.layer[l];
  const float eps = 1e-3f;
  if (L.type == 0) {
#ifndef TCR_EMU
    const int RHt = ds_tile_rows(L), grid = std::min(ds_tiles_per_utt(L, RHt) * n, d->sms);
    // implicit GEMM on wgmma (3xTF32), where the kernel's per-thread im2col walk covers the tile
    if (d->use_tc && L.cin == 1 && L.cout == 64 && (L.kh * L.kw) % 8 == 0 && L.wout <= 64 && im2col_walk_fits(L, RHt, kTcThreads)) {
      const size_t smem_ws = conv_tc_smem<64>(L, RHt, 2).floats * 4;
      if (d->tc_ws && smem_ws <= 220 * 1024 && im2col_walk_fits(L, RHt, kWsProducers) && (L.kh * L.kw / 4) % 2 == 0) {
        auto kws = dscnn_conv_ws_kernel<64>;
        static SmemOptIn optin_ws;
        if (optin_ws.ensure(kws, smem_ws) != cudaSuccess) return TCR_ERR_CUDA;
        TCR_LAUNCH("dscnn_conv_ws", kws, dim3(grid), dim3(kTcThreads), smem_ws, s, L, RHt, n, params, in, out, eps);
        return TCR_OK;
      }
      const size_t smem_tc = conv_tc_smem<64>(L, RHt, 1).floats * 4;
      auto ktc = dscnn_conv_tc_kernel<64>;
      static SmemOptIn optin_tc;
      if (optin_tc.ensure(ktc, smem_tc) != cudaSuccess) return TCR_ERR_CUDA;
      TCR_LAUNCH("dscnn_conv_tc", ktc, dim3(grid), dim3(kTcThreads), smem_tc, s, L, RHt, n, params, in, out, eps);
      return TCR_OK;
    }
#endif
    const size_t smem = conv_smem(L).floats * 4;
    auto kfn = dscnn_conv_kernel;
#ifndef TCR_EMU
    static SmemOptIn optin;
    if (optin.ensure(kfn, smem) != cudaSuccess) return TCR_ERR_CUDA;
#endif
    TCR_LAUNCH("dscnn_conv", kfn, dim3(n), dim3(256), smem, s, L, params, in, out, eps);
  } else {
#ifndef TCR_EMU
    // pointwise conv on the tensor cores (wgmma, 3xTF32): the 64 -> 64 channel blocks with a 3x3 / stride-1 depthwise stage
    if (d->use_tc && L.cin == 64 && L.cout == 64 && L.kh == 3 && L.kw == 3 && L.sh == 1 && L.sw == 1 && L.wout <= 64) {
      const int RHt = ds_tile_rows(L), grid = std::min(ds_tiles_per_utt(L, RHt) * n, d->sms);
      const size_t smem_ws = dsblock_ws_smem<64, 64>(L, RHt).floats * 4;
      if (d->tc_ws && smem_ws <= 226 * 1024 && L.cin / 4 * L.wout <= kWsProducers && L.wout + 2 <= 256 && RHt + 2 <= 256 &&
          (in == d->act[0] || in == d->act[1])) {
        auto kws = dscnn_dsblock_ws_kernel<64, 64>;
        static SmemOptIn optin_ws;
        if (optin_ws.ensure(kws, smem_ws) != cudaSuccess) return TCR_ERR_CUDA;
        if ((int)d->in_maps.size() < d->net.nlayers) d->in_maps.resize(d->net.nlayers);
        tcr_dscnn::InMap& im = d->in_maps[l];
        if (im.ptr != in || im.rh != RHt) {                    // the activations ping-pong between two buffers: encoded once per layer
          const int rc = ds_encode_in_map(&im.map, in, L.cin, L.win, L.hin, d->cfg.max_batch, L.wout + 2, RHt + 2);
          if (rc != TCR_OK) return rc;
          im.ptr = in;
          im.rh = RHt;
        }
        TCR_LAUNCH("dscnn_dsblock_ws", kws, dim3(grid), dim3(kTcThreads), smem_ws, s, im.map, L, RHt, n, params, out, eps);
        return TCR_OK;
      }
      const size_t smem_tc = dsblock_tc_smem<64, 64>(L, RHt).floats * 4;
      if (smem_tc <= 200 * 1024 && (RHt + 2) * (L.wout + 2) <= kDwCells * (kTcThreads / (L.cin / 4))) {   // the kernel's fetch walk
        auto ktc = dscnn_dsblock_tc_kernel<64, 64>;
        static SmemOptIn optin_tc;
        if (optin_tc.ensure(ktc, smem_tc) != cudaSuccess) return TCR_ERR_CUDA;
        TCR_LAUNCH("dscnn_dsblock_tc", ktc, dim3(grid), dim3(kTcThreads), smem_tc, s, L, RHt, n, params, in, out, eps);
        return TCR_OK;
      }
    }
#endif
    // the whole pointwise bank in shared memory when it fits next to a useful tile; else (DS-CNN-L: 276 x 276 fp32 = 305 KB) output-
    // channel tiles of COT, the depthwise output of the tile being reused for every slice
    int COT = L.cout;
    while (COT > 32 && dsblock_smem(L, 1, COT).floats * 4 > 96 * 1024) COT = ((COT / 2) + 3) & ~3;
    int RH = std::min(L.hout, 8);
    while (RH > 1 && dsblock_smem(L, RH, COT).floats * 4 > 100 * 1024) --RH;
    const size_t smem = dsblock_smem(L, RH, COT).floats * 4;
    if (smem > 200 * 1024) { set_error("DS-CNN layer does not fit in shared memory"); return TCR_ERR_UNSUPPORTED; }
    auto kfn = dscnn_dsblock_kernel;
#ifndef TCR_EMU
    static SmemOptIn optin;
    if (optin.ensure(kfn, smem) != cudaSuccess) return TCR_ERR_CUDA;
#endif
    // one utterance per blockIdx.y: batches past kMaxGridRows run as several launches over consecutive utterances
    const size_t in_utt = (size_t)L.hin * L.win * L.cin, out_utt = (size_t)L.hout * L.wout * L.cout;
    for (int first = 0; first < n; first += kMaxGridRows) {
      TCR_LAUNCH("dscnn_dsblock", kfn, dim3(ds_tiles_per_utt(L, RH), std::min(n - first, kMaxGridRows)), dim3(256), smem, s, L, RH, COT,
                 params, in + first * in_utt, out + first * out_utt, eps);
      if (cudaGetLastError() != cudaSuccess) { set_error("DS-CNN block launch failed"); return TCR_ERR_CUDA; }
    }
  }
  return TCR_OK;
}

extern "C" int tcr_dscnn_forward(tcr_dscnn* d, const float* features, const float* params, int32_t n, float* logits, float* probs,
                                 tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !features || !params) { set_error("NULL argument"); return TCR_ERR_INVALID; }
  if (n <= 0 || n > d->cfg.max_batch) { set_error("n outside [1, max_batch]"); return TCR_ERR_INVALID; }
  cudaStream_t s = (cudaStream_t)stream;
  const float* in = features;
  for (int l = 0; l < d->net.nlayers; ++l) {
    float* out = d->act[l & 1];
    const int rc = ds_launch_layer(d, l, params, in, out, n, s);
    if (rc != TCR_OK) return rc;
    in = out;
  }
  const DsLayerDev& last = d->net.layer[d->net.nlayers - 1];
  if (last.cout > 320) { set_error("DS-CNN head supports up to 320 channels"); return TCR_ERR_UNSUPPORTED; }
  TCR_LAUNCH("dscnn_head", dscnn_head_kernel, dim3(n), dim3(256), 0, s, last.hout * last.wout, last.cout, d->net.classes, d->net.fcw,
             d->net.fcb, params, in, logits, probs);
  if (cudaGetLastError() != cudaSuccess) { set_error("DS-CNN launch failed"); return TCR_ERR_CUDA; }
  return TCR_OK;
}

extern "C" int tcr_dscnn_forward_partial(tcr_dscnn* d, const float* features, const float* params, int32_t n, int32_t num_layers,
                                         float* act_out, tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !features || !params || !act_out) { set_error("NULL argument"); return TCR_ERR_INVALID; }
  if (n <= 0 || n > d->cfg.max_batch) { set_error("n outside [1, max_batch]"); return TCR_ERR_INVALID; }
  if (num_layers <= 0 || num_layers > d->net.nlayers) { set_error("num_layers outside [1, number of layers]"); return TCR_ERR_INVALID; }
  cudaStream_t s = (cudaStream_t)stream;
  const float* in = features;
  for (int l = 0; l < num_layers; ++l) {
    float* out = l == num_layers - 1 ? act_out : d->act[l & 1];
    const int rc = ds_launch_layer(d, l, params, in, out, n, s);
    if (rc != TCR_OK) return rc;
    in = out;
  }
  if (cudaGetLastError() != cudaSuccess) { set_error("DS-CNN launch failed"); return TCR_ERR_CUDA; }
  return TCR_OK;
}
