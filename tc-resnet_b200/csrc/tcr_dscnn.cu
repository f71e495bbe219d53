// tcr_dscnn.cu — DS-CNN (Hello-Edge) forward pass for sm_90a: the reference's 2-D-conv comparison model
// (audio_nets/ds_cnn.py:20-118, BASELINE.json config 5), inference mode.
//
//   dscnn_conv_kernel      first layer: kh x kw conv from the single-channel feature map (+bias, BN, ReLU); like the wgmma
//                          first-layer kernels it has a windowed instantiation (WIN = true) that reads utterance u in place from a
//                          listener's feature history (WindowView, tcr_listener.cu) instead of from a [n, height, width] tensor
//   dscnn_dsblock_kernel   depthwise 3x3 (+bias, BN, ReLU) -> pointwise 1x1 (+bias, BN, ReLU) fused per tile of output rows:
//                          the input rows (+halo) and both filter banks are staged in shared memory, the depthwise result
//                          never leaves the SM, the pointwise conv is a register-tiled 4 positions x 4 channels contraction
//   dscnn_head_kernel      global average pool + fully connected (+bias) + softmax
// and the KWS baselines of audio_nets/kws.py on the same handle (sizes 'P' trad_fpool3, 'F' one_fstride4): kws_conv_kernel (FMA
// first layers), kws_bsplit_kernel + kws_conv2_tc_kernel (trad_fpool3's 64 -> 64 conv on wgmma), kws_lin_kernel + kws_head_kernel
// (the dense head); KWSModel's speech_commands nets ('C' low_latency_conv, 'Y' tiny_conv): kws_llconv_kernel (the T x 8 conv as an
// FMA implicit GEMM), kws_tinyconv_kernel (10 x 8 SAME / stride 2), kws_fcs_kernel + kws_fcb_head_kernel (dense head with biases);
// and the 2-D ablations of TC-ResNet8 ('R' ResNet2D8, 'A' ResNet2D8Pool): res2d_conv0_kernel (conv0, the pool
// fused), res2d_block_kernel (one fused residual block), res2d_head_kernel (dscnn_head without the bias); and Honk's ResNets of
// audio_nets/res.py ('E' Res8, 'N' Res8Narrow, 'D' Res15, 'T' Res15Narrow): res_fconv_kernel (f_conv, Res8's pool fused),
// res_conv_kernel (one dilated 3x3 conv, its residual add and BatchNorm in the epilogue), and res2d_head_kernel.
// BatchNorm here has no gamma (slim default scale=False) and uses the moving statistics; bias + BN fold into one
// per-channel (scale, shift) pair computed while staging.
#ifndef TCR_EMU
#include <cuda.h>   // CUtensorMap (types only: the encoder is looked up through the runtime)
#endif
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <initializer_list>

#include "tcr_bn.cuh"
#include "tcr_net.h"

namespace tcr {

struct DsLayerDev {
  int type;                 // 0 conv, 1 separable, 2 (kLayerKws) VALID bias-free conv + ReLU of the KWS baselines, 3 (kLayerRes2d)
                            // a layer of the 2-D ablations (its R2Conv0 / R2Block is in the handle), 4 (kLayerRes) a layer of
                            // Res8 / Res15 (its ResFconv / ResConv is in the handle), 5 (kLayerKwsB) the conv of low_latency_conv or
                            // tiny_conv (its KwsLlConv / KwsTinyConv is in the handle)
  int cin, cout, kh, kw, sh, sw, hin, win, hout, wout, pt, pl;
  int64_t w, b, beta, mm, mv;                // conv / depthwise
  int64_t pw, pb, pbeta, pmm, pmv;           // pointwise (separable only)
};

constexpr int kDsMaxLayers = 16;      // Res15: f_conv and 13 convs (DsNet is host-only)
constexpr int kLayerKws = 2;
constexpr int kLayerRes2d = 3;
constexpr int kLayerRes = 4;
constexpr int kLayerKwsB = 5;
struct DsNet {
  int nlayers, n, classes;
  DsLayerDev layer[kDsMaxLayers];
  int64_t fcw, fcb;
};

// A layer of the KWS baselines (audio_nets/kws.py): VALID, bias-free convolution + ReLU, in [n][hin][win][cin] -> out
// [n][hout][wout][cout] NHWC, w [kh][kw][cin][cout] at params + w; wout counts pooled columns where the layer max-pools over width
// (hout rows are walked in tiles of RH by the FMA kernel).
struct KwsConv {
  int cin, cout, kh, kw, sh, sw, hin, win, hout, wout, RH;
  int64_t w;
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

// Utterance n of the first layer's windowed input: at in + (n / k) * stream + (n % k) * step floats, its height x width features
// back to back.
__device__ __forceinline__ const float* ds_window(const float* in, int n, const WindowView& win) {
  return in + (int64_t)(n / win.k) * win.stream + (int64_t)(n % win.k) * win.step;
}

// ---- first layer: cin == 1 ----
template <bool WIN>
__global__ void __launch_bounds__(256) dscnn_conv_kernel(DsLayerDev L, const float* __restrict__ params, const float* __restrict__ in,
                                                         float* __restrict__ out, float eps, WindowView win) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  const DsSmem S = conv_smem(L);
  const int hp = ds_in_rows(L, L.hout), wp = ds_in_cols(L);      // padded input extent
  float *xs = smem, *ws = smem + S.b, *sc = smem + S.tab, *sf = sc + L.cout;
  const int n = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < hp * wp; i += blockDim.x) {
    const int h = i / wp - L.pt, w = i % wp - L.pl;
    if constexpr (WIN) xs[i] = (h >= 0 && h < L.hin && w >= 0 && w < L.win) ? ds_window(in, n, win)[h * L.win + w] : 0.f;
    else xs[i] = (h >= 0 && h < L.hin && w >= 0 && w < L.win) ? in[((size_t)n * L.hin + h) * L.win + w] : 0.f;
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
  // input rows of the tile starting at output row h0 of utterance n -> xs [hin_t][wp]; WIN: utterance n is a window (ds_window)
  template <bool WIN>
  __device__ __forceinline__ void fetch(const DsLayerDev& L, const float* in, int n, int h0, float* xs, const WindowView& win) const {
    const int hb = h0 * L.sh - L.pt;
    const float* base;
    if constexpr (WIN) base = ds_window(in, n, win) + (int64_t)hb * L.win - L.pl;
    else base = in + ((int64_t)n * L.hin + hb) * L.win - L.pl;
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
template <int CO, bool WIN>
__global__ void __launch_bounds__(kTcThreads, 1) dscnn_conv_ws_kernel(DsLayerDev L, int RH, int n_utt, const float* __restrict__ params,
                                                                      const float* __restrict__ in, float* __restrict__ out, float eps,
                                                                      WindowView win) {
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
      walk.fetch<WIN>(L, in, n, (tile - n * tpu) * RH, xs, win);
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
template <int CO, bool WIN>
__global__ void __launch_bounds__(kTcThreads, 1) dscnn_conv_tc_kernel(DsLayerDev L, int RH, int n_utt, const float* __restrict__ params,
                                                                      const float* __restrict__ in, float* __restrict__ out, float eps,
                                                                      WindowView win) {
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
    walk.fetch<WIN>(L, in, n, (tile - n * tpu) * RH, xs, win);
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

// ---- cnn-trad-fpool3's second convolution (audio_nets/kws.py:242-254) as an implicit GEMM on wgmma (3xTF32) ----
// 10 x 4 VALID, 64 -> 64 channels, ReLU: M = output positions flattened over (utterance, oh, ow), K = 40 taps x 64 channels = 2,560,
// N = 64.  The 655 KB filter bank cannot stay in shared memory, so K is streamed in chunks of 32 (half a tap's channels) through
// a ring of kC2Stages stages, each holding that chunk's A (128 rows, hi / lo) and B (64 columns, hi / lo):
//   warps 0-7   producers: thread 0 bulk-copies the chunk's B (split once per forward by kws_bsplit_kernel into the stage's exact
//               image) and the 256 threads gather A, the 128-byte channel halves of the NHWC input at (oh + i, ow + j), split it
//               and store it in the K-major layout, the next chunk's gathers already in flight; one arrival each, the bulk
//               copy's bytes on the same `full` barrier;
//   warps 8-11  consumer warpgroup: per chunk 3 passes x 4 k-steps of two wgmma m64n64k8 (rows 0-63, 64-127), one commit group
//               per chunk kept in flight: once the previous chunk's group has completed its stage is handed back (`empty`).
//               Every kC2Flush chunks (K = 256) the accumulators are folded into a register sum with fp32 adds and restarted
//               (scale-d = 0): the error of the tensor cores' own accumulation grows with K, and over all 2,560 at once it reached
//               2.1e-5 of the layer's maximum, over the 1e-5 layer bound; in blocks of 256 it is 1.1e-6 to 1.5e-6.
// A tile is 128 consecutive output rows, so tiles span utterances and the last one is partial (its missing rows are zero A rows
// whose accumulator rows are not stored); the grid is persistent and walks the tiles with its own stride.
constexpr int kC2Chunk = 32, kC2Stages = 4, kC2Producers = 256, kC2Threads = kC2Producers + 128, kC2Flush = 8;
constexpr int kC2Lbb = 64 * 4;                                          // B image: K-chunk-of-4 stride in floats (no padding)
constexpr int kC2AFloats = 2 * (kC2Chunk / 4) * kLbaFull;              // A hi, lo [8][kLbaFull]
constexpr int kC2BFloats = 2 * (kC2Chunk / 4) * kC2Lbb;                // B hi, lo [8][64 x 4]: 16 KB, one bulk copy
constexpr int kC2StageFloats = kC2AFloats + kC2BFloats;                // 49,408 bytes, a multiple of 16

// Filter bank w [K][64] -> the B stage image of every chunk c: hi then lo, element (co, k) at (k % 32 / 4) * 256 + co * 4 + k % 4.
__global__ void __launch_bounds__(256) kws_bsplit_kernel(int K, const float* __restrict__ w, float* __restrict__ img) {
  pdl_wait();
  for (int i = blockIdx.x * 256 + threadIdx.x; i < K * 64; i += gridDim.x * 256) {
    const int k = i >> 6, co = i & 63, kk = k % kC2Chunk;
    const float v = __ldg(w + i), hi = tf32_hi(v);
    float* dst = img + (size_t)(k / kC2Chunk) * kC2BFloats + (kk >> 2) * kC2Lbb + co * 4 + (kk & 3);
    dst[0] = hi;
    dst[kC2BFloats / 2] = v - hi;
  }
}

// D[64 x 64] = A B^T (ACC = 0: the accumulator's old value is ignored, scale-d = 0) or D += A B^T (ACC = 1)
template <int ACC>
__device__ __forceinline__ void wgmma_m64n64k8_tf32_sd(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(ACC)
      : "memory");
}
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

__global__ void __launch_bounds__(kC2Threads, 1) kws_conv2_tc_kernel(KwsConv L, int n_utt, const float* __restrict__ bimg,
                                                                     const float* __restrict__ in, float* __restrict__ out) {
  TCR_DYNAMIC_SMEM(smem_raw);
  __shared__ uint64_t full[kC2Stages], empty[kC2Stages];
  float* smem = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x;
  const int npos = L.hout * L.wout, rows = n_utt * npos, ntiles = (rows + 127) / 128;
  const int cpt = L.cin / kC2Chunk, nchunks = L.kh * L.kw * cpt;       // chunks per tap, per tile
  if (tid == 0) {
    for (int s = 0; s < kC2Stages; ++s) {
      mbar_init(&full[s], kC2Producers + 1);                           // + thread 0's expect_tx
      mbar_init(&empty[s], 128);
    }
  }
  pdl_wait();
  __syncthreads();
  if (tid < kC2Producers) {
    const int q = tid & 7, m0 = tid >> 3;                              // float4 q of a row's 32 channels; rows m0 + 32 r
    int64_t base[4];
    bool ok[4];
    uint32_t g = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = tile * 128 + m0 + 32 * r;
        ok[r] = row < rows;
        const int rr = ok[r] ? row : 0, n = rr / npos, p = rr - n * npos, oh = p / L.wout, ow = p - oh * L.wout;
        base[r] = (((int64_t)n * L.hin + oh) * L.win + ow) * L.cin + 4 * q;
      }
      auto load = [&](int c, float4 (&v)[4]) {                        // chunk c's A rows of this thread, into registers
        const int tap = c / cpt, ti = tap / L.kw, tj = tap - ti * L.kw;
        const int64_t off = ((int64_t)ti * L.win + tj) * L.cin + (c - tap * cpt) * kC2Chunk;
#pragma unroll
        for (int r = 0; r < 4; ++r) v[r] = ok[r] ? ldg4(in + base[r] + off) : make_float4(0.f, 0.f, 0.f, 0.f);
      };
      float4 v[4], nxt[4];
      load(0, v);
      for (int c = 0; c < nchunks; ++c, ++g) {
        const int s = g % kC2Stages;
        if (c + 1 < nchunks) load(c + 1, nxt);                         // in flight while this chunk is split and stored
        if (g >= kC2Stages) mbar_wait(&empty[s], ((g / kC2Stages) - 1) & 1);      // the MMAs of chunk g - kC2Stages are done
        float* a_hi = smem + (size_t)s * kC2StageFloats;
        float* a_lo = a_hi + (kC2Chunk / 4) * kLbaFull;
        if (tid == 0) {
          mbar_expect_tx(&full[s], kC2BFloats * 4);
          tma_load_1d(a_hi + kC2AFloats, bimg + (size_t)c * kC2BFloats, kC2BFloats * 4, &full[s]);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float4 hi, lo;
          tf32_split(v[r], hi, lo);
          st4(a_hi + q * kLbaFull + 4 * (m0 + 32 * r), hi);
          st4(a_lo + q * kLbaFull + 4 * (m0 + 32 * r), lo);
          v[r] = nxt[r];
        }
        fence_proxy_async();                                           // operand stores -> visible to the async proxy (wgmma)
        mbar_arrive(&full[s]);
      }
    }
  } else {
    const int wtid = tid - kC2Producers;
    uint32_t g = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      float acc[2][32], sum[2][32];                                    // acc is (re)started by the block's first MMA (scale-d = 0)
#pragma unroll
      for (int i = 0; i < 32; ++i) { sum[0][i] = 0.f; sum[1][i] = 0.f; }
      for (int cb = 0; cb < nchunks; cb += kC2Flush) {                // nchunks is a multiple of kC2Flush (host side)
#pragma unroll
        for (int cc = 0; cc < kC2Flush; ++cc, ++g) {
          const int s = g % kC2Stages;
          mbar_wait(&full[s], (g / kC2Stages) & 1);
          const float* a_hi = smem + (size_t)s * kC2StageFloats;
          const float* b_hi = a_hi + kC2AFloats;
          const uint64_t da_hi = gmma_desc(smem_u32(a_hi), kLbaFull * 4u, 128u);
          const uint64_t da_lo = gmma_desc(smem_u32(a_hi + (kC2Chunk / 4) * kLbaFull), kLbaFull * 4u, 128u);
          const uint64_t db_hi = gmma_desc(smem_u32(b_hi), kC2Lbb * 4u, 128u);
          const uint64_t db_lo = gmma_desc(smem_u32(b_hi + kC2BFloats / 2), kC2Lbb * 4u, 128u);
          wgmma_fence();
#pragma unroll
          for (int pass = 0; pass < 3; ++pass) {                       // lo*hi, hi*lo, hi*hi
            const uint64_t da0 = pass == 0 ? da_lo : da_hi, db0 = pass == 1 ? db_lo : db_hi;
#pragma unroll
            for (int ks = 0; ks < kC2Chunk / 8; ++ks) {
              const uint64_t da = da0 + (uint64_t)((2 * ks * kLbaFull * 4) >> 4), db = db0 + (uint64_t)((2 * ks * kC2Lbb * 4) >> 4);
              if (cc == 0 && pass == 0 && ks == 0) {
                wgmma_m64n64k8_tf32_sd<0>(acc[0], da, db);
                wgmma_m64n64k8_tf32_sd<0>(acc[1], da + (uint64_t)((64 * 16) >> 4), db);
              } else {
                wgmma_m64n64k8_tf32_sd<1>(acc[0], da, db);
                wgmma_m64n64k8_tf32_sd<1>(acc[1], da + (uint64_t)((64 * 16) >> 4), db);
              }
            }
          }
          wgmma_commit();
          if (cc > 0) {
            wgmma_wait_1();                                            // the previous chunk's MMAs have read their stage
            mbar_arrive(&empty[(g - 1) % kC2Stages]);
          }
        }
        wgmma_wait_all();
        mbar_arrive(&empty[(g - 1) % kC2Stages]);
#pragma unroll
        for (int i = 0; i < 32; ++i) { sum[0][i] += acc[0][i]; sum[1][i] += acc[1][i]; }
      }
      // ReLU + NHWC store: accumulator row m of the tile is output row tile * 128 + m (d[4 j + 2 h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e])
      const int r0 = 16 * (wtid >> 5) + ((wtid & 31) >> 2), c0 = 2 * (wtid & 3);
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {                               // rows r0, r0 + 8, r0 + 64, r0 + 72
          const int row = tile * 128 + r0 + 8 * (qq & 1) + 64 * (qq >> 1);
          if (row < rows) {
            const float* a = &sum[qq >> 1][4 * j + 2 * (qq & 1)];
            *reinterpret_cast<float2*>(out + (size_t)row * 64 + 8 * j + c0) = make_float2(fmaxf(a[0], 0.f), fmaxf(a[1], 0.f));
          }
        }
    }
  }
}

// ---- cnn-trad-fpool3's first convolution + ReLU + 1 x 3 max-pool (audio_nets/kws.py:223-240) as an implicit GEMM on wgmma ----
// 20 x 8 VALID, 1 -> 64 channels, 3xTF32: K = 160 taps, N = 64.  The accumulator rows of a tile are 42 pooled outputs x their 3
// pre-pool columns (row m: pooled output tile * 42 + m / 3, column 3 * owp + m % 3; rows 126 and 127 are zero), flattened over
// (utterance, oh, owp), so a pooling window never straddles tiles and only the pooled map reaches HBM.  Persistent, lock-step
// (like dscnn_conv_tc): the split filter bank stays in shared memory for all the CTA's tiles; per tile and half of K, every thread
// gathers its row's 4-tap chunks straight from the feature map (4 taps of a chunk are 4 consecutive columns of one row, read
// through L1) into the K-major A operand (hi / lo), then the four warpgroups each issue the 3 passes x 10 k-steps of one
// m64n32k8 quarter of the accumulator.  Epilogue: ReLU into shared memory (over the A region), then the max over each row
// triple, stored NHWC.  WIN: utterance n is a listener window (ds_window).
constexpr int kC1Pooled = 42, kC1Half = 20;                           // pooled outputs per tile; K chunks of 4 per half of K
constexpr int kC1Ep = 65;                                              // epilogue scratch row stride (floats)
TCR_HD inline size_t conv1_tc_smem_floats(int K4) { return 2 * (size_t)K4 * gmma_lbb(64) + 2 * (size_t)kC1Half * kLbaFull; }
// D[64 x 32] = A B^T (ACC = 0, scale-d = 0) or D += A B^T (ACC = 1)
template <int ACC>
__device__ __forceinline__ void wgmma_m64n32k8_tf32_sd(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "n"(ACC)
      : "memory");
}

template <bool WIN>
__global__ void __launch_bounds__(kTcThreads, 1) kws_conv1_tc_kernel(KwsConv L, int n_utt, const float* __restrict__ params,
                                                                     const float* __restrict__ in, float* __restrict__ out,
                                                                     WindowView win) {
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x;
  const int K = L.kh * L.kw, K4 = K / 4;                              // host side: K4 == 2 * kC1Half, kw a multiple of 4
  constexpr int LBB = gmma_lbb(64);
  float *b_hi = smem, *b_lo = b_hi + (size_t)K4 * LBB;
  float *a_hi = b_lo + (size_t)K4 * LBB, *a_lo = a_hi + kC1Half * kLbaFull;
  float* ep = a_hi;                                                   // [128][kC1Ep] once the tile's MMAs are done
  stage_b<kTcThreads, 64, 1>(params + L.w, K, b_hi, b_lo, tid);
  pdl_wait();
  const int per_utt = L.hout * L.wout, total = n_utt * per_utt, ntiles = (total + kC1Pooled - 1) / kC1Pooled;
  const int g = tid >> 7, wtid = tid & 127, m0 = 64 * (g & 1), col0 = 32 * (g >> 1);    // this warpgroup's quarter
  const uint64_t da_hi = gmma_desc(smem_u32(a_hi + 4 * m0), kLbaFull * 4u, 128u), da_lo = gmma_desc(smem_u32(a_lo + 4 * m0), kLbaFull * 4u, 128u);
  const uint64_t db_hi = gmma_desc(smem_u32(b_hi + 4 * col0), LBB * 4u, 128u), db_lo = gmma_desc(smem_u32(b_lo + 4 * col0), LBB * 4u, 128u);
  fence_proxy_async();                                                // the B operand was written through the generic proxy
  const int m = tid & 127, cq = tid >> 7;                             // the gather: A row m, chunks cq + 4 j of each half
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int p = tile * kC1Pooled + m / 3;
    const bool ok = m < 3 * kC1Pooled && p < total;
    const float* xr = in;
    if (ok) {
      const int n = p / per_utt, r = p - n * per_utt, oh = r / L.wout, owp = r - oh * L.wout;
      const float* utt;
      if constexpr (WIN) utt = ds_window(in, n, win);
      else utt = in + (int64_t)n * L.hin * L.win;
      xr = utt + (int64_t)oh * L.win + 3 * owp + (m - 3 * (m / 3));
    }
    float acc[16];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      for (int c = cq; c < kC1Half; c += 4) {
        const int k0 = 4 * (half * kC1Half + c), i = k0 / L.kw, j = k0 - i * L.kw;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok) {
          const float* s = xr + i * L.win + j;
          v = make_float4(__ldg(s), __ldg(s + 1), __ldg(s + 2), __ldg(s + 3));
        }
        float4 hi, lo;
        tf32_split(v, hi, lo);
        st4(a_hi + c * kLbaFull + 4 * m, hi);
        st4(a_lo + c * kLbaFull + 4 * m, lo);
      }
      fence_proxy_async();                                            // operand stores -> visible to the async proxy (wgmma)
      __syncthreads();
      wgmma_fence();
      // opaque copies: the per-k-step descriptors are formed here, not hoisted out of the tile loop (60 of them would spill)
      uint64_t dal = da_lo, dah = da_hi, dbl = db_lo, dbh = db_hi;
      asm volatile("" : "+l"(dal), "+l"(dah), "+l"(dbl), "+l"(dbh));
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {                          // lo*hi, hi*lo, hi*hi
        const uint64_t da0 = pass == 0 ? dal : dah, db0 = pass == 1 ? dbl : dbh;
#pragma unroll
        for (int ks = 0; ks < kC1Half / 2; ++ks) {
          const uint64_t da = da0 + (uint64_t)((2 * ks * kLbaFull * 4) >> 4);
          const uint64_t db = db0 + (uint64_t)(((2 * ks + half * kC1Half) * LBB * 4) >> 4);
          if (half == 0 && pass == 0 && ks == 0) wgmma_m64n32k8_tf32_sd<0>(acc, da, db);
          else wgmma_m64n32k8_tf32_sd<1>(acc, da, db);
        }
      }
      wgmma_commit();
      wgmma_wait_all();
      __syncthreads();                                                // every warpgroup has read A: refill it / reuse it as `ep`
    }
    // ReLU into ep (d[4 j + 2 h + e] = D[m0 + 16 w + l / 4 + 8 h][col0 + 8 j + 2 (l % 4) + e]), then the max over row triples
    const int r0 = m0 + 16 * (wtid >> 5) + ((wtid & 31) >> 2), c0 = col0 + 2 * (wtid & 3);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        ep[(r0 + 8 * h) * kC1Ep + c0 + 8 * j] = fmaxf(acc[4 * j + 2 * h], 0.f);
        ep[(r0 + 8 * h) * kC1Ep + c0 + 8 * j + 1] = fmaxf(acc[4 * j + 2 * h + 1], 0.f);
      }
    __syncthreads();
    for (int idx = tid; idx < kC1Pooled * 64; idx += kTcThreads) {
      const int pp = idx >> 6, co = idx & 63, po = tile * kC1Pooled + pp;
      if (po < total) {
        const float* e = ep + 3 * pp * kC1Ep + co;
        out[(int64_t)po * 64 + co] = fmaxf(fmaxf(e[0], e[kC1Ep]), e[2 * kC1Ep]);
      }
    }
    __syncthreads();                                                  // ep is the next tile's A
  }
}
#endif

// ---- head: one CTA per utterance ----
// Global average pool, fully connected layer and softmax; BIAS = false is the bias-free fc of the 2-D ablations (res2d_head_kernel).
template <bool BIAS>
__device__ __forceinline__ void dscnn_head(int npos, int C, int classes, int64_t fcw, int64_t fcb, const float* __restrict__ params,
                                           const float* __restrict__ in, float* __restrict__ logits, float* __restrict__ probs) {
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
    float acc = BIAS ? params[fcb + tid] : 0.f;
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
__global__ void __launch_bounds__(256) dscnn_head_kernel(int npos, int C, int classes, int64_t fcw, int64_t fcb,
                                                         const float* __restrict__ params, const float* __restrict__ in,
                                                         float* __restrict__ logits, float* __restrict__ probs) {
  dscnn_head<true>(npos, C, classes, fcw, fcb, params, in, logits, probs);
}

// ---- KWS baselines: FMA convolution, one CTA per (utterance, tile of L.RH output rows), blockIdx.x = n * tiles + tile ----
// cnn-trad-fpool3's first layer (20 x 8, 1 -> 64, ReLU, max-pool 1 x 3 / stride 3: POOL = 3, only the pooled map is stored) and
// cnn-one-fstride4's only one (T x 8, stride 4 in frequency, 1 -> 186); the emulator build, which has no wgmma, also runs the
// 64 -> 64 second layer of trad_fpool3 here.  The tile's input rows are staged in shared memory.  A thread owns CPT consecutive
// output channels (CPT = 4: float4 filter loads, cout a multiple of 4; CPT = 1: any channel count) and RT output rows x CT output
// columns x POOL pre-pool columns, so one filter load feeds RT * CT * POOL * CPT FMAs and one input load CPT.  Consecutive threads
// take consecutive channel groups: a warp's filter loads are one coalesced row and its input loads broadcasts.  Rows and columns
// past the tile re-read its last one and are not stored.  WIN: utterance n is a listener window (ds_window).
constexpr int kKwsMaxStaged = 51200;                                  // floats of input rows the FMA kernel stages (200 KB)
TCR_HD inline int kws_stage_floats(const KwsConv& L) { return ((L.RH - 1) * L.sh + L.kh) * L.win * L.cin; }
template <int POOL, int CPT, int RT, int CT, bool WIN>
__global__ void __launch_bounds__(256, 2) kws_conv_kernel(KwsConv L, const float* __restrict__ params, const float* __restrict__ in,
                                                       float* __restrict__ out, WindowView win) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* xs = reinterpret_cast<float*>(smem_raw);
  const int tpu = (L.hout + L.RH - 1) / L.RH, tid = threadIdx.x;
  const int n = blockIdx.x / tpu, h0 = (blockIdx.x - n * tpu) * L.RH, rh = imin(L.RH, L.hout - h0);
  const int rowlen = L.win * L.cin, staged = ((rh - 1) * L.sh + L.kh) * rowlen;
  const float* src;
  if constexpr (WIN) src = ds_window(in, n, win) + (int64_t)h0 * L.sh * rowlen;
  else src = in + ((int64_t)n * L.hin + (int64_t)h0 * L.sh) * rowlen;
  for (int i = tid; i < staged; i += blockDim.x) xs[i] = src[i];
  __syncthreads();
  const int ncg = L.cout / CPT, ncol = (L.wout + CT - 1) / CT;
  const int ntask = ncg * ncol * ((rh + RT - 1) / RT);
  for (int task = tid; task < ntask; task += blockDim.x) {
    const int cg = task % ncg, t1 = task / ncg, ow0 = (t1 % ncol) * CT, r0 = (t1 / ncol) * RT;
    int xoff[RT][CT];                                             // staged-tile offset of each (row, column)'s first tap
#pragma unroll
    for (int r = 0; r < RT; ++r)
#pragma unroll
      for (int q = 0; q < CT; ++q) xoff[r][q] = imin(r0 + r, rh - 1) * L.sh * rowlen + imin(ow0 + q, L.wout - 1) * POOL * L.sw * L.cin;
    float acc[RT][CT][POOL][CPT];
#pragma unroll
    for (int r = 0; r < RT; ++r)
#pragma unroll
      for (int q = 0; q < CT; ++q)
#pragma unroll
        for (int e = 0; e < POOL; ++e)
#pragma unroll
          for (int k = 0; k < CPT; ++k) acc[r][q][e][k] = 0.f;
    const float* wc = params + L.w + CPT * cg;
    for (int i = 0; i < L.kh; ++i)
      for (int j = 0; j < L.kw; ++j) {
        const float* xb = xs + i * rowlen + j * L.cin;
        const float* wb = wc + (int64_t)(i * L.kw + j) * L.cin * L.cout;
        for (int ci = 0; ci < L.cin; ++ci) {
          float wv[CPT];
          if constexpr (CPT == 4) {
            const float4 w4 = ldg4(wb + (int64_t)ci * L.cout);
            wv[0] = w4.x; wv[1] = w4.y; wv[2] = w4.z; wv[3] = w4.w;
          } else {
            wv[0] = __ldg(wb + (int64_t)ci * L.cout);
          }
#pragma unroll
          for (int r = 0; r < RT; ++r)
#pragma unroll
            for (int q = 0; q < CT; ++q)
#pragma unroll
              for (int e = 0; e < POOL; ++e) {
                const float x = xb[xoff[r][q] + e * L.sw * L.cin + ci];
#pragma unroll
                for (int k = 0; k < CPT; ++k) acc[r][q][e][k] = fmaf(x, wv[k], acc[r][q][e][k]);
              }
        }
      }
#pragma unroll
    for (int r = 0; r < RT; ++r)
#pragma unroll
      for (int q = 0; q < CT; ++q) {
        if (r0 + r < rh && ow0 + q < L.wout) {
          float* o = out + (((int64_t)n * L.hout + h0 + r0 + r) * L.wout + ow0 + q) * L.cout + CPT * cg;
#pragma unroll
          for (int k = 0; k < CPT; ++k) {
            float v = 0.f;                                        // ReLU, then the max over the pooling window
#pragma unroll
            for (int e = 0; e < POOL; ++e) v = fmaxf(v, acc[r][q][e][k]);
            o[k] = v;
          }
        }
      }
  }
}

// ---- KWS baselines' dense head: flatten -> lin (K x 32) -> 128 (-> 128) -> classes, no nonlinearity, then softmax ----
// The matrices are applied one at a time, in the reference's order.  lin is split over K: CTA (utterance group, K chunk s) stages
// kKwsLinK rows of the weights once for kKwsLinU utterances and writes partial sums part[s][u][32]; kws_head_kernel adds the
// chunks in order, so the logits of an utterance do not depend on the batch it is in.
constexpr int kKwsLinK = 256, kKwsLinU = 64, kKwsHeadU = 16;
constexpr size_t kKwsLinSmem = (size_t)(kKwsLinK * 32 + kKwsLinU * (kKwsLinK + 1)) * 4;
struct KwsHead { int K, nsplit, nfc, classes; int64_t lin, fc[2], out; };

__global__ void __launch_bounds__(256) kws_lin_kernel(KwsHead H, int n, const float* __restrict__ params, const float* __restrict__ in,
                                                      float* __restrict__ part) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);                 // [kKwsLinK][32]
  float* xs = ws + kKwsLinK * 32;                                 // [kKwsLinU][kKwsLinK + 1]
  const int s = blockIdx.x % H.nsplit, u0 = (blockIdx.x / H.nsplit) * kKwsLinU, tid = threadIdx.x;
  const int k0 = s * kKwsLinK, kc = imin(kKwsLinK, H.K - k0), nu = imin(kKwsLinU, n - u0);
  for (int i = tid; i < kc * 32; i += blockDim.x) ws[i] = __ldg(params + H.lin + (int64_t)k0 * 32 + i);
  for (int i = tid; i < nu * kc; i += blockDim.x) {               // K need not be a multiple of 4 (one_fstride4: 1,674)
    const int u = i / kc, k = i - u * kc;
    xs[u * (kKwsLinK + 1) + k] = in[(int64_t)(u0 + u) * H.K + k0 + k];
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;                     // lane = output column, warp = utterances warp + 8 i
  float acc[kKwsLinU / 8];
#pragma unroll
  for (int i = 0; i < kKwsLinU / 8; ++i) acc[i] = 0.f;
  for (int k = 0; k < kc; ++k) {
    const float w = ws[k * 32 + lane];
#pragma unroll
    for (int i = 0; i < kKwsLinU / 8; ++i) acc[i] = fmaf(xs[(warp + 8 * i) * (kKwsLinK + 1) + k], w, acc[i]);
  }
#pragma unroll
  for (int i = 0; i < kKwsLinU / 8; ++i)
    if (warp + 8 * i < nu) part[((int64_t)s * n + u0 + warp + 8 * i) * 32 + lane] = acc[i];
}

// kKwsHeadU utterances per CTA of 128 threads: every weight of the 128-wide matrices is loaded once per CTA.
__global__ void __launch_bounds__(128) kws_head_kernel(KwsHead H, int n, const float* __restrict__ params, const float* __restrict__ part,
                                                       float* __restrict__ logits, float* __restrict__ probs) {
  pdl_wait();
  __shared__ float h[2][kKwsHeadU][128];
  __shared__ float s_logit[kKwsHeadU][kMaxClasses];
  const int u0 = blockIdx.x * kKwsHeadU, nu = imin(kKwsHeadU, n - u0), tid = threadIdx.x, C = H.classes;
  for (int i = tid; i < kKwsHeadU * 32; i += blockDim.x) {
    const int u = i >> 5, j = i & 31;
    float a = 0.f;
    if (u < nu)
      for (int s = 0; s < H.nsplit; ++s) a += part[((int64_t)s * n + u0 + u) * 32 + j];
    h[0][u][j] = a;
  }
  __syncthreads();
  int cur = 0, width = 32;
  for (int m = 0; m < H.nfc; ++m, cur ^= 1, width = 128) {
    const float* W = params + H.fc[m];
    float acc[kKwsHeadU];
#pragma unroll
    for (int u = 0; u < kKwsHeadU; ++u) acc[u] = 0.f;
    for (int k = 0; k < width; ++k) {
      const float w = __ldg(W + k * 128 + tid);
#pragma unroll
      for (int u = 0; u < kKwsHeadU; ++u) acc[u] = fmaf(h[cur][u][k], w, acc[u]);
    }
#pragma unroll
    for (int u = 0; u < kKwsHeadU; ++u) h[cur ^ 1][u][tid] = acc[u];
    __syncthreads();
  }
  for (int i = tid; i < nu * C; i += blockDim.x) {
    const int u = i / C, c = i - u * C;
    float a = 0.f;
    for (int k = 0; k < 128; ++k) a = fmaf(h[cur][u][k], __ldg(params + H.out + k * C + c), a);
    s_logit[u][c] = a;
    if (logits) logits[(int64_t)(u0 + u) * C + c] = a;
  }
  __syncthreads();
  if (!probs) return;
  for (int i = tid; i < nu * C; i += blockDim.x) {
    const int u = i / C, c = i - u * C;
    float mx = -3.0e38f;
    for (int k = 0; k < C; ++k) mx = fmaxf(mx, s_logit[u][k]);
    float se = 0.f;
    for (int k = 0; k < C; ++k) se += expf(s_logit[u][k] - mx);
    probs[(int64_t)(u0 + u) * C + c] = expf(s_logit[u][c] - mx) / se;
  }
}

// ---- KWSModel's speech_commands nets (audio_nets/kws.py): low_latency_conv ('C') and tiny_conv ('Y'), evaluation mode ----
// Every layer has a bias.  low_latency_conv: T x 8 VALID conv 1 -> 186 + bias + ReLU, then fc 128, fc 128, fc classes (each + bias,
// no nonlinearity: the training dropouts are the identity).  tiny_conv: 10 x 8 TF-SAME conv at stride 2 x 2, 1 -> 8 + bias + ReLU,
// then fc classes + bias.  Both flatten NHWC.

// low_latency_conv's conv as an implicit GEMM on the FMA pipe: rows m = (utterance, output column), M = n * wout, K = T * 8 taps,
// N = 186 channels padded to 192.  A CTA computes kLlBM rows x 192 channels; a thread 8 rows x 12 channels.  The K loop walks one
// filter row (8 taps) per step: its 8 x kLlBM im2col slice and 8 x 192 weights are staged in shared memory, the next step's loaded
// into registers while the current one is multiplied.  Every output is one fmaf chain in tap order whatever tile it falls in, so
// an utterance's bits do not depend on its batch.  WIN: utterance u is a listener window (ds_window).
constexpr int kLlBM = 128, kLlBN = 192, kLlCout = 186, kLlThreads = 256;
constexpr size_t kLlSmem = (size_t)2 * 8 * (kLlBM + kLlBN) * 4;
struct KwsLlConv { int hin, win, wout, M; int64_t w, b; };
template <bool WIN>
__global__ void __launch_bounds__(kLlThreads, 1) kws_llconv_kernel(KwsLlConv L, const float* __restrict__ params,
                                                                 const float* __restrict__ in, float* __restrict__ out, WindowView win) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* as = reinterpret_cast<float*>(smem_raw);                 // [2][8][kLlBM]
  float* bs = as + 2 * 8 * kLlBM;                                 // [2][8][kLlBN]
  const int tid = threadIdx.x, m0 = blockIdx.x * kLlBM;
  // staging: A row am, taps aj0 .. aj0 + 3; B elements tid + 256 q of the step's [8][192] slice (channels past 186 are zeros)
  const int am = tid & (kLlBM - 1), aj0 = (tid >> 7) * 4;
  const int mrow = imin(m0 + am, L.M - 1), u = mrow / L.wout, col = mrow - u * L.wout;
  const float* arow = (WIN ? ds_window(in, u, win) : in + (int64_t)u * L.hin * L.win) + col + aj0;
  int boff[6];
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    const int e = tid + kLlThreads * q, j = e / kLlBN, c = e - j * kLlBN;
    boff[q] = c < kLlCout ? j * kLlCout + c : -1;
  }
  float ra[4], rb[6];
  auto load = [&](int i) {
#pragma unroll
    for (int k = 0; k < 4; ++k) ra[k] = arow[(int64_t)i * L.win + k];
    const float* wr = params + L.w + (int64_t)i * 8 * kLlCout;
#pragma unroll
    for (int q = 0; q < 6; ++q) rb[q] = boff[q] >= 0 ? __ldg(wr + boff[q]) : 0.f;
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int k = 0; k < 4; ++k) as[(buf * 8 + aj0 + k) * kLlBM + am] = ra[k];
#pragma unroll
    for (int q = 0; q < 6; ++q) bs[buf * 8 * kLlBN + tid + kLlThreads * q] = rb[q];
  };
  const int tx = tid & 15, ty = tid >> 4;                         // channels 12 tx .. 12 tx + 11, rows 8 ty .. 8 ty + 7
  float acc[8][12];
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int c = 0; c < 12; ++c) acc[r][c] = 0.f;
  load(0);
  store(0);
  __syncthreads();
  for (int i = 0; i < L.hin; ++i) {
    const int cur = i & 1;
    if (i + 1 < L.hin) load(i + 1);
    const float* ab = as + cur * 8 * kLlBM + 8 * ty;
    const float* bb = bs + cur * 8 * kLlBN + 12 * tx;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 a0 = ld4(ab + j * kLlBM), a1 = ld4(ab + j * kLlBM + 4);
      const float4 b0 = ld4(bb + j * kLlBN), b1 = ld4(bb + j * kLlBN + 4), b2 = ld4(bb + j * kLlBN + 8);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[12] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w, b2.x, b2.y, b2.z, b2.w};
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 12; ++c) acc[r][c] = fmaf(a[r], b[c], acc[r][c]);
    }
    if (i + 1 < L.hin) store(cur ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int c = 0; c < 12; ++c) {
    const int ch = 12 * tx + c;
    if (ch >= kLlCout) break;
    const float bias = __ldg(params + L.b + ch);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int m = m0 + 8 * ty + r;
      if (m < L.M) out[(int64_t)m * kLlCout + ch] = fmaxf(acc[r][c] + bias, 0.f);
    }
  }
}

// tiny_conv's conv: 10 x 8, TF SAME at stride 2 x 2 (pt rows above, pl columns left: the smaller half of each total), 1 -> 8 +
// bias + ReLU.  One CTA per (utterance, tile of RH output rows), blockIdx.x = n * tiles + tile.  The tile's 2 RH + 8 input rows
// are staged with the padding as zeros (xw = 2 wout + 6 columns), and the taps and bias; a thread computes all 8 channels of one
// output position.  WIN: utterance n is a listener window, padded with zeros at the window's edges like any other input: the
// history frames before it are not read.
struct KwsTinyConv { int hin, win, hout, wout, pt, pl, RH, xw; int64_t w, b; };
TCR_HD inline size_t kws_tiny_smem_floats(const KwsTinyConv& L) { return 648 + (size_t)(2 * L.RH + 8) * L.xw; }
template <bool WIN>
__global__ void __launch_bounds__(256) kws_tinyconv_kernel(KwsTinyConv L, const float* __restrict__ params, const float* __restrict__ in,
                                                           float* __restrict__ out, WindowView win) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);                 // [80 taps][8]
  float* bs = ws + 640;                                           // [8]
  float* xs = ws + 648;                                           // [2 RH + 8][xw]
  const int tpu = (L.hout + L.RH - 1) / L.RH, tid = threadIdx.x;
  const int n = blockIdx.x / tpu, h0 = (blockIdx.x - n * tpu) * L.RH, rh = imin(L.RH, L.hout - h0);
  const float* src = WIN ? ds_window(in, n, win) : in + (int64_t)n * L.hin * L.win;
  const int r0 = 2 * h0 - L.pt, staged = (2 * rh + 8) * L.xw;
  for (int i = tid; i < staged; i += blockDim.x) {
    const int r = i / L.xw, gr = r0 + r, gc = i - r * L.xw - L.pl;
    xs[i] = gr >= 0 && gr < L.hin && gc >= 0 && gc < L.win ? src[(int64_t)gr * L.win + gc] : 0.f;
  }
  for (int i = tid; i < 648; i += blockDim.x) ws[i] = __ldg(params + (i < 640 ? L.w + i : L.b + i - 640));
  __syncthreads();
  for (int p = tid; p < rh * L.wout; p += blockDim.x) {
    const int r = p / L.wout, q = p - r * L.wout;
    const float* x = xs + 2 * r * L.xw + 2 * q;
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    for (int i = 0; i < 10; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v = x[i * L.xw + j];
        const float4 w0 = ld4(ws + (i * 8 + j) * 8), w1 = ld4(ws + (i * 8 + j) * 8 + 4);
        acc[0] = fmaf(v, w0.x, acc[0]); acc[1] = fmaf(v, w0.y, acc[1]); acc[2] = fmaf(v, w0.z, acc[2]); acc[3] = fmaf(v, w0.w, acc[3]);
        acc[4] = fmaf(v, w1.x, acc[4]); acc[5] = fmaf(v, w1.y, acc[5]); acc[6] = fmaf(v, w1.z, acc[6]); acc[7] = fmaf(v, w1.w, acc[7]);
      }
    float* o = out + (((int64_t)n * L.hout + h0 + r) * L.wout + q) * 8;
    st4(o, make_float4(fmaxf(acc[0] + bs[0], 0.f), fmaxf(acc[1] + bs[1], 0.f), fmaxf(acc[2] + bs[2], 0.f), fmaxf(acc[3] + bs[3], 0.f)));
    st4(o + 4, make_float4(fmaxf(acc[4] + bs[4], 0.f), fmaxf(acc[5] + bs[5], 0.f), fmaxf(acc[6] + bs[6], 0.f), fmaxf(acc[7] + bs[7], 0.f)));
  }
}

// Their dense heads.  The first matmul (K = the flattened conv output) is split over K: CTA (utterance group, K chunk s) stages KC
// rows of the weights ([K, N], N <= 32 NQ columns, zero-padded) once for 64 utterances and writes partial sums part[s][u][32 NQ].
// kws_fcb_head_kernel adds the chunks in order and the bias, applies the remaining matrices (+ bias) one at a time, and the
// softmax, so the logits of an utterance do not depend on the batch it is in.  low_latency_conv: first_fc (N = 128, NQ = 4), then
// second_fc and final_fc in the head kernel; tiny_conv: final_fc is the split matmul (N = classes, NQ = 1).
struct KwsFcb { int K, N0, nsplit, nmid, classes; int64_t w0, b0, mid, midb, out, outb; };
template <int NQ, int KC>
constexpr size_t kws_fcs_smem() { return (size_t)(KC * 32 * NQ + 64 * (KC + 1)) * 4; }
template <int NQ, int KC>
__global__ void __launch_bounds__(256) kws_fcs_kernel(KwsFcb H, int n, const float* __restrict__ params, const float* __restrict__ in,
                                                      float* __restrict__ part) {
  pdl_wait();
  constexpr int NP = 32 * NQ;
  TCR_DYNAMIC_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);                 // [KC][NP]
  float* xs = ws + KC * NP;                                       // [64][KC + 1]
  const int s = blockIdx.x % H.nsplit, u0 = (blockIdx.x / H.nsplit) * 64, tid = threadIdx.x;
  const int k0 = s * KC, kc = imin(KC, H.K - k0), nu = imin(64, n - u0);
  for (int i = tid; i < kc * NP; i += blockDim.x) {
    const int k = i / NP, c = i - k * NP;
    ws[i] = c < H.N0 ? __ldg(params + H.w0 + (int64_t)(k0 + k) * H.N0 + c) : 0.f;
  }
  for (int i = tid; i < nu * kc; i += blockDim.x) {
    const int u = i / kc, k = i - u * kc;
    xs[u * (KC + 1) + k] = in[(int64_t)(u0 + u) * H.K + k0 + k];
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;                     // columns lane + 32 q, utterances warp + 8 i
  float acc[8][NQ];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int q = 0; q < NQ; ++q) acc[i][q] = 0.f;
  for (int k = 0; k < kc; ++k) {
    float w[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) w[q] = ws[k * NP + lane + 32 * q];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float x = xs[(warp + 8 * i) * (KC + 1) + k];
#pragma unroll
      for (int q = 0; q < NQ; ++q) acc[i][q] = fmaf(x, w[q], acc[i][q]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (warp + 8 * i < nu)
#pragma unroll
      for (int q = 0; q < NQ; ++q) part[((int64_t)s * n + u0 + warp + 8 * i) * NP + lane + 32 * q] = acc[i][q];
}

// kKwsHeadU utterances per CTA of 128 threads; the partial sums' row stride is N0 rounded up to 32.
__global__ void __launch_bounds__(128) kws_fcb_head_kernel(KwsFcb H, int n, const float* __restrict__ params, const float* __restrict__ part,
                                                           float* __restrict__ logits, float* __restrict__ probs) {
  pdl_wait();
  __shared__ float h[2][kKwsHeadU][128];
  __shared__ float s_logit[kKwsHeadU][kMaxClasses];
  const int u0 = blockIdx.x * kKwsHeadU, nu = imin(kKwsHeadU, n - u0), tid = threadIdx.x, C = H.classes;
  const int NP = (H.N0 + 31) & ~31;
  for (int i = tid; i < kKwsHeadU * H.N0; i += blockDim.x) {
    const int u = i / H.N0, j = i - u * H.N0;
    float a = 0.f;
    if (u < nu) {
      for (int s = 0; s < H.nsplit; ++s) a += part[((int64_t)s * n + u0 + u) * NP + j];
      a += __ldg(params + H.b0 + j);
    }
    h[0][u][j] = a;
  }
  __syncthreads();
  int cur = 0;
  for (int m = 0; m < H.nmid; ++m, cur ^= 1) {                    // 128 -> 128 (+ bias)
    const float* W = params + H.mid;
    float acc[kKwsHeadU];
#pragma unroll
    for (int u = 0; u < kKwsHeadU; ++u) acc[u] = 0.f;
    for (int k = 0; k < 128; ++k) {
      const float w = __ldg(W + k * 128 + tid);
#pragma unroll
      for (int u = 0; u < kKwsHeadU; ++u) acc[u] = fmaf(h[cur][u][k], w, acc[u]);
    }
    const float b = __ldg(params + H.midb + tid);
#pragma unroll
    for (int u = 0; u < kKwsHeadU; ++u) h[cur ^ 1][u][tid] = acc[u] + b;
    __syncthreads();
  }
  for (int i = tid; i < nu * C; i += blockDim.x) {
    const int u = i / C, c = i - u * C;
    float a = h[cur][u][c];                                       // tiny_conv: the split matmul's output are the logits
    if (H.out >= 0) {
      a = 0.f;
      for (int k = 0; k < 128; ++k) a = fmaf(h[cur][u][k], __ldg(params + H.out + k * C + c), a);
      a += __ldg(params + H.outb + c);
    }
    s_logit[u][c] = a;
    if (logits) logits[(int64_t)(u0 + u) * C + c] = a;
  }
  __syncthreads();
  if (!probs) return;
  for (int i = tid; i < nu * C; i += blockDim.x) {
    const int u = i / C, c = i - u * C;
    float mx = -3.0e38f;
    for (int k = 0; k < C; ++k) mx = fmaxf(mx, s_logit[u][k]);
    float se = 0.f;
    for (int k = 0; k < C; ++k) se += expf(s_logit[u][k] - mx);
    probs[(int64_t)(u0 + u) * C + c] = expf(s_logit[u][c] - mx) / se;
  }
}

// ---- ResNet2D8 / ResNet2D8Pool: the paper's 2-D ablations of TC-ResNet8 (audio_nets/tc_resnet.py:6-54, 73-101, debug_2d) ----
// Evaluation mode.  No conv has a bias, and BatchNorm has gamma (TCResNet_arg_scope: center and scale):
// (beta, gamma, moving mean, moving variance) fold into scale = gamma / sqrt(var + eps) and shift = beta - mean * scale.
// Channel counts need not be multiples of 4 (conv0 has 23 at 98 x 40): the block kernel's shared-memory tiles pad them to a
// multiple of 4 with zeros, and zero scale and shift keep the padded intermediate channels at 0.
constexpr int kR2MaxChannels = 128;
struct R2Bn { int64_t beta, gamma, mm, mv; };
__device__ __forceinline__ void r2_fold(const float* p, const R2Bn& bn, int c, int C, float eps, float* sc, float* sf) {
  float s = 0.f, t = 0.f;
  if (c < C) {
    s = p[bn.gamma + c] / sqrtf(p[bn.mv + c] + eps);
    t = fmaf(-p[bn.mm + c], s, p[bn.beta + c]);
  }
  sc[c] = s;
  sf[c] = t;
}
TCR_HD inline int r2_pad4(int c) { return (c + 3) & ~3; }

// conv0: 3 x 3 / stride 1 SAME conv of the single-channel features + BN + ReLU; for ResNet2D8Pool (pool = 4) the 4 x 4 / stride 4
// VALID average pool in the epilogue, so only the pooled map is stored.  One CTA per (utterance, tile of RH output rows),
// blockIdx.x = n * tiles + tile.  The tile's RH * pool + 2 input rows, with SAME's one-pixel zero border, the taps and the folded
// BatchNorm are staged in shared memory.  A thread owns one channel (its 9 taps and BatchNorm in registers) and walks output
// positions 256 / cout apart.  WIN: utterance n is a listener window (ds_window); the border is zeros there too, never the
// neighbouring history frames.
struct R2Conv0 { int hin, win, hout, wout, cout, pool, RH; int64_t w; R2Bn bn; };
TCR_HD inline size_t r2_conv0_smem_floats(const R2Conv0& L) { return (size_t)(L.RH * L.pool + 2) * (L.win + 2) + 11 * (size_t)L.cout; }
template <bool WIN>
__global__ void __launch_bounds__(256) res2d_conv0_kernel(R2Conv0 L, const float* __restrict__ params, const float* __restrict__ in,
                                                          float* __restrict__ out, float eps, WindowView win) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* xs = reinterpret_cast<float*>(smem_raw);
  const int tpu = (L.hout + L.RH - 1) / L.RH, tid = threadIdx.x;
  const int n = blockIdx.x / tpu, h0 = (blockIdx.x - n * tpu) * L.RH, rh = imin(L.RH, L.hout - h0);
  const int xr = L.RH * L.pool + 2, xc = L.win + 2, r0 = h0 * L.pool - 1;       // staged rows, padded width, first input row
  float *ws = xs + xr * xc, *sc = ws + 9 * L.cout, *sf = sc + L.cout;
  const float* src;
  if constexpr (WIN) src = ds_window(in, n, win);
  else src = in + (int64_t)n * L.hin * L.win;
  for (int i = tid; i < xr * xc; i += blockDim.x) {
    const int h = r0 + i / xc, w = i % xc - 1;
    xs[i] = (h >= 0 && h < L.hin && w >= 0 && w < L.win) ? src[(int64_t)h * L.win + w] : 0.f;
  }
  for (int i = tid; i < 9 * L.cout; i += blockDim.x) ws[i] = params[L.w + i];
  for (int c = tid; c < L.cout; c += blockDim.x) r2_fold(params, L.bn, c, L.cout, eps, sc, sf);
  __syncthreads();
  const float inv = 1.f / (float)(L.pool * L.pool);
  const int c = tid % L.cout, pstep = blockDim.x / L.cout, npos = rh * L.wout;   // cout <= kR2MaxChannels < blockDim.x
  if (tid >= pstep * L.cout) return;
  float wk[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) wk[k] = ws[k * L.cout + c];
  const float s = sc[c], t = sf[c];
  int r = (tid / L.cout) / L.wout, ow = (tid / L.cout) - r * L.wout;
  for (int pos = tid / L.cout; pos < npos; pos += pstep) {
    float sum = 0.f;
    for (int py = 0; py < L.pool; ++py)
      for (int px = 0; px < L.pool; ++px) {
        const float* xb = xs + (r * L.pool + py) * xc + ow * L.pool + px;
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
          for (int j = 0; j < 3; ++j) acc = fmaf(xb[i * xc + j], wk[3 * i + j], acc);
        sum += fmaxf(fmaf(acc, s, t), 0.f);
      }
    out[(((int64_t)n * L.hout + h0 + r) * L.wout + ow) * L.cout + c] = L.pool == 1 ? sum : sum * inv;
    ow += pstep;
    while (ow >= L.wout) { ow -= L.wout; ++r; }
  }
}

// A residual block: conv_0 (3 x 3 / stride s, SAME with leading pads pt, pl) + BN + ReLU, conv_1 (3 x 3 / stride 1, SAME) + BN, the
// shortcut (down: 1 x 1 / stride s + BN + ReLU where the channel count changes, else the input), the add and ReLU.  One CTA per
// (utterance, tile of RH x WT output positions), blockIdx.x = n * tiles + tile.  The tile's input (rows and columns of conv_0's
// receptive field around the RH + 2 x WT + 2 intermediate positions conv_1 reads) is staged once; conv_0's output for those
// positions, zero outside the map (conv_1's SAME border), stays in shared memory.  The filter banks pass through shared memory in
// slices of COT output channels, conv_0's first and then conv_1's with the matching slice of down.
struct R2Block {
  int cin, cout, s, hin, win, hout, wout, pt, pl, down;
  int RH, WT, COT;
  int64_t w0, w1, wd;
  R2Bn bn0, bn1, bnd;
};
// Shared-memory layout in floats: x the input tile [xr][xc][cin padded], m the intermediate [RH + 2][WT + 2][cout padded], w one
// filter slice ([9][cin or cout padded][COT], then down's [cin padded][COT]), tab the six folded-BatchNorm tables.
struct R2Smem { size_t m, w, tab, floats; int xr, xc; };
TCR_HD inline R2Smem r2_block_smem(const R2Block& B) {
  const int cip = r2_pad4(B.cin), cop = r2_pad4(B.cout);
  R2Smem S;
  S.xr = (B.RH + 1) * B.s + 3;
  S.xc = (B.WT + 1) * B.s + 3;
  S.m = (size_t)S.xr * S.xc * cip;
  S.w = S.m + (size_t)(B.RH + 2) * (B.WT + 2) * cop;
  S.tab = S.w + (size_t)(9 * (cip > cop ? cip : cop) + (B.down ? cip : 0)) * B.COT;
  S.floats = S.tab + 6 * (size_t)cop;
  return S;
}

// K x K conv of a staged tile for one slice of cot output channels: output position p (npos of them, `cols` per row) reads the
// [.][xc][cip] tile x0 at row (p / cols) * s + i, column (p % cols) * s + j; w is [K * K][cip][cot].  Tasks of kR2TM positions
// (NRT apart) x 4 channels, so that one float4 of the filter feeds kR2TM positions; epi(p, cg, acc) takes each result.
constexpr int kR2TM = 4;
template <int K, class Epi>
__device__ __forceinline__ void r2_conv(const float* x0, int xc, int cip, int s, int npos, int cols, const float* w, int cot, Epi epi) {
  const int ncg = cot >> 2, NRT = (npos + kR2TM - 1) / kR2TM;
  for (int task = threadIdx.x; task < NRT * ncg; task += blockDim.x) {
    const int cg = task % ncg, rt = task / ncg;
    const float* xr[kR2TM];
#pragma unroll
    for (int m = 0; m < kR2TM; ++m) {
      const int p = imin(rt + m * NRT, npos - 1), r = p / cols, c = p - r * cols;
      xr[m] = x0 + ((size_t)r * s * xc + (size_t)c * s) * cip;
    }
    float4 acc[kR2TM];
#pragma unroll
    for (int m = 0; m < kR2TM; ++m) acc[m] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < K; ++i)
      for (int j = 0; j < K; ++j) {
        const float* wk = w + (size_t)(i * K + j) * cip * cot + 4 * cg;
        const int xo = (i * xc + j) * cip;
#pragma unroll 2
        for (int ci = 0; ci < cip; ci += 4) {
          const float4 w0 = ld4(wk + (ci + 0) * cot), w1 = ld4(wk + (ci + 1) * cot), w2 = ld4(wk + (ci + 2) * cot), w3 = ld4(wk + (ci + 3) * cot);
#pragma unroll
          for (int m = 0; m < kR2TM; ++m) {
            const float4 x = ld4(xr[m] + xo + ci);
            float4& a = acc[m];
            a.x = fmaf(x.x, w0.x, a.x); a.y = fmaf(x.x, w0.y, a.y); a.z = fmaf(x.x, w0.z, a.z); a.w = fmaf(x.x, w0.w, a.w);
            a.x = fmaf(x.y, w1.x, a.x); a.y = fmaf(x.y, w1.y, a.y); a.z = fmaf(x.y, w1.z, a.z); a.w = fmaf(x.y, w1.w, a.w);
            a.x = fmaf(x.z, w2.x, a.x); a.y = fmaf(x.z, w2.y, a.y); a.z = fmaf(x.z, w2.z, a.z); a.w = fmaf(x.z, w2.w, a.w);
            a.x = fmaf(x.w, w3.x, a.x); a.y = fmaf(x.w, w3.y, a.y); a.z = fmaf(x.w, w3.z, a.z); a.w = fmaf(x.w, w3.w, a.w);
          }
        }
      }
#pragma unroll
    for (int m = 0; m < kR2TM; ++m)
      if (rt + m * NRT < npos) epi(rt + m * NRT, cg, acc[m]);
  }
}

// Filter slice: w [taps][C][CO] at params + off -> ws [taps][cp][cot], output channels co0 .. co0 + cot, zeros past C and CO.
__device__ __forceinline__ void r2_stage_slice(float* ws, const float* params, int64_t off, int taps, int C, int cp, int CO, int co0, int cot) {
  for (int i = threadIdx.x; i < taps * cp * cot; i += blockDim.x) {
    const int co = i % cot, ci = (i / cot) % cp, k = i / (cot * cp);
    ws[i] = (ci < C && co0 + co < CO) ? params[off + ((int64_t)k * C + ci) * CO + co0 + co] : 0.f;
  }
}

__global__ void __launch_bounds__(256) res2d_block_kernel(R2Block B, const float* __restrict__ params, const float* __restrict__ in,
                                                          float* __restrict__ out, float eps) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  const R2Smem S = r2_block_smem(B);
  const int cip = r2_pad4(B.cin), cop = r2_pad4(B.cout), tid = threadIdx.x;
  const int tcols = (B.wout + B.WT - 1) / B.WT, tpu = ((B.hout + B.RH - 1) / B.RH) * tcols;
  const int n = blockIdx.x / tpu, t = blockIdx.x - n * tpu, h0 = (t / tcols) * B.RH, w0 = (t % tcols) * B.WT;
  const int rh = imin(B.RH, B.hout - h0), wt = imin(B.WT, B.wout - w0), mc = wt + 2;
  float *xs = smem, *ms = smem + S.m, *ws = smem + S.w, *tab = smem + S.tab;
  float *sc0 = tab, *sf0 = tab + cop, *sc1 = tab + 2 * cop, *sf1 = tab + 3 * cop, *scd = tab + 4 * cop, *sfd = tab + 5 * cop;
  // input rows (h0 - 1) * s - pt + [0, xr), columns (w0 - 1) * s - pl + [0, xc): conv_0's taps for intermediate rows h0 - 1 ..
  // h0 + RH and columns w0 - 1 .. w0 + WT; zeros outside the map and past cin
  {
    const int xh0 = (h0 - 1) * B.s - B.pt, xw0 = (w0 - 1) * B.s - B.pl;
    const float* src = in + (int64_t)n * B.hin * B.win * B.cin;
    for (int i = tid; i < S.xr * S.xc * cip; i += blockDim.x) {
      const int c = i % cip, cell = i / cip, h = xh0 + cell / S.xc, w = xw0 + cell % S.xc;
      xs[i] = (c < B.cin && h >= 0 && h < B.hin && w >= 0 && w < B.win) ? src[((int64_t)h * B.win + w) * B.cin + c] : 0.f;
    }
  }
  for (int c = tid; c < cop; c += blockDim.x) {
    r2_fold(params, B.bn0, c, B.cout, eps, sc0, sf0);
    r2_fold(params, B.bn1, c, B.cout, eps, sc1, sf1);
    if (B.down) r2_fold(params, B.bnd, c, B.cout, eps, scd, sfd);
  }
  // conv_0 + BN + ReLU -> ms [rh + 2][wt + 2][cop]
  for (int co0 = 0; co0 < cop; co0 += B.COT) {
    const int cot = imin(B.COT, cop - co0);
    __syncthreads();                                              // the previous slice's readers are done
    r2_stage_slice(ws, params, B.w0, 9, B.cin, cip, B.cout, co0, cot);
    __syncthreads();
    r2_conv<3>(xs, S.xc, cip, B.s, (rh + 2) * mc, mc, ws, cot, [&](int p, int cg, float4 a) {
      const int r = p / mc, c = p - r * mc, h = h0 - 1 + r, w = w0 - 1 + c, co = co0 + 4 * cg;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (h >= 0 && h < B.hout && w >= 0 && w < B.wout) v = bn_relu4(a, ld4(sc0 + co), ld4(sf0 + co));
      st4(ms + (size_t)p * cop + co, v);
    });
  }
  // conv_1 + BN, the shortcut, add, ReLU -> out
  for (int co0 = 0; co0 < cop; co0 += B.COT) {
    const int cot = imin(B.COT, cop - co0);
    __syncthreads();
    r2_stage_slice(ws, params, B.w1, 9, B.cout, cop, B.cout, co0, cot);
    float* wd = ws + (size_t)9 * cop * cot;
    if (B.down) r2_stage_slice(wd, params, B.wd, 1, B.cin, cip, B.cout, co0, cot);
    __syncthreads();
    r2_conv<3>(ms, mc, cop, 1, rh * wt, wt, ws, cot, [&](int p, int cg, float4 a) {
      const int r = p / wt, c = p - r * wt, co = co0 + 4 * cg;
      const float4 s1 = ld4(sc1 + co), t1 = ld4(sf1 + co);
      float4 v = make_float4(fmaf(a.x, s1.x, t1.x), fmaf(a.y, s1.y, t1.y), fmaf(a.z, s1.z, t1.z), fmaf(a.w, s1.w, t1.w));
      // the shortcut's input cell: output (h0 + r, w0 + c) reads input ((h0 + r) * s, (w0 + c) * s)
      const float* xb = xs + ((size_t)((r + 1) * B.s + B.pt) * S.xc + (size_t)(c + 1) * B.s + B.pl) * cip;
      float4 sh;
      if (B.down) {
        float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int ci = 0; ci < cip; ++ci) {
          const float x = xb[ci];
          const float4 k = ld4(wd + (size_t)ci * cot + 4 * cg);
          d.x = fmaf(x, k.x, d.x); d.y = fmaf(x, k.y, d.y); d.z = fmaf(x, k.z, d.z); d.w = fmaf(x, k.w, d.w);
        }
        sh = bn_relu4(d, ld4(scd + co), ld4(sfd + co));
      } else {
        sh = ld4(xb + co);
      }
      v = make_float4(fmaxf(v.x + sh.x, 0.f), fmaxf(v.y + sh.y, 0.f), fmaxf(v.z + sh.z, 0.f), fmaxf(v.w + sh.w, 0.f));
      float* o = out + (((int64_t)n * B.hout + h0 + r) * B.wout + w0 + c) * B.cout + co;
      if ((B.cout & 3) == 0) {
        st4(o, v);
      } else {
        const float vv[4] = {v.x, v.y, v.z, v.w};
        for (int k = 0; k < 4 && co + k < B.cout; ++k) o[k] = vv[k];
      }
    });
  }
}

// head: global average pool, fc (no bias), softmax
__global__ void __launch_bounds__(256) res2d_head_kernel(int npos, int C, int classes, int64_t fcw, const float* __restrict__ params,
                                                         const float* __restrict__ in, float* __restrict__ logits, float* __restrict__ probs) {
  dscnn_head<false>(npos, C, classes, fcw, 0, params, in, logits, probs);
}

// ---- Res8 / Res8Narrow / Res15 / Res15Narrow: Honk's ResNets as the reference builds them (audio_nets/res.py) ----
// Evaluation mode.  Every conv is bias-free, TF SAME at stride 1 and followed by ReLU; BatchNorm has neither beta nor gamma
// (center = scale = False), so the moving statistics fold into scale = 1 / sqrt(var + eps) and shift = -mean * scale.  The head is
// res2d_head_kernel.
struct ResBn { int64_t mm, mv; };
__device__ __forceinline__ void res_fold(const float* p, const ResBn& bn, int c, int C, float eps, float* sc, float* sf) {
  float s = 0.f, t = 0.f;
  if (c < C) {
    s = 1.f / sqrtf(p[bn.mv + c] + eps);
    t = -p[bn.mm + c] * s;
  }
  sc[c] = s;
  sf[c] = t;
}

// 4-byte global -> shared copy; invalid: the destination is zero-filled and nothing is read (cp.async with source size 0).
__device__ __forceinline__ void res_cp4(float* dst, const float* src, bool valid) {
#ifdef TCR_EMU
  *dst = valid ? *src : 0.f;
#else
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 4u : 0u) : "memory");
#endif
}
__device__ __forceinline__ void res_cp_commit() {
#ifndef TCR_EMU
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void res_cp_wait_prev() {             // all but the most recent group have landed
#ifndef TCR_EMU
  asm volatile("cp.async.wait_group 1;" ::: "memory");
#endif
}

// f_conv: 3 x 3 SAME conv of the single-channel features + ReLU; for Res8 (ph x pw = 4 x 3) the stride-1 VALID average pool in the
// same launch, so that only the pooled map reaches HBM.  One CTA per (utterance, tile of RH output rows), blockIdx.x = n * tiles +
// tile.  The tile's input rows with SAME's one-pixel zero border and the taps are staged; with the pool, the RH + ph - 1 rows of
// conv outputs the tile's windows read are staged too.  A thread owns one channel and walks positions 256 / cout apart.  WIN:
// utterance n is a listener window (ds_window); the border is zeros there too, never the neighbouring history frames.
struct ResFconv { int hin, win, hout, wout, cout, ph, pw, RH; int64_t w; };
TCR_HD inline size_t res_fconv_smem_floats(const ResFconv& L) {
  const int cr = L.RH + L.ph - 1;                                 // conv rows of a full tile
  return (size_t)(cr + 2) * (L.win + 2) + (L.ph > 1 ? (size_t)cr * L.win * L.cout : 0) + 9 * (size_t)L.cout;
}
template <bool WIN>
__global__ void __launch_bounds__(256) res_fconv_kernel(ResFconv L, const float* __restrict__ params, const float* __restrict__ in,
                                                        float* __restrict__ out, WindowView win) {
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* xs = reinterpret_cast<float*>(smem_raw);
  const int tpu = (L.hout + L.RH - 1) / L.RH, tid = threadIdx.x, nt = blockDim.x;
  const int n = blockIdx.x / tpu, h0 = (blockIdx.x - n * tpu) * L.RH, rh = imin(L.RH, L.hout - h0);
  const int cr = rh + L.ph - 1, xc = L.win + 2;                   // conv rows of this tile, padded width
  float* cs = xs + (size_t)(L.RH + L.ph + 1) * xc;
  float* ws = cs + (L.ph > 1 ? (size_t)(L.RH + L.ph - 1) * L.win * L.cout : 0);
  const float* src;
  if constexpr (WIN) src = ds_window(in, n, win);
  else src = in + (int64_t)n * L.hin * L.win;
  {  // input rows h0 - 1 .. h0 + cr, columns -1 .. win
    int r = tid / xc, c = tid - r * xc;
    const int dr = nt / xc, dc = nt - dr * xc;
    for (int i = tid; i < (cr + 2) * xc; i += nt) {
      const int h = h0 - 1 + r, w = c - 1;
      xs[i] = (h >= 0 && h < L.hin && w >= 0 && w < L.win) ? src[(int64_t)h * L.win + w] : 0.f;
      r += dr;
      c += dc;
      if (c >= xc) { c -= xc; ++r; }
    }
  }
  for (int i = tid; i < 9 * L.cout; i += nt) ws[i] = params[L.w + i];
  __syncthreads();
  const int c = tid % L.cout, lanes = nt / L.cout;                // cout <= 45 < blockDim.x
  const bool active = tid < lanes * L.cout;
  float wk[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) wk[k] = active ? ws[k * L.cout + c] : 0.f;
  const int dr = lanes / L.win, dc = lanes - dr * L.win;
  if (active) {
    int r = (tid / L.cout) / L.win, ow = (tid / L.cout) - r * L.win;
    for (int q = tid / L.cout; q < cr * L.win; q += lanes) {
      const float* xb = xs + r * xc + ow;
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) acc = fmaf(xb[i * xc + j], wk[3 * i + j], acc);
      const float v = fmaxf(acc, 0.f);
      if (L.ph == 1) out[(((int64_t)n * L.hout + h0 + r) * L.wout + ow) * L.cout + c] = v;
      else cs[((size_t)r * L.win + ow) * L.cout + c] = v;
      r += dr;
      ow += dc;
      if (ow >= L.win) { ow -= L.win; ++r; }
    }
  }
  if (L.ph == 1) return;                                          // uniform across the CTA
  __syncthreads();
  if (!active) return;
  const float inv = 1.f / (float)(L.ph * L.pw);
  const int pr = lanes / L.wout, pc = lanes - pr * L.wout;
  int r = (tid / L.cout) / L.wout, ow = (tid / L.cout) - r * L.wout;
  for (int q = tid / L.cout; q < rh * L.wout; q += lanes) {
    float sum = 0.f;
    for (int py = 0; py < L.ph; ++py)
      for (int px = 0; px < L.pw; ++px) sum += cs[((size_t)(r + py) * L.win + ow + px) * L.cout + c];
    out[(((int64_t)n * L.hout + h0 + r) * L.wout + ow) * L.cout + c] = sum * inv;
    r += pr;
    ow += pc;
    if (ow >= L.wout) { ow -= L.wout; ++r; }
  }
}

// conv{k}: 3 x 3 at dilation d, stride 1, SAME (d zeros on every side), C -> C, then ReLU.  RES = false: then BatchNorm.  RES = true
// (conv{2i+1}, the second conv of block i): + the block's input `res`, then BatchNorm; there is no ReLU after the add.
//
// Persistent CTAs walk tiles of TR whole rows of one utterance (tile t: utterance t / tpu); channels are padded with zeros to CP
// (45 -> 48, 19 -> 20).  Per CTA, once: the filter bank [9][CP][CP] and the folded BatchNorm.  Per tile, three stages, one per tap
// row i: the TR input rows h0 + (i - 1) d .. that the tap row reads, [TR * W][XS] (positions XS floats apart, which keeps a warp's
// eight positions on distinct banks), gathered by 4-byte cp.async (a row of C floats is not 16-byte aligned) with zero fill for
// rows outside the map.  Stages are double-buffered: stage s + 1 is in flight while stage s runs.  A tap's column shift reads
// the same slab d positions over; a position whose shifted column leaves the map reads a zero row instead.
// A thread owns TM positions (SLOTS apart) x TN channels of the tile in registers: CP = 48 as 8 position lanes x 4 channel lanes of
// 12 per warp, CP = 20 as 32 position lanes of all 20 channels.  The epilogue writes ReLU(acc) back into the stage's slab, then
// the tile's rows, contiguous in HBM, are written coalesced with the residual and BatchNorm applied.
// Residual aliasing: in a full forward `out` is the buffer holding the block input `res`; each thread reads its residual element
// before it writes the same element, so neither pointer is __restrict__.
constexpr int kResConvThreads = 256;
template <int CP> struct ResTile;
template <> struct ResTile<48> { static constexpr int CGW = 4, TM = 4; };
template <> struct ResTile<20> { static constexpr int CGW = 1, TM = 2; };
template <int CP> TCR_HD constexpr int res_xs() { return ((CP >> 2) & 1) ? CP : CP + 4; }
template <int CP> TCR_HD constexpr int res_np_max() { return kResConvThreads / 32 * (32 / ResTile<CP>::CGW) * ResTile<CP>::TM; }
template <int CP> TCR_HD inline size_t res_conv_smem_floats(int TR, int W) { return 9 * CP * CP + 3 * CP + 2 * (size_t)TR * W * res_xs<CP>(); }
struct ResConv { int h, w, c, d, TR; int64_t wt; ResBn bn; };

template <int CP, bool RES>
__global__ void __launch_bounds__(kResConvThreads) res_conv_kernel(ResConv L, int n_utt, const float* __restrict__ params,
                                                               const float* __restrict__ in, const float* res, float* out, float eps) {
  constexpr int CGW = ResTile<CP>::CGW, TM = ResTile<CP>::TM, TN = CP / CGW, PG = 32 / CGW, SLOTS = kResConvThreads / 32 * PG;
  constexpr int XS = res_xs<CP>();
  pdl_wait();
  TCR_DYNAMIC_SMEM(smem_raw);
  float* ws = reinterpret_cast<float*>(smem_raw);
  float *sc = ws + 9 * CP * CP, *sf = sc + CP, *zero = sf + CP, *xb = zero + CP;
  const int tid = threadIdx.x, C = L.c, W = L.w, d = L.d, NP = L.TR * W, slab = NP * C;
  const size_t buf = (size_t)NP * XS;
  const int tpu = (L.h + L.TR - 1) / L.TR, ntiles = n_utt * tpu;
  for (int i = tid; i < 9 * CP * CP; i += kResConvThreads) {
    const int co = i % CP, ci = (i / CP) % CP, k = i / (CP * CP);
    ws[i] = (ci < C && co < C) ? params[L.wt + ((int64_t)k * C + ci) * C + co] : 0.f;
  }
  for (int c = tid; c < CP; c += kResConvThreads) {
    res_fold(params, L.bn, c, C, eps, sc, sf);
    zero[c] = 0.f;
  }
  for (int i = tid; i < 2 * NP * (CP - C); i += kResConvThreads) {   // the padded channels of both slabs stay zero
    const int p = i / (CP - C);
    xb[(size_t)p * XS + C + (i - p * (CP - C))] = 0.f;
  }
  // this thread's element walk of a slab (element e of the tile's rows in HBM order -> position p, channel c), stepped without division
  const int p0 = tid / C, c0 = tid - p0 * C, dp = kResConvThreads / C, dc = kResConvThreads - dp * C;
  auto issue = [&](int s) {
    const int t = blockIdx.x + (s / 3) * gridDim.x, i = s - (s / 3) * 3;
    if (t >= ntiles) return;
    const int u = t / tpu, hs = (t - u * tpu) * L.TR + (i - 1) * d;
    const int elo = imax(0, -hs) * W * C, ehi = imax(0, imin(L.TR, L.h - hs)) * W * C;
    const int64_t g0 = ((int64_t)u * L.h + hs) * W * C;
    float* x = xb + (s & 1) * buf;
    int p = p0, c = c0;
    for (int e = tid; e < slab; e += kResConvThreads) {
      const bool v = e >= elo && e < ehi;
      res_cp4(x + (size_t)p * XS + c, v ? in + g0 + e : in, v);
      p += dp;
      c += dc;
      if (c >= C) { c -= C; ++p; }
    }
  };
  // this thread's register tile: positions slot + m * SLOTS of the tile, channels cg * TN ..
  const int lane = tid & 31, slot = (tid >> 5) * PG + lane / CGW, cg = lane % CGW;
  int pos[TM], col[TM];
#pragma unroll
  for (int m = 0; m < TM; ++m) {
    pos[m] = slot + m * SLOTS;
    col[m] = pos[m] % W;
  }
  const int nst = blockIdx.x < ntiles ? 3 * ((ntiles - 1 - blockIdx.x) / gridDim.x + 1) : 0;
  float acc[TM][TN];
  issue(0);
  res_cp_commit();
  for (int s = 0; s < nst; ++s) {
    const int i = s % 3;
    if (s + 1 < nst) issue(s + 1);
    res_cp_commit();
    res_cp_wait_prev();
    __syncthreads();                                              // stage s has landed for every thread
    float* x = xb + (s & 1) * buf;
    if (i == 0) {
#pragma unroll
      for (int m = 0; m < TM; ++m)
#pragma unroll
        for (int k = 0; k < TN; ++k) acc[m][k] = 0.f;
    }
#pragma unroll 1
    for (int j = 0; j < 3; ++j) {
      const int sh = (j - 1) * d;
      const float* xp[TM];
#pragma unroll
      for (int m = 0; m < TM; ++m) {
        const int cc = col[m] + sh;
        xp[m] = (pos[m] < NP && cc >= 0 && cc < W) ? x + (size_t)(pos[m] + sh) * XS : zero;
      }
      const float* wk = ws + (i * 3 + j) * CP * CP + cg * TN;
#pragma unroll 1
      for (int ci = 0; ci < CP; ci += 4) {
        float4 xv[TM];
#pragma unroll
        for (int m = 0; m < TM; ++m) xv[m] = ld4(xp[m] + ci);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float wv[TN];
#pragma unroll
          for (int k = 0; k < TN; k += 4) {
            const float4 w4 = ld4(wk + (ci + q) * CP + k);
            wv[k] = w4.x; wv[k + 1] = w4.y; wv[k + 2] = w4.z; wv[k + 3] = w4.w;
          }
#pragma unroll
          for (int m = 0; m < TM; ++m) {
            const float xq = q == 0 ? xv[m].x : q == 1 ? xv[m].y : q == 2 ? xv[m].z : xv[m].w;
#pragma unroll
            for (int k = 0; k < TN; ++k) acc[m][k] = fmaf(xq, wv[k], acc[m][k]);
          }
        }
      }
    }
    if (i == 2) {
      __syncthreads();                                            // every warp is done reading slab s & 1
#pragma unroll
      for (int m = 0; m < TM; ++m)
        if (pos[m] < NP)
#pragma unroll
          for (int k = 0; k < TN; ++k)
            if (cg * TN + k < C) x[(size_t)pos[m] * XS + cg * TN + k] = fmaxf(acc[m][k], 0.f);
      __syncthreads();
      const int t = blockIdx.x + (s / 3) * gridDim.x, u = t / tpu, h0 = (t - u * tpu) * L.TR;
      const int64_t g0 = ((int64_t)u * L.h + h0) * W * C;
      const int cnt = imin(L.TR, L.h - h0) * W * C;
      // eight residual loads in flight before the first store: `out` may alias `res`, so the compiler cannot hoist them itself
      constexpr int kRun = 8;
      int p = p0, c = c0;
      for (int e0 = tid; e0 < cnt; e0 += kRun * kResConvThreads) {
        float r[kRun];
#pragma unroll
        for (int q = 0; q < kRun; ++q) {
          const int e = e0 + q * kResConvThreads;
          r[q] = (RES && e < cnt) ? res[g0 + e] : 0.f;
        }
#pragma unroll
        for (int q = 0; q < kRun; ++q) {
          const int e = e0 + q * kResConvThreads;
          if (e < cnt) out[g0 + e] = fmaf(x[(size_t)p * XS + c] + r[q], sc[c], sf[c]);
          p += dp;
          c += dc;
          if (c >= C) { c -= C; ++p; }
        }
      }
    }
    __syncthreads();                                              // slab s & 1 is free for stage s + 2
  }
}

}  // namespace tcr

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
using namespace tcr;

// How a layer of DS-CNN S / M / L runs, worked out once by ds_plan_layer in tcr_dscnn_create: the kernel, its tile rows (RHt of the
// wgmma kernels, RH of dscnn_dsblock; 0 for dscnn_conv, which stages a whole utterance), dscnn_dsblock's output-channel slice COT,
// and the dynamic shared memory of the launch.
enum DsKernel { kDsConv, kDsConvTc, kDsConvWs, kDsBlock, kDsBlockTc, kDsBlockWs };
struct DsPlan { int kernel, RH, COT; size_t smem; };

struct tcr_dscnn {
  tcr_dscnn_config cfg;
  DsNet net;
  DsPlan plan[kDsMaxLayers] = {};   // DS-CNN S / M / L: each layer's kernel, tile and shared memory
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
  Frontend fe;               // tcr_dscnn_set_frontend: the wav front-end in front of conv_1 (fe.frames == 0: none yet)
  float* feat = nullptr;     // [max_batch, height, width]: the features of a wav-input forward
  // KWS baselines ('P', 'F'): layers of type kLayerKws, their pooling, the dense head and its buffers
  bool kws = false;
  int pool[kDsMaxLayers] = {};
  KwsHead head = {};
  float* part = nullptr;     // [head.nsplit][max_batch][32]: lin's partial sums per K chunk
  float* bimg = nullptr;     // trad_fpool3: conv2's filter bank split into hi / lo B stage images (kws_bsplit_kernel)
  // 2-D ablations ('R', 'A'): layer 0 is conv0 (+ pool), layers 1-3 the residual blocks; fc's offset
  bool res2d = false;
  R2Conv0 r2conv0 = {};
  R2Block r2block[3] = {};
  int64_t r2fc = 0;
  // Res8 / Res15 ('E', 'N', 'D', 'T'): layer 0 is f_conv (+ pool), layer k + 1 conv{k}; fc's offset
  bool res = false;
  ResFconv rfconv = {};
  ResConv rconv[13] = {};
  int64_t rfc = 0;
  // low_latency_conv / tiny_conv ('C', 'Y'): the conv's plan and the dense head (its partial sums in `part`)
  bool kwsb = false;
  KwsLlConv llconv = {};
  KwsTinyConv tiny = {};
  KwsFcb fcb = {};
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

static int ds_fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  set_error(buf);
  return code;
}

static void ds_same(int len, int k, int s, int* out, int* lead) {
  *out = (len + s - 1) / s;
  const int total = std::max((*out - 1) * s + k - len, 0);
  *lead = total / 2;
}

// The 2-D ablations' layers and variables: conv0 (+ pool), three residual blocks, fc and the dead fc2, named and ordered as
// tcr_param_table's TCResNet8 rows (tcr_api.cu): per conv its weights, BatchNorm beta and gamma, then fc and fc2, then the moving
// statistics per conv.  Also each kernel's tile plan, and the refusals of what the kernels cannot run.
template <class Add>
static int res2d_define(tcr_dscnn* d, Add& add) {
  const tcr_dscnn_config& c = d->cfg;
  const bool pool = c.size == TCR_RES2D8_POOL;
  const char* model = pool ? "ResNet2D8Pool" : "ResNet2D8";
  const double wm = c.width_multiplier == 0.0 ? 1.0 : c.width_multiplier;
  int ch[4] = {16, 24, 32, 48};
  for (int& x : ch) x = (int)((double)x * wm);                     // int(x * width_multiplier), tc_resnet.py:75
  if (ch[0] >= 1 && ch[1] >= 1)                                    // first_c, tc_resnet.py:80: exact integers, one rounded division
    ch[0] = (int)((double)(3ll * c.width * ch[0] + 10ll * ch[0] * ch[1]) / (double)(9 + 10ll * ch[1]));
  for (int i = 0; i < 4; ++i)
    if (ch[i] < 1 || ch[i] > kR2MaxChannels)
      return ds_fail(TCR_ERR_UNSUPPORTED, "%s at width_multiplier %g and width %d needs %d channels in %s; res2d_block takes 1 to %d",
                     model, wm, c.width, ch[i], i ? "a block" : "conv0", kR2MaxChannels);
  struct Conv { std::string name; int k, cin, cout; int64_t w; R2Bn bn; };
  std::vector<Conv> convs = {{"conv0", 3, 1, ch[0], 0, {}}};
  for (int i = 0, cin = ch[0]; i < 3; cin = ch[++i]) {
    const std::string b = "block" + std::to_string(i) + "/";
    if (ch[i + 1] != cin) convs.push_back({b + "down", 1, cin, ch[i + 1], 0, {}});
    convs.push_back({b + "conv" + std::to_string(i) + "_0", 3, cin, ch[i + 1], 0, {}});
    convs.push_back({b + "conv" + std::to_string(i) + "_1", 3, ch[i + 1], ch[i + 1], 0, {}});
  }
  const std::string scope = std::string(model) + "/";
  for (Conv& cv : convs) {
    cv.w = add(scope + cv.name + "/weights", TCR_KIND_WEIGHT, {cv.k, cv.k, cv.cin, cv.cout});
    cv.bn.beta = add(scope + cv.name + "/BatchNorm/beta", TCR_KIND_BETA, {cv.cout});
    cv.bn.gamma = add(scope + cv.name + "/BatchNorm/gamma", TCR_KIND_GAMMA, {cv.cout});
  }
  d->r2fc = add(scope + "fc/weights", TCR_KIND_WEIGHT, {1, 1, ch[3], c.num_classes});
  add(scope + "fc2/weights", TCR_KIND_WEIGHT, {1, 1, ch[3], 2});
  for (Conv& cv : convs) {
    cv.bn.mm = add(scope + cv.name + "/BatchNorm/moving_mean", TCR_KIND_MOVING_MEAN, {cv.cout});
    cv.bn.mv = add(scope + cv.name + "/BatchNorm/moving_variance", TCR_KIND_MOVING_VAR, {cv.cout});
  }
  auto layer = [&](int hin, int win, int hout, int wout, int cin, int cout) {
    DsLayerDev L;
    memset(&L, 0, sizeof(L));
    L.type = kLayerRes2d; L.cin = cin; L.cout = cout; L.hin = hin; L.win = win; L.hout = hout; L.wout = wout;
    d->net.layer[d->net.nlayers++] = L;
    d->act_floats = std::max(d->act_floats, (size_t)hout * wout * cout);
  };
  const size_t kSmemLimit = 227 * 1024;                            // sm_90's opt-in shared memory per block
  const int64_t kGridX = 2147483647;
  R2Conv0& L0 = d->r2conv0;
  L0 = {c.height, c.width, pool ? c.height / 4 : c.height, pool ? c.width / 4 : c.width, ch[0], pool ? 4 : 1, 0, convs[0].w, convs[0].bn};
  L0.RH = std::min(L0.hout, pool ? 2 : 8);                         // 8 conv rows per CTA
  if (r2_conv0_smem_floats(L0) * 4 > kSmemLimit)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res2d_conv0 needs %zu bytes of shared memory at width %d, the limit is %zu",
                   r2_conv0_smem_floats(L0) * 4, c.width, kSmemLimit);
  if ((int64_t)c.max_batch * ((L0.hout + L0.RH - 1) / L0.RH) > kGridX)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res2d_conv0: max_batch %d x %d row tiles exceeds the grid's %lld CTAs", c.max_batch,
                   (L0.hout + L0.RH - 1) / L0.RH, (long long)kGridX);
  layer(c.height, c.width, L0.hout, L0.wout, 1, ch[0]);
  d->flops += 2ll * c.height * c.width * 9 * ch[0];
  int h = L0.hout, w = L0.wout, cin = ch[0];
  size_t ci = 1;
  for (int i = 0; i < 3; ++i) {
    R2Block& B = d->r2block[i];
    memset(&B, 0, sizeof(B));
    B.cin = cin; B.cout = ch[i + 1]; B.down = B.cout != cin; B.s = B.down ? 2 : 1; B.hin = h; B.win = w;
    ds_same(h, 3, B.s, &B.hout, &B.pt);
    ds_same(w, 3, B.s, &B.wout, &B.pl);
    if (B.down) { B.wd = convs[ci].w; B.bnd = convs[ci].bn; ++ci; }
    B.w0 = convs[ci].w; B.bn0 = convs[ci].bn; ++ci;
    B.w1 = convs[ci].w; B.bn1 = convs[ci].bn; ++ci;
    // tile plan: up to 8 x 16 output positions and every output channel at once.  Past 100 KB of shared memory (two CTAs per
    // SM) the filter slice COT halves, to a multiple of 4, until it is at most 32 channels: a sliced layer takes slices of 20 to
    // 32 channels and a shorter last one.  Past 200 KB the tile shrinks.  Then balanced, so that the last tile of a row or
    // column is not a sliver.  The plan depends on the geometry alone, so an utterance's bits do not depend on n.
    B.RH = std::min(B.hout, 8); B.WT = std::min(B.wout, 16); B.COT = r2_pad4(B.cout);
    auto bytes = [&] { return r2_block_smem(B).floats * 4; };
    while (bytes() > 100 * 1024 && B.COT > 32) B.COT = r2_pad4(B.COT / 2);
    while (bytes() > 200 * 1024 && (B.RH > 1 || B.WT > 1)) {
      if (B.WT > B.RH) B.WT = std::max(1, B.WT / 2);
      else B.RH = std::max(1, B.RH / 2);
    }
    B.RH = (B.hout + (B.hout + B.RH - 1) / B.RH - 1) / ((B.hout + B.RH - 1) / B.RH);
    B.WT = (B.wout + (B.wout + B.WT - 1) / B.WT - 1) / ((B.wout + B.WT - 1) / B.WT);
    if (bytes() > kSmemLimit)
      return ds_fail(TCR_ERR_UNSUPPORTED, "res2d_block %d needs %zu bytes of shared memory, the limit is %zu", i, bytes(), kSmemLimit);
    const int64_t tiles = (int64_t)((B.hout + B.RH - 1) / B.RH) * ((B.wout + B.WT - 1) / B.WT);
    if ((int64_t)c.max_batch * tiles > kGridX)
      return ds_fail(TCR_ERR_UNSUPPORTED, "res2d_block %d: max_batch %d x %lld tiles exceeds the grid's %lld CTAs", i, c.max_batch,
                     (long long)tiles, (long long)kGridX);
    layer(h, w, B.hout, B.wout, cin, B.cout);
    d->flops += 2ll * B.hout * B.wout * (9ll * cin * B.cout + 9ll * B.cout * B.cout + (B.down ? (int64_t)cin * B.cout : 0));
    h = B.hout; w = B.wout; cin = B.cout;
  }
  d->flops += 2ll * ch[3] * c.num_classes;
  return TCR_OK;
}

// Honk's ResNets as audio_nets/res.py builds them: f_conv (+ Res8's 4x3 / stride-1 pool), conv0 .. conv{L-1}, fc, all under the
// scope "Res" with slim's default "Conv" sub-scope inside conv{k}; the weights in creation order, then each conv{k}_bn's moving
// statistics.  Also each kernel's tile plan, and the refusals of what the kernels cannot run.
template <class Add>
static int res_define(tcr_dscnn* d, Add& add) {
  const tcr_dscnn_config& c = d->cfg;
  const bool r8 = c.size == TCR_RES8 || c.size == TCR_RES8_NARROW, narrow = c.size == TCR_RES8_NARROW || c.size == TCR_RES15_NARROW;
  const int C = narrow ? 19 : 45, nl = r8 ? 6 : 13;
  const size_t kSmemLimit = 227 * 1024;                            // sm_90's opt-in shared memory per block
  const int64_t kGridX = 2147483647;
  ResFconv& F0 = d->rfconv;
  F0 = {c.height, c.width, r8 ? c.height - 3 : c.height, r8 ? c.width - 2 : c.width, C, r8 ? 4 : 1, r8 ? 3 : 1, 0, 0};
  F0.w = add("Res/f_conv/weights", TCR_KIND_WEIGHT, {3, 3, 1, C});
  int64_t wk[13];
  for (int k = 0; k < nl; ++k) wk[k] = add("Res/conv" + std::to_string(k) + "/Conv/weights", TCR_KIND_WEIGHT, {3, 3, C, C});
  d->rfc = add("Res/fc/weights", TCR_KIND_WEIGHT, {1, 1, C, c.num_classes});
  ResBn bn[13];
  for (int k = 0; k < nl; ++k) {
    bn[k].mm = add("Res/conv" + std::to_string(k) + "_bn/moving_mean", TCR_KIND_MOVING_MEAN, {C});
    bn[k].mv = add("Res/conv" + std::to_string(k) + "_bn/moving_variance", TCR_KIND_MOVING_VAR, {C});
  }
  auto layer = [&](int hin, int win, int hout, int wout, int cin) {
    DsLayerDev L;
    memset(&L, 0, sizeof(L));
    L.type = kLayerRes; L.cin = cin; L.cout = C; L.hin = hin; L.win = win; L.hout = hout; L.wout = wout;
    d->net.layer[d->net.nlayers++] = L;
    d->act_floats = std::max(d->act_floats, (size_t)hout * wout * C);
  };
  // f_conv: up to 8 output rows per CTA, fewer where the staged conv rows pass 100 KB (wide log-mel maps)
  F0.RH = std::min(F0.hout, 8);
  while (F0.RH > 1 && res_fconv_smem_floats(F0) * 4 > 100 * 1024) --F0.RH;
  if (res_fconv_smem_floats(F0) * 4 > kSmemLimit)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res_fconv needs %zu bytes of shared memory at width %d, the limit is %zu",
                   res_fconv_smem_floats(F0) * 4, c.width, kSmemLimit);
  if ((int64_t)c.max_batch * ((F0.hout + F0.RH - 1) / F0.RH) > kGridX)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res_fconv: max_batch %d x %d row tiles exceeds the grid's %lld CTAs", c.max_batch,
                   (F0.hout + F0.RH - 1) / F0.RH, (long long)kGridX);
  layer(c.height, c.width, F0.hout, F0.wout, 1);
  d->flops += 2ll * c.height * c.width * 9 * C;
  // conv{k}: tiles of TR whole rows, as many as the CTA's register tiles cover, then balanced so the last tile is not a sliver.  The
  // plan depends on the geometry alone, so an utterance's bits do not depend on n.
  const int H = F0.hout, W = F0.wout, npmax = narrow ? res_np_max<20>() : res_np_max<48>();
  if (W > npmax)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res_conv tiles whole rows of at most %d positions; the blocks' map is %d wide", npmax, W);
  int TR = std::min(H, npmax / W);
  const int tpu = (H + TR - 1) / TR;
  TR = (H + tpu - 1) / tpu;
  const size_t smem = (narrow ? res_conv_smem_floats<20>(TR, W) : res_conv_smem_floats<48>(TR, W)) * 4;
  if (smem > kSmemLimit)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res_conv needs %zu bytes of shared memory, the limit is %zu", smem, kSmemLimit);
  if ((int64_t)c.max_batch * tpu > kGridX)
    return ds_fail(TCR_ERR_UNSUPPORTED, "res_conv: max_batch %d x %d row tiles exceeds the %lld tiles a launch walks", c.max_batch,
                   tpu, (long long)kGridX);
  for (int k = 0; k < nl; ++k) {
    d->rconv[k] = {H, W, C, r8 ? 1 : 1 << (k / 3), TR, wk[k], bn[k]};   // Res15 dilates: rate 2^(k // 3), res.py:10
    layer(H, W, H, W, C);
    d->flops += 2ll * H * W * 9 * C * C;
  }
  d->flops += 2ll * C * c.num_classes;
  return TCR_OK;
}

// low_latency_conv / tiny_conv as audio_nets/kws.py builds them (create_low_latency_conv_model 293-405, create_tiny_conv_model
// 681-757): top-level TF variables in creation order, each weight followed by its bias.  FLOPs count tiny_conv's full 80-tap kernel
// at every output, padding included.  Also each kernel's plan, and the refusals of what the kernels cannot run.
template <class Add>
static int kwsb_define(tcr_dscnn* d, Add& add) {
  const tcr_dscnn_config& c = d->cfg;
  const bool ll = c.size == TCR_KWS_LOW_LATENCY_CONV;
  const size_t kSmemLimit = 227 * 1024;                            // sm_90's opt-in shared memory per block
  const int64_t kIntMax = 2147483647;
  DsLayerDev L;
  memset(&L, 0, sizeof(L));
  L.type = kLayerKwsB; L.cin = 1; L.hin = c.height; L.win = c.width;
  KwsFcb& H = d->fcb;
  H = {};
  H.classes = c.num_classes;
  H.out = H.outb = -1;
  int64_t K;
  if (ll) {
    if (c.width < 8) return ds_fail(TCR_ERR_UNSUPPORTED, "low_latency_conv needs width >= 8 (its T x 8 conv is VALID), got %d", c.width);
    L.cout = kLlCout; L.kh = c.height; L.kw = 8; L.sh = L.sw = 1; L.hout = 1; L.wout = c.width - 7;
    if ((int64_t)c.max_batch * L.wout > kIntMax)
      return ds_fail(TCR_ERR_UNSUPPORTED, "kws_llconv: max_batch %d x %d output columns exceeds the %lld GEMM rows it indexes",
                     c.max_batch, L.wout, (long long)kIntMax);
    K = (int64_t)L.wout * kLlCout;
  } else {
    L.cout = 8; L.kh = 10; L.kw = 8; L.sh = L.sw = 2;
    ds_same(c.height, 10, 2, &L.hout, &L.pt);
    ds_same(c.width, 8, 2, &L.wout, &L.pl);
    KwsTinyConv& T = d->tiny;
    T = {c.height, c.width, L.hout, L.wout, L.pt, L.pl, std::min(L.hout, 8), 2 * L.wout + 6, 0, 0};
    if (kws_tiny_smem_floats(T) * 4 > kSmemLimit)
      return ds_fail(TCR_ERR_UNSUPPORTED, "kws_tinyconv needs %zu bytes of shared memory at width %d, the limit is %zu",
                     kws_tiny_smem_floats(T) * 4, c.width, kSmemLimit);
    if ((int64_t)c.max_batch * ((T.hout + T.RH - 1) / T.RH) > kIntMax)
      return ds_fail(TCR_ERR_UNSUPPORTED, "kws_tinyconv: max_batch %d x %d row tiles exceeds the grid's %lld CTAs", c.max_batch,
                     (T.hout + T.RH - 1) / T.RH, (long long)kIntMax);
    K = (int64_t)L.hout * L.wout * 8;
  }
  const int KC = ll ? 128 : 256;                                   // kws_fcs_kernel's K chunk
  if (K > kIntMax || (K + KC - 1) / KC * ((c.max_batch + 63) / 64) > kIntMax)
    return ds_fail(TCR_ERR_UNSUPPORTED, "kws_fcs: K = %lld flattened values in chunks of %d for max_batch %d exceeds the grid's %lld CTAs",
                   (long long)K, KC, c.max_batch, (long long)kIntMax);
  H.K = (int)K;
  H.nsplit = (H.K + KC - 1) / KC;
  L.w = add("first_weights", TCR_KIND_WEIGHT, {L.kh, 8, 1, L.cout});
  L.b = add("first_bias", TCR_KIND_BETA, {L.cout});
  d->flops += 2ll * L.hout * L.wout * L.kh * 8 * L.cout;
  if (ll) {
    d->llconv = {c.height, c.width, L.wout, 0, L.w, L.b};
    H.N0 = 128;
    H.nmid = 1;
    H.w0 = add("first_fc_weights", TCR_KIND_WEIGHT, {H.K, 128});
    H.b0 = add("first_fc_bias", TCR_KIND_BETA, {128});
    H.mid = add("second_fc_weights", TCR_KIND_WEIGHT, {128, 128});
    H.midb = add("second_fc_bias", TCR_KIND_BETA, {128});
    H.out = add("final_fc_weights", TCR_KIND_WEIGHT, {128, c.num_classes});
    H.outb = add("final_fc_bias", TCR_KIND_BETA, {c.num_classes});
    d->flops += 2ll * H.K * 128 + 2ll * 128 * 128 + 2ll * 128 * c.num_classes;
  } else {
    d->tiny.w = L.w;
    d->tiny.b = L.b;
    H.N0 = c.num_classes;
    H.w0 = add("final_fc_weights", TCR_KIND_WEIGHT, {H.K, c.num_classes});
    H.b0 = add("final_fc_bias", TCR_KIND_BETA, {c.num_classes});
    d->flops += 2ll * H.K * c.num_classes;
  }
  d->net.layer[d->net.nlayers++] = L;
  d->act_floats = (size_t)L.hout * L.wout * L.cout;
  return TCR_OK;
}

// Tile rows of the wgmma kernels: at most 128 accumulator rows (RH * wout) per tile, balanced (25 rows -> 5 tiles of 5).
static int ds_tile_rows(const DsLayerDev& L) {
  const int cap = std::max(1, std::min(L.hout, 128 / std::max(1, std::min(L.wout, 128))));
  const int tiles = (L.hout + cap - 1) / cap;
  return (L.hout + tiles - 1) / tiles;
}

// The plan of layer l of DS-CNN S / M / L (d->plan[l]), and the refusal of a layer no kernel can run.  wgmma where the layer's shape
// fits the tensor-core kernels (use_tc, TCR_DSCNN_TC; never in the emulator build, which has no wgmma), the register-tiled FMA
// kernels otherwise.  dscnn_conv stages a whole utterance, so its bytes grow with height x width, up to sm_90's 227 KB opt-in;
// dscnn_dsblock shrinks its output-channel slice, then its tile of rows, and stops at 200 KB.  The plan depends on the geometry
// alone, so an utterance's bits do not depend on n.
static int ds_plan_layer(tcr_dscnn* d, int l, const char* scope) {
  const DsLayerDev& L = d->net.layer[l];
  DsPlan& P = d->plan[l];
  if (L.type == 0) {
#ifndef TCR_EMU
    const int RHt = ds_tile_rows(L);
    // implicit GEMM on wgmma (3xTF32), where the kernel's per-thread im2col walk covers the tile
    if (d->use_tc && L.cin == 1 && L.cout == 64 && (L.kh * L.kw) % 8 == 0 && L.wout <= 64 && im2col_walk_fits(L, RHt, kTcThreads)) {
      const size_t smem_ws = conv_tc_smem<64>(L, RHt, 2).floats * 4;
      if (d->tc_ws && smem_ws <= 220 * 1024 && im2col_walk_fits(L, RHt, kWsProducers) && (L.kh * L.kw / 4) % 2 == 0)
        P = {kDsConvWs, RHt, 0, smem_ws};
      else
        P = {kDsConvTc, RHt, 0, conv_tc_smem<64>(L, RHt, 1).floats * 4};
      return TCR_OK;
    }
#endif
    const size_t kSmemLimit = 227 * 1024;                          // sm_90's opt-in shared memory per block
    P = {kDsConv, 0, 0, conv_smem(L).floats * 4};
    if (P.smem > kSmemLimit)
      return ds_fail(TCR_ERR_UNSUPPORTED, "dscnn_conv (%s) needs %zu bytes of shared memory at %d x %d, the limit is %zu", scope, P.smem,
                     d->cfg.height, d->cfg.width, kSmemLimit);
    return TCR_OK;
  }
  // pointwise conv on the tensor cores (wgmma, 3xTF32): the 64 -> 64 channel blocks with a 3x3 / stride-1 depthwise stage.  The
  // warp-specialised kernel where its input tile and producers fit, the lock-step kernel where its fetch walk does.
#ifndef TCR_EMU
  if (d->use_tc && L.cin == 64 && L.cout == 64 && L.kh == 3 && L.kw == 3 && L.sh == 1 && L.sw == 1 && L.wout <= 64) {
    const int RHt = ds_tile_rows(L);
    const size_t smem_ws = dsblock_ws_smem<64, 64>(L, RHt).floats * 4;
    if (d->tc_ws && smem_ws <= 226 * 1024 && L.cin / 4 * L.wout <= kWsProducers && L.wout + 2 <= 256 && RHt + 2 <= 256) {
      P = {kDsBlockWs, RHt, 0, smem_ws};
      return TCR_OK;
    }
    const size_t smem_tc = dsblock_tc_smem<64, 64>(L, RHt).floats * 4;
    if (smem_tc <= 200 * 1024 && (RHt + 2) * (L.wout + 2) <= kDwCells * (kTcThreads / (L.cin / 4))) {
      P = {kDsBlockTc, RHt, 0, smem_tc};
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
  const size_t kBlockLimit = 200 * 1024;
  P = {kDsBlock, RH, COT, dsblock_smem(L, RH, COT).floats * 4};
  if (P.smem > kBlockLimit)
    return ds_fail(TCR_ERR_UNSUPPORTED, "dscnn_dsblock (%s) needs %zu bytes of shared memory at %d x %d, the limit is %zu", scope, P.smem,
                   d->cfg.height, d->cfg.width, kBlockLimit);
  return TCR_OK;
}

extern "C" int tcr_dscnn_create(const tcr_dscnn_config* cfg, tcr_dscnn** out) {
  if (!cfg || !out) { set_error("NULL argument"); return TCR_ERR_INVALID; }
  *out = nullptr;
  const bool kws = cfg->size == TCR_KWS_TRAD_FPOOL3 || cfg->size == TCR_KWS_ONE_FSTRIDE4;
  const bool res2d = cfg->size == TCR_RES2D8 || cfg->size == TCR_RES2D8_POOL;
  const bool res = cfg->size == TCR_RES8 || cfg->size == TCR_RES8_NARROW || cfg->size == TCR_RES15 || cfg->size == TCR_RES15_NARROW;
  const bool kwsb = cfg->size == TCR_KWS_LOW_LATENCY_CONV || cfg->size == TCR_KWS_TINY_CONV;
  if (cfg->size != 'S' && cfg->size != 'M' && cfg->size != 'L' && !kws && !res2d && !res && !kwsb) {
    set_error("DS-CNN size must be 'S', 'M' or 'L', or a KWS baseline: 'P' (trad_fpool3) or 'F' (one_fstride4), or 'C' "
              "(low_latency_conv) or 'Y' (tiny_conv), or a 2-D ablation: 'R' (ResNet2D8) or 'A' (ResNet2D8Pool), or a Honk ResNet: "
              "'E' (Res8), 'N' (Res8Narrow), 'D' (Res15) or 'T' (Res15Narrow)");
    return TCR_ERR_INVALID;
  }
  if (!res2d && cfg->width_multiplier != 0.0)
    return ds_fail(TCR_ERR_INVALID, "width_multiplier (%g) applies to ResNet2D8 / ResNet2D8Pool only; it must be 0 for size '%c'",
                   cfg->width_multiplier, (char)cfg->size);
  if (res2d && !(cfg->width_multiplier >= 0.0 && cfg->width_multiplier < 1e6))
    return ds_fail(TCR_ERR_INVALID, "bad width_multiplier %g", cfg->width_multiplier);
  if (cfg->max_batch <= 0 || cfg->height <= 0 || cfg->width <= 0 || cfg->num_classes <= 0 || cfg->num_classes > kMaxClasses) {
    set_error("bad DS-CNN configuration");
    return TCR_ERR_INVALID;
  }
  if (cfg->size == TCR_KWS_TRAD_FPOOL3 && (cfg->height < 29 || cfg->width < 19)) {
    return ds_fail(TCR_ERR_UNSUPPORTED, "trad_fpool3 needs height >= 29 and width >= 19 (its 20x8 conv, 1x3 pool and 10x4 conv are "
                   "VALID), got %d x %d", cfg->height, cfg->width);
  }
  if (cfg->size == TCR_KWS_ONE_FSTRIDE4 && (int64_t)cfg->height * cfg->width > kKwsMaxStaged) {
    return ds_fail(TCR_ERR_UNSUPPORTED, "one_fstride4 needs height x width <= %d (its conv stages a whole utterance in shared "
                   "memory), got %d x %d", kKwsMaxStaged, cfg->height, cfg->width);
  }
  if (cfg->size == TCR_RES2D8_POOL && (cfg->height < 4 || cfg->width < 4)) {
    return ds_fail(TCR_ERR_UNSUPPORTED, "ResNet2D8Pool needs height >= 4 and width >= 4 (res2d_conv0's 4x4 / stride 4 average pool is "
                   "VALID), got %d x %d", cfg->height, cfg->width);
  }
  if (cfg->size == TCR_KWS_ONE_FSTRIDE4 && cfg->width < 8) {
    return ds_fail(TCR_ERR_UNSUPPORTED, "one_fstride4 needs width >= 8 (its T x 8 conv is VALID), got %d", cfg->width);
  }
  if ((cfg->size == TCR_RES8 || cfg->size == TCR_RES8_NARROW) && (cfg->height < 4 || cfg->width < 3)) {
    return ds_fail(TCR_ERR_UNSUPPORTED, "Res8 / Res8Narrow need height >= 4 and width >= 3 (res_fconv's 4x3 / stride 1 average pool "
                   "is VALID), got %d x %d", cfg->height, cfg->width);
  }
  tcr_dscnn* d = new tcr_dscnn();
  d->cfg = *cfg;
  d->kws = kws;
  d->res2d = res2d;
  d->res = res;
  d->kwsb = kwsb;
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
  if (kws) {
    // audio_nets/kws.py create_trad_fpool3_model (204-290) / create_one_fstride4_model (408-487): top-level TF variables
    auto conv = [&](const char* name, int cout, int kh, int kw, int sw, int pool) {
      DsLayerDev L;
      memset(&L, 0, sizeof(L));
      L.type = kLayerKws; L.cin = cin; L.cout = cout; L.kh = kh; L.kw = kw; L.sh = 1; L.sw = sw; L.hin = h; L.win = w;
      L.hout = h - kh + 1;
      const int wconv = (w - kw) / sw + 1;
      L.wout = wconv / pool;
      L.w = add(name, TCR_KIND_WEIGHT, {kh, kw, cin, cout});
      d->flops += 2ll * L.hout * wconv * kh * kw * cin * cout;
      d->pool[d->net.nlayers] = pool;
      d->net.layer[d->net.nlayers++] = L;
      d->act_floats = std::max(d->act_floats, (size_t)L.hout * L.wout * cout);
      h = L.hout; w = L.wout; cin = cout;
    };
    const bool trad = cfg->size == TCR_KWS_TRAD_FPOOL3;
    if (trad) {
      conv("first_weights", 64, 20, 8, 1, 3);
      conv("second_weights", 64, 10, 4, 1, 1);
    } else {
      conv("first_weights", 186, cfg->height, 8, 4, 1);
    }
    KwsHead& H = d->head;
    H.K = h * w * cin;
    H.nsplit = (H.K + kKwsLinK - 1) / kKwsLinK;
    H.classes = cfg->num_classes;
    H.lin = add(trad ? "linear_weights" : "first_linear_weights", TCR_KIND_WEIGHT, {H.K, 32});
    H.fc[0] = add("first_fc_weights", TCR_KIND_WEIGHT, {32, 128});
    H.nfc = 1;
    if (!trad) H.fc[H.nfc++] = add("second_fc_weights", TCR_KIND_WEIGHT, {128, 128});
    H.out = add("final_fc_weights", TCR_KIND_WEIGHT, {128, cfg->num_classes});
    d->flops += 2ll * H.K * 32 + 2ll * 32 * 128 + (trad ? 0 : 2ll * 128 * 128) + 2ll * 128 * cfg->num_classes;
    defs.clear();
  }
  if (res2d) {
    const int rc = res2d_define(d, add);
    if (rc != TCR_OK) { delete d; return rc; }
    h = d->net.layer[3].hout; w = d->net.layer[3].wout; cin = d->net.layer[3].cout;
    defs.clear();
  }
  if (res) {
    const int rc = res_define(d, add);
    if (rc != TCR_OK) { delete d; return rc; }
    defs.clear();
  }
  if (kwsb) {
    const int rc = kwsb_define(d, add);
    if (rc != TCR_OK) { delete d; return rc; }
    defs.clear();
  }
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
    const int rc = ds_plan_layer(d, d->net.nlayers - 1, df.scope);
    if (rc != TCR_OK) { delete d; return rc; }
    d->act_floats = std::max(d->act_floats, (size_t)L.hout * L.wout * df.depth);
    h = L.hout; w = L.wout; cin = df.depth;
  }
  d->net.classes = cfg->num_classes;
  if (!kws && !res2d && !res && !kwsb) {
    d->net.fcw = add("DSCNN/fc1/weights", TCR_KIND_WEIGHT, {cin, cfg->num_classes});
    d->net.fcb = add("DSCNN/fc1/biases", TCR_KIND_BETA, {cfg->num_classes});
    d->flops += 2ll * cin * cfg->num_classes;
  }
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
  if (kws) {
    const DsLayerDev& L1 = d->net.layer[d->net.nlayers - 1];
    const bool split = L1.cin == 64 && L1.cout == 64;
    if (cudaMalloc((void**)&d->part, (size_t)d->head.nsplit * cfg->max_batch * 32 * sizeof(float)) != cudaSuccess ||
        (split && cudaMalloc((void**)&d->bimg, (size_t)2 * L1.kh * L1.kw * 64 * 64 * sizeof(float)) != cudaSuccess)) {
      tcr_dscnn_destroy(d);
      set_error("cudaMalloc failed for the KWS head / filter buffers");
      return TCR_ERR_CUDA;
    }
  }
  if (kwsb && cudaMalloc((void**)&d->part, (size_t)d->fcb.nsplit * cfg->max_batch * ((d->fcb.N0 + 31) & ~31) * sizeof(float)) !=
                  cudaSuccess) {
    tcr_dscnn_destroy(d);
    set_error("cudaMalloc failed for the KWS head's partial sums");
    return TCR_ERR_CUDA;
  }
  *out = d;
  return TCR_OK;
}

extern "C" int tcr_dscnn_destroy(tcr_dscnn* d) {
  if (!d) return TCR_OK;
  for (int i = 0; i < 2; ++i)
    if (d->act[i]) cudaFree(d->act[i]);
  frontend_free(&d->fe);
  if (d->feat) cudaFree(d->feat);
  if (d->part) cudaFree(d->part);
  if (d->bimg) cudaFree(d->bimg);
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

// The first layer (cin == 1) on the kernel of its plan (ds_plan_layer).  WIN: utterance u is the window `win` describes
// (tcr_listener.cu); the kernel choice is the same.
template <bool WIN>
static int ds_launch_conv(tcr_dscnn* d, int l, const float* params, const float* in, float* out, int32_t n, cudaStream_t s,
                          WindowView win) {
  const DsLayerDev& L = d->net.layer[l];
  const DsPlan& P = d->plan[l];
  const float eps = 1e-3f;
#ifndef TCR_EMU
  const int grid = P.RH ? std::min(ds_tiles_per_utt(L, P.RH) * n, d->sms) : 0;   // wgmma only: dscnn_conv has P.RH = 0
  if (P.kernel == kDsConvWs) {
    auto kws = dscnn_conv_ws_kernel<64, WIN>;
    static SmemOptIn optin_ws;
    if (optin_ws.ensure(kws, P.smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_conv_ws: shared memory opt-in failed");
    TCR_LAUNCH(WIN ? "dscnn_conv_ws:win" : "dscnn_conv_ws", kws, dim3(grid), dim3(kTcThreads), P.smem, s, L, P.RH, n, params, in, out, eps,
               win);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_conv_ws launch failed");
    return TCR_OK;
  }
  if (P.kernel == kDsConvTc) {
    auto ktc = dscnn_conv_tc_kernel<64, WIN>;
    static SmemOptIn optin_tc;
    if (optin_tc.ensure(ktc, P.smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_conv_tc: shared memory opt-in failed");
    TCR_LAUNCH(WIN ? "dscnn_conv_tc:win" : "dscnn_conv_tc", ktc, dim3(grid), dim3(kTcThreads), P.smem, s, L, P.RH, n, params, in, out, eps,
               win);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_conv_tc launch failed");
    return TCR_OK;
  }
#endif
  auto kfn = dscnn_conv_kernel<WIN>;
#ifndef TCR_EMU
  static SmemOptIn optin;
  if (optin.ensure(kfn, P.smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_conv: shared memory opt-in failed");
#endif
  TCR_LAUNCH(WIN ? "dscnn_conv:win" : "dscnn_conv", kfn, dim3(n), dim3(256), P.smem, s, L, params, in, out, eps, win);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_conv launch failed");
  return TCR_OK;
}

// A layer of the KWS baselines.  trad_fpool3's two convs run on wgmma at every geometry the handle accepts: conv1 + pool on
// kws_conv1_tc_kernel, conv2 on kws_bsplit_kernel then kws_conv2_tc_kernel.  one_fstride4's conv runs on the FMA kernel, and so does
// every layer in the emulator build, which has no wgmma.
template <bool WIN>
static int kws_launch_conv(tcr_dscnn* d, int l, const float* params, const float* in, float* out, int32_t n, cudaStream_t s,
                           WindowView win) {
  const DsLayerDev& D = d->net.layer[l];
  KwsConv L = {D.cin, D.cout, D.kh, D.kw, D.sh, D.sw, D.hin, D.win, D.hout, D.wout, std::min(D.hout, 8), D.w};
#ifndef TCR_EMU
  if (D.cin == 1 && D.cout == 64 && d->pool[l] == 3 && D.sh == 1 && D.sw == 1 && D.kw % 4 == 0 && D.kh * D.kw == 8 * kC1Half) {
    const int64_t pooled = (int64_t)n * D.hout * D.wout;
    const int grid = (int)std::min<int64_t>((pooled + kC1Pooled - 1) / kC1Pooled, d->sms);
    const size_t smem = conv1_tc_smem_floats(D.kh * D.kw / 4) * 4;
    auto kfn = kws_conv1_tc_kernel<WIN>;
    static SmemOptIn optin_c1;
    if (optin_c1.ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_conv1_tc: shared memory opt-in failed");
    TCR_LAUNCH(WIN ? "kws_conv1_tc:win" : "kws_conv1_tc", kfn, dim3(grid), dim3(kTcThreads), smem, s, L, (int)n, params, in, out, win);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_conv1_tc launch failed");
    return TCR_OK;
  }
  if (D.cin == 64 && D.cout == 64 && (D.kh * D.kw * D.cin) % (kC2Chunk * kC2Flush) == 0 && d->bimg) {
    const int K = D.kh * D.kw * D.cin;
    TCR_LAUNCH("kws_bsplit", kws_bsplit_kernel, dim3((K * 64 + 255) / 256), dim3(256), 0, s, K, params + D.w, d->bimg);
    const int64_t rows = (int64_t)n * D.hout * D.wout;
    const int grid = (int)std::min<int64_t>((rows + 127) / 128, d->sms);
    const size_t smem = (size_t)kC2Stages * kC2StageFloats * 4;
    static SmemOptIn optin_tc;
    if (optin_tc.ensure(kws_conv2_tc_kernel, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_conv2_tc: shared memory opt-in failed");
    TCR_LAUNCH("kws_conv2_tc", kws_conv2_tc_kernel, dim3(grid), dim3(kC2Threads), smem, s, L, (int)n, d->bimg, in, out);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_conv2_tc launch failed");
    return TCR_OK;
  }
#endif
  const size_t smem = (size_t)kws_stage_floats(L) * 4;
  if (smem > kKwsMaxStaged * sizeof(float))
    return ds_fail(TCR_ERR_UNSUPPORTED, "KWS layer %d: %zu bytes of input rows do not fit in shared memory", l, smem);
  const int tiles = (int)((int64_t)n * ((D.hout + L.RH - 1) / L.RH));
  // a pooled layer (trad_fpool3's first, in the emulator build): 4 channels x 2 rows x 2 pooled columns (x 3) per thread; any
  // other (one_fstride4's single output row of 186 channels; conv2 in the emulator build): one channel x 5 columns
  const bool pooled = d->pool[l] == 3;
  if (!pooled && d->pool[l] != 1) return ds_fail(TCR_ERR_UNSUPPORTED, "KWS layer %d: pooling by %d", l, d->pool[l]);
  if (pooled && D.cout % 4) return ds_fail(TCR_ERR_UNSUPPORTED, "KWS layer %d: a pooled layer needs a multiple of 4 channels", l);
  auto kfn = pooled ? kws_conv_kernel<3, 4, 2, 2, WIN> : kws_conv_kernel<1, 1, 1, 5, WIN>;
#ifndef TCR_EMU
  static SmemOptIn optin3, optin1;
  if ((pooled ? optin3 : optin1).ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_conv: shared memory opt-in failed");
#endif
  TCR_LAUNCH(WIN ? "kws_conv:win" : "kws_conv", kfn, dim3(tiles), dim3(256), smem, s, L, params, in, out, win);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_conv launch failed");
  return TCR_OK;
}

// flatten -> lin (split over K) -> the 128-wide matrices -> logits, softmax
static int kws_head(tcr_dscnn* d, const float* params, const float* in, int n, float* logits, float* probs, cudaStream_t s) {
  const KwsHead& H = d->head;
#ifndef TCR_EMU
  static SmemOptIn optin;
  if (optin.ensure(kws_lin_kernel, kKwsLinSmem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_lin: shared memory opt-in failed");
#endif
  TCR_LAUNCH("kws_lin", kws_lin_kernel, dim3(H.nsplit * ((n + kKwsLinU - 1) / kKwsLinU)), dim3(256), kKwsLinSmem, s, H, n, params, in,
             d->part);
  TCR_LAUNCH("kws_head", kws_head_kernel, dim3((n + kKwsHeadU - 1) / kKwsHeadU), dim3(128), 0, s, H, n, params, d->part, logits, probs);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "KWS head launch failed");
  return TCR_OK;
}

// The conv of low_latency_conv (kws_llconv_kernel) or tiny_conv (kws_tinyconv_kernel); the emulator build runs the same kernels.
template <bool WIN>
static int kwsb_launch_conv(tcr_dscnn* d, const float* params, const float* in, float* out, int32_t n, cudaStream_t s, WindowView win) {
  if (d->cfg.size == TCR_KWS_LOW_LATENCY_CONV) {
    KwsLlConv L = d->llconv;
    L.M = n * L.wout;
    auto kfn = kws_llconv_kernel<WIN>;
    TCR_LAUNCH(WIN ? "kws_llconv:win" : "kws_llconv", kfn, dim3((L.M + kLlBM - 1) / kLlBM), dim3(kLlThreads), kLlSmem, s, L, params,
               in, out, win);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_llconv launch failed");
    return TCR_OK;
  }
  const KwsTinyConv& L = d->tiny;
  const size_t smem = kws_tiny_smem_floats(L) * 4;
  auto kfn = kws_tinyconv_kernel<WIN>;
#ifndef TCR_EMU
  static SmemOptIn optin;
  if (optin.ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_tinyconv: shared memory opt-in failed");
#endif
  const unsigned grid = (unsigned)((int64_t)n * ((L.hout + L.RH - 1) / L.RH));
  TCR_LAUNCH(WIN ? "kws_tinyconv:win" : "kws_tinyconv", kfn, dim3(grid), dim3(256), smem, s, L, params, in, out, win);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_tinyconv launch failed");
  return TCR_OK;
}

// flatten -> the first matmul split over K (kws_fcs: 128 columns for low_latency_conv, the classes for tiny_conv) -> the chunks
// summed in order, the biases, the remaining matrices, logits, softmax (kws_fcb_head)
static int kwsb_head(tcr_dscnn* d, const float* params, const float* in, int n, float* logits, float* probs, cudaStream_t s) {
  const KwsFcb& H = d->fcb;
  const bool ll = d->cfg.size == TCR_KWS_LOW_LATENCY_CONV;
  auto kfn = ll ? kws_fcs_kernel<4, 128> : kws_fcs_kernel<1, 256>;
  const size_t smem = ll ? kws_fcs_smem<4, 128>() : kws_fcs_smem<1, 256>();
#ifndef TCR_EMU
  static SmemOptIn optin4, optin1;
  if ((ll ? optin4 : optin1).ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "kws_fcs: shared memory opt-in failed");
#endif
  TCR_LAUNCH("kws_fcs", kfn, dim3(H.nsplit * ((n + 63) / 64)), dim3(256), smem, s, H, n, params, in, d->part);
  TCR_LAUNCH("kws_fcb_head", kws_fcb_head_kernel, dim3((n + kKwsHeadU - 1) / kKwsHeadU), dim3(128), 0, s, H, n, params, d->part, logits,
             probs);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "KWS head launch failed");
  return TCR_OK;
}

// A layer of the 2-D ablations: 0 is conv0 (+ pool) on res2d_conv0_kernel, 1-3 the residual blocks on res2d_block_kernel.
template <bool WIN>
static int res2d_launch(tcr_dscnn* d, int l, const float* params, const float* in, float* out, int32_t n, cudaStream_t s, WindowView win) {
  const float eps = 1e-3f;
  if (l == 0) {
    const R2Conv0& L = d->r2conv0;
    const size_t smem = r2_conv0_smem_floats(L) * 4;
    auto kfn = res2d_conv0_kernel<WIN>;
#ifndef TCR_EMU
    static SmemOptIn optin;
    if (optin.ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res2d_conv0: shared memory opt-in failed");
#endif
    const unsigned grid = (unsigned)((int64_t)n * ((L.hout + L.RH - 1) / L.RH));
    TCR_LAUNCH(WIN ? "res2d_conv0:win" : "res2d_conv0", kfn, dim3(grid), dim3(256), smem, s, L, params, in, out, eps, win);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res2d_conv0 launch failed");
    return TCR_OK;
  }
  const R2Block& B = d->r2block[l - 1];
  const size_t smem = r2_block_smem(B).floats * 4;
#ifndef TCR_EMU
  static SmemOptIn optin;
  if (optin.ensure(res2d_block_kernel, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res2d_block: shared memory opt-in failed");
#endif
  const unsigned grid = (unsigned)((int64_t)n * ((B.hout + B.RH - 1) / B.RH) * ((B.wout + B.WT - 1) / B.WT));
  TCR_LAUNCH("res2d_block", res2d_block_kernel, dim3(grid), dim3(256), smem, s, B, params, in, out, eps);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res2d_block launch failed");
  return TCR_OK;
}

// conv{k} on res_conv_kernel: a persistent grid of as many CTAs as fit on the device, walking n x tpu row tiles.
template <int CP, bool RES>
static int res_launch_conv(tcr_dscnn* d, const ResConv& R, const float* params, const float* in, const float* res, float* out, int32_t n,
                           cudaStream_t s) {
  const size_t smem = res_conv_smem_floats<CP>(R.TR, R.w) * 4;
  const int tiles = n * ((R.h + R.TR - 1) / R.TR);
  auto kfn = res_conv_kernel<CP, RES>;
  int per_sm = 1;
#ifndef TCR_EMU
  static SmemOptIn optin;
  if (optin.ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res_conv: shared memory opt-in failed");
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kfn, kResConvThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
#endif
  const int grid = std::min(tiles, d->sms * per_sm);
  TCR_LAUNCH(RES ? "res_conv_res" : "res_conv", kfn, dim3(grid), dim3(kResConvThreads), smem, s, R, (int)n, params, in, res, out, 1e-3f);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res_conv launch failed");
  return TCR_OK;
}

// A layer of Res8 / Res15: 0 is f_conv (+ pool) on res_fconv_kernel, l = k + 1 is conv{k} on res_conv_kernel, with the residual for
// odd k (the second conv of a block).  The block input is layer l - 2's output, which both dscnn_forward and forward_partial leave
// in act[l & 1]: in a full forward that is also `out`.
template <bool WIN>
static int res_launch(tcr_dscnn* d, int l, const float* params, const float* in, float* out, int32_t n, cudaStream_t s, WindowView win) {
  if (l == 0) {
    const ResFconv& L = d->rfconv;
    const size_t smem = res_fconv_smem_floats(L) * 4;
    auto kfn = res_fconv_kernel<WIN>;
#ifndef TCR_EMU
    static SmemOptIn optin;
    if (optin.ensure(kfn, smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res_fconv: shared memory opt-in failed");
#endif
    const unsigned grid = (unsigned)((int64_t)n * ((L.hout + L.RH - 1) / L.RH));
    TCR_LAUNCH(WIN ? "res_fconv:win" : "res_fconv", kfn, dim3(grid), dim3(256), smem, s, L, params, in, out, win);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res_fconv launch failed");
    return TCR_OK;
  }
  const ResConv& R = d->rconv[l - 1];
  const bool residual = (l - 1) & 1, narrow = R.c == 19;
  const float* block_in = d->act[l & 1];
  if (narrow) return residual ? res_launch_conv<20, true>(d, R, params, in, block_in, out, n, s)
                              : res_launch_conv<20, false>(d, R, params, in, nullptr, out, n, s);
  return residual ? res_launch_conv<48, true>(d, R, params, in, block_in, out, n, s)
                  : res_launch_conv<48, false>(d, R, params, in, nullptr, out, n, s);
}

// Launches layer l: in [n, hin, win, cin] -> out [n, hout, wout, cout] (NHWC), or for l == 0 with `win` the windows it describes.
// DS-CNN S / M / L run the kernel of the layer's plan, chosen once in tcr_dscnn_create (ds_plan_layer) for every entry point.  The
// warp-specialised block kernel reads its input through a TMA map over max_batch utterances, so only from an activation buffer of
// the handle, which is where every entry point leaves a block's input.
static int ds_launch_layer(tcr_dscnn* d, int l, const float* params, const float* in, float* out, int32_t n, cudaStream_t s,
                           const WindowView* win = nullptr) {
  const DsLayerDev& L = d->net.layer[l];
  const float eps = 1e-3f;
  if (L.type == kLayerKws) {
    if (win) return kws_launch_conv<true>(d, l, params, in, out, n, s, *win);
    return kws_launch_conv<false>(d, l, params, in, out, n, s, WindowView{0, 0, 0});
  }
  if (L.type == kLayerRes2d) {
    if (win) return res2d_launch<true>(d, l, params, in, out, n, s, *win);
    return res2d_launch<false>(d, l, params, in, out, n, s, WindowView{0, 0, 0});
  }
  if (L.type == kLayerRes) {
    if (win) return res_launch<true>(d, l, params, in, out, n, s, *win);
    return res_launch<false>(d, l, params, in, out, n, s, WindowView{0, 0, 0});
  }
  if (L.type == kLayerKwsB) {
    if (win) return kwsb_launch_conv<true>(d, params, in, out, n, s, *win);
    return kwsb_launch_conv<false>(d, params, in, out, n, s, WindowView{0, 0, 0});
  }
  if (L.type == 0) {
    if (win) return ds_launch_conv<true>(d, l, params, in, out, n, s, *win);
    return ds_launch_conv<false>(d, l, params, in, out, n, s, WindowView{0, 0, 0});
  }
  const DsPlan& P = d->plan[l];
#ifndef TCR_EMU
  if (P.kernel == kDsBlockWs || P.kernel == kDsBlockTc) {
    const int grid = std::min(ds_tiles_per_utt(L, P.RH) * n, d->sms);
    if (P.kernel == kDsBlockWs) {
      if (in != d->act[0] && in != d->act[1])
        return ds_fail(TCR_ERR_INVALID, "dscnn_dsblock_ws reads its input through a TMA map over the handle's activation buffers");
      auto kws = dscnn_dsblock_ws_kernel<64, 64>;
      static SmemOptIn optin_ws;
      if (optin_ws.ensure(kws, P.smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_dsblock_ws: shared memory opt-in failed");
      if ((int)d->in_maps.size() < d->net.nlayers) d->in_maps.resize(d->net.nlayers);
      tcr_dscnn::InMap& im = d->in_maps[l];
      if (im.ptr != in || im.rh != P.RH) {                     // the activations ping-pong between two buffers: encoded once per layer
        const int rc = ds_encode_in_map(&im.map, in, L.cin, L.win, L.hin, d->cfg.max_batch, L.wout + 2, P.RH + 2);
        if (rc != TCR_OK) return rc;
        im.ptr = in;
        im.rh = P.RH;
      }
      TCR_LAUNCH("dscnn_dsblock_ws", kws, dim3(grid), dim3(kTcThreads), P.smem, s, im.map, L, P.RH, n, params, out, eps);
      if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_dsblock_ws launch failed");
      return TCR_OK;
    }
    auto ktc = dscnn_dsblock_tc_kernel<64, 64>;
    static SmemOptIn optin_tc;
    if (optin_tc.ensure(ktc, P.smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_dsblock_tc: shared memory opt-in failed");
    TCR_LAUNCH("dscnn_dsblock_tc", ktc, dim3(grid), dim3(kTcThreads), P.smem, s, L, P.RH, n, params, in, out, eps);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_dsblock_tc launch failed");
    return TCR_OK;
  }
#endif
  auto kfn = dscnn_dsblock_kernel;
#ifndef TCR_EMU
  static SmemOptIn optin;
  if (optin.ensure(kfn, P.smem) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_dsblock: shared memory opt-in failed");
#endif
  // one utterance per blockIdx.y: batches past kMaxGridRows run as several launches over consecutive utterances
  const size_t in_utt = (size_t)L.hin * L.win * L.cin, out_utt = (size_t)L.hout * L.wout * L.cout;
  for (int first = 0; first < n; first += kMaxGridRows) {
    TCR_LAUNCH("dscnn_dsblock", kfn, dim3(ds_tiles_per_utt(L, P.RH), std::min(n - first, kMaxGridRows)), dim3(256), P.smem, s, L, P.RH,
               P.COT, params, in + first * in_utt, out + first * out_utt, eps);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "dscnn_dsblock launch failed");
  }
  return TCR_OK;
}

int tcr::dscnn_forward(tcr_dscnn* d, const float* feat, const float* params, int n, float* logits, float* probs, cudaStream_t s,
                       const WindowView* win) {
  const float* in = feat;
  for (int l = 0; l < d->net.nlayers; ++l) {
    float* out = d->act[l & 1];
    const int rc = ds_launch_layer(d, l, params, in, out, n, s, l == 0 ? win : nullptr);
    if (rc != TCR_OK) return rc;
    in = out;
  }
  if (d->kws) return kws_head(d, params, in, n, logits, probs, s);
  if (d->kwsb) return kwsb_head(d, params, in, n, logits, probs, s);
  const DsLayerDev& last = d->net.layer[d->net.nlayers - 1];
  if (d->res2d || d->res) {
    TCR_LAUNCH("res2d_head", res2d_head_kernel, dim3(n), dim3(256), 0, s, last.hout * last.wout, last.cout, d->net.classes,
               d->res ? d->rfc : d->r2fc, params, in, logits, probs);
    if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "res2d_head launch failed");
    return TCR_OK;
  }
  if (last.cout > 320) { set_error("DS-CNN head supports up to 320 channels"); return TCR_ERR_UNSUPPORTED; }
  TCR_LAUNCH("dscnn_head", dscnn_head_kernel, dim3(n), dim3(256), 0, s, last.hout * last.wout, last.cout, d->net.classes, d->net.fcw,
             d->net.fcb, params, in, logits, probs);
  if (cudaGetLastError() != cudaSuccess) { set_error("DS-CNN launch failed"); return TCR_ERR_CUDA; }
  return TCR_OK;
}
const Frontend* tcr::dscnn_frontend(const tcr_dscnn* d) { return d->fe.frames ? &d->fe : nullptr; }
int tcr::dscnn_max_batch(const tcr_dscnn* d) { return d->cfg.max_batch; }

extern "C" int tcr_dscnn_forward(tcr_dscnn* d, const float* features, const float* params, int32_t n, float* logits, float* probs,
                                 tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !features || !params) { set_error("NULL argument"); return TCR_ERR_INVALID; }
  if (n <= 0 || n > d->cfg.max_batch) { set_error("n outside [1, max_batch]"); return TCR_ERR_INVALID; }
  return dscnn_forward(d, features, params, n, logits, probs, (cudaStream_t)stream, nullptr);
}

extern "C" int tcr_dscnn_set_frontend(tcr_dscnn* d, const tcr_config* cfg) {
  pdl_chain_reset();
  if (!d || !cfg) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  int rc = frontend_check(cfg);
  if (rc) return rc;
  int T = 0, F = 0;
  frontend_geometry(*cfg, &T, &F);
  if (T != d->cfg.height || F != d->cfg.width)
    return ds_fail(TCR_ERR_INVALID, "the front-end gives (T, F) = (%d, %d) features, the DS-CNN handle takes (height, width) = (%d, %d)",
                   T, F, d->cfg.height, d->cfg.width);
  if (cudaSetDevice(d->cfg.device) != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "cudaSetDevice(%d) failed", d->cfg.device);
  if (d->feat || d->fe.frames) {
    cudaDeviceSynchronize();                                      // no queued forward may still read the old tables
    frontend_free(&d->fe);
    cudaFree(d->feat);
    d->feat = nullptr;
  }
  tcr_config c = *cfg;
  c.device = d->cfg.device;
  c.max_batch = d->cfg.max_batch;
  rc = frontend_init(&d->fe, &c, d->sms);
  if (!rc && cudaMalloc((void**)&d->feat, (size_t)d->cfg.max_batch * T * F * sizeof(float)) != cudaSuccess)
    rc = ds_fail(TCR_ERR_CUDA, "cudaMalloc failed for the DS-CNN feature buffer");
  if (rc) frontend_free(&d->fe);
  return rc;
}

extern "C" int tcr_dscnn_mfcc_forward(tcr_dscnn* d, const void* wav, int32_t input_kind, float* features, int32_t n, tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !wav || !features) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  if (n <= 0 || n > d->cfg.max_batch) return ds_fail(TCR_ERR_INVALID, "n outside [1, max_batch]");
  if (input_kind != TCR_INPUT_WAV_F32 && input_kind != TCR_INPUT_WAV_PCM16)
    return ds_fail(TCR_ERR_INVALID, "input_kind %d: the front-end takes TCR_INPUT_WAV_F32 or TCR_INPUT_WAV_PCM16", input_kind);
  if (!d->fe.frames) return ds_fail(TCR_ERR_INVALID, "the DS-CNN handle has no front-end (call tcr_dscnn_set_frontend first)");
  return frontend_run(d->fe, wav, input_kind == TCR_INPUT_WAV_PCM16, features, n, (cudaStream_t)stream);
}

extern "C" int tcr_dscnn_forward_input(tcr_dscnn* d, const void* input, int32_t input_kind, const float* params, int32_t n, float* logits,
                                       float* probs, tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !input || !params) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  if (n <= 0 || n > d->cfg.max_batch) return ds_fail(TCR_ERR_INVALID, "n outside [1, max_batch]");
  cudaStream_t s = (cudaStream_t)stream;
  if (input_kind == TCR_INPUT_FEATURES) return dscnn_forward(d, static_cast<const float*>(input), params, n, logits, probs, s, nullptr);
  if (input_kind != TCR_INPUT_WAV_F32 && input_kind != TCR_INPUT_WAV_PCM16) return ds_fail(TCR_ERR_INVALID, "unknown input kind %d", input_kind);
  if (!d->fe.frames) return ds_fail(TCR_ERR_INVALID, "the DS-CNN handle has no front-end (call tcr_dscnn_set_frontend first)");
  const int rc = frontend_run(d->fe, input, input_kind == TCR_INPUT_WAV_PCM16, d->feat, n, s);
  if (rc) return rc;
  return dscnn_forward(d, d->feat, params, n, logits, probs, s, nullptr);
}

extern "C" int tcr_dscnn_eval_accumulate(tcr_dscnn* d, const float* scores, const float* onehot, int32_t n, int32_t topk, int64_t* counts,
                                         tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !scores || !onehot || !counts) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  if (n <= 0) return ds_fail(TCR_ERR_INVALID, "n must be positive (got %d)", n);
  if (topk < 1) return ds_fail(TCR_ERR_INVALID, "topk must be at least 1");
  eval_accumulate_launch(scores, onehot, n, d->cfg.num_classes, topk, counts, (cudaStream_t)stream);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "eval_accumulate launch failed");
  return TCR_OK;
}

extern "C" int tcr_dscnn_eval_collect(tcr_dscnn* d, const float* scores, const float* onehot, int32_t n, int32_t row_offset,
                                      int32_t capacity, float* store_scores, int32_t* store_labels, tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !scores || !onehot || !store_scores || !store_labels) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  if (const char* why = eval_rank_refusal(capacity, d->cfg.num_classes)) return ds_fail(TCR_ERR_INVALID, "capacity %d: %s", capacity, why);
  if (n <= 0 || row_offset < 0 || (int64_t)row_offset + n > capacity)
    return ds_fail(TCR_ERR_INVALID, "rows [%d, %lld) outside the store's %d rows", row_offset, (long long)row_offset + n, capacity);
  eval_collect_launch(scores, onehot, n, d->cfg.num_classes, row_offset, store_scores, store_labels, (cudaStream_t)stream);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "eval_collect launch failed");
  return TCR_OK;
}

extern "C" int tcr_dscnn_eval_rank(tcr_dscnn* d, const float* store_scores, const int32_t* store_labels, int32_t n, void* workspace,
                                   int64_t* workspace_bytes, double* result, tcr_stream stream) {
  pdl_chain_reset();
  if (!d || !workspace_bytes) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  if (const char* why = eval_rank_refusal(n, d->cfg.num_classes)) return ds_fail(TCR_ERR_INVALID, "n %d: %s", n, why);
  const int64_t need = eval_rank_workspace_bytes(n, d->cfg.num_classes);
  if (!workspace) { *workspace_bytes = need; return TCR_OK; }
  if (!store_scores || !store_labels || !result) return ds_fail(TCR_ERR_INVALID, "NULL argument");
  if (*workspace_bytes < need)
    return ds_fail(TCR_ERR_INVALID, "workspace of %lld bytes, %lld needed", (long long)*workspace_bytes, (long long)need);
  eval_rank_launch(store_scores, store_labels, n, d->cfg.num_classes, workspace, result, (cudaStream_t)stream);
  if (cudaGetLastError() != cudaSuccess) return ds_fail(TCR_ERR_CUDA, "eval_rank launch failed");
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
