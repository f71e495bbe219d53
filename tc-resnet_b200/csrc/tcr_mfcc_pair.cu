// tcr_mfcc_pair.cu — the front-end kernel for the BASELINE shape (640-sample window, 320-sample stride, 1024-point real
// FFT; datasets/preprocessors.py:64-96,183-194), two frames per warp with the FFT butterflies in registers.
//
// Same arithmetic as tcr_mfcc.cu (framing, periodic Hann window, real FFT as a 512-point complex FFT + post-processing,
// power | magnitude, banded mel, log(x + 1e-6), DCT-II), restructured around what ncu showed to bound that kernel — the
// shared-memory / L1 data pipe (three Stockham passes, twiddle loads, one mel weight walk per frame) at ~60 % and the issue
// slots at ~50 %:
//   * 512 = 16 x 32.  Pass A: lane n2 holds z[n2 + 32 n1] of BOTH frames of its pair (frame b = frame a shifted by five
//     rows of 32 complex samples, so the pair needs 15 loads instead of 20), multiplies by the window and runs a 16-point
//     DFT in registers (generated straight-line code, the six zero-padding inputs pruned), then the W_512^(n2 k1) twiddle
//     (one table load serves both frames).  ONE exchange through shared memory (rows of 34 float2: conflict-free 64-bit
//     stores, conflict-free 128-bit loads).  Pass B: lane (frame, k1) runs the 32-point DFT over n2 in registers and owns
//     X[k1 + 16 k2], k2 < 32.
//   * real-FFT post-processing pairs bin k with 512 - k: the partner of lane (f, k1) register k2 is lane (f, 16 - k1)
//     register 31 - k2, a static register index, so the pairing is one shuffle per component and no shared-memory pass.
//   * mel by RUNS of bins: the band edges cut the spectrum into 65 runs; a bin of run j rises in band j with weight u and
//     falls in band j - 1 with 1 - u, so with R_j = sum u P and S_j = sum P over the run, band_m = R_m + (S_m+1 - R_m+1).
//     Every bin and ONE weight are read once (167 groups of four instead of the 282 of the band walk), for both frames from
//     one weight load.  The difference S - R loses at most eps / min(1 - u) = 6e-5 relative on a band that a single spectral
//     line dominates (min(1 - u) = 1.05e-3 over the 513 bins); measured against the fp64 restatement (tests/): features 8e-8.
//   * the DCT table sits in shared memory in lane order: one conflict-free 4-byte load per entry serves both frames.
//   * persistent CTAs (three per SM) walk the (utterance, chunk) work items; once every warp has its samples in registers the
//     TMA copy of the next item's samples is issued into the same buffer, so only a CTA's first item waits for HBM.
// Against the one-frame-per-warp kernel this issues fewer warp instructions and fewer shared-memory wavefronts per frame.
#include "tcr_device.cuh"
#include "tcr_fft_reg.cuh"
#include "tcr_mfcc.h"

namespace tcr {

namespace {

constexpr int kNF2 = 512;                    // complex FFT length
constexpr int kRowsIn = 10;                  // window / 2 / 32: rows of 32 complex samples that carry data
constexpr int kRowShift = 5;                 // stride / 2 / 32: frame b starts five rows after frame a
constexpr int kXRow = 34;                    // float2 per exchange row (32 + 2: 16-byte rows, bank stride 4 words)
constexpr int kXbufFloats = 32 * kXRow * 2;  // exchange buffer of a warp: 2 frames x 16 rows
constexpr int kPwStride = 528;               // power spectrum of frame b sits 528 floats after frame a's (other 16 banks)

__device__ __forceinline__ float2 cmul2(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -(a.y * b.y)), fmaf(a.x, b.y, a.y * b.x));
}

// complex sample n of a staged span: (x[2n], x[2n+1]); PCM: int16 scaled by 1/32768 like decode_wav (exact in fp32)
template <bool PCM>
__device__ __forceinline__ float2 raw_pair(const unsigned char* x, int n) {
  if (PCM) {
    const uint32_t u = reinterpret_cast<const uint32_t*>(x)[n];
    return make_float2((float)(short)(u & 0xffffu) * (1.0f / 32768.0f), (float)(short)(u >> 16) * (1.0f / 32768.0f));
  }
  return ld2(reinterpret_cast<const float*>(x) + 2 * n);
}

// |X[k]|^2 and |X[512-k]|^2 (or the magnitudes) of the real FFT from Z[k] and Z[512-k] of the packed complex FFT:
//   E = (Z[k] + conj Z[N-k]) / 2, O = (Z[k] - conj Z[N-k]) / 2, T = e^{-2 pi i k / fft} O, X[k] = E - i T, X[N-k] = conj(E) - i conj(T)
template <bool MAG>
__device__ __forceinline__ void real_fft_bins(float2 zk, float2 zr, float2 tw, float& pa, float& pb) {
  const float2 e = make_float2(0.5f * (zk.x + zr.x), 0.5f * (zk.y - zr.y));
  const float2 o = make_float2(0.5f * (zk.x - zr.x), 0.5f * (zk.y + zr.y));
  const float2 t = make_float2(tw.x * o.x - tw.y * o.y, tw.x * o.y + tw.y * o.x);
  const float ar = e.x + t.y, ai = e.y - t.x;
  const float br = e.x - t.y, bi = e.y + t.x;
  pa = ar * ar + ai * ai;
  pb = br * br + bi * bi;
  if (MAG) {
    pa = sqrtf(pa);
    pb = sqrtf(pb);
  }
}

}  // namespace

// Dynamic shared memory (bytes): [0,16) mbarrier | staged samples (span_max x 4) | W_512^(n2 k1) table [16][32] float2 |
// packed mel weights | per warp: exchange buffer (aliased by the two power spectra) + log-mel vectors of the two frames.
// Persistent CTAs: a CTA walks work items (utterance, chunk of fpb = 2 x warps frames) with stride gridDim.x; one warp per
// frame pair.  As soon as every warp has read its samples into registers (pass A), the TMA copy of the NEXT item's samples
// is issued into the same buffer, so only the first item of a CTA waits for HBM.
template <bool PCM, bool MAG>
__global__ void __launch_bounds__(160, 3) mfcc_pair_kernel(MfccArgs a) {
  TCR_DYNAMIC_SMEM(smem);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr int SB = PCM ? 2 : 4;

  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  unsigned char* s_wav = smem + 16;
  const int span_max = (a.fpb - 1) * a.stride + a.window;
  float* s_twa = reinterpret_cast<float*>(s_wav + (size_t)span_max * 4);
  const float* s_segw = s_twa + 2 * 16 * 32;                 // segment weights (see build_frontend_tables)
  const float* s_dct = s_segw + a.segw_len;                  // DCT entries in lane order [8][5][32]
  const int pair_len = 2 * 16 * 32 + a.segw_len + a.dct_len; // floats staged by one TMA copy
  constexpr int lms = 64;                                    // mel bins (mfcc_pair_supported)
  float* s_warp = s_twa + pair_len + (size_t)warp * (kXbufFloats + 2 * lms);
  const float2* g_tw2 = reinterpret_cast<const float2*>(a.consts + a.c_tw2);
  const float2* g_win = reinterpret_cast<const float2*>(a.consts + a.c_win);

  const int chunks = (a.frames + a.fpb - 1) / a.fpb;
  const int items = a.n_utts * chunks;
  // the runs of bins this lane walks in the three mel passes (constant table, loaded ahead of the dependency wait):
  // start/4 | groups << 8 | (weight offset / 4) << 16
  int run[3];
#pragma unroll
  for (int ps = 0; ps < 3; ++ps) run[ps] = __ldg(&a.seg_meta[32 * ps + lane]);
  auto issue = [&](int item, bool with_consts) {         // thread 0: stage the samples of a work item
    const int utt = item / chunks, f0 = (item - utt * chunks) * a.fpb;
    const int nf = min(a.fpb, a.frames - f0);
    const uint32_t bytes = (uint32_t)((nf - 1) * a.stride + a.window) * SB;
    mbar_expect_tx(bar, bytes + (with_consts ? (uint32_t)pair_len * 4u : 0u));
    tma_load_1d(s_wav, reinterpret_cast<const unsigned char*>(a.wav) + ((size_t)utt * a.clip + (size_t)f0 * a.stride) * SB, bytes, bar);
    if (with_consts) tma_load_1d(s_twa, a.consts + a.c_twa, (uint32_t)pair_len * 4u, bar);
  };
  if (threadIdx.x == 0) mbar_init(bar, 1);
  pdl_wait();                       // the wav buffer and the feature buffer belong to the caller / the previous step
  __syncthreads();
  if (threadIdx.x == 0 && (int)blockIdx.x < items) issue(blockIdx.x, true);

  const int k1 = lane & 15;
  const int partner = (lane & 16) | ((16 - k1) & 15);
  uint32_t phase = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x, phase ^= 1u) {
    const int utt = item / chunks, f0 = (item - utt * chunks) * a.fpb;
    const int nf = min(a.fpb, a.frames - f0);
    const int fa = 2 * warp;                                 // this warp's frame pair (fa, fa + 1) of the chunk
    const bool has_a = fa < nf, has_b = fa + 1 < nf;
    float2* xb = reinterpret_cast<float2*>(s_warp);
    mbar_wait(bar, phase);
    if (has_a) {
      // ---- pass A: framing + window + 16-point DFT over n1 for both frames, twiddle, exchange
      const unsigned char* x = s_wav + (size_t)fa * a.stride * SB;
      float2 raw[kRowsIn + kRowShift];
#pragma unroll
      for (int j = 0; j < kRowsIn + kRowShift; ++j)
        raw[j] = (j < kRowsIn || has_b) ? raw_pair<PCM>(x, lane + 32 * j) : make_float2(0.f, 0.f);
      float2 ina[kRowsIn], inb[kRowsIn];
#pragma unroll
      for (int r = 0; r < kRowsIn; ++r) {
        const float2 w = __ldg(g_win + lane + 32 * r);
        ina[r] = make_float2(raw[r].x * w.x, raw[r].y * w.y);
        inb[r] = make_float2(raw[r + kRowShift].x * w.x, raw[r + kRowShift].y * w.y);
      }
      float2 ya[16], yb[16];
      dft16_in10(ina, ya);
      dft16_in10(inb, yb);
      xb[lane] = ya[0];
      xb[16 * kXRow + lane] = yb[0];
      const float2* twa = reinterpret_cast<const float2*>(s_twa) + lane;
#pragma unroll
      for (int k = 1; k < 16; ++k) {
        const float2 t = twa[32 * k];
        xb[k * kXRow + lane] = cmul2(ya[k], t);
        xb[(16 + k) * kXRow + lane] = cmul2(yb[k], t);
      }
    }
    __syncthreads();                                         // every warp holds its samples in registers / the exchange buffer
    if (threadIdx.x == 0 && item + (int)gridDim.x < items) issue(item + gridDim.x, false);
    if (!has_a) continue;
    float* pw = s_warp + (lane >> 4) * kPwStride;            // this lane's frame; aliases the exchange buffer
    {
      // ---- pass B: 32-point DFT over n2; lane (f, k1) ends up with X[k1 + 16 k2] in X[k2]
      float2 v[32], X[32];
      const float* row = reinterpret_cast<const float*>(xb + lane * kXRow);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 q = ld4(row + 4 * j);
        v[2 * j] = make_float2(q.x, q.y);
        v[2 * j + 1] = make_float2(q.z, q.w);
      }
      dft32(v, X);
      __syncwarp();                                          // every row is in registers: the buffer becomes the power spectra
      // ---- real-FFT post-processing: bin k = k1 + 16 k2 pairs with 512 - k = (16 - k1) + 16 (31 - k2)
#pragma unroll
      for (int k2 = 0; k2 < 16; ++k2) {
        // k1 == 0: 512 - 16 k2 = 16 (32 - k2) lives in this very lane
        const float2 snd = (k1 == 0) ? X[(32 - k2) & 31] : X[31 - k2];
        float2 zr;
        zr.x = __shfl_sync(0xffffffffu, snd.x, partner);
        zr.y = __shfl_sync(0xffffffffu, snd.y, partner);
        const int k = k1 + 16 * k2;
        float pa, pb;
        real_fft_bins<MAG>(X[k2], zr, __ldg(g_tw2 + k), pa, pb);
        pw[k] = pa;
        pw[kNF2 - k] = pb;
      }
      if (k1 == 0) {                                         // bin 256 pairs with itself
        float pa, pb;
        real_fft_bins<MAG>(X[16], X[16], __ldg(g_tw2 + kNF2 / 2), pa, pb);
        pw[kNF2 / 2] = pb;
      }
      if (k1 < 3) pw[kNF2 + 1 + k1] = 0.f;                   // the 4-wide band walk may read three bins past the spectrum
    }
    __syncwarp();
    // ---- mel by runs of bins + log, both frames: lane walks run `lane` (pass 0), run 64 - lane (pass 1) and lane 0 run 32
    // (pass 2); per run R = sum u P (rising part of band j) and S - R = sum (1 - u) P (falling part of band j - 1)
    float* lm = s_warp + kXbufFloats;
    {
      const float* pwa = s_warp;
      const float* pwb = s_warp + kPwStride;
      float ua[3], va[3], ub[3], vb[3];
#pragma unroll
      for (int ps = 0; ps < 3; ++ps) {
        const int groups = (run[ps] >> 8) & 255;
        const float* pa = pwa + ((run[ps] & 255) << 2);
        const float* pb = pwb + ((run[ps] & 255) << 2);
        const float* tw = s_segw + ((run[ps] >> 16) << 2);
        float ra0 = 0.f, ra1 = 0.f, ra2 = 0.f, ra3 = 0.f, sa0 = 0.f, sa1 = 0.f, sa2 = 0.f, sa3 = 0.f;
        float rb0 = 0.f, rb1 = 0.f, rb2 = 0.f, rb3 = 0.f, sb0 = 0.f, sb1 = 0.f, sb2 = 0.f, sb3 = 0.f;
#pragma unroll 2
        for (int q = 0; q < groups; ++q) {
          const float4 t4 = ld4(tw + 4 * q), p4 = ld4(pa + 4 * q), r4 = ld4(pb + 4 * q);
          // marker -1: the bin belongs to a neighbouring run (weight 0, not counted in S)
          const float t0 = fmaxf(t4.x, 0.f), t1 = fmaxf(t4.y, 0.f), t2 = fmaxf(t4.z, 0.f), t3 = fmaxf(t4.w, 0.f);
          const float m0 = t4.x >= 0.f ? 1.f : 0.f, m1 = t4.y >= 0.f ? 1.f : 0.f, m2 = t4.z >= 0.f ? 1.f : 0.f, m3 = t4.w >= 0.f ? 1.f : 0.f;
          ra0 = fmaf(p4.x, t0, ra0); ra1 = fmaf(p4.y, t1, ra1); ra2 = fmaf(p4.z, t2, ra2); ra3 = fmaf(p4.w, t3, ra3);
          sa0 = fmaf(p4.x, m0, sa0); sa1 = fmaf(p4.y, m1, sa1); sa2 = fmaf(p4.z, m2, sa2); sa3 = fmaf(p4.w, m3, sa3);
          rb0 = fmaf(r4.x, t0, rb0); rb1 = fmaf(r4.y, t1, rb1); rb2 = fmaf(r4.z, t2, rb2); rb3 = fmaf(r4.w, t3, rb3);
          sb0 = fmaf(r4.x, m0, sb0); sb1 = fmaf(r4.y, m1, sb1); sb2 = fmaf(r4.z, m2, sb2); sb3 = fmaf(r4.w, m3, sb3);
        }
        ua[ps] = (ra0 + ra1) + (ra2 + ra3);
        va[ps] = ((sa0 + sa1) + (sa2 + sa3)) - ua[ps];
        ub[ps] = (rb0 + rb1) + (rb2 + rb3);
        vb[ps] = ((sb0 + sb1) + (sb2 + sb3)) - ub[ps];
      }
      // band m = R_m + (S - R)_m+1.  Band `lane`: own R of pass 0 + the falling part of run lane + 1 (next lane's pass 0; run 32
      // is lane 0's pass 2).  Band 63 - lane: R of run 63 - lane (next lane's pass 1; run 32 again) + own falling part of pass 1.
      const float va_next = __shfl_down_sync(0xffffffffu, va[0], 1), vb_next = __shfl_down_sync(0xffffffffu, vb[0], 1);
      const float ua_next = __shfl_down_sync(0xffffffffu, ua[1], 1), ub_next = __shfl_down_sync(0xffffffffu, ub[1], 1);
      const float va_32 = __shfl_sync(0xffffffffu, va[2], 0), vb_32 = __shfl_sync(0xffffffffu, vb[2], 0);
      const float ua_32 = __shfl_sync(0xffffffffu, ua[2], 0), ub_32 = __shfl_sync(0xffffffffu, ub[2], 0);
      const bool last = lane == 31;
      // the falling part is a difference: clamp the (rounding-sized) negative values it can take next to a strong line
      const float lo_a = fmaxf(ua[0] + (last ? va_32 : va_next), 0.f), lo_b = fmaxf(ub[0] + (last ? vb_32 : vb_next), 0.f);
      const float hi_a = fmaxf((last ? ua_32 : ua_next) + va[1], 0.f), hi_b = fmaxf((last ? ub_32 : ub_next) + vb[1], 0.f);
      lm[lane] = logf(lo_a + 1e-6f);
      lm[63 - lane] = logf(hi_a + 1e-6f);
      lm[lms + lane] = logf(lo_b + 1e-6f);
      lm[lms + 63 - lane] = logf(hi_b + 1e-6f);
    }
    __syncwarp();
    float* outa = a.feat + (size_t)utt * a.feat_stride + (size_t)(f0 + fa) * a.features;
    float* outb = outa + a.features;
    if (a.use_dct) {
      // DCT-II (40 of 64) for both frames: lane (q, g) = (lane / 8, lane % 8) sums mel rows m = q + 4 i for coefficients
      // c = g + 8 j; rows are folded by D[63-m][c] = (-1)^c D[m][c] (c has the parity of g); the table sits in shared memory
      // in lane order, so each entry is one conflict-free 4-byte load that serves both frames
      const int q = lane >> 3, g = lane & 7;
      float acca[5], accb[5];
#pragma unroll
      for (int j = 0; j < 5; ++j) acca[j] = accb[j] = 0.f;
      const float sgn = (g & 1) ? -1.f : 1.f;
      const float* tab = s_dct + lane;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = q + 4 * i;
        const float va = fmaf(sgn, lm[63 - m], lm[m]);
        const float vb = fmaf(sgn, lm[lms + 63 - m], lm[lms + m]);
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const float d = tab[(i * 5 + j) * 32];
          acca[j] = fmaf(va, d, acca[j]);
          accb[j] = fmaf(vb, d, accb[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        acca[j] += __shfl_xor_sync(0xffffffffu, acca[j], 8);
        accb[j] += __shfl_xor_sync(0xffffffffu, accb[j], 8);
        acca[j] += __shfl_xor_sync(0xffffffffu, acca[j], 16);
        accb[j] += __shfl_xor_sync(0xffffffffu, accb[j], 16);
        if (q == 0) {
          outa[g + 8 * j] = acca[j];
          if (has_b) outb[g + 8 * j] = accb[j];
        }
      }
    } else {
      for (int c = lane; c < a.features; c += 32) {
        outa[c] = lm[c];
        if (has_b) outb[c] = lm[lms + c];
      }
    }
    __syncwarp();
  }
}

bool mfcc_pair_supported(const MfccArgs& a, int fft_length) {
  return fft_length == 2 * kNF2 && a.window == 64 * kRowsIn && a.stride == 64 * kRowShift && a.c_twa >= 0 && (a.fpb % 2) == 0 &&
         a.fpb == 2 * a.warps && a.warps <= 5 && a.mel_bins == 64 && a.seg_meta != nullptr &&
         (a.use_dct ? (a.features == 40 && a.dct_len == 8 * 5 * 32) : a.features == 64);
}

size_t mfcc_pair_smem_bytes(const MfccArgs& a, int warps) {
  const int span_max = (a.fpb - 1) * a.stride + a.window;
  return 16 + (size_t)span_max * 4 + (size_t)(2 * 16 * 32 + a.segw_len + a.dct_len) * 4 + (size_t)warps * (kXbufFloats + 2 * 64) * 4;
}

int mfcc_pair_launch(const MfccArgs& a0, int n, int ctas, cudaStream_t stream) {
  MfccArgs a = a0;
  a.n_utts = n;
  const int items = n * ((a.frames + a.fpb - 1) / a.fpb);
  dim3 grid(ctas < items ? ctas : items, 1, 1);           // persistent: three CTAs per SM walk the work items
  dim3 block(32 * a.warps, 1, 1);
  const size_t smem = mfcc_pair_smem_bytes(a, a.warps);
  auto k = a.pcm16 ? (a.magnitude ? mfcc_pair_kernel<true, true> : mfcc_pair_kernel<true, false>)
                   : (a.magnitude ? mfcc_pair_kernel<false, true> : mfcc_pair_kernel<false, false>);
  const int sel = (a.pcm16 ? 2 : 0) + (a.magnitude ? 1 : 0);
#ifndef TCR_EMU
  static SmemOptIn optin[4];
  if (optin[sel].ensure(k, smem) != cudaSuccess) return 1;
#endif
  TCR_LAUNCH("mfcc", k, grid, block, smem, stream, a);
  return 0;
}

}  // namespace tcr
