// tcr_mfcc.cu — fused MFCC / log-mel front-end for sm_90a.
//
// Replaces the TF graph built by datasets/preprocessors.py:64-96 (_log_mel_spectrogram:
// stft -> power|magnitude -> mel matmul -> log(x + 1e-6)) and :183-194 (MFCC: DCT-II, first
// num_mfccs coefficients) with ONE kernel:
//   * grid = (frame chunks, utterances); a CTA owns FPB consecutive frames of one clip and stages the
//     (FPB-1)*stride + window samples it needs with a single TMA bulk copy (cp.async.bulk + mbarrier);
//   * one warp per frame: periodic-Hann window, real FFT of length fft = 2*NF2 done as a complex
//     Stockham FFT of length NF2 in shared memory (radix 8/4/2 passes, fp32, table twiddles),
//     real-FFT post-processing, power (or magnitude);
//   * banded mel accumulation (<= 2 non-zeros per FFT bin: 942 weights instead of a 513x64 matmul),
//     log(x + 1e-6), 64xF DCT from an L1-resident table, coalesced [N,T,F] store.
// Algorithmic traffic: 4*clip bytes in + 4*T*F bytes out per utterance (64,000 + 7,840 B at T=49).
#include "tcr_device.cuh"
#include "tcr_mfcc.h"

namespace tcr {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 mul_neg_i(float2 a) { return make_float2(a.y, -a.x); }   // a * (-i)

template <int R> __device__ __forceinline__ void dft_small(float2* v);
template <> __device__ __forceinline__ void dft_small<2>(float2* v) {
  float2 a = v[0], b = v[1];
  v[0] = cadd(a, b);
  v[1] = csub(a, b);
}
template <> __device__ __forceinline__ void dft_small<4>(float2* v) {
  float2 a0 = cadd(v[0], v[2]), a1 = csub(v[0], v[2]);
  float2 a2 = cadd(v[1], v[3]), a3 = mul_neg_i(csub(v[1], v[3]));
  v[0] = cadd(a0, a2);
  v[2] = csub(a0, a2);
  v[1] = cadd(a1, a3);
  v[3] = csub(a1, a3);
}
template <> __device__ __forceinline__ void dft_small<8>(float2* v) {
  float2 e[4] = {v[0], v[2], v[4], v[6]};
  float2 o[4] = {v[1], v[3], v[5], v[7]};
  dft_small<4>(e);
  dft_small<4>(o);
  const float h = 0.70710678118654752440f;
  o[1] = make_float2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));     // * (1 - i)/sqrt2
  o[2] = mul_neg_i(o[2]);                                               // * (-i)
  o[3] = make_float2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));    // * (-1 - i)/sqrt2
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    v[k] = cadd(e[k], o[k]);
    v[k + 4] = csub(e[k], o[k]);
  }
}

// Skewed index: one padding slot per 16 complex values keeps the strided Stockham stores 2-way
// (the minimum for 64-bit accesses) instead of 16-way bank conflicted.
__device__ __forceinline__ int zi(int i) { return i + (i >> 4); }

// One Stockham pass of radix R over the warp-private buffer z (N complex values, skewed).
// MAXQ = ceil(N / (32 R)) butterflies per lane, staged in registers so the pass is in place.
template <int R, int MAXQ>
__device__ __forceinline__ void fft_pass(float2* z, int N, int Ns, const float2* __restrict__ tw, int lane) {
  const int nb = N / R;
  const int tstep = N / (Ns * R);
  float2 v[MAXQ][R];
#pragma unroll
  for (int q = 0; q < MAXQ; ++q) {
    const int j = lane + 32 * q;
    if (j < nb) {
      const int k = j & (Ns - 1);
#pragma unroll
      for (int r = 0; r < R; ++r) v[q][r] = z[zi(j + r * nb)];
#pragma unroll
      for (int r = 1; r < R; ++r) v[q][r] = cmul(v[q][r], tw[k * r * tstep]);
      dft_small<R>(v[q]);
    }
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < MAXQ; ++q) {
    const int j = lane + 32 * q;
    if (j < nb) {
      const int k = j & (Ns - 1);
      const int j0 = (j - k) * R + k;
#pragma unroll
      for (int r = 0; r < R; ++r) z[zi(j0 + r * Ns)] = v[q][r];
    }
  }
  __syncwarp();
}

// First pass (Ns = 1: all twiddles are 1) fused with framing: the butterfly inputs are read straight from the staged
// samples, multiplied by the window and packed as complex z[n] = (x[2n] w[2n], x[2n+1] w[2n+1]); n >= window/2 is the zero
// padding up to the FFT length.  PCM: samples are int16 and scaled by 1/32768 like decode_wav (exact in fp32).
template <bool PCM>
__device__ __forceinline__ float2 frame_sample(const void* x, const float2* __restrict__ wtab, int n, int half_w) {
  if (n >= half_w) return make_float2(0.f, 0.f);
  float2 xs;
  if (PCM) {
    const uint32_t u = reinterpret_cast<const uint32_t*>(x)[n];
    xs = make_float2((float)(short)(u & 0xffffu) * (1.0f / 32768.0f), (float)(short)(u >> 16) * (1.0f / 32768.0f));
  } else {
    xs = ld2(reinterpret_cast<const float*>(x) + 2 * n);
  }
  const float2 ws = __ldg(wtab + n);
  return make_float2(xs.x * ws.x, xs.y * ws.y);
}
template <int R, int MAXQ, bool PCM>
__device__ __forceinline__ void fft_first_pass(const void* x, const float2* __restrict__ wtab, int half_w, float2* z, int N, int lane) {
  const int nb = N / R;
  if (R == 8 && half_w == 5 * nb) {
    // the window fills exactly five of the eight butterfly inputs (640-sample window in a 1024-point FFT): the last three are
    // the zero padding, known at compile time, so their loads, bound checks and half of the first butterfly stage fold away
#pragma unroll
    for (int q = 0; q < MAXQ; ++q) {
      const int j = lane + 32 * q;
      if (j < nb) {
        float2 v[R];
#pragma unroll
        for (int r = 0; r < R; ++r) v[r] = r < 5 ? frame_sample<PCM>(x, wtab, j + r * nb, 1 << 30) : make_float2(0.f, 0.f);
        dft_small<R>(v);
#pragma unroll
        for (int r = 0; r < R; ++r) z[zi(j * R + r)] = v[r];
      }
    }
    __syncwarp();
    return;
  }
#pragma unroll
  for (int q = 0; q < MAXQ; ++q) {
    const int j = lane + 32 * q;
    if (j < nb) {
      float2 v[R];
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = frame_sample<PCM>(x, wtab, j + r * nb, half_w);
      dft_small<R>(v);
#pragma unroll
      for (int r = 0; r < R; ++r) z[zi(j * R + r)] = v[r];
    }
  }
  __syncwarp();
}

template <int NF2, bool PCM>
__device__ __forceinline__ void fft_warp(const void* x, const float2* __restrict__ wtab, int half_w, float2* z,
                                         const float2* __restrict__ tw, int lane) {
  if (NF2 == 1024) {
    fft_first_pass<8, 4, PCM>(x, wtab, half_w, z, 1024, lane);
    fft_pass<8, 4>(z, 1024, 8, tw, lane);
    fft_pass<8, 4>(z, 1024, 64, tw, lane);
    fft_pass<2, 16>(z, 1024, 512, tw, lane);
  } else if (NF2 == 512) {
    fft_first_pass<8, 2, PCM>(x, wtab, half_w, z, 512, lane);
    fft_pass<8, 2>(z, 512, 8, tw, lane);
    fft_pass<8, 2>(z, 512, 64, tw, lane);
  } else if (NF2 == 256) {
    fft_first_pass<8, 1, PCM>(x, wtab, half_w, z, 256, lane);
    fft_pass<8, 1>(z, 256, 8, tw, lane);
    fft_pass<4, 2>(z, 256, 64, tw, lane);
  } else if (NF2 == 128) {
    fft_first_pass<8, 1, PCM>(x, wtab, half_w, z, 128, lane);
    fft_pass<4, 1>(z, 128, 8, tw, lane);
    fft_pass<4, 1>(z, 128, 32, tw, lane);
  } else {  // 64
    fft_first_pass<8, 1, PCM>(x, wtab, half_w, z, 64, lane);
    fft_pass<8, 1>(z, 64, 8, tw, lane);
  }
}

// Dynamic shared memory layout (bytes):
//   [0, 16)                         mbarrier
//   wav   : span floats             (TMA destination, 16-byte aligned)
//   tw    : NF2 float2              FFT twiddles exp(-2 pi i n / NF2)
//   per warp: z   (NF2 + NF2/16) float2, pw (NF2 + 1 [+pad]) floats, lm (mel_bins) floats
// ALIAS (fft <= 1024): the power spectrum overwrites the FFT buffer (the bins are staged in registers first), which brings
// the CTA to ~50 KB of shared memory and four CTAs (28 warps) per SM instead of three.
template <int NF2, bool PCM>
__global__ void __launch_bounds__(224, (NF2 <= 512) ? 4 : 2) mfcc_kernel(MfccArgs a) {
  constexpr bool ALIAS = NF2 <= 512;
  TCR_DYNAMIC_SMEM(smem);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int utt = blockIdx.y;
  const int f0 = blockIdx.x * a.fpb;
  const int nf = min(a.fpb, a.frames - f0);
  constexpr int SB = PCM ? 2 : 4;                         // bytes per staged sample

  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  unsigned char* s_wav = smem + 16;
  const int span_max = (a.fpb - 1) * a.stride + a.window;
  // constant block: FFT twiddles | packed mel weights staged in shared memory by one TMA bulk copy; real-FFT twiddles and the
  // window (touched once per frame) stay in global memory / L1
  float* s_const = reinterpret_cast<float*>(s_wav + (size_t)span_max * 4);
  const float2* s_tw = reinterpret_cast<const float2*>(s_const);
  const float* s_melw = s_const + a.c_melw;
  const float2* g_tw2 = reinterpret_cast<const float2*>(a.consts + a.c_tw2);
  const float2* g_win = reinterpret_cast<const float2*>(a.consts + a.c_win);
  const int z_elems = NF2 + (NF2 >> 4);
  const int pw_elems = ALIAS ? 0 : ((NF2 + 4 + 3) / 4) * 4;      // spectrum + 3 zero bins for the 4-wide band loop
  const int per_warp_floats = 2 * z_elems + pw_elems + ((a.mel_bins + 3) & ~3);
  float* s_warp = s_const + a.c_smem + (size_t)warp * per_warp_floats;
  float2* z = reinterpret_cast<float2*>(s_warp);
  float* pw = ALIAS ? s_warp : s_warp + 2 * z_elems;
  float* lm = s_warp + 2 * z_elems + pw_elems;

  const int span = (nf - 1) * a.stride + a.window;   // samples actually needed (span * SB is a multiple of 16)
  if (threadIdx.x == 0) mbar_init(bar, 1);
  pdl_wait();                       // the wav buffer and the feature buffer belong to the caller / the previous step
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, (uint32_t)span * SB + (uint32_t)a.c_smem * 4u);
    tma_load_1d(s_wav, reinterpret_cast<const unsigned char*>(a.wav) + ((size_t)utt * a.clip + (size_t)f0 * a.stride) * SB,
                (uint32_t)span * SB, bar);
    tma_load_1d(s_const, a.consts, (uint32_t)a.c_smem * 4u, bar);
  }
  mbar_wait(bar, 0);
  __syncthreads();

  const int half_w = a.window >> 1;
  for (int f = warp; f < nf; f += nwarps) {
    fft_warp<NF2, PCM>(s_wav + (size_t)f * a.stride * SB, g_win, half_w, z, s_tw, lane);
    // real-FFT post-processing, bins k and NF2-k from the same pair (Z[k], Z[NF2-k]):
    //   E = (Z[k] + conj Z[NF2-k]) / 2, O = (Z[k] - conj Z[NF2-k]) / 2, T = e^{-2 pi i k / fft} O
    //   X[k] = E - i T,  X[NF2-k] = conj(E) - i conj(T) ... written out below in components
    constexpr int NIT = NF2 / 64 + 1;                       // k = lane + 32 it <= NF2 / 2
    if (ALIAS) {
      float2 zk[NIT], zr[NIT];
#pragma unroll
      for (int it = 0; it < NIT; ++it) {
        const int k = lane + 32 * it;
        if (k <= NF2 / 2) {
          zk[it] = z[zi(k)];
          zr[it] = z[zi((NF2 - k) & (NF2 - 1))];
        }
      }
      __syncwarp();                                         // every bin is in registers: the buffer may be overwritten
#pragma unroll
      for (int it = 0; it < NIT; ++it) {
        const int k = lane + 32 * it;
        if (k <= NF2 / 2) {
          const float2 e = make_float2(0.5f * (zk[it].x + zr[it].x), 0.5f * (zk[it].y - zr[it].y));
          const float2 o = make_float2(0.5f * (zk[it].x - zr[it].x), 0.5f * (zk[it].y + zr[it].y));
          const float2 t = cmul(__ldg(&g_tw2[k]), o);
          const float ar = e.x + t.y, ai = e.y - t.x;
          const float br = e.x - t.y, bi = e.y + t.x;
          const float pa = ar * ar + ai * ai, pb = br * br + bi * bi;
          pw[k] = a.magnitude ? sqrtf(pa) : pa;
          pw[NF2 - k] = a.magnitude ? sqrtf(pb) : pb;
        }
      }
    } else {
#pragma unroll 1
      for (int k = lane; k <= NF2 / 2; k += 32) {
        const float2 zk = z[zi(k)];
        const float2 zr = z[zi((NF2 - k) & (NF2 - 1))];
        const float2 e = make_float2(0.5f * (zk.x + zr.x), 0.5f * (zk.y - zr.y));
        const float2 o = make_float2(0.5f * (zk.x - zr.x), 0.5f * (zk.y + zr.y));
        const float2 t = cmul(__ldg(&g_tw2[k]), o);
        const float ar = e.x + t.y, ai = e.y - t.x;          // X[k]
        const float br = e.x - t.y, bi = e.y + t.x;          // X[NF2-k] (imaginary part negated: only |.|^2 is used)
        const float pa = ar * ar + ai * ai, pb = br * br + bi * bi;
        pw[k] = a.magnitude ? sqrtf(pa) : pa;
        pw[NF2 - k] = a.magnitude ? sqrtf(pb) : pb;
      }
    }
    if (lane < 3) pw[NF2 + 1 + lane] = 0.f;                 // the 4-wide band loop may read up to three bins past the spectrum
    __syncwarp();
    // banded mel + log; a lane takes bins i and mel_bins-1-i so short and long bands pair up.  A band starts on a multiple of four
    // FFT bins (its packed weights carry leading / trailing zeros), so the walk is float4 loads and four independent chains.
#pragma unroll 1
    for (int i = lane; 2 * i < a.mel_bins; i += 32) {
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int m = h ? a.mel_bins - 1 - i : i;
        if (h && m == i) break;
        const int start = __ldg(&a.mel_start[m]), len4 = __ldg(&a.mel_len[m]), off = __ldg(&a.mel_off[m]);
        const float* pp = pw + start;
        const float* ww = s_melw + off;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int q = 0; q < len4; ++q) {
          const float4 p4 = ld4(pp + 4 * q), w4 = ld4(ww + 4 * q);
          a0 = fmaf(p4.x, w4.x, a0);
          a1 = fmaf(p4.y, w4.y, a1);
          a2 = fmaf(p4.z, w4.z, a2);
          a3 = fmaf(p4.w, w4.w, a3);
        }
        lm[m] = logf(((a0 + a1) + (a2 + a3)) + 1e-6f);
      }
    }
    __syncwarp();
    float* out = a.feat + (size_t)utt * a.feat_stride + (size_t)(f0 + f) * a.features;
    if (a.use_dct) {
      // DCT: lane (q, g) = (lane / 8, lane % 8) sums mel bins m = q, q + 4, ... for coefficients c = c0 + g, c0 + g + 8, ...;
      // the four quarter sums meet through two shuffles.  A pass covers 64 coefficients (eight per lane), so all 32 lanes
      // stay busy and the accumulators stay eight registers; more than 64 coefficients (up to 128) take a second pass.
      const int q = lane >> 3, g = lane & 7;
      // DCT-II rows are mirror images: D[M-1-m][c] = (-1)^c D[m][c], and c = c0 + g + 8 j has the parity of g (c0 is a
      // multiple of 64), so a lane folds the two halves of the log-mel vector first and walks only M/2 rows (odd M: the
      // middle row is added unfolded).
      const int M = a.mel_bins, half = M >> 1;
      const float sgn = (g & 1) ? -1.f : 1.f;
#pragma unroll 1
      for (int c0 = 0; c0 < a.features; c0 += 64) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        const int nj = min((a.features - c0 + 7) >> 3, 8);
        const int cg = c0 + g;                                // this lane's first coefficient of the pass
        if (a.features == 40) {                             // the usual 40 coefficients: five per lane, no bound checks
#pragma unroll 4
          for (int m = q; m < half; m += 4) {
            const float v = fmaf(sgn, lm[M - 1 - m], lm[m]);
            const float* row = a.dct + m * 40 + g;
#pragma unroll
            for (int j = 0; j < 5; ++j) acc[j] = fmaf(v, __ldg(row + 8 * j), acc[j]);
          }
        } else {
#pragma unroll 4
          for (int m = q; m < half; m += 4) {
            const float v = fmaf(sgn, lm[M - 1 - m], lm[m]);
            const float* row = a.dct + m * a.features + cg;
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (j < nj && cg + 8 * j < a.features) acc[j] = fmaf(v, __ldg(row + 8 * j), acc[j]);
          }
        }
        if ((M & 1) && q == 0) {
          const float v = lm[half];
          const float* row = a.dct + half * a.features + cg;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (j < nj && cg + 8 * j < a.features) acc[j] = fmaf(v, __ldg(row + 8 * j), acc[j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < nj) {
            acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 8);
            acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 16);
            if (q == 0 && cg + 8 * j < a.features) out[cg + 8 * j] = acc[j];
          }
        }
      }
    } else {
      for (int c = lane; c < a.features; c += 32) out[c] = lm[c];
    }
    __syncwarp();
  }
}

size_t mfcc_smem_bytes(const MfccArgs& a, int nf2, int warps) {
  const int span_max = (a.fpb - 1) * a.stride + a.window;
  const int z_elems = nf2 + (nf2 >> 4);
  const int pw_elems = nf2 <= 512 ? 0 : ((nf2 + 4 + 3) / 4) * 4;      // fft <= 1024: the power spectrum aliases the FFT buffer
  const size_t per_warp = (size_t)(2 * z_elems + pw_elems + ((a.mel_bins + 3) & ~3)) * 4;
  return 16 + (size_t)span_max * 4 + (size_t)a.c_smem * 4 + per_warp * warps;
}

// One utterance per blockIdx.y: batches past kMaxGridRows run as several launches over consecutive rows.
int mfcc_launch(const MfccArgs& a, int n, int fft_length, cudaStream_t stream) {
  const int nf2 = fft_length / 2;
  const int warps = a.warps;
  dim3 block(32 * warps, 1, 1);
  const size_t smem = mfcc_smem_bytes(a, nf2, warps);
  for (int first = 0; first < n; first += kMaxGridRows) {
    MfccArgs b = a;
    b.wav = static_cast<const char*>(a.wav) + (size_t)first * a.clip * (a.pcm16 ? 2 : 4);
    b.feat = a.feat + (size_t)first * a.feat_stride;
    dim3 grid((a.frames + a.fpb - 1) / a.fpb, n - first < kMaxGridRows ? n - first : kMaxGridRows, 1);
#ifndef TCR_EMU
#define TCR_MFCC_CASE(NF2)                                                         \
  case NF2: {                                                                      \
    auto k = a.pcm16 ? mfcc_kernel<NF2, true> : mfcc_kernel<NF2, false>;           \
    static SmemOptIn optin[2];                                                     \
    if (optin[a.pcm16 ? 1 : 0].ensure(k, smem) != cudaSuccess) return 1;           \
    TCR_LAUNCH("mfcc", k, grid, block, smem, stream, b);                           \
  } break;
#else
#define TCR_MFCC_CASE(NF2)                         \
  case NF2: {                                      \
    auto k = a.pcm16 ? mfcc_kernel<NF2, true> : mfcc_kernel<NF2, false>; \
    TCR_LAUNCH("mfcc", k, grid, block, smem, stream, b);   \
  } break;
#endif
    switch (nf2) {
      TCR_MFCC_CASE(1024)
      TCR_MFCC_CASE(512)
      TCR_MFCC_CASE(256)
      TCR_MFCC_CASE(128)
      TCR_MFCC_CASE(64)
      default:
        return 2;
    }
#undef TCR_MFCC_CASE
    if (cudaGetLastError() != cudaSuccess) return 1;
  }
  return 0;
}

}  // namespace tcr
