// tcr_listener.cu — continuous-audio listener (include/tcr_b200.h, tcr_listener_*): S streams scored with a sliding window
// of the handle's clip length, hop_frames frames apart, K windows per stream and push.
//
// Per stream the listener keeps a sample row [tail | chunk] (tail = W_s - s samples carried from the previous push) and a
// feature history of carried + K * hop frames (carried = T - hop frames from the previous push).  A push is four launches on
// the caller's stream:
//   listener_stage  the new chunk (fp32, or int16 scaled like decode_wav) into the sample rows behind the tail;
//   mfcc            the K * hop new frames of every stream, written straight into the history behind the carried frames,
//                   by the kernel tcr_mfcc_forward selects for the handle (frame pairs or one frame per warp), so the features
//                   are bit-identical to the per-clip front-end's;
//   forward         the evaluation forward of the listener's model at n = S * K, its first layer reading window u of the batch in
//                   place from the history at (u / K) * stream + (u % K) * hop * F: TC-ResNet's conv0 (conv_fwd_kernel<3, WSMEM,
//                   true>) or DS-CNN's conv_1 (the windowed dscnn_conv* instantiations, tcr_dscnn.cu);
//   listener_roll   the last tail samples and the last carried frames of each stream to the front of their buffers.
// A reset zeroes the sample rows and fills the carried frames with the features of a silent frame (one front-end launch over
// one frame, and listener_reset to copy it): the stream then holds exactly what pushing pre = carried * s + tail zeros would
// have left, so window k of a stream is the clip starting at sample k * hop * s of the zero-prefixed stream.
// Compiled as part of tcr_net_all.cu (the network's single translation unit), not on its own.
#include <stdarg.h>
#include <stdio.h>

#include "tcr_net.h"
#include "tcr_plan.h"

using namespace tcr;

// A listener serves one model: a TC-ResNet handle (h) or a DS-CNN handle (d).  Everything but the forward call goes through the
// model's front-end (fe).
struct tcr_listener {
  tcr_handle* h = nullptr;
  tcr_dscnn* d = nullptr;
  const tcr::Frontend* fe = nullptr;
  int S = 0, hop = 0, chunk = 0, K = 0;
  int tail = 0;                // W_s - s samples carried to the next push
  int row = 0;                 // samples per stream row: tail + chunk
  int carried = 0;             // T - hop frames carried to the next push
  int64_t hist_stride = 0;     // floats per stream of the history: (carried + K * hop) * F
  float* samples = nullptr;    // [S][row]
  float* hist = nullptr;       // [S][carried + K * hop][F]
};

namespace tcr {
namespace {

constexpr int kListenThreads = 256;

int lfail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  set_error(buf);
  return code;
}

// chunk [S][chunk] -> samples[s][tail + i], four samples per thread; PCM: int16 scaled by 1/32768 like decode_wav (exact in fp32)
template <bool PCM>
__global__ void __launch_bounds__(kListenThreads) listener_stage_kernel(const void* in, float* samples, int chunk, int tail, int row) {
  pdl_wait();
  const int s = blockIdx.y;
  const int i4 = blockIdx.x * blockDim.x + threadIdx.x;
  if (4 * i4 >= chunk) return;
  float4 v;
  if (PCM) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(static_cast<const int16_t*>(in) + (size_t)s * chunk) + 2 * i4;
    const uint32_t u0 = p[0], u1 = p[1];
    v = make_float4((float)(short)(u0 & 0xffffu) * (1.0f / 32768.0f), (float)(short)(u0 >> 16) * (1.0f / 32768.0f),
                    (float)(short)(u1 & 0xffffu) * (1.0f / 32768.0f), (float)(short)(u1 >> 16) * (1.0f / 32768.0f));
  } else {
    v = ldg4(static_cast<const float*>(in) + (size_t)s * chunk + 4 * i4);
  }
  st4(samples + (size_t)s * row + tail + 4 * i4, v);
}

// base[i] = base[i + shift] for i < n (float4 units, shift > 0), in place: the CTA walks blocks of blockDim.x in ascending order
// and reads a whole block before writing it, so every read happens before the write of its address.
template <class V>
__device__ __forceinline__ void move_down(V* base, int64_t shift, int64_t n) {
  for (int64_t b = 0; b < n; b += blockDim.x) {
    const int64_t i = b + threadIdx.x;
    V v = {};
    if (i < n) v = base[i + shift];
    __syncthreads();
    if (i < n) base[i] = v;
    __syncthreads();
  }
}

// blockIdx.x = stream; y = 0: the sample tail, y = 1: the carried feature frames.  The history moves in float4 units when every
// stream row, shift and carried length is a multiple of four floats (F % 4 == 0, every TC-ResNet front-end); in floats otherwise
// (e.g. DS-CNN's 10 MFCCs).
template <class V>
__global__ void __launch_bounds__(kListenThreads) listener_roll_kernel(float* samples, float* hist, int row, int chunk, int tail,
                                                                       int64_t hist_stride, int64_t hist_shift, int64_t carry) {
  pdl_wait();
  const int s = blockIdx.x;
  constexpr int kV = sizeof(V) / sizeof(float);
  if (blockIdx.y == 0) move_down(reinterpret_cast<float4*>(samples + (size_t)s * row), chunk / 4, tail / 4);
  else move_down(reinterpret_cast<V*>(hist + (size_t)s * hist_stride), hist_shift / kV, carry / kV);
}

// frames 1 .. carried - 1 of streams first + blockIdx.y = frame 0 (the features of a silent frame)
__global__ void __launch_bounds__(kListenThreads) listener_reset_kernel(float* hist, int64_t hist_stride, int first, int carried,
                                                                        int features) {
  pdl_wait();
  float* hs = hist + (size_t)(first + blockIdx.y) * hist_stride;
  const int n = (carried - 1) * features;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) hs[features + i] = hs[i % features];
}

// Front-end over `frames` frames of rows [first, first + count): samples rows -> history frame `frame0` onwards.
int listener_frontend(tcr_listener* L, int first, int count, int frames, int frame0, cudaStream_t st) {
  MfccArgs a = mfcc_args(*L->fe, L->samples + (size_t)first * L->row, 0,
                         L->hist + (size_t)first * L->hist_stride + (size_t)frame0 * L->fe->features);
  a.clip = L->row;
  a.frames = frames;
  a.feat_stride = L->hist_stride;
  return mfcc_select_launch(*L->fe, a, count, st);
}

int listener_reset_rows(tcr_listener* L, int first, int count, cudaStream_t st) {
  if (cudaMemsetAsync(L->samples + (size_t)first * L->row, 0, (size_t)count * L->row * sizeof(float), st) != cudaSuccess)
    return lfail(TCR_ERR_CUDA, "listener reset: cudaMemsetAsync failed");
  if (L->carried == 0) return TCR_OK;                 // hop == T: no frame outlives a push
  int rc = listener_frontend(L, first, count, 1, 0, st);
  if (rc) return rc;
  if (L->carried > 1) {
    const int n = (L->carried - 1) * L->fe->features;
    for (int f = first; f < first + count; f += kMaxGridRows) {      // one stream per blockIdx.y
      const int rows = std::min(first + count - f, kMaxGridRows);
      TCR_LAUNCH("listener_reset", listener_reset_kernel, dim3((n + kListenThreads - 1) / kListenThreads, rows), dim3(kListenThreads), 0, st,
                 L->hist, L->hist_stride, f, L->carried, L->fe->features);
      if (cudaGetLastError() != cudaSuccess) return lfail(TCR_ERR_CUDA, "listener reset launch failed");
    }
  }
  return TCR_OK;
}

// The new chunk of every stream into the sample rows behind the tail, in slices of at most kMaxGridRows streams (blockIdx.y).
int listener_stage(tcr_listener* L, const void* samples, bool pcm, cudaStream_t st) {
  const size_t in_bytes = pcm ? sizeof(int16_t) : sizeof(float);
  for (int first = 0; first < L->S; first += kMaxGridRows) {
    const dim3 sgrid((L->chunk / 4 + kListenThreads - 1) / kListenThreads, std::min(L->S - first, kMaxGridRows));
    const void* in = static_cast<const char*>(samples) + (size_t)first * L->chunk * in_bytes;
    float* rows = L->samples + (size_t)first * L->row;
    if (pcm) TCR_LAUNCH("listener_stage", listener_stage_kernel<true>, sgrid, dim3(kListenThreads), 0, st, in, rows, L->chunk, L->tail, L->row);
    else TCR_LAUNCH("listener_stage", listener_stage_kernel<false>, sgrid, dim3(kListenThreads), 0, st, in, rows, L->chunk, L->tail, L->row);
    if (cudaGetLastError() != cudaSuccess) return lfail(TCR_ERR_CUDA, "listener stage launch failed");
  }
  return TCR_OK;
}

}  // namespace
}  // namespace tcr

// Shared by both handle types: L->h or L->d and L->fe are set; max_batch and device are the model handle's.
static int listener_create(tcr_listener* L, const tcr_listener_config* cfg, int max_batch, int device, tcr_listener** out) {
  const int T = L->fe->frames, W = L->fe->cfg.window_size_samples, s = L->fe->cfg.window_stride_samples;
  auto refuse = [&](int rc) {
    delete L;
    return rc;
  };
  if (cfg->streams < 1) return refuse(lfail(TCR_ERR_INVALID, "streams must be at least 1 (got %d)", cfg->streams));
  if (cfg->hop_frames < 1 || cfg->hop_frames > T)
    return refuse(lfail(TCR_ERR_INVALID, "hop_frames %d outside [1, T = %d]", cfg->hop_frames, T));
  const int64_t step = (int64_t)cfg->hop_frames * s;
  if (cfg->chunk_samples <= 0 || cfg->chunk_samples % step)
    return refuse(lfail(TCR_ERR_INVALID, "chunk_samples %d is not a positive multiple of hop_frames * window_stride_samples = %lld",
                        cfg->chunk_samples, (long long)step));
  const int K = (int)(cfg->chunk_samples / step);
  if ((int64_t)cfg->streams * K > max_batch)
    return refuse(lfail(TCR_ERR_INVALID, "streams * windows per push = %d * %d exceeds max_batch = %d", cfg->streams, K, max_batch));
  L->S = cfg->streams; L->hop = cfg->hop_frames; L->chunk = cfg->chunk_samples; L->K = K;
  L->tail = W - s;
  L->row = L->tail + L->chunk;
  L->carried = T - L->hop;
  L->hist_stride = (int64_t)(L->carried + K * L->hop) * L->fe->features;
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaMalloc((void**)&L->samples, (size_t)L->S * L->row * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&L->hist, (size_t)L->S * L->hist_stride * sizeof(float)) != cudaSuccess) {
    tcr_listener_destroy(L);
    return lfail(TCR_ERR_CUDA, "listener allocation failed (%d streams)", cfg->streams);
  }
  int rc = listener_reset_rows(L, 0, L->S, nullptr);
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = lfail(TCR_ERR_CUDA, "listener reset failed");
  if (rc) {
    tcr_listener_destroy(L);
    return rc;
  }
  *out = L;
  return TCR_OK;
}

extern "C" int tcr_listener_create(tcr_handle* h, const tcr_listener_config* cfg, tcr_listener** out) {
  pdl_chain_reset();
  if (!h || !cfg || !out) return lfail(TCR_ERR_INVALID, "NULL argument");
  *out = nullptr;
  tcr_listener* L = new tcr_listener();
  L->h = h;
  L->fe = &h->fe;
  return listener_create(L, cfg, h->cfg.max_batch, h->cfg.device, out);
}

extern "C" int tcr_dscnn_listener_create(tcr_dscnn* d, const tcr_listener_config* cfg, tcr_listener** out) {
  pdl_chain_reset();
  if (!d || !cfg || !out) return lfail(TCR_ERR_INVALID, "NULL argument");
  *out = nullptr;
  if (!dscnn_frontend(d)) return lfail(TCR_ERR_INVALID, "the DS-CNN handle has no front-end (call tcr_dscnn_set_frontend first)");
  tcr_listener* L = new tcr_listener();
  L->d = d;
  L->fe = dscnn_frontend(d);
  return listener_create(L, cfg, dscnn_max_batch(d), dscnn_frontend(d)->cfg.device, out);
}

extern "C" int tcr_listener_reset(tcr_listener* L, int32_t stream, tcr_stream stream_) {
  pdl_chain_reset();
  if (!L) return lfail(TCR_ERR_INVALID, "NULL listener");
  if (stream < -1 || stream >= L->S) return lfail(TCR_ERR_INVALID, "stream %d outside [0, %d) (or -1 for all)", stream, L->S);
  return stream < 0 ? listener_reset_rows(L, 0, L->S, (cudaStream_t)stream_) : listener_reset_rows(L, stream, 1, (cudaStream_t)stream_);
}

extern "C" int tcr_listener_push(tcr_listener* L, const void* samples, int32_t input_kind, const float* params, const float* moving,
                                 float* logits, float* probs, tcr_stream stream_) {
  pdl_chain_reset();
  if (!L || !samples || !params || (L->h && !moving))
    return lfail(TCR_ERR_INVALID, "NULL argument (listener, samples, params and, for TC-ResNet, moving are required)");
  if (L->d && moving) return lfail(TCR_ERR_INVALID, "a DS-CNN listener takes moving = NULL: its moving statistics are in params");
  if (input_kind != TCR_INPUT_WAV_F32 && input_kind != TCR_INPUT_WAV_PCM16)
    return lfail(TCR_ERR_INVALID, "input_kind %d: a listener takes TCR_INPUT_WAV_F32 or TCR_INPUT_WAV_PCM16", input_kind);
  if (((uintptr_t)samples & 15) != 0) return lfail(TCR_ERR_INVALID, "samples must be 16-byte aligned");
  const Frontend& fe = *L->fe;
  const bool pcm = input_kind == TCR_INPUT_WAV_PCM16;
  if (pcm && (fe.cfg.window_size_samples % 8 || fe.cfg.window_stride_samples % 8 || L->chunk % 8))
    return lfail(TCR_ERR_UNSUPPORTED, "int16 input needs window, stride and chunk lengths that are multiples of 8 samples");
  cudaStream_t st = (cudaStream_t)stream_;
  int rc = listener_stage(L, samples, pcm, st);
  if (rc) return rc;
  rc = listener_frontend(L, 0, L->S, L->K * L->hop, L->carried, st);
  if (rc) return rc;
  const WindowView win{L->K, L->hist_stride, (int64_t)L->hop * fe.features};
  rc = L->h ? net_forward(L->h, L->hist, params, moving, L->S * L->K, false, 0, nullptr, nullptr, 0.f, logits, probs, nullptr, false, st, &win)
            : dscnn_forward(L->d, L->hist, params, L->S * L->K, logits, probs, st, &win);
  if (rc) {
    char inner[512];
    snprintf(inner, sizeof(inner), "%s", tcr_last_error());
    return lfail(rc, "listener forward launch failed: %s", inner);
  }
  const int64_t shift = (int64_t)L->K * L->hop * fe.features, carry = (int64_t)L->carried * fe.features;
  auto roll = (L->hist_stride % 4 || shift % 4 || carry % 4) ? listener_roll_kernel<float> : listener_roll_kernel<float4>;
  TCR_LAUNCH("listener_roll", roll, dim3(L->S, 2), dim3(kListenThreads), 0, st, L->samples, L->hist, L->row, L->chunk, L->tail,
             L->hist_stride, shift, carry);
  if (cudaGetLastError() != cudaSuccess) return lfail(TCR_ERR_CUDA, "listener launch failed");
  return TCR_OK;
}

extern "C" int tcr_listener_history(const tcr_listener* L, float** history, int32_t* frames) {
  if (!L || !history || !frames) return lfail(TCR_ERR_INVALID, "NULL argument");
  *history = L->hist;
  *frames = L->carried + L->K * L->hop;
  return TCR_OK;
}

extern "C" int tcr_listener_destroy(tcr_listener* L) {
  if (!L) return TCR_OK;
  if (L->samples || L->hist) cudaDeviceSynchronize();   // no queued push may still use the buffers
  if (L->samples) cudaFree(L->samples);
  if (L->hist) cudaFree(L->hist);
  delete L;
  return TCR_OK;
}
