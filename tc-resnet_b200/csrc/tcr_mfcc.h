// tcr_mfcc.h — argument block and launcher of the fused front-end kernel (tcr_mfcc.cu), and the front-end a handle owns.
#pragma once
#include <vector>

#include "tcr_device.cuh"
#include "../../include/tcr_b200.h"

namespace tcr {

// One front-end geometry and its constant tables (Hann window, twiddles, packed mel weights, DCT) and kernel choice, built by
// frontend_init (tcr_api.cu) from the front-end fields of a tcr_config.  A TC-ResNet handle owns one; a DS-CNN handle owns one
// once tcr_dscnn_set_frontend has been called.  mfcc_args / mfcc_select_launch (tcr_net.h) run it.
struct Frontend {
  tcr_config cfg = {};             // only the front-end fields are read: sample rate, clip, window, stride, mel bins, MFCCs, edges, kind
  int frames = 0, features = 0, fft = 0, fpb = 1, fwarps = 1;
  int mfcc_pair = 1, pair_fpb = 10, pair_warps = 5, c_twa = -1, pair_segw_len = 0, pair_dct_len = 0;
  int sms = 1;                     // multiprocessors of the device: the frame-pair kernel's persistent grid
  int* d_seg_meta = nullptr;       // frame-pair front-end kernel (tcr_mfcc_pair.cu)
  float* d_fe_consts = nullptr; int c_tw2 = 0, c_melw = 0, c_win = 0, c_smem = 0;   // front-end constant block (MfccArgs)
  int* d_mel_start = nullptr; int* d_mel_len = nullptr; int* d_mel_off = nullptr;
  float* d_dct = nullptr;
  std::vector<void*> allocs;       // the device tables above
  int64_t bytes = 0;
};

struct MfccArgs {
  const void* wav;          // [N, clip] fp32 samples, or int16 PCM when pcm16 != 0 (clip: the row stride in samples)
  int pcm16;
  float* feat;              // [N, frames, features], utterance u at feat + u * feat_stride
  int clip, window, stride, frames, features, mel_bins;
  int64_t feat_stride;      // floats between two utterances' features: frames * features, or a listener's history row (tcr_listener.cu)
  int fpb;                  // frames per CTA
  int warps;                // warps per CTA (<= 7): a warp takes frames warp, warp + warps, ... of the CTA's chunk
  int magnitude;            // 0: power spectrogram (MFCC path), 1: magnitude (log-mel path)
  int use_dct;              // 1: MFCC, 0: log-mel output
  // constant block (offsets in floats, each section 16-byte aligned); the first c_smem floats are staged in shared memory by
  // one TMA bulk copy:  [0, 2*fft/2) tw exp(-2 pi i n / (fft/2)) | c_melw: packed mel weights | (c_smem) |
  //   c_tw2: tw2 exp(-2 pi i k / fft), k <= fft/2 | c_win: periodic Hann window [window]
  const float* consts; int c_tw2, c_melw, c_win, c_smem;
  int n_utts;               // frame-pair kernel: utterances of the launch (set by mfcc_pair_launch)
  const int* seg_meta; int segw_len, dct_len;   // frame-pair kernel: runs of bins per (pass, lane), section lengths (floats)
  int c_twa;                // frame-pair kernel (tcr_mfcc_pair.cu): section W_512^(n2 k1) [16][32] float2 | segment weights | DCT entries in lane order; -1 when not built
  const int* mel_start;     // [mel_bins] first FFT bin of the band's walk (a multiple of four; leading weights may be zero)
  const int* mel_len;       // [mel_bins] groups of four bins in the walk
  const int* mel_off;       // [mel_bins] offset into mel_w (a multiple of four)
  const float* dct;         // [mel_bins, features]
};

size_t mfcc_smem_bytes(const MfccArgs& a, int nf2, int warps);
int mfcc_launch(const MfccArgs& a, int n, int fft_length, cudaStream_t stream);

// tcr_mfcc_pair.cu: two frames per warp, register-resident 16 x 32 FFT; only the 640 / 320 / 1024 front-end shape, an even
// number of frames per CTA and at most five warps
bool mfcc_pair_supported(const MfccArgs& a, int fft_length);
size_t mfcc_pair_smem_bytes(const MfccArgs& a, int warps);
int mfcc_pair_launch(const MfccArgs& a, int n, int ctas, cudaStream_t stream);   // ctas: persistent grid (3 per SM)

}  // namespace tcr
