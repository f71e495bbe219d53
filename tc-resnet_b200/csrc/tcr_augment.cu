// tcr_augment.cu — the per-clip input stage in front of the MFCC kernel, on the device.
//
// Replaces, for one batch, what the reference's tf.data map does per file on host threads
// (datasets/augmentation_factory.py; called from datasets/audio_data_wrapper.py:37-58 / data_wrapper_base.py:59-89):
//   decode_wav: int16 / 32768 -> f32, crop or zero-pad to desired_samples              (augmentation_factory.py:146-158)
//   silent clips ("" filename): zeros                                                   (:172-178, :193-199)
//   _shift_audio: shift by s in [-L/10, L/10) with zero fill                            (:104-143)
//   _mix_background: clip(background[o : o+L] * volume + foreground, -1, 1)             (:30-101)
// Two inputs share the per-sample body:
//   rows [n, pcm_stride] + one tcr_augment_clip per row: the host made the random draws, so the result is bit-identical to the
//     host restatement for the same draws (TF's own RNG streams are not reproducible, SURVEY.md 8c);
//   a resident dataset (tcr_dataset): row i is gathered from the clip bank at order[position + i], the draws are made here with
//     the counter-based SplitMix64 keyed by (seed, epoch, position) (include/tcr_b200.h states them), and the one-hot labels of
//     the batch are written by the same launch.
// One elementwise pass: 2 B (pcm) + 4 B (background) read, 4 B written per sample -> HBM-bound.
#include "tcr_device.cuh"
#include "tcr_net.h"

namespace tcr {

struct AugArgs {
  const int16_t* pcm; int64_t pcm_stride;      // [n][pcm_stride] int16 samples (only `length` of a row are valid)
  const tcr_augment_clip* clips;               // [n]
  const float* background;                     // concatenated background recordings (may be null: no mixing)
  int64_t background_samples;                  // floats in `background` (0: unknown, offsets are trusted)
  float* out; int clip;                        // [n][clip]
};

// Resident dataset input: the description, the batch's first position in the order, the key of the epoch's draws
struct DatasetArgs {
  tcr_dataset ds;
  int64_t position;
  uint64_t key;                                // splitmix64(seed, epoch)
  float* onehot; int classes;                  // [n][classes]
  float* out; int clip;
};

// One clip of the batch as the per-sample body reads it
struct ClipSrc {
  const int16_t* src;                          // the clip's first sample
  int valid;                                   // samples of `src` to read (crop / zero-pad to the clip length)
  int shift;
  const float* bg;                             // crop of the background recording, null: not mixed
  float volume;
};

__device__ __forceinline__ ClipSrc clip_src(const AugArgs& a, int n) {
  const tcr_augment_clip c = a.clips[n];
  ClipSrc r;
  // decode_wav crops / zero-pads to the clip length; a row never holds more than pcm_stride samples
  r.valid = c.silent ? 0 : max(0, min(min(c.length, a.clip), (int)(a.pcm_stride < 0x7fffffff ? a.pcm_stride : 0x7fffffff)));
  r.src = a.pcm + (size_t)n * a.pcm_stride;
  r.shift = c.shift;
  // a crop that would run past the end of the bank is not mixed in (the host pads short recordings, device_input_stage.py)
  const bool mix = a.background != nullptr && c.bg_offset >= 0 &&
                   (a.background_samples <= 0 || c.bg_offset + (int64_t)a.clip <= a.background_samples);
  r.bg = mix ? a.background + c.bg_offset : nullptr;
  r.volume = c.bg_volume;
  return r;
}

// Gather + draws of row n (include/tcr_b200.h, tcr_dataset).  Every read stays inside the bank and the background bank.
__device__ __forceinline__ ClipSrc clip_src(const DatasetArgs& a, int n) {
  const tcr_dataset& d = a.ds;
  const int64_t p = a.position + n;
  const int64_t idx = d.order[p];
  ClipSrc r;
  r.src = d.samples;
  r.valid = 0;
  if (idx >= 0 && idx < d.num_clips) {
    const tcr_dataset_clip c = d.clips[idx];
    if (c.offset >= 0 && c.offset <= d.num_samples) {
      r.src = d.samples + c.offset;
      r.valid = (int)max(0ll, min((long long)min(c.length, a.clip), (long long)(d.num_samples - c.offset)));
    }
  }
  const uint64_t base = 8ull * (uint64_t)p;
  const int limit = (int)(0.1 * (double)a.clip);          // int(clip_samples * 0.1), augmentation_factory.shift_audio
  r.shift = d.shift && limit > 0 ? (int)(splitmix64(a.key, base + 0) % (uint64_t)(2 * limit)) - limit : 0;
  r.bg = nullptr;
  r.volume = 0.f;
  if (d.mix && d.num_background > 0 && d.background) {
    const uint64_t b = splitmix64(a.key, base + 1) % (uint64_t)d.num_background;
    const int64_t start = d.background_table[2 * b], len = d.background_table[2 * b + 1];
    const int64_t crop = (int64_t)(splitmix64(a.key, base + 2) % (uint64_t)(max((long long)(len - a.clip), 0ll) + 1));
    const bool mixed = d.is_training && uniform01(splitmix64(a.key, base + 3)) < d.background_frequency;
    const float volume = mixed ? uniform01(splitmix64(a.key, base + 4)) * d.background_max_volume : 0.f;
    const int64_t o = start + crop;
    // volume 0 adds 0 * x to every sample: the recording is not read
    if (volume != 0.f && start >= 0 && o + (int64_t)a.clip <= d.background_samples) {
      r.bg = d.background + o;
      r.volume = volume;
    }
  }
  return r;
}

__device__ __forceinline__ void write_onehot(const AugArgs&, int) {}
__device__ __forceinline__ void write_onehot(const DatasetArgs& a, int n) {
  if (blockIdx.x != 0) return;
  const int64_t idx = a.ds.order[a.position + n];
  int label = -1;
  if (idx >= 0 && idx < a.ds.num_clips) label = a.ds.clips[idx].label;
  for (int c = threadIdx.x; c < a.classes; c += blockDim.x) a.onehot[(size_t)n * a.classes + c] = c == label ? 1.f : 0.f;
}

template <typename Args>
__global__ void __launch_bounds__(256) augment_kernel(Args a) {
  pdl_wait();
  const int n = blockIdx.y;
  const ClipSrc c = clip_src(a, n);
  write_onehot(a, n);
  float* dst = a.out + (size_t)n * a.clip;
  for (int i4 = blockIdx.x * blockDim.x + threadIdx.x; 4 * i4 < a.clip; i4 += gridDim.x * blockDim.x) {
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = 4 * i4 + k;
      const int j = i - c.shift;                                     // shift >= 0: zeros in front; shift < 0: zeros at the end
      float fg = 0.f;
      if (i < a.clip && j >= 0 && j < c.valid) fg = (float)c.src[j] * (1.0f / 32768.0f);
      float s = fg;
      if (c.bg && i < a.clip) s = __fadd_rn(__fmul_rn(c.bg[i], c.volume), fg);   // multiply, then add: two roundings like tf.multiply + tf.add
      v[k] = fminf(fmaxf(s, -1.0f), 1.0f);
    }
    if (4 * i4 + 3 < a.clip) {
      st4(dst + 4 * i4, make_float4(v[0], v[1], v[2], v[3]));
    } else {
      for (int k = 0; k < 4 && 4 * i4 + k < a.clip; ++k) dst[4 * i4 + k] = v[k];
    }
  }
}

static int augment_blocks(int clip) { return std::max(1, std::min(8, (clip / 4 + 255) / 256)); }

// One clip per blockIdx.y: batches past kMaxGridRows run as several launches over consecutive rows.  Nonzero: a launch failed.
int augment_launch(const int16_t* pcm, int64_t pcm_stride, const tcr_augment_clip* clips, const float* background, int64_t background_samples,
                   float* out, int clip, int n, cudaStream_t s) {
  for (int first = 0; first < n; first += kMaxGridRows) {
    AugArgs a{pcm + (size_t)first * pcm_stride, pcm_stride, clips + first, background, background_samples, out + (size_t)first * clip, clip};
    TCR_LAUNCH("augment", augment_kernel<AugArgs>, dim3(augment_blocks(clip), std::min(n - first, kMaxGridRows)), dim3(256), 0, s, a);
    if (cudaGetLastError() != cudaSuccess) return 1;
  }
  return 0;
}

// Row i of a slice is row first + i of the batch: its order entry and its draws are keyed by position + first + i.
int dataset_batch_launch(const tcr_dataset& ds, int64_t position, int64_t epoch, uint64_t seed, float* out, float* onehot, int clip,
                         int classes, int n, cudaStream_t s) {
  for (int first = 0; first < n; first += kMaxGridRows) {
    DatasetArgs a{ds, position + first, splitmix64(seed, (uint64_t)epoch), onehot + (size_t)first * classes, classes,
                  out + (size_t)first * clip, clip};
    TCR_LAUNCH("dataset_batch", augment_kernel<DatasetArgs>, dim3(augment_blocks(clip), std::min(n - first, kMaxGridRows)), dim3(256), 0, s, a);
    if (cudaGetLastError() != cudaSuccess) return 1;
  }
  return 0;
}

}  // namespace tcr
