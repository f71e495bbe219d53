/* tcr_b200.h — C ABI of the H100-native TC-ResNet hot path (libtcr_b200.so).
 *
 * The reference (hyperconnect/TC-ResNet) has no FFI: its "plugin API" is Python-level and the
 * arithmetic runs inside TensorFlow 1.13's Session.run.  This header is the boundary a maintainer
 * binds with ctypes (see INTEGRATION.md); each entry point names the reference interface whose
 * arithmetic it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types in signatures.
 *   - every function returns an int status (TCR_OK == 0); tcr_last_error() gives the message of the
 *     last failure on the calling thread.  Functions never throw and never exit.
 *   - the CALLER owns every tensor buffer (device pointers, fp32, row-major) and the stream;
 *     the library owns only the opaque handle and its private workspace.
 *   - one handle per (GPU, stream); a handle is not thread-safe, distinct handles are independent.
 *   - all activations are (N, T, C) row-major with C fastest (== the reference's NHWC [N,T,1,C]);
 *     conv weights are HWIO [k,1,C_in,C_out] exactly as TF stores them, so flat parameter buffers
 *     can be filled from / dumped to reference checkpoints by name (tcr_param_table).
 */
#ifndef TCR_B200_H_
#define TCR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TCR_ABI_VERSION 16

enum {
  TCR_OK = 0,
  TCR_ERR_INVALID = 1,      /* bad argument / unsupported configuration */
  TCR_ERR_CUDA = 2,         /* CUDA runtime or launch failure */
  TCR_ERR_UNSUPPORTED = 3,
  TCR_ERR_COMM = 4          /* NCCL failure or libnccl not loadable */
};

enum { TCR_MODEL_TCRESNET8 = 8, TCR_MODEL_TCRESNET14 = 14 };
enum { TCR_FEATURE_MFCC = 0, TCR_FEATURE_LOG_MEL = 1 };
/* What `input` points at (the `input_is_features` argument / field):
 *   TCR_INPUT_WAV_F32   fp32 samples in [-1,1], the output of contrib_audio.decode_wav + augmentation
 *                       (datasets/audio_data_wrapper.py:57-112);
 *   TCR_INPUT_FEATURES  precomputed features [n,T,F];
 *   TCR_INPUT_WAV_PCM16 int16 PCM samples as stored in the wav files; the kernel applies decode_wav's 1/32768 scaling
 *                       (exact in fp32), so the result is bit-identical to TCR_INPUT_WAV_F32 on the decoded samples.
 *                       Halves the host->device bytes of an un-augmented (evaluation / inference) batch. */
enum { TCR_INPUT_WAV_F32 = 0, TCR_INPUT_FEATURES = 1, TCR_INPUT_WAV_PCM16 = 2 };

typedef struct tcr_handle tcr_handle;
typedef void* tcr_stream;   /* cudaStream_t */

/* Everything that fixes shapes.  Mirrors the flags the reference threads through `args`:
 * datasets/audio_data_wrapper.py:61-110 (sample_rate, clip_duration_ms, window_size_ms,
 * window_stride_ms, num_mel_bins, num_mfccs, lower/upper_edge_hertz), factory/base.py:13-35
 * (num_classes, preprocess_method), factory/audio_nets.py:366-370 (width_multiplier,
 * dropout_keep_prob), audio_nets/tc_resnet.py:102-123 (BN decay 0.997, eps 0.001). */
typedef struct tcr_config {
  int32_t model;                  /* TCR_MODEL_TCRESNET8 | TCR_MODEL_TCRESNET14 (audio_nets/tc_resnet.py:57,65) */
  float   width_multiplier;       /* channels = int(c * width_multiplier); every count must be a multiple of 4 */
  int32_t num_classes;            /* 12 */
  int32_t sample_rate;            /* 16000 */
  int32_t clip_samples;           /* int(sample_rate * clip_duration_ms / 1000) = 16000 */
  int32_t window_size_samples;    /* int(sample_rate * window_size_ms / 1000): 640 (T=49) or 480 (T=98) */
  int32_t window_stride_samples;  /* 320 or 160 */
  int32_t num_mel_bins;           /* 64; at most 128 */
  int32_t num_mfccs;              /* 40; a multiple of 4, at most num_mel_bins (so at most 128); ignored for TCR_FEATURE_LOG_MEL */
  float   lower_edge_hertz;       /* 80 */
  float   upper_edge_hertz;       /* 7600 */
  int32_t feature_kind;           /* TCR_FEATURE_MFCC (power + DCT) | TCR_FEATURE_LOG_MEL (magnitude, no DCT) */
  int32_t max_batch;              /* workspace is sized for this many utterances per call */
  float   bn_decay;               /* 0.997 */
  float   bn_epsilon;             /* 0.001 */
  float   dropout_keep_prob;      /* 0.5 (1.0 disables dropout) */
  float   label_smoothing;        /* 0.0 */
  int32_t device;                 /* CUDA device ordinal */
} tcr_config;

typedef struct tcr_info {
  int32_t abi_version;
  int32_t frames;          /* T  = 1 + (clip - window) / stride */
  int32_t features;        /* F  = num_mfccs or num_mel_bins */
  int32_t fft_length;      /* next pow2 >= window */
  int32_t num_conv_layers; /* conv0 + per block (down?) + 2 */
  int32_t num_blocks;
  int32_t last_channels;
  int32_t last_frames;
  int64_t num_trainable;   /* floats in the flat `params`, `slots`, `grads` buffers */
  int64_t num_moving;      /* floats in the flat BN moving-statistics buffer */
  int64_t forward_flops_per_utt;   /* 2 FLOP per MAC, network only */
  int64_t workspace_bytes;
} tcr_info;

/* Optimizer of a training step (tcr_step_args::optimizer), the choices of helper/trainer.py:171-197 on the accelerated
 * path.  "gd" is TCR_OPT_MOMENTUM with momentum 0. */
enum { TCR_OPT_MOMENTUM = 0, TCR_OPT_ADAM = 1, TCR_OPT_RMSPROP = 2 };

enum { TCR_KIND_WEIGHT = 0, TCR_KIND_BETA = 1, TCR_KIND_GAMMA = 2, TCR_KIND_MOVING_MEAN = 3, TCR_KIND_MOVING_VAR = 4 };

/* One row per TF variable.  `name` is the reference's variable name (e.g.
 * "TCResNet8/block0/conv0_0/BatchNorm/gamma"); trainables come first in
 * tf.trainable_variables() order (offsets into params/slots/grads), then the moving statistics
 * (offsets into the moving buffer).  Replaces the by-name access of common/model_loader.py:87-165
 * and the injection hook helper/trainer.py:145-154. */
typedef struct tcr_param_desc {
  char    name[96];
  int32_t kind;
  int32_t rank;
  int32_t shape[4];
  int64_t offset;
  int64_t numel;
} tcr_param_desc;

struct tcr_augment_clip;
struct tcr_dataset;
/* Arguments of one training step == one `session.run(train_op)` of helper/trainer.py:312-321. */
typedef struct tcr_step_args {
  const float* input;        /* wav [n, clip_samples] in [-1,1], features [n,T,F], or (cast) int16 PCM: see TCR_INPUT_* */
  int32_t      input_is_features;   /* TCR_INPUT_WAV_F32 | TCR_INPUT_FEATURES | TCR_INPUT_WAV_PCM16 */
  const float* onehot;       /* [n, num_classes] fp32 (datasets/audio_data_wrapper.py:113-118) */
  int32_t      n;            /* utterances on THIS rank */
  float*       params;       /* flat trainables, updated in place */
  float*       slots;        /* flat first optimizer slot, updated in place: `<var>/Momentum` (momentum accumulator),
                              * `<var>/Adam` (m, zero-initialised) or `<var>/RMSProp` (ms, initialised to 1.0) */
  float*       moving;       /* flat BN moving mean/variance, updated in place */
  float        learning_rate;
  float        momentum;     /* 0.9 (MomentumOptimizer); RMSPropOptimizer's momentum (0 by default); unused by Adam */
  float        weight_decay; /* 0.001 */
  uint64_t     dropout_seed; /* counter-based RNG seed; ignored when dropout_mask != NULL or keep_prob == 1 */
  const float* dropout_mask; /* optional injected {0,1} mask [n, last_channels] (parity runs) */
  float*       losses;       /* optional device [2]: total_loss, model_loss (factory/audio_nets.py:161-183) */
  float*       logits;       /* optional device [n, num_classes] */
  float*       probs;        /* optional device [n, num_classes] softmax (output/softmax) */
  float*       grads;        /* optional device [num_trainable]: gradient of total_loss actually applied */
  int32_t      apply_update; /* 1: optimizer update + BN moving update; 0: gradients only (params, slots, moving untouched) */
  /* Optional device input stage in front of the front-end (TCR_INPUT_WAV_PCM16 only, see tcr_augment_pcm16): when `clips` is not
   * NULL, `input` holds the wav files' int16 samples [n, pcm_stride] and the step first decodes / shifts / mixes / clips them
   * into an internal fp32 buffer.  Zero-initialise these fields when the stage is not used. */
  const struct tcr_augment_clip* clips;   /* [n]: device memory (tcr_train_step) / pinned host memory (tcr_train_step_host) */
  const float* background;   /* device: concatenated background recordings, may be NULL */
  int64_t      pcm_stride;   /* int16 samples per row of `input`; 0 = clip_samples; at most 2 * clip_samples */
  /* 1: the caller promises that `input` (and `clips`) are final when the call is made, i.e. no work queued on `stream` writes
   * them.  The front-end (input stage + MFCC) of this step then runs on the library's own low-priority stream into one of two
   * feature buffers and overlaps the tail of the previous step (weight-gradient tail, update, the cross-GPU arrival barrier);
   * the rest of the step waits for it on `stream`.  0: everything is ordered on `stream` (the default; zero-initialise).
   * tcr_train_step_host sets it itself: its inputs arrive on the library's copy stream. */
  int32_t      input_resident;
  /* Optimizer (ABI 7).  Zero-initialised, these fields select the momentum step above.  The rules, per parameter in fp32 with
   * g the (rank-averaged) gradient, are TF 1.13's:
   *   TCR_OPT_MOMENTUM  slots = slots*momentum + g;  params -= learning_rate*slots
   *   TCR_OPT_ADAM      alpha = learning_rate*sqrt(1 - beta2_power)/(1 - beta1_power);
   *                     slots += (g - slots)(1 - beta1);  slots2 += (g^2 - slots2)(1 - beta2);
   *                     params -= (slots*alpha)/(sqrt(slots2) + epsilon)                     (tf.train.AdamOptimizer)
   *   TCR_OPT_RMSPROP   slots += (g^2 - slots)(1 - rho);  slots2 = slots2*momentum + g*learning_rate/sqrt(slots + epsilon);
   *                     params -= slots2                                                    (tf.train.RMSPropOptimizer)
   * beta1_power / beta2_power are Adam's beta^t BEFORE this step (beta1 / beta2 at the first step); the caller advances them
   * (beta *= beta) after each submitted step, as TF's finish op does.  They are plain values, so tcr_train_step_host captures
   * them with the call.  Rejected with TCR_ERR_INVALID: an unknown kind, apply_update with Adam / RMSProp and no slots2,
   * beta1_power == 1. */
  int32_t      optimizer;    /* TCR_OPT_MOMENTUM | TCR_OPT_ADAM | TCR_OPT_RMSPROP */
  float*       slots2;       /* flat second slot: `<var>/Adam_1` (v, zero-initialised) or `<var>/RMSProp_1` (mom, zero) */
  float        beta1;        /* Adam: 0.9 */
  float        beta2;        /* Adam: 0.999 */
  float        epsilon;      /* Adam: 1e-8; RMSProp: 1e-10 */
  float        rho;          /* RMSProp decay: 0.9 */
  float        beta1_power;  /* Adam: beta1^t before this step */
  float        beta2_power;  /* Adam: beta2^t before this step */
  /* Exponential moving average of the trained weights (ABI 8), tf.train.ExponentialMovingAverage(decay).apply(variables_to_train)
   * run behind the train op (helper/trainer.py:213-217): after the optimizer step, per TRAINED parameter in fp32 and on the
   * updated weight, ema -= (ema - params) * (1 - ema_decay) (no num_updates, no zero-debias).  Entries of frozen variables
   * (tcr_set_trainable) are not touched.  NULL = off (zero-initialise); with apply_update == 0 nothing is averaged.
   * Rejected with TCR_ERR_INVALID: ema_decay outside [0, 1] when ema is set. */
  float*       ema;          /* flat shadow `<var>/ExponentialMovingAverage` [num_trainable], updated in place */
  float        ema_decay;    /* 0.999 (--ema_decay) */
  /* Resident dataset input (ABI 9, see tcr_dataset).  NULL (zero-initialised): the step reads `input` and `onehot` as above.
   * Otherwise the input stage gathers rows [dataset_position, dataset_position + n) of the dataset's order from the clip bank,
   * augments them with draws keyed by (dataset_seed, dataset_epoch, position) and writes their one-hot labels into a workspace
   * buffer; `input`, `input_is_features`, `onehot`, `clips`, `background` and `pcm_stride` are ignored.  The bank is final when
   * the step is submitted, so input_resident = 1 is valid.  Rejected with TCR_ERR_INVALID: dataset_position < 0 or
   * dataset_position + n > order_length.  tcr_train_step only: tcr_train_step_host rejects it. */
  const struct tcr_dataset* dataset;   /* host pointer to the caller's description, read during the call */
  int64_t      dataset_position;
  int64_t      dataset_epoch;
  uint64_t     dataset_seed;
} tcr_step_args;

int         tcr_abi_version(void);
const char* tcr_last_error(void);

/* Fills *cfg with the BASELINE shape: TCResNet8-1.0, 16 kHz 1 s clips, 40 ms / 20 ms windows (T=49). */
int tcr_config_default(tcr_config* cfg);

/* Builds the layer plan, constant tables (Hann window, FFT twiddles, banded mel weights, DCT) and
 * the device workspace.  Replaces graph construction in AudioNetModel.build
 * (factory/audio_nets.py:41-60) and tc_resnet (audio_nets/tc_resnet.py:6-54). */
int tcr_create(const tcr_config* cfg, tcr_handle** out);
int tcr_destroy(tcr_handle* h);
int tcr_get_info(const tcr_handle* h, tcr_info* out);
int tcr_param_table(const tcr_handle* h, const tcr_param_desc** descs, int32_t* count);

/* Xavier-uniform weights, gamma=1, beta=0, moving mean/var = 0/1, slots = 0
 * (TCResNet_arg_scope, audio_nets/tc_resnet.py:102-123).  Host-side RNG (not TF's), written with
 * cudaMemcpyAsync on `stream`.  Any of params/slots/moving may be NULL. */
int tcr_init_variables(tcr_handle* h, float* params, float* slots, float* moving, uint64_t seed, tcr_stream stream);

/* Front-end only: wav [n, clip_samples] -> features [n, T, F].
 * Replaces MFCCPreprocessor._preprocess / LogMelSpectrogramPreprocessor._preprocess
 * (datasets/preprocessors.py:64-96, 162-170, 183-194). */
int tcr_mfcc_forward(tcr_handle* h, const float* wav, float* features, int32_t n, tcr_stream stream);
/* Same front-end on int16 PCM samples [n, clip_samples] (decode_wav's 1/32768 scaling fused into the framing). */
int tcr_mfcc_forward_pcm16(tcr_handle* h, const int16_t* pcm, float* features, int32_t n, tcr_stream stream);

/* The per-clip input stage in front of the front-end, on the device (SURVEY.md 8f "next" row 1): decode_wav scaling, crop /
 * zero-pad to clip_samples, silent clips, time shift with zero fill, background mix and clip to [-1,1]
 * (datasets/augmentation_factory.py:30-211 as called from datasets/audio_data_wrapper.py:37-58).  The host makes the random
 * draws and passes them per clip, so the output is bit-identical to the host stage for the same draws.
 *   pcm        device int16 [n, pcm_stride]: the wav files' samples (row i holds clips[i].length valid samples)
 *   clips      device [n] tcr_augment_clip
 *   background device float: the background recordings concatenated (NULL: no mixing); bg_offset indexes into it
 *   wav_out    device float [n, clip_samples], what tcr_mfcc_forward / tcr_train_step take as TCR_INPUT_WAV_F32 */
typedef struct tcr_augment_clip {
  int32_t length;      /* valid int16 samples of the clip's row (longer clips are cropped, shorter zero-padded) */
  int32_t shift;       /* _shift_audio: out[i] = in[i - shift], zero outside; 0 for anchored_slice_or_pad */
  int32_t silent;      /* 1: the "" filename of a synthesised silent sample: zeros before the background mix */
  float   bg_volume;   /* 0 when the background is not mixed in (probability 1 - background_frequency, or evaluation) */
  int64_t bg_offset;   /* start of the random crop inside `background` (recording start + crop offset); < 0: none */
} tcr_augment_clip;
int tcr_augment_pcm16(tcr_handle* h, const int16_t* pcm, int64_t pcm_stride, const tcr_augment_clip* clips,
                      const float* background, float* wav_out, int32_t n, tcr_stream stream);
/* Length (floats) of the background bank the `background` pointers refer to: a clip whose crop [bg_offset, bg_offset + clip_samples)
 * does not fit is not mixed (instead of reading past the bank).  0 (default): offsets are trusted.  The host stage pads
 * recordings shorter than a clip, as augmentation_factory.py:60-75 does. */
int tcr_set_background_samples(tcr_handle* h, int64_t samples);

/* A dataset split resident in device memory (ABI 9): every clip decoded once into one int16 bank, each batch gathered and
 * augmented on the device with random draws made in the kernel, so the host does no work per batch (the per-file tf.data map of
 * datasets/audio_data_wrapper.py:37-58 and datasets/augmentation_factory.py:30-211).  Every pointer is device memory owned by
 * the caller; the struct itself is host memory and is read during the call only.
 *
 * Row i of a batch at `position` is clip clips[order[position + i]]: its `length` samples from samples[offset], cropped to
 * clip_samples and zero-padded, then shifted, mixed and clipped exactly as tcr_augment_pcm16 does.  The draws of the row at
 * global position p (an index into `order`) are, with key = splitmix64(seed, epoch) and z_k = splitmix64(key, 8 p + k),
 * splitmix64(s, i) the SplitMix64 output of the state s + 0x9E3779B97F4A7C15 * (i + 1) and u(z) = (z >> 40) / 2^24 in fp32:
 *   shift      z0 % (2 S) - S, S = int(0.1 * clip_samples)                       (`shift` set and S > 0; else 0)
 *   recording  b = z1 % num_background, crop z2 % (length_b - clip_samples + 1)  (`mix` set and num_background > 0)
 *   mixed      is_training && u(z3) < background_frequency
 *   volume     u(z4) * background_max_volume in fp32 when mixed, else 0 (the recording is then not read: 0 * x + y == y)
 * The draws depend on the global position, not on the caller's rank or batch size, so data-parallel ranks reading their rows
 * at position + rank * n get the rows and draws of one device running the global batch.  No read leaves `samples` or
 * `background`: an order entry outside [0, num_clips) is a silent row with an all-zero one-hot row, a clip whose samples lie
 * outside the bank is read only as far as it lies inside, a label outside [0, num_classes) gives an all-zero one-hot row and a
 * crop that does not fit `background_samples` is not mixed. */
typedef struct tcr_dataset_clip {
  int64_t offset;      /* first sample of the clip in `samples` */
  int32_t length;      /* samples stored, at most clip_samples; 0 for a silent sample (the "" filename) */
  int32_t label;       /* class index of the one-hot row */
} tcr_dataset_clip;
typedef struct tcr_dataset {
  const int16_t*          samples;            /* the clip bank: every clip's int16 samples back to back */
  int64_t                 num_samples;
  const tcr_dataset_clip* clips;              /* [num_clips] */
  int64_t                 num_clips;
  const int32_t*          order;              /* [order_length] clip indices: the epoch's shuffled order */
  int64_t                 order_length;
  const float*            background;         /* concatenated background recordings, each at least clip_samples long */
  int64_t                 background_samples;
  const int64_t*          background_table;   /* [num_background][2]: start and length of each recording in `background` */
  int32_t                 num_background;
  int32_t                 shift;              /* 1: anchored_slice_or_pad_with_shift */
  int32_t                 mix;                /* 1: draw a recording and mix it in */
  int32_t                 is_training;        /* 0: volume 0, as the evaluation graph */
  float                   background_frequency;    /* 0.8 */
  float                   background_max_volume;   /* 0.1 */
} tcr_dataset;
/* One batch of a resident dataset: rows [position, position + n) of its order, gathered and augmented (see tcr_dataset) into
 * wav_out [n, clip_samples] (16-byte aligned) and their one-hot labels into onehot_out [n, num_classes], in one launch.
 * For evaluation and inspection; a training step takes the dataset itself (tcr_step_args::dataset).
 * TCR_ERR_INVALID: position < 0 or position + n > order_length, a NULL pointer. */
int tcr_dataset_batch(tcr_handle* h, const tcr_dataset* desc, int64_t position, int64_t epoch, uint64_t seed, int32_t n,
                      float* wav_out, float* onehot_out, tcr_stream stream);

/* Forward pass.  is_training == 0: evaluate_audio.py path (BN moving statistics, dropout identity;
 * helper/base.py:52-125).  is_training == 1: the training graph's forward (batch statistics, dropout)
 * as run by the trainer's in-loop evaluation (helper/trainer.py:436-460); `moving` is not updated.
 * onehot/losses may be NULL; when both are given losses[0..1] = total_loss, model_loss. */
int tcr_forward(tcr_handle* h, const float* input, int32_t input_is_features, const float* params,
                const float* moving, int32_t n, int32_t is_training, uint64_t dropout_seed,
                const float* dropout_mask, const float* onehot, float weight_decay,
                float* logits, float* probs, float* losses, tcr_stream stream);

/* Continuous-audio listener (ABI 10): scores S independent audio streams with a sliding window, the job the deploy graph of
 * factory/audio_nets.py:87-125 is run for, without recomputing a frame of features per window it falls into.
 *
 * A listener belongs to one handle and shares its geometry: T frames, window W_s and stride s samples.  Each push hands it
 * chunk_samples new samples per stream (a multiple of hop_frames * s) and emits exactly K = chunk_samples / (hop_frames * s)
 * windows per stream.  The result equals an offline computation exactly:
 *   1. after create or reset, a stream acts as if pre = (T - hop_frames) * s + (W_s - s) zero samples had already been pushed;
 *   2. window k of a stream (counted from the reset) is made of frames [k * hop_frames, k * hop_frames + T) of that zero-prefixed
 *      sample sequence, i.e. the clip of clip_samples samples that starts at sample k * hop_frames * s; it ends (k + 1) *
 *      hop_frames * s samples after the reset;
 *   3. its logits and softmax equal tcr_forward in evaluation mode (moving BatchNorm statistics, no dropout) on that clip, bit
 *      for bit: a push computes each new frame once with the front-end kernel tcr_mfcc_forward selects for the handle, and conv0
 *      reads every window in place from the stream's feature history; the rest is the evaluation forward at n = S * K.
 * So a stream is just the concatenation of its pushes.
 *
 * The listener owns its persistent state (per stream: the last W_s - s samples and the last T - hop_frames feature frames); it
 * borrows the handle's layer workspace for the forward pass, so a handle and its listeners follow the handle's rule: one stream,
 * not thread-safe.  Training steps may run on the handle between pushes.  (`tcr_stream` is the cudaStream_t type above.)
 *
 * tcr_listener_create  TCR_ERR_INVALID: streams < 1, hop_frames outside [1, T], chunk_samples not a positive multiple of
 *                      hop_frames * s, streams * K > max_batch.  Every stream starts reset; the call synchronises the device.
 * tcr_listener_reset   stream: index of the stream to reset, or -1 for all of them (TCR_ERR_INVALID otherwise).
 * tcr_listener_push    samples: device [S, chunk_samples], fp32 in [-1,1] (TCR_INPUT_WAV_F32) or int16 PCM (TCR_INPUT_WAV_PCM16,
 *                      decode_wav's 1/32768 scaling, bit-identical to the decoded fp32 samples), 16-byte aligned;
 *                      logits / probs: device [S, K, num_classes] or NULL.  TCR_ERR_INVALID: a NULL handle / samples / params,
 *                      a NULL `moving` on a TC-ResNet listener or a non-NULL one on a DS-CNN listener (tcr_dscnn_listener_create),
 *                      another input kind, a misaligned samples pointer.  TCR_ERR_UNSUPPORTED: int16 input with window, stride
 *                      or chunk lengths that are not multiples of 8 samples (as tcr_forward).
 * tcr_listener_destroy frees the listener's buffers (NULL is a no-op); destroy listeners before their handle. */
typedef struct tcr_listener tcr_listener;
typedef struct tcr_listener_config {
  int32_t streams;         /* S */
  int32_t hop_frames;      /* frames between two windows of a stream, in [1, T] */
  int32_t chunk_samples;   /* samples per stream and push, a multiple of hop_frames * window_stride_samples */
} tcr_listener_config;
int tcr_listener_create(tcr_handle* h, const tcr_listener_config* cfg, tcr_listener** out);
int tcr_listener_reset(tcr_listener* L, int32_t stream, tcr_stream stream_);
int tcr_listener_push(tcr_listener* L, const void* samples, int32_t input_kind, const float* params, const float* moving,
                      float* logits, float* probs, tcr_stream stream_);
int tcr_listener_destroy(tcr_listener* L);
/* Inspection: device pointer of the feature history [S][*frames][F] (*frames = T - hop_frames + K * hop_frames).  Between calls,
 * frames [0, T - hop_frames) of each stream are the last T - hop_frames frames of that stream, which the next push's first
 * window starts with (after a reset: the features of silence). */
int tcr_listener_history(const tcr_listener* L, float** history, int32_t* frames);

/* The evaluation consumer behind the forward pass, on the device (SURVEY.md 8f row 3): reduces one batch of scores and
 * one-hot labels to the integers every count-based metric of the reference is a function of, instead of shipping
 * [n, classes] arrays to the host per batch (helper/base.py:52-143, metrics/parser.py:135-147; accuracy, top-5, precision,
 * recall, F1, classification report: metrics/ops/non_tensor_ops.py:64-142, :146-295, :346-).
 *   scores  device [n, classes]: logits or softmax outputs of tcr_forward (arg-max and ranks are the same for both)
 *   onehot  device [n, classes]
 *   counts  device int64 [classes*classes + 2], ACCUMULATED (zero it before the first batch):
 *           [y*classes + p] confusion matrix (true row, predicted column), y and p the np.argmax of the one-hot and score rows:
 *                           the first NaN if the row has one, else the first maximum (+0 and -0 are equal),
 *           [classes*classes] utterances whose true class is among the first `topk` of np.argsort(-scores, kind="stable"): a
 *                           numeric true score ranks after the greater scores and the equal ones at lower class indices, a NaN
 *                           true score after every number and the NaNs at lower indices; topk >= classes counts every row,
 *           [classes*classes + 1] utterances */
int tcr_eval_accumulate(tcr_handle* h, const float* scores, const float* onehot, int32_t n, int32_t topk, int64_t* counts,
                        tcr_stream stream);

/* Ranking metrics on the device (ABI 15): the reference's MAPMetricOp (average_precision_score at macro, micro, weighted and
 * samples) and APMetricOp (per-class AP), metrics/ops/non_tensor_ops.py:15-61, :296-343.  Scores stay on the device for the whole
 * evaluation in a caller-owned store; one ranking pass at the end computes every AP.
 *   tcr_eval_collect  appends rows [row_offset, row_offset + n) of the store: store_scores device fp32 [capacity, classes] <- scores,
 *                     store_labels device int32 [capacity] <- the first maximum of each one-hot row (tcr_eval_accumulate's rule).
 *                     scores MUST be the softmax outputs (tcr_forward's probs), as the reference ranks predictions_onehot: unlike
 *                     the arg-max, a class's ranking across utterances differs between logits and softmax.
 *                     TCR_ERR_INVALID unless capacity * classes <= 2^31 - 1 and the rows lie inside [0, capacity).
 *   tcr_eval_rank     ranks the store's first n rows.  workspace == NULL is the query: *workspace_bytes <- the device bytes the
 *                     pass needs, nothing runs.  Otherwise workspace (device, 256-byte aligned, *workspace_bytes of it) is scratch
 *                     and result (device fp64 [2 * classes + 4]) receives:
 *                       [0, classes)            AP of each class, sklearn's definition: the class's n scores sorted in descending
 *                                               order, equal scores grouped, sum over groups of (R_g - R_{g-1}) * P_g; 0 for a
 *                                               class without positives (sklearn 1.x);
 *                       [classes, 2 * classes)  positives of each class (the support);
 *                       [2 * classes + 0]       macro: the mean of the per-class APs;
 *                       [2 * classes + 1]       micro: the AP of all n * classes (score, is-label) pairs ranked together;
 *                       [2 * classes + 2]       weighted: the per-class APs weighted by their support;
 *                       [2 * classes + 3]       samples: the mean over rows of 1 / |{c : p_c >= p_label}|.
 *                     A NaN score makes every average it enters NaN.  The result is deterministic and depends only on the stored
 *                     rows, not on how many rows each collect call wrote.  TCR_ERR_INVALID unless classes <= 32 and
 *                     1 <= n with n * classes <= 2^31 - 1. */
int tcr_eval_collect(tcr_handle* h, const float* scores, const float* onehot, int32_t n, int32_t row_offset, int32_t capacity,
                     float* store_scores, int32_t* store_labels, tcr_stream stream);
int tcr_eval_rank(tcr_handle* h, const float* store_scores, const int32_t* store_labels, int32_t n, void* workspace,
                  int64_t* workspace_bytes, double* result, tcr_stream stream);

/* Forward + backward + optimizer (momentum, Adam or RMSProp: tcr_step_args::optimizer) + BN moving-average update
 * (helper/trainer.py:171-222, slim.learning.create_train_op).  With a communicator attached (tcr_comm_init) gradients are
 * averaged over ranks with one ncclAllReduce (or the peer-memory exchange) before the update; every rank then applies the
 * same update to the same averaged gradient, so the optimizer state stays identical across replicas. */
int tcr_train_step(tcr_handle* h, const tcr_step_args* args, tcr_stream stream);

/* Which variables the training steps of this handle train (--trainable_scopes: slim.learning.create_train_op's
 * variables_to_train, helper/trainer.py:199-222, resolved by common/tf_utils.py:19-37).  `flags`: one int per TRAINABLE row of
 * tcr_param_table, in table order, nonzero = trained; NULL = every variable (the default).  A frozen variable gets no gradient
 * (0 in tcr_step_args::grads), its parameters and optimizer slots are left bit for bit as they are, and the step skips the
 * backward work only it needed: its weight gradient, and the backward-data chain below the lowest conv with a trained variable
 * (none at all when only fc / fc2 are trained).  Unchanged: the forward pass, total_loss (weight decay over ALL weights), the
 * BatchNorm moving averages of every layer, and the gradients of the trained variables, which are bit-identical to the full
 * step's.  Host-side planning, not per step: the plans are rewritten in place, so no step of this handle may still be queued on
 * the caller's stream (synchronise it first); the streams the handle owns itself are drained by the call.
 * TCR_ERR_INVALID: count != the number of trainable rows, or no flag set. */
int tcr_set_trainable(tcr_handle* h, const int32_t* flags, int32_t count);

/* The same step fed from PINNED HOST memory (the feed_dict / tf.data side of session.run(train_op): helper/trainer.py:312-321,
 * datasets/data_wrapper_base.py:100-108).  `a->input` and `a->onehot` are host pointers (cudaHostAlloc / pin_memory);
 * `a->losses` is ignored; the optimizer fields (and Adam's powers) and ema / ema_decay are taken as they are in this call.  The batch is copied H2D on a private copy stream into one of 3 staging slots, the step runs on
 * `stream` behind it and its two losses are copied back; the call does not wait for the step it submits.  It returns,
 * in losses_out[0..1] and *losses_step, the losses of the step submitted `lag` calls earlier (*losses_step = -1 while
 * fewer than lag+1 steps are outstanding).  lag in [0,2]: 0 = synchronous, 1 = copy/compute overlap, 2 = also keeps
 * kernel launches ahead of the GPU.  The host buffers of a call may be reused once the call `lag`+1 later has
 * returned (or after tcr_host_flush).  tcr_host_flush returns the oldest outstanding losses, *losses_step = -1 when none. */
int tcr_train_step_host(tcr_handle* h, const tcr_step_args* a, int32_t lag, tcr_stream stream, float* losses_out,
                        int64_t* losses_step);
int tcr_host_flush(tcr_handle* h, float* losses_out, int64_t* losses_step);

/* Debug / parity inspection: device pointer of a named workspace tensor after the last call, e.g.
 * "features", "y:conv0", "y:block0/conv0_0", "out:block1", "g:block0/down", "grads".
 * Returns TCR_ERR_INVALID for unknown names. */
int tcr_workspace_tensor(tcr_handle* h, const char* name, float** ptr, int64_t* numel);

/* Data-parallel plumbing (no reference counterpart: const.py:7 hard-wires one device).  The unique id
 * (128 bytes, ncclUniqueId) is created on rank 0 and distributed by the host (torch.distributed). */
int tcr_comm_unique_id(void* id128);
int tcr_comm_init(tcr_handle* h, const void* id128, int32_t rank, int32_t world_size);
/* Parity-test flag (SURVEY.md 8(e)): BatchNorm batch statistics (forward) and BatchNorm-backward sums over the GLOBAL batch of all
 * ranks = the reference's single-device batch of world * n.  One NCCL all-reduce of 2*C floats per BN layer, forward and backward;
 * the step then runs on the per-layer kernels.  Not a production path: the default is local (per-replica) statistics.  No
 * reference counterpart (single device: const.py:7). */
int tcr_comm_set_sync_bn(tcr_handle* h, int32_t enable);

/* Peer-memory gradient exchange over NVLink / NVSwitch (optional, same node, world_size <= 8): every rank exports two CUDA IPC
 * handles (128 bytes: its double-buffered flat gradient and its arrival flags), the host gathers all ranks' handles (rank-major,
 * world_size x 128 bytes) and every rank attaches them.  From then on the update kernel of tcr_train_step announces its gradient
 * in every peer's flag array, waits for all ranks' flags and sums the ranks' gradients itself (fixed rank order: replicas stay
 * bit-identical) — compute and collective in ONE kernel, no ncclAllReduce launch in the step. */
int tcr_comm_p2p_export(tcr_handle* h, void* handles128);
int tcr_comm_p2p_attach(tcr_handle* h, const void* all_handles, int32_t rank, int32_t world_size);
/* Back to ncclAllReduce (e.g. when some rank could not map a peer): unmaps the peers and frees the exported buffers. */
int tcr_comm_p2p_detach(tcr_handle* h);
int tcr_comm_destroy(tcr_handle* h);

/* Measured fp32 FMA peak of the device the handle lives on (TFLOP/s), used as the compute-roofline
 * denominator by bench.py.  Launches a register-resident FMA loop and times it with CUDA events. */
int tcr_measure_fp32_peak(tcr_handle* h, double* tflops, tcr_stream stream);

/* DS-CNN (Hello-Edge) forward pass, inference mode: the reference's 2-D-conv comparison model
 * (audio_nets/ds_cnn.py:20-118; factory/audio_nets.py DSCNN{S,M,L}Model.build_inference; BASELINE.json config 5).
 * features [n, height, width] (== [N,H,W,1]); params = one flat fp32 buffer laid out by tcr_dscnn_param_table
 * (TF variable names "DSCNN/conv_1/weights", ".../batch_norm/moving_mean", "DSCNN/fc1/biases", ...), the BatchNorm moving
 * statistics included.  size: 'S', 'M' or 'L' (64, 172 and 276 channels; the head takes up to 320).
 *
 * The same handle also runs the two Sainath & Parada CNNs of the reference's KWSModel (audio_nets/kws.py), evaluation mode (ABI 12):
 *   size TCR_KWS_TRAD_FPOOL3 ('P', --architecture trad_fpool3): 20x8 conv 1 -> 64 + ReLU, max-pool 1x3 / stride 1x3, 10x4 conv
 *     64 -> 64 + ReLU (every conv VALID, bias-free), then flatten (NHWC order) and the matmuls linear_weights [K, 32],
 *     first_fc_weights [32, 128], final_fc_weights [128, classes], softmax.  Needs height >= 29 and width >= 19.
 *   size TCR_KWS_ONE_FSTRIDE4 ('F', --architecture one_fstride4): height x 8 conv 1 -> 186, stride 4 in frequency + ReLU, then
 *     first_linear_weights [K, 32], first_fc_weights [32, 128], second_fc_weights [128, 128], final_fc_weights [128, classes].
 *     Needs width >= 8 and height x width <= 51,200 (its conv stages a whole utterance in shared memory).
 * Their variables are top-level TF names ("first_weights", ...), all of kind TCR_KIND_WEIGHT; below the geometry bound create
 * returns TCR_ERR_UNSUPPORTED, naming it.  Every tcr_dscnn_* entry point below serves them unchanged; forward_partial's layers
 * are [conv1 + pool, conv2] for 'P' and [conv] for 'F', each written NHWC ([n, hout, wout, cout], the pooled width for 'P''s
 * first), and, as for DS-CNN, the head is not among them.
 *
 * And two of KWSModel's TensorFlow speech_commands nets (audio_nets/kws.py), evaluation mode (ABI 16); every layer has a bias:
 *   size TCR_KWS_LOW_LATENCY_CONV ('C', --architecture low_latency_conv): height x 8 conv 1 -> 186, VALID, stride 1, + bias, ReLU,
 *     then flatten and first_fc, second_fc, final_fc, each + bias with no nonlinearity, softmax.  With W = width - 7: variables
 *     "first_weights" [height, 8, 1, 186], "first_bias" [186], "first_fc_weights" [W * 186, 128], "first_fc_bias" [128],
 *     "second_fc_weights" [128, 128], "second_fc_bias" [128], "final_fc_weights" [128, classes], "final_fc_bias" [classes].
 *     Needs width >= 8 and max_batch x W <= 2^31 - 1 (the conv's GEMM rows).
 *   size TCR_KWS_TINY_CONV ('Y', --architecture tiny_conv): 10 x 8 conv 1 -> 8, TF SAME at stride 2 x 2, + bias, ReLU, then
 *     flatten and final_fc + bias, softmax.  H = ceil(height / 2), W = ceil(width / 2); SAME pads pad_total = max((out - 1) * 2 + k
 *     - in, 0) zeros, pad_total / 2 (rounded down) before (above / left) and the rest after.  Variables "first_weights" [10, 8, 1, 8],
 *     "first_bias" [8], "final_fc_weights" [H * W * 8, classes], "final_fc_bias" [classes].  Takes any height; needs the conv's
 *     staged rows, 4 * (648 + (2 * min(H, 8) + 8) * (2 W + 6)) bytes, within 227 KB of shared memory (width <= 2,388 from height 15 up).
 *   Both: the flattened conv output K (W * 186, or H * W * 8) must be below 2^31, in at most 2^31 - 1 chunk x batch-group CTAs of
 *   the split dense layer.  Weights have kind TCR_KIND_WEIGHT and biases TCR_KIND_BETA.  forward_flops counts 2 x multiply-adds
 *   of the conv and the matmuls (tiny_conv: the full 80-tap kernel at every output), not the bias adds.  forward_partial's only
 *   layer is the conv, NHWC [n, 1, W, 186] or [n, H, W, 8]; the dense head is not among them.
 *
 * And the paper's 2-D ablations of TC-ResNet8 (audio_nets/tc_resnet.py ResNet2D8 / ResNet2D8Pool), evaluation mode (ABI 13):
 *   size TCR_RES2D8 ('R'): conv0 3x3 1 -> c0 + BN + ReLU, then three residual blocks of c1, c2, c3 channels: conv{i}_0 3x3 at stride
 *     s + BN + ReLU, conv{i}_1 3x3 + BN, plus the shortcut, then ReLU.  Where a block changes the channel count, s = 2 and the
 *     shortcut is down (1x1 / stride 2 + BN + ReLU); else s = 1 and the shortcut is the block's input.  Then the global average
 *     pool, fc (1x1, no bias) and softmax.  Every conv is TF SAME (leading pad = total // 2) and bias-free; BatchNorm has gamma,
 *     eps 1e-3, the moving statistics.
 *   size TCR_RES2D8_POOL ('A'): the same with a 4x4 / stride 4 VALID average pool after conv0.  Needs height >= 4 and width >= 4.
 *   Channels: [c0, c1, c2, c3] = int(x * width_multiplier) of [16, 24, 32, 48], then c0 = int((3 width c1 + 10 c1 c2) /
 *   (9 + 10 c2)); every count must be in [1, 128].
 * Variables as tcr_param_table's TCResNet8 rows under the scope "ResNet2D8" / "ResNet2D8Pool", with 2-D shapes ("ResNet2D8/
 * conv0/weights" [3, 3, 1, c0], ".../block0/down/weights" [1, 1, c0, c1], ".../conv0/BatchNorm/gamma", ..., ".../fc/weights"
 * [1, 1, c3, classes], ".../fc2/weights" [1, 1, c3, 2], then the moving statistics); fc2 is loaded but not computed.
 * forward_partial's layers are [conv0 (+ pool), block0, block1, block2], each NHWC.
 *
 * And Honk's ResNets as the reference builds them (audio_nets/res.py Res8 / Res8Narrow / Res15 / Res15Narrow), evaluation mode
 * (ABI 14).  C channels throughout: 45, or 19 for the Narrow variants.  Every conv is 3x3, stride 1, TF SAME, bias-free and followed
 * by ReLU; BatchNorm has no beta and no gamma (y = (x - mean) / sqrt(var + 1e-3), the moving statistics).
 *   f_conv 1 -> C + ReLU (no BatchNorm); Res8 / Res8Narrow only: a 4x3 average pool at stride 1, VALID, so the blocks run on
 *     (height - 3) x (width - 2); needs height >= 4 and width >= 3.
 *   block i = 0 .. L / 2 - 1 on input x: a = BN_{conv2i_bn}(ReLU(conv{2i}(x))), y = BN_{conv2i+1_bn}(ReLU(conv{2i+1}(a)) + x) (no
 *     ReLU after the add).  Res15 has L = 13 convs, so after its six blocks conv12: BN_{conv12_bn}(ReLU(conv12(y))).  Res8 has L = 6.
 *   Res15 / Res15Narrow dilate: conv{k} has rate 2^(k / 3) (1, 1, 1, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16), SAME pads `rate` zeros on
 *     every side.  Res8 does not dilate.
 *   Then the global average pool, fc (1x1, no bias) and softmax.
 * Variables, all under the scope "Res" (slim's conv2d opens the sub-scope "Conv" inside conv{k}): "Res/f_conv/weights" [3, 3, 1, C],
 * "Res/conv{k}/Conv/weights" [3, 3, C, C] for k = 0 .. L - 1, "Res/fc/weights" [1, 1, C, classes] (kind TCR_KIND_WEIGHT), then per
 * k "Res/conv{k}_bn/moving_mean" and ".../moving_variance" [C].  width_multiplier must be 0.  forward_partial's layers are
 * [f_conv (+ pool), conv0, .., conv{L-1}], each NHWC [n, h, w, C] after its epilogue (after BN for conv{2i} and conv12, after the
 * add and BN for conv{2i+1}): 7 layers for Res8, 14 for Res15. */
#define TCR_KWS_TRAD_FPOOL3 'P'
#define TCR_KWS_ONE_FSTRIDE4 'F'
#define TCR_KWS_LOW_LATENCY_CONV 'C'
#define TCR_KWS_TINY_CONV 'Y'
#define TCR_RES2D8 'R'
#define TCR_RES2D8_POOL 'A'
#define TCR_RES8 'E'
#define TCR_RES8_NARROW 'N'
#define TCR_RES15 'D'
#define TCR_RES15_NARROW 'T'
typedef struct tcr_dscnn tcr_dscnn;
typedef struct tcr_dscnn_config {
  int32_t size;          /* 'S' | 'M' | 'L' | TCR_KWS_TRAD_FPOOL3 | TCR_KWS_ONE_FSTRIDE4 | TCR_KWS_LOW_LATENCY_CONV | TCR_KWS_TINY_CONV |
                            TCR_RES2D8 | TCR_RES2D8_POOL | TCR_RES8 | TCR_RES8_NARROW | TCR_RES15 | TCR_RES15_NARROW */
  int32_t height;        /* frames, 49 */
  int32_t width;         /* coefficients, 40 (10 in the reference's DS-CNN recipes) */
  int32_t num_classes;   /* 12 */
  int32_t max_batch;
  int32_t device;
  double width_multiplier; /* TCR_RES2D8 / TCR_RES2D8_POOL only (0 means 1.0); must be 0 for the other sizes.  ABI 13 */
} tcr_dscnn_config;
int tcr_dscnn_create(const tcr_dscnn_config* cfg, tcr_dscnn** out);
int tcr_dscnn_destroy(tcr_dscnn* d);
int tcr_dscnn_param_table(const tcr_dscnn* d, const tcr_param_desc** descs, int32_t* count, int64_t* num_params,
                          int64_t* forward_flops_per_utt);
int tcr_dscnn_forward(tcr_dscnn* d, const float* features, const float* params, int32_t n, float* logits, float* probs,
                      tcr_stream stream);
/* Layers [0, num_layers) of the same forward pass, with the same kernels: the NHWC output [n, hout, wout, cout] of layer
 * num_layers - 1 is written to act_out and nothing else is (for checking one layer at a time against a reference). */
int tcr_dscnn_forward_partial(tcr_dscnn* d, const float* features, const float* params, int32_t n, int32_t num_layers,
                              float* act_out, tcr_stream stream);
/* Evaluation from audio on a DS-CNN handle (ABI 11), the evaluation graph of evaluate_audio.py with a DSCNN{S,M,L}Model
 * (helper/base.py:52-125):
 * tcr_dscnn_set_frontend   gives the handle the front-end of a tcr_config (datasets/preprocessors.py:64-96, 183-194): only the
 *                          front-end fields are read (sample_rate, clip_samples, window / stride, num_mel_bins, num_mfccs, edges,
 *                          feature_kind), with tcr_create's refusals; TCR_ERR_INVALID, naming both shapes, when its (T, F) is not
 *                          the handle's (height, width).  Sizes a feature buffer for max_batch.  The tables are the ones tcr_create
 *                          builds, and the same kernel runs, so the features equal tcr_mfcc_forward's bit for bit.  Calling it
 *                          again replaces the front-end (the call synchronises the device).
 * tcr_dscnn_mfcc_forward   front-end only: wav [n, clip_samples] (TCR_INPUT_WAV_F32 or TCR_INPUT_WAV_PCM16, 16-byte aligned)
 *                          -> features [n, height, width].
 * tcr_dscnn_forward_input  the forward from TCR_INPUT_FEATURES (== tcr_dscnn_forward), TCR_INPUT_WAV_F32 or TCR_INPUT_WAV_PCM16: the
 *                          front-end into the handle's feature buffer, then the same forward, so the result equals
 *                          tcr_dscnn_forward on tcr_dscnn_mfcc_forward's features bit for bit.
 * tcr_dscnn_eval_accumulate  tcr_eval_accumulate's counts (same kernel, same layout) for num_classes of the DS-CNN handle.
 * tcr_dscnn_eval_collect / tcr_dscnn_eval_rank  tcr_eval_collect / tcr_eval_rank (same kernels, same store, workspace and result
 *                          layout, same softmax convention) for num_classes of the DS-CNN handle (ABI 15).
 * tcr_dscnn_listener_create  a tcr_listener (see above) on the DS-CNN handle and its front-end; tcr_listener_reset / _push / _history
 *                          / _destroy are shared, with the same four promises (tcr_dscnn_forward in place of tcr_forward).  Its
 *                          pushes pass moving = NULL.  TCR_ERR_INVALID without a front-end. */
int tcr_dscnn_set_frontend(tcr_dscnn* d, const tcr_config* frontend);
int tcr_dscnn_mfcc_forward(tcr_dscnn* d, const void* wav, int32_t input_kind, float* features, int32_t n, tcr_stream stream);
int tcr_dscnn_forward_input(tcr_dscnn* d, const void* input, int32_t input_kind, const float* params, int32_t n, float* logits,
                            float* probs, tcr_stream stream);
int tcr_dscnn_eval_accumulate(tcr_dscnn* d, const float* scores, const float* onehot, int32_t n, int32_t topk, int64_t* counts,
                              tcr_stream stream);
int tcr_dscnn_eval_collect(tcr_dscnn* d, const float* scores, const float* onehot, int32_t n, int32_t row_offset, int32_t capacity,
                           float* store_scores, int32_t* store_labels, tcr_stream stream);
int tcr_dscnn_eval_rank(tcr_dscnn* d, const float* store_scores, const int32_t* store_labels, int32_t n, void* workspace,
                        int64_t* workspace_bytes, double* result, tcr_stream stream);
int tcr_dscnn_listener_create(tcr_dscnn* d, const tcr_listener_config* cfg, tcr_listener** out);

/* Process-wide launch accounting (no reference counterpart; the reference only logs wall-clock per
 * session.run, helper/trainer.py:312-321).  tcr_launch_count: kernels launched by this library so far.
 * tcr_profile_enable(1) brackets every subsequent launch with CUDA events on its stream (adds overhead:
 * use a separate pass, not the timed region); tcr_profile_read synchronises and returns one row per
 * kernel name ("mfcc", "fwd:block0/conv0_0", "dx:...", "dw:...", "head", "grad_finalize", "update"). */
typedef struct tcr_kernel_stat {
  char    name[64];
  double  total_ms;
  int64_t launches;
} tcr_kernel_stat;
int tcr_profile_enable(int enable);
int tcr_profile_read(const tcr_kernel_stat** stats, int32_t* count);
int tcr_launch_count(uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif  /* TCR_B200_H_ */
