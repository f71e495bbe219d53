// tcr_net.h — host-side launch sequences implemented in tcr_net_fwd.cu / tcr_net_bwd.cu /
// tcr_optim.cu / tcr_comm.cu.  All return 0 or a TCR_ERR_* code (message via tcr::set_error).
#pragma once
#include "tcr_plan.h"

namespace tcr {

void set_error(const char* msg);

int net_alloc_workspace(tcr_handle* h);

// Front-end (tcr_api.cu), the same for every handle type that owns a Frontend: the refusals of a configuration's front-end
// fields, its (T, F), building and freeing the tables, the arguments for `wav` -> `feat` (per-clip geometry), and the launch of
// the kernel the front-end selects for them (the frame-pair kernel where the shape allows and TCR_MFCC_PAIR does not turn it off).
int frontend_check(const tcr_config* cfg);
void frontend_geometry(const tcr_config& cfg, int* frames, int* features);
int frontend_init(Frontend* fe, const tcr_config* cfg, int sms);
void frontend_free(Frontend* fe);
MfccArgs mfcc_args(const Frontend& fe, const void* wav, int pcm16, float* feat);
int mfcc_select_launch(const Frontend& fe, const MfccArgs& a, int n, cudaStream_t stream);
// wav (16-byte aligned; int16 needs window, stride and clip lengths that are multiples of 8) -> features [n, T, F]
int frontend_run(const Frontend& fe, const void* wav, int pcm16, float* features, int n, cudaStream_t stream);

// The first layer reading its utterances as windows of a listener's feature history (tcr_listener.cu) instead of a [n, T, F]
// tensor: utterance u starts at feat + (u / k) * stream + (u % k) * step floats (TC-ResNet conv0, DS-CNN conv_1).
struct WindowView {
  int k;
  int64_t stream, step;
};

// DS-CNN (tcr_dscnn.cu) as the listener sees it: its front-end (nullptr before tcr_dscnn_set_frontend), max_batch, and the
// evaluation forward on features [n, height, width] or on the windows `win` describes.
const Frontend* dscnn_frontend(const tcr_dscnn* d);
int dscnn_max_batch(const tcr_dscnn* d);
int dscnn_forward(tcr_dscnn* d, const float* feat, const float* params, int n, float* logits, float* probs, cudaStream_t s,
                  const WindowView* win);

// Forward pass on features [n, T, F] (or the windows `win` describes).  training: batch-statistics BN (+ dropout); otherwise
// the BN tables are built from `moving`.  backward: the head additionally emits dlogits-derived tensors for the backward pass.
int net_forward(tcr_handle* h, const float* feat, const float* params, const float* moving, int n, bool training,
                uint64_t seed, const float* mask, const float* onehot, float weight_decay, float* logits,
                float* probs, float* losses, bool backward, cudaStream_t s, const WindowView* win = nullptr);

int cluster_size(tcr_handle* h);
StatSrc stat_src(const tcr_handle* h, const ConvPlan& cv, const float* params, int n);
int augment_launch(const int16_t* pcm, int64_t pcm_stride, const tcr_augment_clip* clips, const float* background, int64_t background_samples,
                   float* out, int clip, int n, cudaStream_t s);
// Rows [position, position + n) of a resident dataset's order: gather + draws + augment into out [n][clip], labels into onehot
int dataset_batch_launch(const tcr_dataset& ds, int64_t position, int64_t epoch, uint64_t seed, float* out, float* onehot, int clip,
                         int classes, int n, cudaStream_t s);
int eval_accumulate_launch(const float* scores, const float* onehot, int n, int classes, int topk, int64_t* counts, cudaStream_t s);
// Ranking metrics (tcr_metrics.cu): append a batch to the score store at row_offset; the refusal of a ranking over n rows (nullptr
// when accepted); its workspace bytes; the ranking pass writing result [2 * classes + 4] (layout in include/tcr_b200.h).
int eval_collect_launch(const float* scores, const float* onehot, int n, int classes, int64_t row_offset, float* store_scores,
                        int32_t* store_labels, cudaStream_t s);
const char* eval_rank_refusal(int64_t n, int classes);
int64_t eval_rank_workspace_bytes(int n, int classes);
int eval_rank_launch(const float* store_scores, const int32_t* store_labels, int n, int classes, void* workspace, double* result,
                     cudaStream_t s);
int net_weight_transpose(tcr_handle* h, const float* params, cudaStream_t s);
int sync_records(tcr_handle* h, const float* part, int gc, int cols, float* out, cudaStream_t s);   // SyncBN: sum records, all-reduce
inline bool sync_bn_on(const tcr_handle* h) { return h->sync_bn && h->world > 1 && h->comm; }
inline float bn_inv(const tcr_handle* h, int n, int t) { return 1.0f / ((float)n * (float)t * (sync_bn_on(h) ? (float)h->world : 1.0f)); }
// Resident kernels (tcr_resident.cu): the training forward + head, and the backward-data chain, each as one cooperative kernel with
// SM-resident activations.  ResidentMode says which of them a handle runs; the values are the TCR_RESIDENT settings that force
// them.  The weight gradients always come from the grouped launch (net_weight_gradients).
enum ResidentMode { kResidentOff = 0, kResidentFwd = 1, kResidentFwdBwdData = 3 };
int resident_mode(tcr_handle* h);
int resident_forward(tcr_handle* h, const float* feat, const tcr_step_args* a, cudaStream_t s);
int resident_backward_data(tcr_handle* h, const float* feat, const tcr_step_args* a, cudaStream_t s);
void resident_destroy(tcr_handle* h);
// Backward-data chain as per-layer kernels: every layer's masked gradient and BatchNorm-backward sums, as resident_backward_data.
int net_backward_data(tcr_handle* h, const float* params, int n, cudaStream_t s);
// Every layer's weight gradient in one grouped launch, from the layer gradients either backward-data chain leaves.
int net_weight_gradients(tcr_handle* h, const float* feat, int n, cudaStream_t s);

// Gradient finalisation (+ weight decay), optional NCCL all-reduce, optimizer update, BN moving averages, losses.
int net_update(tcr_handle* h, const tcr_step_args* a, cudaStream_t s);

// Host-side plans that follow the trainable set (tcr_set_trainable, h->train_rows): optimizer segments (tcr_optim.cu), the
// grouped weight-gradient table and the depth of the backward-data chain (tcr_net_bwd.cu).
int build_opt_segments(tcr_handle* h);
int build_dw_table(tcr_handle* h);
int plan_bwd_phases(const tcr_handle* h);
inline int build_trainable_plans(tcr_handle* h) {
  int frozen = 0;
  for (int f : h->train_rows) frozen += f ? 0 : 1;
  h->frozen_rows = frozen;
  h->bwd_phases = plan_bwd_phases(h);
  const int rc = build_dw_table(h);
  return rc ? rc : build_opt_segments(h);
}

int launch_loss_only(tcr_handle* h, const float* params, float weight_decay, int n, float* losses, cudaStream_t s);
int head_groups(int n);


int measure_fp32_peak(tcr_handle* h, double* tflops, cudaStream_t s);

// NCCL through dlopen (tcr_comm.cu): no link-time dependency, the torch-bundled libnccl is reused when loaded.
int comm_unique_id(void* id128);
int comm_init(tcr_handle* h, const void* id128, int rank, int world);
void comm_destroy(tcr_handle* h);
int comm_allreduce_sum(tcr_handle* h, float* buf, int64_t count, cudaStream_t s);
int comm_p2p_export(tcr_handle* h, void* handles128);
int comm_p2p_attach(tcr_handle* h, const void* all_handles, int rank, int world);
void comm_p2p_destroy(tcr_handle* h);
const char* comm_error();

}  // namespace tcr
