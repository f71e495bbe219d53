// tcr_internal.h — layer plan, workspace layout and kernel argument blocks (host + device).
//
// Data layout in HBM (all fp32, row-major, channel fastest == the reference's NHWC [N,T,1,C]):
//   features  [N, T, F]                      written by the MFCC kernel, read by conv0 fwd + conv0 dW
//   y_L       [N, T'_L, C_L]  per conv layer  PRE-BatchNorm conv output (saved for backward)
//   out_i     [N, T'_i, C_i]  per block       relu(bn(y_b) + shortcut), materialised by its first consumer
//   g_L       [N, T'_L, C_L]                  dLoss/d(BN output) after the ReLU mask (backward)
//   bnf_L     [4][C_L]                        finalised BN table: mean, rstd, scale=gamma*rstd, beta
//   fpart/bpart [records][C][2]               partial BatchNorm sums, one record per 8-CTA cluster (tcr_bn.cuh)
//   dwpart_L  [R][k*C_in*C_out]               per-row-chunk partial weight gradients
// Activations are never stored post-BN/ReLU: consumers re-apply the per-channel table on load.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/tcr_b200.h"

namespace tcr {

constexpr int kMaxConvs = 24;
constexpr int kMaxBlocks = 8;
constexpr int kThreads = 256;        // conv fwd / bwd-data CTAs
constexpr int kOptThreads = 256;     // grad_finalize / update CTAs: one w^2 partial sum per grad_finalize CTA
constexpr int kMaxClasses = 32;

// Forward statistics of a layer as its producer kernel left them (tcr_bn.cuh): per-cluster records that the consumer
// sums, or nothing (cpart == nullptr) when the global table is already final.
struct StatSrc {
  const float* cpart;       // [gc][C][2] (sum y, sum y^2)
  int gc;
  const float* gamma; const float* beta;
  float* bnf; float* var;   // published by CTA 0 of the consumer
  float inv_m, eps;
};
struct BsumSrc {            // same for the BatchNorm-backward sums (sum dz, sum dz*xhat)
  const float* cpart;       // [gc][C][2]
  int gc;
  float* bsum;              // [2][C], published by CTA 0 of the consumer
};

// Source of an activation tile: kind 0 = raw tensor, 1 = relu(bn(y)) with table bnf.
struct ActSrc {
  const float* data;
  const float* bnf;   // [4][C]: mean, rstd, scale, beta
  int kind;
  StatSrc st;
};

// ---------------- forward conv kernel (main conv + optional 1x1/stride-2 "down" conv) ----------------
struct FwdArgs {
  // input tile
  int in_kind;              // 0 raw, 1 relu(bn(y)), 2 residual: relu(bn(yb) + shortcut) (also materialises out)
  ActSrc in;                // kind 0/1: the tensor; kind 2: conv_b output (in.kind ignored, bn applied, no relu)
  ActSrc shortcut;          // kind 2 only: raw prev activation / relu(bn(y_down))
  float* out_write;         // kind 2 only: materialised block output [N, t_in, cin]
  int n, U, t_in, cin;
  // main conv
  const float* w; float* y; float* fpart;
  int cout, stride, t_out, pad_left, KS;
  int w_smem;               // 1: filter bank(s) staged in shared memory by one TMA bulk copy
  long long* tl;            // debug timeline (nullptr in production)
  // optional down conv (k=1, stride 2, no padding, same t_out)
  const float* wd; float* yd; float* fpartd; int coutd;
  // training statistics
  int train;
  float eps;
  // windowed input (conv_fwd_kernel<K, WSMEM, true>, in_kind 0 only): utterance u is read at in.data + (u / win_k) * win_stream
  // + (u % win_k) * win_step floats, its T rows of cin floats back to back (a listener's feature history, tcr_listener.cu)
  int win_k;
  int64_t win_stream, win_step;
};

// ---------------- head: residual + pool + dropout + fc + softmax + CE (+ head backward) ----------------
struct HeadArgs {
  ActSrc in;                // conv_b of the last block (bn applied, no relu)
  ActSrc shortcut;          // raw / relu(bn(y_down))
  float* out_write;         // [N, T', C]
  int n, t, c, classes;
  const float* wfc;         // [C, classes]
  const float* onehot;      // may be null (no loss, no backward)
  const float* mask;        // injected dropout mask or null
  uint64_t seed; float keep; int use_dropout; float label_smoothing;
  float* logits; float* probs;   // may be null
  float* loss_part;         // [clusters] sum of per-utterance CE per cluster record
  int backward;             // 1: also produce gblk, BN-backward partial sums and fc dW partials
  float inv_n;              // 1 / n (mean over the local batch)
  float* gout;              // gblk_last [N, T', C]
  // BN-backward sums for conv_b(last) and down(last)
  const float* yb; const float* bnfb; float* bpartb;
  const float* ydn; const float* bnfd; float* bpartd;   // null when the last block has no down conv
  float* dwfc_part;         // [Gh][C*classes]
};

// ---------------- backward-data kernel ----------------
struct DySrc {              // dy = scale * (dz - s1/M - xhat * s2/M), dz optionally masked by (bn(y) > 0)
  const float* dz;          // g tensor
  const float* y;           // pre-BN conv output of this layer
  const float* bnf;         // [4][C]
  const float* bsum;        // [2][C]
  int mask_relu;            // 1: dz *= (bn(y) > 0)   (down conv: its own ReLU is applied here)
  float inv_m;              // 1 / (N * T')
  BsumSrc bs;               // where the sums come from when the producer kernel has just written them
};

struct BwdDataArgs {
  int n, U;
  int w_smem;               // 1: filter bank(s) staged in shared memory by one TMA bulk copy
  // conv whose input gradient we compute
  DySrc dy; const float* w; int cin, cout, k, stride, t_in, t_out, pad_left, KS;
  // optional down conv sharing the same input (k=1, stride 2)
  int has_down; DySrc dyd; const float* wd; int coutd;
  // optional identity shortcut: dx += gid
  const float* gid;
  // epilogue: mask + write g_prev, BN-backward partial sums of the producer layer(s)
  int epi_kind;             // 1: single BN layer (mask bn(yp) > 0); 2: block output (mask out_prev > 0)
  const float* yp; const float* bnfp; float* bpartp;            // kind 1: producer; kind 2: conv_b of prev block
  const float* out_prev;                                        // kind 2
  const float* ypd; const float* bnfpd; float* bpartpd;         // kind 2: down conv of prev block (may be null)
  float* gprev;             // [N, t_in, cin]
};

// ---------------- backward-weight kernel ----------------
struct BwdWeightArgs {
  int n;
  ActSrc x;                 // conv input activation (raw or relu(bn(y)))
  DySrc dy;
  int cin, cout, k, stride, t_in, t_out, pad_left;
  int cot;                  // output-channel tile handled per CTA (multiple of 4, divides cout)
  int RG;                   // row groups inside the CTA
  int R;                    // row chunks (gridDim.y)
  int UB;                   // utterances staged in shared memory at a time
  float* dwpart;            // [R][k*cin*cout]
};

constexpr int kDwThreads = 256;
struct DwLayer {            // one row per conv layer of the grouped weight-gradient launch (static per handle)
  const float* x_data;      // conv input activation; nullptr = the features pointer passed per call
  const float* x_bnf; int x_kind;
  const float* dz; const float* y; const float* bnf; const float* bsum; int mask_relu;
  int cin, cout, k, stride, t_in, t_out, pad_left;
  int cot, RG, R, UB;
  float* dwpart;
  int cta_begin;            // first virtual CTA of this layer
};

// ---------------- optimizer ----------------
struct OptSegment {         // one trainable variable
  int64_t offset, numel;
  const float* part;        // partial sums [R][numel] (weights) or bsum row (gamma/beta), may be null (fc2)
  int R;                    // number of partials to add
  int decay;                // 1: add weight_decay * w
  int train;                // 0: frozen (tcr_set_trainable): gradient 0, no update; still in sum(w^2) when decay
};
struct MovingSegment {      // one BN layer
  int64_t mm_off, mv_off; int c;
  const float* bnf;         // mean at [0][c]
  const float* var;         // biased variance
  int t_out;                // rows per utterance: M = n * t_out, unbiased variance = var * M / (M - 1)
};

struct GradArgs {           // gradient finalisation (sum of partials + weight decay -> flat gradient)
  const OptSegment* segs; int nsegs; int64_t total; int fc_seg; const float* fc_part; int fc_R;
  const float* params; float weight_decay; float* grads; float* l2part;
  float bn_grad_scale;      // 1, or 1/world with SyncBN: every rank then holds the GLOBAL sums for the gamma / beta gradients
};
struct WtLayer { int64_t w_off; float* wT; int k, cin, cout; int64_t begin; };
struct WtArgs { WtLayer layer[kMaxConvs]; int nlayers; int64_t total; const float* params; };

struct Hyper {              // device-resident hyper-parameters (graph replays read fresh values)
  float lr, momentum, weight_decay, one_minus_decay;
  float grad_scale;         // 1 / world_size
  uint64_t seed;
};

}  // namespace tcr

// Row stride (floats) of an activation tile in shared memory: (stride/4) odd keeps 8 lanes reading
// float4s from 8 different rows on 8 distinct bank groups.
#if defined(__CUDACC__)
#define TCR_HD __host__ __device__
#else
#define TCR_HD
#endif
namespace tcr {
TCR_HD inline int chan_stride(int c) { return ((c >> 2) & 1) ? c : c + 4; }
TCR_HD inline int imin(int a, int b) { return a < b ? a : b; }
TCR_HD inline int imax(int a, int b) { return a > b ? a : b; }
}  // namespace tcr
