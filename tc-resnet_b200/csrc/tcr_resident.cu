// tcr_resident.cu — the training step's network part as TWO cooperative kernels whose activations never leave the SM between
// layers: resident_fwd_kernel (all conv layers + head) and resident_bwd_kernel (the backward-data chain).  The weight gradients
// are not computed here: the grouped launch (dw_grouped, two CTAs per SM) reads the layer gradients the backward kernel stores.
//
// Why: BatchNorm's batch statistics force a grid-wide dependency after every conv layer, forward and backward
// (audio_nets/tc_resnet.py:21-41 under TCResNet_arg_scope :102-123; FusedBatchNormGrad in the gradient graph of
// helper/trainer.py:199-211).  As separate launches each layer paid a kernel boundary (~4.5 us), re-staged its tiles from L2 and
// re-fetched its code: 14 conv launches + head, each far longer than its math, stalled on instruction fetch and barriers.  Here:
//   * one CTA of 512 threads per SM owns ceil(n / #SMs) whole utterances for the whole pass; a layer's output stays in shared
//     memory and becomes the next layer's input tile by one smem -> smem pass (BatchNorm + ReLU (+ residual) applied there);
//   * batch statistics travel as per-CTA records through L2 behind a split grid barrier: a CTA arrives as soon as its record is
//     written, then does the work nobody waits for (store the pre-BN output or the layer gradient, prefetch of the next filter
//     bank by TMA and of the next tensors by cp.async) and only then waits;
//   * every CTA sums the records itself (float4 loads, all in flight at once, fixed order: bit-reproducible), CTA 0 publishes;
//   * the phase bodies are non-inlined functions shared by all layers, so their code is fetched once and stays in the I-cache.
// The forward kernel leaves exactly what the multi-kernel forward leaves (plus the transposed filter banks of the backward pass) and
// the backward kernel what the backward-data launches of net_backward_data leave, so either can be paired with the per-layer kernels.
// TCR_RESIDENT = 0: per-layer kernels | 1: resident forward, per-layer backward-data | unset or anything else: both resident
// kernels (resident_state falls back to 1 or 0 where a shape does not fit).
#include <stdio.h>
#include <stdlib.h>

#include "tcr_layer.cuh"
#include "tcr_net.h"

namespace tcr {

constexpr int kResThreads = 512;
constexpr int kResMaxU = 8;          // utterances per CTA the head's scratch is sized for
static_assert(kResMaxU * 1 >= 5, "res_head keeps its [4C + 1] sums in the [kResMaxU][C] dnet region");
constexpr int TMR = 4;               // input rows per thread task of the transposed conv

struct RConv {
  int cin, cout, k, stride, t_in, t_out, pad_left, pad_right;
  long long w_off, gamma_off, beta_off;
  float* y; float* bnf; float* var; float* bsum;
  float* g;                                        // gradient after this layer's ReLU mask (what the grouped weight-gradient launch reads)
  float* frec; float* brec;                        // [G][2*cout] per-CTA records: (sum y, sum y^2) / (sum dz, sum dz*xhat)
  const float* wT;                                 // transposed bank [k][cout][cin]
  int tm, ks;                                      // forward tiling: rows per thread task, k-slices
  int bks;                                         // backward-data k-slices
  int tbl, bs;                                     // float offsets of the [4][cout] table / [2][cout] sums in their smem regions
};
struct RBlock { int a, b, down, c, t; float* out; float* gblk; };

struct ResProgram {                  // static per handle
  int nconvs, nblocks, classes, umax;
  RConv conv[kMaxConvs];
  RBlock blk[kMaxBlocks];
  float eps;
  unsigned* bar;                     // monotonic arrival counter
  // forward layout (float offsets from the dynamic shared memory base)
  int o_w, o_buf0, o_buf1, o_yo, o_sh, o_tbl, o_red, o_head;
  // backward layout
  int b_w, b_ys, b_yp, b_dys, b_dyd, b_pl, b_g[3], b_tbl, b_bs, b_red;
  int b_ys_cap;                      // floats of the b_ys region: it doubles as the backward epilogue's reduction scratch
  // head
  long long fc_off;
  float* loss_part; float* dwfc_part; float* gout; float* bpartb; float* bpartd;
};

struct ResCall {                     // per call
  const float* feat; const float* params; const float* onehot; const float* mask;
  unsigned long long seed; float keep; int use_dropout; float label_smoothing;
  float* logits; float* probs;
  int n; unsigned bar_base; float inv_n;
  long long* tl;                     // debug timeline (TCR_DEBUG_TIMELINE=1): [cta][32] globaltimer stamps, else null
  int phases;                        // backward kernel: phases to run from the last block down (tcr_handle::bwd_phases, >= 1)
};

__device__ __forceinline__ void res_stamp(const ResCall& c, int slot) {
#ifndef TCR_EMU
  if (c.tl && threadIdx.x == 0 && slot < 32) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    c.tl[(size_t)blockIdx.x * 32 + slot] = (long long)t;
  }
#endif
}

// ---- split grid barrier: all CTAs are co-resident (cooperative launch) ----
__device__ __forceinline__ void gbar_arrive(unsigned* ctr) {
#ifndef TCR_EMU
  __syncthreads();                   // every thread's global writes of this phase are issued (CTA-scope order) ...
  if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");   // ... and released at gpu scope
#endif
}
__device__ __forceinline__ void gbar_wait(unsigned* ctr, unsigned target) {
#ifndef TCR_EMU
  if (threadIdx.x == 0) {
    unsigned v;
    for (;;) {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
      if ((int)(v - target) >= 0) break;
    }
  }
  __syncthreads();
#else
  (void)ctr; (void)target;
  emu::gridsync();
#endif
}

// ---- cp.async (LDGSTS): global -> shared without registers; the copies of a thread complete at cp_async_wait_all() ----
__device__ __forceinline__ void cp_async16(float* dst_smem, const float* src) {
#ifndef TCR_EMU
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
#else
  st4(dst_smem, ld4(src));
#endif
}
__device__ __forceinline__ void cp_async_wait_all() {
#ifndef TCR_EMU
  asm volatile("cp.async.wait_all;" ::: "memory");
#endif
}
// n4 float4s from global to shared, asynchronously (every thread issues its share)
__device__ __forceinline__ void res_fetch(float* dst, const float* src, int n4) {
  for (int i = threadIdx.x; i < n4; i += kResThreads) cp_async16(dst + 4 * i, src + 4 * (size_t)i);
}
__device__ __forceinline__ void res_store(float* dst_global, const float* src_smem, int n4) {
  for (int i = threadIdx.x; i < n4; i += kResThreads) st4(dst_global + 4 * (size_t)i, ld4(src_smem + 4 * i));
}

// One TMA bulk copy of up to two filter banks into the weight region; completion on `bar`.
__device__ __forceinline__ void res_load_bank(float* dst, const float* w, unsigned wn, const float* wd, unsigned wdn, uint64_t* bar) {
  if (threadIdx.x == 0) {
    fence_proxy_async();             // earlier generic-proxy accesses of the region are ordered before the async write
    mbar_expect_tx(bar, (wn + wdn) * 4u);
    tma_load_1d(dst, w, wn * 4u, bar);
    if (wdn) tma_load_1d(dst + wn, wd, wdn * 4u, bar);
  }
}

// ------------------------------------------------------------------------------------------------
// Per-CTA records -> per-channel sums.  Up to two record arrays (recA [G][colsA], recB [G][colsB], cols multiples of 4) are
// summed together: thread (q, ch) adds the float4 column q of records ch, ch + nch, ...; all loads of a thread are in flight
// at once.  Chunk sums land in scratch[ch][colsA + colsB]; returns nch.  Ends with __syncthreads().
// ------------------------------------------------------------------------------------------------
__device__ __noinline__ int res_rec_sum(const float* recA, int colsA, const float* recB, int colsB, int G, float* scratch) {
  const int QA = colsA >> 2, Q = (colsA + colsB) >> 2;
  const int nch = imax(1, imin(imin(kResThreads / Q, 8), G));   // few chunks: the fp64 chunk sums of the callers stay short chains
  const int t = threadIdx.x;
  if (t < Q * nch) {
    const int q = t % Q, ch = t / Q;
    const float* base = q < QA ? recA + 4 * q : recB + 4 * (q - QA);
    // 148 records / 8 chunks = 19 loads: one batch, one L2 round trip
    st4(scratch + (size_t)ch * 4 * Q + 4 * q, rec_column_sum<float4, 20>(base, 0, q < QA ? colsA : colsB, ch, nch, G));
  }
  __syncthreads();
  return nch;
}

// BN tables (mean, rstd, gamma*rstd, beta) of one or two layers from their records (pairs c*2+{0,1} = sum y, sum y^2).
struct TblDst { float* tbl; const float* gamma; const float* beta; float* bnf; float* var; int C; float inv_m; };
__device__ __noinline__ void res_tables(const float* recA, const TblDst& A, const float* recB, const TblDst& B, int nlayers, int G,
                                        float eps, float* scratch, bool publish) {
  const int colsA = 2 * A.C, colsB = nlayers > 1 ? 2 * B.C : 0;
  const int nch = res_rec_sum(recA, colsA, recB, colsB, G, scratch);
  const int cols = colsA + colsB;
  for (int j = threadIdx.x; j < A.C + (nlayers > 1 ? B.C : 0); j += kResThreads) {
    const bool second = j >= A.C;
    const TblDst& D = second ? B : A;
    const int c = second ? j - A.C : j, C = D.C;
    bn_channel_finalize(scratch, cols, (second ? colsA : 0) + 2 * c, nch, D.inv_m, eps, D.gamma[c], D.beta[c], C, c, D.tbl, D.bnf, D.var,
                        publish);
  }
  __syncthreads();
}

// BatchNorm-backward sums [2][C] (sum dz, sum dz*xhat) of one or two layers from their records (pairs c*2+q).
struct BsDst { float* sb; float* bsum; int C; };
__device__ __noinline__ void res_bsums(const float* recA, const BsDst& A, const float* recB, const BsDst& B, int nlayers, int G,
                                       float* scratch, bool publish) {
  const int colsA = 2 * A.C, colsB = nlayers > 1 ? 2 * B.C : 0;
  const int nch = res_rec_sum(recA, colsA, recB, colsB, G, scratch);
  const int cols = colsA + colsB;
  for (int i = threadIdx.x; i < cols; i += kResThreads) {
    const bool second = i >= colsA;
    const BsDst& D = second ? B : A;
    bsum_finalize(scratch, cols, i, nch, second ? i - colsA : i, D.C, D.sb, D.bsum, publish);
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// forward conv (+ optional 1x1/stride-2 shortcut conv) from the padded tile x [U][TP][CS], bank in shared memory.
// Output: ys [KS][rcap][cout] k-slice planes, shortcut output ysd [rows][coutd] (compact).
// ------------------------------------------------------------------------------------------------
template <int K, int TM>
__device__ __noinline__ void res_conv(float* smem, int xs_off, int ws_off, int ys_off, int ysd_off, int rcap, int Ue,
                                      int cin, int cout, int coutd, int stride, int t_out, int TP, int CS, int pad_left, int KS) {
  conv_fwd_tasks<K, TM, kResThreads>(smem, WShared{smem, ws_off, ws_off + K * cin * cout}, xs_off, smem + ys_off, smem + ysd_off, rcap,
                                     Ue * t_out, cin, cout, coutd, stride, t_out, TP, CS, pad_left, KS);
}

// One pass: sum the k-slice planes into plane 0 (fixed order) and form this CTA's per-channel (sum y, sum y^2) record.
// Thread (seg, c) walks rows seg, seg + ns, ...; needs C <= blockDim / 2.  red: 2 * blockDim floats.
__device__ __noinline__ void res_reduce_stats(float* ys, int rcap, int KS, int R, int C, float* red, float* rec) {
  const int tid = threadIdx.x;
  const int ns = kResThreads / C;
  const int seg = tid / C, c = tid - seg * C;
  if (seg < ns) {
    float s1 = 0.f, s2 = 0.f;
    for (int r = seg; r < R; r += ns) {
      float v = ys[r * C + c];
      for (int ks = 1; ks < KS; ++ks) v += ys[(size_t)ks * rcap * C + r * C + c];
      if (KS > 1) ys[r * C + c] = v;
      s1 += v;
      s2 = fmaf(v, v, s2);
    }
    red[seg * C + c] = s1;
    red[kResThreads + seg * C + c] = s2;
  }
  __syncthreads();
  if (tid < 2 * C) {
    const int q = tid & 1, cc = tid >> 1;
    float tot = 0.f;
    for (int k = 0; k < ns; ++k) tot += red[q * kResThreads + k * C + cc];
    rec[tid] = tot;                  // record layout: c*2 + q
  }
  __syncthreads();                   // red may be reused
}

// dst padded tile [U][TP][CS] <- relu(bn(src [rows][C])) (tbl != null) or the raw rows (global features); pad rows zeroed.
__device__ __noinline__ void res_stage(const float* src, const float* tbl, float* dst, int Ue, int t, int C, int TP, int CS,
                                       int pad_left, int pad_right) {
  const int c4n = C >> 2;
  zero_pad_rows(dst, Ue, t, c4n, TP, CS, pad_left, pad_left + pad_right, kResThreads);
  // c4 fixed per thread (table entries in registers), rows advance by rstep: no division per element
  const RowWalk w = row_walk(threadIdx.x, kResThreads, c4n);
  const int rows = Ue * t;
  if (w.row < rows) {
    Chan4 k;
    k.mean = k.rstd = k.scale = k.beta = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tbl) k = chan4_load_s(tbl, C, 4 * w.c4);
    int u = w.row / t, tt = w.row - u * t;
    for (int row = w.row; row < rows; row += w.rstep) {
      float4 v = ld4(src + (size_t)row * C + 4 * w.c4);
      if (tbl) v = relu4(chan4_bn(k, v));
      st4(dst + ((size_t)(u * TP + pad_left + tt) * CS + 4 * w.c4), v);
      tt += w.rstep;
      while (tt >= t) { tt -= t; ++u; }
    }
  }
}

// Block output out = relu(bn_b(yb) + shortcut) -> dst (padded for the next conv, or compact for the head) and to global.
//   shortcut = relu(bn_d(yd)) with yd raw in `sh` (compact), or the block input itself read from its padded tile `xin`.
__device__ __noinline__ void res_block_out(const float* yb, const float* tb, const float* sh, const float* td, const float* xin,
                                           int TPx, int CSx, int plx, float* dst, int Ue, int t, int C, int TP, int CS,
                                           int pad_left, int pad_right, float* ogl) {
  const int c4n = C >> 2;
  zero_pad_rows(dst, Ue, t, c4n, TP, CS, pad_left, pad_left + pad_right, kResThreads);
  const RowWalk w = row_walk(threadIdx.x, kResThreads, c4n);
  const int rows = Ue * t;
  if (w.row < rows) {
    const Chan4 kb = chan4_load_s(tb, C, 4 * w.c4);
    Chan4 kd = kb;
    if (sh) kd = chan4_load_s(td, C, 4 * w.c4);
    int u = w.row / t, tt = w.row - u * t;
    for (int row = w.row; row < rows; row += w.rstep) {
      float4 s;
      if (sh) s = relu4(chan4_bn(kd, ld4(sh + (size_t)row * C + 4 * w.c4)));
      else s = ld4(xin + ((size_t)(u * TPx + plx + tt) * CSx + 4 * w.c4));
      const float4 o = relu4(add4(chan4_bn(kb, ld4(yb + (size_t)row * C + 4 * w.c4)), s));
      st4(dst + ((size_t)(u * TP + pad_left + tt) * CS + 4 * w.c4), o);
      if (ogl) st4(ogl + (size_t)row * C + 4 * w.c4, o);
      tt += w.rstep;
      while (tt >= t) { tt -= t; ++u; }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// head on the CTA's utterances (head_tail, tcr_layer.cuh; its inputs are already in shared memory):
//   so [rows][C] block output, syb raw conv_b output, ssh raw shortcut-conv output (or null), tables tb / td.
// The CTA's records: BatchNorm-backward sums of conv_b and of the shortcut conv, cross-entropy, fc weight gradient.
// ------------------------------------------------------------------------------------------------
__device__ __noinline__ void res_head(const ResProgram& P, const ResCall& a, float* smem, const float* so, const float* syb, const float* ssh,
                                      const float* tb, const float* td, int u0, int nu, int cta) {
  const int C = P.blk[P.nblocks - 1].c, T = P.blk[P.nblocks - 1].t, NC = P.classes;
  const int tid = threadIdx.x;
  HeadSmem hs;
  hs.wfc = smem + P.o_head;
  hs.drop = hs.wfc + ((C * NC + 3) & ~3);
  hs.mk = hs.drop + kResMaxU * C;
  hs.dnet = hs.mk + kResMaxU * C;
  hs.logit = hs.dnet + kResMaxU * C;
  hs.dl = hs.logit + kResMaxU * NC;
  hs.loss = hs.dl + kResMaxU * NC;
  hs.red = hs.loss + kResMaxU;                               // [4 * blockDim]
  for (int i = tid; i < C * NC; i += kResThreads) hs.wfc[i] = __ldg(a.params + P.fc_off + i);
  float* sp = hs.dnet;                                       // [4C + 1] sums (8C floats, dead once the sums are formed)
  head_tail<kResThreads>(a, hs, C, T, NC, u0, nu, so, syb, ssh, tb, td, true, P.gout + (size_t)u0 * T * C, sp,
                         P.dwfc_part + (size_t)cta * C * NC);
  __syncthreads();
  for (int i = tid; i < 2 * C; i += kResThreads) {
    P.bpartb[(size_t)cta * 2 * C + i] = sp[i];
    if (P.bpartd) P.bpartd[(size_t)cta * 2 * C + i] = sp[2 * C + i];
  }
  if (tid == 0) P.loss_part[cta] = sp[4 * C];
}

// ------------------------------------------------------------------------------------------------
// forward kernel
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ TblDst res_tbl_dst(const ResCall& c, const RConv& L, float* tblr) {
  return TblDst{tblr + L.tbl, c.params + L.gamma_off, c.params + L.beta_off, L.bnf, L.var, L.cout, 1.0f / ((float)c.n * (float)L.t_out)};
}

__device__ __forceinline__ void res_run_conv(float* smem, const ResProgram& P, const RConv& L, const RConv* D, int xs_off, int Ue, int TP, int CS) {
  const int coutd = D ? D->cout : 0;
  if (L.k == 3) {
    if (L.tm == 2) res_conv<3, 2>(smem, xs_off, P.o_w, P.o_yo, P.o_sh, P.umax * L.t_out, Ue, L.cin, L.cout, coutd, L.stride, L.t_out, TP, CS, L.pad_left, L.ks);
    else res_conv<3, 4>(smem, xs_off, P.o_w, P.o_yo, P.o_sh, P.umax * L.t_out, Ue, L.cin, L.cout, coutd, L.stride, L.t_out, TP, CS, L.pad_left, L.ks);
  } else {
    if (L.tm == 2) res_conv<9, 2>(smem, xs_off, P.o_w, P.o_yo, P.o_sh, P.umax * L.t_out, Ue, L.cin, L.cout, coutd, L.stride, L.t_out, TP, CS, L.pad_left, L.ks);
    else res_conv<9, 4>(smem, xs_off, P.o_w, P.o_yo, P.o_sh, P.umax * L.t_out, Ue, L.cin, L.cout, coutd, L.stride, L.t_out, TP, CS, L.pad_left, L.ks);
  }
}

// Transposed filter banks wT[k][co][ci] for the backward-data pass (wT_source, as in weight_transpose_kernel), spread over the CTAs and
// run in the shadow of the first grid barrier: nobody waits for it before the kernel ends.
__device__ __noinline__ void res_weight_transpose(const ResProgram& P, const float* __restrict__ params, int cta, int G) {
  // one flat index space over all banks, an equal slice per CTA (a per-layer split left the low CTAs with nine dependent
  // round trips and made them the stragglers of the next barrier)
  int total = 0;
  for (int l = 1; l < P.nconvs; ++l) total += P.conv[l].k * P.conv[l].cin * P.conv[l].cout;
  const int per = (total + G - 1) / G;
  const int lo = cta * per, hi = imin(total, lo + per);
  for (int p = lo + (int)threadIdx.x; p < hi; p += kResThreads) {
    int l = 1, base = 0;
    for (;;) {
      const int numel = P.conv[l].k * P.conv[l].cin * P.conv[l].cout;
      if (p < base + numel) break;
      base += numel;
      ++l;
    }
    const RConv& L = P.conv[l];
    const int i = p - base;
    const_cast<float*>(L.wT)[i] = __ldg(params + L.w_off + wT_source(i, L.cin, L.cout));
  }
}

__global__ void __launch_bounds__(kResThreads, 1) resident_fwd_kernel(const __grid_constant__ ResProgram P, const __grid_constant__ ResCall c) {
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem_raw);       // first 16 bytes
  const int tid = threadIdx.x;
  const int G = (int)gridDim.x, cta = (int)blockIdx.x;
  const int ubase = c.n / G, urem = c.n % G;
  const int u0 = cta * ubase + imin(cta, urem), Ue = ubase + (cta < urem ? 1 : 0);
  unsigned wpar = 0;
  unsigned target = c.bar_base;
  uint64_t* fbar = wbar + 1;                                     // second half of the reserved 16 bytes: the feature tile's barrier
  if (tid == 0) { mbar_init(wbar, 1); mbar_init(fbar, 1); }
  __syncthreads();
  float* tblr = smem + P.o_tbl;
  float* red = smem + P.o_red;
  float* ys = smem + P.o_yo;
  float* sh = smem + P.o_sh;
  const int bufo[2] = {P.o_buf0, P.o_buf1};
  const int nb = P.nblocks, nph = 1 + 2 * nb;
  res_stamp(c, 0);
  res_load_bank(smem + P.o_w, c.params + P.conv[0].w_off, (unsigned)(P.conv[0].k * P.conv[0].cin * P.conv[0].cout), nullptr, 0u, wbar);
  {                                   // conv0's input: the T x F feature tiles of this CTA's utterances are one contiguous span:
    const RConv& L0 = P.conv[0];      // one TMA bulk copy into the (still idle) output-plane region, then the padded tile is formed from it
    const unsigned fbytes = (unsigned)(Ue * L0.t_in * L0.cin) * 4u;
    if (tid == 0) {
      mbar_expect_tx(fbar, fbytes);
      tma_load_1d(ys, c.feat + (size_t)u0 * L0.t_in * L0.cin, fbytes, fbar);
    }
    mbar_wait(fbar, 0u);
    res_stage(ys, nullptr, smem + bufo[0], Ue, L0.t_in, L0.cin, L0.pad_left + L0.t_in + L0.pad_right,
              chan_stride(L0.cin), L0.pad_left, L0.pad_right);
  }
  __syncthreads();
  int p = 1;                          // the block input X lives in buf[p], x_a and the block output in buf[1 - p]
  for (int ph = 0; ph < nph; ++ph) {
    const int bi = ph == 0 ? 0 : (ph - 1) >> 1;
    const bool isb = ph > 0 && ((ph - 1) & 1);
    const RBlock& B = P.blk[bi];
    const RConv& L = P.conv[ph == 0 ? 0 : (isb ? B.b : B.a)];
    const RConv* D = (ph > 0 && !isb && B.down >= 0) ? &P.conv[B.down] : nullptr;
    const int TP = L.pad_left + L.t_in + L.pad_right, CS = chan_stride(L.cin);
    const int xin = ph == 0 ? bufo[0] : (isb ? bufo[1 - p] : bufo[p]);
    const int R = Ue * L.t_out, rcap = P.umax * L.t_out;
    const int sl = ph < 3 ? 1 + 8 * ph : 64;
    mbar_wait(wbar, wpar); wpar ^= 1u;
    res_stamp(c, sl);
    res_run_conv(smem, P, L, D, xin, Ue, TP, CS);
    __syncthreads();
    res_stamp(c, sl + 1);
    if (ph + 1 < nph) {               // the bank region is free: the next layer's filters arrive while we reduce / wait
      const RBlock& Bn = P.blk[ph >> 1];                       // block of phase ph + 1
      const bool nb_isb = (ph & 1) == 1;                       // phase ph + 1 is a conv_b
      const RConv& Ln = P.conv[nb_isb ? Bn.b : Bn.a];
      const RConv* Dn = (!nb_isb && Bn.down >= 0) ? &P.conv[Bn.down] : nullptr;
      res_load_bank(smem + P.o_w, c.params + Ln.w_off, (unsigned)(Ln.k * Ln.cin * Ln.cout), Dn ? c.params + Dn->w_off : nullptr,
                    Dn ? (unsigned)(Dn->cin * Dn->cout) : 0u, wbar);
    }
    res_reduce_stats(ys, rcap, L.ks, R, L.cout, red, L.frec + (size_t)cta * 2 * L.cout);
    if (D) res_reduce_stats(sh, rcap, 1, R, D->cout, red, D->frec + (size_t)cta * 2 * D->cout);
    res_stamp(c, sl + 2);
    gbar_arrive(P.bar);
    target += (unsigned)G;
    // nobody waits for these: the pre-BatchNorm outputs go to global memory for the backward pass
    res_store(L.y + (size_t)u0 * L.t_out * L.cout, ys, R * (L.cout >> 2));
    if (D) res_store(D->y + (size_t)u0 * L.t_out * D->cout, sh, R * (D->cout >> 2));
    if (ph == 0) res_weight_transpose(P, c.params, cta, G);
    res_stamp(c, sl + 3);
    gbar_wait(P.bar, target);
    res_stamp(c, sl + 4);
    {
      const TblDst ta = res_tbl_dst(c, L, tblr);
      const TblDst td_ = D ? res_tbl_dst(c, *D, tblr) : ta;
      res_tables(L.frec, ta, D ? D->frec : nullptr, td_, D ? 2 : 1, G, P.eps, red, cta == 0);
    }
    res_stamp(c, sl + 5);
    if (!isb) {
      // x = relu(bn(y)) -> padded tile of the consumer: conv_a of block 0 (after conv0) or this block's conv_b
      const RConv& Cn = P.conv[ph == 0 ? P.blk[0].a : B.b];
      const int dsto = ph == 0 ? bufo[p] : bufo[1 - p];
      res_stage(ys, tblr + L.tbl, smem + dsto, Ue, Cn.t_in, Cn.cin, Cn.pad_left + Cn.t_in + Cn.pad_right, chan_stride(Cn.cin), Cn.pad_left, Cn.pad_right);
      __syncthreads();
    } else {
      // block output -> X of the next block (padded), or compact for the head
      const RConv& A = P.conv[B.a];
      const RConv* Dd = B.down >= 0 ? &P.conv[B.down] : nullptr;
      const int TPa = A.pad_left + A.t_in + A.pad_right, CSa = chan_stride(A.cin);
      float* ogl = B.out + (size_t)u0 * B.t * B.c;
      const float* td = Dd ? tblr + Dd->tbl : nullptr;
      const bool last = bi + 1 == nb;
      const RConv& An = P.conv[last ? B.a : P.blk[bi + 1].a];
      res_block_out(ys, tblr + L.tbl, Dd ? sh : nullptr, td, smem + bufo[p], TPa, CSa, A.pad_left, smem + bufo[1 - p], Ue, B.t, B.c,
                    last ? B.t : An.pad_left + An.t_in + An.pad_right, last ? B.c : chan_stride(An.cin), last ? 0 : An.pad_left,
                    last ? 0 : An.pad_right, ogl);
      __syncthreads();
      if (last) res_head(P, c, smem, smem + bufo[1 - p], ys, Dd ? sh : nullptr, tblr + L.tbl, td, u0, Ue, cta);
      p = 1 - p;
    }
    res_stamp(c, sl + 6);
  }
  res_stamp(c, 31);
}

// ================================================================================================
// backward
// ================================================================================================
// dy = FusedBatchNormGrad(dz) of one layer for the CTA's rows: dz [rows][C] and y [rows][C] in shared memory ->
// dst [U][TPd][COS] (rows at PLd.., pad rows zeroed).  mask: dz *= (bn(y) > 0) first (the shortcut conv's own ReLU).
__device__ __noinline__ void res_dy_stage(const float* dz, const float* y, const float* tbl, const float* sb, float inv_m, int mask,
                                          float* dst, int Ue, int t, int C, int TPd, int PLd, int COS) {
  const int c4n = C >> 2;
  zero_pad_rows(dst, Ue, t, c4n, TPd, COS, PLd, TPd - t, kResThreads);
  const RowWalk w = row_walk(threadIdx.x, kResThreads, c4n);
  const int rows = Ue * t;
  if (w.row < rows) {
    Dy4 d;
    d.dz = nullptr; d.y = nullptr;
    d.mask = mask;
    d.k = chan4_load_s(tbl, C, 4 * w.c4);
    const float4 s1 = ld4(sb + 4 * w.c4), s2 = ld4(sb + C + 4 * w.c4);
    d.s1m = make_float4(s1.x * inv_m, s1.y * inv_m, s1.z * inv_m, s1.w * inv_m);
    d.s2m = make_float4(s2.x * inv_m, s2.y * inv_m, s2.z * inv_m, s2.w * inv_m);
    int u = w.row / t, tt = w.row - u * t;
    for (int row = w.row; row < rows; row += w.rstep) {
      st4(dst + ((size_t)(u * TPd + PLd + tt) * COS + 4 * w.c4),
          dy4_apply(d, ld4(dz + (size_t)row * C + 4 * w.c4), ld4(y + (size_t)row * C + 4 * w.c4)));
      tt += w.rstep;
      while (tt >= t) { tt -= t; ++u; }
    }
  }
}

// Transposed conv (K = 9, convT_tasks in tcr_layer.cuh): dys [U][TPd][COS], dysd [U*t_out][COSD], banks wT [k][cout][cin] |
// wdT [coutd][cin] -> dx planes [KS][rcap][cin].
struct ConvTShape { int cin, cout, coutd, stride, t_in, t_out, pad_left, KS; };
__device__ __noinline__ void res_convT(float* smem, int dys_off, int dysd_off, int ws_off, int wsd_off, int dxs_off, int rcap, int Ue,
                                       int cin, int cout, int coutd, int S, int t_in, int t_out, int pad_left, int TPd, int PLd, int COS,
                                       int COSD, int KS) {
  const ConvTShape g{cin, cout, coutd, S, t_in, t_out, pad_left, KS};
  convT_tasks<9, TMR, kResThreads>(smem, WShared{smem, ws_off, wsd_off}, g, dys_off, dysd_off, smem + dxs_off, rcap, Ue, TPd, PLd, COS, COSD);
}

// Backward epilogue (bwd_epilogue in tcr_layer.cuh) on shared-memory tensors: g stays in shared memory (gdst) for the next phase
// and goes to global memory (gglob) for the grouped weight-gradient launch; the CTA's records go to recp / recpd.
//   kind 1: mask bn(yp) > 0, sums for that layer.  kind 2: mask (previous block's output) > 0, sums for its conv_b (yp, tp) and,
//   when ypd != null, for its shortcut conv.  The block output is read from outp (identity shortcut) or recomputed.
struct ResEpi { const float* gid; int epi_kind; const float* yp; const float* bnfp; const float* out_prev; const float* ypd;
                const float* bnfpd; float* gprev; int cin, KS; };
__device__ __noinline__ void res_bwd_epilogue(const float* dxs, int rcap, int KS, int Rin, int C, const float* gid, int kind,
                                              const float* yp, const float* tp, const float* outp, const float* ypd, const float* tpd,
                                              float* gdst, float* gglob, float* red, int red_cap, float* recp, float* recpd) {
  const ResEpi e{gid, kind, yp, tp, outp, ypd, tpd, gglob, C, KS};
  const int nseg = imax(1, imin(kResThreads / (C >> 2), red_cap / (4 * C)));   // red: [4][nseg][C]
  bwd_epilogue<kResThreads, true>(e, dxs, rcap, Rin, nseg, 0, gdst, red, recp, recpd);
  __syncthreads();
}

// kTrunc: the chain stops after c.phases phases (tcr_set_trainable); the full chain's instantiation has no phase count in it
template <bool kTrunc>
__global__ void __launch_bounds__(kResThreads, 1) resident_bwd_kernel(const __grid_constant__ ResProgram P, const __grid_constant__ ResCall c) {
  TCR_DYNAMIC_SMEM(smem_raw);
  float* smem = reinterpret_cast<float*>(smem_raw);
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem_raw);
  const int tid = threadIdx.x;
  const int G = (int)gridDim.x, cta = (int)blockIdx.x;
  const int ubase = c.n / G, urem = c.n % G;
  const int u0 = cta * ubase + imin(cta, urem), Ue = ubase + (cta < urem ? 1 : 0);
  unsigned wpar = 0;
  unsigned target = c.bar_base;
  if (tid == 0) mbar_init(wbar, 1);
  __syncthreads();
  float* tblr = smem + P.b_tbl;
  float* bsr = smem + P.b_bs;
  float* red = smem + P.b_red;
  float* ysr = smem + P.b_ys;        // y of the layer(s) whose dy is formed: [y_self | y_down]
  float* ypr = smem + P.b_yp;        // tensors of the layer(s) below: [yp | out_prev | ypd]
  const int nb = P.nblocks;
  int gi_b = 0, gi_a = 1, gi_n = 2;  // regions holding gblk (block-level gradient), g_a, and the gradient being produced
  res_stamp(c, 0);
  // every layer's BN table (published by the forward pass) stays in shared memory for the whole kernel
  {                                   // one flat pass over all layers' entries (tbl offsets are cumulative): a single round trip
    const RConv& Ll = P.conv[P.nconvs - 1];
    const int total = Ll.tbl + 4 * Ll.cout;
    for (int i = tid; i < total; i += kResThreads) {
      int l = 0;
      while (l + 1 < P.nconvs && i >= P.conv[l + 1].tbl) ++l;
      tblr[i] = __ldcg(P.conv[l].bnf + (i - P.conv[l].tbl));
    }
  }
  // inputs of the first phase (conv_b of the last block): bank, gradient at the block output, y_b, y_a
  {
    const RBlock& B = P.blk[nb - 1];
    const RConv& Lb = P.conv[B.b];
    const RConv& La = P.conv[B.a];
    const int n4 = Ue * B.t * (B.c >> 2);
    res_load_bank(smem + P.b_w, Lb.wT, (unsigned)(Lb.k * Lb.cin * Lb.cout), nullptr, 0u, wbar);
    res_fetch(smem + P.b_g[gi_b], P.gout + (size_t)u0 * B.t * B.c, n4);
    res_fetch(ysr, Lb.y + (size_t)u0 * B.t * B.c, n4);
    res_fetch(ypr, La.y + (size_t)u0 * B.t * B.c, n4);
  }
  // sums of the last block's conv_b (and shortcut conv) come from the head's records
  {
    const RBlock& B = P.blk[nb - 1];
    const RConv& Lb = P.conv[B.b];
    const BsDst sa{bsr + Lb.bs, Lb.bsum, Lb.cout};
    const RConv* Dd = B.down >= 0 ? &P.conv[B.down] : nullptr;
    const BsDst sd = Dd ? BsDst{bsr + Dd->bs, Dd->bsum, Dd->cout} : sa;
    res_bsums(Lb.brec, sa, Dd ? Dd->brec : nullptr, sd, Dd ? 2 : 1, G, red, cta == 0);
  }
  int slot = 1, done = 0;            // done: phases finished; each ends with the published sums of the layer(s) it produced
  for (int bi = nb - 1; bi >= 0 && (!kTrunc || done < c.phases); --bi) {
    const RBlock& B = P.blk[bi];
    const RConv& La = P.conv[B.a];
    const RConv& Lb = P.conv[B.b];
    const RConv* Dd = B.down >= 0 ? &P.conv[B.down] : nullptr;
    const int R = Ue * B.t;                                  // rows of this block's conv outputs
    // =============== phase Bb: conv_b (k 9, stride 1): gradient at relu(bn(y_a)) ===============
    {
      const int C = B.c, COS = chan_stride(C), PLd = 8, TPd = 8 + B.t + Lb.pad_left, rcap = P.umax * B.t;
      cp_async_wait_all();
      __syncthreads();
      res_stamp(c, slot);
      res_dy_stage(smem + P.b_g[gi_b], ysr, tblr + Lb.tbl, bsr + Lb.bs, 1.0f / ((float)c.n * (float)Lb.t_out), 0, smem + P.b_dys, Ue, B.t, C,
                   TPd, PLd, COS);
      mbar_wait(wbar, wpar); wpar ^= 1u;
      __syncthreads();
      res_convT(smem, P.b_dys, 0, P.b_w, 0, P.b_pl, rcap, Ue, C, C, 0, 1, B.t, B.t, Lb.pad_left, TPd, PLd, COS, 0, Lb.bks);
      __syncthreads();
      res_stamp(c, slot + 1);
      res_bwd_epilogue(smem + P.b_pl, rcap, Lb.bks, R, C, nullptr, 1, ypr, tblr + La.tbl, nullptr, nullptr, nullptr, smem + P.b_g[gi_a],
                       La.g + (size_t)u0 * B.t * C, ysr, P.b_ys_cap, La.brec + (size_t)cta * 2 * C, nullptr);
      res_stamp(c, slot + 2);
      gbar_arrive(P.bar);
      target += (unsigned)G;
      // ---- nobody waits for the rest of this phase: the next phase's (conv_a) tensors and bank(s) travel during the barrier ----
      if (!kTrunc || ++done < c.phases) {
        const int Ca = La.cin, Rin = Ue * La.t_in;
        res_fetch(ysr, La.y + (size_t)u0 * B.t * C, R * (C >> 2));
        if (Dd) res_fetch(ysr + P.umax * B.t * C, Dd->y + (size_t)u0 * B.t * C, R * (C >> 2));
        {                               // y / out of the layer(s) below into ypr (the epilogue has consumed y_a)
          const int n4 = Rin * (Ca >> 2), cap = P.umax * La.t_in * Ca;
          if (bi > 0) {
            const RBlock& Bp = P.blk[bi - 1];
            res_fetch(ypr, P.conv[Bp.b].y + (size_t)u0 * La.t_in * Ca, n4);
            res_fetch(ypr + cap, (Bp.down >= 0 ? P.conv[Bp.down].y : Bp.out) + (size_t)u0 * La.t_in * Ca, n4);
          } else {
            res_fetch(ypr, P.conv[0].y + (size_t)u0 * La.t_in * Ca, n4);
          }
        }
        res_load_bank(smem + P.b_w, La.wT, (unsigned)(La.k * La.cin * La.cout), Dd ? Dd->wT : nullptr, Dd ? (unsigned)(Dd->cin * Dd->cout) : 0u, wbar);
      }
      res_stamp(c, slot + 3);
      gbar_wait(P.bar, target);
      res_stamp(c, slot + 4);
      const BsDst sa{bsr + La.bs, La.bsum, La.cout};
      res_bsums(La.brec, sa, nullptr, sa, 1, G, red, cta == 0);
      slot += 5;
    }
    if (kTrunc && done == c.phases) break;
    // =============== phase Ba: conv_a (k 9, stride S) + shortcut conv / identity: gradient at the block input ===============
    {
      const int C = B.c, Ca = La.cin, S = La.stride, COS = chan_stride(C);
      const int PLd = (9 - 1) / S, PRd = imax(0, (La.t_in - 1 + La.pad_left) / S - (La.t_out - 1)), TPd = PLd + B.t + PRd;
      const int rcap = P.umax * La.t_in, Rin = Ue * La.t_in, cap = rcap * Ca;
      const float inv_m = 1.0f / ((float)c.n * (float)B.t);
      cp_async_wait_all();
      __syncthreads();
      res_stamp(c, slot);
      res_dy_stage(smem + P.b_g[gi_a], ysr, tblr + La.tbl, bsr + La.bs, inv_m, 0, smem + P.b_dys, Ue, B.t, C, TPd, PLd, COS);
      if (Dd) res_dy_stage(smem + P.b_g[gi_b], ysr + P.umax * B.t * C, tblr + Dd->tbl, bsr + Dd->bs, inv_m, 1, smem + P.b_dyd, Ue, B.t, C, B.t, 0, COS);
      mbar_wait(wbar, wpar); wpar ^= 1u;
      __syncthreads();
      res_convT(smem, P.b_dys, P.b_dyd, P.b_w, P.b_w + 9 * Ca * C, P.b_pl, rcap, Ue, Ca, C, Dd ? C : 0, S, La.t_in, B.t, La.pad_left, TPd, PLd,
                COS, COS, La.bks);
      __syncthreads();
      res_stamp(c, slot + 1);
      const float* gid = Dd ? nullptr : smem + P.b_g[gi_b];     // identity shortcut: the block-level gradient passes through
      if (bi > 0) {
        const RBlock& Bp = P.blk[bi - 1];
        const RConv& Lpb = P.conv[Bp.b];
        const RConv* Lpd = Bp.down >= 0 ? &P.conv[Bp.down] : nullptr;
        res_bwd_epilogue(smem + P.b_pl, rcap, La.bks, Rin, Ca, gid, 2, ypr, tblr + Lpb.tbl, Lpd ? nullptr : ypr + cap, Lpd ? ypr + cap : nullptr,
                         Lpd ? tblr + Lpd->tbl : nullptr, smem + P.b_g[gi_n], Bp.gblk + (size_t)u0 * La.t_in * Ca, ysr,
                         P.b_ys_cap, Lpb.brec + (size_t)cta * 2 * Ca,
                         Lpd ? Lpd->brec + (size_t)cta * 2 * Ca : nullptr);
      } else {
        res_bwd_epilogue(smem + P.b_pl, rcap, La.bks, Rin, Ca, gid, 1, ypr, tblr + P.conv[0].tbl, nullptr, nullptr, nullptr, smem + P.b_g[gi_n],
                         P.conv[0].g + (size_t)u0 * La.t_in * Ca, ysr, P.b_ys_cap, P.conv[0].brec + (size_t)cta * 2 * Ca,
                         nullptr);
      }
      res_stamp(c, slot + 2);
      gbar_arrive(P.bar);
      target += (unsigned)G;
      // ---- nobody waits for the rest of this phase: the next phase's tensors (ysr and ypr are dead) and bank travel ----
      if (kTrunc ? ++done < c.phases : bi > 0) {   // (truncated: done < phases implies bi > 0)
        const RBlock& Bp = P.blk[bi - 1];
        const RConv& Lpb = P.conv[Bp.b];
        res_fetch(ysr, Lpb.y + (size_t)u0 * Bp.t * Bp.c, Ue * Bp.t * (Bp.c >> 2));
        res_fetch(ypr, P.conv[Bp.a].y + (size_t)u0 * Bp.t * Bp.c, Ue * Bp.t * (Bp.c >> 2));
        res_load_bank(smem + P.b_w, Lpb.wT, (unsigned)(Lpb.k * Lpb.cin * Lpb.cout), nullptr, 0u, wbar);
      }
      res_stamp(c, slot + 3);
      gbar_wait(P.bar, target);
      res_stamp(c, slot + 4);
      if (bi > 0) {
        const RBlock& Bp = P.blk[bi - 1];
        const RConv& Lpb = P.conv[Bp.b];
        const RConv* Lpd = Bp.down >= 0 ? &P.conv[Bp.down] : nullptr;
        const BsDst sa{bsr + Lpb.bs, Lpb.bsum, Lpb.cout};
        const BsDst sd = Lpd ? BsDst{bsr + Lpd->bs, Lpd->bsum, Lpd->cout} : sa;
        res_bsums(Lpb.brec, sa, Lpd ? Lpd->brec : nullptr, sd, Lpd ? 2 : 1, G, red, cta == 0);
      } else {
        const RConv& L0 = P.conv[0];
        const BsDst sa{bsr + L0.bs, L0.bsum, L0.cout};
        res_bsums(L0.brec, sa, nullptr, sa, 1, G, red, cta == 0);
      }
      slot += 5;
      const int t = gi_b; gi_b = gi_n; gi_n = t;               // the produced gradient is the next block's gblk
    }
  }
  res_stamp(c, 31);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct ResidentState {
  ResProgram prog;
  size_t smem_f = 0, smem_b = 0;
  int grid_max = 0;                  // CTAs that can be co-resident (one per SM)
  int umax = 0;
  int mode = kResidentOff;           // which kernels of the step run resident (ResidentMode)
  unsigned bar_next = 0;             // value the arrival counter will have when the next launch starts
};

static void res_pick_tile(RConv& L, const RConv* D, int umax, int plane_budget_floats) {
  const int R = umax * L.t_out;
  double best = 1e30;
  L.tm = 4; L.ks = 1;
  for (int tm = 4; tm >= 2; tm -= 2) {
    for (int ks = 1; ks <= L.k; ++ks) {
      if (L.k % ks) continue;
      if ((long)ks * R * L.cout > plane_budget_floats) continue;
      const int nrt = (R + tm - 1) / tm;
      const long tmain = (long)nrt * (L.cout / 4) * ks, tdown = D ? (long)nrt * (D->cout / 4) : 0;
      const double wmain = (double)tm * (L.k / ks) * L.cin, wdown = (double)tm * L.cin;
      // rounds of 512 threads: main tasks first, the shorter shortcut tasks fill the last round
      const long full = tmain / kResThreads, rest = tmain % kResThreads;
      double cost = full * wmain;
      if (rest + tdown > 0) cost += rest > 0 ? wmain : wdown;
      if (rest + tdown > kResThreads) cost += wdown * ((rest + tdown - 1) / kResThreads);
      cost *= tm == 2 ? 1.2 : 1.0;                // smaller register tile: more shared-memory loads per FMA
      cost += ks > 1 ? 0.05 * ks * L.cin : 0.0;   // plane reduction
      if (cost < best - 1e-9) { best = cost; L.tm = tm; L.ks = ks; }
    }
  }
}

// k-slices of the transposed conv: enough tasks for 512 threads, planes within the budget
static int res_pick_bks(const RConv& L, int umax, int plane_budget_floats) {
  const int S = L.stride, NT0 = (L.k + S - 1) / S;
  const int rows = (L.t_in + TMR - 1) / TMR + (S > 1 ? 1 : 0);
  int best = 1;
  double best_cost = 1e30;
  for (int ks = 1; ks <= NT0; ++ks) {
    const int mps = (NT0 + ks - 1) / ks;
    if ((NT0 + mps - 1) / mps != ks) continue;
    if ((long)ks * umax * L.t_in * L.cin > plane_budget_floats) continue;
    const long tasks = (long)ks * umax * rows * (L.cin / 4);
    const double cost = (double)((tasks + kResThreads - 1) / kResThreads) * mps + 0.05 * ks;
    if (cost < best_cost - 1e-9) { best_cost = cost; best = ks; }
  }
  return best;
}

static ResidentState* resident_state(tcr_handle* h) {
  if (h->resident) return (ResidentState*)h->resident;
  ResidentState* S = new ResidentState();
  h->resident = S;
  // default: both resident kernels, ahead of the resident forward alone by the backward-data launches they save
  int want = kResidentFwdBwdData;
  if (const char* e = getenv("TCR_RESIDENT")) {
    const int v = atoi(e);
    if (v == kResidentOff || v == kResidentFwd) want = v;
  }
  if (h->sync_bn) want = kResidentOff;   // SyncBN lives in the per-layer kernels' launch sequence (NCCL between launches)
  if (want == kResidentOff) return S;
  int sms = 3;                       // emulator: a few CTAs exercise ragged ownership
#ifndef TCR_EMU
  int dev = 0, coop = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  if (!coop) return S;
#endif
  const int umax = (h->cfg.max_batch + sms - 1) / sms;
  if (umax > kResMaxU || h->c_last > kResThreads / 2 || h->cfg.num_classes > 32) return S;
  ResProgram& P = S->prog;
  memset(&P, 0, sizeof(P));
  P.nconvs = (int)h->convs.size();
  P.nblocks = (int)h->blocks.size();
  P.classes = h->cfg.num_classes;
  P.eps = h->cfg.bn_epsilon;
  P.umax = umax;
  int tbl = 0, bs = 0;
  for (int l = 0; l < P.nconvs; ++l) {
    const ConvPlan& cv = h->convs[l];
    RConv& L = P.conv[l];
    L.cin = cv.cin; L.cout = cv.cout; L.k = cv.k; L.stride = cv.stride; L.t_in = cv.t_in; L.t_out = cv.t_out;
    L.pad_left = cv.pad_left;
    L.pad_right = std::max((cv.t_out - 1) * cv.stride + cv.k - cv.pad_left - cv.t_in, 0);
    L.w_off = cv.w_off; L.gamma_off = cv.gamma_off; L.beta_off = cv.beta_off;
    L.y = cv.y; L.bnf = cv.bnf; L.var = cv.var; L.bsum = cv.bsum; L.g = cv.g; L.frec = cv.fpart; L.brec = cv.bpart; L.wT = cv.wT;
    L.tbl = tbl; L.bs = bs;
    tbl += 4 * cv.cout;
    bs += 2 * cv.cout;
    if (cv.cout > kResThreads / 2) return S;                       // single-pass statistics need 2C <= blockDim
    if (cv.k != 9 && cv.k != 3 && cv.k != 1) return S;
  }
  if (h->convs[0].k != 3) return S;
  for (int b = 0; b < P.nblocks; ++b) {
    const BlockPlan& bp = h->blocks[b];
    P.blk[b] = RBlock{bp.a, bp.b, bp.down, bp.c, bp.t, bp.out, bp.gblk};
    if (h->convs[bp.a].k != 9 || h->convs[bp.b].k != 9) return S;
  }
  auto al = [](int v) { return (v + 3) & ~3; };
  auto tile_floats = [&](const ConvPlan& cv) {
    const int pr = std::max((cv.t_out - 1) * cv.stride + cv.k - cv.pad_left - cv.t_in, 0);
    return umax * (cv.pad_left + cv.t_in + pr) * chan_stride(cv.cin);
  };
  auto down_of = [&](int l) -> const ConvPlan* {
    for (auto& bp : h->blocks)
      if (bp.a == l && bp.down >= 0) return &h->convs[bp.down];
    return nullptr;
  };
  // ---------------- forward layout ----------------
  const int plane_budget = 9 * 1024;                               // floats: k-slice planes of one layer
  int wmax = 0, plane_max = 0, sh_max = 0;
  for (int l = 0; l < P.nconvs; ++l) {
    const ConvPlan& cv = h->convs[l];
    if (cv.k == 1) continue;                                       // shortcut convs ride with their block's conv_a
    const ConvPlan* dn = down_of(l);
    res_pick_tile(P.conv[l], dn ? &P.conv[dn - &h->convs[0]] : nullptr, umax, plane_budget);
    P.conv[l].bks = l == 0 ? 1 : res_pick_bks(P.conv[l], umax, plane_budget);
    wmax = std::max(wmax, (int)cv.wnumel() + (dn ? (int)dn->wnumel() : 0));
    plane_max = std::max(plane_max, P.conv[l].ks * umax * cv.t_out * cv.cout);
    if (dn) sh_max = std::max(sh_max, umax * dn->t_out * dn->cout);
  }
  plane_max = std::max(plane_max, umax * h->convs[0].t_in * h->convs[0].cin);      // the raw feature tiles land there first (TMA)
  // ping-pong of the two tile buffers (see the kernel): conv0's input in buf0, block input X in buf[p], x_a and the block
  // output in buf[1 - p], p flips per block
  int bufsz[2] = {tile_floats(h->convs[0]), 0};
  {
    int p = 1;
    for (size_t b = 0; b < h->blocks.size(); ++b) {
      const BlockPlan& bp = h->blocks[b];
      bufsz[p] = std::max(bufsz[p], tile_floats(h->convs[bp.a]));
      bufsz[1 - p] = std::max(bufsz[1 - p], tile_floats(h->convs[bp.b]));
      const int outsz = b + 1 < h->blocks.size() ? tile_floats(h->convs[h->blocks[b + 1].a]) : umax * bp.t * bp.c;
      bufsz[1 - p] = std::max(bufsz[1 - p], outsz);
      p = 1 - p;
    }
  }
  const int red_floats = 4 * kResThreads;                          // statistics scratch / record chunk sums
  {
    int o = 4;                                                     // mbarrier
    P.o_w = o; o += al(wmax);
    P.o_buf0 = o; o += al(bufsz[0]);
    P.o_buf1 = o; o += al(bufsz[1]);
    P.o_yo = o; o += al(plane_max);
    P.o_sh = o; o += al(std::max(sh_max, 4));
    P.o_tbl = o; o += al(tbl);
    P.o_red = o; o += red_floats;
    P.o_head = o;
    o += al(h->c_last * P.classes) + 3 * kResMaxU * h->c_last + 2 * kResMaxU * P.classes + kResMaxU + 4 * kResThreads + 8;
    S->smem_f = (size_t)al(o) * 4;
  }
  // ---------------- backward layout ----------------
  {
    int ysmax = 0, ypmax = 0, dysmax = 0, dydmax = 0, plmax = 0;
    for (size_t b = 0; b < h->blocks.size(); ++b) {
      const BlockPlan& bp = h->blocks[b];
      const ConvPlan& ca = h->convs[bp.a];
      const ConvPlan& cb = h->convs[bp.b];
      const int C = bp.c, COS = chan_stride(C), rows = umax * bp.t;
      ysmax = std::max(ysmax, rows * C * (bp.down >= 0 ? 2 : 1));
      ypmax = std::max(ypmax, std::max(rows * C, umax * ca.t_in * ca.cin * (b > 0 ? 2 : 1)));
      // phase Bb
      dysmax = std::max(dysmax, umax * (8 + bp.t + cb.pad_left) * COS);
      plmax = std::max(plmax, P.conv[bp.b].bks * rows * C);
      // phase Ba
      const int S_ = ca.stride, PLd = 8 / S_, PRd = std::max(0, (ca.t_in - 1 + ca.pad_left) / S_ - (ca.t_out - 1));
      dysmax = std::max(dysmax, umax * (PLd + bp.t + PRd) * COS);
      if (bp.down >= 0) dydmax = std::max(dydmax, rows * COS);
      plmax = std::max(plmax, P.conv[bp.a].bks * umax * ca.t_in * ca.cin);
    }
    // conv0's rows and the input features are never staged here, but these sizes decide which shapes fit the kernel: without
    // them TCResNet14-1.0 at N=512 (T=49) would move from the per-layer backward-data kernels to this one.
    const ConvPlan& c0 = h->convs[0];
    ysmax = std::max(ysmax, umax * c0.t_out * c0.cout);
    ypmax = std::max(ypmax, umax * c0.t_in * c0.cin);
    dysmax = std::max(dysmax, umax * c0.t_out * chan_stride(c0.cout));
    int o = 4;
    P.b_w = o; o += al(wmax);
    ysmax = std::max(ysmax, 1024);                                 // epilogue scratch [4][nseg][C] lives here
    plmax = std::max(plmax, red_floats);                           // the record sums' scratch aliases the (then dead) planes
    P.b_ys = o; o += al(ysmax);
    P.b_ys_cap = al(ysmax);
    P.b_yp = o; o += al(ypmax);
    P.b_dys = o; o += al(dysmax);
    P.b_dyd = o; o += al(std::max(dydmax, 4));
    P.b_pl = o; o += al(plmax);
    {                                // the three gradient regions rotate (see the kernel); each is sized for what it ever holds
      int gsz[3] = {0, 0, 0}, gb = 0, ga = 1, gn = 2;
      for (int b = (int)h->blocks.size() - 1; b >= 0; --b) {
        const BlockPlan& bp = h->blocks[b];
        const ConvPlan& ca = h->convs[bp.a];
        gsz[gb] = std::max(gsz[gb], umax * bp.t * bp.c);
        gsz[ga] = std::max(gsz[ga], umax * bp.t * bp.c);
        gsz[gn] = std::max(gsz[gn], umax * ca.t_in * ca.cin);
        std::swap(gb, gn);
      }
      for (int i = 0; i < 3; ++i) { P.b_g[i] = o; o += al(gsz[i]); }
    }
    P.b_tbl = o; o += al(tbl);
    P.b_bs = o; o += al(bs);
    P.b_red = P.b_pl;
    S->smem_b = (size_t)al(o) * 4;
  }
  S->umax = umax;
  P.bar = h->d_gridbar;
  P.fc_off = h->fc_off;
  P.loss_part = h->d_loss_part; P.dwfc_part = h->d_dwfc_part;
  const BlockPlan& lb = h->blocks.back();
  P.gout = lb.gblk;
  P.bpartb = h->convs[lb.b].bpart;
  P.bpartd = lb.down >= 0 ? h->convs[lb.down].bpart : nullptr;
#ifndef TCR_EMU
  if (S->smem_f > 227 * 1024) return S;
  // the opt-in limit is a property of the FUNCTION, shared by every handle of the process: it is only ever raised
  static SmemOptIn optin_f, optin_b, optin_t;
  if (optin_f.ensure(resident_fwd_kernel, S->smem_f) != cudaSuccess) return S;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resident_fwd_kernel, kResThreads, S->smem_f) != cudaSuccess || per_sm < 1) return S;
  if (want == kResidentFwdBwdData) {
    if (S->smem_b > 227 * 1024 ||
        optin_b.ensure(resident_bwd_kernel<false>, S->smem_b) != cudaSuccess || optin_t.ensure(resident_bwd_kernel<true>, S->smem_b) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resident_bwd_kernel<false>, kResThreads, S->smem_b) != cudaSuccess || per_sm < 1 ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resident_bwd_kernel<true>, kResThreads, S->smem_b) != cudaSuccess || per_sm < 1)
      want = kResidentFwd;
  }
#endif
  S->grid_max = sms;
  S->mode = want;
  if (getenv("TCR_RESIDENT_VERBOSE")) {
    fprintf(stderr, "[tcr] resident mode %d, umax %d, smem fwd %zu B, bwd %zu B\n", S->mode, umax, S->smem_f, S->smem_b);
    for (int l = 0; l < P.nconvs; ++l)
      fprintf(stderr, "[tcr]   conv %d: %dx%d k%d s%d t%d->%d  fwd tm %d ks %d  bwd ks %d\n", l, P.conv[l].cin, P.conv[l].cout, P.conv[l].k,
              P.conv[l].stride, P.conv[l].t_in, P.conv[l].t_out, P.conv[l].tm, P.conv[l].ks, P.conv[l].bks);
  }
  return S;
}

void resident_destroy(tcr_handle* h) {
  delete (ResidentState*)h->resident;
  h->resident = nullptr;
}

// The resident kernels run where the activations of ceil(max_batch / #SMs) utterances and the largest filter bank fit in one
// SM's shared memory; see resident_state for what TCR_RESIDENT and SyncBN select.
int resident_mode(tcr_handle* h) { return resident_state(h)->mode; }

static int res_launch(tcr_handle* h, const char* name, void (*kernel)(const ResProgram, const ResCall), int G, size_t smem, const ResCall& c,
                      cudaStream_t s) {
  ResidentState* S = resident_state(h);
#ifndef TCR_EMU
  prof_begin(name, s);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(G); cfg.blockDim = dim3(kResThreads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  pdl_enabled();                     // this launch is fully ordered behind the previous kernel; later ones may chain on it
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, S->prog, c);
  prof_end(s);
  if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return TCR_ERR_CUDA; }
#else
  (void)name; (void)s;
  emu::launch_cooperative(dim3(G), dim3(kResThreads), smem, [&]() { kernel(S->prog, c); });
#endif
  return 0;
}

static ResCall res_call(tcr_handle* h, const float* feat, const tcr_step_args* a) {
  ResCall c;
  memset(&c, 0, sizeof(c));
  c.feat = feat; c.params = a->params; c.onehot = a->onehot; c.mask = a->dropout_mask;
  c.seed = a->dropout_seed; c.keep = h->cfg.dropout_keep_prob;
  c.use_dropout = h->cfg.dropout_keep_prob < 1.0f ? 1 : 0;
  c.label_smoothing = h->cfg.label_smoothing;
  c.logits = a->logits ? a->logits : h->d_logits;
  c.probs = a->probs ? a->probs : h->d_probs;
  c.n = a->n; c.inv_n = 1.0f / (float)a->n;
  c.tl = h->d_timeline;
  return c;
}

// Training-mode forward + head (with head backward) on features [n, T, F]; leaves what net_forward(..., backward=true) leaves.
int resident_forward(tcr_handle* h, const float* feat, const tcr_step_args* a, cudaStream_t s) {
  ResidentState* S = resident_state(h);
  const int G = std::min(S->grid_max, a->n);
  ResCall c = res_call(h, feat, a);
  c.bar_base = S->bar_next;
  S->bar_next += (unsigned)G * (unsigned)(1 + 2 * h->blocks.size());
  // per-CTA records: consumers sum G of them; the BN tables are final (published by CTA 0)
  for (auto& cv : h->convs) { cv.f_gc = 0; cv.b_gc = 0; }
  const BlockPlan& lb = h->blocks.back();
  h->convs[lb.b].b_gc = G;
  if (lb.down >= 0) h->convs[lb.down].b_gc = G;
  h->loss_gc = G;
  h->fc_records = G;
  return res_launch(h, "resident_fwd", resident_fwd_kernel, G, S->smem_f, c, s);
}

// The backward-data chain as the resident kernel.  It leaves every layer's masked gradient (ConvPlan::g, BlockPlan::gblk) and
// the published BatchNorm-backward sums, i.e. what the conv_bwd_data launches of net_backward_data leave, down to the depth
// the trainable set needs (tcr_handle::bwd_phases; the caller launches nothing when that is 0).
int resident_backward_data(tcr_handle* h, const float* feat, const tcr_step_args* a, cudaStream_t s) {
  ResidentState* S = resident_state(h);
  const int G = std::min(S->grid_max, a->n);
  ResCall c = res_call(h, feat, a);
  c.tl = h->d_timeline ? h->d_timeline + 148 * 32 : nullptr;
  c.bar_base = S->bar_next;
  c.phases = h->bwd_phases;                           // the chain stops at the lowest conv with a trained variable
  S->bar_next += (unsigned)G * (unsigned)c.phases;    // one grid barrier per phase run
  for (auto& cv : h->convs) cv.b_gc = 0;              // every layer's sums are published: nobody sums records afterwards
  const bool full = c.phases == 2 * (int)h->blocks.size();
  return res_launch(h, "resident_bwd_data", full ? resident_bwd_kernel<false> : resident_bwd_kernel<true>, G, S->smem_b, c, s);
}

}  // namespace tcr
