// tcr_net_bwd.cu — TC-ResNet backward kernels for sm_90a (fp32 FMA pipe).
//
// Replaces the gradient graph slim.learning.create_train_op builds (helper/trainer.py:199-211):
// Conv2DBackpropInput / Conv2DBackpropFilter / FusedBatchNormGrad / ReluGrad per layer.
//   conv_bwd_data_kernel<K>   : dy = FusedBatchNormGrad(dz) is formed while staging the tile (the two per-channel
//                               sums s1 = sum dz, s2 = sum dz*xhat are added up from the producer kernel's per-cluster
//                               records in the prologue, tcr_bn.cuh);
//                               dx = conv^T(dy, W) [+ the block's 1x1 shortcut conv^T] [+ identity gradient];
//                               epilogue applies the consumer-side ReLU mask, writes the next dz and emits the
//                               partial (s1, s2) of the layer(s) below, reduced over the 8 CTAs of a thread-block cluster
//                               through distributed shared memory into one record per cluster.
//                               Stride-2 transposed convs are split by output-row parity so no FMA is spent on
//                               the zeros of a dilated gradient.
//   conv_bwd_weight_kernel<K> : dW[k,ci,co] = sum_rows x[row+k, ci] * dy[row, co]; each thread owns 2 ci x 4 co
//                               x K taps in registers, CTAs split (co tile, row chunk); row-chunk partials are
//                               reduced in a fixed order by the optimizer kernel (deterministic, no atomics).
#include "tcr_layer.cuh"
#include "tcr_net.h"

namespace tcr {

constexpr int TMB = 4;   // input rows per thread task (backward-data)

// ------------------------------------------------------------------------------------------------
// backward data
// ------------------------------------------------------------------------------------------------
template <int K, bool WSMEM>
__device__ __forceinline__ void conv_bwd_data_body(const BwdDataArgs& a, const int vb, unsigned char* smem_raw, MbarCtx& mb) {
  float* smem = reinterpret_cast<float*>(smem_raw);
  const int tid = threadIdx.x;
  const int S = a.stride;
  const int u0 = vb * a.U;
  const int Ue = imax(0, imin(a.U, a.n - u0));        // 0: a CTA that only pads the grid to whole clusters
  const int COS = chan_stride(a.cout);
  const int PLd = (K - 1) / S;
  const int PRd = imax(0, (a.t_in - 1 + a.pad_left) / S - (a.t_out - 1));
  const int TPd = PLd + a.t_out + PRd;
  const int COSD = a.has_down ? chan_stride(a.coutd) : 0;
  const int Rin_max = a.U * a.t_in;
  // shared memory: [mbarrier | W | W_down | dy tile | dy_down tile | dx planes | scratch]
  uint64_t* bar = mb.bar;
  float* ws = smem + 4;
  const int wn = WSMEM ? K * a.cin * a.cout : 0;
  const int wdn = (WSMEM && a.has_down) ? a.cin * a.coutd : 0;
  float* wsd = ws + wn;
  if (WSMEM) {
    if (!mb.ready) {
      if (tid == 0) mbar_init(bar, 1);
      __syncthreads();
      mb.ready = true;
    }
    if (tid == 0) {
      fence_proxy_async();
      mbar_expect_tx(bar, (uint32_t)(wn + wdn) * 4u);
      tma_load_1d(ws, a.w, (uint32_t)wn * 4u, bar);
      if (wdn) tma_load_1d(wsd, a.wd, (uint32_t)wdn * 4u, bar);
    }
  }
  float* dys = wsd + wdn;                                            // [U][TPd][COS]
  float* dysd = dys + (size_t)a.U * TPd * COS;                       // [U][t_out][COSD]
  // dx planes start past BOTH the staged tiles and the epilogue scratch `red` (which aliases the filter bank / dy tiles from
  // `ws` on): with the filters read through L1/L2 and a small tile, `red` is the larger of the two.
  float* tiles_end = dysd + (a.has_down ? (size_t)a.U * a.t_out * COSD : 0);
  const int red_floats = 4 * imax(1, kThreads / (a.cin >> 2)) * a.cin;
  float* dxs = ws + imax((int)(tiles_end - ws), red_floats);         // [KS][Rin_max][cin]
  float* red = ws;                                                   // [4][nseg][cin]: aliases the filter bank / dy tiles,
                                                                     // which are dead once the transposed conv is done
  float* stat = dxs + (size_t)a.KS * Rin_max * a.cin;                // BN-backward sums: [2][cout] + [2][coutd] while staging,
  float* sb_main = stat;                                             // then this CTA's [4*cin] partial sums of the epilogue
  float* sb_down = stat + 2 * a.cout;
  float* stat_scratch = stat + imax(4 * a.cin, 2 * a.cout + 2 * a.coutd);   // [kThreads]
  const int ws_off = (int)(ws - smem), wsd_off = (int)(wsd - smem), dys_off = (int)(dys - smem), dysd_off = (int)(dysd - smem);

  // ---- stage dy (BatchNorm backward applied on load) ----
  {
    const int c4n = a.cout >> 2, npad = PLd + PRd;
    for (int idx = tid; idx < Ue * npad * c4n; idx += kThreads) {
      const int c4 = idx % c4n, pr = (idx / c4n) % npad, u = idx / (c4n * npad);
      const int row = pr < PLd ? pr : a.t_out + pr;
      st4(dys + ((size_t)(u * TPd + row) * COS + 4 * c4), make_float4(0.f, 0.f, 0.f, 0.f));
    }
    pdl_wait();                     // the transposed filter bank (TMA above) was written at the start of the step
    // raw (dz, y) rows are requested BEFORE the BatchNorm-backward sums are built: the two global round trips overlap
    constexpr int PF = 4;
    const RowWalk w = row_walk(tid, kThreads, c4n);
    const int rows = Ue * a.t_out;
    const size_t grow = (size_t)u0 * a.t_out;
    float4 pdz[PF], py[PF];
#pragma unroll
    for (int i = 0; i < PF; ++i) {
      const int row = w.row + i * w.rstep;
      pdz[i] = py[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < rows) {
        const size_t gofs = (grow + row) * a.cout + 4 * w.c4;
        pdz[i] = ld4(a.dy.dz + gofs);
        py[i] = ld4(a.dy.y + gofs);
      }
    }
    bsum_build(a.dy.bs, a.dy.bsum, a.cout, sb_main, stat_scratch, vb == 0);
    if (a.has_down) bsum_build(a.dyd.bs, a.dyd.bsum, a.coutd, sb_down, stat_scratch, vb == 0);
    if (w.row < rows) {
      const Dy4 d = dy4_make(a.dy, a.cout, 4 * w.c4, sb_main);
      int u = w.row / a.t_out, t = w.row - u * a.t_out;
      auto place = [&](float4 dz, float4 y) {
        st4(dys + ((size_t)(u * TPd + PLd + t) * COS + 4 * w.c4), dy4_apply(d, dz, y));
        t += w.rstep;
        while (t >= a.t_out) { t -= a.t_out; ++u; }
      };
#pragma unroll
      for (int i = 0; i < PF; ++i)
        if (w.row + i * w.rstep < rows) place(pdz[i], py[i]);
      for (int row = w.row + PF * w.rstep; row < rows; row += w.rstep) {
        const size_t gofs = (grow + row) * a.cout + 4 * w.c4;
        place(ld4(a.dy.dz + gofs), ld4(a.dy.y + gofs));
      }
    }
    if (a.has_down) {
      const int d4n = a.coutd >> 2;
      const RowWalk wd = row_walk(tid, kThreads, d4n);
      if (wd.row < rows) {
        const Dy4 d = dy4_make(a.dyd, a.coutd, 4 * wd.c4, sb_down);
        for (int row = wd.row; row < rows; row += wd.rstep)
          st4(dysd + ((size_t)row * COSD + 4 * wd.c4), dy4_load(d, (grow + row) * a.coutd + 4 * wd.c4));
      }
    }
  }
  if (WSMEM) { mbar_wait(bar, mb.parity); mb.parity ^= 1u; }
  __syncthreads();

  // ---- transposed conv (+ shortcut conv^T) into the dx planes ----
  if (WSMEM) convT_tasks<K, TMB, kThreads>(smem, WShared{smem, ws_off, wsd_off}, a, dys_off, dysd_off, dxs, Rin_max, Ue, TPd, PLd, COS, COSD);
  else convT_tasks<K, TMB, kThreads>(smem, WGlobal{a.w, a.wd}, a, dys_off, dysd_off, dxs, Rin_max, Ue, TPd, PLd, COS, COSD);
  __syncthreads();

  // ---- epilogue: dz of the layer(s) below + partial BatchNorm-backward sums, one record per cluster ----
  bwd_epilogue<kThreads, false>(a, dxs, Rin_max, Ue * a.t_in, imax(1, kThreads / (a.cin >> 2)), (size_t)u0 * a.t_in, nullptr, red, stat,
                                stat + 2 * a.cin);
  const PubSeg segs[2] = {{stat, 2 * a.cin, a.bpartp}, {stat + 2 * a.cin, (a.epi_kind == 2 && a.ypd) ? 2 * a.cin : 0, a.bpartpd}};
  cluster_publish(segs, vb);
}

template <int K, bool WSMEM>
__global__ void __launch_bounds__(kThreads) conv_bwd_data_kernel(BwdDataArgs a) {
  TCR_DYNAMIC_SMEM(smem_raw);
  MbarCtx mb{reinterpret_cast<uint64_t*>(smem_raw), 0u, false};
  pdl_trigger();
  conv_bwd_data_body<K, WSMEM>(a, blockIdx.x, smem_raw, mb);
}

// Transposed filter banks wT[k][co][ci] for the backward-data kernels (all conv layers, one launch).  `params`
// is caller-owned and may change between calls, so the copy is refreshed at the start of every backward pass
// (65 K - 300 K floats: a few microseconds).
__device__ __forceinline__ void weight_transpose_body(const WtArgs& a, const int64_t p) {
  if (p >= a.total) return;
  int l = 0;
  while (l + 1 < a.nlayers && p >= a.layer[l + 1].begin) ++l;
  const WtLayer L = a.layer[l];
  const int64_t i = p - L.begin;
  L.wT[i] = a.params[L.w_off + wT_source(i, L.cin, L.cout)];
}
__global__ void __launch_bounds__(256) weight_transpose_kernel(WtArgs a) {
  pdl_wait();
  weight_transpose_body(a, (int64_t)blockIdx.x * 256 + threadIdx.x);
}

// ------------------------------------------------------------------------------------------------
// backward weight
// ------------------------------------------------------------------------------------------------
template <int K>
__device__ __forceinline__ void dw_body(const BwdWeightArgs& a, int bx, int by, float* smem) {
  const int tid = threadIdx.x;
  const int cot0 = bx * a.cot;
  const int upc = (a.n + a.R - 1) / a.R;                       // utterances per row chunk
  const int ubeg = by * upc, uend = imin(a.n, ubeg + upc);
  const int pad_right = imax((a.t_out - 1) * a.stride + K - a.pad_left - a.t_in, 0);
  const int TP = a.pad_left + a.t_in + pad_right;
  const int CI2 = a.cin >> 1;
  const int NP = CI2 * (a.cot >> 2);
  float* xs = smem;                                            // [UB][TP][cin]
  float* dys = xs + (size_t)a.UB * TP * a.cin;                 // [UB * t_out][cot]
  float* tblx = dys + (size_t)a.UB * a.t_out * a.cot;          // [4][cin] BN table of the input layer
  float* sbw = tblx + 4 * a.cin;                               // [2][cout] BN-backward sums of this layer
  float* wscr = sbw + 2 * a.cout;                              // [kDwThreads] scratch
  if (a.x.kind == 1) bn_table_build(a.x.st, a.x.bnf, a.cin, tblx, wscr, false);
  bsum_build(a.dy.bs, a.dy.bsum, a.cout, sbw, wscr, bx == 0 && by == 0);   // conv0: no backward-data kernel published its sums
  const int rg = tid / NP, pr = tid - rg * NP;
  const int ci2 = pr % CI2, co4 = pr / CI2;
  const bool worker = rg < a.RG;

  float4 acc[K][2];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k][0] = acc[k][1] = make_float4(0.f, 0.f, 0.f, 0.f);

  const int c4n = a.cin >> 2, d4n = a.cot >> 2, npad = a.pad_left + pad_right;
  for (int ub0 = ubeg; ub0 < uend; ub0 += a.UB) {
    const int Ue = imin(a.UB, uend - ub0);
    zero_pad_rows(xs, Ue, a.t_in, c4n, TP, a.cin, a.pad_left, npad, (int)blockDim.x);
    {
      const RowWalk w = row_walk(tid, (int)blockDim.x, c4n);
      const int rows = Ue * a.t_in;
      if (w.row < rows) {
        const Act4 src = act4_make(a.x, a.cin, 4 * w.c4, tblx);
        int u = w.row / a.t_in, t = w.row - u * a.t_in;
        for (int row = w.row; row < rows; row += w.rstep) {
          st4(xs + ((size_t)(u * TP + a.pad_left + t) * a.cin + 4 * w.c4),
              act4_load(src, ((size_t)ub0 * a.t_in + row) * a.cin + 4 * w.c4));
          t += w.rstep;
          while (t >= a.t_in) { t -= a.t_in; ++u; }
        }
      }
    }
    {
      const RowWalk w = row_walk(tid, (int)blockDim.x, d4n);
      const int rows = Ue * a.t_out;
      if (w.row < rows) {
        const Dy4 d = dy4_make(a.dy, a.cout, cot0 + 4 * w.c4, sbw);
        for (int row = w.row; row < rows; row += w.rstep)
          st4(dys + (size_t)row * a.cot + 4 * w.c4, dy4_load(d, ((size_t)ub0 * a.t_out + row) * a.cout + cot0 + 4 * w.c4));
      }
    }
    __syncthreads();
    if (worker) {
      // worker rg takes t = rg, rg + RG, ... of every staged utterance: no division in the row loop
      const int xstep = a.stride * a.cin;
      int xu = (int)(xs - smem) + 2 * ci2, du = (int)(dys - smem) + 4 * co4;
      for (int u = 0; u < Ue; ++u, xu += TP * a.cin, du += a.t_out * a.cot) {
        int xrow = xu + rg * xstep, drow = du + rg * a.cot;
        for (int t = rg; t < a.t_out; t += a.RG, xrow += a.RG * xstep, drow += a.RG * a.cot) {
          const float4 d = ld4(smem + drow);
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const float2 x = ld2(smem + xrow + k * a.cin);
            acc[k][0].x = fmaf(x.x, d.x, acc[k][0].x); acc[k][0].y = fmaf(x.x, d.y, acc[k][0].y);
            acc[k][0].z = fmaf(x.x, d.z, acc[k][0].z); acc[k][0].w = fmaf(x.x, d.w, acc[k][0].w);
            acc[k][1].x = fmaf(x.y, d.x, acc[k][1].x); acc[k][1].y = fmaf(x.y, d.y, acc[k][1].y);
            acc[k][1].z = fmaf(x.y, d.z, acc[k][1].z); acc[k][1].w = fmaf(x.y, d.w, acc[k][1].w);
          }
        }
      }
    }
    __syncthreads();
  }
  // ---- fixed-order reduction over the row groups of this CTA, then one partial per (row chunk, weight) ----
  float* scratch = smem;                                       // [(RG-1)][NP][K][8], tiles and tables are dead now
  if (worker && rg > 0) {
    float* sc = scratch + ((size_t)(rg - 1) * NP + pr) * K * 8;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      st4(sc + k * 8, acc[k][0]);
      st4(sc + k * 8 + 4, acc[k][1]);
    }
  }
  __syncthreads();
  if (worker && rg == 0) {
    for (int g = 1; g < a.RG; ++g) {
      const float* sc = scratch + ((size_t)(g - 1) * NP + pr) * K * 8;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        acc[k][0] = add4(acc[k][0], ld4(sc + k * 8));
        acc[k][1] = add4(acc[k][1], ld4(sc + k * 8 + 4));
      }
    }
    float* out = a.dwpart + (size_t)by * K * a.cin * a.cout;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      st4(out + ((size_t)k * a.cin + 2 * ci2) * a.cout + cot0 + 4 * co4, acc[k][0]);
      st4(out + ((size_t)k * a.cin + 2 * ci2 + 1) * a.cout + cot0 + 4 * co4, acc[k][1]);
    }
  }
}

// All layers' weight gradients in ONE launch: virtual CTA -> (layer, output-channel tile, row chunk) through a
// static table, so ~600 CTAs of 256 threads keep every SM busy instead of ten serial 64-CTA launches.
__device__ __forceinline__ void dw_grouped_body(const DwLayer* __restrict__ layers, int nlayers, int n, const float* __restrict__ feat,
                                                long long* tl, const int vb, unsigned char* smem_raw, const BsumSrc& bs0, float inv_scale) {
  float* smem = reinterpret_cast<float*>(smem_raw);
  tl_stamp(tl, 4096 + vb, 0);
  int l = 0;
  while (l + 1 < nlayers && vb >= layers[l + 1].cta_begin) ++l;
  const DwLayer L = layers[l];
  const int local = vb - L.cta_begin;
  const int ncot = L.cout / L.cot;
  BwdWeightArgs a;
  a.n = n;
  a.x = ActSrc{L.x_data ? L.x_data : feat, L.x_bnf, L.x_kind, StatSrc{}};     // tables were published during the forward pass
  a.dy = DySrc{L.dz, L.y, L.bnf, L.bsum, L.mask_relu, 1.0f / ((float)n * (float)L.t_out) * inv_scale, l == 0 ? bs0 : BsumSrc{nullptr, 0, nullptr}};
  a.cin = L.cin; a.cout = L.cout; a.k = L.k; a.stride = L.stride; a.t_in = L.t_in; a.t_out = L.t_out;
  a.pad_left = L.pad_left; a.cot = L.cot; a.RG = L.RG; a.R = L.R; a.UB = L.UB; a.dwpart = L.dwpart;
  const int bx = local % ncot, by = local / ncot;
  tl_stamp(tl, 4096 + vb, 1);
  if (L.k == 9) dw_body<9>(a, bx, by, smem);
  else if (L.k == 3) dw_body<3>(a, bx, by, smem);
  else dw_body<1>(a, bx, by, smem);
  tl_stamp(tl, 4096 + vb, 2);
  if (tl && threadIdx.x == 0) { tl[(size_t)(4096 + vb) * 8 + 3] = l; tl[(size_t)(4096 + vb) * 8 + 4] = (long long)by; }
}
__global__ void __launch_bounds__(kDwThreads, 2) dw_grouped_kernel(const DwLayer* __restrict__ layers, int nlayers, int n,
                                                                const float* __restrict__ feat, long long* tl, BsumSrc bs0, float inv_scale) {
  TCR_DYNAMIC_SMEM(smem_raw);
  pdl_wait();
  dw_grouped_body(layers, nlayers, n, feat, tl, (int)blockIdx.x, smem_raw, bs0, inv_scale);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static constexpr size_t kSmemBudgetW = 64 * 1024;

static size_t bwd_data_smem(const ConvPlan& cv, const ConvPlan* dn, int U, int KS, bool w_smem) {
  const int S = cv.stride;
  const int PLd = (cv.k - 1) / S;
  const int PRd = std::max(0, (cv.t_in - 1 + cv.pad_left) / S - (cv.t_out - 1));
  const int TPd = PLd + cv.t_out + PRd;
  const int ncig = cv.cin / 4;
  const int nseg = std::max(1, kThreads / ncig);
  size_t f = (size_t)U * TPd * chan_stride(cv.cout) + (dn ? (size_t)U * cv.t_out * chan_stride(dn->cout) : 0);
  f += (w_smem ? (size_t)cv.wnumel() + (dn ? (size_t)dn->wnumel() : 0) : 0);
  f = std::max(f, (size_t)4 * nseg * cv.cin);            // epilogue scratch aliases the filter bank + dy tiles
  f += 4 + (size_t)KS * U * cv.t_in * cv.cin;
  f += std::max((size_t)4 * cv.cin, (size_t)2 * cv.cout + (dn ? (size_t)2 * dn->cout : 0)) + kThreads;   // BN-backward sums / partials
  return f * 4;
}

double tile_cost(int sms, int n, int U, int occ, bool wsm);     // tcr_net_fwd.cu

// false: not even the smallest tile (one utterance, one slice, filters through L1/L2) fits in `limit` bytes (see pick_fwd_tile)
static bool pick_bwd_tile(int sms, const ConvPlan& cv, const ConvPlan* dn, int n, size_t limit, int* U_out, int* KS_out, int* wsm_out) {
  const size_t wbytes = ((size_t)cv.wnumel() + (dn ? (size_t)dn->wnumel() : 0)) * 4;
  const int S = cv.stride, NT0 = (cv.k + S - 1) / S;
  double best = 1e30;
  *U_out = 1; *KS_out = 1; *wsm_out = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const bool wsm = pass < 2;
    const int occ = (pass & 1) ? 1 : 2;
    const size_t budget = occ == 2 ? kSmemBudget : kSmemMax;
    if (wsm && wbytes + 16 * 1024 > budget) continue;
    for (int U = std::min(16, std::max(1, (n + sms * occ - 1) / (sms * occ))); U >= 1; --U) {
      int best_ks = 0;
      double best_cost = 1e30;
      for (int KS = 1; KS <= NT0; ++KS) {
        const int mps = (NT0 + KS - 1) / KS;
        if ((NT0 + mps - 1) / mps != KS) continue;   // skip slice counts that leave empty slices
        const int rows = (cv.t_in + TMB - 1) / TMB + (S > 1 ? 1 : 0);
        const long tasks = (long)KS * U * rows * (cv.cin / 4);
        const double cost = (double)((tasks + kThreads - 1) / kThreads) * mps;
        if (cost < best_cost - 1e-9 && bwd_data_smem(cv, dn, U, KS, wsm) <= budget) {
          best_cost = cost;
          best_ks = KS;
        }
      }
      if (!best_ks) continue;
      const double c = tile_cost(sms, n, U, occ, wsm);
      if (c < best - 1e-9) { best = c; *U_out = U; *KS_out = best_ks; *wsm_out = wsm ? 1 : 0; }
      break;
    }
  }
  return best < 1e30 || bwd_data_smem(cv, dn, 1, 1, false) <= limit;
}

static size_t bwd_weight_smem(const ConvPlan& cv, int cot, int RG, int UB) {
  const int pad_right = std::max((cv.t_out - 1) * cv.stride + cv.k - cv.pad_left - cv.t_in, 0);
  const int TP = cv.pad_left + cv.t_in + pad_right;
  const size_t tiles = ((size_t)UB * TP * cv.cin + (size_t)UB * cv.t_out * cot + 4 * cv.cin + 2 * cv.cout + kDwThreads) * 4;
  const size_t np = (size_t)(cv.cin / 2) * (cot / 4);
  const size_t scratch = (size_t)(RG - 1) * np * cv.k * 8 * 4;
  return std::max(tiles, scratch);
}

// Static per-layer choice of (output-channel tile, row groups, row chunks, staged utterances) for 256-thread CTAs:
// the tile that keeps most threads busy, chunks of roughly equal work (~0.7 M MAC) so all layers together give a
// few waves of CTAs.
void plan_bwd_weight(tcr_handle* h) {
  // Per layer: the LARGEST output-channel tile that fits 256 threads (tiny tiles re-stage the same x tile many times) and at
  // most 4 row groups.  Row chunks: ONE wave of CTAs (SMs x 2) with equal predicted duration.  The time of a CTA is modelled
  // as ~ utterances x (0.9 + MACs per utterance and tile / 70e3): the K=1 shortcut convs are staging-bound, the others
  // FMA-bound.  Chunks of equal MACs would leave long conv0 chunks and a late second wave; balanced, the launch is bounded by
  // sum(tau_l x tiles_l) x N / (2 x SMs).
  struct L { ConvPlan* cv; int cot, ncot; double tau; };
  std::vector<L> ls;
  for (auto& cv : h->convs) {
    // output-channel tile: the LARGEST that fits 256 threads (a thread owns 2 ci x 4 co x K taps).  A smaller tile with more row
    // groups keeps more threads busy (75-84 % instead of 56-63 % on 48- and 36-channel layers) but re-stages the x tile per
    // tile and is slower on TCResNet8 and TCResNet14-1.5.
    int cot = 4;
    for (int c = 4; c <= cv.cout; c += 4)
      if (cv.cout % c == 0 && (cv.cin / 2) * (c / 4) <= kDwThreads) cot = c;
    const double macs = (double)cv.t_out * cv.k * cv.cin * cot;
    ls.push_back(L{&cv, cot, cv.cout / cot, 0.9 + macs / 70e3});
  }
  const int n = h->cfg.max_batch;
  int slots = 2 * h->sms, upc_cap = 256;
  if (const char* e = getenv("TCR_DW_SLOTS")) slots = atoi(e);              // tuning knobs (tools/sweep_dw.sh)
  if (const char* e = getenv("TCR_DW_UPC")) upc_cap = atoi(e);
  auto ctas_at = [&](double D) {
    long c = 0;
    for (auto& l : ls) {
      const int upc = std::max(1, std::min(upc_cap, (int)(D / l.tau)));
      c += (long)l.ncot * ((n + upc - 1) / upc);
    }
    return c;
  };
  double D = 1.0;
  while (ctas_at(D) > slots && D < 1e5) D *= 1.05;
  for (auto& l : ls) {
    ConvPlan& cv = *l.cv;
    const int np = (cv.cin / 2) * (l.cot / 4);
    int RG = std::max(1, std::min(4, kDwThreads / np));
    const int upc = std::max(1, std::min(upc_cap, (int)(D / l.tau)));     // utterances per chunk
    const int R = std::max(1, (n + upc - 1) / upc);
    int UB = 8;
    while (UB > 1 && bwd_weight_smem(cv, l.cot, RG, UB) > kSmemBudgetW) --UB;
    while (RG > 1 && bwd_weight_smem(cv, l.cot, RG, UB) > kSmemBudget) --RG;
    cv.dw_cot = l.cot;
    cv.dw_RG = RG;
    cv.dw_R = R;
    cv.dw_UB = UB;
  }
}

// What the per-layer path can run, checked once when the handle is created (after plan_bwd_weight): a handle tcr_create accepts
// can always evaluate (tcr_forward runs only these kernels) and always train with TCR_RESIDENT=0.  No layer has more than
// kThreads / 2 channels, the head keeps its two-CTAs-per-SM budget; every convolution's smallest forward and backward-data tile (one
// utterance per CTA) and its planned weight-gradient tile must fit in what one CTA may opt in to.  The resident kernels are not
// part of it: where their layout does not fit, the step falls back to these.
int net_check_envelope(tcr_handle* h) {
  char msg[256];
  auto refuse = [&](const std::string& what, size_t need, size_t limit) {
    snprintf(msg, sizeof(msg), "%s needs %zu B of shared memory, limit %zu B: shorten the clip or the width", what.c_str(), need, limit);
    set_error(msg);
    return TCR_ERR_UNSUPPORTED;
  };
  // the one-pass BatchNorm statistics of the per-layer kernels (tile_stats, records_sum) give each of a layer's 2 x C columns
  // one of the CTA's kThreads threads
  int c_max = 0;
  for (const ConvPlan& cv : h->convs) c_max = std::max(c_max, cv.cout);
  if (2 * c_max > kThreads) {
    snprintf(msg, sizeof(msg), "%s has a %d-channel layer, the per-layer kernels' BatchNorm statistics take at most %d channels: lower the width",
             h->scope.c_str(), c_max, kThreads / 2);
    set_error(msg);
    return TCR_ERR_UNSUPPORTED;
  }
  const size_t limit = h->smem_optin;
  int U, KS, wsm;
  const ConvPlan& c0 = h->convs[0];
  if (!pick_fwd_tile(h->sms, c0, nullptr, 1, limit, &U, &KS, &wsm))
    return refuse("forward tile of " + h->scope + "/" + c0.name, fwd_smem_bytes(c0, nullptr, 1, 1, false), limit);
  for (const BlockPlan& b : h->blocks) {
    const ConvPlan& ca = h->convs[b.a];
    const ConvPlan& cb = h->convs[b.b];
    const ConvPlan* dn = b.down >= 0 ? &h->convs[b.down] : nullptr;
    if (!pick_fwd_tile(h->sms, ca, dn, 1, limit, &U, &KS, &wsm))
      return refuse("forward tile of " + h->scope + "/" + ca.name, fwd_smem_bytes(ca, dn, 1, 1, false), limit);
    if (!pick_fwd_tile(h->sms, cb, nullptr, 1, limit, &U, &KS, &wsm))
      return refuse("forward tile of " + h->scope + "/" + cb.name, fwd_smem_bytes(cb, nullptr, 1, 1, false), limit);
    if (!pick_bwd_tile(h->sms, ca, dn, 1, limit, &U, &KS, &wsm))
      return refuse("backward-data tile of " + h->scope + "/" + ca.name, bwd_data_smem(ca, dn, 1, 1, false), limit);
    if (!pick_bwd_tile(h->sms, cb, nullptr, 1, limit, &U, &KS, &wsm))
      return refuse("backward-data tile of " + h->scope + "/" + cb.name, bwd_data_smem(cb, nullptr, 1, 1, false), limit);
  }
  for (const ConvPlan& cv : h->convs) {
    const size_t need = bwd_weight_smem(cv, cv.dw_cot, cv.dw_RG, cv.dw_UB);
    if (need > limit) return refuse("weight-gradient tile of " + h->scope + "/" + cv.name, need, limit);
  }
  if (head_smem_bytes(h) > kSmemBudget) {
    char what[128];
    snprintf(what, sizeof(what), "head tile of %s (T_last %d, %d channels)", h->scope.c_str(), h->t_last, h->c_last);
    return refuse(what, head_smem_bytes(h), kSmemBudget);
  }
  return 0;
}

// Device table of the grouped weight-gradient launch (pointers are workspace addresses: static per handle).  Only the layers
// whose weights are trained (tcr_set_trainable) are in it; each keeps its own row partition (plan_bwd_weight), so its partial
// sums, and its gradient, are those of the full table.
int build_dw_table(tcr_handle* h) {
  std::vector<DwLayer> tab;
  int cta = 0;
  size_t smem = 0;
  auto add = [&](ConvPlan& cv, const float* xd, const float* xb, int xk, const float* dz, int mask) {
    if (!h->conv_w_trained((int)(&cv - &h->convs[0]))) return;
    DwLayer L;
    L.x_data = xd; L.x_bnf = xb; L.x_kind = xk;
    L.dz = dz; L.y = cv.y; L.bnf = cv.bnf; L.bsum = cv.bsum; L.mask_relu = mask;
    L.cin = cv.cin; L.cout = cv.cout; L.k = cv.k; L.stride = cv.stride; L.t_in = cv.t_in; L.t_out = cv.t_out;
    L.pad_left = cv.pad_left; L.cot = cv.dw_cot; L.RG = cv.dw_RG; L.R = cv.dw_R; L.UB = cv.dw_UB;
    L.dwpart = cv.dwpart;
    L.cta_begin = cta;
    cta += (cv.cout / cv.dw_cot) * cv.dw_R;
    smem = std::max(smem, bwd_weight_smem(cv, cv.dw_cot, cv.dw_RG, cv.dw_UB));
    tab.push_back(L);
  };
  ConvPlan& c0 = h->convs[0];
  add(c0, nullptr, nullptr, 0, c0.g, 0);                       // x = features (pointer supplied per call)
  for (size_t i = 0; i < h->blocks.size(); ++i) {
    BlockPlan& b = h->blocks[i];
    ConvPlan& ca = h->convs[b.a];
    ConvPlan& cb = h->convs[b.b];
    const float* xd = i == 0 ? c0.y : h->blocks[i - 1].out;
    const float* xb = i == 0 ? c0.bnf : nullptr;
    const int xk = i == 0 ? 1 : 0;
    add(ca, xd, xb, xk, ca.g, 0);
    if (b.down >= 0) add(h->convs[b.down], xd, xb, xk, b.gblk, 1);
    add(cb, ca.y, ca.bnf, 1, b.gblk, 0);
  }
  h->dw_ctas = cta;
  h->dw_smem = smem;
  h->n_dw_layers = (int)tab.size();
  h->dw_conv0 = h->conv_w_trained(0) ? 1 : 0;
  if (!h->d_dw_layers) {             // sized for every layer: a later tcr_set_trainable rewrites it in place
    void* p = nullptr;
    if (cudaMalloc(&p, h->convs.size() * sizeof(DwLayer)) != cudaSuccess) return TCR_ERR_CUDA;
    h->allocs.push_back(p);
    h->d_dw_layers = (DwLayer*)p;
  }
  if (!tab.empty() && cudaMemcpy(h->d_dw_layers, tab.data(), tab.size() * sizeof(DwLayer), cudaMemcpyHostToDevice) != cudaSuccess)
    return TCR_ERR_CUDA;
  return 0;
}

// Backward-data phases a step runs: 2 per block from the last block down ((1) conv_b -> g of conv_a, (2) conv_a + shortcut ->
// gradient at the block input), only as deep as the lowest conv with a trained variable needs.  conv_b / down of block i read
// gblk_i (phase (2) of block i + 1), conv_a of block i phase (1) of block i, conv0 phase (2) of block 0.  0: only fc / fc2.
// The last block's conv_b / down take phase (1) as well: the head leaves their BatchNorm-backward sums as records, and the
// resident kernel publishes them (with its own summation order) when it starts.
int plan_bwd_phases(const tcr_handle* h) {
  const int nb = (int)h->blocks.size();
  int phases = h->conv_any_trained(0) ? 2 * nb : 0;
  for (int i = 0; i < nb; ++i) {
    const BlockPlan& b = h->blocks[(size_t)i];
    const int above = 2 * (nb - 1 - i);
    if (h->conv_any_trained(b.b) || (b.down >= 0 && h->conv_any_trained(b.down))) phases = std::max(phases, std::max(above, 1));
    if (h->conv_any_trained(b.a)) phases = std::max(phases, above + 1);
  }
  return phases;
}

template <int K, bool WSMEM>
static int launch_bwd_data(const char* name, const BwdDataArgs& a, int groups, size_t smem, cudaStream_t s, int cluster) {
  auto kfn = conv_bwd_data_kernel<K, WSMEM>;
#ifndef TCR_EMU
  static SmemOptIn optin;           // one per template instantiation
  if (optin.ensure(kfn, smem) != cudaSuccess) return TCR_ERR_CUDA;
#endif
  TCR_LAUNCH_CLUSTER(name, kfn, dim3(groups), dim3(kThreads), smem, s, cluster, a);
  return 0;
}

static BsumSrc bsum_src(const tcr_handle* h, const ConvPlan& cv) {
  if (sync_bn_on(h) && cv.b_gc) return BsumSrc{cv.bsync, 1, cv.bsum};          // SyncBN: the sums over all ranks as one record
  return BsumSrc{cv.b_gc ? cv.bpart : nullptr, cv.b_gc, cv.bsum};
}
static DySrc make_dy(const tcr_handle* h, const ConvPlan& cv, const float* dz, int mask, int n) {
  return DySrc{dz, cv.y, cv.bnf, cv.bsum, mask, bn_inv(h, n, cv.t_out), bsum_src(h, cv)};
}

// *gc_out: per-cluster records of BatchNorm-backward sums this launch leaves for the layer(s) below (0 when recording)
static int bwd_data(tcr_handle* h, ConvPlan& cv, ConvPlan* dn, BwdDataArgs a, int n, cudaStream_t s, int* gc_out) {
  int U, KS, wsm;
  if (!pick_bwd_tile(h->sms, cv, dn, n, h->smem_optin, &U, &KS, &wsm)) {   // tcr_create refuses such a handle (net_check_envelope)
    set_error("backward-data tile does not fit in shared memory");
    return TCR_ERR_UNSUPPORTED;
  }
  a.n = n; a.U = U; a.w_smem = wsm;
  a.w = cv.wT; a.cin = cv.cin; a.cout = cv.cout; a.k = cv.k; a.stride = cv.stride;
  a.t_in = cv.t_in; a.t_out = cv.t_out; a.pad_left = cv.pad_left; a.KS = KS;
  a.has_down = dn ? 1 : 0;
  a.wd = dn ? dn->wT : nullptr;
  a.coutd = dn ? dn->cout : 0;
  const int groups = (n + U - 1) / U;
  const size_t smem = bwd_data_smem(cv, dn, U, KS, wsm != 0);
  *gc_out = 0;
  const int CL = cluster_size(h);
  const int grid = (groups + CL - 1) / CL * CL;
  *gc_out = grid / CL;
  switch (cv.k) {
    case 9: return wsm ? launch_bwd_data<9, true>(("dx:" + cv.name).c_str(), a, grid, smem, s, CL)
                       : launch_bwd_data<9, false>(("dx:" + cv.name).c_str(), a, grid, smem, s, CL);
    default: set_error("unsupported kernel width"); return TCR_ERR_UNSUPPORTED;
  }
}

// Transposed filter banks for the backward-data kernels: launched at the START of the step (it only reads params), so the
// first backward kernel can prefetch its bank before its programmatic-dependency wait.
int net_weight_transpose(tcr_handle* h, const float* params, cudaStream_t s) {
  WtArgs w;
  w.nlayers = 0;
  w.total = 0;
  w.params = params;
  for (auto& cv : h->convs) {
    if (&cv == &h->convs[0]) continue;               // conv0 needs no input gradient
    w.layer[w.nlayers++] = WtLayer{cv.w_off, cv.wT, cv.k, cv.cin, cv.cout, w.total};
    w.total += cv.wnumel();
  }
  TCR_LAUNCH("weight_transpose", weight_transpose_kernel, dim3((unsigned)((w.total + 255) / 256)), dim3(256), 0, s, w);
  return 0;
}

// BatchNorm-backward sums of one layer from the per-cluster records its producer left, published to ConvPlan::bsum.  A truncated
// backward-data chain (tcr_set_trainable) leaves the records of its lowest layers without the consumer launch that would
// publish them; this is that consumer's prologue (bsum_build with the same 256 threads, hence the same bits).
__global__ void __launch_bounds__(kThreads) bsum_publish_kernel(BsumSrc bs, int C) {
  pdl_wait();
  __shared__ float sb[kThreads], scratch[kThreads];
  bsum_build(bs, bs.bsum, C, sb, scratch, true);
}
static int publish_bsums(tcr_handle* h, int l, cudaStream_t s) {
  if (!h->conv_any_trained(l)) return 0;
  const ConvPlan& cv = h->convs[(size_t)l];
  TCR_LAUNCH("records_sum", bsum_publish_kernel, dim3(1), dim3(kThreads), 0, s, bsum_src(h, cv), cv.cout);
  return 0;
}

int net_backward_data(tcr_handle* h, const float* params, int n, cudaStream_t s) {
  const int nb = (int)h->blocks.size(), phases = h->bwd_phases;
  int done = 0;
  for (int i = nb - 1; i >= 0 && done < phases; --i) {
    BlockPlan& b = h->blocks[i];
    ConvPlan& ca = h->convs[b.a];
    ConvPlan& cb = h->convs[b.b];
    ConvPlan* dn = b.down >= 0 ? &h->convs[b.down] : nullptr;
    // (1) conv_b: dx is the gradient at relu(bn(y_a)); epilogue masks with bn(y_a) > 0 and sums for BN_a
    {
      BwdDataArgs a;
      memset(&a, 0, sizeof(a));
      a.dy = make_dy(h, cb, b.gblk, 0, n);
      a.epi_kind = 1;
      a.yp = ca.y; a.bnfp = ca.bnf; a.bpartp = ca.bpart; a.gprev = ca.g;
      int gc = 0;
      int rc = bwd_data(h, cb, nullptr, a, n, s, &gc);
      if (rc) return rc;
      ca.b_gc = gc;
      if (sync_bn_on(h) && (rc = sync_records(h, ca.bpart, gc, 2 * ca.cout, ca.bsync, s))) return rc;
    }
    if (++done == phases) {          // truncated after (1): conv_a's records and the shortcut conv's are still unpublished
      int rc = publish_bsums(h, b.a, s);
      if (!rc && b.down >= 0) rc = publish_bsums(h, b.down, s);
      return rc;
    }
    // (2) conv_a (+ down conv | identity): dx is the gradient at the block input
    {
      BwdDataArgs a;
      memset(&a, 0, sizeof(a));
      a.dy = make_dy(h, ca, ca.g, 0, n);
      if (dn) a.dyd = make_dy(h, *dn, b.gblk, 1, n);
      else a.gid = b.gblk;
      if (i > 0) {
        BlockPlan& pb = h->blocks[i - 1];
        ConvPlan& pcb = h->convs[pb.b];
        a.epi_kind = 2;
        a.out_prev = pb.out;
        a.yp = pcb.y; a.bnfp = pcb.bnf; a.bpartp = pcb.bpart;
        if (pb.down >= 0) {
          ConvPlan& pd = h->convs[pb.down];
          a.ypd = pd.y; a.bnfpd = pd.bnf; a.bpartpd = pd.bpart;
        }
        a.gprev = pb.gblk;
      } else {
        ConvPlan& c0 = h->convs[0];
        a.epi_kind = 1;
        a.yp = c0.y; a.bnfp = c0.bnf; a.bpartp = c0.bpart; a.gprev = c0.g;
      }
      int gc = 0;
      int rc = bwd_data(h, ca, dn, a, n, s, &gc);
      if (rc) return rc;
      if (i > 0) {
        BlockPlan& pb = h->blocks[i - 1];
        h->convs[pb.b].b_gc = gc;
        if (pb.down >= 0) h->convs[pb.down].b_gc = gc;
        if (sync_bn_on(h)) {
          ConvPlan& q = h->convs[pb.b];
          if ((rc = sync_records(h, q.bpart, gc, 2 * q.cout, q.bsync, s))) return rc;
          if (pb.down >= 0) {
            ConvPlan& qd = h->convs[pb.down];
            if ((rc = sync_records(h, qd.bpart, gc, 2 * qd.cout, qd.bsync, s))) return rc;
          }
        }
      } else {
        h->convs[0].b_gc = gc;
        if (sync_bn_on(h) && (rc = sync_records(h, h->convs[0].bpart, gc, 2 * h->convs[0].cout, h->convs[0].bsync, s))) return rc;
      }
    }
    if (++done == phases && i > 0) {  // truncated after (2): the previous block's conv_b / shortcut records are unpublished
      const BlockPlan& pb = h->blocks[i - 1];
      int rc = publish_bsums(h, pb.b, s);
      if (!rc && pb.down >= 0) rc = publish_bsums(h, pb.down, s);
      return rc;
    }
  }
  // conv0's records: its weight-gradient CTAs sum them (net_weight_gradients); without its weights in that launch, here
  if (phases == 2 * nb && !h->dw_conv0) return publish_bsums(h, 0, s);
  return 0;
}

// weight gradients: every layer's inputs are final now -> one grouped launch over all layers
int net_weight_gradients(tcr_handle* h, const float* feat, int n, cudaStream_t s) {
  if (h->dw_ctas == 0) return 0;     // no conv weight is trained
  if (h->dw_smem > h->smem_optin) { set_error("weight-gradient tile does not fit in shared memory"); return TCR_ERR_UNSUPPORTED; }
  {
    auto kfn = dw_grouped_kernel;
#ifndef TCR_EMU
    static SmemOptIn optin;
    if (optin.ensure(kfn, h->dw_smem) != cudaSuccess) return TCR_ERR_CUDA;
#endif
    // conv0's BatchNorm-backward sums have no backward-data consumer: its weight-gradient CTAs add the records themselves.
    // Row 0 of a table without conv0 is a layer whose sums are published: it reads them like every other row.
    const ConvPlan& c0 = h->convs[0];
    const BsumSrc bs0 = h->dw_conv0 ? bsum_src(h, c0) : BsumSrc{nullptr, 0, nullptr};
    const float inv_scale = sync_bn_on(h) ? 1.0f / (float)h->world : 1.0f;         // SyncBN: BatchNorm-backward means over the global rows
    TCR_LAUNCH("dw_grouped", kfn, dim3(h->dw_ctas), dim3(kDwThreads), h->dw_smem, s, h->d_dw_layers, h->n_dw_layers, n, feat, h->d_timeline, bs0,
               inv_scale);
  }
  return 0;
}

}  // namespace tcr
