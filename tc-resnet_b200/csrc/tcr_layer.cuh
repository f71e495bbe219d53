// tcr_layer.cuh — the layer computations of TC-ResNet, written once for both kernel paths: the per-layer kernels
// (tcr_net_fwd.cu, tcr_net_bwd.cu: 256 threads, one launch per layer) inline them, and the resident kernels (tcr_resident.cu:
// 512 threads, one launch per pass) call them from their non-inlined phase functions.  NT is the thread count of the CTA.
#pragma once
#include "tcr_bn.cuh"

namespace tcr {

__device__ __forceinline__ float4 mask_pos4(float4 v, float4 z) {
  return make_float4(z.x > 0.f ? v.x : 0.f, z.y > 0.f ? v.y : 0.f, z.z > 0.f ? v.z : 0.f, z.w > 0.f ? v.w : 0.f);
}
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }

// Zero the pad rows of a padded tile [Ue][TP][CS]: rows [0, pad_left) and the npad - pad_left rows after the t data rows.
__device__ __forceinline__ void zero_pad_rows(float* tile, int Ue, int t, int c4n, int TP, int CS, int pad_left, int npad, int nthreads) {
  for (int idx = threadIdx.x; idx < Ue * npad * c4n; idx += nthreads) {
    const int c4 = idx % c4n, pr = (idx / c4n) % npad, u = idx / (c4n * npad);
    const int row = pr < pad_left ? pr : t + pr;
    st4(tile + ((size_t)(u * TP + row) * CS + 4 * c4), make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

// Offset in the filter bank w[k][cin][cout] of entry i of its transpose wT[k][cout][ci] (the backward-data layout).
// (k from i / (cin * cout), not from i / cin: the latter costs weight_transpose_kernel two registers.)
template <class I>
__device__ __forceinline__ int64_t wT_source(I i, int cin, int cout) {
  const int ci = (int)(i % cin), co = (int)((i / cin) % cout), k = (int)(i / ((I)cin * cout));
  return ((int64_t)k * cin + ci) * cout + co;
}

// Where the FMA loops read a filter bank (main conv, and the block's 1x1 shortcut conv) from.  Shared memory: 32-bit float
// offsets from the shared-memory base, so the inner loop is LDS.128 + FFMA + integer adds.  Global: LDG.128 through L1/L2, with
// 64-bit offsets to the tap's slice (Off).
struct WShared {
  using Ptr = int; using Off = int;
  const float* smem; int main, down;
  __device__ __forceinline__ Ptr bank(bool is_down) const { return is_down ? down : main; }
  __device__ __forceinline__ float4 ld(Ptr p) const { return ld4(smem + p); }
};
struct WGlobal {
  using Ptr = const float*; using Off = size_t;
  const float* main; const float* down;
  __device__ __forceinline__ Ptr bank(bool is_down) const { return is_down ? down : main; }
  __device__ __forceinline__ float4 ld(Ptr p) const { return ldg4(p); }
};

// ------------------------------------------------------------------------------------------------
// Forward conv, register-tiled: task = (k-slice, row tile of TM, 4 output channels) of the [K,1] conv of the padded tile
// x [U][TP][CS] (at float offset xs_off), then tasks of the 1x1/stride-2 shortcut conv (coutd > 0) from the same tile.
// Output: k-slice planes ys [KS][rcap][cout], shortcut output ysd [R][coutd].
// ------------------------------------------------------------------------------------------------
template <int K, int TM, int NT, class W>
__device__ __forceinline__ void conv_fwd_tasks(const float* smem, const W& w, int xs_off, float* ys, float* ysd, int rcap, int R, int cin,
                                               int cout, int coutd, int stride, int t_out, int TP, int CS, int pad_left, int KS) {
  const int NRT = (R + TM - 1) / TM;
  const int NCG = cout >> 2;
  const int KPS = K / KS;
  const int ntasks = NRT * NCG * KS;
  const int NCGD = coutd >> 2;
  const int ntasks_all = ntasks + NRT * NCGD;
  for (int task = threadIdx.x; task < ntasks_all; task += NT) {
    const bool is_down = task >= ntasks;
    const int tk = is_down ? task - ntasks : task;
    const int ncg = is_down ? NCGD : NCG;
    const int cg = tk % ncg;
    const int rt = (tk / ncg) % NRT;
    const int ks = is_down ? 0 : tk / (ncg * NRT);
    int xo[TM];
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int r = imin(rt + i * NRT, R - 1);      // rows of a task are NRT apart: adjacent lanes -> adjacent rows
      const int u = r / t_out, t = r - u * t_out;
      xo[i] = xs_off + (is_down ? (u * TP + pad_left + 2 * t) : (u * TP + t * stride)) * CS;
    }
    float4 acc[TM];
#pragma unroll
    for (int i = 0; i < TM; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int k_lo = is_down ? 0 : ks * KPS, k_hi = is_down ? 1 : k_lo + KPS;
    const int co_n = is_down ? coutd : cout;
    const typename W::Ptr wb = w.bank(is_down) + 4 * cg;
    for (int k = k_lo; k < k_hi; ++k) {
      typename W::Ptr wk = wb + (typename W::Off)k * cin * co_n;
      const int xk = k * CS;
#pragma unroll 2
      for (int ci = 0; ci < cin; ci += 4, wk += 4 * co_n) {
        const float4 w0 = w.ld(wk), w1 = w.ld(wk + co_n), w2 = w.ld(wk + 2 * co_n), w3 = w.ld(wk + 3 * co_n);
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          const float4 x = ld4(smem + xo[i] + xk + ci);
          acc[i].x = fmaf(x.x, w0.x, acc[i].x); acc[i].y = fmaf(x.x, w0.y, acc[i].y);
          acc[i].z = fmaf(x.x, w0.z, acc[i].z); acc[i].w = fmaf(x.x, w0.w, acc[i].w);
          acc[i].x = fmaf(x.y, w1.x, acc[i].x); acc[i].y = fmaf(x.y, w1.y, acc[i].y);
          acc[i].z = fmaf(x.y, w1.z, acc[i].z); acc[i].w = fmaf(x.y, w1.w, acc[i].w);
          acc[i].x = fmaf(x.z, w2.x, acc[i].x); acc[i].y = fmaf(x.z, w2.y, acc[i].y);
          acc[i].z = fmaf(x.z, w2.z, acc[i].z); acc[i].w = fmaf(x.z, w2.w, acc[i].w);
          acc[i].x = fmaf(x.w, w3.x, acc[i].x); acc[i].y = fmaf(x.w, w3.y, acc[i].y);
          acc[i].z = fmaf(x.w, w3.z, acc[i].z); acc[i].w = fmaf(x.w, w3.w, acc[i].w);
        }
      }
    }
    float* dst = is_down ? ysd : ys + ks * rcap * cout;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int r = rt + i * NRT;
      if (r < R) st4(dst + r * co_n + 4 * cg, acc[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Transposed conv (backward data), one parity class of input rows at a time, so a stride-2 conv spends no FMA on the zeros
// of the dilated gradient: input row t belongs to class p = (t + pad_left) % S and receives taps k = p + S m from dy row
// (t + pad_left - p) / S - m.  Plus the 1x1/stride-2 shortcut conv^T on even rows (coutd > 0).
// dy tile [U][TPd][COS] at dys_off (rows at PLd..), shortcut dy [U*t_out][COSD] at dysd_off, banks wT [k][cout][cin] |
// wdT [coutd][cin] -> dx planes dxs [KS][rcap][cin].
// g: the layer's shape (cin, cout, coutd, stride, t_in, t_out, pad_left, KS), read in place: the per-layer kernel passes its
// argument block, so these stay operands in the constant bank instead of taking registers.
// ------------------------------------------------------------------------------------------------
template <int K, int TMB, int NT, class W, class A>
__device__ __forceinline__ void convT_tasks(const float* smem, const W& w, const A& g, int dys_off, int dysd_off, float* dxs, int rcap, int Ue,
                                            int TPd, int PLd, int COS, int COSD) {
  const int S = g.stride;
  const int NCIG = g.cin >> 2;
  int t0[2], np[2], nrt[2];
#pragma unroll 1
  for (int p = 0; p < 2; ++p) {
    t0[p] = ((p - g.pad_left) % S + S) % S;
    np[p] = (p < S && t0[p] < g.t_in) ? (g.t_in - t0[p] + S - 1) / S : 0;
    nrt[p] = (np[p] + TMB - 1) / TMB;
  }
  const int NRTU = nrt[0] + nrt[1];
  const int NT0 = (K + S - 1) / S;
  const int MPS = (NT0 + g.KS - 1) / g.KS;
  const int ntasks = g.KS * Ue * NRTU * NCIG;
  for (int task = threadIdx.x; task < ntasks; task += NT) {
    const int cig = task % NCIG;
    int q = task / NCIG;
    const int rtu = q % NRTU;
    q /= NRTU;
    const int u = q % Ue, ks = q / Ue;
    const int p = rtu >= nrt[0] ? 1 : 0;
    const int rt = rtu - p * nrt[0];
    int dyo[TMB], tt[TMB];
#pragma unroll
    for (int i = 0; i < TMB; ++i) {
      const int j = imin(rt + i * nrt[p], np[p] - 1);   // rows of a task are nrt apart: adjacent lanes -> adjacent rows
      tt[i] = t0[p] + S * j;
      const int b = (tt[i] + g.pad_left - p) / S;
      dyo[i] = dys_off + (u * TPd + PLd + b) * COS;
    }
    float4 acc[TMB];
#pragma unroll
    for (int i = 0; i < TMB; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int NTp = (K - p + S - 1) / S;                 // taps of class p
    const int m_lo = ks * MPS, m_hi = imin(NTp, m_lo + MPS);
    for (int m = m_lo; m < m_hi; ++m) {
      // wT[k][co][ci]: lanes (adjacent cig) read adjacent float4s -> no bank conflicts
      const int dm = m * COS;
      typename W::Ptr wk = w.bank(false) + (typename W::Off)(p + S * m) * g.cout * g.cin + 4 * cig;
#pragma unroll 2
      for (int co = 0; co < g.cout; co += 4, wk += 4 * g.cin) {
        const float4 w0 = w.ld(wk), w1 = w.ld(wk + g.cin), w2 = w.ld(wk + 2 * g.cin), w3 = w.ld(wk + 3 * g.cin);
#pragma unroll
        for (int i = 0; i < TMB; ++i) {
          const float4 d = ld4(smem + dyo[i] - dm + co);
          acc[i].x = fmaf(d.x, w0.x, fmaf(d.y, w1.x, fmaf(d.z, w2.x, fmaf(d.w, w3.x, acc[i].x))));
          acc[i].y = fmaf(d.x, w0.y, fmaf(d.y, w1.y, fmaf(d.z, w2.y, fmaf(d.w, w3.y, acc[i].y))));
          acc[i].z = fmaf(d.x, w0.z, fmaf(d.y, w1.z, fmaf(d.z, w2.z, fmaf(d.w, w3.z, acc[i].z))));
          acc[i].w = fmaf(d.x, w0.w, fmaf(d.y, w1.w, fmaf(d.z, w2.w, fmaf(d.w, w3.w, acc[i].w))));
        }
      }
    }
    if (g.coutd && ks == 0 && (t0[p] & 1) == 0) {        // 1x1 stride-2 shortcut conv touches even input rows only
      int ddo[TMB];
#pragma unroll
      for (int i = 0; i < TMB; ++i) ddo[i] = dysd_off + (u * g.t_out + (tt[i] >> 1)) * COSD;
      typename W::Ptr wk = w.bank(true) + 4 * cig;        // wdT[co][ci]
      for (int co = 0; co < g.coutd; co += 4, wk += 4 * g.cin) {
        const float4 w0 = w.ld(wk), w1 = w.ld(wk + g.cin), w2 = w.ld(wk + 2 * g.cin), w3 = w.ld(wk + 3 * g.cin);
#pragma unroll
        for (int i = 0; i < TMB; ++i) {
          const float4 d = ld4(smem + ddo[i] + co);
          acc[i].x = fmaf(d.x, w0.x, fmaf(d.y, w1.x, fmaf(d.z, w2.x, fmaf(d.w, w3.x, acc[i].x))));
          acc[i].y = fmaf(d.x, w0.y, fmaf(d.y, w1.y, fmaf(d.z, w2.y, fmaf(d.w, w3.y, acc[i].y))));
          acc[i].z = fmaf(d.x, w0.z, fmaf(d.y, w1.z, fmaf(d.z, w2.z, fmaf(d.w, w3.z, acc[i].z))));
          acc[i].w = fmaf(d.x, w0.w, fmaf(d.y, w1.w, fmaf(d.z, w2.w, fmaf(d.w, w3.w, acc[i].w))));
        }
      }
    }
#pragma unroll
    for (int i = 0; i < TMB; ++i)
      if (rt + i * nrt[p] < np[p]) st4(dxs + ((size_t)ks * rcap + (size_t)u * g.t_in + tt[i]) * g.cin + 4 * cig, acc[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// Backward-data epilogue.  Per row: dx = sum of the k-slice planes dxs [KS][rcap][cin] (+ the identity gradient gid); g = dx
// masked by the consumer-side ReLU; (sum g, sum g*xhat) of the layer(s) below.
//   epi_kind 1: mask bn(yp) > 0, sums for that layer (table bnfp).
//   epi_kind 2: mask (previous block's output) > 0, sums for its conv_b (yp, bnfp) and, when ypd != null, for its shortcut conv
//   (ypd, bnfpd; additionally masked by bn_d(ypd) > 0).
// g goes to gprev.  nseg row segments per channel group leave their sums in red [4][nseg][cin]; the CTA's record then goes to
// rec [cin][2] (and recd [cin][2] for the shortcut conv).  No trailing barrier.
// e: gid, epi_kind, yp, bnfp, out_prev, ypd, bnfpd, gprev, cin, KS, read in place (the per-layer kernel passes its argument block).
// Global row tensors are indexed from row row0.  RESIDENT (the resident kernel: tensors and tables in shared memory, rows from 0):
// the tables are read from shared memory, g is also kept in gdst, and with a shortcut conv below the block output is recomputed
// exactly as the forward pass formed it, bn_b(yp) + relu(bn_d(ypd)), instead of being read from out_prev.
// ------------------------------------------------------------------------------------------------
template <int NT, bool RESIDENT, class A>
__device__ __forceinline__ void bwd_epilogue(const A& e, const float* dxs, int rcap, int Rin, int nseg, size_t row0, float* gdst, float* red,
                                             float* rec, float* recd) {
  const int tid = threadIdx.x;
  const int NCIG = e.cin >> 2;
  const int seg = tid / NCIG, cig = tid - seg * NCIG;
  const bool has_pd = e.epi_kind == 2 && e.ypd;
  float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1, sd1 = s1, sd2 = s1;
  if (seg < nseg) {
    const Chan4 kp = RESIDENT ? chan4_load_s(e.bnfp, e.cin, 4 * cig) : chan4_load(e.bnfp, e.cin, 4 * cig);
    Chan4 kpd = kp;
    if (has_pd) kpd = RESIDENT ? chan4_load_s(e.bnfpd, e.cin, 4 * cig) : chan4_load(e.bnfpd, e.cin, 4 * cig);
    for (int r = seg; r < Rin; r += nseg) {
      const size_t go = (row0 + r) * e.cin + 4 * cig;
      float4 v = ld4(dxs + (size_t)r * e.cin + 4 * cig);
      for (int ks = 1; ks < e.KS; ++ks) v = add4(v, ld4(dxs + ((size_t)ks * rcap + r) * e.cin + 4 * cig));
      if (e.gid) v = add4(v, ld4(e.gid + go));
      const float4 yv = ld4(e.yp + go);
      float4 zd = make_float4(0.f, 0.f, 0.f, 0.f);        // RESIDENT: bn_d(ypd), formed once per row (ypd itself is reloaded below:
      if (RESIDENT && has_pd) zd = chan4_bn(kpd, ld4(e.ypd + go));   // holding it across the row costs the resident kernel a spill)
      float4 g;
      if (e.epi_kind == 1) g = mask_pos4(v, chan4_bn(kp, yv));
      else if (RESIDENT && has_pd) g = mask_pos4(v, add4(chan4_bn(kp, yv), relu4(zd)));
      else g = mask_pos4(v, ld4(e.out_prev + go));
      if (RESIDENT) st4(gdst + (size_t)r * e.cin + 4 * cig, g);
      st4(e.gprev + go, g);
      s1 = add4(s1, g);
      s2 = add4(s2, mul4(g, chan4_xhat(kp, yv)));
      if (has_pd) {
        const float4 yd = ld4(e.ypd + go);
        const float4 gs = mask_pos4(g, RESIDENT ? zd : chan4_bn(kpd, yd));
        sd1 = add4(sd1, gs);
        sd2 = add4(sd2, mul4(gs, chan4_xhat(kpd, yd)));
      }
    }
    float* r0 = red + ((size_t)seg * e.cin + 4 * cig);
    st4(r0, s1);
    st4(r0 + (size_t)nseg * e.cin, s2);
    st4(r0 + (size_t)2 * nseg * e.cin, sd1);
    st4(r0 + (size_t)3 * nseg * e.cin, sd2);
  }
  __syncthreads();
  const int nq = has_pd ? 4 : 2;
  for (int i = tid; i < nq * e.cin; i += NT) {
    const int qd = i / e.cin, c = i - qd * e.cin;
    float s = 0.f;
    for (int sg = 0; sg < nseg; ++sg) s += red[((size_t)qd * nseg + sg) * e.cin + c];
    ((qd >> 1) ? recd : rec)[c * 2 + (qd & 1)] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Head on the CTA's nu utterances once the block output so [nu*T][C] is in shared memory: average pool, dropout, fc (no bias),
// softmax cross-entropy; with `backward` also the head backward: dlogits -> fc^T, dropout, AvgPoolGrad -> gradient at the block
// output (gout [nu*T][C]), the BatchNorm-backward sums of conv_b (raw output syb, table tb) and of the shortcut conv (raw output
// syd, table td; null for an identity shortcut), and the fc weight-gradient record dwfc [C][NC].  The CTA's [4C + 1] sums are left
// in sp: conv_b (c*2+q), shortcut conv (c*2+q), cross-entropy; the caller publishes them.  The fc weights are in hs.wfc.
// A: the call's arguments (onehot, mask, seed, keep, use_dropout, label_smoothing, logits, probs, inv_n).
// ------------------------------------------------------------------------------------------------
struct HeadSmem { float* wfc; float* drop; float* mk; float* dnet; float* logit; float* dl; float* loss; float* red; };

template <int NT, class A>
__device__ __forceinline__ void head_tail(const A& a, const HeadSmem& hs, int C, int T, int NC, int u0, int nu, const float* so,
                                          const float* syb, const float* syd, const float* tb, const float* td, bool backward, float* gout,
                                          float* sp, float* dwfc) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rows = nu * T;
  // average pool + dropout
#pragma unroll 1
  for (int i = tid; i < nu * C; i += NT) {
    const int u = i / C, cc = i - u * C;
    float acc = 0.f;
    for (int t = 0; t < T; ++t) acc += so[(u * T + t) * C + cc];
    const float pooled = acc / (float)T;
    float mk = 1.f, dropped = pooled;
    if (a.use_dropout) {
      const size_t gi = (size_t)(u0 + u) * C + cc;
      mk = a.mask ? a.mask[gi] : floorf(a.keep + uniform01(a.seed, (uint64_t)gi));
      dropped = pooled / a.keep * mk;                       // tf.nn.dropout: x / keep_prob * floor(keep_prob + U)
    }
    hs.drop[i] = dropped;
    hs.mk[i] = mk;
  }
  __syncthreads();
  // fc: one warp per (utterance, class)
#pragma unroll 1
  for (int o = warp; o < nu * NC; o += NT / 32) {
    const int u = o / NC, k = o - u * NC;
    float p = 0.f;
    for (int cc = lane; cc < C; cc += 32) p = fmaf(hs.drop[u * C + cc], hs.wfc[cc * NC + k], p);
    p = warp_sum(p);
    if (lane == 0) hs.logit[o] = p;
  }
  __syncthreads();
  // softmax cross-entropy: one warp per utterance, lane k keeps class k (NC <= 32)
#pragma unroll 1
  for (int u = warp; u < nu; u += NT / 32) {
    const bool act = lane < NC;
    const float logit = act ? hs.logit[u * NC + lane] : 0.f;
    const float mx = warp_max(act ? logit : -3.0e38f);
    const float e = act ? expf(logit - mx) : 0.f;
    const float se = warp_sum(e);
    const float prob = e / se;
    const float logp = (logit - mx) - logf(se);
    const size_t gi = (size_t)(u0 + u) * NC + lane;
    if (act) {
      if (a.logits) a.logits[gi] = logit;
      if (a.probs) a.probs[gi] = prob;
    }
    float loss_n = 0.f, dl = 0.f;
    if (a.onehot) {
      float lab = act ? a.onehot[gi] : 0.f;
      if (a.label_smoothing > 0.f && act) lab = lab * (1.f - a.label_smoothing) + a.label_smoothing / (float)NC;
      const float labsum = warp_sum(lab);
      loss_n = -warp_sum(act ? lab * logp : 0.f);
      dl = act ? (prob * labsum - lab) * a.inv_n : 0.f;
    }
    if (act) hs.dl[u * NC + lane] = dl;
    if (lane == 0) hs.loss[u] = loss_n;
  }
  __syncthreads();
  if (!backward) return;

  // d logits -> d pooled (fc^T, dropout, AvgPoolGrad)
#pragma unroll 1
  for (int i = tid; i < nu * C; i += NT) {
    const int u = i / C, cc = i - u * C;
    float d = 0.f;
    for (int k = 0; k < NC; ++k) d = fmaf(hs.dl[u * NC + k], hs.wfc[cc * NC + k], d);
    if (a.use_dropout) d = d / a.keep * hs.mk[i];
    hs.dnet[i] = d / (float)T;
  }
  __syncthreads();
  // gradient at the block output and the BN-backward partial sums: thread (seg, c) walks rows seg, seg + SEG, ...
  const int SEG = NT / C;
  const int seg = tid / C, c = tid - seg * C;
  if (seg < SEG) {
    float sb1 = 0.f, sb2 = 0.f, sd1 = 0.f, sd2 = 0.f;
    const float mb_ = tb[c], rb_ = tb[C + c];
    const float md_ = syd ? td[c] : 0.f, rd_ = syd ? td[C + c] : 0.f, sd_ = syd ? td[2 * C + c] : 0.f, bd_ = syd ? td[3 * C + c] : 0.f;
#pragma unroll 1
    for (int r = seg; r < rows; r += SEG) {
      const int u = r / T;
      const float g = so[r * C + c] > 0.f ? hs.dnet[u * C + c] : 0.f;
      gout[r * C + c] = g;
      sb1 += g;
      sb2 = fmaf(g, (syb[r * C + c] - mb_) * rb_, sb2);
      if (syd) {
        const float yd = syd[r * C + c];
        const float gs = fmaf(yd - md_, sd_, bd_) > 0.f ? g : 0.f;
        sd1 += gs;
        sd2 = fmaf(gs, (yd - md_) * rd_, sd2);
      }
    }
    hs.red[(0 * SEG + seg) * C + c] = sb1;
    hs.red[(1 * SEG + seg) * C + c] = sb2;
    hs.red[(2 * SEG + seg) * C + c] = sd1;
    hs.red[(3 * SEG + seg) * C + c] = sd2;
  }
  __syncthreads();
#pragma unroll 1
  for (int i = tid; i < 4 * C; i += NT) {
    const int q = i / C, cc = i - q * C;
    float s = 0.f;
    for (int k = 0; k < SEG; ++k) s += hs.red[(q * SEG + k) * C + cc];
    sp[(q >> 1) * 2 * C + cc * 2 + (q & 1)] = s;
  }
  if (tid == 0) {
    float s = 0.f;
    for (int u = 0; u < nu; ++u) s += hs.loss[u];
    sp[4 * C] = s;
  }
#pragma unroll 1
  for (int i = tid; i < C * NC; i += NT) {
    const int cc = i / NC, k = i - cc * NC;
    float s = 0.f;
    for (int u = 0; u < nu; ++u) s = fmaf(hs.drop[u * C + cc], hs.dl[u * NC + k], s);
    if (nu > 0) dwfc[i] = s;                              // cluster-padding CTAs own no record
  }
}

}  // namespace tcr
