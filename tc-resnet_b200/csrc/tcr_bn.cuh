// tcr_bn.cuh — BatchNorm table helpers shared by forward and backward kernels.
// bnf layout: [4][C] = mean, rstd, scale (= gamma * rstd), beta.
#pragma once
#include "tcr_device.cuh"
#include "tcr_internal.h"

namespace tcr {

__device__ __forceinline__ float4 relu4(float4 v) {
  return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
}
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// z = (y - mean) * scale + beta
__device__ __forceinline__ float4 bn_apply4(float4 y, const float* __restrict__ bnf, int C, int c) {
  const float4 mean = ldc4(bnf + c), scale = ldc4(bnf + 2 * C + c), beta = ldc4(bnf + 3 * C + c);
  return make_float4(fmaf(y.x - mean.x, scale.x, beta.x), fmaf(y.y - mean.y, scale.y, beta.y),
                     fmaf(y.z - mean.z, scale.z, beta.z), fmaf(y.w - mean.w, scale.w, beta.w));
}
__device__ __forceinline__ float bn_apply1(float y, const float* __restrict__ bnf, int C, int c) {
  return fmaf(y - ldc1(bnf + c), ldc1(bnf + 2 * C + c), ldc1(bnf + 3 * C + c));
}
// xhat = (y - mean) * rstd
__device__ __forceinline__ float4 bn_xhat4(float4 y, const float* __restrict__ bnf, int C, int c) {
  const float4 mean = ldc4(bnf + c), rstd = ldc4(bnf + C + c);
  return make_float4((y.x - mean.x) * rstd.x, (y.y - mean.y) * rstd.y, (y.z - mean.z) * rstd.z, (y.w - mean.w) * rstd.w);
}

// Activation source: raw tensor or relu(bn(y)).
__device__ __forceinline__ float4 act_load4(const ActSrc& s, size_t ofs, int C, int c) {
  float4 v = ld4(s.data + ofs);
  if (s.kind == 1) v = relu4(bn_apply4(v, s.bnf, C, c));
  return v;
}

// dy = scale * (dz - s1/M - xhat * s2/M); dz optionally masked by the layer's own ReLU (bn(y) > 0).
__device__ __forceinline__ float4 dy_load4(const DySrc& d, size_t ofs, int C, int c) {
  float4 dz = ld4(d.dz + ofs);
  const float4 y = ld4(d.y + ofs);
  const float4 mean = ldc4(d.bnf + c), rstd = ldc4(d.bnf + C + c), scale = ldc4(d.bnf + 2 * C + c);
  if (d.mask_relu) {
    const float4 beta = ldc4(d.bnf + 3 * C + c);
    if (fmaf(y.x - mean.x, scale.x, beta.x) <= 0.f) dz.x = 0.f;
    if (fmaf(y.y - mean.y, scale.y, beta.y) <= 0.f) dz.y = 0.f;
    if (fmaf(y.z - mean.z, scale.z, beta.z) <= 0.f) dz.z = 0.f;
    if (fmaf(y.w - mean.w, scale.w, beta.w) <= 0.f) dz.w = 0.f;
  }
  const float4 s1 = ldc4(d.bsum + c), s2 = ldc4(d.bsum + C + c);
  const float im = d.inv_m;
  float4 r;
  r.x = scale.x * (dz.x - s1.x * im - (y.x - mean.x) * rstd.x * (s2.x * im));
  r.y = scale.y * (dz.y - s1.y * im - (y.y - mean.y) * rstd.y * (s2.y * im));
  r.z = scale.z * (dz.z - s1.z * im - (y.z - mean.z) * rstd.z * (s2.z * im));
  r.w = scale.w * (dz.w - s1.w * im - (y.w - mean.w) * rstd.w * (s2.w * im));
  return r;
}

// ---- per-channel constants hoisted into registers -------------------------------------------------
// Staging loops give every thread a FIXED group of 4 channels and walk rows, so the BN table entries (and the
// BN-backward sums) are loaded once per thread instead of once per element.
struct Chan4 { float4 mean, rstd, scale, beta; };
__device__ __forceinline__ Chan4 chan4_load(const float* __restrict__ bnf, int C, int c) {
  Chan4 k;
  k.mean = ldc4(bnf + c); k.rstd = ldc4(bnf + C + c); k.scale = ldc4(bnf + 2 * C + c); k.beta = ldc4(bnf + 3 * C + c);
  return k;
}
__device__ __forceinline__ Chan4 chan4_load_s(const float* tbl, int C, int c) {       // table in shared memory
  Chan4 k;
  k.mean = ld4(tbl + c); k.rstd = ld4(tbl + C + c); k.scale = ld4(tbl + 2 * C + c); k.beta = ld4(tbl + 3 * C + c);
  return k;
}
__device__ __forceinline__ float4 chan4_bn(const Chan4& k, float4 y) {
  return make_float4(fmaf(y.x - k.mean.x, k.scale.x, k.beta.x), fmaf(y.y - k.mean.y, k.scale.y, k.beta.y),
                     fmaf(y.z - k.mean.z, k.scale.z, k.beta.z), fmaf(y.w - k.mean.w, k.scale.w, k.beta.w));
}
__device__ __forceinline__ float4 chan4_xhat(const Chan4& k, float4 y) {
  return make_float4((y.x - k.mean.x) * k.rstd.x, (y.y - k.mean.y) * k.rstd.y, (y.z - k.mean.z) * k.rstd.z, (y.w - k.mean.w) * k.rstd.w);
}
// activation source with hoisted constants
struct Act4 { const float* data; Chan4 k; int kind; };
__device__ __forceinline__ Act4 act4_make(const ActSrc& s, int C, int c, const float* tbl) {
  Act4 a;
  a.data = s.data; a.kind = s.kind;
  if (s.kind == 1) a.k = chan4_load_s(tbl, C, c);
  return a;
}
__device__ __forceinline__ float4 act4_load(const Act4& a, size_t ofs) {
  float4 v = ld4(a.data + ofs);
  if (a.kind == 1) v = relu4(chan4_bn(a.k, v));
  return v;
}
// dy = scale * (dz - s1/M - xhat * s2/M) with hoisted constants
struct Dy4 { const float* dz; const float* y; Chan4 k; float4 s1m, s2m; int mask; };
__device__ __forceinline__ Dy4 dy4_make(const DySrc& d, int C, int c, const float* sb) {   // sb: [2][C] sums in shared memory
  Dy4 r;
  r.dz = d.dz; r.y = d.y; r.mask = d.mask_relu;
  r.k = chan4_load(d.bnf, C, c);
  const float4 s1 = ld4(sb + c), s2 = ld4(sb + C + c);
  const float im = d.inv_m;
  r.s1m = make_float4(s1.x * im, s1.y * im, s1.z * im, s1.w * im);
  r.s2m = make_float4(s2.x * im, s2.y * im, s2.z * im, s2.w * im);
  return r;
}
__device__ __forceinline__ float4 dy4_apply(const Dy4& d, float4 dz, const float4 y) {
  if (d.mask) {
    const float4 z = chan4_bn(d.k, y);
    if (z.x <= 0.f) dz.x = 0.f;
    if (z.y <= 0.f) dz.y = 0.f;
    if (z.z <= 0.f) dz.z = 0.f;
    if (z.w <= 0.f) dz.w = 0.f;
  }
  float4 r;
  r.x = d.k.scale.x * (dz.x - d.s1m.x - (y.x - d.k.mean.x) * d.k.rstd.x * d.s2m.x);
  r.y = d.k.scale.y * (dz.y - d.s1m.y - (y.y - d.k.mean.y) * d.k.rstd.y * d.s2m.y);
  r.z = d.k.scale.z * (dz.z - d.s1m.z - (y.z - d.k.mean.z) * d.k.rstd.z * d.s2m.z);
  r.w = d.k.scale.w * (dz.w - d.s1m.w - (y.w - d.k.mean.w) * d.k.rstd.w * d.s2m.w);
  return r;
}
__device__ __forceinline__ float4 dy4_load(const Dy4& d, size_t ofs) { return dy4_apply(d, ld4(d.dz + ofs), ld4(d.y + ofs)); }

// 2-D walk of a [rows][c4n] float4 grid by the CTA: c4 fixed per thread, rows advance by rstep.
// Threads beyond rstep * c4n idle (row = huge).
struct RowWalk { int c4, row, rstep; };
__device__ __forceinline__ RowWalk row_walk(int tid, int nthreads, int c4n) {
  RowWalk w;
  w.rstep = nthreads / c4n;
  w.c4 = tid % c4n;
  w.row = tid / c4n;
  if (w.row >= w.rstep) w.row = 1 << 29;
  return w;
}

// ---- cross-CTA BatchNorm statistics: cluster reduce in the producer, table in the consumer -------------------------
// Producer: every CTA leaves its per-channel partial sums in its OWN shared memory; the CTAs of a thread-block cluster add
// them through distributed shared memory (rank order) and write one record per cluster, part[cluster][cols].  No atomics,
// no fences, no "last CTA" tail: the kernel ends when its tiles are done.  (A launch without a cluster dimension is a
// cluster of one: one record per CTA, which is what the persistent kernel's finalize phases read.)
// Consumer: the next kernel sums the <= 32..64 records per channel in its prologue (every CTA, redundantly, from L2) and
// keeps the finished table in shared memory; CTA 0 also publishes it for the kernels further down the stream.
// Everything is summed in a fixed order, so the step stays bit-reproducible.
struct PubSeg { const float* sp; int n; float* g; };   // shared-memory partials, column count, global records [cluster][n]
template <int NSEG>
__device__ __forceinline__ void cluster_publish(const PubSeg (&seg)[NSEG], int vb) {
  cluster_sync_all();
  const int CL = (int)cluster_nctarank(), r = (int)cluster_ctarank();
  const int cid = vb / CL;
  int total = 0;
#pragma unroll
  for (int k = 0; k < NSEG; ++k) total += seg[k].n;
  for (int col = r + CL * (int)threadIdx.x; col < total; col += CL * (int)blockDim.x) {
    int k = 0, c = col;
#pragma unroll
    for (int j = 0; j < NSEG - 1; ++j)
      if (k == j && c >= seg[j].n) { c -= seg[j].n; k = j + 1; }
    const float* sp = seg[k].sp + c;
    float s = 0.f;
    if (CL == 8) {
      s = sum_dsmem8(sp);
    } else {
      for (int q = 0; q < CL; ++q) s += ld_dsmem(sp, (unsigned)q);
    }
    seg[k].g[(size_t)cid * seg[k].n + c] = s;
  }
  cluster_sync_all();               // nobody exits (and releases its shared memory) while a peer may still read it
}

// ---- record sums and their per-channel finalisation, shared by the per-layer and the resident kernels ----------------------
__device__ __forceinline__ float rec_ld(const float* p, float) { return __ldcg(p); }
__device__ __forceinline__ float4 rec_ld(const float* p, float4) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float rec_add(float a, float b) { return a + b; }
__device__ __forceinline__ float4 rec_add(float4 a, float4 b) { return add4(a, b); }

// Sum of records ch, ch + nch, ch + 2 nch, ... < G of column `col` (V = float) or of the four columns from `col` (V = float4) of
// records `stride` floats apart, in a fixed order; DEPTH loads of a thread are in flight at once.
template <class V, int DEPTH>
__device__ __forceinline__ V rec_column_sum(const float* p, int col, int stride, int ch, int nch, int G) {
  V s = V{};
  for (int g0 = ch; g0 < G; g0 += DEPTH * nch) {
    V v[DEPTH];
#pragma unroll
    for (int j = 0; j < DEPTH; ++j) {
      const int g = g0 + j * nch;
      v[j] = g < G ? rec_ld(p + (size_t)g * stride + col, V{}) : V{};
    }
#pragma unroll
    for (int j = 0; j < DEPTH; ++j) s = rec_add(s, v[j]);
  }
  return s;
}

// One BatchNorm channel from the nch chunk sums of its (sum y, sum y^2) at scratch[ch * cols + col + {0,1}]: mean, variance and
// rstd in fp64, the table entry tbl[4][C] (mean, rstd, gamma * rstd, beta) and, with `publish`, the global table and variance.
__device__ __forceinline__ void bn_channel_finalize(const float* scratch, int cols, int col, int nch, float inv_m, float eps, float gamma,
                                                    float beta, int C, int c, float* tbl, float* bnf, float* var, bool publish) {
  double s1 = 0.0, s2 = 0.0;
  for (int ch = 0; ch < nch; ++ch) {
    s1 += (double)scratch[ch * cols + col];
    s2 += (double)scratch[ch * cols + col + 1];
  }
  const double mean = s1 * (double)inv_m;
  double v = s2 * (double)inv_m - mean * mean;
  if (v < 0.0) v = 0.0;
  const double rstd = 1.0 / sqrt(v + (double)eps);
  const float fm = (float)mean, fr = (float)rstd, fs = (float)((double)gamma * rstd);
  tbl[c] = fm; tbl[C + c] = fr; tbl[2 * C + c] = fs; tbl[3 * C + c] = beta;
  if (publish) {
    bnf[c] = fm; bnf[C + c] = fr; bnf[2 * C + c] = fs; bnf[3 * C + c] = beta;
    var[c] = (float)v;
  }
}

// One BatchNorm-backward sum (record column j = c*2 + q) from its nch chunk sums at scratch[ch * cols + i] -> sb[q][C] and, with
// `publish`, the global bsum[q][C].
__device__ __forceinline__ void bsum_finalize(const float* scratch, int cols, int i, int nch, int j, int C, float* sb, float* bsum, bool publish) {
  double s = 0.0;
  for (int ch = 0; ch < nch; ++ch) s += (double)scratch[ch * cols + i];
  const float f = (float)s;
  sb[(j & 1) * C + (j >> 1)] = f;
  if (publish) bsum[(j & 1) * C + (j >> 1)] = f;
}

// Sum `gc` records of `cols` floats each: thread i < cols * nch takes column i % cols and records i / cols, + nch, ...
// (loads batched kRecB deep); the nch chunk sums land in scratch[chunk * cols + col].  Needs cols <= blockDim.x.
constexpr int kRecB = 32;          // records in flight per thread: one batch covers 32 records x column chunks
__device__ __forceinline__ int records_sum(const float* part, int gc, int cols, float* scratch) {
  const int nch = imax(1, (int)blockDim.x / cols);
  const int i = threadIdx.x;
  if (i < cols * nch) {
    const int col = i % cols, ch = i / cols;
    scratch[ch * cols + col] = rec_column_sum<float, kRecB>(part, col, cols, ch, nch, gc);
  }
  return nch;
}

// BN table of one layer in shared memory tbl[4][C] (mean, rstd, scale, beta).  st.cpart == nullptr: the global table is
// already final (persistent kernel / eval tables) and is only copied.  Block-wide; ends with __syncthreads().
__device__ __forceinline__ void bn_table_build(const StatSrc& st, const float* bnf_global, int C, float* tbl, float* scratch, bool publish) {
  if (!st.cpart) {
    for (int i = threadIdx.x; i < 4 * C; i += blockDim.x) tbl[i] = ldc1(bnf_global + i);
    __syncthreads();
    return;
  }
  const int nch = records_sum(st.cpart, st.gc, 2 * C, scratch);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    bn_channel_finalize(scratch, 2 * C, 2 * c, nch, st.inv_m, st.eps, st.gamma[c], st.beta[c], C, c, tbl, st.bnf, st.var, publish);
  __syncthreads();
}

// Two tables of the same width (a block's conv_b and its shortcut conv) in ONE pass: the record loads of both layers are in
// flight together and the two barriers are shared.  Falls back to two passes when 4C columns exceed the block.
__device__ __forceinline__ void bn_table_build2(const StatSrc& sa, const float* bnf_a, float* tbl_a, const StatSrc& sb, const float* bnf_b,
                                                float* tbl_b, int C, float* scratch, bool publish) {
  const int cols = 4 * C;
  if (!sa.cpart || !sb.cpart || cols > (int)blockDim.x) {
    bn_table_build(sa, bnf_a, C, tbl_a, scratch, publish);
    bn_table_build(sb, bnf_b, C, tbl_b, scratch, publish);
    return;
  }
  const int nch = (int)blockDim.x / cols;
  const int i = threadIdx.x;
  if (i < cols * nch) {
    const int col = i % cols, ch = i / cols;
    const bool second = col >= 2 * C;
    const StatSrc& st = second ? sb : sa;
    scratch[ch * cols + col] = rec_column_sum<float, kRecB>(st.cpart, second ? col - 2 * C : col, 2 * C, ch, nch, st.gc);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * C; j += blockDim.x) {
    const bool second = j >= C;
    const int c = second ? j - C : j;
    const StatSrc& st = second ? sb : sa;
    bn_channel_finalize(scratch, cols, (second ? 2 * C : 0) + 2 * c, nch, st.inv_m, st.eps, st.gamma[c], st.beta[c], C, c,
                        second ? tbl_b : tbl_a, st.bnf, st.var, publish);
  }
  __syncthreads();
}

// BN-backward sums of one layer in shared memory sb[2][C] (sum dz, sum dz*xhat), same conventions.
__device__ __forceinline__ void bsum_build(const BsumSrc& bs, const float* bsum_global, int C, float* sb, float* scratch, bool publish) {
  if (!bs.cpart) {
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sb[i] = ldc1(bsum_global + i);
    __syncthreads();
    return;
  }
  const int nch = records_sum(bs.cpart, bs.gc, 2 * C, scratch);
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) bsum_finalize(scratch, 2 * C, i, nch, i, C, sb, bs.bsum, publish);
  __syncthreads();
}

// Per-channel (sum y, sum y^2) of a [rows][C] shared-memory tile -> part_out[c*2 + {0,1}] (shared memory), ONE pass.
// Requires C <= blockDim.x.  red: 2 * blockDim.x floats of scratch.  The cross-CTA combination is then a plain
// fixed-order sum; var = E[y^2] - mean^2 is formed once per channel in fp64 (relative error ~1e-7 (1 + mean^2/var)).
__device__ __forceinline__ void tile_stats(const float* tile, int rows, int C, float* red, float* part_out) {
  const int tid = threadIdx.x;
  const int ns = imax(1, (int)blockDim.x / C);
  const int seg = tid / C, c = tid - seg * C;
  const bool act = seg < ns;
  if (act) {
    float s1 = 0.f, s2 = 0.f;
    for (int r = seg; r < rows; r += ns) {
      const float v = tile[r * C + c];
      s1 += v;
      s2 = fmaf(v, v, s2);
    }
    red[seg * C + c] = s1;
    red[blockDim.x + seg * C + c] = s2;
  }
  __syncthreads();
  if (tid < 2 * C) {
    const int q = tid / C, cc = tid - q * C;
    float tot = 0.f;
    for (int k = 0; k < ns; ++k) tot += red[q * blockDim.x + k * C + cc];
    part_out[(size_t)cc * 2 + q] = tot;
  }
  __syncthreads();
}

}  // namespace tcr
