// tcr_metrics.cu — the evaluation consumer right behind the forward pass, on the device (SURVEY.md 8f row 3).
//
// The reference's evaluator pulls `predictions_onehot` [num_samples, classes] and the labels to the host after every batch
// (helper/base.py:52-143, metrics/parser.py:135-147) and computes accuracy / top-5 / precision / recall / F1 / the classification
// report with sklearn (metrics/ops/non_tensor_ops.py:64-142, :146-295, :346-).  All of these are functions of the confusion
// matrix plus one top-k counter, so the batch is reduced to classes^2 + 2 integers where the scores already are:
//   counts[y * C + p] += 1     y = arg-max of the one-hot label row, p = arg-max of the score row (first maximum, like np.argmax)
//   counts[C * C]     += 1     when the true class ranks among the top k scores (ties broken by the lower class index)
//   counts[C * C + 1] += 1     per utterance
// Integer atomics: exact and order-independent, so the result is bit-identical to the host computation.
#include "tcr_device.cuh"
#include "tcr_net.h"

#include <algorithm>
#include <climits>

namespace tcr {

__global__ void __launch_bounds__(256) eval_accumulate_kernel(const float* __restrict__ scores, const float* __restrict__ onehot, int n, int C,
                                                              int topk, unsigned long long* counts) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = scores + (size_t)i * C;
  const float* l = onehot + (size_t)i * C;
  int y = 0, p = 0;
  float ly = l[0], sp = s[0];
  for (int c = 1; c < C; ++c) {
    if (l[c] > ly) { ly = l[c]; y = c; }
    if (s[c] > sp) { sp = s[c]; p = c; }
  }
  const float sy = s[y];
  int rank = 0;                       // classes ranked before the true one by a stable descending sort
  for (int c = 0; c < C; ++c) rank += (s[c] > sy || (s[c] == sy && c < y)) ? 1 : 0;
  atomicAdd(counts + (size_t)y * C + p, 1ull);
  if (rank < topk) atomicAdd(counts + (size_t)C * C, 1ull);
  atomicAdd(counts + (size_t)C * C + 1, 1ull);
}

int eval_accumulate_launch(const float* scores, const float* onehot, int n, int classes, int topk, int64_t* counts, cudaStream_t s) {
  TCR_LAUNCH("eval_accumulate", eval_accumulate_kernel, dim3((n + 255) / 256), dim3(256), 0, s, scores, onehot, n, classes, topk,
             reinterpret_cast<unsigned long long*>(counts));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Ranking metrics: the reference's MAPMetricOp (average_precision_score at macro / micro / weighted / samples) and APMetricOp
// (per-class AP), metrics/ops/non_tensor_ops.py:15-61, :296-343, on the softmax outputs (metrics/parser.py:135-147).
//
// eval_collect_kernel appends a batch of scores and label indices to a caller-owned store; eval_rank ranks the n stored rows once:
//   1. every (row, class) pair becomes one 64-bit item: [63:32] a key whose ascending order is the descending score order (+0 and -0
//      one key, like np.diff; every NaN one key, ranked first), [5:1] the class, [0] whether the class is the row's label;
//   2. an LSD radix sort (stable, 8-bit digits, one tile of 2,048 items per CTA) over the four key bytes gives the micro ranking
//      (one segment of n * classes), and one more stable pass over the class gives every class's ranking (classes segments of n);
//   3. per ranking, an exclusive scan of (group start, positive) pairs gives, at the end of each group of equal scores, the group's
//      positives and the cumulative positives and rank, so the group adds positives_g * TP_g / N_g (sklearn's sum of
//      (R_g - R_{g-1}) * P_g times the segment's positives); the group's first item records the cumulative positives before it;
//   4. the sums run in fixed chunks with a fixed reduction tree, then one fixed-order reduction per segment.
// Every intermediate depends only on the multiset of stored pairs, so the result is bit-identical however the rows were collected.
namespace {

constexpr int kRankThreads = 256;
constexpr int kRadixItems = 8;
constexpr int kRadixTile = kRankThreads * kRadixItems;   // items per CTA of a radix pass
constexpr int kScanItems = 16;
constexpr int kScanChunk = kRankThreads * kScanItems;    // elements per CTA of the exclusive scan
constexpr int kSumChunk = kRankThreads * 32;             // items (or rows) per CTA of the AP sums

__device__ __forceinline__ uint32_t rank_key(float x) {
  if (x != x) return 0u;
  uint32_t b = __float_as_uint(x == 0.0f ? 0.0f : x);
  b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);       // ascending in x
  return ~b;                                              // ascending in -x; no number maps to 0
}

__device__ __forceinline__ uint32_t item_key(uint64_t it) { return (uint32_t)(it >> 32); }

// fixed-order sum over the CTA: thread partials, then a fixed shuffle tree per warp, then warp totals in order
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double warp_sum[kRankThreads / 32];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = v;
  __syncthreads();
  double total = 0.0;
  for (int w = 0; w < kRankThreads / 32; ++w) total += warp_sum[w];
  __syncthreads();
  return total;
}

}  // namespace

__global__ void __launch_bounds__(256) eval_collect_kernel(const float* __restrict__ scores, const float* __restrict__ onehot, int n, int C,
                                                           float* __restrict__ store, int* __restrict__ labels) {
  pdl_wait();
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * C) return;
  store[e] = scores[e];
  if (e % C) return;
  const float* l = onehot + e;
  int y = 0;
  float ly = l[0];
  for (int c = 1; c < C; ++c)
    if (l[c] > ly) { ly = l[c]; y = c; }
  labels[e / C] = y;
}

__global__ void __launch_bounds__(256) rank_items_kernel(const float* __restrict__ store, const int* __restrict__ labels, int64_t L, int C,
                                                         uint64_t* __restrict__ items) {
  pdl_wait();
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= L) return;
  const int c = (int)(e % C);
  items[e] = ((uint64_t)rank_key(store[e]) << 32) | ((uint64_t)c << 1) | (labels[e / C] == c ? 1u : 0u);
}

// Radix pass, first half: the digit counts of one tile, digit-major (hist[d * tiles + tile]) so that one exclusive scan over the
// whole array gives every (digit, tile) its first output position.
__global__ void __launch_bounds__(256) rank_hist_kernel(const uint64_t* __restrict__ in, int64_t L, int shift, int tiles,
                                                        uint64_t* __restrict__ hist) {
  __shared__ unsigned cnt[256];
  pdl_wait();
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kRadixTile + threadIdx.x;
  for (int k = 0; k < kRadixItems; ++k) {
    const int64_t e = base + (int64_t)k * kRankThreads;
    if (e < L) atomicAdd(&cnt[(unsigned)(in[e] >> shift) & 255u], 1u);
  }
  __syncthreads();
  hist[(int64_t)threadIdx.x * tiles + blockIdx.x] = cnt[threadIdx.x];
}

// Radix pass, second half: stable scatter.  Warp w holds items [w * 256, w * 256 + 256) of the tile, 32 per step in order; an item's
// rank among equal digits is (earlier warps) + (earlier steps of its warp) + (lower lanes of its step, found with eight ballots).
__global__ void __launch_bounds__(256) rank_scatter_kernel(const uint64_t* __restrict__ in, uint64_t* __restrict__ out, int64_t L, int shift,
                                                           int tiles, const uint64_t* __restrict__ offsets) {
  __shared__ unsigned wcnt[kRankThreads / 32][256];
  pdl_wait();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < (kRankThreads / 32) * 256; i += kRankThreads) (&wcnt[0][0])[i] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kRadixTile + (int64_t)w * (32 * kRadixItems) + lane;
  const unsigned lower = (1u << lane) - 1u;
  uint64_t item[kRadixItems];
  unsigned rank[kRadixItems];
#pragma unroll
  for (int k = 0; k < kRadixItems; ++k) {
    const bool valid = base + k * 32 < L;
    item[k] = valid ? in[base + k * 32] : 0ull;
    const unsigned d = (unsigned)(item[k] >> shift) & 255u;
    unsigned peers = __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const unsigned m = __ballot_sync(0xffffffffu, (d >> b) & 1u);
      peers &= ((d >> b) & 1u) ? m : ~m;
    }
    const unsigned before = wcnt[w][d];
    rank[k] = before + __popc(peers & lower);
    __syncwarp();
    if (valid && (peers & lower) == 0) wcnt[w][d] = before + __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {
    unsigned acc = 0;
    for (int k = 0; k < kRankThreads / 32; ++k) {
      const unsigned c = wcnt[k][threadIdx.x];
      wcnt[k][threadIdx.x] = acc;
      acc += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kRadixItems; ++k) {
    if (base + k * 32 >= L) break;
    const unsigned d = (unsigned)(item[k] >> shift) & 255u;
    out[offsets[(int64_t)d * tiles + blockIdx.x] + wcnt[w][d] + rank[k]] = item[k];
  }
}

// Exclusive scan of a uint64 array in place, in chunks of kScanChunk: chunk totals, one CTA scanning the totals, then each chunk.
namespace {
__device__ uint64_t scan_chunk(uint64_t* a, int64_t begin, int64_t len, uint64_t carry, bool write) {
  __shared__ uint64_t warp_tot[kRankThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t p = begin + (int64_t)threadIdx.x * kScanItems;
  uint64_t v[kScanItems], sum = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    v[k] = p + k < len ? a[p + k] : 0ull;
    sum += v[k];
  }
  uint64_t inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  uint64_t run = carry + inc - sum, total = 0;
  for (int k = 0; k < kRankThreads / 32; ++k) {
    if (k < w) run += warp_tot[k];
    total += warp_tot[k];
  }
  if (write) {
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      if (p + k < len) a[p + k] = run;
      run += v[k];
    }
  }
  __syncthreads();
  return total;
}
}  // namespace

__global__ void __launch_bounds__(256) scan_totals_kernel(uint64_t* a, int64_t len, uint64_t* totals) {
  pdl_wait();
  const uint64_t t = scan_chunk(a, (int64_t)blockIdx.x * kScanChunk, len, 0ull, false);
  if (threadIdx.x == 0) totals[blockIdx.x] = t;
}

__global__ void __launch_bounds__(256) scan_top_kernel(uint64_t* totals, int64_t chunks) {
  pdl_wait();
  uint64_t carry = 0;
  for (int64_t b = 0; b < chunks; b += kScanChunk) carry += scan_chunk(totals, b, chunks, carry, true);
}

__global__ void __launch_bounds__(256) scan_apply_kernel(uint64_t* a, int64_t len, const uint64_t* totals) {
  pdl_wait();
  scan_chunk(a, (int64_t)blockIdx.x * kScanChunk, len, totals[blockIdx.x], true);
}

namespace {
__device__ __forceinline__ bool group_start(const uint64_t* items, int64_t e, int64_t seglen) {
  return e % seglen == 0 || item_key(items[e - 1]) != item_key(items[e]);
}
}  // namespace

// flags[e] = (item e starts a group of equal scores) << 32 | (item e is a positive); exclusive-scanned in place afterwards
__global__ void __launch_bounds__(256) ap_flags_kernel(const uint64_t* __restrict__ items, int64_t L, int64_t seglen, uint64_t* __restrict__ flags) {
  pdl_wait();
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= L) return;
  flags[e] = ((uint64_t)group_start(items, e, seglen) << 32) | (items[e] & 1u);
}

// After the scan: each group's first item records the positives before the group; each segment's first item the positives before
// the segment, and the last item the total.
__global__ void __launch_bounds__(256) ap_groups_kernel(const uint64_t* __restrict__ items, const uint64_t* __restrict__ scanned, int64_t L,
                                                        int64_t seglen, uint32_t* __restrict__ group_tp, uint32_t* __restrict__ seg_tp) {
  pdl_wait();
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= L) return;
  const uint64_t s = scanned[e];
  if (group_start(items, e, seglen)) group_tp[s >> 32] = (uint32_t)s;
  if (e % seglen == 0) seg_tp[e / seglen] = (uint32_t)s;
  if (e == L - 1) seg_tp[L / seglen] = (uint32_t)s + (uint32_t)(items[e] & 1u);
}

// Sum of positives_g * TP_g / N_g over the group ends in chunk blockIdx.x of segment blockIdx.y -> partial[y * gridDim.x + x]
__global__ void __launch_bounds__(256) ap_sum_kernel(const uint64_t* __restrict__ items, const uint64_t* __restrict__ scanned, int64_t seglen,
                                                     const uint32_t* __restrict__ group_tp, const uint32_t* __restrict__ seg_tp,
                                                     double* __restrict__ partial) {
  pdl_wait();
  const int64_t seg0 = (int64_t)blockIdx.y * seglen;
  const int64_t stop = (int64_t)(blockIdx.x + 1) * kSumChunk, end = stop < seglen ? stop : seglen;
  const uint32_t tp0 = seg_tp[blockIdx.y];
  double acc = 0.0;
  for (int64_t j = (int64_t)blockIdx.x * kSumChunk + threadIdx.x; j < end; j += kRankThreads) {
    const int64_t e = seg0 + j;
    const uint64_t it = items[e];
    if (j + 1 < seglen && item_key(items[e + 1]) == item_key(it)) continue;     // not the last item of its group
    const uint64_t s = scanned[e];
    const uint32_t tp = (uint32_t)s + (uint32_t)(it & 1u);                     // positives up to and including e
    const bool first = j == 0 || item_key(items[e - 1]) != item_key(it);
    const uint32_t group = (uint32_t)(s >> 32) + (first ? 1u : 0u) - 1u;
    const uint32_t in_group = tp - group_tp[group];
    if (in_group) acc += (double)in_group * (double)(tp - tp0) / (double)(j + 1);
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) partial[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = t;
}

// Samples AP: a row has one positive, so its AP is 1 / |{c : p_c >= p_label}|; NaN when any of its scores is NaN
__global__ void __launch_bounds__(256) ap_samples_kernel(const float* __restrict__ store, const int* __restrict__ labels, int n, int C,
                                                         double* __restrict__ partial) {
  pdl_wait();
  const int stop = (int)(blockIdx.x + 1) * kSumChunk, end = stop < n ? stop : n;
  double acc = 0.0;
  for (int i = blockIdx.x * kSumChunk + threadIdx.x; i < end; i += kRankThreads) {
    const float* s = store + (int64_t)i * C;
    const int y = labels[i];
    bool nan = y < 0 || y >= C;
    const float sy = nan ? 0.0f : s[y];
    int above = 0;
    for (int c = 0; c < C; ++c) {
      nan |= s[c] != s[c];
      above += s[c] >= sy ? 1 : 0;
    }
    acc += nan ? (double)NAN : 1.0 / (double)above;
  }
  const double t = block_sum(acc);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}

// out[y] = sum of in[y * len, (y + 1) * len) in a fixed order
__global__ void __launch_bounds__(256) row_sum_kernel(const double* __restrict__ in, int64_t len, double* __restrict__ out) {
  pdl_wait();
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < len; i += kRankThreads) acc += in[(int64_t)blockIdx.x * len + i];
  const double t = block_sum(acc);
  if (threadIdx.x == 0) out[blockIdx.x] = t;
}

// result: [0, C) AP per class, [C, 2C) positives per class, then macro, micro, weighted and samples
__global__ void eval_rank_finish_kernel(const uint64_t* __restrict__ class_items, int n, int C, const double* __restrict__ sums,
                                        const uint32_t* __restrict__ class_tp, const uint32_t* __restrict__ micro_tp, double* __restrict__ result) {
  pdl_wait();
  if (threadIdx.x) return;
  double macro = 0.0, weighted = 0.0, support = 0.0;
  bool any_nan = false;
  for (int c = 0; c < C; ++c) {
    const uint32_t pos = class_tp[c + 1] - class_tp[c];
    const bool nan = item_key(class_items[(int64_t)c * n]) == 0u;
    const double ap = nan ? (double)NAN : (pos ? sums[c] / (double)pos : 0.0);
    any_nan |= nan;
    result[c] = ap;
    result[C + c] = (double)pos;
    macro += ap;
    weighted += ap * (double)pos;
    support += (double)pos;
  }
  const uint32_t micro_pos = micro_tp[1] - micro_tp[0];
  result[2 * C] = macro / (double)C;
  result[2 * C + 1] = any_nan ? (double)NAN : (micro_pos ? sums[C] / (double)micro_pos : 0.0);
  result[2 * C + 2] = support > 0.0 ? weighted / support : 0.0;
  result[2 * C + 3] = sums[C + 1] / (double)n;
}

int eval_collect_launch(const float* scores, const float* onehot, int n, int classes, int64_t row_offset, float* store_scores,
                        int32_t* store_labels, cudaStream_t s) {
  const int64_t total = (int64_t)n * classes;
  TCR_LAUNCH("eval_collect", eval_collect_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s, scores, onehot, n, classes,
             store_scores + row_offset * classes, store_labels + row_offset);
  return 0;
}

namespace {
struct RankWorkspace {
  int64_t L, tiles, hist_len, scan_chunks, micro_chunks, class_chunks, sample_chunks, bytes;
  size_t items_a, items_b, group_tp, hist, totals, partial, sums, class_tp, micro_tp;
};

RankWorkspace rank_workspace(int n, int C) {
  RankWorkspace w{};
  w.L = (int64_t)n * C;
  w.tiles = (w.L + kRadixTile - 1) / kRadixTile;
  w.hist_len = 256 * w.tiles;
  w.scan_chunks = (std::max(w.L, w.hist_len) + kScanChunk - 1) / kScanChunk;
  w.micro_chunks = (w.L + kSumChunk - 1) / kSumChunk;
  w.class_chunks = ((int64_t)n + kSumChunk - 1) / kSumChunk;
  w.sample_chunks = w.class_chunks;
  size_t off = 0;
  auto take = [&off](int64_t bytes) { const size_t at = off; off += ((size_t)bytes + 255) & ~(size_t)255; return at; };
  w.items_a = take(8 * w.L);
  w.items_b = take(8 * w.L);
  w.group_tp = take(4 * w.L);
  w.hist = take(8 * w.hist_len);
  w.totals = take(8 * w.scan_chunks);
  w.partial = take(8 * (w.micro_chunks + C * w.class_chunks + w.sample_chunks));
  w.sums = take(8 * (C + 2));
  w.class_tp = take(4 * (C + 1));
  w.micro_tp = take(4 * 2);
  w.bytes = (int64_t)off;
  return w;
}

void scan_launch(uint64_t* a, int64_t len, uint64_t* totals, cudaStream_t s) {
  const int64_t chunks = (len + kScanChunk - 1) / kScanChunk;
  TCR_LAUNCH("rank_scan", scan_totals_kernel, dim3((unsigned)chunks), dim3(kRankThreads), 0, s, a, len, totals);
  TCR_LAUNCH("rank_scan", scan_top_kernel, dim3(1), dim3(kRankThreads), 0, s, totals, chunks);
  TCR_LAUNCH("rank_scan", scan_apply_kernel, dim3((unsigned)chunks), dim3(kRankThreads), 0, s, a, len, (const uint64_t*)totals);
}

void radix_pass(const uint64_t* in, uint64_t* out, int shift, const RankWorkspace& w, unsigned char* ws, cudaStream_t s) {
  uint64_t* hist = reinterpret_cast<uint64_t*>(ws + w.hist);
  TCR_LAUNCH("rank_hist", rank_hist_kernel, dim3((unsigned)w.tiles), dim3(kRankThreads), 0, s, in, w.L, shift, (int)w.tiles, hist);
  scan_launch(hist, w.hist_len, reinterpret_cast<uint64_t*>(ws + w.totals), s);
  TCR_LAUNCH("rank_scatter", rank_scatter_kernel, dim3((unsigned)w.tiles), dim3(kRankThreads), 0, s, in, out, w.L, shift, (int)w.tiles,
             (const uint64_t*)hist);
}

// AP sums of `segs` rankings of seglen items each (sorted `items`; `scratch` holds L uint64) -> partial [segs][chunks] -> sums[segs]
void ap_launch(const uint64_t* items, uint64_t* scratch, int64_t seglen, int segs, int64_t chunks, double* partial, double* sums,
               uint32_t* seg_tp, const RankWorkspace& w, unsigned char* ws, cudaStream_t s) {
  const unsigned grid = (unsigned)((w.L + 255) / 256);
  uint32_t* group_tp = reinterpret_cast<uint32_t*>(ws + w.group_tp);
  TCR_LAUNCH("ap_flags", ap_flags_kernel, dim3(grid), dim3(256), 0, s, items, w.L, seglen, scratch);
  scan_launch(scratch, w.L, reinterpret_cast<uint64_t*>(ws + w.totals), s);
  TCR_LAUNCH("ap_groups", ap_groups_kernel, dim3(grid), dim3(256), 0, s, items, (const uint64_t*)scratch, w.L, seglen, group_tp, seg_tp);
  TCR_LAUNCH("ap_sum", ap_sum_kernel, dim3((unsigned)chunks, (unsigned)segs), dim3(kRankThreads), 0, s, items, (const uint64_t*)scratch,
             seglen, (const uint32_t*)group_tp, (const uint32_t*)seg_tp, partial);
  TCR_LAUNCH("ap_sum", row_sum_kernel, dim3((unsigned)segs), dim3(kRankThreads), 0, s, (const double*)partial, chunks, sums);
}
}  // namespace

const char* eval_rank_refusal(int64_t n, int classes) {
  if (classes < 1 || classes > kMaxClasses) return "classes outside [1, kMaxClasses]";
  if (n < 1) return "n must be positive";
  if (n * classes > INT32_MAX) return "n * classes exceeds 2^31 - 1";
  return nullptr;
}

int64_t eval_rank_workspace_bytes(int n, int classes) { return rank_workspace(n, classes).bytes; }

int eval_rank_launch(const float* store_scores, const int32_t* store_labels, int n, int classes, void* workspace, double* result,
                     cudaStream_t s) {
  const RankWorkspace w = rank_workspace(n, classes);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  uint64_t* a = reinterpret_cast<uint64_t*>(ws + w.items_a);
  uint64_t* b = reinterpret_cast<uint64_t*>(ws + w.items_b);
  double* partial = reinterpret_cast<double*>(ws + w.partial);
  double* sums = reinterpret_cast<double*>(ws + w.sums);
  uint32_t* class_tp = reinterpret_cast<uint32_t*>(ws + w.class_tp);
  uint32_t* micro_tp = reinterpret_cast<uint32_t*>(ws + w.micro_tp);
  TCR_LAUNCH("rank_items", rank_items_kernel, dim3((unsigned)((w.L + 255) / 256)), dim3(256), 0, s, store_scores, store_labels, w.L,
             classes, a);
  for (int shift = 32; shift < 64; shift += 16) {       // the four key bytes, least significant first: a -> b -> a
    radix_pass(a, b, shift, w, ws, s);
    radix_pass(b, a, shift + 8, w, ws, s);
  }
  ap_launch(a, b, w.L, 1, w.micro_chunks, partial, sums + classes, micro_tp, w, ws, s);
  radix_pass(a, b, 1, w, ws, s);                         // stable by class: every class's ranking, in class order
  double* class_partial = partial + w.micro_chunks;
  ap_launch(b, a, n, classes, w.class_chunks, class_partial, sums, class_tp, w, ws, s);
  double* sample_partial = class_partial + classes * w.class_chunks;
  TCR_LAUNCH("ap_samples", ap_samples_kernel, dim3((unsigned)w.sample_chunks), dim3(kRankThreads), 0, s, store_scores, store_labels, n,
             classes, sample_partial);
  TCR_LAUNCH("ap_samples", row_sum_kernel, dim3(1), dim3(kRankThreads), 0, s, (const double*)sample_partial, w.sample_chunks,
             sums + classes + 1);
  TCR_LAUNCH("eval_rank_finish", eval_rank_finish_kernel, dim3(1), dim3(32), 0, s, (const uint64_t*)b, n, classes, (const double*)sums,
             (const uint32_t*)class_tp, (const uint32_t*)micro_tp, result);
  return 0;
}

}  // namespace tcr
