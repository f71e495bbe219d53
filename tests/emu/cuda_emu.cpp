// cuda_emu.cpp — fiber scheduler behind tests/emu/cuda_emu.h (TEST-ONLY, see header).
// Ordinary launches run one block at a time; cooperative launches keep every block's fibers alive so that
// emu::gridsync() can be a barrier over the whole grid (use small grids: every thread owns a stack).
#include "cuda_emu.h"

namespace emu {

static State g_state;
State& st() { return g_state; }

namespace {
struct Fiber {
  ucontext_t ctx;
  ThreadCtx tc;
  bool done = true;
  char* stack = nullptr;
  size_t stack_bytes = 0;
  int block = 0, lane = 0, warp = 0;
};
struct WarpState {
  int count = 0;
  unsigned gen = 0;
  int alive = 0;
  uint64_t slots[32];
};
struct BlockState {
  int alive = 0, count = 0;
  unsigned gen = 0;
  std::vector<WarpState> warps;
  std::vector<unsigned char> smem;
};

std::vector<Fiber> g_fibers;
std::vector<BlockState> g_blocks;
ucontext_t g_sched;
const std::function<void()>* g_body = nullptr;
int g_cur = 0, g_total_alive = 0, g_grid_count = 0;
unsigned g_cluster = 1;   // CTAs per cluster of the running launch (1: ordinary / cooperative launches)
unsigned g_grid_gen = 0;
unsigned long long g_progress = 0;

Fiber& me() { return g_fibers[g_cur]; }
void yield() { swapcontext(&me().ctx, &g_sched); }

void on_exit_thread() {
  Fiber& f = me();
  f.done = true;
  ++g_progress;
  BlockState& b = g_blocks[f.block];
  WarpState& w = b.warps[f.warp];
  w.slots[f.lane] = 0;
  --w.alive;
  --b.alive;
  --g_total_alive;
  if (w.alive > 0 && w.count == w.alive) { w.count = 0; ++w.gen; }
  if (b.alive > 0 && b.count == b.alive) { b.count = 0; ++b.gen; }
  if (g_total_alive > 0 && g_grid_count == g_total_alive) { g_grid_count = 0; ++g_grid_gen; }
}

void fiber_entry() {
  (*g_body)();
  on_exit_thread();
  swapcontext(&me().ctx, &g_sched);
  abort();  // never resumed
}

void run(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body, const std::vector<uint3>& bids,
         size_t stack_bytes) {
  const int n = (int)(block.x * block.y * block.z);
  const int nb = (int)bids.size();
  if (n <= 0 || n > 1024) { fprintf(stderr, "emu: bad block size %d\n", n); abort(); }
  if ((int)g_fibers.size() < n * nb) g_fibers.resize((size_t)n * nb);
  if ((int)g_blocks.size() < nb) g_blocks.resize(nb);
  g_body = &body;
  g_state.bdim = block;
  g_state.gdim = grid;
  g_total_alive = n * nb;
  g_grid_count = 0;
  for (int b = 0; b < nb; ++b) {
    BlockState& bs = g_blocks[b];
    bs.alive = n;
    bs.count = 0;
    bs.warps.assign((n + 31) / 32, WarpState());
    bs.smem.resize(smem_bytes + 2048);
    unsigned char* base = (unsigned char*)(((uintptr_t)bs.smem.data() + 1023) & ~(uintptr_t)1023);
    memset(base, 0xFF, smem_bytes);  // NaN poison
    for (int i = 0; i < n; ++i) {
      Fiber& f = g_fibers[(size_t)b * n + i];
      if (f.stack_bytes < stack_bytes) {
        free(f.stack);
        f.stack = (char*)malloc(stack_bytes);
        f.stack_bytes = stack_bytes;
      }
      f.done = false;
      f.block = b;
      f.warp = i / 32;
      f.lane = i % 32;
      f.tc.tid = uint3{(unsigned)(i % block.x), (unsigned)((i / block.x) % block.y), (unsigned)(i / (block.x * block.y))};
      f.tc.bid = bids[b];
      f.tc.smem = base;
      getcontext(&f.ctx);
      f.ctx.uc_stack.ss_sp = f.stack;
      f.ctx.uc_stack.ss_size = f.stack_bytes;
      f.ctx.uc_link = nullptr;
      makecontext(&f.ctx, fiber_entry, 0);
      bs.warps[i / 32].alive++;
    }
  }
  while (g_total_alive > 0) {
    const unsigned long long before = g_progress;
    for (int i = 0; i < n * nb; ++i) {
      if (g_fibers[i].done) continue;
      g_cur = i;
      g_state.cur = &g_fibers[i].tc;
      swapcontext(&g_sched, &g_fibers[i].ctx);
    }
    if (g_total_alive > 0 && g_progress == before) {
      fprintf(stderr, "emu: deadlock: %d threads stuck at a barrier\n", g_total_alive);
      abort();
    }
  }
  g_state.cur = nullptr;
}
}  // namespace

void syncthreads() {
  BlockState& b = g_blocks[me().block];
  const unsigned gen = b.gen;
  ++g_progress;  // an arrival is progress (deadlock detector)
  if (++b.count == b.alive) {
    b.count = 0;
    ++b.gen;
  } else {
    while (b.gen == gen) yield();
  }
}

void syncwarp() {
  WarpState& w = g_blocks[me().block].warps[me().warp];
  const unsigned gen = w.gen;
  ++g_progress;
  if (++w.count == w.alive) {
    w.count = 0;
    ++w.gen;
  } else {
    while (w.gen == gen) yield();
  }
}

void gridsync() {
  const unsigned gen = g_grid_gen;
  ++g_progress;
  if (++g_grid_count == g_total_alive) {
    g_grid_count = 0;
    ++g_grid_gen;
  } else {
    while (g_grid_gen == gen) yield();
  }
}

int lane_id() { return me().lane; }

uint64_t warp_exchange(uint64_t v, int src_lane) {
  WarpState& w = g_blocks[me().block].warps[me().warp];
  w.slots[me().lane] = v;
  syncwarp();
  const uint64_t r = w.slots[src_lane & 31];
  syncwarp();
  return r;
}

unsigned ballot(int pred) {
  WarpState& w = g_blocks[me().block].warps[me().warp];
  w.slots[me().lane] = pred ? 1 : 0;
  syncwarp();
  unsigned m = 0;
  for (int i = 0; i < 32; ++i)
    if (w.slots[i]) m |= 1u << i;
  syncwarp();
  return m;
}

// CUDA's launch bounds (compute capability 9.0): a launch outside them fails with cudaErrorInvalidConfiguration before any block runs
static bool refused(dim3 grid, dim3 block) {
  const unsigned long long threads = (unsigned long long)block.x * block.y * block.z;
  const bool bad = grid.x < 1 || grid.x > 2147483647u || grid.y < 1 || grid.y > 65535u || grid.z < 1 || grid.z > 65535u ||
                   threads < 1 || threads > 1024 || block.z > 64;
  if (bad) g_state.last_error = cudaErrorInvalidConfiguration;
  return bad;
}

int launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body) {
  if (refused(grid, block)) return cudaErrorInvalidConfiguration;
  std::vector<uint3> one(1);
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        one[0] = uint3{bx, by, bz};
        run(grid, block, smem_bytes, body, one, 256 * 1024);
      }
  return cudaSuccess;
}

unsigned cluster_rank() { return g_cluster > 1 ? (unsigned)me().block : 0u; }
unsigned cluster_size() { return g_cluster; }
void cluster_sync() {
  if (g_cluster > 1) gridsync();   // a cluster launch keeps exactly one cluster alive per run
  else syncthreads();
}
const void* dsmem(const void* local, unsigned rank) {
  if (g_cluster <= 1) return local;
  const unsigned char* mine = me().tc.smem;
  const unsigned char* theirs = g_fibers[(size_t)rank * (g_state.bdim.x * g_state.bdim.y * g_state.bdim.z)].tc.smem;
  return theirs + ((const unsigned char*)local - mine);
}

int launch_cluster(dim3 grid, dim3 block, size_t smem_bytes, unsigned cluster, const std::function<void()>& body) {
  if (cluster <= 1) return launch(grid, block, smem_bytes, body);
  if (refused(grid, block)) return cudaErrorInvalidConfiguration;
  if (grid.x % cluster != 0 || grid.y != 1 || grid.z != 1) { fprintf(stderr, "emu: grid %u not a multiple of cluster %u\n", grid.x, cluster); abort(); }
  std::vector<uint3> blocks(cluster);
  g_cluster = cluster;
  for (unsigned c0 = 0; c0 < grid.x; c0 += cluster) {
    for (unsigned r = 0; r < cluster; ++r) blocks[r] = uint3{c0 + r, 0, 0};
    run(grid, block, smem_bytes, body, blocks, 128 * 1024);
  }
  g_cluster = 1;
  return cudaSuccess;
}

int launch_cooperative(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body) {
  if (refused(grid, block)) return cudaErrorInvalidConfiguration;
  std::vector<uint3> all;
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) all.push_back(uint3{bx, by, bz});
  run(grid, block, smem_bytes, body, all, 128 * 1024);
  return cudaSuccess;
}

}  // namespace emu
