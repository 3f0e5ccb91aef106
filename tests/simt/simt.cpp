// TEST INFRASTRUCTURE: scheduler of the SIMT emulator (see simt.h).
#include "simt.h"

namespace simt {
Block *g_blk = nullptr;
uint3 g_threadIdx, g_blockIdx;
dim3 g_blockDim, g_gridDim;
void *g_shared_handles[1024];
unsigned g_shared_ctr = 0;
long long g_clock = 0;

static const size_t kStack = 256 * 1024;
static std::vector<char *> g_stacks;

// MPMB_SIMT_ORDER: 0 = CTAs and threads in index order (default), 1 = both reversed, 2 = CTAs in a pseudo-random
// order (different per launch) and threads reversed on odd launches.  A kernel whose result depends on which CTA or
// thread runs first — an inter-CTA race, an unordered reduction — gives different bits under different orders.
static int sched_order() {
  static int o = -1;
  if (o < 0) { const char *e = getenv("MPMB_SIMT_ORDER"); o = e ? atoi(e) : 0; }
  return o;
}
static unsigned long long g_launch_no = 0;

static void trampoline() {
  Block *b = g_blk;
  b->body();
  Thread &t = b->th[b->cur];
  t.state = 2;
  b->done++;
  b->warps[t.tid >> 5].exited |= 1u << (t.tid & 31u);
  swapcontext(&t.ctx, &b->main);
}

void yield() {
  Block *b = g_blk;
  Thread &t = b->th[b->cur];
  swapcontext(&t.ctx, &b->main);
  g_threadIdx.x = t.tid;  // restored by the scheduler as well; kept for clarity
}

void run(unsigned grid, unsigned block, const std::function<void()> &body) {
  if (block == 0 || grid == 0) return;
  while (g_stacks.size() < block) g_stacks.push_back((char *)malloc(kStack));
  Block blk;
  blk.n = block;
  blk.th.resize(block);
  blk.warps.resize((block + 31) / 32);
  blk.body = body;
  g_blockDim = dim3(block);
  g_gridDim = dim3(grid);
  Block *prev = g_blk;
  g_blk = &blk;
  const int order = sched_order();
  const unsigned long long launch = g_launch_no++;
  std::vector<unsigned> bids(grid);
  for (unsigned i = 0; i < grid; i++) bids[i] = order == 1 ? grid - 1 - i : i;
  if (order == 2) {  // Fisher-Yates with a per-launch LCG
    unsigned long long st = 0x9E3779B97F4A7C15ull * (launch + 1);
    for (unsigned i = grid; i > 1; i--) { st = st * 6364136223846793005ull + 1442695040888963407ull; std::swap(bids[i - 1], bids[(st >> 33) % i]); }
  }
  const bool rev_threads = order == 1 || (order == 2 && (launch & 1));
  for (unsigned bi = 0; bi < grid; bi++) {
    const unsigned bid = bids[bi];
    g_blockIdx.x = bid; g_blockIdx.y = g_blockIdx.z = 0;
    blk.at_barrier = blk.done = 0;
    blk.or_acc[0] = blk.or_acc[1] = 0;
    for (auto &w : blk.warps) { w.phase = 0; w.arrived = w.released = 0; w.exited = 0; }
    // lanes that do not exist count as exited
    if (block % 32) blk.warps.back().exited = ~0u << (block % 32);
    for (unsigned t = 0; t < block; t++) {
      Thread &th = blk.th[t];
      th.tid = t; th.state = 0; th.stack = g_stacks[t]; th.or_gen = 0;
      getcontext(&th.ctx);
      th.ctx.uc_stack.ss_sp = th.stack;
      th.ctx.uc_stack.ss_size = kStack;
      th.ctx.uc_link = &blk.main;
      makecontext(&th.ctx, trampoline, 0);
    }
    unsigned long long rounds_without_progress = 0;
    while (blk.done < block) {
      unsigned progressed = 0;
      for (unsigned tt = 0; tt < block; tt++) {
        const unsigned t = rev_threads ? block - 1 - tt : tt;
        Thread &th = blk.th[t];
        if (th.state != 0) continue;
        blk.cur = (int)t;
        g_threadIdx.x = t; g_threadIdx.y = g_threadIdx.z = 0;
        unsigned done_before = blk.done, bar_before = blk.at_barrier;
        swapcontext(&blk.main, &th.ctx);
        progressed += (blk.done != done_before) || (blk.at_barrier != bar_before) || 1;  // a resumed thread ran some code
      }
      // release the block barrier when every live thread has arrived
      if (blk.at_barrier && blk.at_barrier + blk.done == block) {
        for (auto &th : blk.th) if (th.state == 1) th.state = 0;
        blk.at_barrier = 0;
        rounds_without_progress = 0;
        continue;
      }
      bool any_runnable = false;
      for (auto &th : blk.th) any_runnable |= th.state == 0;
      if (!any_runnable && blk.done < block) {
        fprintf(stderr, "simt: deadlock in block %u: %u threads at __syncthreads, %u done, %u total\n", bid, blk.at_barrier, blk.done, block);
        abort();
      }
      if (++rounds_without_progress > 50000000ull) { fprintf(stderr, "simt: livelock (warp collective never completed) in block %u\n", bid); abort(); }
    }
  }
  g_blk = prev;
}

long long *warp_exchange(unsigned mask, long long v, unsigned *participants) {
  Block *b = g_blk;
  unsigned l = g_threadIdx.x & 31u;
  Warp &w = b->warps[g_threadIdx.x >> 5];
  while (w.phase == 1) yield();  // the previous collective is still being read
  w.val[l] = v;
  w.arrived |= 1u << l;
  for (;;) {
    unsigned expect = mask & ~w.exited;
    if (w.phase == 1) break;
    if ((w.arrived & expect) == expect) { w.phase = 1; w.released = 0; break; }
    yield();
  }
  *participants = w.arrived & mask;
  return w.val;
}
void warp_release(unsigned mask) {
  Block *b = g_blk;
  unsigned l = g_threadIdx.x & 31u;
  Warp &w = b->warps[g_threadIdx.x >> 5];
  w.released |= 1u << l;
  unsigned expect = w.arrived & mask;
  if ((w.released & expect) == expect) { w.phase = 0; w.arrived = 0; w.released = 0; }
}
}  // namespace simt

// emulated device allocations (simt.h): the live count; simt_fail_allocation(k) makes the k-th cudaMalloc from now fail
// (k = 0: none) and returns how many allocations the previous setting still had to go (0: it has fired, or there was none)
namespace simt {
long long g_live_allocs = 0;
long long g_fail_in = 0;
}  // namespace simt
extern "C" long long simt_device_allocations() { return simt::g_live_allocs; }
extern "C" long long simt_fail_allocation(long long k) {
  const long long left = simt::g_fail_in;
  simt::g_fail_in = k > 0 ? k : 0;
  return left;
}

void __syncthreads() {
  simt::Block *b = simt::g_blk;
  simt::Thread &t = b->th[b->cur];
  t.state = 1;
  b->at_barrier++;
  simt::yield();
}
int __syncthreads_or(int pred) {
  simt::Block *b = simt::g_blk;
  simt::Thread &t = b->th[b->cur];
  const int g = t.or_gen;
  t.or_gen ^= 1;
  if (pred) b->or_acc[g] = 1;
  __syncthreads();
  const int r = b->or_acc[g];
  b->or_acc[g ^ 1] = 0;  // the other accumulator: everybody has read its last value (they all passed this barrier)
  return r;
}
void __syncwarp(unsigned mask) {
  unsigned part;
  simt::warp_exchange(mask, 0, &part);
  simt::warp_release(mask);
}
