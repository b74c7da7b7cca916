// TEST INFRASTRUCTURE ONLY: scheduler of the cooperative-fiber CUDA emulator (see include/cuda_runtime.h).
#include <cuda_runtime.h>

#include <algorithm>

// the runtime entry points the host code of the kernels' translation units calls
extern "C" cudaError_t cudaGetLastError(void) { return cudaSuccess; }
extern "C" const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
extern "C" cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, enum cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
extern "C" cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return cudaSuccess; }
extern "C" cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
extern "C" cudaError_t cudaDeviceGetAttribute(int* v, enum cudaDeviceAttr, int) { *v = 4; return cudaSuccess; }

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;

namespace emu {
ucontext_t g_sched;
Fiber* g_cur = nullptr;
std::vector<Fiber>* g_fibers = nullptr;
Barrier g_warp_bar[64], g_block_bar;
unsigned long long g_slot[64][32];
int g_block_threads = 0;
char* dyn_smem = nullptr;
std::function<void()> g_body;
long long g_progress = 0;
long long g_tick = 0;
int g_async_max = 0;
static unsigned long long g_rng = 0x9E3779B97F4A7C15ull;
struct Ev { long long due; std::function<void()> fn; };
static std::vector<Ev> g_fifo, g_any;
static size_t g_fifo_head = 0;
unsigned rnd() { g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17; return (unsigned)(g_rng >> 32); }
static long long delay() { return g_async_max > 0 ? (long long)(rnd() % (unsigned)(g_async_max + 1)) : 0; }
void defer_ordered(std::function<void()> fn) {
  if (g_async_max <= 0 && g_fifo_head == g_fifo.size()) { fn(); return; }
  long long due = g_tick + delay();
  if (g_fifo_head < g_fifo.size() && due < g_fifo.back().due) due = g_fifo.back().due;  // in issue order
  g_fifo.push_back(Ev{due, std::move(fn)});
}
void defer_unordered(std::function<void()> fn) {
  if (g_async_max <= 0) { fn(); return; }
  g_any.push_back(Ev{g_tick + delay(), std::move(fn)});
}
static bool fire_due(bool all) {
  bool fired = false;
  while (g_fifo_head < g_fifo.size() && (all || g_fifo[g_fifo_head].due <= g_tick)) { auto fn = std::move(g_fifo[g_fifo_head].fn); ++g_fifo_head; fn(); fired = true; }
  if (g_fifo_head == g_fifo.size()) { g_fifo.clear(); g_fifo_head = 0; }
  for (size_t i = 0; i < g_any.size();) {
    if (all || g_any[i].due <= g_tick) { auto fn = std::move(g_any[i].fn); g_any.erase(g_any.begin() + i); fn(); fired = true; }
    else ++i;
  }
  return fired;
}
unsigned g_mma_a[64][32][4], g_mma_b[64][32][2];
std::vector<Wgmma> g_wg_open[2048];
std::vector<std::vector<Wgmma>> g_wg_groups[2048];
std::vector<Copy> g_cp_open[2048];
std::vector<std::vector<Copy>> g_cp_groups[2048];
Barrier g_named_bar[16];

static void trampoline() {
  g_body();
  g_cur->done = true;
  ++g_progress;
  swapcontext(&g_cur->ctx, &g_sched);
}

void run_block(std::function<void()> body, dim3 block) {
  const int n = (int)(block.x * block.y * block.z);
  if (n > 2048) { fprintf(stderr, "emu: block of %d threads\n", n); abort(); }
  g_block_threads = n;
  if (getenv("EMU_TRACE") && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) fprintf(stderr, "emu: launch with %d threads per block\n", n);
  g_body = body;
  for (auto& b : g_warp_bar) b = Barrier();
  g_block_bar = Barrier();
  for (int t = 0; t < 2048; ++t) { g_cp_open[t].clear(); g_cp_groups[t].clear(); g_wg_open[t].clear(); g_wg_groups[t].clear(); }
  for (auto& b : g_named_bar) b = Barrier();
  std::vector<Fiber> fibers(n);
  g_fibers = &fibers;
  for (int t = 0; t < n; ++t) {
    Fiber& f = fibers[t];
    f.stack.resize(256 * 1024);
    f.tid = uint3{(unsigned)(t % block.x), (unsigned)((t / block.x) % block.y), (unsigned)(t / (block.x * block.y))};
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack.data();
    f.ctx.uc_stack.ss_size = f.stack.size();
    f.ctx.uc_link = &g_sched;
    makecontext(&f.ctx, trampoline, 0);
  }
  {
    const char* e = getenv("EMU_ASYNC");
    g_async_max = e ? atoi(e) : 0;
    const char* sd = getenv("EMU_SEED");
    if (sd) g_rng = 0x9E3779B97F4A7C15ull ^ ((unsigned long long)atoll(sd) * 0xD1342543DE82EF95ull + blockIdx.x * 977u + blockIdx.y * 131u + blockIdx.z);
  }
  const bool shuffle = getenv("EMU_SEED") != nullptr;
  std::vector<int> order(n);
  for (int t = 0; t < n; ++t) order[t] = t;
  int left = n, stalled = 0;
  while (left > 0) {
    const long long before = g_progress;
    ++g_tick;
    const bool fired = fire_due(false);
    if (shuffle)  // resume the threads in a different order every pass (warps stay collectively correct: collectives rendezvous)
      for (int t = n - 1; t > 0; --t) std::swap(order[t], order[rnd() % (unsigned)(t + 1)]);
    for (int oi = 0; oi < n; ++oi) {
      Fiber& f = fibers[order[oi]];
      if (f.done) continue;
      g_cur = &f;
      threadIdx = f.tid;
      swapcontext(&g_sched, &f.ctx);
      if (f.done) --left;
    }
    // A pass without a single arrival / completion is not yet a deadlock (a thread may have moved silently from one wait to the
    // next, an asynchronous operation may still be in flight), but thousands in a row are: everybody spins on something nobody
    // will ever signal.
    const bool pending = g_fifo_head < g_fifo.size() || !g_any.empty();
    stalled = (g_progress == before && !fired && !pending) ? stalled + 1 : 0;
    if (left > 0 && stalled > 4000) {
      fprintf(stderr, "emu: deadlock -- %d threads of block (%u,%u,%u) wait for something the others never signal\n", left, blockIdx.x, blockIdx.y, blockIdx.z);
      abort();
    }
  }
  fire_due(true);  // e.g. a trailing prefetch nobody waited for
  g_fibers = nullptr;
}
}  // namespace emu
