// TEST INFRASTRUCTURE ONLY -- a stand-in for <cuda_runtime.h> that lets the *simple* kernels of hqq_b200/csrc (no wgmma, TMA,
// cp.async, mma.sync or inline PTX on their path) be compiled by g++ and EXECUTED ON THE CPU by a cooperative-fiber emulator:
// every CUDA thread of a block is a ucontext fiber, warp collectives (__shfl_xor_sync, __any_sync, __all_sync, __syncwarp) and
// __syncthreads are rendezvous points between fibers.  It exists so that kernels written without access to a GPU can be executed
// and compared with the oracle before their first GPU run (tests/test_emu_cpu.py).  Nothing in the hqq_b200 package includes,
// links or loads this; the product path has no CPU arithmetic.
#pragma once
#define __shared__ static
#include <ucontext.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#include "vector_types.h"  // real CUDA header: float4, uint2, dim3, ... and crt/host_defines.h (empty __device__/__global__ for g++)

#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif

// ---- runtime API surface: the REAL declarations (types, enums, C prototypes); the handful of functions the host side of the
// .cu files calls are DEFINED by emu_runtime.cpp (memcpy/memset/no-ops), nothing links libcudart
#include <cuda.h>  // driver TYPES only (CUtensorMap, CUresult): nothing is linked
#include <cuda_runtime_api.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
template <typename F> inline cudaError_t cudaFuncSetAttribute(F*, cudaFuncAttribute, int) { return cudaSuccess; }
template <typename F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F*, int, size_t) { *n = 2; return cudaSuccess; }

// ---- the emulator ------------------------------------------------------------------------------------------------------------
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;

namespace emu {

struct Fiber {
  ucontext_t ctx;
  std::vector<char> stack;
  bool done = false;
  uint3 tid;
};
struct Barrier { int count = 0; unsigned gen = 0; };

extern ucontext_t g_sched;
extern Fiber* g_cur;
extern std::vector<Fiber>* g_fibers;
extern Barrier g_warp_bar[64], g_block_bar;
extern unsigned long long g_slot[64][32];
extern int g_block_threads;
extern char* dyn_smem;
extern std::function<void()> g_body;
extern long long g_progress;

// Asynchronous engines (TMA, tensor core, cp.async-with-mbarrier) are modelled as deferred events: with EMU_ASYNC=<n> an operation
// takes effect a random number (0..n) of scheduler passes after it was issued -- tensor-core operations in issue order, copies in
// any order -- so a kernel that reads a stage without waiting for its barrier, or refills one the tensor core has not read yet,
// computes garbage here too.  EMU_ASYNC unset: everything completes at issue.  EMU_SEED seeds the delays and shuffles the order
// in which threads are resumed.
extern long long g_tick;
extern int g_async_max;
void defer_ordered(std::function<void()> fn);    // tensor-core queue (FIFO)
void defer_unordered(std::function<void()> fn);  // copy engines
unsigned rnd();

inline int linear_tid() { return (int)(threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)); }
inline void yield() { Fiber* f = g_cur; swapcontext(&f->ctx, &g_sched); }
inline void arrive(Barrier& b, int need) {
  const unsigned gen = b.gen;
  ++g_progress;
  if (++b.count == need) { b.count = 0; ++b.gen; }
  else while (b.gen == gen) yield();
}
inline int warp_lanes(int warp) { const int left = g_block_threads - 32 * warp; return left < 32 ? left : 32; }
inline void warp_barrier() { const int w = linear_tid() >> 5; arrive(g_warp_bar[w], warp_lanes(w)); }

template <typename T> inline T shfl(T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  const int t = linear_tid(), w = t >> 5, l = t & 31;
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  g_slot[w][l] = bits;
  warp_barrier();
  const unsigned long long got = g_slot[w][src_lane & 31];
  warp_barrier();
  T r;
  memcpy(&r, &got, sizeof(T));
  return r;
}
inline int vote(bool p, bool all) {
  const int t = linear_tid(), w = t >> 5, l = t & 31, n = warp_lanes(w);
  g_slot[w][l] = p ? 1ull : 0ull;
  warp_barrier();
  int cnt = 0;
  for (int i = 0; i < n; ++i) cnt += (int)g_slot[w][i];
  warp_barrier();
  return all ? (cnt == n) : (cnt > 0);
}

void run_block(std::function<void()> body, dim3 block);

template <typename K, typename... A>
void launch(K kernel, dim3 grid, dim3 block, size_t smem, A... args) {
  gridDim = grid; blockDim = block;
  std::vector<char> dyn(smem + 2048);
  dyn_smem = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(dyn.data()) + 1023) & ~(uintptr_t)1023);
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        blockIdx = uint3{bx, by, bz};
        run_block([&]() { kernel(args...); }, block);
      }
}
template <typename K>
struct Bound {
  K k; dim3 grid, block; size_t smem;
  template <typename... A> void operator()(A... a) { launch(k, grid, block, smem, a...); }
};
template <typename K> inline Bound<K> bind(K k, dim3 g, dim3 b, size_t s = 0, cudaStream_t = nullptr) { return Bound<K>{k, g, b, s}; }

}  // namespace emu

namespace emu {
// ---- warp-level tensor-core op used by the small-M forward: mma.sync.aligned.m16n8k16.row.col.f32.{f16,bf16} ----------------
// A collective: every lane deposits its fragments, then computes its four outputs from the assembled 16x16 / 16x8 tiles
// (PTX ISA fragment layouts; products of two 16-bit floats are exact in fp32, the k-sum runs in index order).
extern unsigned g_mma_a[64][32][4], g_mma_b[64][32][2];
template <typename T> float half_bits_to_float(unsigned short h);
template <typename T>
inline void mma_m16n8k16(float (&d)[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1, bool zero_c) {
  const int t = linear_tid(), w = t >> 5, l = t & 31, g = l >> 2, q = l & 3;
  g_mma_a[w][l][0] = a0; g_mma_a[w][l][1] = a1; g_mma_a[w][l][2] = a2; g_mma_a[w][l][3] = a3;
  g_mma_b[w][l][0] = b0; g_mma_b[w][l][1] = b1;
  warp_barrier();
  auto A = [&](int r, int k) {
    const unsigned reg = g_mma_a[w][(r & 7) * 4 + ((k & 7) >> 1)][(r >= 8 ? 1 : 0) + (k >= 8 ? 2 : 0)];
    return half_bits_to_float<T>((unsigned short)((reg >> (16 * (k & 1))) & 0xFFFFu));
  };
  auto B = [&](int k, int n) {
    const unsigned reg = g_mma_b[w][n * 4 + ((k & 7) >> 1)][k >= 8 ? 1 : 0];
    return half_bits_to_float<T>((unsigned short)((reg >> (16 * (k & 1))) & 0xFFFFu));
  };
  float out[4];
  for (int i = 0; i < 4; ++i) {
    const int r = g + ((i & 2) ? 8 : 0), n = 2 * q + (i & 1);
    float acc = zero_c ? 0.0f : d[i];
    for (int k = 0; k < 16; ++k) { volatile float p = A(r, k) * B(k, n); volatile float s2 = acc + p; acc = s2; }
    out[i] = acc;
  }
  warp_barrier();
  for (int i = 0; i < 4; ++i) d[i] = out[i];
}
template <> inline float half_bits_to_float<__half>(unsigned short h) { __half_raw r; r.x = h; return __half2float(__half(r)); }
template <> inline float half_bits_to_float<__nv_bfloat16>(unsigned short h) { unsigned u = (unsigned)h << 16; float f; memcpy(&f, &u, 4); return f; }
inline unsigned prmt(unsigned a, unsigned b, unsigned s) {  // prmt.b32, default mode
  const unsigned long long src = ((unsigned long long)b << 32) | a;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) {
    const unsigned sel = (s >> (4 * i)) & 0xFu;
    unsigned byte = (unsigned)((src >> (8 * (sel & 7))) & 0xFFu);
    if (sel & 8) byte = (byte & 0x80u) ? 0xFFu : 0x00u;
    r |= byte << (8 * i);
  }
  return r;
}
inline unsigned lop3(unsigned a, unsigned b, unsigned c, unsigned lut) {
  unsigned r = 0;
  for (int m = 0; m < 8; ++m)
    if ((lut >> m) & 1u) r |= ((m & 4) ? a : ~a) & ((m & 2) ? b : ~b) & ((m & 1) ? c : ~c);
  return r;
}

}  // namespace emu

// ---- functional model of the Hopper tensor-core path used by csrc/linear_gemm.cu --------------------------------------------
// mbarrier (arrival count + transaction bytes + phase), TMA 2-D tile loads with SWIZZLE_128B, wgmma shared-memory descriptors
// (K-major, SWIZZLE_128B), wgmma.mma_async m64nNk16 f32 += f16/bf16 into each thread's register fragment, commit_group /
// wait_group.  What is modelled is the LOGIC (addresses, swizzles, fragment layouts, phases, who waits for whom) -- a protocol
// that deadlocks here is reported by the scheduler -- not timing, proxies or memory ordering.
namespace emu {
struct Mbar { uint16_t init, pending; int32_t tx; };  // the 8 bytes of the kernel's uint64_t; phase in the sign of `init`'s top bit
static_assert(sizeof(Mbar) == 8, "mbarrier model must fit the 64-bit object");
extern Barrier g_named_bar[16];
inline uint32_t smem_offset(const void* p) { return (uint32_t)(reinterpret_cast<const char*>(p) - dyn_smem); }
inline char* smem_ptr(uint32_t off) { return dyn_smem + off; }
inline Mbar* mb(uint64_t* bar) { return reinterpret_cast<Mbar*>(bar); }
inline unsigned mbar_phase(uint64_t* bar) { return mb(bar)->init >> 15; }
inline void mbar_check(uint64_t* bar) {
  Mbar* m = mb(bar);
  if (m->pending == 0 && m->tx == 0) { m->init ^= 0x8000u; m->pending = m->init & 0x7FFFu; }
}
inline void mbar_init(uint64_t* bar, uint32_t count) { Mbar* m = mb(bar); m->init = (uint16_t)count; m->pending = (uint16_t)count; m->tx = 0; ++g_progress; }
inline void mbar_arrive(uint64_t* bar) {
  Mbar* m = mb(bar);
  if (m->pending == 0) { fprintf(stderr, "emu: mbarrier over-arrival\n"); abort(); }
  --m->pending; ++g_progress; mbar_check(bar);
}
inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { mb(bar)->tx += (int32_t)bytes; mbar_arrive(bar); }
inline void mbar_complete_tx(uint64_t* bar, uint32_t bytes) { mb(bar)->tx -= (int32_t)bytes; ++g_progress; mbar_check(bar); }
inline void mbar_wait(uint64_t* bar, uint32_t parity) { while (mbar_phase(bar) == (parity & 1u)) yield(); }  // spinning is not progress
struct TMap { const char* base; uint64_t dims[2]; uint64_t stride_bytes; uint32_t box[2]; uint32_t esize; uint32_t swz; };
static_assert(sizeof(TMap) <= sizeof(CUtensorMap), "fake tensor map must fit the opaque CUtensorMap");
inline CUresult encode_tiled(CUtensorMap* out, CUtensorMapDataType dt, cuuint32_t rank, void* gaddr, const cuuint64_t* dims, const cuuint64_t* strides,
                             const cuuint32_t* box, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle sw, CUtensorMapL2promotion,
                             CUtensorMapFloatOOBfill) {
  // what the model covers: 16-bit tiles of 64 elements with SWIZZLE_128B (the MMA operands), and plain byte tiles (the packed weights)
  const bool bytes = dt == CU_TENSOR_MAP_DATA_TYPE_UINT8;
  if (rank != 2) return CUDA_ERROR_INVALID_VALUE;
  if (!bytes && (sw != CU_TENSOR_MAP_SWIZZLE_128B || box[0] * 2 != 128)) return CUDA_ERROR_INVALID_VALUE;
  if (bytes && (sw != CU_TENSOR_MAP_SWIZZLE_NONE || box[0] % 16 != 0)) return CUDA_ERROR_INVALID_VALUE;
  if (strides[0] % 16 != 0 || (reinterpret_cast<uintptr_t>(gaddr) % 16) != 0) return CUDA_ERROR_INVALID_VALUE;  // the hardware's constraints
  TMap t{reinterpret_cast<const char*>(gaddr), {dims[0], dims[1]}, strides[0], {box[0], box[1]}, bytes ? 1u : 2u, bytes ? 0u : 1u};
  memset(out, 0, sizeof(*out));
  memcpy(out, &t, sizeof(t));
  return CUDA_SUCCESS;
}
inline void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  TMap t;
  memcpy(&t, map, sizeof(t));
  char* dst = reinterpret_cast<char*>(smem_dst);
  if (smem_offset(dst) % (t.swz ? 1024 : 128)) { fprintf(stderr, "emu: TMA destination misaligned\n"); abort(); }
  defer_unordered([=]() {
    if (t.swz) {
      for (uint32_t j = 0; j < t.box[1]; ++j) {
        const long long row = (long long)c1 + j;
        for (uint32_t ch = 0; ch < 8; ++ch) {  // 128-byte rows, SWIZZLE_128B: 16-byte chunk index XOR (row % 8)
          char* d = dst + j * 128 + ((ch ^ (j & 7)) << 4);
          const long long k = (long long)c0 + ch * 8;
          if (row >= 0 && row < (long long)t.dims[1] && k >= 0 && k + 8 <= (long long)t.dims[0]) memcpy(d, t.base + row * t.stride_bytes + k * 2, 16);
          else if (row >= 0 && row < (long long)t.dims[1] && k >= 0 && k < (long long)t.dims[0]) {  // ragged inside a chunk: element-wise
            for (int e = 0; e < 8; ++e) {
              if (k + e < (long long)t.dims[0]) memcpy(d + 2 * e, t.base + row * t.stride_bytes + (k + e) * 2, 2);
              else memset(d + 2 * e, 0, 2);
            }
          } else memset(d, 0, 16);  // out-of-range elements are zero-filled and still count as transferred bytes
        }
      }
    } else {
      for (uint32_t j = 0; j < t.box[1]; ++j) {
        const long long row = (long long)c1 + j;
        for (uint32_t b = 0; b < t.box[0]; ++b) {
          const long long col = (long long)c0 + b;
          dst[j * t.box[0] + b] = (row >= 0 && row < (long long)t.dims[1] && col >= 0 && col < (long long)t.dims[0]) ? t.base[row * t.stride_bytes + col] : 0;
        }
      }
    }
    mbar_complete_tx(bar, t.box[0] * t.box[1] * t.esize);
  });
}
inline float smem_half(uint32_t start, int row, int k, bool bf16) {  // K-major SWIZZLE_128B operand element
  uint32_t logical = start + (uint32_t)(row >> 3) * 1024u + (uint32_t)(row & 7) * 128u + (uint32_t)k * 2u;
  const uint32_t phys = logical ^ (((logical >> 7) & 7u) << 4);
  unsigned short h;
  memcpy(&h, dyn_smem + phys, 2);
  return bf16 ? half_bits_to_float<__nv_bfloat16>(h) : half_bits_to_float<__half>(h);
}
// wgmma.mma_async: operands are read when the operation EXECUTES.  The model runs a thread's wgmma groups at the latest moment
// the program may rely on their results or on their operands no longer being needed -- its wgmma.wait_group -- so a kernel
// that frees a stage before the group reading it has retired multiplies overwritten data.
struct Wgmma { float* d; int N; uint32_t sa, sb; bool accumulate, bf16; };
extern std::vector<Wgmma> g_wg_open[2048];               // per thread: wgmmas not yet committed
extern std::vector<std::vector<Wgmma>> g_wg_groups[2048];  // per thread: committed groups, oldest first
inline void wgmma_now(const Wgmma& w) {
  // thread (warp ww, lane l) of the warpgroup owns rows 16 ww + l/4 (+ 8), columns 8 j + 2 (l % 4) (+ 1): d[4 j + 2 h + e]
  const int tw = linear_tid() & 127, ww = tw >> 5, l = tw & 31;
  for (int j = 0; j < w.N / 8; ++j)
    for (int h = 0; h < 2; ++h)
      for (int e = 0; e < 2; ++e) {
        const int r = 16 * ww + (l >> 2) + 8 * h, n = 8 * j + 2 * (l & 3) + e;
        float acc = w.accumulate ? w.d[4 * j + 2 * h + e] : 0.0f;
        for (int k = 0; k < 16; ++k) acc += smem_half(w.sa, r, k, w.bf16) * smem_half(w.sb, n, k, w.bf16);
        w.d[4 * j + 2 * h + e] = acc;
      }
  ++g_progress;
}
inline void wgmma_f16(float* d, int N, uint64_t adesc, uint64_t bdesc, bool accumulate, bool bf16) {
  if (N < 8 || N > 256 || N % 8 || (adesc >> 62) != 1 || (bdesc >> 62) != 1 || ((adesc >> 32) & 0x3FFFu) != 64 || ((bdesc >> 32) & 0x3FFFu) != 64) {
    fprintf(stderr, "emu: unsupported wgmma descriptor\n");
    abort();
  }
  const uint32_t sa = (uint32_t)(adesc & 0x3FFFu) << 4, sb = (uint32_t)(bdesc & 0x3FFFu) << 4;
  g_wg_open[linear_tid()].push_back(Wgmma{d, N, sa, sb, accumulate, bf16});
}
inline void wgmma_commit() { const int t = linear_tid(); g_wg_groups[t].push_back(std::move(g_wg_open[t])); g_wg_open[t].clear(); }
inline void wgmma_wait(int allow_pending) {
  auto& q = g_wg_groups[linear_tid()];
  while ((int)q.size() > allow_pending) {
    for (const Wgmma& w : q.front()) wgmma_now(w);
    q.erase(q.begin());
  }
}
inline void sts(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) { const uint32_t v[4] = {a, b, c, d}; memcpy(dyn_smem + addr, v, 16); }
inline void sts(uint32_t addr, uint32_t a, uint32_t b) { const uint32_t v[2] = {a, b}; memcpy(dyn_smem + addr, v, 8); }
inline void named_barrier(int id, int n) { arrive(g_named_bar[id & 15], n); }
// cp.async: a copy is only guaranteed to have landed after the thread's wait_group (or the mbarrier it signals) says so.  The
// model performs it at the LATEST moment the program may rely on -- a kernel that consumes a ring slot too early reads old bytes.
struct Copy { void* dst; const void* src; int bytes; };
extern std::vector<Copy> g_cp_open[2048];               // per thread: copies of the group that is still open
extern std::vector<std::vector<Copy>> g_cp_groups[2048];  // per thread: committed groups, oldest first
inline void cp_async(void* dst, const void* src, int bytes) { g_cp_open[linear_tid()].push_back(Copy{dst, src, bytes}); }
inline void cp_async_commit() { const int t = linear_tid(); g_cp_groups[t].push_back(std::move(g_cp_open[t])); g_cp_open[t].clear(); }
inline void cp_async_wait(int allow_pending) {
  auto& q = g_cp_groups[linear_tid()];
  while ((int)q.size() > allow_pending) {
    for (const Copy& c : q.front()) memcpy(c.dst, c.src, (size_t)c.bytes);
    q.erase(q.begin());
  }
}
// cp.async.mbarrier.arrive.noinc: the barrier is signalled when all of this thread's earlier copies have landed -- a deferred event
inline void cp_async_mbar_arrive(uint64_t* bar) {
  const int t = linear_tid();
  std::vector<Copy> mine = std::move(g_cp_open[t]);
  g_cp_open[t].clear();
  defer_unordered([mine, bar]() {
    for (const Copy& c : mine) memcpy(c.dst, c.src, (size_t)c.bytes);
    mbar_arrive(bar);
  });
}
}  // namespace emu
inline unsigned atomicAdd(unsigned* p, unsigned v) { const unsigned old = *p; *p = old + v; return old; }
inline void __threadfence() {}
template <typename T> inline void __stcg(T* p, T v) { *p = v; }
template <typename T> inline T __ldcg(const T* p) { return *p; }

// generated sources replace  kernel<<<g, b, s, st>>>(args)  by  EMU_LAUNCH((kernel), g, b, s, st)(args)
#define EMU_LAUNCH(k, ...) ::emu::bind(k, __VA_ARGS__)

// cudaLaunchKernelEx (programmatic dependent launch attributes are meaningless here: blocks and kernels run one after another)
template <typename... E, typename... A>
inline cudaError_t cudaLaunchKernelEx(const cudaLaunchConfig_t* cfg, void (*kernel)(E...), A&&... args) {
  ::emu::launch(kernel, cfg->gridDim, cfg->blockDim, cfg->dynamicSmemBytes, args...);
  return cudaSuccess;
}

// ---- device intrinsics ---------------------------------------------------------------------------------------------------------
inline void __syncthreads() { emu::arrive(emu::g_block_bar, emu::g_block_threads); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp_barrier(); }
template <typename T> inline T __shfl_xor_sync(unsigned, T v, int o) { return emu::shfl(v, (emu::linear_tid() & 31) ^ o); }
template <typename T> inline T __shfl_sync(unsigned, T v, int src) { return emu::shfl(v, src); }
inline int __any_sync(unsigned, int p) { return emu::vote(p != 0, false); }
inline int __all_sync(unsigned, int p) { return emu::vote(p != 0, true); }

template <typename T> inline T __ldg(const T* p) { return *p; }
// one IEEE operation each: build with -ffp-contract=off so that nothing is fused
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
inline float __frcp_rn(float a) { volatile float r = 1.0f / a; return r; }
inline float __log2f(float a) { return log2f(a); }
inline float __expf(float a) { return expf(a); }
inline float rsqrtf(float a) { return 1.0f / sqrtf(a); }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
