// Decode-harness glue kernels (SURVEY.md 8 f-2: the caller of HQQLinear.forward, NOT the hot path): the few tiny ops
// between the fused linears of a Llama-style block at batch 1, written so a decode step is 8 launches per block
// instead of ~25 framework kernels.  fp16/bf16, one token.  All kernels are PDL-aware (griddepcontrol) so their
// launch latency overlaps the tail of the previous kernel inside a CUDA graph.
#ifndef HQQ_EMU
#include <cooperative_groups.h>
#endif
#include <type_traits>

#include "common.cuh"

namespace hqq {

#ifdef HQQ_EMU
// CPU emulation (tests/emu): kernels and blocks run one after another, so the L2 prefetch and the system-scope accesses are
// plain code; the cluster argmax (DSMEM) is not emulated
__device__ __forceinline__ uint32_t ld_sys_u32(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
__device__ __forceinline__ void prefetch_l2(const void*) {}
// shared-memory integer atomics of the sampling kernel: the emulator resumes a block's threads one at a time and switches only
// at collectives, so a plain read-modify-write is atomic there
__device__ __forceinline__ void smem_add(unsigned* p, unsigned v) { *p += v; }
__device__ __forceinline__ void smem_add(unsigned long long* p, unsigned long long v) { *p += v; }
__device__ __forceinline__ void smem_max(unsigned* p, unsigned v) { if (v > *p) *p = v; }
__device__ __forceinline__ void smem_max(unsigned long long* p, unsigned long long v) { if (v > *p) *p = v; }
__device__ __forceinline__ uint32_t umulhi32(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
__device__ __forceinline__ unsigned long long f32_to_u64_rn(float a) { return (unsigned long long)llrintf(a); }  // 0 <= a < 2^63
#else
__device__ __forceinline__ uint32_t ld_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void smem_add(unsigned* p, unsigned v) { atomicAdd(p, v); }
__device__ __forceinline__ void smem_add(unsigned long long* p, unsigned long long v) { atomicAdd(p, v); }
__device__ __forceinline__ void smem_max(unsigned* p, unsigned v) { atomicMax(p, v); }
__device__ __forceinline__ void smem_max(unsigned long long* p, unsigned long long v) { atomicMax(p, v); }
__device__ __forceinline__ uint32_t umulhi32(uint32_t a, uint32_t b) { return __umulhi(a, b); }
__device__ __forceinline__ unsigned long long f32_to_u64_rn(float a) { return __float2ull_rn(a); }
#endif

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < nw; ++i) s += red[i];
  __syncthreads();
  return s;
}

// h += delta (optional); y = rmsnorm(h) * w         (one CTA per row of [rows, H]; H <= 8 * blockDim)
template <typename T>
__global__ void __launch_bounds__(1024) add_rmsnorm_kernel(T* __restrict__ h, const T* __restrict__ delta, const T* __restrict__ w,
                                                           T* __restrict__ y, int H, float eps) {
  __shared__ float red[32];
  {
    const long long row = (long long)blockIdx.x * H;  // batched decode: one sequence per CTA
    h += row;
    y += row;
    if (delta) delta += row;
  }
  pdl_launch_dependents();
  pdl_wait();
  float v[8];
  int n = 0;
  float ss = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x, ++n) {
    float x = to_f32<T>(h[i]);
    if (delta) {
      x = to_f32<T>(from_f32<T>(x + to_f32<T>(delta[i])));  // residual stream stays in T, like h = h + o in the framework
      h[i] = from_f32<T>(x);
    }
    v[n] = x;
    ss += x * x;
  }
  const float tot = block_sum(ss, red);
  const float inv = rsqrtf(tot / (float)H + eps);
  n = 0;
  for (int i = threadIdx.x; i < H; i += blockDim.x, ++n) y[i] = from_f32<T>(to_f32<T>(from_f32<T>(v[n] * inv)) * to_f32<T>(w[i]));
}

// Same as add_rmsnorm_kernel, but the residual delta is the sum of `tp` tagged partial vectors that the peers' row-parallel
// kernels scattered into this rank's exchange buffer (see SKArgs in linear_small.cu).  As the last consumer of a token it
// bumps the step counter the exchange tags are derived from.
template <typename T>
__global__ void __launch_bounds__(1024) add_rmsnorm_tp_kernel(T* __restrict__ h, const uint32_t* red_data, int* step_ctr, int x_index, int x_per_step,
                                                              int tp, const T* __restrict__ w, T* __restrict__ y, int H, float eps) {
  __shared__ float red[32];
  pdl_launch_dependents();
  pdl_wait();
  const int step = *reinterpret_cast<volatile int*>(step_ctr);
  const uint32_t ex = (uint32_t)step * (uint32_t)x_per_step + (uint32_t)x_index;
  const uint32_t tag = ex & 0xFFFFu;
  const uint32_t* part = red_data + (size_t)(ex & 1u) * tp * H;
  float v[8];
  int n = 0;
  float ss = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x, ++n) {
    float d = 0.f;
    for (int r = 0; r < tp; ++r) {
      uint32_t wv;
      do { wv = ld_sys_u32(part + (size_t)r * H + i); } while ((wv >> 16) != tag);
      const unsigned short hb = (unsigned short)(wv & 0xFFFFu);
      d += to_f32<T>(*reinterpret_cast<const T*>(&hb));
    }
    float x = to_f32<T>(from_f32<T>(to_f32<T>(h[i]) + to_f32<T>(from_f32<T>(d))));
    h[i] = from_f32<T>(x);
    v[n] = x;
    ss += x * x;
  }
  const float tot = block_sum(ss, red);
  const float inv = rsqrtf(tot / (float)H + eps);
  n = 0;
  for (int i = threadIdx.x; i < H; i += blockDim.x, ++n) y[i] = from_f32<T>(to_f32<T>(from_f32<T>(v[n] * inv)) * to_f32<T>(w[i]));
  if (threadIdx.x == 0) *step_ctr = step + 1;
}

// y = silu(g) * u
template <typename T>
__global__ void __launch_bounds__(256) silu_mul_kernel(const T* __restrict__ g, const T* __restrict__ u, T* __restrict__ y, int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float a = to_f32<T>(g[i]);
    const float s = to_f32<T>(from_f32<T>(a / (1.0f + __expf(-a))));
    y[i] = from_f32<T>(s * to_f32<T>(u[i]));
  }
}

// ---- mixture-of-experts router and combine (Mixtral-style sparse MLP) -------------------------------------------------------
// Router: one CTA per token row m of x [M, H]; router [E, H].
//   l[e] = T(sum_k x[m][k] router[e][k])  (fp32 sum, one rounding to T: transformers computes F.linear in the model dtype)
//   p = softmax(l) in fp32; the k largest p, ties to the lower expert index, in descending order; w_j = p_j / sum_j p_j (fp32)
// ids / weights [M, k] take them in that order.  The last CTA to finish (a ticket counter, reset to zero by that CTA) groups the
// M k pairs by expert: pairs of expert e are the slots [off[e], off[e] + cnt[e]) in ascending token order, token[slot] the row a
// pair came from, pair_of[m][j] the slot of (m, j).  Every thread of that CTA owns a contiguous run of tokens, counts its pairs per
// expert, and a scan over the threads in thread order hands each run its first slot per expert: no atomics touch the output.
constexpr int kRouteThreads = 256;
constexpr int kMaxExperts = 64;

template <typename T>
__global__ void __launch_bounds__(kRouteThreads) moe_route_kernel(const T* __restrict__ x, const T* __restrict__ router, int M, int H, int E, int k,
                                                                 int* __restrict__ ids, float* __restrict__ weights, int* __restrict__ pair_of,
                                                                 int* __restrict__ off, int* __restrict__ cnt, int* __restrict__ token,
                                                                 unsigned* ticket) {
  __shared__ float part[kRouteThreads / 32][kMaxExperts];
  __shared__ unsigned short run[kMaxExperts * kRouteThreads];  // [e][thread]: pairs of expert e in the thread's tokens, then its next slot
  __shared__ int first[kMaxExperts];
  __shared__ int is_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m = blockIdx.x;
  pdl_launch_dependents();
  pdl_wait();
  const T* xr = x + (long long)m * H;
  for (int e = 0; e < E; ++e) {
    const T* wr = router + (long long)e * H;
    float acc = 0.0f;
    for (int i = tid * 8; i < H; i += kRouteThreads * 8) {
      const Vec<T, 8> a = *reinterpret_cast<const Vec<T, 8>*>(xr + i);
      const Vec<T, 8> b = *reinterpret_cast<const Vec<T, 8>*>(wr + i);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += to_f32<T>(a.v[j]) * to_f32<T>(b.v[j]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) part[warp][e] = acc;
  }
  __syncthreads();
  if (tid == 0) {
    float p[kMaxExperts];
    float mx = -INFINITY;
    for (int e = 0; e < E; ++e) {
      float l = 0.0f;
      for (int w = 0; w < kRouteThreads / 32; ++w) l += part[w][e];
      p[e] = to_f32<T>(from_f32<T>(l));
      mx = fmaxf(mx, p[e]);
    }
    float sum = 0.0f;
    for (int e = 0; e < E; ++e) { p[e] = expf(p[e] - mx); sum += p[e]; }
    for (int e = 0; e < E; ++e) p[e] = p[e] / sum;
    unsigned long long taken = 0;
    int sel[8];
    float top = 0.0f;
    for (int j = 0; j < k; ++j) {
      int best = -1;
      for (int e = 0; e < E; ++e)
        if (!((taken >> e) & 1ull) && (best < 0 || p[e] > p[best])) best = e;  // strict: the lower index keeps a tie
      taken |= 1ull << best;
      sel[j] = best;
      top += p[best];
    }
    for (int j = 0; j < k; ++j) {
      ids[(long long)m * k + j] = sel[j];
      weights[(long long)m * k + j] = p[sel[j]] / top;
    }
    __threadfence();
    is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // ---- the last CTA: group the pairs by expert
  const int per = (M + kRouteThreads - 1) / kRouteThreads;
  const int t0 = min(M, tid * per), t1 = min(M, t0 + per);
  for (int e = 0; e < E; ++e) run[e * kRouteThreads + tid] = 0;
  for (int t = t0; t < t1; ++t)
    for (int j = 0; j < k; ++j) ++run[__ldcg(ids + (long long)t * k + j) * kRouteThreads + tid];
  __syncthreads();
  if (tid < E) {  // exclusive scan over the threads, in thread order (a count never exceeds M <= 65535)
    int c = 0;
    for (int i = 0; i < kRouteThreads; ++i) {
      const int v = run[tid * kRouteThreads + i];
      run[tid * kRouteThreads + i] = (unsigned short)c;
      c += v;
    }
    first[tid] = c;  // the expert's pair count, for now
  }
  __syncthreads();
  if (tid == 0) {
    int o = 0;
    for (int e = 0; e < E; ++e) {
      const int c = first[e];
      off[e] = o; cnt[e] = c; first[e] = o;
      o += c;
    }
    *ticket = 0;  // every launch leaves the counter at zero (graph replays)
  }
  __syncthreads();
  for (int t = t0; t < t1; ++t)
    for (int j = 0; j < k; ++j) {
      const int e = __ldcg(ids + (long long)t * k + j);
      const int slot = first[e] + run[e * kRouteThreads + tid]++;
      token[slot] = t;
      pair_of[(long long)t * k + j] = slot;
    }
}

// Combine: delta[m] = sum over token m's k pairs in ascending expert id of T(y[pair] * w), accumulated in T from 0 -- the arithmetic
// of transformers' MixtralExperts (fp32 product, .to(dtype), index_add_ one expert at a time).  One CTA per row.
template <typename T>
__global__ void __launch_bounds__(256) moe_combine_kernel(const T* __restrict__ y, const int* __restrict__ ids, const float* __restrict__ weights,
                                                         const int* __restrict__ pair_of, T* __restrict__ delta, int H, int k) {
  __shared__ int s_pair[8];
  __shared__ float s_w[8];
  const int m = blockIdx.x;
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) {
    int e[8];
    for (int j = 0; j < k; ++j) { e[j] = ids[(long long)m * k + j]; s_pair[j] = pair_of[(long long)m * k + j]; s_w[j] = weights[(long long)m * k + j]; }
    for (int j = 1; j < k; ++j)  // insertion sort by expert id (ids of a token are distinct)
      for (int i = j; i > 0 && e[i - 1] > e[i]; --i) {
        const int te = e[i]; e[i] = e[i - 1]; e[i - 1] = te;
        const int tp = s_pair[i]; s_pair[i] = s_pair[i - 1]; s_pair[i - 1] = tp;
        const float tw = s_w[i]; s_w[i] = s_w[i - 1]; s_w[i - 1] = tw;
      }
  }
  __syncthreads();
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    T acc = from_f32<T>(0.0f);
    for (int j = 0; j < k; ++j) {
      const T term = from_f32<T>(to_f32<T>(y[(long long)s_pair[j] * H + h]) * s_w[j]);
      acc = from_f32<T>(to_f32<T>(acc) + to_f32<T>(term));
    }
    delta[(long long)m * H + h] = acc;
  }
}

// Paged KV cache (PAGED instantiations of the ragged kernels): a cache is a pool of pages [pages, n_kv, 64, 128], a page holding 64
// positions of one sequence for every kv head, and row p of slot b, kv head h lives at row (table[b][p / 64] n_kv + h) 64 + p % 64 of
// the pool; table is int32 [batch, L / 64].  Decode tiles (16 positions) and prefill tiles (64), aligned to absolute positions, never
// straddle a page: one table read per tile.  Nothing else changes -- arithmetic, tiling, chunks, tickets, merge order.  Like pos, the
// table entries are read before griddepcontrol.wait, so they must have been written by an earlier, completed launch.
constexpr int kPage = 64;
struct PageTable { const int* table; };
struct NoPages {};  // the contiguous-cache instantiations
template <bool PAGED> using PageArg = typename std::conditional<PAGED, PageTable, NoPages>::type;

// pool row of position p of kv head kvh through the slot's table row tab
__device__ __forceinline__ long long page_row(const int* tab, int n_kv, int kvh, int p) {
  return ((long long)tab[p >> 6] * n_kv + kvh) * kPage + (p & (kPage - 1));
}

// RoPE (rotate-half, cos/sin tables [L, hd]) + KV-cache append + single-token GQA attention over cache[0..pos].
// grid = n_q_heads, block = 256 threads (8 warps).  caches are [n_kv_heads, L, hd], hd = 128.
// The step streams ~5 GB of weights between two visits of a layer's cache, so the rows are cold in DRAM and the kernel is
// bound by load latency, not bandwidth: (1) rows 0..pos-1 were written by earlier steps, so they are prefetched into L2
// BEFORE griddepcontrol.wait, under the tail of the q/k/v kernel (pos itself is only written by the non-PDL kernel that ends
// a step, a full barrier); (2) both position loops keep 8-16 independent loads in flight per thread.
// SEQPOS (ragged batches, BATCH only): sequence b sits at its own position pos_p[b], and everything derived from the position --
// the prefetched rows, the RoPE row, the written row, the loop bounds -- follows it.
// PAGED (SEQPOS only): the caches are page pools and every row, the prefetched ones included, is found through the slot's table row.
constexpr int kAttnThreads = 256;
template <typename T, bool BATCH, bool SEQPOS = false, bool PAGED = false>
__global__ void __launch_bounds__(kAttnThreads) rope_attn_decode_kernel(const T* __restrict__ q_in, const T* __restrict__ k_in, const T* __restrict__ v_in,
                                                                        const T* __restrict__ cos_t, const T* __restrict__ sin_t,
                                                                        T* __restrict__ k_cache, T* __restrict__ v_cache, const long long* __restrict__ pos_p,
                                                                        T* __restrict__ out, int n_q, int n_kv, int L, int hd, float scale,
                                                                        const PageArg<PAGED> pg) {
  extern __shared__ float sm[];  // q[hd] | knew[hd] | p[L]  (later reused as [8][hd] partial outputs) | red[32]
  constexpr int NW = kAttnThreads / 32;
  float* qs = sm;
  float* ks = sm + hd;
  float* ps = sm + 2 * hd;
  float* red = sm + max(2 * hd + L, NW * hd);
  const int h = blockIdx.x, kvh = h / (n_q / n_kv), d = threadIdx.x;
  if constexpr (BATCH) {  // sequence blockIdx.y of the lock-step batch (all at the same position); the one-sequence
    const long long b = blockIdx.y;  // instantiation is the kernel as it was (its position loops lost 1 us per layer at 200
    q_in += b * n_q * hd; out += b * n_q * hd;  // cached positions when the offsets were applied unconditionally)
    k_in += b * n_kv * hd; v_in += b * n_kv * hd;
    if constexpr (!PAGED) { k_cache += b * n_kv * L * hd; v_cache += b * n_kv * L * hd; }
  }
  static_assert(BATCH || !SEQPOS, "per-sequence positions need the batch layout");
  static_assert(SEQPOS || !PAGED, "a paged cache needs per-sequence positions");
  const int* tab = nullptr;
  if constexpr (PAGED) tab = pg.table + (long long)blockIdx.y * (L / kPage);
  // cache row (in units of hd elements) of position t of this head
  auto row = [&](int t) -> long long {
    if constexpr (PAGED) return page_row(tab, n_kv, kvh, t);
    else return (long long)kvh * L + t;
  };
  const int pos = (int)pos_p[SEQPOS ? blockIdx.y : 0];
  pdl_launch_dependents();
  if constexpr (PAGED) {
    // the same lines page by page: a row is two 128-byte lines (hd 128, 16-bit T)
    const char* kb = reinterpret_cast<const char*>(k_cache);
    const char* vb = reinterpret_cast<const char*>(v_cache);
    for (int i = d; i < 2 * pos; i += kAttnThreads) {
      const long long off = row(i >> 1) * (hd * (int)sizeof(T)) + ((i & 1) << 7);
      prefetch_l2(kb + off);
      prefetch_l2(vb + off);
    }
  } else {
    // one 128-byte line per prefetch; pos rows of hd * sizeof(T) bytes each in both caches
    const char* kb = reinterpret_cast<const char*>(k_cache + (long long)kvh * L * hd);
    const char* vb = reinterpret_cast<const char*>(v_cache + (long long)kvh * L * hd);
    const int lines = (int)(((long long)pos * hd * (int)sizeof(T)) >> 7);
    for (int i = d; i < lines; i += kAttnThreads) {
      prefetch_l2(kb + ((long long)i << 7));
      prefetch_l2(vb + ((long long)i << 7));
    }
  }
  pdl_wait();
  const int half = hd / 2;
  // rope: x*cos + rotate_half(x)*sin, computed in T like the framework ops
  if (d < hd) {
    const float c = to_f32<T>(cos_t[(long long)pos * hd + d]), s = to_f32<T>(sin_t[(long long)pos * hd + d]);
    const float qx = to_f32<T>(q_in[h * hd + d]);
    const float qr = (d < half) ? -to_f32<T>(q_in[h * hd + d + half]) : to_f32<T>(q_in[h * hd + d - half]);
    qs[d] = to_f32<T>(from_f32<T>(to_f32<T>(from_f32<T>(qx * c)) + to_f32<T>(from_f32<T>(qr * s))));
    const float kx = to_f32<T>(k_in[kvh * hd + d]);
    const float kr = (d < half) ? -to_f32<T>(k_in[kvh * hd + d + half]) : to_f32<T>(k_in[kvh * hd + d - half]);
    const T kn = from_f32<T>(to_f32<T>(from_f32<T>(kx * c)) + to_f32<T>(from_f32<T>(kr * s)));
    ks[d] = to_f32<T>(kn);
    if (h % (n_q / n_kv) == 0) {  // one head of the group owns the cache write
      k_cache[row(pos) * hd + d] = kn;
      v_cache[row(pos) * hd + d] = v_in[kvh * hd + d];
    }
  }
  __syncthreads();
  // scores: thread t handles positions t, t+blockDim, ... (a whole 256-byte row each, all 16 loads in flight at once);
  // the current position uses the freshly rotated k
  float mx = -INFINITY;
  for (int t = d; t <= pos; t += kAttnThreads) {
    float acc = 0.f;
    if (t == pos) {
      for (int i = 0; i < hd; ++i) acc += qs[i] * ks[i];
    } else {
      const T* kr = k_cache + row(t) * hd;
      Vec<T, 8> kv[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) kv[i] = *reinterpret_cast<const Vec<T, 8>*>(kr + i * 8);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += qs[i * 8 + j] * to_f32<T>(kv[i].v[j]);
      }
    }
    acc *= scale;
    ps[t] = acc;
    mx = fmaxf(mx, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((d & 31) == 0) red[d >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < NW; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int t = d; t <= pos; t += kAttnThreads) {
    const float e = __expf(ps[t] - mx);
    ps[t] = e;
    sum += e;
  }
  const float tot = block_sum(sum, red);
  const float ps_last = ps[pos];
  // output: warp w takes positions w, w+8, ... and each lane four consecutive dimensions (one 8-byte load per position);
  // eight positions per warp are loaded before any is consumed.  The eight partial outputs meet in shared memory.
  {
    const int w = d >> 5, l = d & 31;
    float o4[4] = {0.f, 0.f, 0.f, 0.f};
    const T* vbase = v_cache + (long long)kvh * L * hd + 4 * l;
    auto vrow = [&](int t) -> const T* {  // lane's four dims of position t
      if constexpr (PAGED) return v_cache + row(t) * hd + 4 * l;
      else return vbase + (long long)t * hd;
    };
    int t = w;
    for (; t + 7 * NW < pos; t += 8 * NW) {
      Vec<T, 4> vv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) vv[u] = *reinterpret_cast<const Vec<T, 4>*>(vrow(t + u * NW));
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float pt = ps[t + u * NW];
#pragma unroll
        for (int j = 0; j < 4; ++j) o4[j] += pt * to_f32<T>(vv[u].v[j]);
      }
    }
    for (; t < pos; t += NW) {
      const Vec<T, 4> vv = *reinterpret_cast<const Vec<T, 4>*>(vrow(t));
      const float pt = ps[t];
#pragma unroll
      for (int j = 0; j < 4; ++j) o4[j] += pt * to_f32<T>(vv.v[j]);
    }
    __syncthreads();  // q, k and the probabilities are dead now: reuse the front of the buffer for the cross-warp reduction
    float* part = sm;  // [NW][hd] floats (the launcher sizes the buffer for max(2*hd + L, NW*hd) + 32)
#pragma unroll
    for (int j = 0; j < 4; ++j) part[w * hd + 4 * l + j] = o4[j];
    __syncthreads();
    if (d < hd) {
      float o = 0.f;
#pragma unroll
      for (int i = 0; i < NW; ++i) o += part[i * hd + d];
      o += ps_last * to_f32<T>(v_in[kvh * hd + d]);
      out[h * hd + d] = from_f32<T>(o / tot);
    }
  }
}

// Split-KV GQA attention for one decoded token at long context (DESIGN.md 3.5): RoPE + KV-cache append + attention over
// cache[0..pos] with the cached positions split into S contiguous chunks, one CTA per (chunk, kv head, sequence).
//
// Each CTA handles all G = n_q / n_kv query heads of its group, so every K/V row crosses HBM once, not G times.  Both products
// run on mma.sync m16n8k16 with the (at most 8) heads as the n = 8 dimension:
//   scores^T [16 positions x 8 heads] = K tile [16 x 128] . Q^T       (K from shared memory, Q^T in registers)
//   O^T      [128 dims x 8 heads]    += V^T [128 x 16] . P^T           (V^T from shared memory, P^T from the score fragments)
// Each of the 8 warps streams the 16-position tiles w, w+8, ... of its CTA's chunk through a private cp.async ring (its stages and
// their layout depend on the cache format: 16-bit, or HQQ 8- or 4-bit levels dequantised into the MMA fragments) and keeps an online
// softmax in fp32; P is rounded to T for the MMA and the row sum adds the rounded values.  The warps meet in shared memory in warp order,
// the CTA publishes its partial (m, l, o[G][128]) to the workspace, and the last CTA of a (sequence, kv head) -- found with a
// fence and a ticket -- combines the S partials in split order, writes out with one rounding to T and resets the ticket.
//
// S = max(1, min(SMs / n_kv, ceil(cache_len / 16))) is fixed at launch (graph replay advances *pos without re-capture); each CTA
// derives its chunk from *pos: c = ceil((pos + 1) / S) rounded up to 16, split s covers [s c, min((s + 1) c, pos + 1)).
namespace {

constexpr int kSplitWarps = 8;
constexpr int kSplitThreads = 32 * kSplitWarps;
constexpr int kSplitStages = 3;
constexpr int kSplitTile = 16;      // positions per tile: the m dimension of the score MMA
constexpr int kSplitMaxGroup = 8;   // query heads per kv head: the n dimension of both MMAs
constexpr int kSplitMaxLen = 131072;
constexpr int kHd = 128;
constexpr int kTileBytes = kSplitTile * kHd * 2;                          // one K or V tile, 4 KB
constexpr int kStageBytes = 2 * kTileBytes;
constexpr int kRingBytes = kSplitWarps * kSplitStages * kStageBytes;      // 192 KB
constexpr int kPartFloats = kHd + 2;                                      // per head: m, l, o[128]

template <typename T> __device__ __forceinline__ uint32_t bits16(T v) { return (uint32_t)*reinterpret_cast<const unsigned short*>(&v); }

// byte offset of 16-byte chunk c of row r inside a [16][128] tile
__device__ __forceinline__ int swz(int r, int c) { return r * 256 + ((c ^ (r & 7)) << 4); }

__device__ __forceinline__ void split_cp16(void* smem, const void* g) {
#ifdef HQQ_EMU
  ::emu::cp_async(smem, g, 16);
#else
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(g) : "memory");
#endif
}
#ifdef HQQ_EMU
__device__ __forceinline__ void split_commit() { ::emu::cp_async_commit(); }
template <int N> __device__ __forceinline__ void split_wait() { ::emu::cp_async_wait(N); }
#else
__device__ __forceinline__ void split_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void split_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#endif

// ldmatrix.x4 (TRANS: .trans): lane l supplies the row address p of row l % 8 of matrix l / 8 and receives r[j] of matrix j
template <bool TRANS>
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], const char* p) {
#ifdef HQQ_EMU
  const int l = threadIdx.x & 31;
  for (int j = 0; j < 4; ++j) {
    if (!TRANS) {
      const char* src = __shfl_sync(0xffffffffu, p, j * 8 + (l >> 2));
      r[j] = *reinterpret_cast<const uint32_t*>(src + 4 * (l & 3));
    } else {  // element (row 2 (l % 4) + {0, 1}, column l / 4) of the stored matrix
      const char* s0 = __shfl_sync(0xffffffffu, p, j * 8 + 2 * (l & 3));
      const char* s1 = __shfl_sync(0xffffffffu, p, j * 8 + 2 * (l & 3) + 1);
      r[j] = (uint32_t)*reinterpret_cast<const unsigned short*>(s0 + 2 * (l >> 2)) |
             ((uint32_t)*reinterpret_cast<const unsigned short*>(s1 + 2 * (l >> 2)) << 16);
    }
  }
#else
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  if (TRANS)
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
  else
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
#endif
}

// d += A[16x16] . B[16x8], fp32 accumulate
template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
#ifdef HQQ_EMU
  ::emu::mma_m16n8k16<T>(d, a[0], a[1], a[2], a[3], b0, b1, false);
#else
  if constexpr (std::is_same<T, __half>::value)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
#endif
}

// x*cos + rotate_half(x)*sin at dim d of the head row x, with the cos / sin rows of its position: each product and the sum rounded
// to T, as rope_attn_decode_kernel rounds them (a cache row written by any kernel is bit for bit the row a decode step writes)
template <typename T>
__device__ __forceinline__ T rope_rounded(const T* x, int d, const T* cos_row, const T* sin_row) {
  constexpr int half = kHd / 2;
  const float c = to_f32<T>(cos_row[d]), s = to_f32<T>(sin_row[d]);
  const float xv = to_f32<T>(x[d]);
  const float xr = (d < half) ? -to_f32<T>(x[d + half]) : to_f32<T>(x[d - half]);
  return from_f32<T>(to_f32<T>(from_f32<T>(xv * c)) + to_f32<T>(from_f32<T>(xr * s)));
}

// One 16-position tile of the online softmax of the split kernels for lane (g, qd): columns 2 qd, 2 qd + 1 (heads, or the verify
// kernel's (t, h) columns), scores s of positions p0 and p0 + 8, column u seeing the positions below lim_u.  P is rounded to T for the
// MMA and l adds the rounded values.  b0, b1: the P^T fragment of the V^T . P^T MMA (k = position, n = column g): positions 2 qd,
// 2 qd + 1 (+ 8) sit in lanes (2 qd, g / 2) and (2 qd + 1, g / 2).  GUARD: a tile may lie wholly past a column's last key, so a column
// with no key yet keeps m = -inf, l = 0, o = 0; without it every tile holds a key of every column and the running max is finite.
template <typename T, bool GUARD>
__device__ __forceinline__ void softmax_tile(const float (&s)[4], float scale_log2, int p0, int lim0, int lim1, float (&m)[2], float (&l)[2],
                                             float (&o)[8][4], int g, int qd, uint32_t& b0, uint32_t& b1) {
  const float x0 = p0 < lim0 ? s[0] * scale_log2 : -INFINITY, x1 = p0 < lim1 ? s[1] * scale_log2 : -INFINITY;
  const float x2 = p0 + 8 < lim0 ? s[2] * scale_log2 : -INFINITY, x3 = p0 + 8 < lim1 ? s[3] * scale_log2 : -INFINITY;
  float t0 = fmaxf(x0, x2), t1 = fmaxf(x1, x3);
#pragma unroll
  for (int off = 4; off < 32; off <<= 1) {
    t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, off));
    t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, off));
  }
  const float n0 = fmaxf(m[0], t0), n1 = fmaxf(m[1], t1);
  float r0 = n0, r1 = n1;
  if constexpr (GUARD) {
    r0 = n0 == -INFINITY ? 0.f : n0;
    r1 = n1 == -INFINITY ? 0.f : n1;
  }
  const float a0 = exp2f(m[0] - r0), a1 = exp2f(m[1] - r1);
  m[0] = n0; m[1] = n1;
  const T p00 = from_f32<T>(exp2f(x0 - r0)), p01 = from_f32<T>(exp2f(x1 - r1));
  const T p10 = from_f32<T>(exp2f(x2 - r0)), p11 = from_f32<T>(exp2f(x3 - r1));
  l[0] = l[0] * a0 + (to_f32<T>(p00) + to_f32<T>(p10));
  l[1] = l[1] * a1 + (to_f32<T>(p01) + to_f32<T>(p11));
#pragma unroll
  for (int mt = 0; mt < 8; ++mt) { o[mt][0] *= a0; o[mt][1] *= a1; o[mt][2] *= a0; o[mt][3] *= a1; }
  const uint32_t lo = bits16(p00) | (bits16(p01) << 16), hi = bits16(p10) | (bits16(p11) << 16);
  const int src = 8 * qd + (g >> 1), sh = (g & 1) * 16;
  const uint32_t lo0 = __shfl_sync(0xffffffffu, lo, src), lo1 = __shfl_sync(0xffffffffu, lo, src + 4);
  const uint32_t hi0 = __shfl_sync(0xffffffffu, hi, src), hi1 = __shfl_sync(0xffffffffu, hi, src + 4);
  b0 = ((lo0 >> sh) & 0xFFFFu) | (((lo1 >> sh) & 0xFFFFu) << 16);
  b1 = ((hi0 >> sh) & 0xFFFFu) | (((hi1 >> sh) & 0xFFFFu) << 16);
}

// Lane (g, qd)'s share of its warp's partials of columns 2 qd, 2 qd + 1, w0 pointing at the first one's [m, l, o[128]]: l summed over
// the lanes of a column, O^T row g (+ 8) of step mt being dim Dims::odim(mt, g, 0 (1)).  Every lane must call it.
template <class Dims>
__device__ __forceinline__ void put_partial(float* w0, const float (&m)[2], float (&l)[2], const float (&o)[8][4], int g) {
#pragma unroll
  for (int off = 4; off < 32; off <<= 1) {
    l[0] += __shfl_xor_sync(0xffffffffu, l[0], off);
    l[1] += __shfl_xor_sync(0xffffffffu, l[1], off);
  }
  float* w1 = w0 + kPartFloats;
  if (g == 0) { w0[0] = m[0]; w0[1] = l[0]; w1[0] = m[1]; w1[1] = l[1]; }
#pragma unroll
  for (int mt = 0; mt < 8; ++mt) {
    w0[2 + Dims::odim(mt, g, 0)] = o[mt][0]; w1[2 + Dims::odim(mt, g, 0)] = o[mt][1];
    w0[2 + Dims::odim(mt, g, 1)] = o[mt][2]; w1[2 + Dims::odim(mt, g, 1)] = o[mt][3];
  }
}

// The end of the split kernels, once the warp partials wp [NW][WC][m, l, o[128]] are in shared memory: this CTA's partial of its nc
// columns to the workspace part [S][PC][m, l, o[128]], the ticket, and in the last CTA of the group the merge of all S partials into
// row out_row(c) of column c.
template <typename T, int WC, typename OutRow>
__device__ __forceinline__ void split_merge(const float* wp, float* __restrict__ part, unsigned* __restrict__ tickets, int* last, int S, int split,
                                           int PC, int nc, int tid, OutRow out_row) {
  constexpr int NW = kSplitWarps;
  // this CTA's partial, warps in order (an empty chunk, or a column with no key in it, publishes m = -inf, l = 0, o = 0)
  for (int i = tid; i < nc * kHd; i += kSplitThreads) {
    const int c = i >> 7, d = i & (kHd - 1);
    float M = -INFINITY;
    for (int w = 0; w < NW; ++w) M = fmaxf(M, wp[(w * WC + c) * kPartFloats]);
    float lsum = 0.f, osum = 0.f;
    if (M != -INFINITY) {
      for (int w = 0; w < NW; ++w) {
        const float* e = wp + (w * WC + c) * kPartFloats;
        const float f = exp2f(e[0] - M);
        lsum += f * e[1];
        osum += f * e[2 + d];
      }
    }
    float* dst = part + ((long long)split * PC + c) * kPartFloats;
    if (d == 0) { dst[0] = M; dst[1] = lsum; }
    dst[2 + d] = osum;
  }
  __threadfence();  // the partial is visible device-wide before the ticket counts it
  __syncthreads();
  if (tid == 0) *last = atomicAdd(tickets, 1u) == (unsigned)(S - 1);
  __syncthreads();
  if (!*last) return;
  __threadfence();
  // last CTA of the group: all S partials, split order, one rounding to T.  Split 0 holds key 0, which every column sees: M is finite
  for (int i = tid; i < nc * kHd; i += kSplitThreads) {
    const int c = i >> 7, d = i & (kHd - 1);
    float M = -INFINITY;
    for (int sp = 0; sp < S; ++sp) M = fmaxf(M, __ldcg(part + ((long long)sp * PC + c) * kPartFloats));
    float lsum = 0.f, osum = 0.f;
    for (int sp = 0; sp < S; ++sp) {
      const float* e = part + ((long long)sp * PC + c) * kPartFloats;
      const float f = exp2f(__ldcg(e) - M);
      lsum += f * __ldcg(e + 1);
      osum += f * __ldcg(e + 2 + d);
    }
    out_row(c)[d] = from_f32<T>(osum / lsum);
  }
  if (tid == 0) *tickets = 0u;  // ready for the next launch (graph replay needs no memset)
}

// 8-bit HQQ KV cache (DESIGN.md 3.5).  A cache row of one kv head is Quantizer.quantize(row, nbits=8, group_size=gs, axis=1,
// optimize=False): levels uint8 [128] and per-group scale / zero [128 / gs] in T; the attended row is T(T(q - z) * s), what
// hqq_b200_dequantize gives.
//
// kv8_quant4: a 128-element row held four per lane (lane l: elements 4 l .. 4 l + 3).  Group min / max over gs / 4 lanes, then
// init_group (maxv 255, zero not rounded) and quant_level as quantize.cu does for an 8-bit layer without the solver.  Returns the
// four levels (byte j: element 4 l + j) and the scale (1 / s) and zero of the lane's group rounded to T.  MAXV 15 is the 4-bit
// cache's quantiser (levels in [0, 15], one per byte, unpacked).
template <typename T, int MAXV = 255>
__device__ __forceinline__ uint32_t kv8_quant4(const float (&x)[4], int gs, T& scale, T& zero) {
  float mn = fminf(fminf(x[0], x[1]), fminf(x[2], x[3])), mx = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3]));
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    if (o < gs / 4) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
  }
  GroupState st;
  init_group(mn, mx, MAXV, 0, st);
  uint32_t q = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) q |= (uint32_t)quant_level(x[j], st.s, st.z, (float)MAXV) << (8 * j);
  scale = from_f32<T>(__frcp_rn(st.s));  // quantize.py:154 scale = 1.0 / scale, then the meta cast to T
  zero = from_f32<T>(st.z);
  return q;
}

template <typename T> struct Pair;
template <> struct Pair<__half> { using type = __half2; };
template <> struct Pair<__nv_bfloat16> { using type = __nv_bfloat162; };

// The two levels in bytes 2 HI, 2 HI + 1 of w -> T(T(q - z) * s) each, packed as a T2 (byte 2 HI in the low half): T(q) exactly,
// then one rounded T subtraction and one rounded T product per element (z, s: T2 of the two elements' zero and scale).
// fp16: half2(1024 + q) by bit pattern (0x64qq; one prmt for both), minus 1024 exactly.  bf16 (8 significant bits cannot hold
// 1024 + q): float 2^23 + q by bit pattern, minus 2^23, packed to bf16x2 exactly.
template <typename T, int HI>
__device__ __forceinline__ uint32_t kv8_deq2(uint32_t w, typename Pair<T>::type z, typename Pair<T>::type s) {
  typename Pair<T>::type q;
  if constexpr (std::is_same<T, __half>::value) {
    const uint32_t h = prmt(w, 0x64646464u, HI ? 0x4342u : 0x4140u);
    q = __hsub2(*reinterpret_cast<const __half2*>(&h), __half2half2(__ushort_as_half((unsigned short)0x6400u)));
  } else {
    const float a = __fsub_rn(__uint_as_float(prmt(w, 0x4B000000u, 0x7540u | (2 * HI))), 8388608.0f);
    const float b = __fsub_rn(__uint_as_float(prmt(w, 0x4B000000u, 0x7540u | (2 * HI + 1))), 8388608.0f);
    q = __floats2bfloat162_rn(a, b);
  }
  const typename Pair<T>::type r = __hmul2(__hsub2(q, z), s);
  return *reinterpret_cast<const uint32_t*>(&r);
}

// 4-bit HQQ KV cache (DESIGN.md 3.5).  A cache row of one kv head is Quantizer.quantize(row, nbits=4, group_size=gs, axis=1,
// optimize=False) with gs 32 or 64, packed as the reference's 4bit_u8 packing of that row: 64 bytes, byte d = q[d] << 4 | q[d + 64];
// meta [128 / gs] T.  The attended row is T(T(q - z) * s), what oracle.dequantize gives.  16-byte chunk c of a row holds dims
// 16 c .. 16 c + 15 (high nibbles) and 64 + 16 c .. (low nibbles), each half inside one group.
//
// kv4_pack: the levels of kv8_quant4<T, 15> (lane l: elements 4 l .. 4 l + 3, one per byte) -> the packed bytes 4 l .. 4 l + 3 of
// the row in lanes 0..15 (lanes 16..31 hold elements 64 .. 127, whose levels are the low nibbles).  Every lane must call it.
__device__ __forceinline__ uint32_t kv4_pack(uint32_t q) { return (q << 4) | __shfl_xor_sync(0xffffffffu, q, 16); }
// kv4_unpack: packed bytes 4 l' .. 4 l' + 3 -> the levels (one per byte) of elements 4 l' .. (hi) or 64 + 4 l' .. (lo)
__device__ __forceinline__ uint32_t kv4_unpack(uint32_t w, bool hi) { return (hi ? w >> 4 : w) & 0x0F0F0F0Fu; }

// The levels in bits 0..3 and 16..19 of t (other bits ignored) -> T(T(q - z) * s) each, packed as a T2 (bits 0..3 in the low half):
// T(q) exactly, then one rounded T subtraction and one rounded T product per element, as kv8_deq2.  fp16: half2(1024 + q) by bit
// pattern (0x640q), minus 1024 exactly; bf16: bf16(128 + q) by bit pattern (0x430q), minus 128 exactly.
template <typename T>
__device__ __forceinline__ uint32_t kv4_deq2(uint32_t t, typename Pair<T>::type z, typename Pair<T>::type s) {
  using T2 = typename Pair<T>::type;
  const uint32_t m = std::is_same<T, __half>::value ? 0x64006400u : 0x43004300u;
  const uint32_t h = (t & 0x000F000Fu) | m;
  const T2 q = __hsub2(*reinterpret_cast<const T2*>(&h), *reinterpret_cast<const T2*>(&m));
  const T2 r = __hmul2(__hsub2(q, z), s);
  return *reinterpret_cast<const uint32_t*>(&r);
}

// The warp row quantiser of the quantised caches: the 128-element row x (lane l: elements 4 l .. 4 l + 3) quantised by kv8_quant4 to
// BITS bits, its levels stored at lq (BITS 4: packed by kv4_pack, 64 bytes written by lanes 0..15) and each group's scale and zero at
// s[group], z[group].  Returns the lane's four levels (one per byte) and, in sc / ze, their group's meta.  Every lane must call it.
template <typename T, int BITS>
__device__ __forceinline__ uint32_t kv_quant_row(const float (&x)[4], int gs, uint8_t* lq, T* s, T* z, T& sc, T& ze) {
  const int lane = (int)threadIdx.x & 31;
  const uint32_t lv = kv8_quant4<T, (1 << BITS) - 1>(x, gs, sc, ze);
  if constexpr (BITS == 8) {
    *reinterpret_cast<uint32_t*>(lq + 4 * lane) = lv;
  } else {
    const uint32_t pk = kv4_pack(lv);
    if (lane < 16) *reinterpret_cast<uint32_t*>(lq + 4 * lane) = pk;
  }
  if ((4 * lane) % gs == 0) {
    s[4 * lane / gs] = sc;
    z[4 * lane / gs] = ze;
  }
  return lv;
}

// The cache formats of rope_attn_decode_split_kernel.  A format holds the cache pointers -- level arrays k and v with rows of kRowBytes
// bytes, copied in 16-byte chunks -- and supplies what differs between formats:
//   - the stage layout: each warp's ring has kStages stages of kStageBytes, the K then the V levels of a 16-position tile (kLvlBytes
//     each, chunk c of row r at slot(r, c)), then the format's meta (4 arrays of kMetaBytes); the smem a CTA needs (kSmemBytes);
//   - the per-(sequence, kv head) advance of the pointers (contiguous caches);
//   - the staging of a tile's meta rows and the row-pos patch of that meta in a tile staged before the wait;
//   - the fresh row pos: the kFreshBytes after the rotated k, v hold it in cache format (none: the rotated rows are that), and split 0
//     writes it to the cache;
//   - the head-dim permutation, the same for both operands of a product (so the products are unchanged): the Q^T fragment dims
//     (k slots 2 qd + {0, 1} of step kk are dims qdim(kk, qd) + {0, 1}, slots 2 qd + {8, 9} kQPair dims further) and the O^T -> dim
//     map odim(mt, g, hi) (O^T row g + 8 hi of step mt);
//   - the score MMA loop (K . Q^T) and the V^T . P^T loop over one staged tile.
//
// 16-bit cache: [16][128] T tiles of 16-byte chunks XOR-swizzled by row, read through ldmatrix (conflict-free) in 3 stages of 8 KB.
template <typename T>
struct KvF16 {
  static constexpr int kStages = kSplitStages, kRowBytes = 2 * kHd, kFreshBytes = 0;
  static constexpr int kLvlBytes = kTileBytes, kStageBytes = 2 * kLvlBytes;
  static constexpr int kRingBytes = kSplitWarps * kStages * kStageBytes;  // 192 KB
  static constexpr int kSmemBytes = kRingBytes + (kSplitMaxGroup + 2) * kHd * 2 + kFreshBytes + 16;  // + q [8][128], k, v, the fresh row, the flag
  static constexpr int kQPair = 8;
  T* k;
  T* v;

  __device__ static int slot(int r, int c) { return swz(r, c); }
  __device__ static int qdim(int kk, int qd) { return 16 * kk + 2 * qd; }
  __device__ static int odim(int mt, int g, int hi) { return 16 * mt + g + 8 * hi; }
  __device__ void advance(long long kv, int L) { k += kv * L * kHd; v += kv * L * kHd; }
  __device__ void stage_meta(char*, long long, int, int, int, bool, const char*) const {}
  __device__ void patch_meta(char*, int, int, const char*) const {}
  // kf: the rotated k row, then v.  Split 0 writes them to the cache row pr (no CTA of this launch reads it).
  __device__ void fresh(const T* kf, char*, bool write, long long pr, int tid) const {
    if (write && tid < kHd) {
      k[pr * kHd + tid] = kf[tid];
      v[pr * kHd + tid] = kf[kHd + tid];
    }
  }
  // The append's store (rope_append_rows_kernel): lane l's elements 4 l .. 4 l + 3 of a rotated k row (isv 0) or a v row to cache row
  // crow.  Returns them as the cache holds them, packed as two T2.
  __device__ uint2 put(int isv, long long crow, const T (&x)[4]) const {
    const int lane = (int)threadIdx.x & 31;
    T* dst = (isv ? v : k) + crow * kHd + 4 * lane;
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = x[j];
    uint2 y;
    y.x = bits16(x[0]) | (bits16(x[1]) << 16);
    y.y = bits16(x[2]) | (bits16(x[3]) << 16);
    return y;
  }
  __device__ void scores(float (&s)[4], const char* st, const uint32_t (&qb)[8][2], int lane) const {
    const int kr = (lane & 7) + ((lane >> 3) & 1) * 8, kc = lane >> 4;  // ldmatrix row / chunk, K (a0..a3: rows +8, then k +8)
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      uint32_t a[4];
      ldsm4<false>(a, st + swz(kr, 2 * kk + kc));
      mma16816<T>(s, a, qb[kk][0], qb[kk][1]);
    }
  }
  __device__ void pv(float (&o)[8][4], const char* st, uint32_t b0, uint32_t b1, int lane) const {
    const int vr = (lane & 7) + ((lane >> 4) & 1) * 8, vc = (lane >> 3) & 1;  // V^T (a0..a3: dims +8, then positions +8)
    const char* vt = st + kLvlBytes;
#pragma unroll
    for (int mt = 0; mt < 8; ++mt) {
      uint32_t a[4];
      ldsm4<true>(a, vt + swz(vr, 2 * mt + vc));
      mma16816<T>(o[mt], a, b0, b1);
    }
  }
};

// HQQ cache of BITS 8 (gs 64 or 128) or 4 (gs 32 or 64): levels [.., L, 128 BITS / 8] uint8, meta k_s, k_z, v_s, v_z [.., L, 128 / gs]
// T, dequantised straight into the MMA fragments.  The meta of a stage is k scale | k zero | v scale | v zero [16][kNg], kNg the most
// groups a row has; the fresh row is its levels [2][kRowBytes] and meta [4][kNg].  A meta chunk of 16 bytes spans 8 / ng rows.
//   8 bits: 4 stages of 4352 bytes, level rows of 8 chunks XOR-swizzled by row.  Lane (g, qd) takes K dims 32 qd .. 32 qd + 31 of
//     positions g, g + 8 (k slot 2 qd + {0, 1, 8, 9} of step kk is dim 32 qd + 4 kk + {0..3}) and V dims 16 g .. 16 g + 15 of positions
//     2 qd + {0, 1, 8, 9} (O^T row g / g + 8 of step mt is dim 16 g + 2 mt / + 1): two 16-byte loads a row, one group each.
//   4 bits: 6 stages of 2560 bytes, the 16 level rows of a tile filling 8 lines of 128 bytes, line l = r / 2 holding chunk
//     (4 (r & 1) + c) ^ 2 (l & 3) -- conflict-free for the K reads (16 bytes a lane) and the V reads (8 bytes a lane).  Lane (g, qd)
//     takes K chunk qd of positions g, g + 8 (k slot 2 qd + {0, 1, 8, 9} of step kk is dim 16 qd + 4 kk + {0..3} for kk < 4, the high
//     nibbles, and 64 + 16 qd + 4 (kk - 4) + {0..3} for kk >= 4, the low nibbles), and V bytes 8 g .. 8 g + 7 of positions
//     2 qd + {0, 1, 8, 9} (O^T row g of step mt is dim 8 g + mt, the high nibble of byte 8 g + mt; row g + 8 is dim 64 + 8 g + mt, its
//     low nibble).  Each lane's K half-row and V half-row span two groups, one per nibble.
template <typename T, int BITS>
struct KvHqq {
  static_assert(BITS == 8 || BITS == 4, "8- or 4-bit levels");
  static constexpr int kNg = BITS == 8 ? 2 : 4;
  static constexpr int kStages = BITS == 8 ? 4 : 6, kRowBytes = kHd * BITS / 8, kMetaBytes = kSplitTile * kNg * 2;
  static constexpr int kFreshBytes = 2 * kRowBytes + 4 * kNg * 2;
  static constexpr int kLvlBytes = kSplitTile * kRowBytes, kStageBytes = 2 * kLvlBytes + 4 * kMetaBytes;
  static constexpr int kRingBytes = kSplitWarps * kStages * kStageBytes;  // 136 KB (8 bits), 120 KB (4 bits)
  static constexpr int kSmemBytes = kRingBytes + (kSplitMaxGroup + 2) * kHd * 2 + kFreshBytes + 16;
  static constexpr int kQPair = 2;
  uint8_t* k;
  T* k_s;
  T* k_z;
  uint8_t* v;
  T* v_s;
  T* v_z;
  int gs;
  int ng;  // 128 / gs groups a row

  // group of dim d: d / gs without a division by the run-time gs, which the compiler will not hoist out of the tile loop
  __device__ int grp(int d) const { return d * ng / kHd; }

  __device__ static int slot(int r, int c) {
    if constexpr (BITS == 8) return r * kHd + ((c ^ (r & 7)) << 4);
    else return (r >> 1) * 128 + (((((r & 1) << 2) | c) ^ (((r >> 1) & 3) << 1)) << 4);
  }
  __device__ static int qdim(int kk, int qd) {
    if constexpr (BITS == 8) return 32 * qd + 4 * kk;
    else return kk < 4 ? 16 * qd + 4 * kk : 64 + 16 * qd + 4 * (kk - 4);
  }
  __device__ static int odim(int mt, int g, int hi) {
    if constexpr (BITS == 8) return 16 * g + 2 * mt + hi;
    else return 8 * g + mt + 64 * hi;
  }
  __device__ void advance(long long kv, int L) {
    k += kv * L * kRowBytes; v += kv * L * kRowBytes;
    k_s += kv * L * ng; k_z += kv * L * ng; v_s += kv * L * ng; v_z += kv * L * ng;
  }
  // Meta rows < pos from the cache, row pos from the fresh meta fx once `fresh`, rows past pos zero (they dequantise to 0).  A chunk
  // that reaches row pos (or sits on a misaligned address) is staged row by row.
  __device__ void stage_meta(char* st, long long rt, int t0, int pos, int lane, bool fresh, const char* fx) const {
    if (lane < 8 * ng) {  // 4 arrays x 2 ng chunks
      const T* fm = reinterpret_cast<const T*>(fx + 2 * kRowBytes);
      const int a = lane / (2 * ng), j = lane % (2 * ng), rows = 8 / ng, r0 = j * rows;
      const T* src = (a == 0 ? k_s : a == 1 ? k_z : a == 2 ? v_s : v_z) + (rt + (t0 + r0)) * ng;
      char* dst = st + 2 * kLvlBytes + a * kMetaBytes + j * 16;
      if (t0 + r0 + rows <= pos && ((uintptr_t)src & 15) == 0) {
        split_cp16(dst, src);
      } else {
        for (int e = 0; e < 8; ++e) {
          const int p = t0 + r0 + e / ng;
          if (p < pos) reinterpret_cast<T*>(dst)[e] = src[e];
          else if (p > pos) reinterpret_cast<T*>(dst)[e] = from_f32<T>(0.f);
          else if (fresh) reinterpret_cast<T*>(dst)[e] = fm[kNg * a + e % ng];
        }
      }
    }
  }
  __device__ void patch_meta(char* st, int r, int lane, const char* fx) const {
    if (lane >= 16 && lane < 16 + 4 * ng) {
      const T* fm = reinterpret_cast<const T*>(fx + 2 * kRowBytes);
      const int a = (lane - 16) / ng, e = (lane - 16) % ng;
      reinterpret_cast<T*>(st + 2 * kLvlBytes + a * kMetaBytes)[r * ng + e] = fm[kNg * a + e];
    }
  }
  // Warp 0 quantises the rotated k row kf, warp 1 the v row after it, into the fresh row fx.  In split 0 warps 2 and 3 quantise the same
  // rows into cache row pr: the same bits, from warps that would otherwise wait at the barrier.  Ends with a barrier.
  __device__ void fresh(const T* kf, char* fx, bool write, long long pr, int tid) const {
    const int warp = tid >> 5, lane = tid & 31, isv = warp & 1;
    if (warp < 2 || (write && warp < 4)) {
      float x[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = to_f32<T>(kf[isv * kHd + 4 * lane + j]);
      T* fm = reinterpret_cast<T*>(fx + 2 * kRowBytes);
      const bool own = warp < 2;
      uint8_t* lq = own ? reinterpret_cast<uint8_t*>(fx) + isv * kRowBytes : (isv ? v : k) + pr * kRowBytes;
      T* ls = own ? fm + 2 * isv * kNg : (isv ? v_s : k_s) + pr * ng;
      T* lz = own ? fm + (2 * isv + 1) * kNg : (isv ? v_z : k_z) + pr * ng;
      T sc, ze;
      kv_quant_row<T, BITS>(x, gs, lq, ls, lz, sc, ze);
    }
    __syncthreads();
  }
  // The append's store, as KvF16::put: the row quantised by kv_quant_row into cache row crow (the levels and meta fresh writes for
  // the same row); returns the lane's elements as the cache holds them, T(T(q - z) * s) (kv8_deq2).  Every lane must call it.
  __device__ uint2 put(int isv, long long crow, const T (&x)[4]) const {
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = to_f32<T>(x[j]);
    T sc, ze;
    const uint32_t lv = kv_quant_row<T, BITS>(f, gs, (isv ? v : k) + crow * kRowBytes, (isv ? v_s : k_s) + crow * ng, (isv ? v_z : k_z) + crow * ng, sc, ze);
    typename Pair<T>::type s2, z2;
    s2.x = s2.y = sc;
    z2.x = z2.y = ze;
    uint2 y;
    y.x = kv8_deq2<T, 0>(lv, z2, s2);
    y.y = kv8_deq2<T, 1>(lv, z2, s2);
    return y;
  }
  __device__ void scores(float (&s)[4], const char* st, const uint32_t (&qb)[8][2], int lane) const {
    const int g = lane >> 2, qd = lane & 3;
    const T* ms = reinterpret_cast<const T*>(st + 2 * kLvlBytes);
    constexpr int MA = kMetaBytes / 2;  // T elements per meta array
    if constexpr (BITS == 8) {
      const int gk = grp(32 * qd);  // the group of the lane's K dims
      const uint4 ka0 = *reinterpret_cast<const uint4*>(st + slot(g, 2 * qd)), ka1 = *reinterpret_cast<const uint4*>(st + slot(g, 2 * qd + 1));
      const uint4 kb0 = *reinterpret_cast<const uint4*>(st + slot(g + 8, 2 * qd)), kb1 = *reinterpret_cast<const uint4*>(st + slot(g + 8, 2 * qd + 1));
      typename Pair<T>::type sa, sb, za, zb;  // rows g and g + 8, both halves alike
      sa.x = sa.y = ms[g * ng + gk]; sb.x = sb.y = ms[(g + 8) * ng + gk];
      za.x = za.y = ms[MA + g * ng + gk]; zb.x = zb.y = ms[MA + (g + 8) * ng + gk];
      const uint32_t wa[8] = {ka0.x, ka0.y, ka0.z, ka0.w, ka1.x, ka1.y, ka1.z, ka1.w};
      const uint32_t wb[8] = {kb0.x, kb0.y, kb0.z, kb0.w, kb1.x, kb1.y, kb1.z, kb1.w};
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        uint32_t a[4];
        a[0] = kv8_deq2<T, 0>(wa[kk], za, sa);
        a[2] = kv8_deq2<T, 1>(wa[kk], za, sa);
        a[1] = kv8_deq2<T, 0>(wb[kk], zb, sb);
        a[3] = kv8_deq2<T, 1>(wb[kk], zb, sb);
        mma16816<T>(s, a, qb[kk][0], qb[kk][1]);
      }
    } else {
      const int gkh = grp(16 * qd), gkl = grp(64 + 16 * qd);  // the groups of the lane's K dims (high, low nibbles)
      const uint4 ka = *reinterpret_cast<const uint4*>(st + slot(g, qd)), kb = *reinterpret_cast<const uint4*>(st + slot(g + 8, qd));
      typename Pair<T>::type sah, sal, sbh, sbl, zah, zal, zbh, zbl;  // rows g (a) and g + 8 (b), high and low nibbles
      sah.x = sah.y = ms[g * ng + gkh]; sal.x = sal.y = ms[g * ng + gkl];
      sbh.x = sbh.y = ms[(g + 8) * ng + gkh]; sbl.x = sbl.y = ms[(g + 8) * ng + gkl];
      zah.x = zah.y = ms[MA + g * ng + gkh]; zal.x = zal.y = ms[MA + g * ng + gkl];
      zbh.x = zbh.y = ms[MA + (g + 8) * ng + gkh]; zbl.x = zbl.y = ms[MA + (g + 8) * ng + gkl];
      const uint32_t wa[4] = {ka.x, ka.y, ka.z, ka.w}, wb[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        // bytes 4 w, 4 w + 1 (dims +0, +1) and 4 w + 2, 4 w + 3 (dims +2, +3) of each row, one byte per 16-bit half
        const uint32_t a01 = prmt(wa[w], 0u, 0x4140u), a23 = prmt(wa[w], 0u, 0x4342u);
        const uint32_t b01 = prmt(wb[w], 0u, 0x4140u), b23 = prmt(wb[w], 0u, 0x4342u);
        uint32_t a[4];
        a[0] = kv4_deq2<T>(a01 >> 4, zah, sah); a[1] = kv4_deq2<T>(b01 >> 4, zbh, sbh);
        a[2] = kv4_deq2<T>(a23 >> 4, zah, sah); a[3] = kv4_deq2<T>(b23 >> 4, zbh, sbh);
        mma16816<T>(s, a, qb[w][0], qb[w][1]);
        a[0] = kv4_deq2<T>(a01, zal, sal); a[1] = kv4_deq2<T>(b01, zbl, sbl);
        a[2] = kv4_deq2<T>(a23, zal, sal); a[3] = kv4_deq2<T>(b23, zbl, sbl);
        mma16816<T>(s, a, qb[w + 4][0], qb[w + 4][1]);
      }
    }
  }
  __device__ void pv(float (&o)[8][4], const char* st, uint32_t b0, uint32_t b1, int lane) const {
    const int g = lane >> 2, qd = lane & 3, r0 = 2 * qd;
    const T* vs = reinterpret_cast<const T*>(st + 2 * kLvlBytes + 2 * kMetaBytes);
    const T* vz = reinterpret_cast<const T*>(st + 2 * kLvlBytes + 3 * kMetaBytes);
    const char* vt = st + kLvlBytes;
    if constexpr (BITS == 8) {
      // V^T: positions r = 2 qd + {0, 1, 8, 9}, dims 16 g .. 16 g + 15 (one 16-byte chunk each)
      const int gv = grp(16 * g);  // the group of the lane's V dims
      const uint4 v0 = *reinterpret_cast<const uint4*>(vt + slot(r0, g)), v1 = *reinterpret_cast<const uint4*>(vt + slot(r0 + 1, g));
      const uint4 v8 = *reinterpret_cast<const uint4*>(vt + slot(r0 + 8, g)), v9 = *reinterpret_cast<const uint4*>(vt + slot(r0 + 9, g));
      typename Pair<T>::type s01, s89, z01, z89;  // positions r0, r0 + 1 and r0 + 8, r0 + 9
      s01.x = vs[r0 * ng + gv]; s01.y = vs[(r0 + 1) * ng + gv];
      s89.x = vs[(r0 + 8) * ng + gv]; s89.y = vs[(r0 + 9) * ng + gv];
      z01.x = vz[r0 * ng + gv]; z01.y = vz[(r0 + 1) * ng + gv];
      z89.x = vz[(r0 + 8) * ng + gv]; z89.y = vz[(r0 + 9) * ng + gv];
      const uint32_t w0[4] = {v0.x, v0.y, v0.z, v0.w}, w1[4] = {v1.x, v1.y, v1.z, v1.w};
      const uint32_t w8[4] = {v8.x, v8.y, v8.z, v8.w}, w9[4] = {v9.x, v9.y, v9.z, v9.w};
#pragma unroll
      for (int wi = 0; wi < 4; ++wi) {
        // dims 16 g + 4 wi .. + 3 are bytes 0..3 of word wi; interleave the two positions of each pair: [p.b, p'.b, p.b+1, p'.b+1]
        const uint32_t lo01 = prmt(w0[wi], w1[wi], 0x5140u), hi01 = prmt(w0[wi], w1[wi], 0x7362u);
        const uint32_t lo89 = prmt(w8[wi], w9[wi], 0x5140u), hi89 = prmt(w8[wi], w9[wi], 0x7362u);
        uint32_t a[4];
        // step mt = 2 wi: dims 16 g + 4 wi (+ 1); step 2 wi + 1: dims 16 g + 4 wi + 2 (+ 3)
        a[0] = kv8_deq2<T, 0>(lo01, z01, s01); a[1] = kv8_deq2<T, 1>(lo01, z01, s01);
        a[2] = kv8_deq2<T, 0>(lo89, z89, s89); a[3] = kv8_deq2<T, 1>(lo89, z89, s89);
        mma16816<T>(o[2 * wi], a, b0, b1);
        a[0] = kv8_deq2<T, 0>(hi01, z01, s01); a[1] = kv8_deq2<T, 1>(hi01, z01, s01);
        a[2] = kv8_deq2<T, 0>(hi89, z89, s89); a[3] = kv8_deq2<T, 1>(hi89, z89, s89);
        mma16816<T>(o[2 * wi + 1], a, b0, b1);
      }
    } else {
      // V^T: positions r = 2 qd + {0, 1, 8, 9}, bytes 8 g .. 8 g + 7 (half of chunk g / 2)
      const int gvh = grp(8 * g), gvl = grp(64 + 8 * g);  // the groups of the lane's V dims (high, low nibbles)
      const int cb = 8 * (g & 1);
      const uint2 v0 = *reinterpret_cast<const uint2*>(vt + slot(r0, g >> 1) + cb), v1 = *reinterpret_cast<const uint2*>(vt + slot(r0 + 1, g >> 1) + cb);
      const uint2 v8 = *reinterpret_cast<const uint2*>(vt + slot(r0 + 8, g >> 1) + cb), v9 = *reinterpret_cast<const uint2*>(vt + slot(r0 + 9, g >> 1) + cb);
      typename Pair<T>::type s01h, s01l, s89h, s89l, z01h, z01l, z89h, z89l;  // positions r0, r0 + 1 / r0 + 8, r0 + 9; high / low nibbles
      s01h.x = vs[r0 * ng + gvh]; s01h.y = vs[(r0 + 1) * ng + gvh]; s01l.x = vs[r0 * ng + gvl]; s01l.y = vs[(r0 + 1) * ng + gvl];
      s89h.x = vs[(r0 + 8) * ng + gvh]; s89h.y = vs[(r0 + 9) * ng + gvh]; s89l.x = vs[(r0 + 8) * ng + gvl]; s89l.y = vs[(r0 + 9) * ng + gvl];
      z01h.x = vz[r0 * ng + gvh]; z01h.y = vz[(r0 + 1) * ng + gvh]; z01l.x = vz[r0 * ng + gvl]; z01l.y = vz[(r0 + 1) * ng + gvl];
      z89h.x = vz[(r0 + 8) * ng + gvh]; z89h.y = vz[(r0 + 9) * ng + gvh]; z89l.x = vz[(r0 + 8) * ng + gvl]; z89l.y = vz[(r0 + 9) * ng + gvl];
      const uint32_t w0[2] = {v0.x, v0.y}, w1[2] = {v1.x, v1.y}, w8[2] = {v8.x, v8.y}, w9[2] = {v9.x, v9.y};
#pragma unroll
      for (int mt = 0; mt < 8; ++mt) {
        // byte mt of each position: the two positions of a pair side by side (bits 0..7 and 16..23)
        const uint32_t sel = (mt & 3) | ((4 + (mt & 3)) << 8);
        const uint32_t t01 = prmt(w0[mt >> 2], w1[mt >> 2], sel), t89 = prmt(w8[mt >> 2], w9[mt >> 2], sel);
        uint32_t a[4];
        a[0] = kv4_deq2<T>(t01 >> 4, z01h, s01h); a[1] = kv4_deq2<T>(t01, z01l, s01l);
        a[2] = kv4_deq2<T>(t89 >> 4, z89h, s89h); a[3] = kv4_deq2<T>(t89, z89l, s89l);
        mma16816<T>(o[mt], a, b0, b1);
      }
    }
  }
};

// grid = (S, n_kv, batch), block = 256.  q / out [batch, n_q * 128], k / v [batch, n_kv * 128], the cache arrays of cc [batch, n_kv, L, .].
// part: [batch, n_kv, S, G, 2 + 128] floats (m, l, o per head), tickets: [batch, n_kv] uint32, zero between launches.
// SEQPOS: sequence b at its own position pos_p[b]; its chunk, staged rows, RoPE row and written row follow it (S stays fixed).
// PAGED (SEQPOS only): the cache arrays are page pools [pages, n_kv, 64, .]; a tile's rows are found with one read of the table row.
template <typename T, class Cache, bool SEQPOS = false, bool PAGED = false>
__global__ void __launch_bounds__(kSplitThreads, 1)
    rope_attn_decode_split_kernel(const T* __restrict__ q_in, const T* __restrict__ k_in, const T* __restrict__ v_in, const T* __restrict__ cos_t,
                                  const T* __restrict__ sin_t, Cache cc, const long long* __restrict__ pos_p, T* __restrict__ out,
                                  float* __restrict__ part, unsigned* __restrict__ tickets, int n_q, int n_kv, int L, float scale_log2,
                                  const PageArg<PAGED> pg) {
  extern __shared__ __align__(16) char smem[];
  constexpr int NW = kSplitWarps, ST = Cache::kStages, CH = Cache::kRowBytes / 16;  // CH: 16-byte chunks a level row
  static_assert(NW * kSplitMaxGroup * kPartFloats * 4 <= Cache::kRingBytes, "the warp partials reuse the ring");
  static_assert(SEQPOS || !PAGED, "a paged cache needs per-sequence positions");
  const int S = (int)gridDim.x, split = (int)blockIdx.x, kvh = (int)blockIdx.y, b = (int)blockIdx.z;
  const int G = n_q / n_kv;
  const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
  const int* tab = nullptr;
  if constexpr (PAGED) tab = pg.table + (long long)b * (L / kPage);
  {
    const long long kv = (long long)b * n_kv + kvh;
    if constexpr (!PAGED) cc.advance(kv, L);
    k_in += kv * kHd; v_in += kv * kHd;
    q_in += ((long long)b * n_q + (long long)kvh * G) * kHd; out += ((long long)b * n_q + (long long)kvh * G) * kHd;
    part += kv * S * G * kPartFloats;
    tickets += kv;
  }
  char* ring = smem + warp * ST * Cache::kStageBytes;
  T* qs = reinterpret_cast<T*>(smem + Cache::kRingBytes);  // rotated q [8][128]
  T* kf = qs + kSplitMaxGroup * kHd;                        // rotated k and v of position pos
  T* vf = kf + kHd;
  char* fx = reinterpret_cast<char*>(vf + kHd);  // the format's fresh row pos, if the rotated rows are not that
  const char* fr = Cache::kFreshBytes ? fx : reinterpret_cast<const char*>(kf);  // fresh K levels, the V levels kRowBytes later
  int* last = reinterpret_cast<int*>(fx + Cache::kFreshBytes);

  // *pos was written by a completed launch (the step's final, non-programmatic kernel): it may be read before the wait
  const int pos = (int)pos_p[SEQPOS ? b : 0], n_pos = pos + 1;
  const int chunk = (((n_pos + S - 1) / S) + kSplitTile - 1) / kSplitTile * kSplitTile;
  const int c0 = min(split * chunk, n_pos), c1 = min(c0 + chunk, n_pos);
  const int n_tiles = (c1 - c0 + kSplitTile - 1) / kSplitTile;
  const int my_tiles = warp < n_tiles ? (n_tiles - warp + NW - 1) / NW : 0;  // tiles warp, warp + NW, ... of the chunk
  pdl_launch_dependents();

  // Stage local tile i into its ring slot: rows < pos from the cache (cp.async), row pos from this launch's fresh row once `fresh`
  // (the cache row is written by another CTA of this launch), rows past pos zero (finite: their probability is 0).
  auto issue = [&](int i, bool fresh) {
    if (i < my_tiles) {
      const int t0 = c0 + (warp + i * NW) * kSplitTile;
      char* st = ring + (i % ST) * Cache::kStageBytes;
      long long rt = 0;  // cache row of position 0 of the tile's page, minus the page's first position
      if constexpr (PAGED) rt = page_row(tab, n_kv, kvh, t0) - t0;
#pragma unroll 4
      for (int j = lane; j < 2 * kSplitTile * CH; j += 32) {
        const int isv = j / (kSplitTile * CH), r = (j / CH) % kSplitTile, c = j % CH, p = t0 + r;
        char* dst = st + isv * Cache::kLvlBytes + Cache::slot(r, c);
        if (p < pos) {
          split_cp16(dst, reinterpret_cast<const char*>(isv ? cc.v : cc.k) + (rt + p) * Cache::kRowBytes + c * 16);
        } else if (p > pos || fresh) {
          uint4 val;
          val.x = val.y = val.z = val.w = 0u;
          if (p == pos) val = *reinterpret_cast<const uint4*>(fr + isv * Cache::kRowBytes + c * 16);
          *reinterpret_cast<uint4*>(dst) = val;
        }
      }
      cc.stage_meta(st, rt, t0, pos, lane, fresh, fx);
    }
    split_commit();  // always (possibly empty): every iteration waits on the same group count
  };
  // cache rows < pos were written by earlier launches: the first ST - 1 tiles stream in under the previous kernel's tail
#pragma unroll
  for (int i = 0; i < ST - 1; ++i) issue(i, false);
  pdl_wait();

  for (int i = tid; i < (G + 1) * kHd; i += kSplitThreads) {
    const int h = i >> 7, d = i & (kHd - 1);
    const T r = rope_rounded<T>(h < G ? q_in + h * kHd : k_in, d, cos_t + (long long)pos * kHd, sin_t + (long long)pos * kHd);
    if (h < G) {
      qs[h * kHd + d] = r;
    } else {
      kf[d] = r;
      vf[d] = v_in[d];
    }
  }
  __syncthreads();
  long long pr = pos;  // cache row of position pos: one writer per (sequence, kv head), split 0
  if constexpr (PAGED) {
    if (split == 0) pr = page_row(tab, n_kv, kvh, pos);
  }
  cc.fresh(kf, fx, split == 0, pr, tid);
  if (pos >= c0 && pos < c1) {  // row pos in a tile staged before the wait: its owner fills it in now
    const int ti = (pos - c0) / kSplitTile, i = ti / NW;
    if (ti % NW == warp && i < ST - 1) {
      const int r = pos - (c0 + ti * kSplitTile);
      char* st = ring + (i % ST) * Cache::kStageBytes;
      if (lane < 2 * CH) {
        const int isv = lane / CH, c = lane % CH;
        *reinterpret_cast<uint4*>(st + isv * Cache::kLvlBytes + Cache::slot(r, c)) = *reinterpret_cast<const uint4*>(fr + isv * Cache::kRowBytes + c * 16);
      }
      cc.patch_meta(st, r, lane, fx);
    }
  }
  // Q^T fragments (B operand of the score MMA, n = head g) in the format's dims
  uint32_t qb[8][2];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const T* qr = qs + g * kHd + Cache::qdim(kk, qd);
    qb[kk][0] = g < G ? *reinterpret_cast<const uint32_t*>(qr) : 0u;
    qb[kk][1] = g < G ? *reinterpret_cast<const uint32_t*>(qr + Cache::kQPair) : 0u;
  }

  // lane (g, qd) holds the running max / sum of heads 2 qd, 2 qd + 1 and O^T rows g (+ 8) of each step mt of those heads
  float o[8][4];
#pragma unroll
  for (int mt = 0; mt < 8; ++mt) o[mt][0] = o[mt][1] = o[mt][2] = o[mt][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int i = 0; i < my_tiles; ++i) {
    __syncwarp();  // every lane is done with the slot the next issue overwrites
    issue(i + ST - 1, true);
    split_wait<ST - 1>();
    __syncwarp();  // this tile's copies and plain stores of every lane are visible to the warp
    const char* st = ring + (i % ST) * Cache::kStageBytes;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    cc.scores(s, st, qb, lane);
    uint32_t b0, b1;  // every tile holds position c0 + 16 j < c1
    softmax_tile<T, false>(s, scale_log2, c0 + (warp + i * NW) * kSplitTile + g, c1, c1, m, l, o, g, qd, b0, b1);
    cc.pv(o, st, b0, b1, lane);
  }
  split_wait<0>();
  __syncthreads();  // every warp is done with the ring: it now holds the warp partials [NW][8][m, l, o[128]]
  float* wp = reinterpret_cast<float*>(smem);
  put_partial<Cache>(wp + (warp * kSplitMaxGroup + 2 * qd) * kPartFloats, m, l, o, g);
  __syncthreads();
  split_merge<T, kSplitMaxGroup>(wp, part, tickets, last, S, split, G, G, tid, [&](int h) { return out + h * kHd; });
}

int split_count(int n_kv, int cache_len) {
  const int by_sm = sm_count() / n_kv;
  const int by_len = (int)cdiv(cache_len, kSplitTile);
  return max(1, min(by_sm, by_len));
}

// Speculative verify attention (DESIGN.md 3.5): slot b feeds T = K + 1 rows at positions pos[b] .. pos[b] + T - 1, of which the
// n[b] = min(T, L - pos[b]) that fit in the cache are valid; row t attends over cache rows 0 .. pos[b] + t.  The schedule is
// rope_attn_decode_split_kernel's -- grid (S, ., batch) with S fixed at launch, 16-position tiles through per-warp 3-stage cp.async
// rings, K.Q^T and V^T.P^T on mma.sync m16n8k16, online softmax in fp32, a ticketed merge in split order -- with three changes:
//   - the MMA n dimension is the (t, h) columns of one GQA group, column c = t G + h (T G <= 64), in n-tiles of 8.  A CTA holds
//     kVerTiles n-tiles; the column groups of a kv head are spread over grid.y = n_kv * n_cg, each re-reading the same chunk;
//   - every attended row comes from the cache (the DEVPOS append writes rows pos .. pos + n - 1 just before this launch).  Rows < pos
//     may be staged before griddepcontrol.wait; rows pos .. are loaded after it.  Each chunk covers [0, pos + n);
//   - column (t, h) masks key positions > pos + t.  A tile can lie wholly past a column's last key, so the running max is guarded
//     (a column with no key yet keeps m = -inf, l = 0, o = 0).
// q / out [batch T, n_q 128] (row b T + t, q rotated), caches [batch, n_kv, L, 128] or (PAGED) pools [pages, n_kv, 64, 128].
// part [batch, n_kv, n_cg, S, 8 kVerTiles, 2 + 128] floats, tickets [batch, n_kv, n_cg] uint32, zero between launches.
// KV8: the caches hold HQQ 8-bit levels (uint8, same layout) with meta [.., 128 / gs] T; each staged 16-byte chunk is the
// dequantisation T(T(q - z) * s) of 8 levels (kv8_deq2, what hqq_b200_dequantize gives), loaded and stored synchronously instead of
// through cp.async; the tile layout, the MMAs and everything after them are those of the 16-bit cache.  KV8 with BITS 4: the 4-bit
// cache (packed levels [.., 64], gs 32 or 64); chunk c's 8 levels are the high (c < 8) or low nibbles of bytes 8 (c % 8) .. + 7.
constexpr int kVerTiles = 2;                     // n-tiles per CTA (no spills at 2: DESIGN.md 3.5)
constexpr int kVerCols = 8 * kVerTiles;          // columns per CTA
constexpr int kVerMaxCols = 64;                  // T G
constexpr int kVerMaxT = 8;                      // K + 1
static_assert(kSplitWarps * kVerCols * kPartFloats * 4 <= kRingBytes, "the warp partials reuse the ring");
template <typename T> struct Kv8Meta { const T* k_s; const T* k_z; const T* v_s; const T* v_z; int gs; };
struct NoKv8 {};
template <typename T, bool KV8> using Kv8Arg = typename std::conditional<KV8, Kv8Meta<T>, NoKv8>::type;
template <typename T, bool KV8> using CacheT = typename std::conditional<KV8, uint8_t, T>::type;

template <typename T, bool PAGED = false, bool KV8 = false, int BITS = 8>
__global__ void __launch_bounds__(kSplitThreads, 1)
    attn_verify_split_kernel(const T* __restrict__ q, const CacheT<T, KV8>* __restrict__ k_cache, const CacheT<T, KV8>* __restrict__ v_cache,
                             const long long* __restrict__ pos_p, T* __restrict__ out, float* __restrict__ part, unsigned* __restrict__ tickets, int n_q,
                             int n_kv, int L, int TQ, float scale_log2, const PageArg<PAGED> pg, Kv8Arg<T, KV8> m8) {
  extern __shared__ __align__(16) char smem[];
  constexpr int NW = kSplitWarps, ST = kSplitStages, NT = kVerTiles, NC = kVerCols;
  const int G = n_q / n_kv, C = TQ * G, n_cg = (C + NC - 1) / NC;
  const int S = (int)gridDim.x, split = (int)blockIdx.x, kvh = (int)blockIdx.y / n_cg, cg = (int)blockIdx.y % n_cg, b = (int)blockIdx.z;
  const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
  constexpr int RW = KV8 ? kHd * BITS / 8 : kHd;  // cache elements a row
  const int* tab = nullptr;
  if constexpr (PAGED) tab = pg.table + (long long)b * (L / kPage);
  {
    const long long kv = (long long)b * n_kv + kvh;
    if constexpr (!PAGED) {
      k_cache += kv * L * RW; v_cache += kv * L * RW;
      if constexpr (KV8) {
        const int ng = kHd / m8.gs;
        m8.k_s += kv * L * ng; m8.k_z += kv * L * ng; m8.v_s += kv * L * ng; m8.v_z += kv * L * ng;
      }
    }
    part += (kv * n_cg + cg) * S * NC * kPartFloats;
    tickets += kv * n_cg + cg;
  }
  char* ring = smem + warp * ST * kStageBytes;
  int* last = reinterpret_cast<int*>(smem + kRingBytes);

  // *pos was written by a completed launch (the previous step's accept kernel): it may be read before the wait
  const int pos = (int)pos_p[b], end = pos + min(TQ, L - pos);
  const int chunk = (((end + S - 1) / S) + kSplitTile - 1) / kSplitTile * kSplitTile;
  const int c0 = min(split * chunk, end), c1 = min(c0 + chunk, end);
  const int n_tiles = (c1 - c0 + kSplitTile - 1) / kSplitTile;
  const int my_tiles = warp < n_tiles ? (n_tiles - warp + NW - 1) / NW : 0;
  pdl_launch_dependents();

  // 16-byte chunk c of cache row `row` (K or V) into dst: cp.async, or (KV8) 8 levels dequantised with their group's meta
  auto stage16 = [&](char* dst, int isv, long long row, int c, bool async) {
    if constexpr (KV8) {
      uint2 w;
      if constexpr (BITS == 8) {
        w = *reinterpret_cast<const uint2*>((isv ? v_cache : k_cache) + row * kHd + c * 8);
      } else {
        const uint2 p = *reinterpret_cast<const uint2*>((isv ? v_cache : k_cache) + row * RW + (c & 7) * 8);
        w.x = kv4_unpack(p.x, c < 8);
        w.y = kv4_unpack(p.y, c < 8);
      }
      const long long mi = row * (kHd / m8.gs) + (c * 8) / m8.gs;
      typename Pair<T>::type s2, z2;
      s2.x = s2.y = (isv ? m8.v_s : m8.k_s)[mi];
      z2.x = z2.y = (isv ? m8.v_z : m8.k_z)[mi];
      uint4 o;
      o.x = kv8_deq2<T, 0>(w.x, z2, s2); o.y = kv8_deq2<T, 1>(w.x, z2, s2);
      o.z = kv8_deq2<T, 0>(w.y, z2, s2); o.w = kv8_deq2<T, 1>(w.y, z2, s2);
      *reinterpret_cast<uint4*>(dst) = o;
    } else if (async) {
      split_cp16(dst, (isv ? v_cache : k_cache) + row * kHd + c * 8);
    } else {
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>((isv ? v_cache : k_cache) + row * kHd + c * 8);
    }
  };
  // Stage local tile i into its ring slot: rows below lim from the cache (cp.async), rows past the chunk zero (finite, P = 0).
  // Before the wait lim = pos; rows pos .. c1 - 1 of those tiles are filled in after it.
  auto issue = [&](int i, int lim) {
    if (i < my_tiles) {
      const int t0 = c0 + (warp + i * NW) * kSplitTile;
      char* st = ring + (i % ST) * kStageBytes;
      long long rt = 0;
      if constexpr (PAGED) rt = page_row(tab, n_kv, kvh, t0) - t0;
#pragma unroll 4
      for (int j = lane; j < 2 * kSplitTile * 16; j += 32) {
        const int isv = j >> 8, r = (j >> 4) & 15, c = j & 15, p = t0 + r;
        char* dst = st + isv * kTileBytes + swz(r, c);
        if (p < c1) {
          if (p < lim) stage16(dst, isv, rt + p, c, true);
        } else {
          uint4 z;
          z.x = z.y = z.z = z.w = 0u;
          *reinterpret_cast<uint4*>(dst) = z;
        }
      }
    }
    split_commit();
  };
#pragma unroll
  for (int i = 0; i < ST - 1; ++i) issue(i, pos);
  pdl_wait();
  for (int i = 0; i < ST - 1 && i < my_tiles; ++i) {  // rows pos .. of the tiles staged before the wait, written by the append
    const int t0 = c0 + (warp + i * NW) * kSplitTile;
    if (t0 + kSplitTile <= pos) continue;
    char* st = ring + (i % ST) * kStageBytes;
    long long rt = 0;
    if constexpr (PAGED) rt = page_row(tab, n_kv, kvh, t0) - t0;
    for (int j = lane; j < 2 * kSplitTile * 16; j += 32) {
      const int isv = j >> 8, r = (j >> 4) & 15, c = j & 15, p = t0 + r;
      if (p >= pos && p < c1) stage16(st + isv * kTileBytes + swz(r, c), isv, rt + p, c, false);
    }
  }
  // Q^T fragments of n-tile j: column cg NC + 8 j + g = (t, h); columns past T G are zero.  Lane (g, qd) owns the scores of columns
  // 8 j + 2 qd + {0, 1}; lim[j][u] is the first key position such a column does not see.
  uint32_t qb[NT][8][2];
  int lim[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int col = cg * NC + 8 * j + g;
    const bool ok = col < C;
    const T* qr = q + (((long long)b * TQ + (ok ? col / G : 0)) * n_q + (long long)kvh * G + (ok ? col % G : 0)) * kHd + 2 * qd;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      qb[j][kk][0] = ok ? *reinterpret_cast<const uint32_t*>(qr + kk * 16) : 0u;
      qb[j][kk][1] = ok ? *reinterpret_cast<const uint32_t*>(qr + kk * 16 + 8) : 0u;
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int cu = cg * NC + 8 * j + 2 * qd + u;
      lim[j][u] = cu < C ? min(pos + cu / G + 1, c1) : c1;
    }
  }

  float o[NT][8][4];
  float m[NT][2], l[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int mt = 0; mt < 8; ++mt) o[j][mt][0] = o[j][mt][1] = o[j][mt][2] = o[j][mt][3] = 0.f;
    m[j][0] = m[j][1] = -INFINITY;
    l[j][0] = l[j][1] = 0.f;
  }
  const int kr = (lane & 7) + ((lane >> 3) & 1) * 8, kc = lane >> 4;
  const int vr = (lane & 7) + ((lane >> 4) & 1) * 8, vc = (lane >> 3) & 1;
  for (int i = 0; i < my_tiles; ++i) {
    __syncwarp();
    issue(i + ST - 1, c1);
    split_wait<ST - 1>();
    __syncwarp();
    const char* kt = ring + (i % ST) * kStageBytes;
    const char* vt = kt + kTileBytes;
    float s[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      uint32_t a[4];
      ldsm4<false>(a, kt + swz(kr, 2 * kk + kc));
#pragma unroll
      for (int j = 0; j < NT; ++j) mma16816<T>(s[j], a, qb[j][kk][0], qb[j][kk][1]);
    }
    const int p0 = c0 + (warp + i * NW) * kSplitTile + g;
    uint32_t pb[NT][2];
#pragma unroll
    for (int j = 0; j < NT; ++j) softmax_tile<T, true>(s[j], scale_log2, p0, lim[j][0], lim[j][1], m[j], l[j], o[j], g, qd, pb[j][0], pb[j][1]);
#pragma unroll
    for (int mt = 0; mt < 8; ++mt) {
      uint32_t a[4];
      ldsm4<true>(a, vt + swz(vr, 2 * mt + vc));
#pragma unroll
      for (int j = 0; j < NT; ++j) mma16816<T>(o[j][mt], a, pb[j][0], pb[j][1]);
    }
  }
  split_wait<0>();
  __syncthreads();  // every warp is done with the ring: it now holds the warp partials [NW][NC][m, l, o[128]]
  float* wp = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int j = 0; j < NT; ++j) put_partial<KvF16<T>>(wp + (warp * NC + 8 * j + 2 * qd) * kPartFloats, m[j], l[j], o[j], g);
  __syncthreads();
  split_merge<T, NC>(wp, part, tickets, last, S, split, NC, min(NC, C - cg * NC), tid, [&](int c) {  // this CTA's real columns
    const int col = cg * NC + c;
    return out + (((long long)b * TQ + col / G) * n_q + (long long)kvh * G + col % G) * kHd;
  });
}

// Prompt-lookup drafts (DESIGN.md 3.5).  Slot b knows n = pos[b] + 1 tokens: hist[b][0 .. pos - 1] and tok[b] at pos.  Take the
// longest g in {3, 2, 1} for which some j with j + g <= n - 1 has hist[j .. j + g - 1] == the last g known tokens, the largest such
// j, and draft d_{i+1} = token j + g + i while j + g + i < n, else -1; no match: every draft -1.  grid = batch, block = kNgramThreads:
// one pass over j with the three match lengths, then block max reductions.
constexpr int kNgramThreads = 512;
__global__ void __launch_bounds__(kNgramThreads) ngram_draft_kernel(const int* __restrict__ hist, const long long* __restrict__ pos_p,
                                                                    const long long* __restrict__ tok, long long* __restrict__ drafts, int L, int K) {
  __shared__ int red[3][kNgramThreads / 32];
  __shared__ int best[3];
  pdl_launch_dependents();
  pdl_wait();
  const int b = (int)blockIdx.x, tid = (int)threadIdx.x;
  const int* h = hist + (long long)b * L;
  const int pos = (int)pos_p[b], n = pos + 1, last = (int)tok[b];
  const int s2 = n >= 2 ? h[n - 2] : 0, s3 = n >= 3 ? h[n - 3] : 0;
  int j1 = -1, j2 = -1, j3 = -1;  // every compared token lies below pos: from hist
  for (int j = tid; j + 1 <= n - 1; j += kNgramThreads) {
    const int a0 = h[j];
    if (a0 == last) j1 = j;
    if (j + 2 <= n - 1) {
      const int a1 = h[j + 1];
      if (a0 == s2 && a1 == last) j2 = j;
      if (j + 3 <= n - 1 && a0 == s3 && a1 == s2 && h[j + 2] == last) j3 = j;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    j1 = max(j1, __shfl_xor_sync(0xffffffffu, j1, o));
    j2 = max(j2, __shfl_xor_sync(0xffffffffu, j2, o));
    j3 = max(j3, __shfl_xor_sync(0xffffffffu, j3, o));
  }
  if ((tid & 31) == 0) { red[0][tid >> 5] = j1; red[1][tid >> 5] = j2; red[2][tid >> 5] = j3; }
  __syncthreads();
  if (tid < 3) {
    int v = -1;
    for (int w = 0; w < kNgramThreads / 32; ++w) v = max(v, red[tid][w]);
    best[tid] = v;
  }
  __syncthreads();
  const int gl = best[2] >= 0 ? 3 : best[1] >= 0 ? 2 : best[0] >= 0 ? 1 : 0;
  const int j = gl ? best[gl - 1] : 0;
  for (int i = tid; i < K; i += kNgramThreads) {
    const int at = j + gl + i;
    drafts[(long long)b * K + i] = (gl && at < n) ? (at == pos ? (long long)last : (long long)h[at]) : -1ll;
  }
}

// Greedy accept (DESIGN.md 3.5): slot b verified the window [tok, d1 .. dK] at pos .. pos + K with targets t_r = argmax of row r.
// n = min(K + 1, L - pos); a = the largest r < n with d_i == t_{i-1} for every i <= r.  Emits d1 .. da, t_a (tokens [batch, K + 1],
// -1 padded), n_new = a + 1; hist[pos .. pos + a] = the accepted window; pos = (pos + a + 1) mod L; tok = next_tok = t_a.
// grid = ceil(batch / 128), block = 128: one thread per slot.
__global__ void __launch_bounds__(128) spec_accept_kernel(const long long* __restrict__ targets, const long long* __restrict__ drafts,
                                                          long long* __restrict__ pos_p, long long* __restrict__ tok, long long* __restrict__ next_tok,
                                                          int* __restrict__ hist, long long* __restrict__ tokens, long long* __restrict__ n_new, int batch,
                                                          int K, int L) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (b >= batch) return;
  const int T = K + 1, pos = (int)pos_p[b], n = min(T, L - pos);
  const long long* tg = targets + (long long)b * T;
  const long long* d = drafts + (long long)b * K;
  int a = 0;
  while (a + 1 < n && d[a] == tg[a]) ++a;
  int* hr = hist + (long long)b * L;
  hr[pos] = (int)tok[b];
  for (int i = 1; i <= a; ++i) hr[pos + i] = (int)d[i - 1];
  for (int i = 0; i < T; ++i) tokens[(long long)b * T + i] = i < a ? d[i] : (i == a ? tg[a] : -1ll);
  pos_p[b] = (pos + a + 1) % L;
  tok[b] = next_tok[b] = tg[a];
  n_new[b] = a + 1;
}

// Prompt prefill (DESIGN.md 3.5): a chunk of T positions pos0 .. pos0 + T - 1 of every sequence.
//
// rope_append_rows_kernel writes rope(k) and v into cache rows [pos0, pos0 + T) and rope(q) into q_out, rounding exactly as
// rope_attn_decode_kernel does, so a cache row is bit for bit the row a decode step writes from the same k and v.
//
// attn_prefill_kernel: causal GQA attention of the chunk's T queries over cache rows 0 .. pos0 + t (FlashAttention-2 style on
// mma.sync m16n8k16).  A CTA owns 128 rows (t, h) = (row / G, row % G) of one (kv head, sequence), so each K/V tile is staged once
// for all G <= 8 heads of the group; each of the 8 warps owns 16 rows for the whole key range:
//   S [16 rows x 64 positions]  = Q [16 x 128] . K^T        (Q fragments in registers, K from shared memory through ldmatrix)
//   O [16 rows x 128 dims]     += P [16 x 64]  . V           (P from the S accumulators, V through ldmatrix.trans, O in fp32)
// K/V tiles of 64 positions, aligned to absolute positions, stream through a 3-stage cp.async ring shared by the CTA (16-byte
// chunks XOR-swizzled by row).  Rows at or past pos0 + T are never loaded: their slots are zero.  Online softmax in fp32 with
// exp2f; P is rounded to T for the second MMA and the row sum adds the rounded values; one rounding to T at the end.  A tile that
// lies wholly past a row's position leaves its m, l and o bit for bit unchanged (scale 1, P = 0), and tile 0 -- which every row
// sees -- comes first, so a row's output depends only on its q row and cache rows 0 .. p: not on pos0 / T chunking, batch or
// which rows share its CTA.  No atomics, no workspace.  Query blocks with the longest key range are scheduled first.
constexpr int kPreWarps = 8;
constexpr int kPreThreads = 32 * kPreWarps;
constexpr int kPreRows = 16 * kPreWarps;                  // (position, head) rows per CTA
constexpr int kPreTile = 64;                              // key positions per tile
constexpr int kPreStages = 3;
constexpr int kPreTileBytes = kPreTile * kHd * 2;         // one K or V tile, 16 KB
constexpr int kPreStageBytes = 2 * kPreTileBytes;
constexpr int kPreSmemBytes = kPreStages * kPreStageBytes;  // 96 KB

// Variable-length prefill (VARLEN instantiations of the prefill attention, the VarlenRows layout of the append and the staging refill):
// slot b contributes n_tok[b] >= 0 rows at positions pos0[b] .. pos0[b] + n_tok[b] - 1, packed in slot order from token row row0[b] =
// sum of n_tok[b'] for b' < b (equal lengths give the b T + t layout).  The grids are sized by the longest slot; CTAs past their slot's
// rows exit, so a slot with no rows is neither read nor written.  The arrays travel by value in the parameter block (3 KB), so a launch
// needs no upload and no workspace.
//
// The row layouts of rope_append_rows_kernel: place(t, b, L, p, row) gives CTA (t, b) = (blockIdx.x, blockIdx.y) its position p and
// token row, or returns false when the CTA has nothing to do; kStages says whether the layout writes staging rows.
constexpr int kVarlenMaxBatch = 256;
struct VarlenRows {
  int pos0[kVarlenMaxBatch];
  int n_tok[kVarlenMaxBatch];
  int row0[kVarlenMaxBatch];
  static constexpr bool kStages = true;
  __device__ bool place(int t, int b, int, int& p, long long& row) const {
    if (t >= n_tok[b]) return false;  // past this slot's rows
    p = pos0[b] + t;
    row = (long long)row0[b] + t;
    return true;
  }
};
struct NoVarlen {};  // the fixed-length instantiations: their uniform pos0 / T are the scalar arguments
template <bool VARLEN> using VarlenArg = typename std::conditional<VARLEN, VarlenRows, NoVarlen>::type;
// The fixed-length append: T rows a slot at the uniform positions pos0 .. pos0 + T - 1, row b T + t.
struct FixedRows {
  int pos0, T;
  static constexpr bool kStages = true;
  __device__ bool place(int t, int b, int, int& p, long long& row) const {
    p = pos0 + t;
    row = (long long)b * T + t;
    return true;
  }
};
// Device positions (the speculative verify step): slot b's T rows b T + t go to positions pos[b] + t, and only the
// n[b] = min(T, L - pos[b]) rows that fit in the cache are rotated and written.  pos is read before griddepcontrol.wait, so it must
// have been written by an earlier, completed launch (the previous step's accept kernel).  No staging rows: the verify attention
// dequantises the cache itself.
struct DevPos {
  const long long* pos;
  int T;
  static constexpr bool kStages = false;
  __device__ bool place(int t, int b, int L, int& p, long long& row) const {
    const int p0 = (int)pos[b];
    if (t >= L - p0) return false;  // past the end of the cache: neither written nor rotated
    p = p0 + t;
    row = (long long)b * T + t;
    return true;
  }
};

// The prefill and verify append of every cache format and row layout.  Each k and v row goes to the cache through the format's put:
// KvF16 copies it, KvHqq quantises it as the split decode kernel quantises row pos (the same levels and meta bit for bit).  A quantised
// format under a staging layout also writes the row as the cache holds it to the staging pair k_st / v_st [batch, n_kv, L, 128] T at
// the same row, which the prefill attention reads.
// grid = (T | max T, batch), block = 256: threads take the q elements in turn, then warp w the rows w, w + 8, ... of the 2 n_kv rows
// of a position (k and v of each kv head), four elements per lane.  q / q_out [rows, n_q 128], k / v [rows, n_kv 128], caches
// [batch, n_kv, L, .] in the format's layout.  PAGED: page pools (the staging pair stays contiguous), the CTA's position found with one
// table read.
template <typename T, typename Cache, typename Rows, bool PAGED>
__global__ void __launch_bounds__(256) rope_append_rows_kernel(const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v,
                                                               const T* __restrict__ cos_t, const T* __restrict__ sin_t, const Cache cache,
                                                               T* __restrict__ k_st, T* __restrict__ v_st, T* __restrict__ q_out, int n_q, int n_kv,
                                                               int L, const Rows rows, const PageArg<PAGED> pg) {
  static_assert(!PAGED || !std::is_same<Rows, FixedRows>::value, "a paged cache needs per-slot positions");
  constexpr bool kStage = Rows::kStages && !std::is_same<Cache, KvF16<T>>::value;
  const int b = (int)blockIdx.y;
  int p;
  long long row;
  if (!rows.place((int)blockIdx.x, b, L, p, row)) return;
  Cache c = cache;
  {
    const long long kv = (long long)b * n_kv;
    q += row * n_q * kHd; q_out += row * n_q * kHd;
    k += row * n_kv * kHd; v += row * n_kv * kHd;
    if constexpr (!PAGED) c.advance(kv, L);
    if constexpr (kStage) { k_st += kv * L * kHd; v_st += kv * L * kHd; }
  }
  long long c0 = 0;  // PAGED: pool row of position p of kv head 0
  if constexpr (PAGED) c0 = page_row(pg.table + (long long)b * (L / kPage), n_kv, 0, p);
  pdl_launch_dependents();
  pdl_wait();
  const T* cs = cos_t + (long long)p * kHd;
  const T* sn = sin_t + (long long)p * kHd;
  for (int i = (int)threadIdx.x; i < n_q * kHd; i += (int)blockDim.x) {
    const int h = i >> 7, d = i & (kHd - 1);
    q_out[h * kHd + d] = rope_rounded<T>(q + h * kHd, d, cs, sn);
  }
  const int warp = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  for (int r = warp; r < 2 * n_kv; r += (int)blockDim.x >> 5) {
    const int kvh = r >> 1, isv = r & 1;
    T x[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = isv ? v[kvh * kHd + 4 * lane + j] : rope_rounded<T>(k + kvh * kHd, 4 * lane + j, cs, sn);
    const long long crow = PAGED ? c0 + (long long)kvh * kPage : (long long)kvh * L + p;
    const uint2 y = c.put(isv, crow, x);
    if constexpr (kStage) *reinterpret_cast<uint2*>((isv ? v_st : k_st) + ((long long)kvh * L + p) * kHd + 4 * lane) = y;
  }
}

// Prefill into a paged 8-bit cache: staging rows [0, pos0[b]) of every slot with n_tok[b] > 0, dequantised from the page pools through
// the table with the rows kernel's arithmetic (kv8_deq2: T(T(q - z) * s), what hqq_b200_dequantize gives).  grid = (max pos0, batch),
// block = 256: warp w takes rows w, w + 8, ... of the 2 n_kv rows of a position, four elements per lane.  The table is read before the
// wait, the pools after it.  BITS 4: the 4-bit cache (lane l unpacks the high nibbles of bytes 4 l .. 4 l + 3, lane 16 + l their
// low nibbles).  PAGED false (BITS 4 only): the contiguous caches [batch, n_kv, L, .], pg unused.
template <typename T, int BITS = 8, bool PAGED = true>
__global__ void __launch_bounds__(256) kv8_stage_paged_kernel(const uint8_t* __restrict__ k_q, const T* __restrict__ k_s, const T* __restrict__ k_z,
                                                              const uint8_t* __restrict__ v_q, const T* __restrict__ v_s, const T* __restrict__ v_z,
                                                              T* __restrict__ k_st, T* __restrict__ v_st, int n_kv, int L, int gs, const VarlenRows vl,
                                                              const PageArg<PAGED> pg) {
  constexpr int LB = kHd * BITS / 8;  // level bytes a row
  const int p = (int)blockIdx.x, b = (int)blockIdx.y, ng = kHd / gs;
  if (vl.n_tok[b] == 0 || p >= vl.pos0[b]) return;  // slot outside the chunk, or a row the rows kernel writes
  long long c0;  // cache row of position p of kv head 0; kv head h at c0 + h * rs
  long long rs;
  if constexpr (PAGED) {
    c0 = page_row(pg.table + (long long)b * (L / kPage), n_kv, 0, p);
    rs = kPage;
  } else {
    c0 = (long long)b * n_kv * L + p;
    rs = L;
  }
  pdl_launch_dependents();
  pdl_wait();
  const int warp = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  for (int r = warp; r < 2 * n_kv; r += (int)blockDim.x >> 5) {
    const int kvh = r >> 1, isv = r & 1, grp = 4 * lane / gs;
    const long long crow = c0 + (long long)kvh * rs;
    uint32_t lv;
    if constexpr (BITS == 8) lv = *reinterpret_cast<const uint32_t*>((isv ? v_q : k_q) + crow * kHd + 4 * lane);
    else lv = kv4_unpack(*reinterpret_cast<const uint32_t*>((isv ? v_q : k_q) + crow * LB + 4 * (lane & 15)), lane < 16);
    typename Pair<T>::type s2, z2;
    s2.x = s2.y = (isv ? v_s : k_s)[crow * ng + grp];
    z2.x = z2.y = (isv ? v_z : k_z)[crow * ng + grp];
    uint2 y;
    y.x = kv8_deq2<T, 0>(lv, z2, s2);
    y.y = kv8_deq2<T, 1>(lv, z2, s2);
    *reinterpret_cast<uint2*>((isv ? v_st : k_st) + (((long long)b * n_kv + kvh) * L + p) * kHd + 4 * lane) = y;
  }
}

// grid = (n_kv, batch, ceil(T G / 128)), block = 256: the query block is the slowest grid index, so the blocks with the longest key
// range are dispatched first across all kv heads and sequences.  q (rotated) / out [batch T, n_q 128] (row b T + t), caches
// [batch, n_kv, L, 128].  VARLEN: grid = (n_kv, batch, ceil(max T G / 128)), rows as VarlenRows lays them out; the query blocks
// past a slot's rows exit.  PAGED (VARLEN only): page pools, one table read per 64-position tile (a tile is one page).
template <typename T, bool VARLEN = false, bool PAGED = false>
__global__ void __launch_bounds__(kPreThreads, 1)
    attn_prefill_kernel(const T* __restrict__ q, const T* __restrict__ k_cache, const T* __restrict__ v_cache, T* __restrict__ out, int pos0,
                        int n_tok, int n_q, int n_kv, int L, float scale_log2, const VarlenArg<VARLEN> vl, const PageArg<PAGED> pg) {
  static_assert(VARLEN || !PAGED, "a paged cache needs the variable-length layout");
  static_assert(kPreTile == kPage, "a prefill tile is one page");
  extern __shared__ __align__(16) char smem[];
  constexpr int ST = kPreStages;
  const int G = n_q / n_kv;
  const int rb = (int)(gridDim.z - 1 - blockIdx.z), kvh = (int)blockIdx.x, b = (int)blockIdx.y;  // longest query blocks first
  long long qrow0 = (long long)b * n_tok;  // token row of the slot's first position
  if constexpr (VARLEN) {
    pos0 = vl.pos0[b];
    n_tok = vl.n_tok[b];
    qrow0 = vl.row0[b];
    if (rb * kPreRows >= n_tok * G) return;  // past this slot's query rows
  }
  const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
  if constexpr (!PAGED) {
    const long long kv = (long long)b * n_kv + kvh;
    k_cache += kv * L * kHd; v_cache += kv * L * kHd;
  }
  const int* tab = nullptr;
  if constexpr (PAGED) tab = pg.table + (long long)b * (L / kPage);
  const int n_rows = n_tok * G, row0 = rb * kPreRows;
  const int n_tiles = (pos0 + (min(row0 + kPreRows, n_rows) - 1) / G) / kPreTile + 1;  // through the CTA's last position
  const int lim = pos0 + n_tok;                                                          // rows >= lim are never loaded
  const int wr0 = row0 + warp * 16;
  const int w_end = wr0 < n_rows ? pos0 + (min(wr0 + 15, n_rows - 1)) / G : -1;          // the warp's last position
  // the lane's rows g and g + 8 of the warp: position and q / out row (rows past the chunk compute on zero q and are not stored)
  const int ra = wr0 + g, rb8 = wr0 + g + 8;
  const bool va = ra < n_rows, vb = rb8 < n_rows;
  const int pa = pos0 + (va ? ra / G : n_tok - 1), pb = pos0 + (vb ? rb8 / G : n_tok - 1);
  const long long oa = (qrow0 + (pa - pos0)) * n_q * kHd + (long long)(kvh * G + ra % G) * kHd;
  const long long ob = (qrow0 + (pb - pos0)) * n_q * kHd + (long long)(kvh * G + rb8 % G) * kHd;
  pdl_launch_dependents();
  pdl_wait();

  auto issue = [&](int j) {
    if (j < n_tiles) {
      const int t0 = j * kPreTile;
      char* st = smem + (j % ST) * kPreStageBytes;
      long long rt = 0;  // cache row of position 0 of the tile's page, minus the page's first position
      if constexpr (PAGED) rt = page_row(tab, n_kv, kvh, t0) - t0;
#pragma unroll 4
      for (int c = tid; c < 2 * kPreTile * 16; c += kPreThreads) {
        const int isv = c >> 10, r = (c >> 4) & (kPreTile - 1), ch = c & 15, p = t0 + r;
        char* dst = st + isv * kPreTileBytes + swz(r, ch);
        if (p < lim) {
          split_cp16(dst, (isv ? v_cache : k_cache) + (rt + p) * kHd + ch * 8);
        } else {
          uint4 z;
          z.x = z.y = z.z = z.w = 0u;
          *reinterpret_cast<uint4*>(dst) = z;
        }
      }
    }
    split_commit();  // always (possibly empty): every iteration waits on the same group count
  };
#pragma unroll
  for (int i = 0; i < ST - 1; ++i) issue(i);

  // Q fragments (A operand of the score MMA): rows g, g + 8; dims 16 kk + 2 qd + {0, 1} and + 8
  uint32_t qf[8][4];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const int d = kk * 16 + 2 * qd;
    qf[kk][0] = va ? *reinterpret_cast<const uint32_t*>(q + oa + d) : 0u;
    qf[kk][1] = vb ? *reinterpret_cast<const uint32_t*>(q + ob + d) : 0u;
    qf[kk][2] = va ? *reinterpret_cast<const uint32_t*>(q + oa + d + 8) : 0u;
    qf[kk][3] = vb ? *reinterpret_cast<const uint32_t*>(q + ob + d + 8) : 0u;
  }
  // lane (g, qd) holds m, l (its share of the row sum) and O columns 8 dt + 2 qd + {0, 1} of rows g (index 0) and g + 8 (index 1)
  float o[16][4];
#pragma unroll
  for (int dt = 0; dt < 16; ++dt) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const int kr = (lane & 7) + ((lane >> 4) & 1) * 8, kc = (lane >> 3) & 1;  // K as the B operand: n-tile pairs, then k + 8
  const int vr = (lane & 7) + ((lane >> 3) & 1) * 8, vc = lane >> 4;         // V through .trans: positions + 8, then dims + 8
  for (int j = 0; j < n_tiles; ++j) {
    split_wait<ST - 2>();
    __syncthreads();  // tile j is visible to every warp, and every warp is done with the slot the next issue overwrites
    issue(j + ST - 1);
    const int t0 = j * kPreTile;
    if (t0 > w_end) continue;  // wholly past every row of this warp: it would change nothing
    const char* kt = smem + (j % ST) * kPreStageBytes;
    const char* vt = kt + kPreTileBytes;
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t kb[4];
        ldsm4<false>(kb, kt + swz(16 * np + kr, 2 * kk + kc));
        mma16816<T>(s[2 * np], qf[kk], kb[0], kb[1]);
        mma16816<T>(s[2 * np + 1], qf[kk], kb[2], kb[3]);
      }
    }
    float x0 = -INFINITY, x1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int kp = t0 + 8 * nt + 2 * qd;
      s[nt][0] = kp <= pa ? s[nt][0] * scale_log2 : -INFINITY;
      s[nt][1] = kp + 1 <= pa ? s[nt][1] * scale_log2 : -INFINITY;
      s[nt][2] = kp <= pb ? s[nt][2] * scale_log2 : -INFINITY;
      s[nt][3] = kp + 1 <= pb ? s[nt][3] * scale_log2 : -INFINITY;
      x0 = fmaxf(x0, fmaxf(s[nt][0], s[nt][1]));
      x1 = fmaxf(x1, fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, off));
      x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, off));
    }
    const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);  // finite: tile 0 holds position 0, which every row sees
    const float a0 = exp2f(m0 - n0), a1 = exp2f(m1 - n1);
    m0 = n0; m1 = n1;
    uint32_t pf[8][2];  // P rounded to T, packed as the A operand of the second MMA
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const T e0 = from_f32<T>(exp2f(s[nt][0] - n0)), e1 = from_f32<T>(exp2f(s[nt][1] - n0));
      const T e2 = from_f32<T>(exp2f(s[nt][2] - n1)), e3 = from_f32<T>(exp2f(s[nt][3] - n1));
      r0 += to_f32<T>(e0) + to_f32<T>(e1);
      r1 += to_f32<T>(e2) + to_f32<T>(e3);
      pf[nt][0] = bits16(e0) | (bits16(e1) << 16);
      pf[nt][1] = bits16(e2) | (bits16(e3) << 16);
    }
    l0 = l0 * a0 + r0;
    l1 = l1 * a1 + r1;
#pragma unroll
    for (int dt = 0; dt < 16; ++dt) { o[dt][0] *= a0; o[dt][1] *= a0; o[dt][2] *= a1; o[dt][3] *= a1; }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t pa4[4] = {pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1]};
#pragma unroll
      for (int dp = 0; dp < 8; ++dp) {
        uint32_t vb4[4];
        ldsm4<true>(vb4, vt + swz(16 * kk + vr, 2 * dp + vc));
        mma16816<T>(o[2 * dp], pa4, vb4[0], vb4[1]);
        mma16816<T>(o[2 * dp + 1], pa4, vb4[2], vb4[3]);
      }
    }
  }
  split_wait<0>();
#pragma unroll
  for (int off = 1; off < 4; off <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, off);
    l1 += __shfl_xor_sync(0xffffffffu, l1, off);
  }
#pragma unroll
  for (int dt = 0; dt < 16; ++dt) {
    const int d = dt * 8 + 2 * qd;
    if (va) {
      const T y[2] = {from_f32<T>(o[dt][0] / l0), from_f32<T>(o[dt][1] / l0)};
      *reinterpret_cast<uint32_t*>(out + oa + d) = bits16(y[0]) | (bits16(y[1]) << 16);
    }
    if (vb) {
      const T y[2] = {from_f32<T>(o[dt][2] / l1), from_f32<T>(o[dt][3] / l1)};
      *reinterpret_cast<uint32_t*>(out + ob + d) = bits16(y[0]) | (bits16(y[1]) << 16);
    }
  }
}

// The checks both prefill entry points share; returns HQQ_OK or the error code (message set).
int prefill_args(const char* name, int pos0, int n_tok, int n_q, int n_kv, int L, int hd, int batch, int dtype) {
  HQQ_REQUIRE(dtype == HQQ_F16 || dtype == HQQ_BF16, HQQ_E_INVALID, "%s: dtype must be f16/bf16", name);
  HQQ_REQUIRE(batch > 0 && batch <= 65535, HQQ_E_INVALID, "%s: batch %d", name, batch);
  HQQ_REQUIRE(hd == kHd && n_kv > 0 && n_kv <= 65535 && n_q > 0 && n_q % n_kv == 0 && n_q / n_kv <= kSplitMaxGroup && L > 0 && L <= kSplitMaxLen,
              HQQ_E_UNSUPPORTED, "%s: needs head_dim 128, n_q_heads %% n_kv_heads == 0, n_q_heads / n_kv_heads <= 8, cache_len <= 131072 (got %d, %d/%d, %d)",
              name, hd, n_q, n_kv, L);
  HQQ_REQUIRE(n_tok >= 1 && pos0 >= 0 && n_tok <= L && pos0 <= L - n_tok, HQQ_E_INVALID, "%s: needs 1 <= T and pos0 + T <= cache_len (pos0=%d T=%d cache_len=%d)",
              name, pos0, n_tok, L);
  return HQQ_OK;
}

// The checks of the three variable-length prefill entry points: the shape checks of prefill_args, then the host arrays pos0 / n_tok
// of `batch` slots into vl (with the packed row offsets) and the longest slot's row count into max_t.
int varlen_args(const char* name, const int* pos0, const int* n_tok, int n_q, int n_kv, int L, int hd, int batch, int dtype, VarlenRows& vl,
                int& max_t) {
  HQQ_REQUIRE(pos0 && n_tok, HQQ_E_INVALID, "%s: null pos0 / n_tok", name);
  HQQ_REQUIRE(batch > 0 && batch <= kVarlenMaxBatch, HQQ_E_INVALID, "%s: batch %d (1 .. %d)", name, batch, kVarlenMaxBatch);
  if (int rc = prefill_args(name, 0, 1, n_q, n_kv, L, hd, batch, dtype)) return rc;
  long long rows = 0;
  max_t = 0;
  for (int b = 0; b < batch; ++b) {
    HQQ_REQUIRE(n_tok[b] >= 0 && pos0[b] >= 0 && n_tok[b] <= L && pos0[b] <= L - n_tok[b], HQQ_E_INVALID,
                "%s: slot %d needs 0 <= T, 0 <= pos0 and pos0 + T <= cache_len (pos0=%d T=%d cache_len=%d)", name, b, pos0[b], n_tok[b], L);
    vl.pos0[b] = pos0[b];
    vl.n_tok[b] = n_tok[b];
    vl.row0[b] = (int)rows;
    rows += n_tok[b];
    max_t = max(max_t, n_tok[b]);
    HQQ_REQUIRE(rows <= 65535, HQQ_E_INVALID, "%s: at most 65535 rows in all slots", name);
  }
  HQQ_REQUIRE(rows >= 1, HQQ_E_INVALID, "%s: needs at least one row", name);
  return HQQ_OK;
}

// ---- sampling: temperature, top-k, top-p and a Gumbel race (hqq_b200_glue_sample; the definition is in include/hqq_b200.h) --------
// One CTA of 1024 threads per row.  Each 16-bit value maps to a monotone ordered key (-0 with +0), so the top-k pivot and the top-p
// threshold are keys, found by a radix select: a 256-bin histogram of the high byte, then one of the low byte inside the bin that
// holds the answer.  Counts and fixed-point masses round(w * 2^32), w = exp((l - max) / T) <= 1, are integers summed with shared
// atomics: any order gives the same bits.  Passes over the row: without a filter one (the race); with a filter three --
//   1. high-byte counts and the maximum;
//   2. low-byte counts and masses inside the top-k pivot bin, high-byte masses above it;
//   3. the race over the kept elements.  When the top-p threshold lies in a higher bin than the top-k pivot, this pass also sums
//      the low-byte masses of that bin and keeps one race winner per low byte there; the threshold then picks among those.
// The race skips the Philox draw and the logarithms of an element that cannot win: g <= 16.64, so l / T + 17 below the key of an
// element this thread has already kept is a loss.
constexpr int kSampleThreads = 1024;
constexpr float kGumbelMax = 17.0f;  // above the largest g, -log(-log(1 - 2^-24)) = 16.64

__device__ __forceinline__ uint32_t sample_key(uint32_t bits) {
  if (bits == 0x8000u) bits = 0;  // -0 orders with +0
  return (bits & 0x8000u) ? (~bits & 0xFFFFu) : (bits | 0x8000u);
}

template <typename T> __device__ __forceinline__ float sample_key_value(uint32_t k) {
  const unsigned short bits = (unsigned short)((k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu));
  return to_f32<T>(*reinterpret_cast<const T*>(&bits));
}

// Philox4x32-10 (Salmon et al., SC'11): counter c, key (k0, k1)
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = umulhi32(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = umulhi32(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
  }
}

__device__ __forceinline__ unsigned long long sample_mass(float l, float m, float temperature) {
  return f32_to_u64_rn(expf(__fdiv_rn(__fsub_rn(l, m), temperature)) * 4294967296.0f);
}

// Warp 0: the bin b of bins[0..256) where the sum from bin 255 down first reaches target, and the sum of the bins above b.
// Needs 1 <= target <= the sum of all bins.
template <typename C>
__device__ __forceinline__ void find_from_top(const C* bins, unsigned long long target, int* bin_out, unsigned long long* above_out) {
  const int lane = threadIdx.x & 31;
  unsigned long long s = 0;
  for (int j = 0; j < 8; ++j) s += bins[lane * 8 + j];
  unsigned long long suf = s;  // sum of lanes lane..31
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_sync(0xffffffffu, suf, lane + o < 32 ? lane + o : 31);
    if (lane + o < 32) suf += t;
  }
  unsigned long long above = suf - s;
  if (above < target && target <= suf) {
    for (int j = 7; j >= 0; --j) {
      const unsigned long long c = bins[lane * 8 + j];
      if (above + c >= target) { *bin_out = lane * 8 + j; *above_out = above; break; }
      above += c;
    }
  }
}

// warp sum of bins[0..256)
__device__ __forceinline__ unsigned long long warp_bin_sum(const unsigned long long* bins) {
  unsigned long long s = 0;
  for (int j = 0; j < 8; ++j) s += bins[(threadIdx.x & 31) * 8 + j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// A row's Philox counter words: word 1 in w1, words 2 and 3 returned as one 64-bit value (word 0 is i / 4).  StepKeys (hqq_b200_glue_sample):
// (row, *counter).  PosKeys (hqq_b200_glue_sample_pos): row r is slot r / T at position pos[slot] + r % T, giving (slot, position,
// 0x80000000 | seq[slot] & 0x7FFFFFFF).
struct StepKeys { const unsigned long long* counter; };
struct PosKeys { const long long* pos; const long long* seq; int T; };

__device__ __forceinline__ unsigned long long sample_counter(StepKeys k, uint32_t row, uint32_t& w1) {
  w1 = row;
  return __ldg(k.counter);
}

__device__ __forceinline__ unsigned long long sample_counter(PosKeys k, uint32_t row, uint32_t& w1) {
  const uint32_t slot = row / (uint32_t)k.T;
  const uint32_t p = (uint32_t)(__ldg(k.pos + slot) + (long long)(row - slot * (uint32_t)k.T));
  w1 = slot;
  return (unsigned long long)(0x80000000u | ((uint32_t)__ldg(k.seq + slot) & 0x7FFFFFFFu)) << 32 | p;
}

// A row's temperature, top_k and top_p.  ScalarParams (hqq_b200_glue_sample, _pos): one set for the launch, by value.  SlotParams
// (hqq_b200_glue_sample_slots): device arrays indexed by the slot r / T, read after the PDL wait; temperature 0 asks for the argmax.
struct ScalarParams { float temperature; int top_k; float top_p; static constexpr bool kSlots = false; };
struct SlotParams { const float* temperature; const int* top_k; const float* top_p; int T; static constexpr bool kSlots = true; };

__device__ __forceinline__ void sample_params(ScalarParams p, uint32_t, float& t, int& k, float& tp) { t = p.temperature; k = p.top_k; tp = p.top_p; }

__device__ __forceinline__ void sample_params(SlotParams p, uint32_t row, float& t, int& k, float& tp) {
  const uint32_t slot = row / (uint32_t)p.T;
  t = __ldg(p.temperature + slot); k = __ldg(p.top_k + slot); tp = __ldg(p.top_p + slot);
}

template <typename T, typename Keys, typename Params>
__global__ void __launch_bounds__(kSampleThreads, 1) sample_kernel(const T* __restrict__ logits, int n, long long ld, Params params, uint32_t seed_lo,
                                                                uint32_t seed_hi, Keys keys, long long* __restrict__ out) {
  __shared__ unsigned cnt_hi[256], cnt_lo[256];
  __shared__ unsigned long long mass_hi[256], mass_lo[256], best_lo[256], red[32];
  __shared__ unsigned max_key;
  __shared__ int sel_bin;
  __shared__ unsigned long long sel_above, sel_target;
  const int tid = threadIdx.x;
  const uint32_t row = blockIdx.x;
  const T* x = logits + (long long)row * ld;
  for (int i = tid; i < 256; i += kSampleThreads) { cnt_hi[i] = 0; cnt_lo[i] = 0; mass_hi[i] = 0; mass_lo[i] = 0; best_lo[i] = 0; }
  if (tid == 0) { max_key = 0; sel_bin = 0; sel_above = 0; }
  pdl_launch_dependents();
  pdl_wait();
  float temperature, top_p;
  int top_k;
  sample_params(params, row, temperature, top_k, top_p);
  const bool greedy = Params::kSlots && temperature == 0.0f;  // the race below takes the largest value, first index on ties
  const bool use_k = !greedy && top_k > 0 && top_k < n, use_p = !greedy && top_p < 1.0f;
  uint32_t word1;
  const unsigned long long ctr = sample_counter(keys, row, word1);  // counter words 2, 3
  __syncthreads();
  auto each = [&](auto&& f) {
    for (int i = tid * 8; i < n; i += kSampleThreads * 8) {
      if (i + 8 <= n) {
        const Vec<T, 8> v = *reinterpret_cast<const Vec<T, 8>*>(x + i);
#pragma unroll
        for (int j = 0; j < 8; ++j) f(i + j, v.v[j]);
      } else {
        for (int j = i; j < n; ++j) f(j, x[j]);
      }
    }
  };

  int hb_k = -1, lb_k = 0;   // top-k pivot key hb_k << 8 | lb_k; hb_k -1: no top-k
  uint32_t thr = 0;          // kept: key >= thr ...
  int split = -1;            // ... or, when split >= 0: high byte > split, or high byte == split and low byte >= the top-p low byte
  unsigned long long p_left = 0;  // split >= 0: the mass the low bytes of bin `split` must still supply
  if (use_k || use_p) {
    unsigned mk = 0;
    each([&](int, T v) {
      const uint32_t k = sample_key(bits16(v));
      smem_add(&cnt_hi[k >> 8], 1u);
      mk = k > mk ? k : mk;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned t = __shfl_xor_sync(0xffffffffu, mk, o); mk = t > mk ? t : mk; }
    if ((tid & 31) == 0) smem_max(&max_key, mk);
    __syncthreads();
    if (use_k && tid < 32) find_from_top(cnt_hi, (unsigned long long)top_k, &sel_bin, &sel_above);
    __syncthreads();
    const unsigned long long k_left = (unsigned long long)top_k - sel_above;
    if (use_k) hb_k = sel_bin;
    const float m = sample_key_value<T>(max_key);
    each([&](int, T v) {
      const uint32_t k = sample_key(bits16(v));
      const int hi = (int)(k >> 8);
      if (hi < hb_k || (hi > hb_k && !use_p)) return;
      const unsigned long long w = use_p ? sample_mass(to_f32<T>(v), m, temperature) : 0ull;
      if (hi == hb_k) {
        smem_add(&cnt_lo[k & 255u], 1u);
        if (w) smem_add(&mass_lo[k & 255u], w);
      } else if (w) {
        smem_add(&mass_hi[hi], w);
      }
    });
    __syncthreads();
    if (use_k) {
      if (tid < 32) find_from_top(cnt_lo, k_left, &sel_bin, &sel_above);
      __syncthreads();
      lb_k = sel_bin;
      thr = ((uint32_t)hb_k << 8) | (uint32_t)lb_k;
      if (tid < 256 && tid < lb_k) mass_lo[tid] = 0;  // the pivot bin keeps its low bytes >= lb_k
      __syncthreads();
    }
    if (use_p) {
      if (tid < 32) {
        if (hb_k >= 0) {
          const unsigned long long s = warp_bin_sum(mass_lo);
          if (tid == 0) mass_hi[hb_k] = s;
        }
        __syncwarp();
        const unsigned long long total = warp_bin_sum(mass_hi);
        const unsigned long long target = (unsigned long long)ceil((double)top_p * (double)total);
        if (tid == 0) sel_target = target;
        find_from_top(mass_hi, target, &sel_bin, &sel_above);
      }
      __syncthreads();
      const int hb_p = sel_bin;
      p_left = sel_target - sel_above;
      __syncthreads();
      if (hb_p == hb_k) {  // the threshold lies in the pivot bin, whose low-byte masses are at hand
        if (tid < 32) find_from_top(mass_lo, p_left, &sel_bin, &sel_above);
        __syncthreads();
        thr = ((uint32_t)hb_p << 8) | (uint32_t)sel_bin;
      } else {
        split = hb_p;
        for (int i = tid; i < 256; i += kSampleThreads) mass_lo[i] = 0;
        __syncthreads();
      }
    }
  }

  // the race: the kept element with the largest l / T + g (lowest index on equal keys), g = -log(-log u) from Philox
  unsigned long long best = 0;
  float best_r = -INFINITY;
  long long pq = -1;
  uint32_t ph[4] = {0, 0, 0, 0};
  const float m_p = split >= 0 ? sample_key_value<T>(max_key) : 0.0f;
  each([&](int i, T v) {
    const uint32_t k = sample_key(bits16(v));
    if (greedy) {  // the ordered 16-bit key in place of l / T + g
      const unsigned long long key = ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)i);
      if (key > best) best = key;
      return;
    }
    bool edge = false;
    if (split >= 0) {
      const int hi = (int)(k >> 8);
      if (hi < split) return;
      edge = hi == split;
    } else if (k < thr) {
      return;
    }
    const float l = to_f32<T>(v);
    if (edge) {
      const unsigned long long w = sample_mass(l, m_p, temperature);
      if (w) smem_add(&mass_lo[k & 255u], w);
    }
    const float lt = __fdiv_rn(l, temperature);
    if (__fadd_rn(lt, kGumbelMax) < best_r) return;
    if ((long long)(i >> 2) != pq) {
      pq = i >> 2;
      ph[0] = (uint32_t)pq; ph[1] = word1; ph[2] = (uint32_t)ctr; ph[3] = (uint32_t)(ctr >> 32);
      philox4x32_10(ph, seed_lo, seed_hi);
    }
    const int wi = i & 3;
    const uint32_t word = wi == 0 ? ph[0] : wi == 1 ? ph[1] : wi == 2 ? ph[2] : ph[3];
    const float u = ((float)(word >> 9) + 0.5f) * 0x1p-23f;  // exact: 24 significant bits at most
    const float r = __fadd_rn(lt, -logf(-logf(u)));
    const uint32_t ur = __float_as_uint(r);
    const unsigned long long key = ((unsigned long long)((ur & 0x80000000u) ? ~ur : (ur | 0x80000000u)) << 32) | (0xFFFFFFFFu - (uint32_t)i);
    if (edge) {
      smem_max(&best_lo[k & 255u], key);
    } else if (key > best) {
      best = key;
      best_r = r;
    }
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o); best = t > best ? t : best; }
  if ((tid & 31) == 0) red[tid >> 5] = best;
  __syncthreads();
  if (tid < 32) {
    best = red[tid];
    if (split >= 0) {  // the top-p low byte of bin `split`, then the winners of the low bytes at or above it
      find_from_top(mass_lo, p_left, &sel_bin, &sel_above);
      __syncwarp();
      const int lb = *reinterpret_cast<volatile int*>(&sel_bin);
      for (int j = 0; j < 8; ++j) {
        const int bin = tid * 8 + j;
        if (bin >= lb && best_lo[bin] > best) best = best_lo[bin];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o); best = t > best ? t : best; }
    if (tid == 0) out[row] = (long long)(0xFFFFFFFFu - (uint32_t)(best & 0xFFFFFFFFull));
  }
}

// ---- repetition, frequency and presence penalties (hqq_b200_glue_penalize; the definition is in include/hqq_b200.h) ---------------
// CTA (x, s) takes columns [x * kPenChunk, (x + 1) * kPenChunk) of every row of slot s, one column per thread and pass.  The thread
// whose column is tok[s] reads counts[s][tok] once, penalises all of the slot's rows with the count plus one and stores that
// count back; no other thread touches the entry, so the increment needs no atomic and every row sees this step's token.
constexpr int kPenThreads = 256;
constexpr int kPenChunk = 1024;  // 126 CTAs over one row of the 128256-entry vocabulary

template <typename T>
__global__ void __launch_bounds__(kPenThreads) penalize_kernel(const T* __restrict__ logits, int n, long long ld, int rows_per_slot,
                                                               const float* __restrict__ rep, const float* __restrict__ freq,
                                                               const float* __restrict__ pres, int* __restrict__ counts,
                                                               const unsigned char* __restrict__ prompt, const long long* __restrict__ tok,
                                                               T* __restrict__ out, long long ld_out) {
  const int slot = blockIdx.y;
  pdl_launch_dependents();
  pdl_wait();
  const float r = __ldg(rep + slot), f = __ldg(freq + slot), p = __ldg(pres + slot);
  const long long t = tok ? __ldg(tok + slot) : -1;
  int* cnt = counts + (long long)slot * n;
  const unsigned char* pr = prompt + (long long)slot * n;
  const int end = min(n, (int)(blockIdx.x + 1) * kPenChunk);
  for (int i = blockIdx.x * kPenChunk + threadIdx.x; i < end; i += kPenThreads) {
    const int c = cnt[i] + (i == t);
    if (i == t) cnt[i] = c;
    const bool seen = c > 0 || pr[i];
    const float fc = __fmul_rn(f, (float)c);
    for (int j = 0; j < rows_per_slot; ++j) {
      const long long row = (long long)slot * rows_per_slot + j;
      T v = logits[row * ld + i];
      if (seen) {
        float x = to_f32<T>(v);
        x = x < 0.0f ? __fmul_rn(x, r) : __fdiv_rn(x, r);
        if (c > 0) x = __fsub_rn(__fsub_rn(x, fc), p);
        v = from_f32<T>(x);
      }
      out[row * ld_out + i] = v;
    }
  }
}

}  // namespace

#ifndef HQQ_EMU
// argmax over n logits -> int64 index (first index on ties).  One thread-block cluster of 8 CTAs: each scans an
// interleaved eighth of the row, the eight candidates meet in CTA 0's shared memory over DSMEM (no workspace, one launch).
// key_offset >= 0 (vocabulary-sharded lm_head under tensor parallelism): out[0] = (ordered(max) >> 1) << 32 | (0xFFFFFFFF -
// (key_offset + index)) -- a signed 64-bit key whose MAX over the ranks is the global argmax with the first index on ties
// (ordered() is the usual monotone float -> uint32 map; fp16/bf16 values leave the low mantissa bits of the float zero, so the
// shift that keeps the sign bit clear loses nothing).
constexpr int kArgmaxCtas = 8;
//
// tp > 0 (hqq_b200_glue_argmax_tp): the key exchange happens in this launch.  Bits 32..43 of a key are the same for every fp16 /
// bf16 value of one sign (they are below the 16-bit value's precision), so they can carry a 12-bit tag of the token step without
// disturbing the order, as long as every rank uses the same tag in the same step.  CTA 0 stores its tagged key into slot
// [parity][rank] of every peer's key area (one aligned 8-byte store each: value, index and tag arrive together), polls its own
// slots [parity][0..tp) until all carry this step's tag, and writes the winner's index to out[0].  Two parities suffice: a rank
// cannot finish step s+1 before every peer has sent its step s+1 key, which a peer does only after it has read step s.
struct KeyPeers { unsigned long long* p[8]; };
template <typename T>
__global__ void __cluster_dims__(kArgmaxCtas, 1, 1) __launch_bounds__(1024) argmax_kernel(const T* __restrict__ x, int n, long long* __restrict__ out,
                                                                                            long long key_offset, KeyPeers peers, int tp, int tp_rank,
                                                                                            const int* __restrict__ step_ctr) {
  namespace cg = cooperative_groups;
  __shared__ float bv[32];
  __shared__ int bi[32];
  __shared__ float cv[kArgmaxCtas];
  __shared__ int ci[kArgmaxCtas];
  __shared__ unsigned long long xkey;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  pdl_launch_dependents();
  pdl_wait();
  float best = -INFINITY;
  int idx = 0;
  for (int i = (rank * 1024 + (int)threadIdx.x) * 8; i < n; i += kArgmaxCtas * 1024 * 8) {
    if (i + 8 <= n) {
      const Vec<T, 8> v = *reinterpret_cast<const Vec<T, 8>*>(x + i);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float f = to_f32<T>(v.v[j]); if (f > best) { best = f; idx = i + j; } }
    } else {
      for (int j = i; j < n; ++j) { const float f = to_f32<T>(x[j]); if (f > best) { best = f; idx = j; } }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
  }
  if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = idx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
      if (bv[i] > best || (bv[i] == best && bi[i] < idx)) { best = bv[i]; idx = bi[i]; }
    cluster.map_shared_rank(cv, 0)[rank] = best;
    cluster.map_shared_rank(ci, 0)[rank] = idx;
  }
  cluster.sync();
  if (rank == 0 && threadIdx.x == 0) {
    best = cv[0]; idx = ci[0];
    for (int i = 1; i < kArgmaxCtas; ++i)
      if (cv[i] > best || (cv[i] == best && ci[i] < idx)) { best = cv[i]; idx = ci[i]; }
    if (key_offset < 0) {
      out[0] = idx;
    } else {
      const uint32_t u = __float_as_uint(best);
      const uint32_t ord = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      const unsigned long long key = ((unsigned long long)(ord >> 1) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)(key_offset + idx));
      if (tp <= 0) out[0] = (long long)key;
      else xkey = key;
    }
  }
  if (tp > 0 && rank == 0) {  // uniform per CTA
    __syncthreads();
    if ((int)threadIdx.x < 32) {
      const int seq = *reinterpret_cast<const volatile int*>(step_ctr);  // already bumped by this token's final norm: >= 1
      const unsigned long long tag = (unsigned long long)((unsigned)seq & 0xFFFu) << 32, tmask = 0xFFFull << 32;
      const int par = seq & 1, t = (int)threadIdx.x;
      long long got = 0;  // keys are non-negative
      if (t < tp) {
        const unsigned long long mine = (xkey & ~tmask) | tag;
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(peers.p[t] + par * tp + tp_rank), "l"(mine) : "memory");
        const unsigned long long* slot = peers.p[tp_rank] + par * tp + t;
        unsigned long long v;
        unsigned spins = 0;  // a peer that never arrives (it died) ends in a launch failure, not in a GPU that spins for ever
        do {
          asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(slot) : "memory");
          if (++spins == (1u << 27)) __trap();
        } while ((v & tmask) != tag);
        got = (long long)v;
      }
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) { const long long ov = __shfl_xor_sync(0xffffffffu, got, o); got = ov > got ? ov : got; }
      if (t == 0) out[0] = (long long)(0xFFFFFFFFu - (uint32_t)((unsigned long long)got & 0xFFFFFFFFull));
    }
  }
}

#endif  // !HQQ_EMU

}  // namespace hqq

using namespace hqq;

extern "C" int hqq_b200_glue_add_rmsnorm_rows(void* h, const void* delta, const void* weight, void* y, int rows, int H, float eps, int dtype,
                                              void* stream) {
  HQQ_REQUIRE(h && weight && y && H > 0 && H <= 8 * 1024 && rows > 0 && rows <= 65535, HQQ_E_INVALID,
              "hqq_b200_glue_add_rmsnorm: bad arguments (rows=%d H=%d)", rows, H);
  cudaStream_t st = (cudaStream_t)stream;
  const int threads = H > 2048 ? 1024 : 256;  // at most 8 elements per thread (the kernels keep them in registers)
  if (dtype == HQQ_F16) return launch_pdl("add_rmsnorm", add_rmsnorm_kernel<__half>, dim3(rows), dim3(threads), 0, st, (__half*)h, (const __half*)delta, (const __half*)weight, (__half*)y, H, eps);
  if (dtype == HQQ_BF16) return launch_pdl("add_rmsnorm", add_rmsnorm_kernel<__nv_bfloat16>, dim3(rows), dim3(threads), 0, st, (__nv_bfloat16*)h, (const __nv_bfloat16*)delta, (const __nv_bfloat16*)weight, (__nv_bfloat16*)y, H, eps);
  set_error("hqq_b200_glue_add_rmsnorm: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_add_rmsnorm(void* h, const void* delta, const void* weight, void* y, int H, float eps, int dtype, void* stream) {
  return hqq_b200_glue_add_rmsnorm_rows(h, delta, weight, y, 1, H, eps, dtype, stream);
}

extern "C" int hqq_b200_glue_add_rmsnorm_tp(void* h, const void* red_data, int* step_ctr, int x_index, int x_per_step, int tp, const void* weight,
                                            void* y, int H, float eps, int dtype, void* stream) {
  HQQ_REQUIRE(h && red_data && step_ctr && weight && y && H > 0 && H <= 8 * 1024 && tp >= 1 && tp <= 8 && x_per_step > 0, HQQ_E_INVALID,
              "hqq_b200_glue_add_rmsnorm_tp: bad arguments (H=%d tp=%d)", H, tp);
  cudaStream_t st = (cudaStream_t)stream;
  const int threads = H > 2048 ? 1024 : 256;  // at most 8 elements per thread (the kernels keep them in registers)
  if (dtype == HQQ_F16) return launch_pdl("add_rmsnorm_tp", add_rmsnorm_tp_kernel<__half>, dim3(1), dim3(threads), 0, st, (__half*)h, (const uint32_t*)red_data, step_ctr, x_index, x_per_step, tp, (const __half*)weight, (__half*)y, H, eps);
  if (dtype == HQQ_BF16) return launch_pdl("add_rmsnorm_tp", add_rmsnorm_tp_kernel<__nv_bfloat16>, dim3(1), dim3(threads), 0, st, (__nv_bfloat16*)h, (const uint32_t*)red_data, step_ctr, x_index, x_per_step, tp, (const __nv_bfloat16*)weight, (__nv_bfloat16*)y, H, eps);
  set_error("hqq_b200_glue_add_rmsnorm_tp: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_silu_mul(const void* gate, const void* up, void* y, int n, int dtype, void* stream) {
  HQQ_REQUIRE(gate && up && y && n > 0, HQQ_E_INVALID, "hqq_b200_glue_silu_mul: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)cdiv(n, 256));
  if (dtype == HQQ_F16) return launch_pdl("silu_mul", silu_mul_kernel<__half>, grid, dim3(256), 0, st, (const __half*)gate, (const __half*)up, (__half*)y, n);
  if (dtype == HQQ_BF16) return launch_pdl("silu_mul", silu_mul_kernel<__nv_bfloat16>, grid, dim3(256), 0, st, (const __nv_bfloat16*)gate, (const __nv_bfloat16*)up, (__nv_bfloat16*)y, n);
  set_error("hqq_b200_glue_silu_mul: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_moe_route(const void* x, const void* router, int M, int H, int n_experts, int k, int32_t* ids, float* weights,
                                       int32_t* pair_of, int32_t* expert_off, int32_t* expert_cnt, int32_t* pair_token, void* ticket, int dtype,
                                       void* stream) {
  HQQ_REQUIRE(x && router && ids && weights && pair_of && expert_off && expert_cnt && pair_token && ticket, HQQ_E_INVALID,
              "hqq_b200_glue_moe_route: null pointer");
  HQQ_REQUIRE(n_experts >= 2 && n_experts <= kMaxExperts, HQQ_E_INVALID, "hqq_b200_glue_moe_route: n_experts must be in [2, %d] (got %d)", kMaxExperts,
              n_experts);
  HQQ_REQUIRE(k >= 1 && k <= 8 && k <= n_experts, HQQ_E_INVALID, "hqq_b200_glue_moe_route: k must be in [1, min(8, n_experts)] (got %d)", k);
  HQQ_REQUIRE(M >= 1 && M <= 65535, HQQ_E_INVALID, "hqq_b200_glue_moe_route: M must be in [1, 65535] (got %d)", M);
  HQQ_REQUIRE(H > 0 && H % 8 == 0 && aligned(x, 16) && aligned(router, 16), HQQ_E_INVALID,
              "hqq_b200_glue_moe_route: H must be a positive multiple of 8 and x / router 16-byte aligned (H=%d)", H);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == HQQ_F16)
    return launch_pdl("moe_route", moe_route_kernel<__half>, dim3(M), dim3(kRouteThreads), 0, st, (const __half*)x, (const __half*)router, M, H,
                      n_experts, k, (int*)ids, weights, (int*)pair_of, (int*)expert_off, (int*)expert_cnt, (int*)pair_token, (unsigned*)ticket);
  if (dtype == HQQ_BF16)
    return launch_pdl("moe_route", moe_route_kernel<__nv_bfloat16>, dim3(M), dim3(kRouteThreads), 0, st, (const __nv_bfloat16*)x,
                      (const __nv_bfloat16*)router, M, H, n_experts, k, (int*)ids, weights, (int*)pair_of, (int*)expert_off, (int*)expert_cnt,
                      (int*)pair_token, (unsigned*)ticket);
  set_error("hqq_b200_glue_moe_route: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_moe_combine(const void* y, const int32_t* ids, const float* weights, const int32_t* pair_of, void* delta, int M, int H,
                                         int k, int dtype, void* stream) {
  HQQ_REQUIRE(y && ids && weights && pair_of && delta, HQQ_E_INVALID, "hqq_b200_glue_moe_combine: null pointer");
  HQQ_REQUIRE(M >= 1 && M <= 65535 && H > 0 && k >= 1 && k <= 8, HQQ_E_INVALID, "hqq_b200_glue_moe_combine: bad shape (M=%d H=%d k=%d)", M, H, k);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == HQQ_F16)
    return launch_pdl("moe_combine", moe_combine_kernel<__half>, dim3(M), dim3(256), 0, st, (const __half*)y, (const int*)ids, weights,
                      (const int*)pair_of, (__half*)delta, H, k);
  if (dtype == HQQ_BF16)
    return launch_pdl("moe_combine", moe_combine_kernel<__nv_bfloat16>, dim3(M), dim3(256), 0, st, (const __nv_bfloat16*)y, (const int*)ids, weights,
                      (const int*)pair_of, (__nv_bfloat16*)delta, H, k);
  set_error("hqq_b200_glue_moe_combine: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

// The checks every paged entry point adds: a table, whole pages, at least one page besides the sink.
static int paged_args(const char* name, const int* table, int cache_len, int n_pages) {
  HQQ_REQUIRE(table, HQQ_E_INVALID, "%s: null page table", name);
  HQQ_REQUIRE(cache_len > 0 && cache_len % kPage == 0, HQQ_E_INVALID, "%s: cache_len must be a multiple of %d (got %d)", name, kPage, cache_len);
  HQQ_REQUIRE(n_pages >= 1, HQQ_E_INVALID, "%s: n_pages must be >= 1 (got %d)", name, n_pages);
  return HQQ_OK;
}

// table == nullptr: contiguous caches; else page pools (seqpos only)
static int rope_attn_decode_batch(const char* name, bool seqpos, const void* q, const void* k, const void* v, const void* cos_table,
                                  const void* sin_table, void* k_cache, void* v_cache, const int* table, const int64_t* pos, void* out, int n_q_heads,
                                  int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream) {
  HQQ_REQUIRE(q && k && v && cos_table && sin_table && k_cache && v_cache && pos && out, HQQ_E_INVALID, "%s: null pointer", name);
  HQQ_REQUIRE(batch > 0 && batch <= 65535, HQQ_E_INVALID, "%s: batch %d", name, batch);
  HQQ_REQUIRE(head_dim == 128 && n_kv_heads > 0 && n_q_heads % n_kv_heads == 0 && cache_len > 0 && cache_len <= 8192, HQQ_E_UNSUPPORTED,
              "%s: needs head_dim 128, cache_len <= 8192", name);
  cudaStream_t st = (cudaStream_t)stream;
  const int body = 2 * head_dim + cache_len > 8 * head_dim ? 2 * head_dim + cache_len : 8 * head_dim;
  const size_t smem = (size_t)(body + 32) * sizeof(float);
  const float scale = 1.0f / sqrtf((float)head_dim);
  auto go = [&](auto kernel, auto tag, auto pg) {
    using T = decltype(tag);
    return launch_pdl("rope_attn_decode", kernel, dim3(n_q_heads, batch), dim3(kAttnThreads), smem, st, (const T*)q, (const T*)k, (const T*)v,
                      (const T*)cos_table, (const T*)sin_table, (T*)k_cache, (T*)v_cache, (const long long*)pos, (T*)out, n_q_heads, n_kv_heads,
                      cache_len, head_dim, scale, pg);
  };
  const PageTable pt{table};
  if (dtype == HQQ_F16) {
    if (table) return go(rope_attn_decode_kernel<__half, true, true, true>, __half(), pt);
    if (seqpos) return go(rope_attn_decode_kernel<__half, true, true>, __half(), NoPages());
    return batch > 1 ? go(rope_attn_decode_kernel<__half, true>, __half(), NoPages()) : go(rope_attn_decode_kernel<__half, false>, __half(), NoPages());
  }
  if (dtype == HQQ_BF16) {
    if (table) return go(rope_attn_decode_kernel<__nv_bfloat16, true, true, true>, __nv_bfloat16(), pt);
    if (seqpos) return go(rope_attn_decode_kernel<__nv_bfloat16, true, true>, __nv_bfloat16(), NoPages());
    return batch > 1 ? go(rope_attn_decode_kernel<__nv_bfloat16, true>, __nv_bfloat16(), NoPages())
                     : go(rope_attn_decode_kernel<__nv_bfloat16, false>, __nv_bfloat16(), NoPages());
  }
  set_error("%s: dtype must be f16/bf16", name);
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_rope_attn_decode_batch(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                              void* k_cache, void* v_cache, const int64_t* pos, void* out, int n_q_heads, int n_kv_heads,
                                              int cache_len, int head_dim, int batch, int dtype, void* stream) {
  return rope_attn_decode_batch("hqq_b200_glue_rope_attn_decode", false, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr, pos, out, n_q_heads,
                                n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_batch_seqpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                     void* k_cache, void* v_cache, const int64_t* pos, void* out, int n_q_heads, int n_kv_heads,
                                                     int cache_len, int head_dim, int batch, int dtype, void* stream) {
  return rope_attn_decode_batch("hqq_b200_glue_rope_attn_decode_batch_seqpos", true, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr, pos, out,
                                n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_batch_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                          void* k_pool, void* v_pool, const int* table, const int64_t* pos, void* out, int n_q_heads,
                                                          int n_kv_heads, int cache_len, int head_dim, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_rope_attn_decode_batch_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  return rope_attn_decode_batch(name, true, q, k, v, cos_table, sin_table, k_pool, v_pool, table, pos, out, n_q_heads, n_kv_heads, cache_len, head_dim,
                                batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                              void* k_cache, void* v_cache, const int64_t* pos, void* out, int n_q_heads, int n_kv_heads,
                                              int cache_len, int head_dim, int dtype, void* stream) {
  return hqq_b200_glue_rope_attn_decode_batch(q, k, v, cos_table, sin_table, k_cache, v_cache, pos, out, n_q_heads, n_kv_heads, cache_len, head_dim, 1,
                                              dtype, stream);
}

extern "C" size_t hqq_b200_glue_rope_attn_decode_split_workspace_bytes(int n_q_heads, int n_kv_heads, int head_dim, int batch) {
  if (n_kv_heads <= 0 || n_q_heads <= 0 || n_q_heads % n_kv_heads || head_dim <= 0 || batch <= 0) return 0;
  const size_t s_max = (size_t)max(1, sm_count() / n_kv_heads);
  const size_t groups = (size_t)batch * n_kv_heads;
  return groups * s_max * (size_t)(n_q_heads / n_kv_heads) * (size_t)(head_dim + 2) * sizeof(float) + groups * sizeof(unsigned);
}

// The group sizes of a quantised cache: 64 or 128 for 8 bits, 32 or 64 for 4 bits (a 4-bit row of one group has no 4bit_u8 packing)
static int kv_group_args(const char* name, int bits, int group_size) {
  if (bits == 8) {
    HQQ_REQUIRE(group_size == 64 || group_size == 128, HQQ_E_UNSUPPORTED, "%s: group_size must be 64 or 128 (got %d)", name, group_size);
  } else {
    HQQ_REQUIRE(group_size == 32 || group_size == 64, HQQ_E_UNSUPPORTED, "%s: group_size must be 32 or 64 (got %d)", name, group_size);
  }
  return HQQ_OK;
}

// bits 16: k_cache / v_cache are the 16-bit caches (meta, gs unused); bits 8 or 4: they are the HQQ level caches, meta = {k_scale,
// k_zero, v_scale, v_zero} and gs their group size.  table == nullptr: contiguous caches; else page pools (seqpos only).
static int rope_attn_decode_split(const char* name, int bits, bool seqpos, const void* q, const void* k, const void* v, const void* cos_table,
                                  const void* sin_table, void* k_cache, void* v_cache, void* const* meta, int gs, const int* table, const int64_t* pos,
                                  void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch, int dtype,
                                  void* stream) {
  const bool quant = bits != 16;
  HQQ_REQUIRE(q && k && v && cos_table && sin_table && k_cache && v_cache && (!quant || (meta[0] && meta[1] && meta[2] && meta[3])) && pos && out &&
                  workspace,
              HQQ_E_INVALID, "%s: null pointer", name);
  HQQ_REQUIRE(batch > 0 && batch <= 65535, HQQ_E_INVALID, "%s: batch %d", name, batch);
  if (quant) {
    HQQ_REQUIRE(((uintptr_t)workspace & 3) == 0 && ((uintptr_t)k_cache & 15) == 0 && ((uintptr_t)v_cache & 15) == 0, HQQ_E_INVALID,
                "%s: workspace must be 4-byte and the level caches 16-byte aligned", name);
  } else {
    HQQ_REQUIRE(((uintptr_t)workspace & 3) == 0, HQQ_E_INVALID, "%s: workspace must be 4-byte aligned", name);
  }
  HQQ_REQUIRE(head_dim == kHd && n_kv_heads > 0 && n_kv_heads <= 65535 && n_q_heads % n_kv_heads == 0 && n_q_heads / n_kv_heads >= 1 &&
                  n_q_heads / n_kv_heads <= kSplitMaxGroup && cache_len > 0 && cache_len <= kSplitMaxLen,
              HQQ_E_UNSUPPORTED, "%s: needs head_dim 128, n_q_heads / n_kv_heads <= 8, cache_len <= 131072%s", name,
              quant ? ", group_size 64 or 128" : "");
  if (quant) {
    if (int rc = kv_group_args(name, bits, gs)) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int S = split_count(n_kv_heads, cache_len);
  const int G = n_q_heads / n_kv_heads;
  const size_t part_bytes = (size_t)batch * n_kv_heads * max(1, sm_count() / n_kv_heads) * G * kPartFloats * sizeof(float);
  float* part = (float*)workspace;
  unsigned* tickets = (unsigned*)((char*)workspace + part_bytes);
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)head_dim);
  const dim3 grid((unsigned)S, (unsigned)n_kv_heads, (unsigned)batch);
  auto launch = [&](auto tag, auto sp, auto pg, auto cache) {
    using E = decltype(tag);
    using C = decltype(cache);
    constexpr bool SP = decltype(sp)::value;
    constexpr bool PG = std::is_same<decltype(pg), PageTable>::value;
    if (int rc = reserve_smem<rope_attn_decode_split_kernel<E, C, SP, PG>>(C::kSmemBytes)) return rc;
    return launch_pdl(bits == 16 ? "rope_attn_decode_split" : bits == 8 ? "rope_attn_decode_split_kv8" : "rope_attn_decode_split_kv4",
                      rope_attn_decode_split_kernel<E, C, SP, PG>, grid, dim3(kSplitThreads), C::kSmemBytes, st, (const E*)q, (const E*)k, (const E*)v,
                      (const E*)cos_table, (const E*)sin_table, cache, (const long long*)pos, (E*)out, part, tickets, n_q_heads, n_kv_heads, cache_len,
                      scale_log2, pg);
  };
  auto go = [&](auto tag, auto sp, auto pg) {
    using E = decltype(tag);
    if (bits == 16) return launch(tag, sp, pg, KvF16<E>{(E*)k_cache, (E*)v_cache});
    if (bits == 8)
      return launch(tag, sp, pg, KvHqq<E, 8>{(uint8_t*)k_cache, (E*)meta[0], (E*)meta[1], (uint8_t*)v_cache, (E*)meta[2], (E*)meta[3], gs, kHd / gs});
    return launch(tag, sp, pg, KvHqq<E, 4>{(uint8_t*)k_cache, (E*)meta[0], (E*)meta[1], (uint8_t*)v_cache, (E*)meta[2], (E*)meta[3], gs, kHd / gs});
  };
  const PageTable pt{table};
  if (dtype == HQQ_F16) {
    if (table) return go(__half(), std::true_type(), pt);
    return seqpos ? go(__half(), std::true_type(), NoPages()) : go(__half(), std::false_type(), NoPages());
  }
  if (dtype == HQQ_BF16) {
    if (table) return go(__nv_bfloat16(), std::true_type(), pt);
    return seqpos ? go(__nv_bfloat16(), std::true_type(), NoPages()) : go(__nv_bfloat16(), std::false_type(), NoPages());
  }
  set_error("%s: dtype must be f16/bf16", name);
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_rope_attn_decode_split(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                    void* k_cache, void* v_cache, const int64_t* pos, void* out, void* workspace, int n_q_heads,
                                                    int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream) {
  return rope_attn_decode_split("hqq_b200_glue_rope_attn_decode_split", 16, false, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr, 0,
                                nullptr, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_seqpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                           void* k_cache, void* v_cache, const int64_t* pos, void* out, void* workspace, int n_q_heads,
                                                           int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream) {
  return rope_attn_decode_split("hqq_b200_glue_rope_attn_decode_split_seqpos", 16, true, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr, 0,
                                nullptr, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                          void* k_pool, void* v_pool, const int* table, const int64_t* pos, void* out, void* workspace,
                                                          int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch, int n_pages, int dtype,
                                                          void* stream) {
  const char* name = "hqq_b200_glue_rope_attn_decode_split_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  return rope_attn_decode_split(name, 16, true, q, k, v, cos_table, sin_table, k_pool, v_pool, nullptr, 0, table, pos, out, workspace, n_q_heads,
                                n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_kv8(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                        void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                        const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len,
                                                        int head_dim, int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_attn_decode_split("hqq_b200_glue_rope_attn_decode_split_kv8", 8, false, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size,
                                nullptr, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_kv8_seqpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                               void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                               const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads,
                                                               int cache_len, int head_dim, int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_attn_decode_split("hqq_b200_glue_rope_attn_decode_split_kv8_seqpos", 8, true, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size,
                                nullptr, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_kv8_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                              void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                              const int* table, const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads,
                                                              int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_rope_attn_decode_split_kv8_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_attn_decode_split(name, 8, true, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size, table, pos, out, workspace, n_q_heads,
                                n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_kv4(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                        void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                        const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len,
                                                        int head_dim, int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_attn_decode_split("hqq_b200_glue_rope_attn_decode_split_kv4", 4, false, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size,
                                nullptr, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_kv4_seqpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                               void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                               const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads,
                                                               int cache_len, int head_dim, int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_attn_decode_split("hqq_b200_glue_rope_attn_decode_split_kv4_seqpos", 4, true, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size,
                                nullptr, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_attn_decode_split_kv4_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                              void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero,
                                                              const int* table, const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads,
                                                              int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_rope_attn_decode_split_kv4_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_attn_decode_split(name, 4, true, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size, table, pos, out, workspace, n_q_heads,
                                n_kv_heads, cache_len, head_dim, batch, dtype, stream);
}

// The checks of the device-position entry points: the prefill shape checks, 1 <= T <= 8 rows per slot, T G <= 64 columns.
static int spec_args(const char* name, int T, int n_q, int n_kv, int L, int hd, int batch, int dtype) {
  if (int rc = prefill_args(name, 0, 1, n_q, n_kv, L, hd, batch, dtype)) return rc;
  HQQ_REQUIRE(T >= 1 && T <= kVerMaxT && T <= L, HQQ_E_INVALID, "%s: needs 1 <= T <= %d and T <= cache_len (T=%d)", name, kVerMaxT, T);
  HQQ_REQUIRE(T * (n_q / n_kv) <= kVerMaxCols, HQQ_E_UNSUPPORTED, "%s: T * n_q_heads / n_kv_heads must be <= %d", name, kVerMaxCols);
  return HQQ_OK;
}

// The row layout of an append: uniform pos0 / T (FixedRows), host pos0_v / n_tok_v of `batch` slots (VarlenRows), or device positions
// pos with T rows a slot (DevPos)
enum AppendRows { kAppendFixed, kAppendVarlen, kAppendDevPos };

// Every append entry point (rope_append_rows_kernel).  bits 16: k_cache / v_cache are the 16-bit caches (meta, gs unused); bits 8 or 4:
// they are the HQQ level caches, meta = {k_scale, k_zero, v_scale, v_zero} and gs their group size.  paged: page pools through table.
// k_stage / v_stage: the staging pair of a quantised cache under the host-position layouts (unused otherwise).
static int rope_append_rows(const char* name, int bits, AppendRows lay, bool paged, const void* q, const void* k, const void* v,
                            const void* cos_table, const void* sin_table, void* k_cache, void* v_cache, void* const* meta, int gs,
                            const int* table, void* k_stage, void* v_stage, void* q_out, int pos0, int T, const int* pos0_v,
                            const int* n_tok_v, const int64_t* pos, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch,
                            int n_pages, int dtype, void* stream) {
  const bool quant = bits != 16, dev = lay == kAppendDevPos;
  if (paged && dev) {  // the device-position forms check the table before the pointers
    if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  }
  HQQ_REQUIRE(q && k && v && cos_table && sin_table && k_cache && v_cache && (!quant || (meta[0] && meta[1] && meta[2] && meta[3])) &&
                  (!quant || dev || (k_stage && v_stage)) && q_out && (!dev || pos),
              HQQ_E_INVALID, "%s: null pointer", name);
  if (paged && !dev) {
    if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  }
  VarlenRows vl;
  int max_t = 0;
  if (lay == kAppendVarlen) {
    if (int rc = varlen_args(name, pos0_v, n_tok_v, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, vl, max_t)) return rc;
  } else if (dev) {
    if (int rc = spec_args(name, T, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype)) return rc;
  } else if (int rc = prefill_args(name, pos0, T, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype)) {
    return rc;
  }
  if (quant) {
    if (int rc = kv_group_args(name, bits, gs)) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)(lay == kAppendVarlen ? max_t : T), (unsigned)batch);
  auto launch = [&](auto tag, auto cache, auto rows, auto pg) {
    using E = decltype(tag);
    constexpr bool PG = std::is_same<decltype(pg), PageTable>::value;
    return launch_pdl(name, rope_append_rows_kernel<E, decltype(cache), decltype(rows), PG>, grid, dim3(256), 0, st, (const E*)q, (const E*)k,
                      (const E*)v, (const E*)cos_table, (const E*)sin_table, cache, (E*)k_stage, (E*)v_stage, (E*)q_out, n_q_heads, n_kv_heads,
                      cache_len, rows, pg);
  };
  auto by_rows = [&](auto tag, auto cache) {
    const PageTable pt{table};
    if (lay == kAppendFixed) return launch(tag, cache, FixedRows{pos0, T}, NoPages());
    if (lay == kAppendVarlen) return paged ? launch(tag, cache, vl, pt) : launch(tag, cache, vl, NoPages());
    const DevPos dp{(const long long*)pos, T};
    return paged ? launch(tag, cache, dp, pt) : launch(tag, cache, dp, NoPages());
  };
  auto by_format = [&](auto tag) {
    using E = decltype(tag);
    if (bits == 16) return by_rows(tag, KvF16<E>{(E*)k_cache, (E*)v_cache});
    if (bits == 8) return by_rows(tag, KvHqq<E, 8>{(uint8_t*)k_cache, (E*)meta[0], (E*)meta[1], (uint8_t*)v_cache, (E*)meta[2], (E*)meta[3], gs, kHd / gs});
    return by_rows(tag, KvHqq<E, 4>{(uint8_t*)k_cache, (E*)meta[0], (E*)meta[1], (uint8_t*)v_cache, (E*)meta[2], (E*)meta[3], gs, kHd / gs});
  };
  return dtype == HQQ_F16 ? by_format(__half()) : by_format(__nv_bfloat16());
}

extern "C" int hqq_b200_glue_rope_append_rows(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table, void* k_cache,
                                              void* v_cache, void* q_out, int pos0, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                              int batch, int dtype, void* stream) {
  return rope_append_rows("hqq_b200_glue_rope_append_rows", 16, kAppendFixed, false, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr, 0,
                          nullptr, nullptr, nullptr, q_out, pos0, T, nullptr, nullptr, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch, 0,
                          dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_varlen(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                     void* k_cache, void* v_cache, void* q_out, const int* pos0, const int* n_tok, int n_q_heads,
                                                     int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream) {
  return rope_append_rows("hqq_b200_glue_rope_append_rows_varlen", 16, kAppendVarlen, false, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr,
                          0, nullptr, nullptr, nullptr, q_out, 0, 0, pos0, n_tok, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch, 0, dtype,
                          stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                    void* k_pool, void* v_pool, const int* table, void* q_out, const int* pos0, const int* n_tok,
                                                    int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch, int n_pages, int dtype,
                                                    void* stream) {
  return rope_append_rows("hqq_b200_glue_rope_append_rows_paged", 16, kAppendVarlen, true, q, k, v, cos_table, sin_table, k_pool, v_pool, nullptr, 0,
                          table, nullptr, nullptr, q_out, 0, 0, pos0, n_tok, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch, n_pages, dtype,
                          stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_devpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                     void* k_cache, void* v_cache, void* q_out, const int64_t* pos, int T, int n_q_heads,
                                                     int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream) {
  return rope_append_rows("hqq_b200_glue_rope_append_rows_devpos", 16, kAppendDevPos, false, q, k, v, cos_table, sin_table, k_cache, v_cache, nullptr,
                          0, nullptr, nullptr, nullptr, q_out, 0, T, nullptr, nullptr, pos, n_q_heads, n_kv_heads, cache_len, head_dim, batch, 0, dtype,
                          stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_devpos_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                           void* k_pool, void* v_pool, const int* table, void* q_out, const int64_t* pos, int T,
                                                           int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch, int n_pages, int dtype,
                                                           void* stream) {
  return rope_append_rows("hqq_b200_glue_rope_append_rows_devpos_paged", 16, kAppendDevPos, true, q, k, v, cos_table, sin_table, k_pool, v_pool,
                          nullptr, 0, table, nullptr, nullptr, q_out, 0, T, nullptr, nullptr, pos, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          n_pages, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv8(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table, void* k_q,
                                                  void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* k_stage, void* v_stage,
                                                  void* q_out, int pos0, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                  int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv8", 8, kAppendFixed, false, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size,
                          nullptr, k_stage, v_stage, q_out, pos0, T, nullptr, nullptr, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch, 0,
                          dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv8_varlen(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                         void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* k_stage,
                                                         void* v_stage, void* q_out, const int* pos0, const int* n_tok, int n_q_heads, int n_kv_heads,
                                                         int cache_len, int head_dim, int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv8_varlen", 8, kAppendVarlen, false, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, nullptr, k_stage, v_stage, q_out, 0, 0, pos0, n_tok, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          0, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv8_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                        void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, const int* table,
                                                        void* k_stage, void* v_stage, void* q_out, const int* pos0, const int* n_tok, int n_q_heads,
                                                        int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype,
                                                        void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv8_paged", 8, kAppendVarlen, true, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, table, k_stage, v_stage, q_out, 0, 0, pos0, n_tok, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          n_pages, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv8_devpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                         void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* q_out,
                                                         const int64_t* pos, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                         int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv8_devpos", 8, kAppendDevPos, false, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, nullptr, nullptr, nullptr, q_out, 0, T, nullptr, nullptr, pos, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          0, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv8_devpos_paged(const void* q, const void* k, const void* v, const void* cos_table,
                                                               const void* sin_table, void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale,
                                                               void* v_zero, const int* table, void* q_out, const int64_t* pos, int T, int n_q_heads,
                                                               int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages,
                                                               int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv8_devpos_paged", 8, kAppendDevPos, true, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, table, nullptr, nullptr, q_out, 0, T, nullptr, nullptr, pos, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          n_pages, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv4(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table, void* k_q,
                                                  void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* k_stage, void* v_stage,
                                                  void* q_out, int pos0, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                  int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv4", 4, kAppendFixed, false, q, k, v, cos_table, sin_table, k_q, v_q, meta, group_size,
                          nullptr, k_stage, v_stage, q_out, pos0, T, nullptr, nullptr, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch, 0,
                          dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv4_varlen(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                         void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* k_stage,
                                                         void* v_stage, void* q_out, const int* pos0, const int* n_tok, int n_q_heads, int n_kv_heads,
                                                         int cache_len, int head_dim, int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv4_varlen", 4, kAppendVarlen, false, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, nullptr, k_stage, v_stage, q_out, 0, 0, pos0, n_tok, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          0, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv4_paged(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                        void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, const int* table,
                                                        void* k_stage, void* v_stage, void* q_out, const int* pos0, const int* n_tok, int n_q_heads,
                                                        int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype,
                                                        void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv4_paged", 4, kAppendVarlen, true, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, table, k_stage, v_stage, q_out, 0, 0, pos0, n_tok, nullptr, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          n_pages, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv4_devpos(const void* q, const void* k, const void* v, const void* cos_table, const void* sin_table,
                                                         void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale, void* v_zero, void* q_out,
                                                         const int64_t* pos, int T, int n_q_heads, int n_kv_heads, int cache_len, int head_dim,
                                                         int group_size, int batch, int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv4_devpos", 4, kAppendDevPos, false, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, nullptr, nullptr, nullptr, q_out, 0, T, nullptr, nullptr, pos, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          0, dtype, stream);
}

extern "C" int hqq_b200_glue_rope_append_rows_kv4_devpos_paged(const void* q, const void* k, const void* v, const void* cos_table,
                                                               const void* sin_table, void* k_q, void* k_scale, void* k_zero, void* v_q, void* v_scale,
                                                               void* v_zero, const int* table, void* q_out, const int64_t* pos, int T, int n_q_heads,
                                                               int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages,
                                                               int dtype, void* stream) {
  void* const meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return rope_append_rows("hqq_b200_glue_rope_append_rows_kv4_devpos_paged", 4, kAppendDevPos, true, q, k, v, cos_table, sin_table, k_q, v_q, meta,
                          group_size, table, nullptr, nullptr, q_out, 0, T, nullptr, nullptr, pos, n_q_heads, n_kv_heads, cache_len, head_dim, batch,
                          n_pages, dtype, stream);
}

extern "C" int hqq_b200_glue_attn_prefill(const void* q_rot, const void* k_cache, const void* v_cache, void* out, int pos0, int T, int n_q_heads,
                                          int n_kv_heads, int cache_len, int head_dim, int batch, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_attn_prefill";
  HQQ_REQUIRE(q_rot && k_cache && v_cache && out, HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = prefill_args(name, pos0, T, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)head_dim);
  const dim3 grid((unsigned)n_kv_heads, (unsigned)batch, (unsigned)cdiv((int64_t)T * (n_q_heads / n_kv_heads), kPreRows));  // z <= 8192
  auto go = [&](auto tag) {
    using E = decltype(tag);
    if (int rc = reserve_smem<attn_prefill_kernel<E>>(kPreSmemBytes)) return rc;
    return launch_pdl("attn_prefill", attn_prefill_kernel<E>, grid, dim3(kPreThreads), kPreSmemBytes, st, (const E*)q_rot, (const E*)k_cache,
                      (const E*)v_cache, (E*)out, pos0, T, n_q_heads, n_kv_heads, cache_len, scale_log2, NoVarlen(), NoPages());
  };
  return dtype == HQQ_F16 ? go(__half()) : go(__nv_bfloat16());
}

extern "C" int hqq_b200_glue_attn_prefill_varlen(const void* q_rot, const void* k_cache, const void* v_cache, void* out, const int* pos0,
                                                 const int* n_tok, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch, int dtype,
                                                 void* stream) {
  const char* name = "hqq_b200_glue_attn_prefill_varlen";
  HQQ_REQUIRE(q_rot && k_cache && v_cache && out, HQQ_E_INVALID, "%s: null pointer", name);
  VarlenRows vl;
  int max_t = 0;
  if (int rc = varlen_args(name, pos0, n_tok, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, vl, max_t)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)head_dim);
  const dim3 grid((unsigned)n_kv_heads, (unsigned)batch, (unsigned)cdiv((int64_t)max_t * (n_q_heads / n_kv_heads), kPreRows));  // z <= 8192
  auto go = [&](auto tag) {
    using E = decltype(tag);
    if (int rc = reserve_smem<attn_prefill_kernel<E, true>>(kPreSmemBytes)) return rc;
    return launch_pdl("attn_prefill_varlen", attn_prefill_kernel<E, true>, grid, dim3(kPreThreads), kPreSmemBytes, st, (const E*)q_rot,
                      (const E*)k_cache, (const E*)v_cache, (E*)out, 0, 0, n_q_heads, n_kv_heads, cache_len, scale_log2, vl, NoPages());
  };
  return dtype == HQQ_F16 ? go(__half()) : go(__nv_bfloat16());
}

// Staging rows [0, pos0[b]) of the slots with n_tok[b] > 0 from a quantised cache: page pools through the table, or (table == nullptr,
// 4 bits only) the contiguous caches
static int kvq_stage(const char* name, int bits, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q, const void* v_scale,
                     const void* v_zero, const int* table, void* k_stage, void* v_stage, const int* pos0, const int* n_tok, int n_kv_heads, int cache_len,
                     int head_dim, int group_size, int batch, int dtype, void* stream) {
  HQQ_REQUIRE(k_q && k_scale && k_zero && v_q && v_scale && v_zero && k_stage && v_stage, HQQ_E_INVALID, "%s: null pointer", name);
  VarlenRows vl;
  int max_t = 0;
  if (int rc = varlen_args(name, pos0, n_tok, n_kv_heads, n_kv_heads, cache_len, head_dim, batch, dtype, vl, max_t)) return rc;
  if (int rc = kv_group_args(name, bits, group_size)) return rc;
  int max_p = 0;  // rows to refill: [0, pos0[b]) of the slots in the chunk
  for (int b = 0; b < batch; ++b)
    if (vl.n_tok[b] > 0) max_p = max(max_p, vl.pos0[b]);
  if (max_p == 0) return HQQ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  auto go = [&](auto tag, auto kernel, auto pg) {
    using E = decltype(tag);
    return launch_pdl(name, kernel, dim3((unsigned)max_p, (unsigned)batch), dim3(256), 0, st, (const uint8_t*)k_q, (const E*)k_scale, (const E*)k_zero,
                      (const uint8_t*)v_q, (const E*)v_scale, (const E*)v_zero, (E*)k_stage, (E*)v_stage, n_kv_heads, cache_len, group_size, vl, pg);
  };
  const PageTable pt{table};
  if (bits == 8)
    return dtype == HQQ_F16 ? go(__half(), kv8_stage_paged_kernel<__half>, pt) : go(__nv_bfloat16(), kv8_stage_paged_kernel<__nv_bfloat16>, pt);
  if (table)
    return dtype == HQQ_F16 ? go(__half(), kv8_stage_paged_kernel<__half, 4>, pt) : go(__nv_bfloat16(), kv8_stage_paged_kernel<__nv_bfloat16, 4>, pt);
  return dtype == HQQ_F16 ? go(__half(), kv8_stage_paged_kernel<__half, 4, false>, NoPages())
                          : go(__nv_bfloat16(), kv8_stage_paged_kernel<__nv_bfloat16, 4, false>, NoPages());
}

extern "C" int hqq_b200_glue_kv8_stage_paged(const void* k_q, const void* k_scale, const void* k_zero, const void* v_q, const void* v_scale,
                                             const void* v_zero, const int* table, void* k_stage, void* v_stage, const int* pos0, const int* n_tok,
                                             int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_kv8_stage_paged";
  HQQ_REQUIRE(k_q && k_scale && k_zero && v_q && v_scale && v_zero && k_stage && v_stage, HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  return kvq_stage(name, 8, k_q, k_scale, k_zero, v_q, v_scale, v_zero, table, k_stage, v_stage, pos0, n_tok, n_kv_heads, cache_len, head_dim,
                   group_size, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_kv4_stage_paged(const void* k_q, const void* k_scale, const void* k_zero, const void* v_q, const void* v_scale,
                                             const void* v_zero, const int* table, void* k_stage, void* v_stage, const int* pos0, const int* n_tok,
                                             int n_kv_heads, int cache_len, int head_dim, int group_size, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_kv4_stage_paged";
  HQQ_REQUIRE(k_q && k_scale && k_zero && v_q && v_scale && v_zero && k_stage && v_stage, HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  return kvq_stage(name, 4, k_q, k_scale, k_zero, v_q, v_scale, v_zero, table, k_stage, v_stage, pos0, n_tok, n_kv_heads, cache_len, head_dim,
                   group_size, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_kv4_stage(const void* k_q, const void* k_scale, const void* k_zero, const void* v_q, const void* v_scale, const void* v_zero,
                                       void* k_stage, void* v_stage, const int* pos0, const int* n_tok, int n_kv_heads, int cache_len, int head_dim,
                                       int group_size, int batch, int dtype, void* stream) {
  return kvq_stage("hqq_b200_glue_kv4_stage", 4, k_q, k_scale, k_zero, v_q, v_scale, v_zero, nullptr, k_stage, v_stage, pos0, n_tok, n_kv_heads, cache_len,
                   head_dim, group_size, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_attn_prefill_paged(const void* q_rot, const void* k_pool, const void* v_pool, const int* table, void* out, const int* pos0,
                                                const int* n_tok, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int batch, int n_pages,
                                                int dtype, void* stream) {
  const char* name = "hqq_b200_glue_attn_prefill_paged";
  HQQ_REQUIRE(q_rot && k_pool && v_pool && out, HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  VarlenRows vl;
  int max_t = 0;
  if (int rc = varlen_args(name, pos0, n_tok, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype, vl, max_t)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)head_dim);
  const dim3 grid((unsigned)n_kv_heads, (unsigned)batch, (unsigned)cdiv((int64_t)max_t * (n_q_heads / n_kv_heads), kPreRows));  // z <= 8192
  auto go = [&](auto tag) {
    using E = decltype(tag);
    if (int rc = reserve_smem<attn_prefill_kernel<E, true, true>>(kPreSmemBytes)) return rc;
    return launch_pdl("attn_prefill_paged", attn_prefill_kernel<E, true, true>, grid, dim3(kPreThreads), kPreSmemBytes, st, (const E*)q_rot,
                      (const E*)k_pool, (const E*)v_pool, (E*)out, 0, 0, n_q_heads, n_kv_heads, cache_len, scale_log2, vl, PageTable{table});
  };
  return dtype == HQQ_F16 ? go(__half()) : go(__nv_bfloat16());
}

// ---- speculative decoding (DESIGN.md 3.5)
// column groups of one kv head in the verify attention
static int verify_groups(int n_q_heads, int n_kv_heads, int T) { return (int)cdiv((int64_t)T * (n_q_heads / n_kv_heads), kVerCols); }

extern "C" size_t hqq_b200_glue_attn_verify_split_workspace_bytes(int n_q_heads, int n_kv_heads, int head_dim, int T, int batch) {
  if (n_kv_heads <= 0 || n_q_heads <= 0 || n_q_heads % n_kv_heads || head_dim <= 0 || T < 1 || batch <= 0) return 0;
  const size_t s_max = (size_t)max(1, sm_count() / n_kv_heads);
  const size_t groups = (size_t)batch * n_kv_heads * verify_groups(n_q_heads, n_kv_heads, T);
  return groups * s_max * kVerCols * (size_t)(head_dim + 2) * sizeof(float) + groups * sizeof(unsigned);
}

// table == nullptr: contiguous caches; meta == nullptr: 16-bit caches, else the quantised cache's {k_scale, k_zero, v_scale, v_zero}
// with `bits` 8 or 4
static int attn_verify_split(const char* name, const void* q_rot, const void* k_cache, const void* v_cache, const void* const* meta, int gs,
                             const int* table, const int64_t* pos, void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len,
                             int head_dim, int T, int batch, int dtype, void* stream, int bits = 8) {
  HQQ_REQUIRE(q_rot && k_cache && v_cache && pos && out && workspace, HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = spec_args(name, T, n_q_heads, n_kv_heads, cache_len, head_dim, batch, dtype)) return rc;
  if (meta) {
    HQQ_REQUIRE(meta[0] && meta[1] && meta[2] && meta[3], HQQ_E_INVALID, "%s: null pointer", name);
    if (int rc = kv_group_args(name, bits, gs)) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int S = split_count(n_kv_heads, cache_len), n_cg = verify_groups(n_q_heads, n_kv_heads, T);
  const size_t part_bytes = (size_t)batch * n_kv_heads * n_cg * max(1, sm_count() / n_kv_heads) * kVerCols * kPartFloats * sizeof(float);
  float* part = (float*)workspace;
  unsigned* tickets = (unsigned*)((char*)workspace + part_bytes);
  const float scale_log2 = 1.4426950408889634f / sqrtf((float)head_dim);
  const dim3 grid((unsigned)S, (unsigned)(n_kv_heads * n_cg), (unsigned)batch);
  constexpr int smem = kRingBytes + 16;
  auto run = [&](auto tag, auto pg, auto paged, auto kv8, auto nbits) -> int {
    using E = decltype(tag);
    constexpr bool PG = decltype(paged)::value, K8 = decltype(kv8)::value;
    constexpr int NB = decltype(nbits)::value;
    using C = CacheT<E, K8>;
    Kv8Arg<E, K8> m8;
    if constexpr (K8) m8 = Kv8Meta<E>{(const E*)meta[0], (const E*)meta[1], (const E*)meta[2], (const E*)meta[3], gs};
    if (int rc = reserve_smem<attn_verify_split_kernel<E, PG, K8, NB>>(smem)) return rc;
    return launch_pdl(K8 ? (NB == 4 ? "attn_verify_split_kv4" : "attn_verify_split_kv8") : "attn_verify_split", attn_verify_split_kernel<E, PG, K8, NB>,
                      grid, dim3(kSplitThreads), smem, st, (const E*)q_rot, (const C*)k_cache, (const C*)v_cache, (const long long*)pos, (E*)out, part,
                      tickets, n_q_heads, n_kv_heads, cache_len, T, scale_log2, pg, m8);
  };
  using B8 = std::integral_constant<int, 8>;
  auto by_dtype = [&](auto pg, auto paged, auto kv8, auto nbits) {
    return dtype == HQQ_F16 ? run(__half(), pg, paged, kv8, nbits) : run(__nv_bfloat16(), pg, paged, kv8, nbits);
  };
  const PageTable pt{table};
  if (meta && bits == 4) {
    using B4 = std::integral_constant<int, 4>;
    return table ? by_dtype(pt, std::true_type(), std::true_type(), B4()) : by_dtype(NoPages(), std::false_type(), std::true_type(), B4());
  }
  if (meta) return table ? by_dtype(pt, std::true_type(), std::true_type(), B8()) : by_dtype(NoPages(), std::false_type(), std::true_type(), B8());
  return table ? by_dtype(pt, std::true_type(), std::false_type(), B8()) : by_dtype(NoPages(), std::false_type(), std::false_type(), B8());
}

extern "C" int hqq_b200_glue_attn_verify_split(const void* q_rot, const void* k_cache, const void* v_cache, const int64_t* pos, void* out,
                                               void* workspace, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int T, int batch, int dtype,
                                               void* stream) {
  return attn_verify_split("hqq_b200_glue_attn_verify_split", q_rot, k_cache, v_cache, nullptr, 0, nullptr, pos, out, workspace, n_q_heads, n_kv_heads,
                           cache_len, head_dim, T, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_attn_verify_split_paged(const void* q_rot, const void* k_pool, const void* v_pool, const int* table, const int64_t* pos,
                                                     void* out, void* workspace, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int T,
                                                     int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_attn_verify_split_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  return attn_verify_split(name, q_rot, k_pool, v_pool, nullptr, 0, table, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, T, batch,
                           dtype, stream);
}

extern "C" int hqq_b200_glue_attn_verify_split_kv8(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q,
                                                   const void* v_scale, const void* v_zero, const int64_t* pos, void* out, void* workspace, int n_q_heads,
                                                   int n_kv_heads, int cache_len, int head_dim, int group_size, int T, int batch, int dtype,
                                                   void* stream) {
  const void* meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return attn_verify_split("hqq_b200_glue_attn_verify_split_kv8", q_rot, k_q, v_q, meta, group_size, nullptr, pos, out, workspace, n_q_heads,
                           n_kv_heads, cache_len, head_dim, T, batch, dtype, stream);
}

extern "C" int hqq_b200_glue_attn_verify_split_kv8_paged(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q,
                                                         const void* v_scale, const void* v_zero, const int* table, const int64_t* pos, void* out,
                                                         void* workspace, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                                         int T, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_attn_verify_split_kv8_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  const void* meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return attn_verify_split(name, q_rot, k_q, v_q, meta, group_size, table, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, T, batch,
                           dtype, stream);
}

extern "C" int hqq_b200_glue_attn_verify_split_kv4(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q,
                                                   const void* v_scale, const void* v_zero, const int64_t* pos, void* out, void* workspace, int n_q_heads,
                                                   int n_kv_heads, int cache_len, int head_dim, int group_size, int T, int batch, int dtype,
                                                   void* stream) {
  const void* meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return attn_verify_split("hqq_b200_glue_attn_verify_split_kv4", q_rot, k_q, v_q, meta, group_size, nullptr, pos, out, workspace, n_q_heads,
                           n_kv_heads, cache_len, head_dim, T, batch, dtype, stream, 4);
}

extern "C" int hqq_b200_glue_attn_verify_split_kv4_paged(const void* q_rot, const void* k_q, const void* k_scale, const void* k_zero, const void* v_q,
                                                         const void* v_scale, const void* v_zero, const int* table, const int64_t* pos, void* out,
                                                         void* workspace, int n_q_heads, int n_kv_heads, int cache_len, int head_dim, int group_size,
                                                         int T, int batch, int n_pages, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_attn_verify_split_kv4_paged";
  if (int rc = paged_args(name, table, cache_len, n_pages)) return rc;
  const void* meta[4] = {k_scale, k_zero, v_scale, v_zero};
  return attn_verify_split(name, q_rot, k_q, v_q, meta, group_size, table, pos, out, workspace, n_q_heads, n_kv_heads, cache_len, head_dim, T, batch,
                           dtype, stream, 4);
}

extern "C" int hqq_b200_glue_ngram_draft(const int32_t* hist, const int64_t* pos, const int64_t* tok, int64_t* drafts, int cache_len, int K, int batch,
                                         void* stream) {
  const char* name = "hqq_b200_glue_ngram_draft";
  HQQ_REQUIRE(hist && pos && tok && drafts, HQQ_E_INVALID, "%s: null pointer", name);
  HQQ_REQUIRE(cache_len > 0 && cache_len <= kSplitMaxLen && K >= 1 && K < kVerMaxT && batch > 0 && batch <= 65535, HQQ_E_INVALID,
              "%s: needs 0 < cache_len <= %d, 1 <= K <= %d, 0 < batch <= 65535 (cache_len=%d K=%d batch=%d)", name, kSplitMaxLen, kVerMaxT - 1, cache_len,
              K, batch);
  return launch_pdl("ngram_draft", ngram_draft_kernel, dim3((unsigned)batch), dim3(kNgramThreads), 0, (cudaStream_t)stream, (const int*)hist,
                    (const long long*)pos, (const long long*)tok, (long long*)drafts, cache_len, K);
}

extern "C" int hqq_b200_glue_spec_accept(const int64_t* targets, const int64_t* drafts, int64_t* pos, int64_t* tok, int64_t* next_tok, int32_t* hist,
                                         int64_t* tokens, int64_t* n_new, int cache_len, int K, int batch, void* stream) {
  const char* name = "hqq_b200_glue_spec_accept";
  HQQ_REQUIRE(targets && drafts && pos && tok && next_tok && hist && tokens && n_new, HQQ_E_INVALID, "%s: null pointer", name);
  HQQ_REQUIRE(cache_len > 0 && cache_len <= kSplitMaxLen && K >= 1 && K < kVerMaxT && batch > 0 && batch <= 65535, HQQ_E_INVALID,
              "%s: needs 0 < cache_len <= %d, 1 <= K <= %d, 0 < batch <= 65535 (cache_len=%d K=%d batch=%d)", name, kSplitMaxLen, kVerMaxT - 1, cache_len,
              K, batch);
  return launch_pdl("spec_accept", spec_accept_kernel, dim3((unsigned)cdiv(batch, 128)), dim3(128), 0, (cudaStream_t)stream, (const long long*)targets,
                    (const long long*)drafts, (long long*)pos, (long long*)tok, (long long*)next_tok, (int*)hist, (long long*)tokens, (long long*)n_new,
                    batch, K, cache_len);
}

template <typename Keys, typename Params>
static int sample_launch(const char* name, const void* logits, int n, int ld, int rows, Params params, uint64_t seed, Keys keys, int64_t* out, int dtype,
                         void* stream) {
  HQQ_REQUIRE(dtype == HQQ_F16 || dtype == HQQ_BF16, HQQ_E_INVALID, "%s: dtype must be f16/bf16", name);
  if constexpr (!Params::kSlots) {
    const float temperature = params.temperature, top_p = params.top_p;
    HQQ_REQUIRE(temperature > 0.0f && temperature <= 3.40282347e38f, HQQ_E_INVALID, "%s: temperature must be finite and > 0 (got %g)", name, (double)temperature);
    HQQ_REQUIRE(params.top_k >= 0, HQQ_E_INVALID, "%s: top_k must be >= 0 (got %d)", name, params.top_k);
    HQQ_REQUIRE(top_p > 0.0f && top_p <= 1.0f, HQQ_E_INVALID, "%s: top_p must lie in (0, 1] (got %g)", name, (double)top_p);
  }
  HQQ_REQUIRE(n > 0 && ld >= n && rows > 0 && rows <= 65535, HQQ_E_INVALID, "%s: needs n > 0, ld >= n and 1 <= rows <= 65535 (n=%d ld=%d rows=%d)", name,
              n, ld, rows);
  HQQ_REQUIRE(aligned(logits, 16) && ld % 8 == 0, HQQ_E_INVALID, "%s: rows must start on 16-byte boundaries (logits 16-byte aligned, ld %% 8 == 0; ld=%d)",
              name, ld);
  cudaStream_t st = (cudaStream_t)stream;
  auto go = [&](auto t) {
    using E = decltype(t);
    return launch_pdl("sample", sample_kernel<E, Keys, Params>, dim3((unsigned)rows), dim3(kSampleThreads), 0, st, (const E*)logits, n, (long long)ld,
                      params, (uint32_t)seed, (uint32_t)(seed >> 32), keys, (long long*)out);
  };
  return dtype == HQQ_F16 ? go(__half()) : go(__nv_bfloat16());
}

static int rows_per_slot_args(const char* name, int rows_per_slot, int rows) {
  HQQ_REQUIRE(rows_per_slot >= 1 && rows_per_slot <= 8 && rows % rows_per_slot == 0, HQQ_E_INVALID,
              "%s: needs 1 <= rows_per_slot <= 8 dividing rows (rows_per_slot=%d rows=%d)", name, rows_per_slot, rows);
  return HQQ_OK;
}

extern "C" int hqq_b200_glue_sample(const void* logits, int n, int ld, int rows, float temperature, int top_k, float top_p, uint64_t seed,
                                    const uint64_t* counter, int64_t* out, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_sample";
  HQQ_REQUIRE(logits && counter && out, HQQ_E_INVALID, "%s: null pointer", name);
  return sample_launch(name, logits, n, ld, rows, ScalarParams{temperature, top_k, top_p}, seed, StepKeys{(const unsigned long long*)counter}, out, dtype,
                       stream);
}

extern "C" int hqq_b200_glue_sample_pos(const void* logits, int n, int ld, int rows, float temperature, int top_k, float top_p, uint64_t seed,
                                        int rows_per_slot, const int64_t* pos, const int64_t* seq, int64_t* out, int dtype, void* stream) {
  const char* name = "hqq_b200_glue_sample_pos";
  HQQ_REQUIRE(logits && pos && seq && out, HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = rows_per_slot_args(name, rows_per_slot, rows)) return rc;
  return sample_launch(name, logits, n, ld, rows, ScalarParams{temperature, top_k, top_p}, seed,
                       PosKeys{(const long long*)pos, (const long long*)seq, rows_per_slot}, out, dtype, stream);
}

extern "C" int hqq_b200_glue_sample_slots(const void* logits, int n, int ld, int rows, int rows_per_slot, const float* temperature, const int32_t* top_k,
                                          const float* top_p, uint64_t seed, const uint64_t* counter, const int64_t* pos, const int64_t* seq, int64_t* out,
                                          int dtype, void* stream) {
  const char* name = "hqq_b200_glue_sample_slots";
  HQQ_REQUIRE(logits && temperature && top_k && top_p && out && (pos ? seq != nullptr : counter != nullptr), HQQ_E_INVALID, "%s: null pointer", name);
  if (int rc = rows_per_slot_args(name, rows_per_slot, rows)) return rc;
  const SlotParams params{temperature, (const int*)top_k, top_p, rows_per_slot};
  if (pos)
    return sample_launch(name, logits, n, ld, rows, params, seed, PosKeys{(const long long*)pos, (const long long*)seq, rows_per_slot}, out, dtype, stream);
  return sample_launch(name, logits, n, ld, rows, params, seed, StepKeys{(const unsigned long long*)counter}, out, dtype, stream);
}

extern "C" int hqq_b200_glue_penalize(const void* logits, int n, int ld, int rows, int rows_per_slot, const float* repetition, const float* frequency,
                                      const float* presence, int32_t* counts, const uint8_t* prompt, const int64_t* tok, void* out, int ld_out, int dtype,
                                      void* stream) {
  const char* name = "hqq_b200_glue_penalize";
  HQQ_REQUIRE(logits && repetition && frequency && presence && counts && prompt && out, HQQ_E_INVALID, "%s: null pointer", name);
  HQQ_REQUIRE(dtype == HQQ_F16 || dtype == HQQ_BF16, HQQ_E_INVALID, "%s: dtype must be f16/bf16", name);
  HQQ_REQUIRE(n > 0 && ld >= n && ld_out >= n && rows > 0, HQQ_E_INVALID, "%s: needs n > 0, ld >= n, ld_out >= n and rows >= 1 (n=%d ld=%d ld_out=%d rows=%d)",
              name, n, ld, ld_out, rows);
  if (int rc = rows_per_slot_args(name, rows_per_slot, rows)) return rc;
  HQQ_REQUIRE(rows / rows_per_slot <= 65535, HQQ_E_INVALID, "%s: at most 65535 slots (rows=%d rows_per_slot=%d)", name, rows, rows_per_slot);
  HQQ_REQUIRE(aligned(out, 16) && ld_out % 8 == 0, HQQ_E_INVALID, "%s: output rows must start on 16-byte boundaries (out 16-byte aligned, ld_out %% 8 == 0; "
              "ld_out=%d)", name, ld_out);
  const char *a = (const char*)logits, *b = (const char*)out;
  const long long span_in = ((long long)(rows - 1) * ld + n) * 2, span_out = ((long long)(rows - 1) * ld_out + n) * 2;
  HQQ_REQUIRE(b >= a + span_in || a >= b + span_out, HQQ_E_INVALID, "%s: out must not overlap logits", name);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)cdiv(n, kPenChunk), (unsigned)(rows / rows_per_slot));
  auto go = [&](auto t) {
    using E = decltype(t);
    return launch_pdl("penalize", penalize_kernel<E>, grid, dim3(kPenThreads), 0, st, (const E*)logits, n, (long long)ld, rows_per_slot, repetition, frequency,
                      presence, (int*)counts, (const unsigned char*)prompt, (const long long*)tok, (E*)out, (long long)ld_out);
  };
  return dtype == HQQ_F16 ? go(__half()) : go(__nv_bfloat16());
}

#ifndef HQQ_EMU
extern "C" int hqq_b200_glue_argmax(const void* logits, int n, int64_t* out, int dtype, void* stream) {
  HQQ_REQUIRE(logits && out && n > 0, HQQ_E_INVALID, "hqq_b200_glue_argmax: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == HQQ_F16) return launch_pdl("argmax", argmax_kernel<__half>, dim3(kArgmaxCtas), dim3(1024), 0, st, (const __half*)logits, n, (long long*)out, -1LL, KeyPeers{}, 0, 0, (const int*)nullptr);
  if (dtype == HQQ_BF16) return launch_pdl("argmax", argmax_kernel<__nv_bfloat16>, dim3(kArgmaxCtas), dim3(1024), 0, st, (const __nv_bfloat16*)logits, n, (long long*)out, -1LL, KeyPeers{}, 0, 0, (const int*)nullptr);
  set_error("hqq_b200_glue_argmax: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_argmax_key(const void* logits, int n, int64_t index_offset, int64_t* out_key, int dtype, void* stream) {
  HQQ_REQUIRE(logits && out_key && n > 0 && index_offset >= 0 && index_offset + n <= 0xFFFFFFFFll, HQQ_E_INVALID, "hqq_b200_glue_argmax_key: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == HQQ_F16) return launch_pdl("argmax_key", argmax_kernel<__half>, dim3(kArgmaxCtas), dim3(1024), 0, st, (const __half*)logits, n, (long long*)out_key, (long long)index_offset, KeyPeers{}, 0, 0, (const int*)nullptr);
  if (dtype == HQQ_BF16) return launch_pdl("argmax_key", argmax_kernel<__nv_bfloat16>, dim3(kArgmaxCtas), dim3(1024), 0, st, (const __nv_bfloat16*)logits, n, (long long*)out_key, (long long)index_offset, KeyPeers{}, 0, 0, (const int*)nullptr);
  set_error("hqq_b200_glue_argmax_key: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_glue_argmax_tp(const void* logits, int n, int64_t index_offset, void* const* peer_keys, int tp, int rank, const int* step_ctr,
                                       int64_t* out, int dtype, void* stream) {
  HQQ_REQUIRE(logits && out && peer_keys && step_ctr && n > 0 && index_offset >= 0 && index_offset + n <= 0xFFFFFFFFll && tp >= 1 && tp <= 8 &&
                  rank >= 0 && rank < tp,
              HQQ_E_INVALID, "hqq_b200_glue_argmax_tp: bad arguments (n=%d tp=%d rank=%d)", n, tp, rank);
  KeyPeers kp = {};
  for (int i = 0; i < tp; ++i) {
    HQQ_REQUIRE(peer_keys[i] && ((uintptr_t)peer_keys[i] & 7) == 0, HQQ_E_INVALID, "hqq_b200_glue_argmax_tp: key area %d must be 8-byte aligned", i);
    kp.p[i] = (unsigned long long*)peer_keys[i];
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == HQQ_F16) return launch_pdl("argmax_tp", argmax_kernel<__half>, dim3(kArgmaxCtas), dim3(1024), 0, st, (const __half*)logits, n, (long long*)out, (long long)index_offset, kp, tp, rank, step_ctr);
  if (dtype == HQQ_BF16) return launch_pdl("argmax_tp", argmax_kernel<__nv_bfloat16>, dim3(kArgmaxCtas), dim3(1024), 0, st, (const __nv_bfloat16*)logits, n, (long long*)out, (long long)index_offset, kp, tp, rank, step_ctr);
  set_error("hqq_b200_glue_argmax_tp: dtype must be f16/bf16");
  return HQQ_E_INVALID;
}
#endif  // !HQQ_EMU
