// Quantizer.quantize on sm_90a: min/max init -> proximal (half-quadratic) zero-point solver with the
// reference's whole-tensor early stop -> round/clamp -> bit-pack.  Three launches, no host sync:
//
//   K1 solver_kernel     every group runs ALL `iters` iterations on-chip (weights stay in registers),
//                        writes its zero-point trajectory hist[it][g] and adds its share of the
//                        per-iteration error sums into a per-block partial (fixed order -> deterministic)
//   K2 stop_kernel       one block: reduces the partials in a fixed order (float64), replays the
//                        reference's `if err < best: best = err else: break` and publishes the slot to use
//   K3 quant_pack_kernel W_q = clamp(rint(W*s + z_sel)) packed into the reference's slab layout,
//                        plus scale_out = 1/s, zero_out = z_sel
//
// Reference: hqq/core/quantize.py:102-176, hqq/core/optimize.py:96-108,201-255 (float32 path).
// Arithmetic notes (see DESIGN.md "parity"): everything is fp32 with explicit non-fused mul/add where the
// final W_q depends on it; inside the solver W_r = (W_q - z) * (1/s) replaces the division and
// |x|^(p-1) is ex2(p-1 * lg2|x|) on the SFU -- both perturb the zero-point at the 1e-7 relative level.
#include <math.h>
#include <stdlib.h>

#include "common.cuh"

namespace hqq {

static constexpr int kMaxIters = 64;
static constexpr int kSolverThreads = 256;

struct SolverArgs {
  const void* W;
  long long total, G;  // elements, groups
  int gs;
  int maxv, round_zero, iters, lp_is_one;
  float inv_beta, pm1;
  float thr;  // |W - W_r| below this shrinks to exactly 0 (see solver_axis1_kernel); 0 disables the shortcut
  const float* s_init;  // optional [G]: caller-supplied inverse scale / zero (optimize_weights_proximal seam)
  const float* z_init;
  float* s_inv;     // [G]   inverse scale (the solver's `scale`)
  float* hist;      // [iters+1][G] zero-point trajectory, slot 0 = initial zero
  double* partial;  // [gridDim.x][iters]
};

__device__ __forceinline__ float rint_magic(float t) {
  // round-half-even for |t| < 2^22; beyond that the result is still >= 2^22-ish in magnitude with the
  // right sign, so the clamp that always follows yields the same level as rintf would.
  return __fsub_rn(__fadd_rn(t, 12582912.0f), 12582912.0f);
}

struct GroupState {
  float s, rs, z;
};

__device__ __forceinline__ void init_group_ext(const SolverArgs& a, long long g, bool valid, GroupState& st) {
  const float s = valid ? a.s_init[g] : 1.0f;
  st.s = s;
  st.rs = __frcp_rn(s);
  st.z = valid ? a.z_init[g] : 0.0f;
}

__device__ __forceinline__ void init_group(float mn, float mx, int maxv, int round_zero, GroupState& st) {
  // quantize.py:126-134 ; `max_v / denom` is reciprocal(denom) * max_v in torch (two roundings)
  float denom = __fsub_rn(mx, mn);
  float s = __fmul_rn(__frcp_rn(denom), (float)maxv);
  if (fabsf(denom) <= 1e-4f) s = 1.0f;
  s = fminf(s, 2e4f);
  float z = __fmul_rn(-mn, s);
  if (round_zero) z = rintf(z);
  st.s = s;
  st.rs = __frcp_rn(s);
  st.z = z;
}

// Group mean of the zero-point terms: float64 accumulation (the terms are float32 values of magnitude <= 2^nbits, so the sum of a
// group is exact or within one float64 ulp), rounded to float32 once -- torch.mean's result on the reference's CPU path
// (vectorised float32 partial sums) equals this level for level on every golden fixture, where a float32 shuffle tree lands one
// ulp away in about half of the groups and flips a rounding tie now and then.  The order of the float64 additions is fixed
// (lane-local sequence, then xor-shuffle tree), so results stay deterministic and identical across the solver variants.
__device__ __forceinline__ float zero_mean(double zs, int gs) {
  // sum / n: for a power-of-two n the product with 1/n is exact (no double division; n is a compile-time constant on the
  // register-resident paths), otherwise the float64 quotient, rounded to float32 once either way
  if ((gs & (gs - 1)) == 0) return (float)(zs * (1.0 / (double)gs));
  return (float)(zs / (double)gs);
}

// One solver update for one element; returns its contribution to the zero-point sum.
__device__ __forceinline__ float solver_elem(float w, const GroupState& st, float fmaxv, float inv_beta, float pm1,
                                             int lp_is_one, float& errsum) {
  float q = rint_magic(__fadd_rn(__fmul_rn(w, st.s), st.z));
  q = fminf(fmaxf(q, 0.0f), fmaxv);
  float wr = __fmul_rn(__fsub_rn(q, st.z), st.rs);
  float d = __fsub_rn(w, wr);
  float a = fabsf(d);
  errsum += a;
  float e;
  if (lp_is_one) {
    e = fmaxf(__fsub_rn(a, inv_beta), 0.0f);
  } else {
    float p = exp2f(pm1 * __log2f(a));  // a^(p-1); a == 0 -> +inf (p<1) -> e == 0, as in the reference
    e = fmaxf(__fsub_rn(a, __fmul_rn(inv_beta, p)), 0.0f);
  }
  e = copysignf(e, d);
  return __fsub_rn(q, __fmul_rn(__fsub_rn(w, e), st.s));
}

template <typename TIn>
__device__ __forceinline__ void load8_group(const TIn* base, int l, int L, float (&w)[8]);
template <>
__device__ __forceinline__ void load8_group<float>(const float* base, int l, int L, float (&w)[8]) {
  // two coalesced float4 loads: chunk c covers elements (c*L + l)*4 .. +3 of the group
  float4 a = __ldg(reinterpret_cast<const float4*>(base) + l);
  float4 b = __ldg(reinterpret_cast<const float4*>(base) + L + l);
  w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
  w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}
// 16-bit sources use the SAME element-to-lane assignment as float32 (chunk c of lane l = elements (c*L + l)*4 .. +3), so that
// quantising a half tensor is bit-identical to quantising its float32 copy (tensor.float() is exact, quantize.py:102).
template <>
__device__ __forceinline__ void load8_group<__half>(const __half* base, int l, int L, float (&w)[8]) {
  const uint2 a = __ldg(reinterpret_cast<const uint2*>(base) + l);
  const uint2 b = __ldg(reinterpret_cast<const uint2*>(base) + L + l);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
    w[2 * j] = fa.x; w[2 * j + 1] = fa.y;
    w[4 + 2 * j] = fb.x; w[4 + 2 * j + 1] = fb.y;
  }
}
template <>
__device__ __forceinline__ void load8_group<__nv_bfloat16>(const __nv_bfloat16* base, int l, int L, float (&w)[8]) {
  const uint2 a = __ldg(reinterpret_cast<const uint2*>(base) + l);
  const uint2 b = __ldg(reinterpret_cast<const uint2*>(base) + L + l);
  const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&a);
  const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&b);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float2 fa = __bfloat1622float2(ha[j]), fb = __bfloat1622float2(hb[j]);
    w[2 * j] = fa.x; w[2 * j + 1] = fa.y;
    w[4 + 2 * j] = fb.x; w[4 + 2 * j + 1] = fb.y;
  }
}

// Adds this warp's per-iteration error into its private shared-memory row, then (at kernel end) the block
// sums its warps in a fixed order.  No atomics anywhere -> bit-reproducible error sums.
struct ErrAcc {
  double* row;  // smem [kMaxIters] private to the warp
  __device__ __forceinline__ void add(int it, float errsum) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) errsum += __shfl_xor_sync(0xffffffffu, errsum, o);
    if ((threadIdx.x & 31) == 0) row[it] += (double)errsum;
  }
};

__device__ __forceinline__ void block_flush_errors(double (*err_w)[kMaxIters], int iters, double* partial) {
  __syncthreads();
  if ((int)threadIdx.x < iters) {
    double s = 0.0;
    for (int w = 0; w < kSolverThreads / 32; ++w) s += err_w[w][threadIdx.x];
    partial[(long long)blockIdx.x * iters + threadIdx.x] = s;
  }
}

// ---- K1, axis = 1: group = gs contiguous elements = L lanes x 8 elements, weights in registers -------------------------
// Two exact shortcuts over the plain 20-iteration loop (solver_generic_kernel below is that plain loop; the results are
// bit-identical, tests/test_quantize_gpu.py::test_register_solver_equals_plain_loop):
//  (1) shrink_lp_op(x) is exactly 0 wherever |x| - (1/beta)|x|^(p-1) <= 0, i.e. |x| <= beta^(-1/(2-p)) (0.170 for the
//      default beta = 10, p = 0.7; optimize.py:96-108).  Quantisation errors of real weight matrices are far below that,
//      so W_e = 0, `W_f - W_e` = W_f and the update collapses to z = mean(W_q - W_f*scale): no SFU work, and W_f*scale is
//      loop-invariant.  The warp falls back to the full formula whenever any of its elements is at or above `thr`
//      (= 0.9 x the root, a 10 % margin against the 2^-22 error of ex2/lg2) -- a warp-uniform branch.
//  (2) one iteration is a deterministic function of the group's zero-point alone.  Once z_{i+1} == z_i (bitwise) every later
//      iteration repeats the same W_q, error and zero, so the warp stops as soon as all of its groups sit on a fixed point and
//      writes the remaining trajectory slots / error sums without recomputing them (measured on Gaussian weights: a group is
//      fixed after 3.4 iterations on average, a warp of four groups after 7.4, instead of 20).
template <typename TIn, int L>
__global__ void __launch_bounds__(kSolverThreads) solver_axis1_kernel(SolverArgs a) {
  __shared__ double err_w[kSolverThreads / 32][kMaxIters];
  for (int i = threadIdx.x; i < (kSolverThreads / 32) * kMaxIters; i += blockDim.x) (&err_w[0][0])[i] = 0.0;
  __syncthreads();
  double* row = err_w[threadIdx.x >> 5];
  constexpr int GPW = 32 / L;
  const int lane = threadIdx.x & 31, l = lane % L;
  const long long warp_global = (long long)blockIdx.x * (kSolverThreads / 32) + (threadIdx.x >> 5);
  const long long warp_stride = (long long)gridDim.x * (kSolverThreads / 32);
  const float fmaxv = (float)a.maxv;
  const float thr = a.thr;
  const TIn* W = reinterpret_cast<const TIn*>(a.W);

  for (long long gb = warp_global * GPW; gb < a.G; gb += warp_stride * GPW) {  // warp-uniform
    const long long g = gb + lane / L;
    const bool valid = g < a.G;
    float w[8];
    if (valid) {
      load8_group<TIn>(W + g * (long long)a.gs, l, L, w);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = 0.0f;
    }
    float mn = w[0], mx = w[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) { mn = fminf(mn, w[j]); mx = fmaxf(mx, w[j]); }
#pragma unroll
    for (int o = 1; o < L; o <<= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    GroupState st;
    if (a.s_init) init_group_ext(a, g, valid, st);
    else init_group(mn, mx, a.maxv, a.round_zero, st);
    if (valid && l == 0) { a.s_inv[g] = st.s; a.hist[g] = st.z; }
    float ws[8];  // W_f * scale, the same rounding solver_elem applies every iteration
#pragma unroll
    for (int j = 0; j < 8; ++j) ws[j] = __fmul_rn(w[j], st.s);
    float ew = 0.0f;  // warp-wide error sum of the last iteration executed
    int it = 0;
    while (it < a.iters) {
      float errsum = 0.0f, amax = 0.0f;
      double zs = 0.0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float q = rint_magic(__fadd_rn(ws[j], st.z));
        q = fminf(fmaxf(q, 0.0f), fmaxv);
        const float wr = __fmul_rn(__fsub_rn(q, st.z), st.rs);
        const float ad = fabsf(__fsub_rn(w[j], wr));
        errsum += ad;
        amax = fmaxf(amax, ad);
        zs += (double)__fsub_rn(q, ws[j]);
      }
      if (__any_sync(0xffffffffu, !(amax < thr))) {  // some |W - W_r| may survive the shrinkage: full formula for the warp
        zs = 0.0;
        float unused = 0.0f;
#pragma unroll
        for (int j = 0; j < 8; ++j) zs += (double)solver_elem(w[j], st, fmaxv, a.inv_beta, a.pm1, a.lp_is_one, unused);
      }
#pragma unroll
      for (int o = 1; o < L; o <<= 1) zs += __shfl_xor_sync(0xffffffffu, zs, o);
      const float znew = zero_mean(zs, 8 * L);  // torch.mean = sum / n, exactly as solver_axis1_kernel
      if (valid && l == 0) a.hist[(long long)(it + 1) * a.G + g] = znew;
      ew = valid ? errsum : 0.0f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ew += __shfl_xor_sync(0xffffffffu, ew, o);  // same order as ErrAcc::add
      if (lane == 0) row[it] += (double)ew;
      const bool fixed = !valid || __float_as_uint(znew) == __float_as_uint(st.z);
      st.z = znew;
      ++it;
      if (__all_sync(0xffffffffu, fixed)) break;
    }
    // iterations it .. iters-1 would reproduce (st.z, ew) exactly: fill their slots without recomputing them
    __syncwarp();
    if (valid)
      for (int t = it + l; t < a.iters; t += L) a.hist[(long long)(t + 1) * a.G + g] = st.z;
    for (int t = it + lane; t < a.iters; t += 32) row[t] += (double)ew;
    __syncwarp();
  }
  block_flush_errors(err_w, a.iters, a.partial);
}

// ---- K1, axis = 0: group g = column g of the [GS, C] view, one thread per group; the two exact shortcuts of
// solver_axis1_kernel (32 groups per warp: the warp leaves once all 32 zero-points repeat) ------------------------------------
template <typename TIn, int GS>
__global__ void __launch_bounds__(kSolverThreads) solver_axis0_kernel(SolverArgs a) {
  __shared__ double err_w[kSolverThreads / 32][kMaxIters];
  for (int i = threadIdx.x; i < (kSolverThreads / 32) * kMaxIters; i += blockDim.x) (&err_w[0][0])[i] = 0.0;
  __syncthreads();
  double* row = err_w[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const long long C = a.G;
  const float fmaxv = (float)a.maxv;
  const float thr = a.thr;
  const TIn* W = reinterpret_cast<const TIn*>(a.W);
  const long long stride = (long long)gridDim.x * kSolverThreads;
  const long long first = (long long)blockIdx.x * kSolverThreads + (threadIdx.x & ~31);
  for (long long gb = first; gb < C; gb += stride) {  // warp-uniform trip count
    const long long g = gb + lane;
    const bool valid = g < C;
    float w[GS];
#pragma unroll
    for (int j = 0; j < GS; ++j) w[j] = valid ? to_f32<TIn>(W[(long long)j * C + g]) : 0.0f;
    float mn = w[0], mx = w[0];
#pragma unroll
    for (int j = 1; j < GS; ++j) { mn = fminf(mn, w[j]); mx = fmaxf(mx, w[j]); }
    GroupState st;
    if (a.s_init) init_group_ext(a, g, valid, st);
    else init_group(mn, mx, a.maxv, a.round_zero, st);
    if (valid) { a.s_inv[g] = st.s; a.hist[g] = st.z; }
    float ew = 0.0f;
    int it = 0;
    while (it < a.iters) {
      float errsum = 0.0f, amax = 0.0f;
      double zs = 0.0;
#pragma unroll
      for (int j = 0; j < GS; ++j) {
        const float ws = __fmul_rn(w[j], st.s);
        float q = rint_magic(__fadd_rn(ws, st.z));
        q = fminf(fmaxf(q, 0.0f), fmaxv);
        const float wr = __fmul_rn(__fsub_rn(q, st.z), st.rs);
        const float ad = fabsf(__fsub_rn(w[j], wr));
        errsum += ad;
        amax = fmaxf(amax, ad);
        zs += (double)__fsub_rn(q, ws);
      }
      if (__any_sync(0xffffffffu, !(amax < thr))) {
        zs = 0.0;
        float unused = 0.0f;
#pragma unroll
        for (int j = 0; j < GS; ++j) zs += (double)solver_elem(w[j], st, fmaxv, a.inv_beta, a.pm1, a.lp_is_one, unused);
      }
      const float znew = zero_mean(zs, GS);
      if (valid) a.hist[(long long)(it + 1) * a.G + g] = znew;
      ew = valid ? errsum : 0.0f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ew += __shfl_xor_sync(0xffffffffu, ew, o);
      if (lane == 0) row[it] += (double)ew;
      const bool fixed = !valid || __float_as_uint(znew) == __float_as_uint(st.z);
      st.z = znew;
      ++it;
      if (__all_sync(0xffffffffu, fixed)) break;
    }
    __syncwarp();
    if (valid)
      for (int t = it; t < a.iters; ++t) a.hist[(long long)(t + 1) * a.G + g] = st.z;
    for (int t = it + lane; t < a.iters; t += 32) row[t] += (double)ew;
    __syncwarp();
  }
  block_flush_errors(err_w, a.iters, a.partial);
}

// ---- K1, generic path: one warp per group, any gs / axis; elements are re-read (L1/L2) every iteration --
template <typename TIn>
__global__ void __launch_bounds__(kSolverThreads) solver_generic_kernel(SolverArgs a, int axis) {
  __shared__ double err_w[kSolverThreads / 32][kMaxIters];
  for (int i = threadIdx.x; i < (kSolverThreads / 32) * kMaxIters; i += blockDim.x) (&err_w[0][0])[i] = 0.0;
  __syncthreads();
  ErrAcc acc{err_w[threadIdx.x >> 5]};
  const int lane = threadIdx.x & 31;
  const long long warp_global = (long long)blockIdx.x * (kSolverThreads / 32) + (threadIdx.x >> 5);
  const long long warp_stride = (long long)gridDim.x * (kSolverThreads / 32);
  const float fmaxv = (float)a.maxv;
  const TIn* W = reinterpret_cast<const TIn*>(a.W);
  const long long estride = (axis == 1) ? 1 : a.G;
  for (long long g = warp_global; g < a.G; g += warp_stride) {
    const TIn* base = (axis == 1) ? W + g * (long long)a.gs : W + g;
    float mn = INFINITY, mx = -INFINITY;
    for (int e = lane; e < a.gs; e += 32) {
      float w = to_f32<TIn>(base[(long long)e * estride]);
      mn = fminf(mn, w); mx = fmaxf(mx, w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    GroupState st;
    if (a.s_init) init_group_ext(a, g, true, st);
    else init_group(mn, mx, a.maxv, a.round_zero, st);
    if (lane == 0) { a.s_inv[g] = st.s; a.hist[g] = st.z; }
    for (int it = 0; it < a.iters; ++it) {
      float errsum = 0.0f;
      double zs = 0.0;
      for (int e = lane; e < a.gs; e += 32) {
        float w = to_f32<TIn>(base[(long long)e * estride]);
        zs += (double)solver_elem(w, st, fmaxv, a.inv_beta, a.pm1, a.lp_is_one, errsum);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) zs += __shfl_xor_sync(0xffffffffu, zs, o);
      st.z = zero_mean(zs, a.gs);
      if (lane == 0) a.hist[(long long)(it + 1) * a.G + g] = st.z;
      acc.add(it, errsum);
    }
  }
  block_flush_errors(err_w, a.iters, a.partial);
}

// ---- K2: fixed-order reduction of the error partials + the reference's early-stop rule -----------------
// Sharded quantisation (SURVEY 8e, optimize.py:239-247 compares a WHOLE-tensor mean): with `sums_out` the kernel stops after the
// reduction and hands the `iters` float64 error sums of this shard to the caller, who adds the shards' sums (one all-reduce of
// iters x 8 bytes) and comes back with `sums_in` (global sums) and the global element count in `total`.
__global__ void __launch_bounds__(1024) stop_kernel(const double* __restrict__ partial, int nblocks, int iters, long long total,
                                                    int32_t* __restrict__ info, float* __restrict__ err_out,
                                                    const double* __restrict__ sums_in, double* __restrict__ sums_out) {
  __shared__ double e[kMaxIters];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (sums_in) {
    if ((int)threadIdx.x < iters) e[threadIdx.x] = sums_in[threadIdx.x];
  } else {
    for (int it = warp; it < iters; it += 32) {
      double s = 0.0;
      for (int b = lane; b < nblocks; b += 32) s += partial[(long long)b * iters + it];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) e[it] = s;
    }
  }
  __syncthreads();
  if (sums_out) {
    if ((int)threadIdx.x < iters) sums_out[threadIdx.x] = e[threadIdx.x];
    return;
  }
  if (threadIdx.x == 0) {
    // optimize.py:236-247: best = inf; for i: err = mean|W - W_r| (float32); if err < best: best = err else break
    float best = INFINITY;
    int done = 0;
    for (int it = 0; it < iters; ++it) {
      float err = (float)(e[it] / (double)total);
      if (err_out) err_out[it] = err;
      done = it + 1;
      if (err < best) best = err; else break;
    }
    if (err_out) for (int it = done; it < iters; ++it) err_out[it] = (float)(e[it] / (double)total);
    info[0] = done;  // iterations the reference would have executed
    info[1] = done;  // hist slot holding the zero it returns (slot i+1 = zero after iteration i)
    info[2] = 0; info[3] = 0;
  }
}

// ---- K3: final rounding with the selected zero + slab packing + meta outputs ---------------------------
template <int NBITS> struct QPk {
  static constexpr int F = 8 / NBITS;
  using T = uint8_t;
  __device__ __forceinline__ static int shift(int f) { return 8 - NBITS * (f + 1); }
};
template <> struct QPk<3> {
  static constexpr int F = 10;
  using T = int32_t;
  __device__ __forceinline__ static int shift(int f) { return 27 - 3 * f; }
};

template <int NBITS, typename TIn, int V, int AXIS>
__global__ void __launch_bounds__(256) quant_pack_kernel(const TIn* __restrict__ W, const float* __restrict__ s_inv,
                                                         const float* __restrict__ hist, const int32_t* __restrict__ info,
                                                         typename QPk<NBITS>::T* __restrict__ out, long long n, long long total,
                                                         long long gdiv, long long G, int maxv, float* __restrict__ scale_out,
                                                         float* __restrict__ zero_out) {
  using P = QPk<NBITS>;
  const int sel = info ? info[1] : 0;
  const float* __restrict__ zero = hist + (long long)sel * G;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long i = tid * V;
  if (i < n) {
    Vec<typename P::T, V> o;
#pragma unroll
    for (int j = 0; j < V; ++j) o.v[j] = 0;
#pragma unroll
    for (int f = 0; f < P::F; ++f) {
      const long long e = i + (long long)f * n;
      if (e < total) {
        Vec<TIn, V> w = *reinterpret_cast<const Vec<TIn, V>*>(W + e);
        float s[V], z[V];
        if (AXIS == 1) {
          const long long g = e / gdiv;
          const float sg = s_inv[g], zg = zero[g];
#pragma unroll
          for (int j = 0; j < V; ++j) { s[j] = sg; z[j] = zg; }
        } else {
          const long long c = e % gdiv;
#pragma unroll
          for (int j = 0; j < V; ++j) { s[j] = s_inv[c + j]; z[j] = zero[c + j]; }
        }
#pragma unroll
        for (int j = 0; j < V; ++j) {
          // optimize.py:254 / quantize.py:147: round(W*scale + zero).clamp(min,max); mul and add round separately
          // rint and the float -> int conversion as float adds (ncu: this kernel was bound by the conversion pipe): below 2^22
          // rint_magic is rintf, beyond it the clamp decides alike; a clamped level (0 .. 255) + 1.5 * 2^23 carries it in its low bits
          float t = rint_magic(__fadd_rn(__fmul_rn(to_f32<TIn>(w.v[j]), s[j]), z[j]));
          t = fminf(fmaxf(t, 0.0f), (float)maxv);
          const uint32_t q = __float_as_uint(__fadd_rn(t, 12582912.0f)) & 0xFFu;
          o.v[j] = (typename P::T)((uint32_t)o.v[j] | (q << P::shift(f)));
        }
      }
    }
    *reinterpret_cast<Vec<typename P::T, V>*>(out + i) = o;
  }
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (long long g = tid; g < G; g += nthreads) {
    scale_out[g] = __frcp_rn(s_inv[g]);  // quantize.py:154 scale = 1.0 / scale
    zero_out[g] = zero[g];
  }
}

// ---------------------------------------------------------------------------------------------------------
struct Layout {
  long long total, G, R, C, n_packed;
  int nblocks;
  size_t off_s, off_hist, off_partial, off_info, bytes;
};

static bool fast_axis1(int gs) { return gs == 8 || gs == 16 || gs == 32 || gs == 64 || gs == 128 || gs == 256; }
static bool fast_axis0(int gs) { return gs == 8 || gs == 16 || gs == 32 || gs == 64; }

static Layout make_layout(long long N, long long K, int gs, int nbits, int axis, int iters) {
  Layout L;
  L.total = N * K;
  L.G = L.total / gs;
  L.R = (axis == 1) ? L.G : gs;
  L.C = (axis == 1) ? gs : L.G;
  const int F = fields_of(nbits);
  L.n_packed = ((nbits == 3) ? cdiv(L.R, 10) : L.R / F) * L.C;
  long long per_block;
  if (axis == 1 && fast_axis1(gs)) per_block = (kSolverThreads / (gs / 8));
  else if (axis == 0 && fast_axis0(gs)) per_block = kSolverThreads;
  else per_block = kSolverThreads / 32;
  long long nb = cdiv(L.G, per_block);
  const long long cap = (long long)kNumSMs * 8;
  L.nblocks = (int)(nb < 1 ? 1 : (nb > cap ? cap : nb));
  auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
  size_t o = 0;
  L.off_s = o; o = up(o + sizeof(float) * L.G);
  L.off_hist = o; o = up(o + sizeof(float) * L.G * (size_t)(iters + 1));
  L.off_partial = o; o = up(o + sizeof(double) * (size_t)L.nblocks * (iters > 0 ? iters : 1));
  L.off_info = o; o = up(o + 64);
  L.bytes = o;
  return L;
}

// HQQ_B200_PLAIN_SOLVER=1 (test hook, read per call): every configuration runs solver_generic_kernel, the plain loop without
// the two shortcuts -- the GPU tests use it to show the register-resident kernels bit-identical to it.
static bool plain_solver() {
  const char* e = getenv("HQQ_B200_PLAIN_SOLVER");
  return e && e[0] == '1';
}

template <typename TIn>
static int launch_solver(const SolverArgs& a, int axis, int nblocks, cudaStream_t st) {
  if (axis == 1 && fast_axis1(a.gs) && !plain_solver()) {
    switch (a.gs / 8) {
      case 1: solver_axis1_kernel<TIn, 1><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 2: solver_axis1_kernel<TIn, 2><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 4: solver_axis1_kernel<TIn, 4><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 8: solver_axis1_kernel<TIn, 8><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 16: solver_axis1_kernel<TIn, 16><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 32: solver_axis1_kernel<TIn, 32><<<nblocks, kSolverThreads, 0, st>>>(a); break;
    }
  } else if (axis == 0 && fast_axis0(a.gs) && !plain_solver()) {
    switch (a.gs) {
      case 8: solver_axis0_kernel<TIn, 8><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 16: solver_axis0_kernel<TIn, 16><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 32: solver_axis0_kernel<TIn, 32><<<nblocks, kSolverThreads, 0, st>>>(a); break;
      case 64: solver_axis0_kernel<TIn, 64><<<nblocks, kSolverThreads, 0, st>>>(a); break;
    }
  } else {
    solver_generic_kernel<TIn><<<nblocks, kSolverThreads, 0, st>>>(a, axis);
  }
  HQQ_LAUNCH_CHECK("hqq_b200_quantize/solver");
  return HQQ_OK;
}

template <int NBITS, typename TIn>
static int launch_quant_pack(const void* W, const float* s_inv, const float* hist, const int32_t* info, void* out, const Layout& L,
                             int gs, int axis, int maxv, float* scale_out, float* zero_out, cudaStream_t st) {
  using PT = typename QPk<NBITS>::T;
  const long long n = L.n_packed;
  const size_t a_in = 4 * sizeof(TIn) >= 16 ? 16 : 4 * sizeof(TIn);
  bool vec = (n % 4 == 0) && (L.total % 4 == 0) && aligned(W, a_in) && aligned(out, 4 * sizeof(PT)) &&
             (axis == 1 ? (gs % 4 == 0) : (L.C % 4 == 0));
  const long long gdiv = (axis == 1) ? gs : L.C;
  // 16-bit sources: 8 packed elements per thread -> 16-byte loads of W instead of 8-byte ones
  const bool vec8 = vec && sizeof(TIn) == 2 && axis == 1 && (n % 8 == 0) && (L.total % 8 == 0) &&
                    (gs % 8 == 0) && aligned(W, 16) && aligned(out, 8 * sizeof(PT) >= 16 ? 16 : 8 * sizeof(PT));
  if (vec8) {
    unsigned grid = (unsigned)cdiv(cdiv(n, 8), 256);
    quant_pack_kernel<NBITS, TIn, 8, 1><<<grid, 256, 0, st>>>((const TIn*)W, s_inv, hist, info, (PT*)out, n, L.total, gdiv, L.G, maxv, scale_out, zero_out);
  } else if (vec) {
    unsigned grid = (unsigned)cdiv(cdiv(n, 4), 256);
    if (axis == 1) quant_pack_kernel<NBITS, TIn, 4, 1><<<grid, 256, 0, st>>>((const TIn*)W, s_inv, hist, info, (PT*)out, n, L.total, gdiv, L.G, maxv, scale_out, zero_out);
    else quant_pack_kernel<NBITS, TIn, 4, 0><<<grid, 256, 0, st>>>((const TIn*)W, s_inv, hist, info, (PT*)out, n, L.total, gdiv, L.G, maxv, scale_out, zero_out);
  } else {
    unsigned grid = (unsigned)cdiv(n, 256);
    if (axis == 1) quant_pack_kernel<NBITS, TIn, 1, 1><<<grid, 256, 0, st>>>((const TIn*)W, s_inv, hist, info, (PT*)out, n, L.total, gdiv, L.G, maxv, scale_out, zero_out);
    else quant_pack_kernel<NBITS, TIn, 1, 0><<<grid, 256, 0, st>>>((const TIn*)W, s_inv, hist, info, (PT*)out, n, L.total, gdiv, L.G, maxv, scale_out, zero_out);
  }
  HQQ_LAUNCH_CHECK("hqq_b200_quantize/quant_pack");
  return HQQ_OK;
}

// phase 0: everything; 1: solver + this shard's error sums -> err_sums (trajectories stay in the workspace); 2: early stop from the
// caller's global err_sums / total_override, then round + pack on the same workspace
template <typename TIn>
static int quantize_typed(const void* W, long long N, long long K, int gs, int nbits, int maxv, int axis, int round_zero, int optimize,
                          float lp_norm, float beta, int iters, const float* s_init, const float* z_init, void* Wq, float* scale_out,
                          float* zero_out, int32_t* info_out, float* err_out, char* ws, const Layout& L, cudaStream_t st, int phase = 0,
                          double* err_sums = nullptr, long long total_override = 0) {
  SolverArgs a;
  a.W = W; a.total = L.total; a.G = L.G; a.gs = gs;
  a.s_init = s_init; a.z_init = z_init;
  a.maxv = maxv; a.round_zero = round_zero; a.iters = optimize ? iters : 0;
  a.lp_is_one = (lp_norm == 1.0f); a.inv_beta = 1.0f / beta; a.pm1 = lp_norm - 1.0f;
  // below thr the shrinkage is exactly zero: lp = 1 -> |x| <= 1/beta; lp < 1 -> |x| <= beta^(-1/(2-lp)) (10 % margin for the SFU)
  a.thr = a.lp_is_one ? a.inv_beta : (lp_norm < 1.0f ? 0.9f * (float)pow((double)a.inv_beta, 1.0 / (2.0 - (double)lp_norm)) : 0.0f);
  a.s_inv = reinterpret_cast<float*>(ws + L.off_s);
  a.hist = reinterpret_cast<float*>(ws + L.off_hist);
  a.partial = reinterpret_cast<double*>(ws + L.off_partial);
  int32_t* info = reinterpret_cast<int32_t*>(ws + L.off_info);
  int rc = HQQ_OK;
  if (phase != 2) {
    rc = launch_solver<TIn>(a, axis, L.nblocks, st);
    if (rc) return rc;
  }
  if (a.iters > 0) {
    if (phase == 1) stop_kernel<<<1, 1024, 0, st>>>(a.partial, L.nblocks, a.iters, L.total, info, nullptr, nullptr, err_sums);
    else if (phase == 2) stop_kernel<<<1, 1024, 0, st>>>(a.partial, L.nblocks, a.iters, total_override, info, err_out, err_sums, nullptr);
    else stop_kernel<<<1, 1024, 0, st>>>(a.partial, L.nblocks, a.iters, L.total, info, err_out, nullptr, nullptr);
    HQQ_LAUNCH_CHECK("hqq_b200_quantize/stop");
  }
  if (phase == 1) return HQQ_OK;
  const int32_t* sel = a.iters > 0 ? info : nullptr;
  switch (nbits) {
    case 8: rc = launch_quant_pack<8, TIn>(W, a.s_inv, a.hist, sel, Wq, L, gs, axis, a.maxv, scale_out, zero_out, st); break;
    case 4: rc = launch_quant_pack<4, TIn>(W, a.s_inv, a.hist, sel, Wq, L, gs, axis, a.maxv, scale_out, zero_out, st); break;
    case 3: rc = launch_quant_pack<3, TIn>(W, a.s_inv, a.hist, sel, Wq, L, gs, axis, a.maxv, scale_out, zero_out, st); break;
    case 2: rc = launch_quant_pack<2, TIn>(W, a.s_inv, a.hist, sel, Wq, L, gs, axis, a.maxv, scale_out, zero_out, st); break;
    case 1: rc = launch_quant_pack<1, TIn>(W, a.s_inv, a.hist, sel, Wq, L, gs, axis, a.maxv, scale_out, zero_out, st); break;
  }
  if (rc) return rc;
  if (info_out) {
    if (a.iters > 0) {
      cudaError_t e = cudaMemcpyAsync(info_out, info, 4 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
      HQQ_REQUIRE(e == cudaSuccess, HQQ_E_CUDA, "hqq_b200_quantize: info copy failed: %s", cudaGetErrorString(e));
    } else {
      cudaError_t e = cudaMemsetAsync(info_out, 0, 4 * sizeof(int32_t), st);
      HQQ_REQUIRE(e == cudaSuccess, HQQ_E_CUDA, "hqq_b200_quantize: info memset failed: %s", cudaGetErrorString(e));
    }
  }
  return HQQ_OK;
}

}  // namespace hqq

using namespace hqq;

static int check_quant_args(int64_t N, int64_t K, int gs, int nbits, int axis, int iters) {
  HQQ_REQUIRE(valid_nbits(nbits), HQQ_E_INVALID, "nbits=%d not supported.", nbits);
  HQQ_REQUIRE(axis == 0 || axis == 1, HQQ_E_INVALID, "axis should be either 0 or 1");
  HQQ_REQUIRE(N > 0 && K > 0 && gs > 0, HQQ_E_INVALID, "hqq_b200_quantize: bad shape N=%lld K=%lld group_size=%d", (long long)N, (long long)K, gs);
  HQQ_REQUIRE((N * K) % gs == 0, HQQ_E_INVALID, "group_size should be divisble by the total tensor dimensions. shape: [%lld, %lld], group_size: %d",
              (long long)N, (long long)K, gs);
  HQQ_REQUIRE(iters >= 0 && iters <= kMaxIters, HQQ_E_INVALID, "hqq_b200_quantize: iters=%d outside [0,%d]", iters, kMaxIters);
  const long long total = N * K, G = total / gs;
  const long long R = (axis == 1) ? G : gs;
  HQQ_REQUIRE(nbits == 3 || R % fields_of(nbits) == 0, HQQ_E_INVALID,
              "hqq_b200_quantize: %lld grouped rows cannot be packed %d per byte", R, fields_of(nbits));
  return HQQ_OK;
}

extern "C" size_t hqq_b200_quantize_workspace_bytes(int64_t N, int64_t K, int group_size, int nbits, int axis, int iters) {
  if (check_quant_args(N, K, group_size, nbits, axis, iters)) return 0;
  return make_layout(N, K, group_size, nbits, axis, iters).bytes;
}

extern "C" int hqq_b200_quantize_ex(const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int max_level,
                                    int axis, int round_zero, int optimize, float lp_norm, float beta, int iters,
                                    const float* inv_scale_init, const float* zero_init, void* W_q_out, float* scale_out,
                                    float* zero_out, int32_t* info_out, float* err_out, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  int rc = check_quant_args(N, K, group_size, nbits, axis, iters);
  if (rc) return rc;
  HQQ_REQUIRE(W && W_q_out && scale_out && zero_out && workspace, HQQ_E_INVALID, "hqq_b200_quantize: null pointer");
  HQQ_REQUIRE(beta > 0.0f, HQQ_E_INVALID, "hqq_b200_quantize: beta must be positive");
  HQQ_REQUIRE((inv_scale_init == nullptr) == (zero_init == nullptr), HQQ_E_INVALID, "hqq_b200_quantize: scale/zero init must be given together");
  HQQ_REQUIRE(max_level >= 1 && max_level <= (1 << nbits) - 1, HQQ_E_INVALID, "hqq_b200_quantize: max_level=%d does not fit %d bits", max_level, nbits);
  if (!optimize) iters = 0;
  Layout L = make_layout(N, K, group_size, nbits, axis, iters);
  HQQ_REQUIRE(workspace_bytes >= L.bytes, HQQ_E_WORKSPACE, "hqq_b200_quantize: workspace %zu < required %zu bytes", workspace_bytes, L.bytes);
  HQQ_REQUIRE(aligned(workspace, 256), HQQ_E_INVALID, "hqq_b200_quantize: workspace must be 256-byte aligned");
  HQQ_REQUIRE(aligned(W, 16), HQQ_E_INVALID, "hqq_b200_quantize: W must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = reinterpret_cast<char*>(workspace);
  switch (src_dtype) {
    case HQQ_F32: return quantize_typed<float>(W, N, K, group_size, nbits, max_level, axis, round_zero, optimize, lp_norm, beta, iters, inv_scale_init, zero_init, W_q_out, scale_out, zero_out, info_out, err_out, ws, L, st);
    case HQQ_F16: return quantize_typed<__half>(W, N, K, group_size, nbits, max_level, axis, round_zero, optimize, lp_norm, beta, iters, inv_scale_init, zero_init, W_q_out, scale_out, zero_out, info_out, err_out, ws, L, st);
    case HQQ_BF16: return quantize_typed<__nv_bfloat16>(W, N, K, group_size, nbits, max_level, axis, round_zero, optimize, lp_norm, beta, iters, inv_scale_init, zero_init, W_q_out, scale_out, zero_out, info_out, err_out, ws, L, st);
  }
  set_error("hqq_b200_quantize: unsupported source dtype %d (need f32/f16/bf16)", src_dtype);
  return HQQ_E_INVALID;
}

static int quantize_phase(int phase, const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int axis, int round_zero,
                          float lp_norm, float beta, int iters, void* W_q_out, float* scale_out, float* zero_out, int32_t* info_out,
                          float* err_out, double* err_sums, int64_t total, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_quant_args(N, K, group_size, nbits, axis, iters);
  if (rc) return rc;
  HQQ_REQUIRE(W && workspace && err_sums && iters >= 1, HQQ_E_INVALID, "hqq_b200_quantize_shard: null pointer or no iterations");
  HQQ_REQUIRE(phase == 1 || (W_q_out && scale_out && zero_out && total >= N * K), HQQ_E_INVALID, "hqq_b200_quantize_shard_finish: null output or bad global element count");
  HQQ_REQUIRE(beta > 0.0f, HQQ_E_INVALID, "hqq_b200_quantize: beta must be positive");
  Layout L = make_layout(N, K, group_size, nbits, axis, iters);
  HQQ_REQUIRE(workspace_bytes >= L.bytes, HQQ_E_WORKSPACE, "hqq_b200_quantize: workspace %zu < required %zu bytes", workspace_bytes, L.bytes);
  HQQ_REQUIRE(aligned(workspace, 256) && aligned(W, 16) && aligned(err_sums, 8), HQQ_E_INVALID, "hqq_b200_quantize_shard: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = reinterpret_cast<char*>(workspace);
  const int maxv = (1 << nbits) - 1;
  switch (src_dtype) {
    case HQQ_F32: return quantize_typed<float>(W, N, K, group_size, nbits, maxv, axis, round_zero, 1, lp_norm, beta, iters, nullptr, nullptr, W_q_out, scale_out, zero_out, info_out, err_out, ws, L, st, phase, err_sums, total);
    case HQQ_F16: return quantize_typed<__half>(W, N, K, group_size, nbits, maxv, axis, round_zero, 1, lp_norm, beta, iters, nullptr, nullptr, W_q_out, scale_out, zero_out, info_out, err_out, ws, L, st, phase, err_sums, total);
    case HQQ_BF16: return quantize_typed<__nv_bfloat16>(W, N, K, group_size, nbits, maxv, axis, round_zero, 1, lp_norm, beta, iters, nullptr, nullptr, W_q_out, scale_out, zero_out, info_out, err_out, ws, L, st, phase, err_sums, total);
  }
  set_error("hqq_b200_quantize: unsupported source dtype %d (need f32/f16/bf16)", src_dtype);
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_quantize_shard_begin(const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int axis,
                                             int round_zero, float lp_norm, float beta, int iters, double* err_sums_out, void* workspace,
                                             size_t workspace_bytes, void* stream) {
  return quantize_phase(1, W, src_dtype, N, K, group_size, nbits, axis, round_zero, lp_norm, beta, iters, nullptr, nullptr, nullptr, nullptr, nullptr,
                        err_sums_out, 0, workspace, workspace_bytes, stream);
}

extern "C" int hqq_b200_quantize_shard_finish(const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int axis,
                                              int round_zero, float lp_norm, float beta, int iters, const double* err_sums,
                                              int64_t total_elements, void* W_q_out, float* scale_out, float* zero_out, int32_t* info_out,
                                              float* err_out, void* workspace, size_t workspace_bytes, void* stream) {
  return quantize_phase(2, W, src_dtype, N, K, group_size, nbits, axis, round_zero, lp_norm, beta, iters, W_q_out, scale_out, zero_out, info_out,
                        err_out, const_cast<double*>(err_sums), total_elements, workspace, workspace_bytes, stream);
}

extern "C" int hqq_b200_quantize(const void* W, int src_dtype, int64_t N, int64_t K, int group_size, int nbits, int axis,
                                 int round_zero, int optimize, float lp_norm, float beta, int iters, void* W_q_out, float* scale_out,
                                 float* zero_out, int32_t* info_out, float* err_out, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  return hqq_b200_quantize_ex(W, src_dtype, N, K, group_size, nbits, (1 << nbits) - 1, axis, round_zero, optimize, lp_norm, beta, iters,
                              nullptr, nullptr, W_q_out, scale_out, zero_out, info_out, err_out, workspace, workspace_bytes, stream);
}
