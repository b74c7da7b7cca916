// BitPack pack / unpack and the standalone dequantize kernels (sm_90a).
//
// The reference's "slab interleave" (hqq/core/bitpack.py) is one-dimensional once the matrix
// is flattened: with n = packed_rows*cols packed elements, field f of packed element i is the
// unpacked element i + f*n.  All three kernels below are therefore 1-D streaming kernels:
// each thread owns V consecutive packed elements (one 8/16-byte load) and touches the F
// slabs with fully coalesced 16-byte accesses.  They are HBM-bound: bytes = in + out.
#include "common.cuh"

namespace hqq {

template <int NBITS> struct Pk {
  static constexpr int F = 8 / NBITS;
  using T = uint8_t;
  static constexpr unsigned MASK = (1u << NBITS) - 1u;
  __device__ __forceinline__ static int shift(int f) { return 8 - NBITS * (f + 1); }
};
template <> struct Pk<3> {
  static constexpr int F = 10;
  using T = int32_t;
  static constexpr unsigned MASK = 7u;
  __device__ __forceinline__ static int shift(int f) { return 27 - 3 * f; }
};

template <typename T> __device__ __forceinline__ long long to_ll(T v) { return (long long)v; }
template <> __device__ __forceinline__ long long to_ll<__half>(__half v) { return (long long)__half2float(v); }
template <> __device__ __forceinline__ long long to_ll<__nv_bfloat16>(__nv_bfloat16 v) { return (long long)__bfloat162float(v); }

// ---------------------------------------------------------------------------------------
// pack: out[i] = OR_f  (in[i + f*n] << shift_f)      (bitpack.py:24-28,43-52,69-91,115-128)
// uint8 path reproduces torch's modulo-256 behaviour of `.to(uint8)` and `uint8 << k`.
// ---------------------------------------------------------------------------------------
template <int NBITS, typename TIn, int V>
__global__ void __launch_bounds__(256) pack_kernel(const TIn* __restrict__ in, typename Pk<NBITS>::T* __restrict__ out,
                                                   long long n, long long n_in) {
  using P = Pk<NBITS>;
  long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (i >= n) return;
  Vec<typename P::T, V> o;
#pragma unroll
  for (int j = 0; j < V; ++j) o.v[j] = 0;
#pragma unroll
  for (int f = 0; f < P::F; ++f) {
    long long e = i + (long long)f * n;
    if (e < n_in) {  // only the 3-bit path has (zero) padding; n_in % V == 0 when V > 1
      Vec<TIn, V> w = *reinterpret_cast<const Vec<TIn, V>*>(in + e);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        long long q = to_ll<TIn>(w.v[j]);
        if (NBITS == 3) {
          o.v[j] = (typename P::T)((uint32_t)o.v[j] | ((uint32_t)(int32_t)q << P::shift(f)));
        } else {
          o.v[j] = (typename P::T)((uint32_t)o.v[j] | ((((uint32_t)q & 0xFFu) << P::shift(f)) & 0xFFu));
        }
      }
    }
  }
  *reinterpret_cast<Vec<typename P::T, V>*>(out + i) = o;
}

// ---------------------------------------------------------------------------------------
// unpack: out[i + f*n] = (in[i] >> shift_f) & mask    (bitpack.py:31-38,55-64,95-110,131-144)
// ---------------------------------------------------------------------------------------
template <int NBITS, typename TOut, int V>
__global__ void __launch_bounds__(256) unpack_kernel(const typename Pk<NBITS>::T* __restrict__ in, TOut* __restrict__ out, long long n) {
  using P = Pk<NBITS>;
  long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (i >= n) return;
  Vec<typename P::T, V> p = *reinterpret_cast<const Vec<typename P::T, V>*>(in + i);
#pragma unroll
  for (int f = 0; f < P::F; ++f) {
    Vec<TOut, V> o;
#pragma unroll
    for (int j = 0; j < V; ++j) o.v[j] = level_to<TOut>(((uint32_t)p.v[j] >> P::shift(f)) & P::MASK);
    *reinterpret_cast<Vec<TOut, V>*>(out + i + (long long)f * n) = o;
  }
}

// ---------------------------------------------------------------------------------------
// dequantize: out[e] = (T(q_e) - zero[g(e)]) * scale[g(e)], e = i + f*n < total
//   axis 1: g(e) = e / gs          (grouped matrix [R, gs], meta [R,1])
//   axis 0: g(e) = e % C           (grouped matrix [gs, C], meta [1,C])
// (quantize.py:184-199; hqq_aten_cuda_kernel.cu:35-428 implements the axis-0 case only)
// ---------------------------------------------------------------------------------------
template <int NBITS, typename T, int V, int AXIS>
__global__ void __launch_bounds__(256) dequant_kernel(const typename Pk<NBITS>::T* __restrict__ in, const T* __restrict__ scale,
                                                      const T* __restrict__ zero, T* __restrict__ out, long long n,
                                                      long long total, long long gdiv /* gs (axis1) or C (axis0) */) {
  using P = Pk<NBITS>;
  long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (i >= n) return;
  Vec<typename P::T, V> p = *reinterpret_cast<const Vec<typename P::T, V>*>(in + i);
#pragma unroll
  for (int f = 0; f < P::F; ++f) {
    long long e = i + (long long)f * n;
    if (e >= total) continue;  // 3-bit zero padding (quantize.py:190-195 slices it off)
    Vec<T, V> o;
    if (AXIS == 1) {
      long long g = e / gdiv;  // all V elements share the group (V | gs)
      T s = scale[g], z = zero[g];
#pragma unroll
      for (int j = 0; j < V; ++j) o.v[j] = dequant_one<T>(((uint32_t)p.v[j] >> P::shift(f)) & P::MASK, z, s);
    } else {
      long long c = e % gdiv;  // V consecutive columns (V | C)
      Vec<T, V> s = *reinterpret_cast<const Vec<T, V>*>(scale + c);
      Vec<T, V> z = *reinterpret_cast<const Vec<T, V>*>(zero + c);
#pragma unroll
      for (int j = 0; j < V; ++j) o.v[j] = dequant_one<T>(((uint32_t)p.v[j] >> P::shift(f)) & P::MASK, z.v[j], s.v[j]);
    }
    *reinterpret_cast<Vec<T, V>*>(out + e) = o;
  }
}

// ---------------------------------------------------------------------------------------
// host dispatch
// ---------------------------------------------------------------------------------------
static inline unsigned grid_for(long long n, int V) { return (unsigned)cdiv(cdiv(n, V), 256); }

template <int NBITS, typename TIn>
static int launch_pack(const void* in, void* out, long long n, long long n_in, cudaStream_t st) {
  using PT = typename Pk<NBITS>::T;
  bool vec = (n % 4 == 0) && (n_in % 4 == 0) && aligned(in, 4 * sizeof(TIn) >= 16 ? 16 : 4 * sizeof(TIn)) && aligned(out, 4 * sizeof(PT));
  if (n == 0) return HQQ_OK;
  if (vec)
    pack_kernel<NBITS, TIn, 4><<<grid_for(n, 4), 256, 0, st>>>((const TIn*)in, (PT*)out, n, n_in);
  else
    pack_kernel<NBITS, TIn, 1><<<grid_for(n, 1), 256, 0, st>>>((const TIn*)in, (PT*)out, n, n_in);
  HQQ_LAUNCH_CHECK("hqq_b200_pack");
  return HQQ_OK;
}

template <int NBITS>
static int pack_dtype(const void* in, int in_dtype, void* out, long long n, long long n_in, cudaStream_t st) {
  switch (in_dtype) {
    case HQQ_F32: return launch_pack<NBITS, float>(in, out, n, n_in, st);
    case HQQ_F16: return launch_pack<NBITS, __half>(in, out, n, n_in, st);
    case HQQ_BF16: return launch_pack<NBITS, __nv_bfloat16>(in, out, n, n_in, st);
    case HQQ_U8: return launch_pack<NBITS, uint8_t>(in, out, n, n_in, st);
    case HQQ_I32: return launch_pack<NBITS, int32_t>(in, out, n, n_in, st);
    case HQQ_I64: return launch_pack<NBITS, int64_t>(in, out, n, n_in, st);
  }
  set_error("hqq_b200_pack: unsupported input dtype %d", in_dtype);
  return HQQ_E_INVALID;
}

template <int NBITS, typename TOut>
static int launch_unpack(const void* in, void* out, long long n, cudaStream_t st) {
  using PT = typename Pk<NBITS>::T;
  if (n == 0) return HQQ_OK;
  bool vec = (n % 8 == 0) && aligned(in, 8 * sizeof(PT) >= 16 ? 16 : 8 * sizeof(PT)) && aligned(out, 8 * sizeof(TOut) >= 16 ? 16 : 8 * sizeof(TOut));
  if (vec)
    unpack_kernel<NBITS, TOut, 8><<<grid_for(n, 8), 256, 0, st>>>((const PT*)in, (TOut*)out, n);
  else
    unpack_kernel<NBITS, TOut, 1><<<grid_for(n, 1), 256, 0, st>>>((const PT*)in, (TOut*)out, n);
  HQQ_LAUNCH_CHECK("hqq_b200_unpack");
  return HQQ_OK;
}

template <int NBITS>
static int unpack_dtype(const void* in, void* out, int out_dtype, long long n, cudaStream_t st) {
  switch (out_dtype) {
    case HQQ_F32: return launch_unpack<NBITS, float>(in, out, n, st);
    case HQQ_F16: return launch_unpack<NBITS, __half>(in, out, n, st);
    case HQQ_BF16: return launch_unpack<NBITS, __nv_bfloat16>(in, out, n, st);
    case HQQ_U8: return launch_unpack<NBITS, uint8_t>(in, out, n, st);
    case HQQ_I32: return launch_unpack<NBITS, int32_t>(in, out, n, st);
    case HQQ_I64: return launch_unpack<NBITS, int64_t>(in, out, n, st);
  }
  set_error("hqq_b200_unpack: unsupported output dtype %d", out_dtype);
  return HQQ_E_INVALID;
}

template <int NBITS, typename T>
static int launch_dequant(const void* Wq, const void* scale, const void* zero, void* out, long long n, long long total,
                          int gs, long long C, int axis, cudaStream_t st) {
  using PT = typename Pk<NBITS>::T;
  if (total == 0) return HQQ_OK;
  const size_t a_in = 8 * sizeof(PT) >= 16 ? 16 : 8 * sizeof(PT);
  bool vec = (n % 8 == 0) && (total % 8 == 0) && aligned(Wq, a_in) && aligned(out, 16);
  if (axis == 1) {
    vec = vec && (gs % 8 == 0);
    if (vec)
      dequant_kernel<NBITS, T, 8, 1><<<grid_for(n, 8), 256, 0, st>>>((const PT*)Wq, (const T*)scale, (const T*)zero, (T*)out, n, total, gs);
    else
      dequant_kernel<NBITS, T, 1, 1><<<grid_for(n, 1), 256, 0, st>>>((const PT*)Wq, (const T*)scale, (const T*)zero, (T*)out, n, total, gs);
  } else {
    vec = vec && (C % 8 == 0) && aligned(scale, 16) && aligned(zero, 16);
    if (vec)
      dequant_kernel<NBITS, T, 8, 0><<<grid_for(n, 8), 256, 0, st>>>((const PT*)Wq, (const T*)scale, (const T*)zero, (T*)out, n, total, C);
    else
      dequant_kernel<NBITS, T, 1, 0><<<grid_for(n, 1), 256, 0, st>>>((const PT*)Wq, (const T*)scale, (const T*)zero, (T*)out, n, total, C);
  }
  HQQ_LAUNCH_CHECK("hqq_b200_dequantize");
  return HQQ_OK;
}

template <int NBITS>
static int dequant_dtype(const void* Wq, const void* scale, const void* zero, void* out, long long n, long long total, int gs,
                         long long C, int axis, int dtype, cudaStream_t st) {
  switch (dtype) {
    case HQQ_F32: return launch_dequant<NBITS, float>(Wq, scale, zero, out, n, total, gs, C, axis, st);
    case HQQ_F16: return launch_dequant<NBITS, __half>(Wq, scale, zero, out, n, total, gs, C, axis, st);
    case HQQ_BF16: return launch_dequant<NBITS, __nv_bfloat16>(Wq, scale, zero, out, n, total, gs, C, axis, st);
  }
  set_error("hqq_b200_dequantize: unsupported dtype %d (need f32/f16/bf16)", dtype);
  return HQQ_E_INVALID;
}

}  // namespace hqq

using namespace hqq;

#define HQQ_NBITS_SWITCH(nbits, CALL)                      \
  switch (nbits) {                                         \
    case 8: return CALL(8);                                \
    case 4: return CALL(4);                                \
    case 3: return CALL(3);                                \
    case 2: return CALL(2);                                \
    case 1: return CALL(1);                                \
  }

extern "C" int hqq_b200_pack(int nbits, const void* in, int in_dtype, void* out, int64_t rows, int64_t cols, void* stream) {
  HQQ_REQUIRE(valid_nbits(nbits), HQQ_E_INVALID, "hqq_b200_pack: nbits=%d not supported", nbits);
  HQQ_REQUIRE(rows >= 0 && cols >= 0, HQQ_E_INVALID, "hqq_b200_pack: negative shape");
  HQQ_REQUIRE((in && out) || rows * cols == 0, HQQ_E_INVALID, "hqq_b200_pack: null pointer");
  const int F = fields_of(nbits);
  // the reference slices W_q[:step] | W_q[step:] and fails on a ragged split (bitpack.py:26-28)
  HQQ_REQUIRE(nbits == 3 || rows % F == 0, HQQ_E_INVALID,
              "hqq_b200_pack: %lld rows is not a multiple of %d (%d-bit packs %d rows per byte)", (long long)rows, F, nbits, F);
  const long long prow = (nbits == 3) ? cdiv(rows, 10) : rows / F;
  const long long n = prow * cols, n_in = rows * cols;
  cudaStream_t st = (cudaStream_t)stream;
#define CALL(B) pack_dtype<B>(in, in_dtype, out, n, n_in, st)
  HQQ_NBITS_SWITCH(nbits, CALL)
#undef CALL
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_unpack(int nbits, const void* in, void* out, int out_dtype, int64_t packed_rows, int64_t cols, void* stream) {
  HQQ_REQUIRE(valid_nbits(nbits), HQQ_E_INVALID, "hqq_b200_unpack: nbits=%d not supported", nbits);
  HQQ_REQUIRE(packed_rows >= 0 && cols >= 0, HQQ_E_INVALID, "hqq_b200_unpack: negative shape");
  HQQ_REQUIRE((in && out) || packed_rows * cols == 0, HQQ_E_INVALID, "hqq_b200_unpack: null pointer");
  const long long n = packed_rows * cols;
  cudaStream_t st = (cudaStream_t)stream;
#define CALL(B) unpack_dtype<B>(in, out, out_dtype, n, st)
  HQQ_NBITS_SWITCH(nbits, CALL)
#undef CALL
  return HQQ_E_INVALID;
}

extern "C" int hqq_b200_dequantize(const void* W_q, const void* scale, const void* zero, void* out, int64_t N, int64_t K,
                                   int group_size, int nbits, int axis, int dtype, void* stream) {
  HQQ_REQUIRE(valid_nbits(nbits), HQQ_E_INVALID, "hqq_b200_dequantize: nbits=%d not supported", nbits);
  HQQ_REQUIRE(axis == 0 || axis == 1, HQQ_E_INVALID, "axis should be either 0 or 1");
  HQQ_REQUIRE(N >= 0 && K >= 0 && group_size > 0, HQQ_E_INVALID, "hqq_b200_dequantize: bad shape N=%lld K=%lld gs=%d", (long long)N, (long long)K, group_size);
  const long long total = N * K;
  HQQ_REQUIRE(total % group_size == 0, HQQ_E_INVALID, "group_size should be divisble by the total tensor dimensions. shape: [%lld, %lld], group_size: %d",
              (long long)N, (long long)K, group_size);
  HQQ_REQUIRE((W_q && scale && zero && out) || total == 0, HQQ_E_INVALID, "hqq_b200_dequantize: null pointer");
  const long long R = (axis == 1) ? total / group_size : group_size;  // rows of the grouped matrix
  const long long C = total / R;
  const int F = fields_of(nbits);
  HQQ_REQUIRE(nbits == 3 || R % F == 0, HQQ_E_INVALID, "hqq_b200_dequantize: %lld grouped rows not a multiple of %d", R, F);
  const long long prow = (nbits == 3) ? cdiv(R, 10) : R / F;
  const long long n = prow * C;
  cudaStream_t st = (cudaStream_t)stream;
#define CALL(B) dequant_dtype<B>(W_q, scale, zero, out, n, total, group_size, C, axis, dtype, st)
  HQQ_NBITS_SWITCH(nbits, CALL)
#undef CALL
  return HQQ_E_INVALID;
}
